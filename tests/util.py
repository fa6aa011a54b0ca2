"""Shared helpers for the parity tests."""
import torch

from frosting_b200 import scenes


def scene(P, W, H, seed, sh_degree, device, bg=0.0):
    cam = scenes.make_camera(W, H, device=device)
    g = scenes.random_gaussians(P, cam, seed, device=device)
    rs = scenes.settings_for(cam, sh_degree, bg=torch.full((3,), float(bg)), device=device)
    return cam, g, rs


def regime_gaussians(P, cam, seed, sh_coeffs=16, n_behind=0, device="cpu"):
    """Free Gaussians for the per-Gaussian backward's edge cases, shuffled so that warps mix them: centres outside the
    1.3 tanfov guard band in x only, y only and both (large enough to reach into the image), view depths in (0.21, 0.4]
    (within 2x of the 0.2 near plane), needles whose projected variances stay below the 0.3 dilation, raw quaternions of
    norm 0.3 .. 3 (half of them outside [0.5, 2]; scales shrunk by 1 / |q|^2 to keep the splat's size), and rows with one
    or two colour channels driven below zero.  `n_behind` rows behind the camera form one contiguous run in the middle.
    Any camera: the scene is built in its view space and moved to the world."""
    g = torch.Generator().manual_seed(seed)
    U = lambda n, lo, hi: lo + (hi - lo) * torch.rand(n, generator=g)
    sign = lambda n: torch.where(torch.rand(n, generator=g) < 0.5, -1.0, 1.0)
    fx = cam.image_width / (2 * cam.tanfovx)
    tx, ty = cam.tanfovx, cam.tanfovy
    z = U(P, 2.0, 10.0)
    x, y = U(P, -1.0, 1.0) * z * tx, U(P, -1.0, 1.0) * z * ty
    scales = (1.5 * z / fx)[:, None] * torch.exp(0.5 * torch.randn(P, 3, generator=g))
    kind = torch.randint(0, 8, (P,), generator=g)     # 1 guard x, 2 guard y, 3 guard x+y, 4 near, 5 needle, else plain
    for k, gx, gy in ((1, True, False), (2, False, True), (3, True, True)):
        r = kind == k
        n = int(r.sum())
        z[r] = U(n, 3.0, 8.0)
        x[r] = (sign(n) * U(n, 1.33, 1.5) * tx if gx else U(n, -0.8, 0.8) * tx) * z[r]
        y[r] = (sign(n) * U(n, 1.33, 1.6) * ty if gy else U(n, -0.8, 0.8) * ty) * z[r]
        scales[r] = (U(n, 0.06, 0.12) * z[r])[:, None] * torch.exp(0.2 * torch.randn(n, 3, generator=g))
    r = kind == 4
    n = int(r.sum())
    z[r] = U(n, 0.21, 0.4)
    x[r], y[r] = U(n, -0.9, 0.9) * z[r] * tx, U(n, -0.9, 0.9) * z[r] * ty
    scales[r] = (1.5 * z[r] / fx)[:, None] * torch.exp(0.5 * torch.randn(n, 3, generator=g))
    r = kind == 5
    n = int(r.sum())
    needle = torch.full((n, 3), 1e-3) * (z[r] / fx)[:, None]
    needle[torch.arange(n), torch.randint(0, 3, (n,), generator=g)] = U(n, 0.1, 0.4) * z[r] / fx
    scales[r] = needle
    q = torch.randn(P, 4, generator=g)
    q = q / q.norm(dim=1, keepdim=True)
    lam = torch.where(torch.rand(P, generator=g) < 0.5, U(P, 0.5, 2.0),
                      torch.where(torch.rand(P, generator=g) < 0.5, U(P, 0.3, 0.5), U(P, 2.0, 3.0)))
    rotations = q * lam[:, None]
    scales = scales / lam.clamp_min(1.0)[:, None] ** 2
    opacities = U(P, 0.05, 0.6)[:, None]
    shs = torch.randn(P, sh_coeffs, 3, generator=g) * 0.1
    shs[:, 0] = torch.rand(P, 3, generator=g) + 0.2
    dark = torch.rand(P, generator=g) < 0.25
    chans = torch.rand(P, 3, generator=g) < 0.5
    chans[torch.arange(P), torch.randint(0, 3, (P,), generator=g)] = True       # one channel on, one off: never
    chans[torch.arange(P), torch.randint(0, 3, (P,), generator=g)] = False      # all three, mostly not none
    shs[:, 0] = torch.where(dark[:, None] & chans, torch.full_like(shs[:, 0], -4.0), shs[:, 0])
    if n_behind:
        mid = P // 2
        z[mid:mid + n_behind] = -3.0
    means = torch.stack([x, y, z], 1)
    c2w = torch.linalg.inv(cam.w2c.double())
    means = (torch.cat([means.double(), torch.ones(P, 1, dtype=torch.float64)], 1) @ c2w.t())[:, :3].float()
    out = dict(means3D=means, scales=scales.float(), rotations=rotations.float(), opacities=opacities.float(),
               shs=shs.float())
    return {k: v.contiguous().to(device) for k, v in out.items()}


def rel_err_stats(a, b):
    """Gradient tolerance used throughout: error relative to the tensor's scale, plus the fraction of
    significant elements whose own relative error exceeds 1e-3."""
    a, b = a.double().flatten(), b.double().flatten()
    scale = b.abs().max().clamp_min(1e-30)
    diff = (a - b).abs()
    max_rel_to_scale = (diff.max() / scale).item()
    sig = b.abs() > 1e-4 * scale
    if sig.any():
        el = diff[sig] / b.abs()[sig]
        frac_bad = (el > 1e-3).double().mean().item()
    else:
        frac_bad = 0.0
    return max_rel_to_scale, frac_bad


def blend_regime_gaussians(P, cam, seed, n_deep=0, device="cpu"):
    """Free Gaussians (precomputed colours) for the blend kernels' edge cases, built in the view space of `cam` from
    pixel positions and sizes: an opaque wall of small splats (half of them at opacity > 0.99, i.e. past the 0.99
    clamp) bounded by a slanted sharp edge, so that sub-tiles on the edge hold saturated and never-saturating pixels
    side by side; a cloud of anisotropic splats of opacity 0.02 .. 0.7 over the middle; ~0.2 % wide faint splats whose
    opacity is within 2e-3 above 1/255, so that their alpha crosses 1/255 over whole pixel disks; and an empty strip at
    the right edge (empty sub-tiles).  `n_deep` extra faint splats centred in one tile push its list past 8192
    entries (the global-memory sort class)."""
    g = torch.Generator().manual_seed(seed)
    U = lambda n, lo, hi: lo + (hi - lo) * torch.rand(n, generator=g)
    W, H = cam.image_width, cam.image_height
    fx = W / (2 * cam.tanfovx)
    fy = H / (2 * cam.tanfovy)
    n_faint = max(P // 500, 20)
    n_wall = (P - n_faint) * 2 // 5
    n_cloud = P - n_faint - n_wall
    u, v, z, sig, op = [], [], [], [], []
    # the wall: left of the line u = 0.3 W + 0.25 v
    vw = U(n_wall, 0, H)
    u.append(U(n_wall, 0, 1) * (0.3 * W + 0.25 * vw)); v.append(vw); z.append(U(n_wall, 3.0, 4.0))
    sig.append(U(n_wall, 0.8, 2.0))
    op.append(torch.where(torch.rand(n_wall, generator=g) < 0.5, U(n_wall, 0.993, 1.0), U(n_wall, 0.5, 0.95)))
    # the cloud, behind the wall's depth range in part
    u.append(U(n_cloud, 0.2 * W, W - 80)); v.append(U(n_cloud, 0, H)); z.append(U(n_cloud, 2.0, 10.0))
    sig.append(U(n_cloud, 1.0, 8.0)); op.append(U(n_cloud, 0.02, 0.7))
    # faint and wide: alpha = op G crosses 1/255 where G = 1/255 / op, within ~0.06 sigma of the centre
    u.append(U(n_faint, 0.25 * W, W - 100)); v.append(U(n_faint, 10, H - 10)); z.append(U(n_faint, 2.0, 10.0))
    sig.append(U(n_faint, 30.0, 60.0)); op.append((1.0 / 255.0) * (1 + U(n_faint, 1e-4, 2e-3)))
    if n_deep:
        tx = (W // 32) * 16
        u.append(U(n_deep, tx, tx + 16)); v.append(U(n_deep, 16, 32)); z.append(U(n_deep, 2.0, 10.0))
        sig.append(U(n_deep, 0.5, 1.5)); op.append(U(n_deep, 0.01, 0.05))
    u, v, z, sig, op = (torch.cat(a) for a in (u, v, z, sig, op))
    N = u.shape[0]
    x = (u - 0.5 * (W - 1)) / fx * z
    y = (v - 0.5 * (H - 1)) / fy * z
    scales = (sig * z / fx)[:, None] * torch.exp(0.25 * torch.randn(N, 3, generator=g))
    q = torch.randn(N, 4, generator=g)
    rotations = q / q.norm(dim=1, keepdim=True)
    colors = torch.rand(N, 3, generator=g)
    perm = torch.randperm(N, generator=g)
    means = torch.stack([x, y, z], 1)
    c2w = torch.linalg.inv(cam.w2c.double())
    means = (torch.cat([means.double(), torch.ones(N, 1, dtype=torch.float64)], 1) @ c2w.t())[:, :3].float()
    out = dict(means3D=means, scales=scales.float(), rotations=rotations.float(), opacities=op.float()[:, None],
               colors=colors.float())
    return {k: v[perm].contiguous().to(device) for k, v in out.items()}
