"""Synthetic cameras and scenes for tests and bench.py (SURVEY.md section 8d, BASELINE.md section 4).

Camera conventions restate the reference so that the same tensors can be fed to both rasterizers:
  getProjectionMatrix   frosting_utils/graphics_utils.py:65-85
  getWorld2View         frosting_utils/graphics_utils.py:38-50
  GSCamera matrices     frosting_scene/cameras.py:203-212 (world_view_transform = W2C^T,
                        full_proj_transform = world_view_transform @ P^T, camera_center = inv(W2C^T)[3,:3])
Frosting's mesh-bound parameterisation restates frosting_scene/frosting_model.py:
  prism cells           :676,705,709-710 (shell_cells_verts: inner v0..v2, outer v0..v2)
  points                :713-726 (softmax of 6 barycentric logits x cell vertices)
  activations           :729-734,765,798
  cell assignment       :476-495, barycentric init :503-509
Everything is generated on the CPU with a seeded torch.Generator (bit-reproducible across boxes) and
moved to the requested device.
"""
import math
from types import SimpleNamespace

import torch

from .rasterizer import GaussianRasterizationSettings

ZNEAR, ZFAR = 0.01, 100.0


def get_projection_matrix(znear, zfar, fovX, fovY):
    tan_y, tan_x = math.tan(fovY / 2), math.tan(fovX / 2)
    top, right = tan_y * znear, tan_x * znear
    bottom, left = -top, -right
    P = torch.zeros(4, 4)
    P[0, 0] = 2.0 * znear / (right - left)
    P[1, 1] = 2.0 * znear / (top - bottom)
    P[0, 2] = (right + left) / (right - left)
    P[1, 2] = (top + bottom) / (top - bottom)
    P[3, 2] = 1.0
    P[2, 2] = zfar / (zfar - znear)
    P[2, 3] = -(zfar * znear) / (zfar - znear)
    return P


def make_camera(W, H, w2c=None, fovx_deg=60.0, device="cpu"):
    """GSCamera-like namespace.  w2c: 4x4 world-to-camera (COLMAP axes: x right, y down, z forward)."""
    if w2c is None:
        w2c = torch.eye(4)
    w2c = w2c.float()
    tanfovx = math.tan(math.radians(fovx_deg) / 2)
    tanfovy = tanfovx * H / W
    fovx, fovy = 2 * math.atan(tanfovx), 2 * math.atan(tanfovy)
    world_view = w2c.t().contiguous()
    proj = get_projection_matrix(ZNEAR, ZFAR, fovx, fovy).t().contiguous()
    full = world_view @ proj
    campos = torch.linalg.inv(world_view)[3, :3].contiguous()
    return SimpleNamespace(
        image_width=W, image_height=H, tanfovx=tanfovx, tanfovy=tanfovy, FoVx=fovx, FoVy=fovy,
        world_view_transform=world_view.to(device), projection_matrix=proj.to(device),
        full_proj_transform=full.to(device), camera_center=campos.to(device), w2c=w2c)


def look_at_w2c(eye, target, up=(0.0, -1.0, 0.0)):
    """World-to-camera for a camera at `eye` looking at `target` (z forward, y down)."""
    eye = torch.tensor(eye, dtype=torch.float64)
    target = torch.tensor(target, dtype=torch.float64)
    upv = torch.tensor(up, dtype=torch.float64)
    z = target - eye
    z = z / z.norm()
    x = torch.linalg.cross(-upv, z)     # right
    if x.norm() < 1e-8:
        x = torch.tensor([1.0, 0.0, 0.0], dtype=torch.float64)
    x = x / x.norm()
    y = torch.linalg.cross(z, x)        # down
    R = torch.stack([x, y, z])          # rows: camera axes in world
    w2c = torch.eye(4, dtype=torch.float64)
    w2c[:3, :3] = R
    w2c[:3, 3] = -R @ eye
    return w2c.float()


def ring_cameras(n, W, H, centre=(0.0, 0.0, 6.0), radius=6.0, device="cpu"):
    cams = []
    for i in range(n):
        a = 2 * math.pi * i / n
        eye = (centre[0] + radius * math.sin(a), centre[1], centre[2] - radius * math.cos(a))
        cams.append(make_camera(W, H, look_at_w2c(eye, centre), device=device))
    return cams


def settings_for(cam, sh_degree, bg=None, device=None, scale_modifier=1.0, debug=False):
    device = device or cam.world_view_transform.device
    if bg is None:
        bg = torch.zeros(3)
    return GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width),
        tanfovx=cam.tanfovx, tanfovy=cam.tanfovy, bg=bg.float().to(device), scale_modifier=scale_modifier,
        viewmatrix=cam.world_view_transform.to(device), projmatrix=cam.full_proj_transform.to(device),
        sh_degree=sh_degree, campos=cam.camera_center.to(device), prefiltered=False, debug=debug)


def random_gaussians(P, cam, seed, device="cpu", sh_coeffs=16, large_frac=0.005, near_frac=0.02):
    """Free Gaussians in the frustum of `cam` (identity W2C assumed): SURVEY.md 8d recipe."""
    g = torch.Generator().manual_seed(seed)
    W = cam.image_width
    fx = W / (2 * cam.tanfovx)
    z = torch.rand(P, generator=g) * 8 + 2
    n_near = int(P * near_frac)
    if n_near:
        z[:n_near] = torch.rand(n_near, generator=g) * 1.2 - 1.0
    x = (torch.rand(P, generator=g) * 2 - 1) * 1.1 * z.abs() * cam.tanfovx
    y = (torch.rand(P, generator=g) * 2 - 1) * 1.1 * z.abs() * cam.tanfovy
    means = torch.stack([x, y, z], 1)
    # move into world space if the camera is not at the origin
    c2w = torch.linalg.inv(cam.w2c.double())
    means = (torch.cat([means.double(), torch.ones(P, 1, dtype=torch.float64)], 1) @ c2w.t())[:, :3].float()
    z_med = 6.0
    s0 = 1.5 * z_med / fx
    scales = s0 * torch.exp(0.5 * torch.randn(P, 3, generator=g))
    n_large = int(P * large_frac)
    if n_large:
        idx = torch.randperm(P, generator=g)[:n_large]
        scales[idx] *= 20
    q = torch.randn(P, 4, generator=g)
    rotations = q / q.norm(dim=1, keepdim=True)
    opacities = torch.rand(P, 1, generator=g) * 0.9 + 0.05
    shs = torch.randn(P, sh_coeffs, 3, generator=g) * 0.1
    shs[:, 0] = torch.randn(P, 3, generator=g)
    out = dict(means3D=means, scales=scales, rotations=rotations, opacities=opacities, shs=shs)
    return {k: v.contiguous().to(device) for k, v in out.items()}


def uv_sphere(n_lat, n_lon, radius=3.0, centre=(0.0, 0.0, 6.0)):
    """Closed UV sphere: 2 + (n_lat-1)*n_lon vertices, 2*n_lon*(n_lat-1) faces."""
    th = torch.linspace(0, math.pi, n_lat + 1)[1:-1]                    # polar, without the poles
    ph = torch.arange(n_lon) * (2 * math.pi / n_lon)
    st, ct = torch.sin(th)[:, None], torch.cos(th)[:, None]
    ring = torch.stack([st * torch.cos(ph)[None], ct.expand(-1, n_lon), st * torch.sin(ph)[None]], -1)  # [n_lat-1,n_lon,3]
    normals = torch.cat([torch.tensor([[0.0, 1.0, 0.0]]), ring.reshape(-1, 3), torch.tensor([[0.0, -1.0, 0.0]])])
    verts = normals * radius + torch.tensor(centre)
    nr = n_lat - 1

    def vid(i, j):
        return 1 + i * n_lon + (j % n_lon)
    j = torch.arange(n_lon)
    faces = []
    top = torch.stack([torch.zeros(n_lon, dtype=torch.long), 1 + (j + 1) % n_lon, 1 + j], 1)
    faces.append(top)
    for i in range(nr - 1):
        a, b = vid(i, j), vid(i, j + 1)
        c, d = vid(i + 1, j), vid(i + 1, j + 1)
        faces.append(torch.stack([a, b, d], 1))
        faces.append(torch.stack([a, d, c], 1))
    last = 1 + nr * n_lon
    bot = torch.stack([torch.full((n_lon,), last, dtype=torch.long), vid(nr - 1, j), vid(nr - 1, j + 1)], 1)
    faces.append(bot)
    return verts.float().contiguous(), torch.cat(faces).int().contiguous(), normals.float().contiguous()


def frosting_layer(P, cam, seed, n_faces_target=1_000_000, device="cpu", sh_coeffs=16, thickness=0.02,
                   n_min_per_cell=1, view_distance=7.5, n_background=0, behind_frac=0.25):
    """Frosting-layer scene: Gaussians bound to prism cells over a UV-sphere base mesh.

    Returns the *learnable parameters* (bary logits, opacity logits, log scales, raw quaternions, SH dc/rest)
    plus the mesh and `_point_cell_indices`; `frosting_attributes()` turns them into rasterizer inputs.
    `n_background` > 0 adds Frosting's background Gaussians (the six `bg_*` keys, frosting_model.py:564-591): free
    Gaussians outside the base mesh's bounding box, on a thick spherical shell around the scene, `behind_frac` of them
    behind the ring cameras (radius 6 around the sphere's centre); `frosting_background_attributes()` maps them.  They
    come from a generator of their own, so the mesh-bound tensors are the same with or without them.
    """
    g = torch.Generator().manual_seed(seed)
    n_lon = max(8, int(round(math.sqrt(n_faces_target / 2.0) * math.sqrt(2.0))))
    n_lat = max(4, n_faces_target // (2 * n_lon) + 1)
    verts, faces, normals = uv_sphere(n_lat, n_lon)
    F = faces.shape[0]
    inner = verts - thickness * normals
    outer = verts + thickness * normals
    fl = faces.long()
    # cell volumes ~ base triangle area (constant thickness)
    tri = verts[fl]
    area = torch.linalg.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]).norm(dim=1) * 0.5
    base = torch.arange(F).repeat(n_min_per_cell)[:P]
    n_extra = P - base.shape[0]
    if n_extra > 0:
        extra = torch.multinomial(area / area.sum(), n_extra, replacement=True, generator=g)
        cells = torch.cat([base, extra])
    else:
        cells = base
    # barycentric init: spacings of sorted uniforms (uniform on the simplex), stored as logits
    u = torch.sort(torch.rand(P, 5, generator=g), dim=1).values
    u = torch.cat([torch.zeros(P, 1), u, torch.ones(P, 1)], 1)
    bary = (u[:, 1:] - u[:, :-1]).clamp_min(1e-6)
    bary_logits = bary.log()
    fx = cam.image_width / (2 * cam.tanfovx)
    s0 = 1.5 * view_distance / fx     # median screen-space sigma ~1.5 px at the viewing distance
    log_scales = math.log(s0) + 0.5 * torch.randn(P, 3, generator=g)
    log_scales[:, 2] -= 1.0    # flatter along one axis, like surface-aligned splats
    quats = torch.randn(P, 4, generator=g)
    opacity_logits = torch.logit(torch.rand(P, generator=g) * 0.9 + 0.05)
    sh_dc = torch.randn(P, 1, 3, generator=g)
    sh_rest = torch.randn(P, sh_coeffs - 1, 3, generator=g) * 0.1
    params = dict(bary_logits=bary_logits, opacity_logits=opacity_logits, log_scales=log_scales, quats=quats,
                  sh_dc=sh_dc, sh_rest=sh_rest)
    mesh = dict(verts=verts, faces=faces, inner=inner, outer=outer, cells=cells)
    if n_background > 0:
        params.update(_background_gaussians(n_background, verts, fx, seed, sh_coeffs, behind_frac))
    params = {k: v.contiguous().to(device) for k, v in params.items()}
    mesh = {k: v.contiguous().to(device) for k, v in mesh.items()}
    return params, mesh


def _background_gaussians(n, verts, fx, seed, sh_coeffs, behind_frac):
    g = torch.Generator().manual_seed(seed + 0x6267)           # separate stream: the mesh-bound draws are unchanged
    lo, hi = verts.min(0).values, verts.max(0).values
    centre, half = (lo + hi) / 2, (hi - lo) / 2
    n_behind = int(n * behind_frac)
    d = torch.randn(n, 3, generator=g)
    d[:, 1] *= 0.5                                                # flatter towards the ring's plane
    d = d / d.norm(dim=1, keepdim=True)
    # distance along d at which the ray leaves the bounding box: beyond it a point is background (frosting_model.py:567-574)
    t_box = (half[None] / d.abs().clamp_min(1e-6)).min(1).values * 1.05
    # a thick shell: in front of the ring cameras (between the box and radius 5.5, the ring being at 6) or behind them
    u = torch.rand(n, generator=g)
    r = t_box + u * (5.5 - t_box).clamp_min(0.0)
    r[:n_behind] = torch.maximum(t_box[:n_behind], 7.0 + u[:n_behind] * 8.0)
    points = centre + r[:, None] * d
    s0 = 1.5 * r[:, None] / fx
    log_scales = torch.log(s0) + 0.5 * torch.randn(n, 3, generator=g)
    return dict(bg_points=points.float(), bg_opacity_logits=torch.logit(torch.rand(n, generator=g) * 0.9 + 0.05),
                bg_log_scales=log_scales.float(), bg_quats=torch.randn(n, 4, generator=g),
                bg_sh_dc=torch.randn(n, 1, 3, generator=g), bg_sh_rest=torch.randn(n, sh_coeffs - 1, 3, generator=g) * 0.1)


def frosting_attributes(params, mesh):
    """Learnable parameters -> rasterizer inputs, as Frosting's properties do (frosting_model.py:713-799)."""
    faces = mesh["faces"].long()
    shell = torch.stack([mesh["inner"], mesh["outer"]], 1)            # n_verts, 2, 3
    cells_verts = shell[faces].transpose(-2, -3)                      # n_faces, 2, 3, 3
    bary = torch.softmax(params["bary_logits"], dim=-1)
    points = (bary[..., None] * cells_verts[mesh["cells"]].reshape(-1, 6, 3)).sum(dim=-2)
    return dict(
        means3D=points,
        opacities=torch.sigmoid(params["opacity_logits"].view(-1, 1)),
        scales=torch.exp(params["log_scales"]),
        rotations=torch.nn.functional.normalize(params["quats"], dim=-1),
        shs=torch.cat([params["sh_dc"], params["sh_rest"]], dim=1),
    )


def frosting_background_attributes(params):
    """Background parameters -> rasterizer inputs, as Frosting's bg_* properties do (frosting_model.py:801-876): points
    as they are, sigmoid, cat(dc, rest), exp, normalize."""
    return dict(
        means3D=params["bg_points"],
        opacities=torch.sigmoid(params["bg_opacity_logits"].view(-1, 1)),
        scales=torch.exp(params["bg_log_scales"]),
        rotations=torch.nn.functional.normalize(params["bg_quats"], dim=-1),
        shs=torch.cat([params["bg_sh_dc"], params["bg_sh_rest"]], dim=1),
    )
