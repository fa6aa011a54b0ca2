"""SuGaR's depth-normal consistency on the GPU against float64, bit reproducibility, no host read-back, and the fused
route (features as extra channels of the colour frame) against the reference's two-pass route.

Three results from the same float32 inputs: ours, R32 (the torch restatement in float32 on the GPU: the reference's own
arithmetic) and R64 (the restatement in float64).  The bar, as for the SDF regulariser: ours may be at most twice as
far from R64 as R32 is, plus 1e-6 of R64's size --
  - a loss: |ours - R64| <= 2 |R32 - R64| + 1e-6 |R64|;
  - each tensor, on the largest error and on the 99.9th percentile of the errors: err(ours) <= 2 err(R32) + 1e-6 max|R64|.
"""
import os

import numpy as np
import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import scenes, sugar_dn
from tests import refgold

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_sugar_dn.npz")
LEAVES = ("points", "scaling", "quaternions")


def _quantile(x, q):
    x = x.reshape(-1)
    return float(x.kthvalue(max(1, int(round(q * x.numel())))).values) if x.numel() else 0.0


def assert_bar(ours, r32, r64, label):
    ours, r32, r64 = ours.double(), r32.double(), r64.double()
    if r64.dim() == 0:
        assert float((ours - r64).abs()) <= 2 * float((r32 - r64).abs()) + 1e-6 * float(r64.abs()), \
            (label, float(ours), float(r32), float(r64))
        return
    err_o, err_r = (ours - r64).abs(), (r32 - r64).abs()
    floor = 1e-6 * float(r64.abs().max()) if r64.numel() else 0.0
    for stat in (lambda e: float(e.max()), lambda e: _quantile(e, 0.999)):
        lhs, rhs = stat(err_o), 2 * stat(err_r) + floor
        assert lhs <= rhs, (label, lhs, stat(err_r), floor)


def camera(W, H):
    return scenes.make_camera(W, H, scenes.look_at_w2c((1.0, -0.6, 0.5), (0.0, 0.0, 6.0)), device=DEV)


# ---- features ------------------------------------------------------------------------------------------------------

def check_features(sc, rs, cot, label):
    leaves = {k: sc[k].clone().requires_grad_(True) for k in LEAVES}
    feats = fb.depth_normal_features(*leaves.values(), rs)
    ours = [feats.detach()] + list(torch.autograd.grad(feats, list(leaves.values()), cot))
    refs = {}
    for dtype in (torch.float32, torch.float64):
        ref_leaves = [sc[k].to(dtype).requires_grad_(True) for k in LEAVES]
        f = sugar_dn.torch_reference_features(*ref_leaves, rs.viewmatrix.to(dtype), rs.campos.to(dtype))
        g = torch.autograd.grad(f, ref_leaves, cot.to(dtype), allow_unused=True)
        refs[dtype] = [f.detach()] + [torch.zeros_like(l) if x is None else x for x, l in zip(g, ref_leaves)]
    for name, o, a, b in zip(("features",) + LEAVES, ours, refs[torch.float32], refs[torch.float64]):
        assert_bar(o, a, b, (label, name))
    assert not ours[2].any()                         # dL/dscaling: exactly zero, as a tensor


@pytest.mark.parametrize("P", [1, 17, 2000, 200_000, 1_000_000])
def test_features_against_float64(P):
    sc = {k: v.to(DEV) for k, v in scenes.sugar_scene(P, P + 3, K=1).items() if k != "knn_idx"}
    rs = scenes.settings_for(camera(64, 48), 0, device=DEV)
    cot = torch.randn(P, 3, generator=torch.Generator().manual_seed(P)).to(DEV)
    check_features(sc, rs, cot, P)


def test_features_golden_edge_cases():
    """Tied scales, a normal perpendicular to the view ray (sign 0) and a raw quaternion, under the golden's camera."""
    z = np.load(GOLD)
    w2c = torch.from_numpy(z["cam_perm/w2c"])
    rs = scenes.settings_for(scenes.make_camera(64, 40, w2c, device=DEV), 0, device=DEV)
    sc = {k: torch.from_numpy(z[k]).to(DEV) for k in LEAVES}
    check_features(sc, rs, torch.from_numpy(z["cot"]).to(DEV), "golden")
    feats = fb.depth_normal_features(*sc.values(), rs)
    assert torch.allclose(feats.cpu().double(), torch.from_numpy(z["f64/features"]), rtol=0, atol=1e-5)
    assert float(feats[6, 1].detach()) == 0.0 and float(feats[6, 2].detach()) == 0.0


# ---- loss ----------------------------------------------------------------------------------------------------------

def check_loss(dn, rs, label, upstream=1.0):
    leaf = dn.clone().requires_grad_(True)
    loss = fb.depth_normal_consistency(leaf, rs)
    (g,) = torch.autograd.grad(loss, [leaf], torch.tensor(upstream, device=DEV))
    for dtype in (torch.float32, torch.float64):
        x = dn.to(dtype).requires_grad_(True)
        ref = sugar_dn.torch_reference_loss(x, rs.viewmatrix.to(dtype), rs.projmatrix.to(dtype))
        (rg,) = torch.autograd.grad(ref, [x], torch.tensor(upstream, device=DEV, dtype=dtype), allow_unused=True)
        rg = torch.zeros_like(x) if rg is None else rg
        if dtype == torch.float32:
            r32 = (ref.detach(), rg)
        else:
            r64 = (ref.detach(), rg)
    assert_bar(loss.detach(), r32[0], r64[0], (label, "loss"))
    assert_bar(g, r32[1], r64[1], (label, "dL/ddn"))
    return loss.detach(), g


def synthetic(H, W, seed):
    """A smooth surface in front of the camera with a background corner (depth 0), a step, and normal channels that
    reach past |xy|^2 = 1 on a tenth of the pixels (never exactly 1)."""
    g = torch.Generator().manual_seed(seed)
    y, x = torch.meshgrid(torch.arange(H, dtype=torch.float64), torch.arange(W, dtype=torch.float64), indexing="ij")
    depth = 5.0 + 0.4 * torch.sin(7.0 * x / W) * torch.cos(5.0 * y / H) + 0.3 * x / W
    depth = torch.where(x > 0.6 * W, depth + 1.0, depth)
    depth = torch.where((y < 0.3 * H) & (x < 0.3 * W), torch.zeros_like(depth), depth)
    nxy = 0.6 * (2 * torch.rand(2, H, W, generator=g, dtype=torch.float64) - 1)
    over = torch.rand(H, W, generator=g, dtype=torch.float64) < 0.1
    nxy[:, over] = torch.tensor([0.9, -0.8], dtype=torch.float64)[:, None]
    return torch.cat([depth[None], nxy]).float().contiguous().to(DEV)


@pytest.mark.parametrize("H,W", [(1080, 1920), (1079, 1917), (33, 47), (17, 17), (3, 40), (40, 3), (4, 4)])
def test_loss_synthetic_against_float64(H, W):
    rs = scenes.settings_for(camera(W, H), 0, device=DEV)
    for upstream in (1.0, -0.05):
        check_loss(synthetic(H, W, H * W), rs, (H, W), upstream)


def render_dn(P, W, H, seed):
    """The fused route's image: sugar_scene's features blended as extra channels of a colour frame, background 0."""
    sc = {k: v.to(DEV) for k, v in scenes.sugar_scene(P, seed, K=1).items() if k != "knn_idx"}
    rs = scenes.settings_for(camera(W, H), 0, device=DEV)
    feats = fb.depth_normal_features(sc["points"], sc["scaling"], sc["quaternions"], rs)
    _, radii, dn = fb.GaussianRasterizer(rs)(
        means3D=sc["points"], means2D=torch.zeros(P, 3, device=DEV), opacities=sc["strengths"],
        colors_precomp=torch.full((P, 3), 0.5, device=DEV), scales=sc["scaling"], rotations=sc["quaternions"],
        extra_features=feats)
    return dn.detach().contiguous(), rs, radii


@pytest.mark.parametrize("P,W,H", [(2000, 96, 160), (200_000, 1920, 1080), (1_000_000, 1917, 1079)])
def test_loss_rendered_against_float64(P, W, H):
    dn, rs, radii = render_dn(P, W, H, 11)
    assert int((radii > 0).sum()) > 0 and bool((dn[0] == 0).any()) and bool((dn[0] > 0).any())
    check_loss(dn, rs, (P, W, H))


def test_loss_golden_edge_images():
    z = np.load(GOLD)
    names = [k[4:-3] for k in z.files if k.startswith("img_") and k.endswith("/dn")]
    assert {"1x1", "2x5", "3x3", "23x37"} <= set(names)
    for name in names:
        dn = torch.from_numpy(z[f"img_{name}/dn"]).to(DEV)
        H, W = dn.shape[1:]
        cam = scenes.make_camera(W, H, device=DEV)
        cam.world_view_transform = torch.from_numpy(z[f"img_{name}/view"]).to(DEV)
        cam.full_proj_transform = torch.from_numpy(z[f"img_{name}/proj"]).to(DEV)
        rs = scenes.settings_for(cam, 0, device=DEV)
        loss, g = check_loss(dn, rs, name)
        if H < 3 or W < 3:
            assert float(loss) == 1.0 and not g.any()


def test_exact_unit_xy_gives_torchs_infinite_gradient():
    """At |xy|^2 == 1 exactly the sqrt's backward divides by zero: +-inf where the rendered normal's partner n_d has a
    z component, NaN where the upstream is 0 (border pixels); torch's values, reproduced."""
    H, W = 20, 24
    dn = synthetic(H, W, 5)
    dn[1, 5:9, 5:9], dn[2, 5:9, 5:9] = 0.6, 0.8                 # 0.36 + 0.64 == 1 in float32
    dn[1, 0, 3], dn[2, 0, 3] = 0.6, 0.8                          # on the border
    assert bool((dn[1] * dn[1] + dn[2] * dn[2] == 1).any())
    rs = scenes.settings_for(camera(W, H), 0, device=DEV)
    leaf = dn.clone().requires_grad_(True)
    (g,) = torch.autograd.grad(fb.depth_normal_consistency(leaf, rs), [leaf])
    x = dn.clone().requires_grad_(True)
    (rg,) = torch.autograd.grad(sugar_dn.torch_reference_loss(x, rs.viewmatrix, rs.projmatrix), [x])
    for c in (1, 2):
        assert torch.equal(torch.isinf(g[c]), torch.isinf(rg[c])) and torch.equal(torch.isnan(g[c]), torch.isnan(rg[c]))
        inf = torch.isinf(rg[c])
        assert bool(inf.any()) and torch.equal(torch.sign(g[c][inf]), torch.sign(rg[c][inf]))
    assert bool(torch.isnan(g[1, 0, 3]))


def test_two_runs_are_bit_identical():
    dn, rs, _ = render_dn(200_000, 1920, 1080, 3)
    sc = {k: v.to(DEV) for k, v in scenes.sugar_scene(50_000, 4, K=1).items() if k != "knn_idx"}
    cot = torch.randn(50_000, 3, generator=torch.Generator().manual_seed(0)).to(DEV)

    def run():
        leaf = dn.clone().requires_grad_(True)
        loss = fb.depth_normal_consistency(leaf, rs)
        (g,) = torch.autograd.grad(loss, [leaf])
        leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
        f = fb.depth_normal_features(*leaves, rs)
        return [loss.detach(), g, f.detach(), *torch.autograd.grad(f, leaves, cot)]

    a, b = run(), run()
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_no_host_read_back_and_no_grad_forward():
    dn, rs, _ = render_dn(2000, 160, 96, 7)
    sc = {k: v.to(DEV) for k, v in scenes.sugar_scene(2000, 7, K=1).items() if k != "knn_idx"}
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    leaf = dn.clone().requires_grad_(True)
    cot = torch.randn(2000, 3, device=DEV)

    def calls():
        f = fb.depth_normal_features(*leaves, rs)
        gf = torch.autograd.grad(f, leaves, cot)
        loss = fb.depth_normal_consistency(leaf, rs)
        gl = torch.autograd.grad(loss, [leaf])
        return f, gf, loss, gl

    calls()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = calls()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    with torch.no_grad():
        loss = fb.depth_normal_consistency(leaf, rs)
        f = fb.depth_normal_features(*leaves, rs)
    assert not loss.requires_grad and loss.grad_fn is None and f.grad_fn is None
    assert torch.equal(loss, out[2].detach()) and torch.equal(f, out[0].detach())


def test_fused_route_matches_the_reference_two_pass_route(cuda_device):
    """The trainer's step: colour frame + L1-DSSIM + 0.05 x consistency.  Fused: features as extra channels of the colour
    frame, then the CUDA loss.  Reference: the compiled reference rasterizer's colour pass, plus a second pass with the
    features as colors_precomp and background 0, plus the float32 torch loss (recorded by tests/refgold.py)."""
    dev = cuda_device
    P, W, H, D = 60_000, 400, 304, 3
    sc = {k: v.to(dev) for k, v in scenes.sugar_scene(P, 21, K=1).items() if k != "knn_idx"}
    cam = camera(W, H)
    rs = scenes.settings_for(cam, D, device=dev)
    gen = torch.Generator().manual_seed(9)
    shs = (0.2 * torch.randn(P, 16, 3, generator=gen)).to(dev)
    gt = torch.rand(3, H, W, generator=gen).to(dev)
    g = dict(means3D=sc["points"], opacities=sc["strengths"], scales=sc["scaling"], rotations=sc["quaternions"],
             shs=shs)

    def compute():
        from oracle import refdgr
        kw = dict(scales=g["scales"], rotations=g["rotations"])
        leaves = {k: v.clone().requires_grad_(True) for k, v in g.items()}
        f3 = sugar_dn.torch_reference_features(leaves["means3D"], g["scales"], leaves["rotations"], rs.viewmatrix,
                                               rs.campos)
        ref1 = refdgr.forward(rs, g["means3D"], g["opacities"], shs=g["shs"], **kw)
        rs2 = rs._replace(bg=torch.zeros(3, device=dev))
        ref2 = refdgr.forward(rs2, g["means3D"], g["opacities"], colors_precomp=f3.detach(), **kw)
        color = ref1["color"].clone().requires_grad_(True)
        dn = ref2["color"].clone().requires_grad_(True)
        loss = fb.l1_dssim_loss(color, gt) + 0.05 * sugar_dn.torch_reference_loss(dn, rs.viewmatrix, rs.projmatrix)
        g_color, g_dn = torch.autograd.grad(loss, [color, dn])
        rb1 = refdgr.backward(rs, ref1, g["means3D"], g_color, shs=g["shs"], **kw)
        rb2 = refdgr.backward(rs2, ref2, g["means3D"], g_dn, colors_precomp=f3.detach(), **kw)
        g_m3, g_rot = torch.autograd.grad(f3, [leaves["means3D"], leaves["rotations"]], rb2["colors"])
        out = {"g_" + k: rb1[k] + rb2[k] for k in ("means3D", "opacities", "scales", "rotations")}
        out["g_means3D"] = out["g_means3D"] + g_m3
        out["g_rotations"] = out["g_rotations"] + g_rot
        return dict(out, loss=float(loss.detach()), radii=ref1["radii"], g_sh=rb1["sh"])
    ref = refgold.case("sugar_dn_fused_route", compute, [g["means3D"], g["opacities"], g["shs"], g["scales"],
                                                         g["rotations"], gt])

    leaves = {k: v.clone().requires_grad_(True) for k, v in g.items()}
    feats = fb.depth_normal_features(leaves["means3D"], leaves["scales"], leaves["rotations"], rs)
    rgb, radii, dn = fb.GaussianRasterizer(rs)(
        means3D=leaves["means3D"], means2D=torch.zeros(P, 3, device=dev, requires_grad=True),
        opacities=leaves["opacities"], shs=leaves["shs"], scales=leaves["scales"], rotations=leaves["rotations"],
        extra_features=feats)
    loss = fb.l1_dssim_loss(rgb, gt) + 0.05 * fb.depth_normal_consistency(dn, rs)
    loss.backward()
    assert ref.equal("radii", radii)
    assert abs(float(loss.detach()) - ref["loss"]) <= 1e-5 * abs(ref["loss"])
    got = dict(means3D=leaves["means3D"].grad, opacities=leaves["opacities"].grad, scales=leaves["scales"].grad,
               rotations=leaves["rotations"].grad, sh=leaves["shs"].grad)
    for k, v in got.items():
        m, frac = ref.close("g_" + k, v)
        assert m <= 1e-3 and frac <= 5e-3, (k, m, frac)
