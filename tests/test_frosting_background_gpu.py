"""Background Gaussians in frosting mode (frosting_model.py:564-591, :801-876): `frosting_render` with the six `bg_*`
parameters against the attribute-kernel route, Frosting's torch chain, the mesh-only frame and torch.optim.Adam."""
import os

import numpy as np
import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import _lib, optim, scenes
from frosting_b200.frosting_render import BG_KEYS, MESH_KEYS
from tests.util import rel_err_stats

pytestmark = pytest.mark.gpu


def _layer(dev, W, H, n_mesh, n_bg, faces, M=16, seed=11, occl=True):
    cam = scenes.make_camera(W, H, device=dev)
    params, mesh = scenes.frosting_layer(n_mesh, cam, seed, n_faces_target=faces, device=dev, view_distance=4.5,
                                         sh_coeffs=M, n_background=n_bg)
    fv = None
    if occl:
        _, fv, _ = fb.rasterize_mesh(mesh["verts"], mesh["faces"], cam.full_proj_transform, H, W, mark_last_on_bg=True)
    return cam, params, mesh, fv


def _leaves(params, mesh):
    p = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    m = dict(mesh)
    m["inner"] = mesh["inner"].clone().requires_grad_(True)
    m["outer"] = mesh["outer"].clone().requires_grad_(True)
    return p, m


@pytest.mark.parametrize("W,H,n_mesh,n_bg,faces,occl,M,D", [
    (320, 200, 50_000, 20_000, 8000, True, 16, 3),
    (200, 120, 3001, 500, 500, False, 16, 3),
    (320, 200, 20_003, 6000, 4000, True, 9, 2),
])
def test_frosting_mode_with_background_equals_the_two_step_route(cuda_device, W, H, n_mesh, n_bg, faces, occl, M, D):
    """n_mesh is not a multiple of 32: one warp of preprocess and of the per-Gaussian backward mixes mesh and background
    rows.  Bit-identical image and radii, gradients equal up to the blend backward's atomic order, exact zeros for
    unrendered rows -- also in a caller-owned sink that is dirty on entry."""
    dev = cuda_device
    assert n_mesh % 32
    cam, params, mesh, fv = _layer(dev, W, H, n_mesh, n_bg, faces, M=M, occl=occl)
    rs = scenes.settings_for(cam, D, device=dev)
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(3)).to(dev)
    res = []
    for fn in (fb.frosting_render, fb.frosting_render_two_step):
        p, m = _leaves(params, mesh)
        color, radii = fn(p, m, rs, face_visible=fv)
        (color * cot).sum().backward()
        res.append((color, radii, p, m))
    (c1, r1, p1, m1), (c2, r2, p2, m2) = res
    assert r1.shape == (n_mesh + n_bg,)
    assert torch.equal(r1, r2)
    assert 0 < int((r1[:n_mesh] > 0).sum()) and 0 < int((r1[n_mesh:] > 0).sum()) < n_bg
    assert torch.equal(c1.view(torch.int32), c2.view(torch.int32))
    for k in p1:
        mx, frac = rel_err_stats(p1[k].grad, p2[k].grad)
        assert mx <= 1e-3 and frac <= 1e-3, (k, mx, frac)
        dead = (r1[n_mesh:] if k in BG_KEYS else r1[:n_mesh]) <= 0
        assert float(p1[k].grad[dead].abs().sum()) == 0.0, k
        assert float(p1[k].grad.abs().sum()) > 0.0, k
    for k in ("inner", "outer"):
        mx, _ = rel_err_stats(m1[k].grad, m2[k].grad)
        assert mx <= 1e-3, (k, mx)
    sink = {k: torch.full_like(v, 7.0) for k, v in params.items()}
    p3 = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    color, radii = fb.frosting_render(p3, mesh, rs, face_visible=fv, grad_sink=sink)
    (color * cot).sum().backward()
    for k in p1:
        mx, _ = rel_err_stats(sink[k].view_as(p1[k].grad), p1[k].grad)
        assert mx <= 1e-3 and p3[k].grad is None, (k, mx)
        dead = (radii[n_mesh:] if k in BG_KEYS else radii[:n_mesh]) <= 0
        assert float(sink[k][dead].abs().sum()) == 0.0, k


def test_frosting_mode_with_background_against_the_torch_chain(cuda_device):
    """Frosting's own construction: torch properties for both blocks, cat, render_mask (trailing ones for the background),
    plain rasterizer.  Attribute values agree to ~1 ulp: statistical bounds as for the mesh-only frame."""
    dev = cuda_device
    W, H, n_mesh, n_bg = 320, 200, 50_000, 20_000
    cam, params, mesh, fv = _layer(dev, W, H, n_mesh, n_bg, 8000, seed=9)
    rs = scenes.settings_for(cam, 3, device=dev)
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(7)).to(dev)
    p1 = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    color1, radii1 = fb.frosting_render(p1, mesh, rs, face_visible=fv)
    (color1 * cot).sum().backward()
    p3 = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    a, b = scenes.frosting_attributes(p3, mesh), scenes.frosting_background_attributes(p3)
    a = {k: torch.cat([a[k], b[k]]) for k in a}
    P = n_mesh + n_bg
    mask = fb.gaussian_render_mask(fv, mesh["cells"], P)
    color3, radii3 = fb.GaussianRasterizer(rs)(means3D=a["means3D"], means2D=torch.zeros(P, 3, device=dev),
                                               opacities=a["opacities"], shs=a["shs"], scales=a["scales"],
                                               rotations=a["rotations"], visibility_mask=mask)
    (color3 * cot).sum().backward()
    d = (color1 - color3).abs()
    assert (d > 1e-4).float().mean().item() < 1e-3 and d.max().item() < 2e-2
    assert (radii1 != radii3).float().mean().item() < 1e-3
    for k in p1:
        m, frac = rel_err_stats(p1[k].grad, p3[k].grad)
        assert m <= 2e-2 and frac <= 2e-2, (k, m, frac)


def test_background_behind_the_camera_changes_nothing(cuda_device):
    """Every background Gaussian behind the camera: the frame is the mesh-only frame bit for bit and the background
    gradients are exact zeros."""
    dev = cuda_device
    W, H, n_mesh, n_bg = 320, 200, 30_001, 4000
    cam, params, mesh, fv = _layer(dev, W, H, n_mesh, n_bg, 6000, seed=4)
    rs = scenes.settings_for(cam, 3, device=dev)
    # the camera sits at the origin looking down +z (identity W2C): z < 0 is behind it
    pts = params["bg_points"].clone()
    pts[:, 2] = -1.0 - pts[:, 2].abs()
    params["bg_points"] = pts
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(5)).to(dev)
    mesh_only = {k: params[k] for k in MESH_KEYS}
    p0 = {k: v.detach().clone().requires_grad_(True) for k, v in mesh_only.items()}
    c0, r0 = fb.frosting_render(p0, mesh, rs, face_visible=fv)
    (c0 * cot).sum().backward()
    p1 = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    c1, r1 = fb.frosting_render(p1, mesh, rs, face_visible=fv)
    (c1 * cot).sum().backward()
    assert torch.equal(c0.view(torch.int32), c1.view(torch.int32))
    assert torch.equal(r0, r1[:n_mesh]) and int((r1[n_mesh:] != 0).sum()) == 0
    for k in BG_KEYS:
        assert float(p1[k].grad.abs().sum()) == 0.0, k
    for k in MESH_KEYS:
        mx, frac = rel_err_stats(p1[k].grad, p0[k].grad)
        assert mx <= 1e-3 and frac <= 1e-3, (k, mx, frac)


def test_background_attribute_kernels_against_the_reference_property_goldens(cuda_device):
    """The background rows of fb200_frosting_attributes / _backward against vectors produced by executing the reference's
    bg_* property source (tests/golden/make_frosting_attr_golden.py): values 1e-6, gradients 2e-5 of scale."""
    dev = cuda_device
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frosting_bg_attrs.npz"))
    n_mesh = 37           # a few mesh rows in front: the background rows are written behind them, in place
    cam = scenes.make_camera(64, 48, device=dev)
    params, mesh = scenes.frosting_layer(n_mesh, cam, 2, n_faces_target=64, device=dev,
                                         sh_coeffs=z["param_bg_sh_rest"].shape[1] + 1)
    for k in z.files:
        if k.startswith("param_"):
            params[k[len("param_"):]] = torch.from_numpy(z[k]).to(dev)
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in params.items()}
    out = fb.frosting_attributes_fused(leaves, mesh)
    cot_total = {}
    for k, v in out.items():
        ref = torch.from_numpy(z[f"out_{k}"]).to(dev)
        got = v[n_mesh:].reshape(ref.shape)
        assert (got - ref).abs().max().item() <= 1e-6 * max(1.0, ref.abs().max().item()), k
        cot = torch.zeros_like(v)
        cot[n_mesh:] = torch.from_numpy(z[f"cot_{k}"]).to(dev).reshape(cot[n_mesh:].shape)
        cot_total[k] = cot
    sum((out[k] * cot_total[k]).sum() for k in out).backward()
    for k in BG_KEYS:
        ref = torch.from_numpy(z[f"grad_{k}"]).to(dev)
        assert (leaves[k].grad.reshape(ref.shape) - ref).abs().max().item() <= 2e-5 * ref.abs().max().item(), k


def test_frosting_adam_with_background_groups_equals_torch_adam(cuda_device):
    """frosting_render into FrostingAdam's sink (mesh rows sparse, background groups dense) steps like torch.optim.Adam
    over the reference's twelve groups on the dense autograd gradients; state_dict round-trips; bg_points is
    scheduled."""
    dev = cuda_device
    W, H, n_mesh, n_bg = 240, 160, 30_000, 8000
    cam, params, mesh, fv = _layer(dev, W, H, n_mesh, n_bg, 5000, seed=5)
    rs = scenes.settings_for(cam, 3, device=dev)
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    fo = optim.FrostingAdam.for_frosting(params, spatial_lr_scale=2.0)
    names = [g["name"] for g in fo.param_groups]
    assert names == ["bary_coords", "sh_coordinates_dc", "sh_coordinates_rest", "opacities", "scales", "quaternions",
                     "bg_points", "bg_opacities", "bg_sh_coordinates_dc", "bg_sh_coordinates_rest", "bg_scales",
                     "bg_quaternions"]
    o = optim.OptimizationParams()
    assert [g["lr"] for g in fo.param_groups[6:]] == pytest.approx(
        [o.position_lr_init * 2.0, o.opacity_lr, o.feature_lr, o.feature_lr / 20.0, o.scaling_lr, o.rotation_lr])
    # the background groups carry no row structure even when they have as many rows as the mesh block
    assert fo.slabs.row_width[6:] == [0] * 6
    ref_params = {n: params[n].detach().clone().requires_grad_(True) for n in fo.slabs.names}
    ref = torch.optim.Adam([{"params": [ref_params[n]], "lr": g["lr"], "name": g["name"]}
                            for n, g in zip(fo.slabs.names, fo.param_groups)], lr=0.0, eps=1e-15)
    for step in range(2):
        fo.slabs.grad_slab.fill_(float("nan"))
        color, radii = fb.frosting_render(fo.params, mesh, rs, face_visible=fv, grad_sink=fo.grads)
        (color * cot).sum().backward()
        assert set(fo.grads.sparse_names) == set(MESH_KEYS)
        fo.step()
        ref.zero_grad()
        c2, _ = fb.frosting_render(ref_params, mesh, rs, face_visible=fv)
        (c2 * cot).sum().backward()
        ref.step()
        for n in fo.slabs.names:
            # the two renders' gradients differ by the blend backward's atomic order; Adam's first steps are ~lr * sign(g),
            # so an element whose tiny gradient changes sign moves the other way: count those, they must be rare
            a, b = fo.params[n].detach(), ref_params[n].detach()
            off = ((a - b).abs() > 1e-6 * (1.0 + b.abs())).double().mean().item()
            assert off <= 2e-3, (n, step, off)
            assert not torch.equal(b, params[n]), n          # the group did move
    sd = fo.state_dict()
    ref2 = torch.optim.Adam([{"params": [ref_params[n]], "lr": 0.0, "name": g["name"]}
                             for n, g in zip(fo.slabs.names, fo.param_groups)], lr=0.0, eps=1e-15)
    ref2.load_state_dict(sd)
    fo2 = optim.FrostingAdam.for_frosting(params)
    fo2.load_state_dict(ref2.state_dict())
    assert fo2.current_iteration == 2
    assert torch.equal(fo2.exp_avg, fo.exp_avg) and torch.equal(fo2.exp_avg_sq, fo.exp_avg_sq)
    lr = fo.update_learning_rate(15_000)
    sched = optim.get_expon_lr_func(o.position_lr_init * 2.0, o.position_lr_final * 2.0,
                                    lr_delay_mult=o.position_lr_delay_mult, max_steps=o.position_lr_max_steps)
    assert fo.param_groups[6]["lr"] == pytest.approx(sched(15_000)) == lr    # the last scheduled group's lr, as the reference
    assert fo.param_groups[0]["lr"] == pytest.approx(np.sqrt(0.005 * 0.00005))


def test_misaligned_grad_sink_is_rejected_before_the_backward(cuda_device):
    """A sink view at an odd element offset is contiguous, but the backward stores gradient rows with 128-bit accesses:
    it is refused before the library is called."""
    dev = cuda_device
    cam, params, mesh, _ = _layer(dev, 200, 120, 3001, 500, 500, occl=False)
    rs = scenes.settings_for(cam, 3, device=dev)
    p, m = _leaves(params, mesh)
    sink = {k: torch.zeros_like(v) for k, v in params.items()}
    sink["quats"] = torch.zeros(params["quats"].numel() + 1, device=dev)[1:].view_as(params["quats"])
    assert sink["quats"].is_contiguous() and sink["quats"].data_ptr() % 16
    color, _ = fb.frosting_render(p, m, rs, grad_sink=sink)
    launches = _lib.kernel_launches()
    with pytest.raises(RuntimeError, match="16-byte aligned"):
        color.sum().backward()
    assert _lib.kernel_launches() == launches
