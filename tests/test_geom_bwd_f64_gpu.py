"""The per-Gaussian backward (csrc/geom_bwd.cu) element by element against its float64 model (oracle/geom_f64.py).

The kernel's input is the blend backward's accumulator record of each Gaussian (fb200_layout.geom_acc) and the forward's
colour clamp bits (geom_clamped).  Both are read back after the frame, so the model sees exactly what the kernel consumed:
no atomic-order noise, no sampling, no fraction of elements allowed off.  Every element of every gradient output of
every rendered row must satisfy

    |g32 - g64| <= TAU * m64 + 1e-30,

m64 being the element's componentwise condition (geom_f64.vjp_by_slot).  The only rows left out are those whose float32
and float64 guard-band decisions can differ (|t.x / t.z| within 1e-6 relative of 1.3 tanfov); there must be < 0.1 % of
them.  The scenes populate, on purpose and asserted, each regime where this kernel can be wrong: the guard band crossed
in x only, y only and both, a clamped colour channel beside unclamped ones, view depth within 2x of the 0.2 near plane,
needles under the 0.3 dilation, raw quaternions of norm outside [0.5, 2]; with scale modifiers 0.6, 1 and 1.7, SH rows
of 1, 9, 16 and 20 coefficients at degrees 0-3 and a camera off the origin.  Every path of the kernel runs: the in-place
walk (dense rows: unrendered rows exactly 0 in NaN-poisoned buffers; P % 32 != 0 and a run of unrendered rows), the list
walk (unrendered rows untouched), the precomputed covariance / colour inputs, and frosting mode (mesh and background rows
in one warp, occlusion lookup, shell vertex gradients).

TAU is more than ten times the largest |g32 - g64| / m64 observed on an H100 (sm_90a build) over these cases, OBSERVED;
a kernel that drops the guard-band mask of d/dt.x exceeds the bound by a ratio of ~0.1."""
import ctypes as C

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import _lib, scenes
from frosting_b200._lib import Grads, Inputs, Params, Workspace
from frosting_b200.frosting_render import BG_KEYS, MESH_KEYS, FrostingBlock
from oracle import geom_f64
from tests.util import regime_gaussians

pytestmark = pytest.mark.gpu

OBSERVED = 6.3e-5       # largest |g32 - g64| / m64 on an H100 80GB HBM3 (700 W) over every case of this file: d(scale)
TAU = 7e-4
W, H = 320, 208
P = 20_011             # P % 32 == 11
N_BEHIND = 100         # one run of unrendered rows (three whole warps of them and two partial ones)
REGIME_MIN = 0.03


def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _run(rs, P, M, D, inp, grads, dev):
    """Forward (two-phase, exactly sized binning) and backward through the C ABI; returns radii, the accumulator
    records [P,12] and the clamp bits [P,3] the per-Gaussian backward consumed."""
    L = _lib.lib()
    prm = Params(P=P, sh_degree=D, sh_coeffs=M, image_width=W, image_height=H, tanfovx=float(rs.tanfovx),
                 tanfovy=float(rs.tanfovy), scale_modifier=float(rs.scale_modifier), prefiltered=0, debug=0, extra=None)
    t = dict(bg=rs.bg.contiguous(), view=rs.viewmatrix.contiguous(), proj=rs.projmatrix.contiguous(),
             campos=rs.campos.contiguous())
    inp.d_background, inp.d_viewmatrix, inp.d_projmatrix, inp.d_campos = (_p(t[k]) for k in ("bg", "view", "proj",
                                                                                             "campos"))
    geom = torch.empty(L.fb200_geom_bytes(P), dtype=torch.uint8, device=dev)
    image = torch.empty(L.fb200_image_bytes(W, H), dtype=torch.uint8, device=dev)
    status = torch.zeros(_lib.FB200_STATUS_WORDS, dtype=torch.int32, device=dev)
    ws = Workspace(d_geom=geom.data_ptr(), geom_bytes=geom.numel(), d_image=image.data_ptr(), image_bytes=image.numel(),
                   d_binning=None, binning_bytes=0, binning_capacity=0, d_status=status.data_ptr(),
                   acc_zeroed_by_forward=0, h_status=None)
    color = torch.empty(3, H, W, device=dev)
    radii = torch.empty(P, dtype=torch.int32, device=dev)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    _lib.check(L.fb200_forward_geometry(C.byref(prm), C.byref(inp), C.byref(ws), _p(radii), stream))
    R = max(int(status[_lib.ST_NUM_RENDERED]), 1)
    binning = torch.empty(L.fb200_binning_bytes(R), dtype=torch.uint8, device=dev)
    ws.d_binning, ws.binning_bytes, ws.binning_capacity = binning.data_ptr(), binning.numel(), R
    _lib.check(L.fb200_forward_raster(C.byref(prm), C.byref(inp), C.byref(ws), _p(color), _p(radii), stream))
    cot = torch.randn(3, H, W, generator=torch.Generator().manual_seed(P % 97)).to(dev)
    _lib.check(L.fb200_backward(C.byref(prm), C.byref(inp), C.byref(ws), _p(radii), _p(cot), C.byref(grads), stream))
    torch.cuda.synchronize(dev)
    v = _lib.workspace_views(geom, image, binning, P, W, H, R, R)
    acc = v["acc"].clone()
    bits = v["clamped"].clone()
    clamped = torch.stack([(bits >> c) & 1 for c in range(3)], 1).bool()
    assert int(status[_lib.ST_OVERFLOW]) == 0
    return radii, acc, clamped


def _guard_ok(cam64, means):
    """Rows whose float32 and float64 guard-band decisions cannot differ."""
    rx, ry = geom_f64.guard_ratio(cam64, means)
    return ((rx - 1).abs() > 1e-6) & ((ry - 1).abs() > 1e-6)


def _check(name, g32, g64, m64, worst):
    r = geom_f64.excess(g32, g64, m64)
    bad = geom_f64.outside(g32, g64, m64, TAU)
    worst[name] = max(worst.get(name, 0.0), float(r.max()) if r.numel() else 0.0)
    assert not bool(bad.any()), (name, int(bad.sum()), float(r.max()))


def _regimes(cam64, rows, g, clamped, mod):
    """Share of the rows in each regime, computed from the rows themselves."""
    rx, ry = geom_f64.guard_ratio(cam64, g["means3D"][rows])
    t = torch.cat([g["means3D"][rows].double(), torch.ones(len(rows), 1, dtype=torch.float64, device=rows.device)], 1)
    depth = (t @ cam64.view)[:, 2]
    cov = geom_f64.projected_cov(cam64, g["means3D"][rows].double(), g["scales"][rows].double(),
                                 g["rotations"][rows].double())
    lam = torch.linalg.eigvalsh(cov)
    qn = g["rotations"][rows].norm(dim=1)
    cl = clamped[rows]
    share = lambda m: float(m.double().mean())
    return dict(guard_x=share((rx > 1) & (ry <= 1)), guard_y=share((ry > 1) & (rx <= 1)), guard_xy=share((rx > 1) & (ry > 1)),
                clamp_mixed=share(cl.any(1) & ~cl.all(1)), near=share(depth <= 0.4), needle=share(lam.max(1).values < 0.3),
                quat_norm=share((qn < 0.5) | (qn > 2)))


def _camera(dev):
    return scenes.ring_cameras(8, W, H, device=dev)[3]


CASES = [  # D, M, scale modifier, sparse_rows
    (3, 16, 1.7, 0),
    (0, 1, 0.6, 0),
    (2, 9, 1.0, 0),
    (3, 20, 0.6, 1),
    (1, 16, 1.7, 1),
]


@pytest.mark.parametrize("D,M,mod,sparse", CASES)
def test_every_gradient_element_matches_the_float64_model(cuda_device, D, M, mod, sparse):
    dev = cuda_device
    cam = _camera(dev)
    rs = scenes.settings_for(cam, D, scale_modifier=mod, device=dev)
    g = regime_gaussians(P, cam, 40 + D + M, sh_coeffs=M, n_behind=N_BEHIND, device=dev)
    nan = lambda *shape: torch.full(shape, float("nan"), device=dev)
    out = dict(means2D=nan(P, 3), opacities=nan(P, 1), means3D=nan(P, 3), shs=nan(P, M, 3), scales=nan(P, 3),
               rotations=nan(P, 4))
    inp = Inputs(d_means3D=_p(g["means3D"]), d_shs=_p(g["shs"]), d_opacities=_p(g["opacities"]),
                 d_scales=_p(g["scales"]), d_rotations=_p(g["rotations"]))
    grads = Grads(d_dL_dmeans2D=_p(out["means2D"]), d_dL_dopacity=_p(out["opacities"]), d_dL_dmeans3D=_p(out["means3D"]),
                  d_dL_dsh=_p(out["shs"]), d_dL_dscales=_p(out["scales"]), d_dL_drotations=_p(out["rotations"]),
                  sparse_rows=sparse)
    radii, acc, clamped = _run(rs, P, M, D, inp, grads, dev)
    rendered = radii > 0
    dead = ~rendered
    assert bool(dead[P // 2:P // 2 + N_BEHIND].all())
    for k, v in out.items():
        if sparse:
            assert bool(v[dead].isnan().all()), k          # the list walk leaves unrendered rows alone
        else:
            assert bool((v[dead] == 0).all()), k           # the in-place walk writes exact zeros there
    cam64 = geom_f64.Camera(rs)
    rows = torch.nonzero(rendered).flatten()
    ok = _guard_ok(cam64, g["means3D"][rows])
    assert float((~ok).double().mean()) < 1e-3
    rows = rows[ok]
    shares = _regimes(cam64, rows, g, clamped, mod)
    print(f"\nD={D} M={M} mod={mod} sparse={sparse}: {len(rows)} rows compared, {int((~ok).sum())} left out; {shares}")
    assert all(v >= REGIME_MIN for v in shares.values()), shares
    # dL/dmeans2D is the record's first two slots, bit for bit
    assert torch.equal(out["means2D"][rows, :2], acc[rows, :2]) and bool((out["means2D"][rows, 2] == 0).all())
    g64, m64 = geom_f64.splat_grads(cam64, acc[rows].double(), clamped=clamped[rows], D=D, **{k: g[k][rows] for k in g})
    worst = {}
    for k in ("means3D", "opacities", "scales", "rotations", "shs"):
        _check(k, out[k][rows], g64[k], m64[k], worst)
    print("max |g32 - g64| / m64:", worst)


@pytest.mark.parametrize("sparse", [0, 1])
def test_precomputed_covariance_and_colours_match_the_float64_model(cuda_device, sparse):
    dev = cuda_device
    cam = _camera(dev)
    rs = scenes.settings_for(cam, 0, scale_modifier=1.7, device=dev)      # the modifier does not apply to cov3D
    g = regime_gaussians(P, cam, 77, sh_coeffs=1, n_behind=N_BEHIND, device=dev)
    R = geom_f64.rotation_rows(g["rotations"].double())
    S = R.transpose(-1, -2) @ (R * (g["scales"].double() ** 2)[:, :, None])
    cov3D = S[:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]].float().contiguous()
    colors = (torch.rand(P, 3, generator=torch.Generator().manual_seed(3)) * 1.4 - 0.2).to(dev)
    nan = lambda *shape: torch.full(shape, float("nan"), device=dev)
    out = dict(means2D=nan(P, 3), opacities=nan(P, 1), means3D=nan(P, 3), colors=nan(P, 3), cov3D=nan(P, 6))
    inp = Inputs(d_means3D=_p(g["means3D"]), d_colors_precomp=_p(colors), d_opacities=_p(g["opacities"]),
                 d_cov3D_precomp=_p(cov3D))
    grads = Grads(d_dL_dmeans2D=_p(out["means2D"]), d_dL_dcolors=_p(out["colors"]), d_dL_dopacity=_p(out["opacities"]),
                  d_dL_dmeans3D=_p(out["means3D"]), d_dL_dcov3D=_p(out["cov3D"]), sparse_rows=sparse)
    radii, acc, clamped = _run(rs, P, 0, 0, inp, grads, dev)
    dead = radii <= 0
    for k, v in out.items():
        assert bool(v[dead].isnan().all() if sparse else (v[dead] == 0).all()), k
    cam64 = geom_f64.Camera(rs)
    rows = torch.nonzero(~dead).flatten()
    ok = _guard_ok(cam64, g["means3D"][rows])
    assert float((~ok).double().mean()) < 1e-3
    rows = rows[ok]
    # precomputed colours are not clamped by the rasterizer: dL/dcolors is the record's colour slots as they are
    assert torch.equal(out["colors"][rows], acc[rows, 6:9])
    assert torch.equal(out["means2D"][rows, :2], acc[rows, :2])
    g64, m64 = geom_f64.splat_grads(cam64, acc[rows].double(), means3D=g["means3D"][rows],
                                    opacities=g["opacities"][rows], cov3D=cov3D[rows], colors=colors[rows])
    worst = {}
    for k in ("means3D", "opacities", "cov3D"):
        _check(k, out[k][rows], g64[k], m64[k], worst)
    print(f"\nprecomputed, sparse={sparse}: {len(rows)} rows; max |g32 - g64| / m64:", worst)


@pytest.mark.parametrize("M,D,mod", [(9, 2, 1.0), (16, 3, 1.3)])
def test_frosting_parameter_gradients_match_the_float64_model(cuda_device, M, D, mod):
    """Frosting mode through the parameter block of frosting_render's FrostingBlock: the chain rule through softmax
    barycentrics, sigmoid, exp, normalize and dc | rest, mesh and background rows in one warp (n_mesh % 32 != 0), the
    occlusion lookup on, the shell vertex gradients scatter-added.  Rows that were not rendered stay as they were."""
    dev = cuda_device
    n_mesh, n_bg = 20_003, 5000
    cam = scenes.ring_cameras(8, W, H, device=dev)[1]
    params, mesh = scenes.frosting_layer(n_mesh, cam, 21 + M, n_faces_target=4000, device=dev, view_distance=4.5,
                                         sh_coeffs=M, n_background=n_bg)
    _, fv, _ = fb.rasterize_mesh(mesh["verts"], mesh["faces"], cam.full_proj_transform, H, W, mark_last_on_bg=True)
    shell = dict(mesh, inner=mesh["inner"].clone().requires_grad_(True), outer=mesh["outer"].clone().requires_grad_(True))
    blk = FrostingBlock(params, shell, fv)
    assert blk.n_mesh % 32 and blk.vert_grad
    fg, d = blk.grad_targets(None)
    for k in MESH_KEYS + BG_KEYS:
        d[k].fill_(float("nan"))
    m2 = torch.full((blk.rows, 3), float("nan"), device=dev)
    rs = scenes.settings_for(cam, D, scale_modifier=mod, device=dev)
    inp = Inputs(n_cell_points=0, frosting=C.addressof(blk.fp))
    grads = Grads(d_dL_dmeans2D=_p(m2), sparse_rows=1, frosting=C.addressof(fg))
    radii, acc, clamped = _run(rs, blk.rows, M, D, inp, grads, dev)
    rendered = radii > 0
    mesh_rows = torch.nonzero(rendered[:n_mesh]).flatten()
    bg_rows = torch.nonzero(rendered[n_mesh:]).flatten()
    assert 0 < len(mesh_rows) < n_mesh and 0 < len(bg_rows) < n_bg
    for k in MESH_KEYS + BG_KEYS:
        dead = ~(rendered[n_mesh:] if k in BG_KEYS else rendered[:n_mesh])
        assert bool(d[k][dead].isnan().all()), k
    assert bool(m2[~rendered].isnan().all())
    frame_rows = torch.nonzero(rendered).flatten()
    assert torch.equal(m2[frame_rows, :2], acc[frame_rows, :2]) and bool((m2[frame_rows, 2] == 0).all())
    # guard-band decisions from the float64 attributes
    cam64 = geom_f64.Camera(rs)
    p64 = {k: v.double() for k, v in params.items()}
    m64_mesh = dict(mesh, inner=mesh["inner"].double(), outer=mesh["outer"].double())
    means = torch.cat([scenes.frosting_attributes(p64, m64_mesh)["means3D"], p64["bg_points"]])
    ok = _guard_ok(cam64, means)
    assert float((~ok[frame_rows]).double().mean()) < 1e-3
    mesh_rows = mesh_rows[ok[mesh_rows]]
    bg_rows = bg_rows[ok[n_mesh + bg_rows]]
    t = blk.tensors
    g64, m64 = geom_f64.frosting_grads(cam64, acc.double(), clamped, D, {k: t[k] for k in MESH_KEYS + BG_KEYS},
                                       dict(faces=t["faces"], cells=t["cells"], inner=t["inner_verts"],
                                            outer=t["outer_verts"]), mesh_rows, bg_rows)
    worst = {}
    for k in MESH_KEYS:
        _check(k, d[k][mesh_rows].reshape(g64[k].shape), g64[k], m64[k], worst)
    for k in BG_KEYS:
        _check(k, d[k][bg_rows].reshape(g64[k].shape), g64[k], m64[k], worst)
    # shell vertices touched only by rows left out of the comparison are not compared
    left = torch.ones(t["inner_verts"].shape[0], dtype=torch.bool, device=dev)
    out_rows = torch.nonzero(rendered[:n_mesh] & ~ok[:n_mesh]).flatten()
    left[t["faces"].long()[t["cells"][out_rows]].flatten()] = False
    for k, name in (("inner", "inner_verts"), ("outer", "outer_verts")):
        _check(k, d[name][left], g64[k][left], m64[k][left], worst)
    qn = torch.cat([params["quats"][mesh_rows], params["bg_quats"][bg_rows]]).norm(dim=1)
    print(f"\nfrosting M={M} D={D} mod={mod}: {len(mesh_rows)} mesh + {len(bg_rows)} background rows, quaternion norm "
          f"outside [0.5, 2]: {float(((qn < 0.5) | (qn > 2)).double().mean()):.3f}; max |g32 - g64| / m64:", worst)
