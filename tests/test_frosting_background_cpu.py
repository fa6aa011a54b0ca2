"""Background Gaussians of frosting mode, host side: argument checks of the new entry points (no CUDA call is reached),
the struct-size query, the torch restatement of Frosting's bg_* properties against the reference's own source, and the
scene generator's compatibility with the frames it produced before."""
import ctypes as C
import hashlib
import os

import numpy as np
import torch

from frosting_b200 import _lib, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
D = C.c_void_p(0x1000)            # 16-byte aligned dummy device pointer: never dereferenced, the checks fail first
ODD = C.c_void_p(0x1004)          # 4-byte aligned only


def _frame(n_mesh=10, n_bg=5):
    prm = _lib.Params(P=n_mesh + n_bg, sh_degree=3, sh_coeffs=16, image_width=64, image_height=64, tanfovx=0.5,
                      tanfovy=0.5, scale_modifier=1.0, prefiltered=0, debug=0)
    fp = _lib.FrostingParams(P=n_mesh, n_verts=4, n_faces=2, sh_rest=15, d_bary_logits=D, d_cells=D, d_faces=D,
                             d_inner_verts=D, d_outer_verts=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D,
                             d_sh_rest=D)
    inp = _lib.Inputs(d_background=D, d_viewmatrix=D, d_projmatrix=D, d_campos=D, frosting=C.addressof(fp))
    bg = _lib.FrostingBackground(n=n_bg, d_points=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D, d_sh_rest=D)
    bgg = _lib.FrostingBackgroundGrads(d_points=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D, d_sh_rest=D)
    fg = _lib.FrostingGrads(d_bary_logits=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D, d_sh_rest=D)
    grads = _lib.Grads(sparse_rows=1, frosting=C.addressof(fg))
    return prm, fp, inp, bg, bgg, fg, grads


def _fwd(L, prm, inp, bg):
    return L.fb200_frosting_forward(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()),
                                    C.byref(bg) if bg is not None else None, None, None, None)


def _bwd(L, prm, inp, bg, grads, bgg):
    # a workspace that passes the size checks, so that the gradient checks behind them are reached; every call below
    # fails one of those, so no kernel is ever launched on these dummy pointers
    big = 1 << 40
    ws = _lib.Workspace(d_geom=D, geom_bytes=big, d_image=D, image_bytes=big, d_status=D)
    return L.fb200_frosting_backward(C.byref(prm), C.byref(inp), C.byref(ws),
                                     C.byref(bg) if bg is not None else None, D, D, C.byref(grads),
                                     C.byref(bgg) if bgg is not None else None, None)


def _err(L):
    return L.fb200_last_error().decode()


def test_frosting_entry_points_reject_bad_background_arguments():
    L = _lib.lib()
    keep = _frame()
    prm, fp, inp, bg, bgg, fg, grads = keep
    # a valid background block gets past every frosting check (the empty workspace is the first thing missing)
    assert _fwd(L, prm, inp, bg) == -1 and "workspace pointers missing" in _err(L)
    for entry in (lambda b: L.fb200_frosting_forward_geometry(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()),
                                                              C.byref(b), None, None),
                  lambda b: L.fb200_frosting_forward_raster(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()),
                                                            C.byref(b), None, None, None)):
        assert entry(bg) == -1 and "workspace pointers missing" in _err(L)
        bg.n = 4
        assert entry(bg) == -1 and "do not match the parameter block" in _err(L)
        bg.n = 5
    # P != frosting->P + n
    prm.P = 14
    assert _fwd(L, prm, inp, bg) == -1 and "do not match the parameter block" in _err(L)
    assert _fwd(L, prm, inp, None) == -1 and "do not match the parameter block" in _err(L)
    prm.P = 10
    assert _fwd(L, prm, inp, None) == -1 and "workspace pointers missing" in _err(L)    # NULL: the mesh-only frame
    bg.n = 0
    assert _fwd(L, prm, inp, bg) == -1 and "workspace pointers missing" in _err(L)      # n == 0: the same
    bg.n = -1
    prm.P = 9
    assert _fwd(L, prm, inp, bg) == -1 and "n must be >= 0" in _err(L)
    bg.n, prm.P = 5, 15
    # a missing pointer, each of the six
    for f in ("d_points", "d_opacity_logits", "d_log_scales", "d_quats", "d_sh_dc", "d_sh_rest"):
        setattr(bg, f, None)
        assert _fwd(L, prm, inp, bg) == -1 and "missing parameter pointer" in _err(L), f
        setattr(bg, f, D)
    # misaligned quaternions, parameters and gradients
    bg.d_quats = ODD
    assert _fwd(L, prm, inp, bg) == -1 and "quats must be 16-byte aligned" in _err(L)
    bg.d_quats = D
    bgg.d_quats = ODD
    assert _bwd(L, prm, inp, bg, grads, bgg) == -1 and "dL/dquats must be 16-byte aligned" in _err(L)
    bgg.d_quats = D
    for f in ("d_points", "d_opacity_logits", "d_log_scales", "d_quats", "d_sh_dc", "d_sh_rest"):
        setattr(bgg, f, None)
        assert _bwd(L, prm, inp, bg, grads, bgg) == -1 and "gradient pointers missing" in _err(L), f
        setattr(bgg, f, D)
    # gradients without parameters, parameters without gradients
    assert _bwd(L, prm, inp, bg, grads, None) == -1 and "exactly when there are background" in _err(L)
    prm.P = 10
    assert _bwd(L, prm, inp, None, grads, bgg) == -1 and "exactly when there are background" in _err(L)
    # the new entry points are frosting mode only
    inp.frosting = None
    assert _fwd(L, prm, inp, bg) == -1 and "frosting mode (fb200_inputs.frosting) required" in _err(L)


def test_background_attribute_entry_points_reject_bad_arguments():
    L = _lib.lib()
    _, _, _, bg, bgg, _, _ = keep = _frame()
    out = [D] * 5
    assert L.fb200_frosting_background_attributes(None, 15, *out, None) == -1 and "null background" in _err(L)
    assert L.fb200_frosting_background_attributes(C.byref(bg), -1, *out, None) == -1 and "sh_rest" in _err(L)
    assert L.fb200_frosting_background_attributes(C.byref(bg), 15, D, D, D, ODD, D, None) == -1 and \
        "rotations must be 16-byte aligned" in _err(L)
    assert L.fb200_frosting_background_attributes(C.byref(bg), 15, D, None, D, D, D, None) == -1 and \
        "missing output pointer" in _err(L)
    bg.d_quats = ODD
    assert L.fb200_frosting_background_attributes(C.byref(bg), 15, *out, None) == -1 and "quats must be" in _err(L)
    bg.d_quats = D
    up = [D] * 5
    assert L.fb200_frosting_background_attributes_backward(C.byref(bg), 15, None, *up, None, None) == -1 and \
        "exactly when there are background" in _err(L)
    bgg.d_sh_dc = None
    assert L.fb200_frosting_background_attributes_backward(C.byref(bg), 15, None, *up, C.byref(bgg), None) == -1 and \
        "gradient pointers missing" in _err(L)
    bgg.d_sh_dc = D
    assert L.fb200_frosting_background_attributes_backward(C.byref(bg), 15, None, D, D, D, ODD, D, C.byref(bgg),
                                                           None) == -1 and "dL/drotations" in _err(L)
    assert L.fb200_frosting_background_attributes_backward(C.byref(bg), 15, None, D, None, D, D, D, C.byref(bgg),
                                                           None) == -1 and "upstream gradient" in _err(L)
    del keep


def test_background_struct_sizes_match_the_mirrors():
    L = _lib.lib()
    out = (C.c_size_t * 2)()
    assert L.fb200_frosting_background_struct_sizes(out) == 0
    assert list(out) == [C.sizeof(_lib.FrostingBackground), C.sizeof(_lib.FrostingBackgroundGrads)] == [56, 48]
    assert L.fb200_frosting_background_struct_sizes(None) == -1


def test_torch_background_properties_match_the_reference_goldens():
    """scenes.frosting_background_attributes (the GPU tests' oracle) against the reference's bg_* source executed by
    tests/golden/make_frosting_bg_attr_golden.py: values 1e-6, gradients 2e-5 of scale."""
    z = np.load(os.path.join(HERE, "golden", "frosting_bg_attrs.npz"))
    leaf = {k[len("param_"):]: torch.from_numpy(z[k]).requires_grad_(True) for k in z.files if k.startswith("param_")}
    assert len(leaf) == 6
    out = scenes.frosting_background_attributes(leaf)
    for k, v in out.items():
        ref = torch.from_numpy(z[f"out_{k}"])
        assert v.shape == ref.shape, k
        assert (v - ref).abs().max().item() <= 1e-6 * max(1.0, ref.abs().max().item()), k
    sum((out[k] * torch.from_numpy(z[f"cot_{k}"])).sum() for k in out).backward()
    for k, v in leaf.items():
        ref = torch.from_numpy(z[f"grad_{k}"])
        assert (v.grad - ref).abs().max().item() <= 2e-5 * ref.abs().max().item(), k


def _digest(*dicts):
    h = hashlib.sha256()
    for d in dicts:
        for k in sorted(d):
            h.update(k.encode())
            h.update(d[k].contiguous().numpy().tobytes())
    return h.hexdigest()


def test_frosting_layer_without_background_is_unchanged():
    """n_background=0 (the default) returns the tensors and keys the generator returned before background Gaussians
    existed (digest pinned from that version), and n_background > 0 leaves the mesh-bound draws untouched."""
    cam = scenes.make_camera(160, 96)
    pinned = "27daff4a6f0470d131e2324e6060c02aea1e3d7b9db33027fba4e927ddb08675"
    assert _digest(*scenes.frosting_layer(3001, cam, 17, n_faces_target=500)) == pinned
    assert _digest(*scenes.frosting_layer(3001, cam, 17, n_faces_target=500, n_background=0)) == pinned
    p, m = scenes.frosting_layer(3001, cam, 17, n_faces_target=500, n_background=700)
    assert _digest({k: v for k, v in p.items() if not k.startswith("bg_")}, m) == pinned
    assert {k: tuple(p[k].shape) for k in p if k.startswith("bg_")} == {
        "bg_points": (700, 3), "bg_opacity_logits": (700,), "bg_log_scales": (700, 3), "bg_quats": (700, 4),
        "bg_sh_dc": (700, 1, 3), "bg_sh_rest": (700, 15, 3)}
    # Frosting's definition of a background Gaussian: outside the base mesh's bounding box (frosting_model.py:567-574)
    lo, hi = m["verts"].min(0).values, m["verts"].max(0).values
    assert not bool(((p["bg_points"] > lo) & (p["bg_points"] < hi)).all(1).any())

