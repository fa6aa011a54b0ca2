"""Background Gaussians of frosting mode, host side: argument checks of the entry points (no CUDA call is reached), the
torch restatement of Frosting's bg_* properties against the reference's own source, and the scene generator's
compatibility with the frames it produced before."""
import ctypes as C
import hashlib
import os

import numpy as np
import torch

from frosting_b200 import _lib, scenes

HERE = os.path.dirname(os.path.abspath(__file__))
D = C.c_void_p(0x1000)            # 16-byte aligned dummy device pointer: never dereferenced, the checks fail first
ODD = C.c_void_p(0x1004)          # 4-byte aligned only


BG = ("d_bg_points", "d_bg_opacity_logits", "d_bg_log_scales", "d_bg_quats", "d_bg_sh_dc", "d_bg_sh_rest")


def _frame(n_mesh=10, n_bg=5):
    prm = _lib.Params(P=n_mesh + n_bg, sh_degree=3, sh_coeffs=16, image_width=64, image_height=64, tanfovx=0.5,
                      tanfovy=0.5, scale_modifier=1.0, prefiltered=0, debug=0)
    fp = _lib.FrostingParams(P=n_mesh, n_verts=4, n_faces=2, sh_rest=15, d_bary_logits=D, d_cells=D, d_faces=D,
                             d_inner_verts=D, d_outer_verts=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D,
                             d_sh_rest=D, n_bg=n_bg, **{f: D for f in BG})
    inp = _lib.Inputs(d_background=D, d_viewmatrix=D, d_projmatrix=D, d_campos=D, frosting=C.addressof(fp))
    fg = _lib.FrostingGrads(d_bary_logits=D, d_opacity_logits=D, d_log_scales=D, d_quats=D, d_sh_dc=D, d_sh_rest=D,
                            **{f: D for f in BG})
    grads = _lib.Grads(sparse_rows=1, frosting=C.addressof(fg))
    return prm, fp, inp, fg, grads


def _fwd(L, prm, inp):
    return L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()), None, None, None)


def _bwd(L, prm, inp, grads):
    # a workspace that passes the size checks, so that the gradient checks behind them are reached; every call below
    # fails one of those, so no kernel is ever launched on these dummy pointers
    big = 1 << 40
    ws = _lib.Workspace(d_geom=D, geom_bytes=big, d_image=D, image_bytes=big, d_status=D)
    return L.fb200_backward(C.byref(prm), C.byref(inp), C.byref(ws), D, D, C.byref(grads), None)


def _err(L):
    return L.fb200_last_error().decode()


def test_frosting_entry_points_reject_bad_background_arguments():
    L = _lib.lib()
    keep = _frame()
    prm, fp, inp, fg, grads = keep
    # valid background rows get past every frosting check (the empty workspace is the first thing missing)
    assert _fwd(L, prm, inp) == -1 and "workspace pointers missing" in _err(L)
    for entry in (lambda: L.fb200_forward_geometry(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()), None, None),
                  lambda: L.fb200_forward_raster(C.byref(prm), C.byref(inp), C.byref(_lib.Workspace()), None, None,
                                                 None)):
        assert entry() == -1 and "workspace pointers missing" in _err(L)
        fp.n_bg = 4
        assert entry() == -1 and "do not match the parameter block" in _err(L)
        fp.n_bg = 5
    # P != frosting->P + n_bg, with and without background rows
    prm.P = 14
    assert _fwd(L, prm, inp) == -1 and "do not match the parameter block" in _err(L)
    fp.n_bg = 0
    assert _fwd(L, prm, inp) == -1 and "do not match the parameter block" in _err(L)
    prm.P = 10
    assert _fwd(L, prm, inp) == -1 and "workspace pointers missing" in _err(L)     # n_bg == 0: the mesh-only frame
    fp.n_bg, prm.P = -1, 9
    assert _fwd(L, prm, inp) == -1 and "n_bg must be >= 0" in _err(L)
    fp.n_bg, prm.P = 5, 15
    # a missing pointer, each of the six
    for f in BG:
        setattr(fp, f, None)
        assert _fwd(L, prm, inp) == -1 and "missing parameter pointer" in _err(L), f
        setattr(fp, f, D)
    # misaligned quaternions, parameters and gradients
    fp.d_bg_quats = ODD
    assert _fwd(L, prm, inp) == -1 and "quats must be 16-byte aligned" in _err(L)
    fp.d_bg_quats = D
    fg.d_bg_quats = ODD
    assert _bwd(L, prm, inp, grads) == -1 and "dL/dquats must be 16-byte aligned" in _err(L)
    fg.d_bg_quats = D
    for f in BG:
        setattr(fg, f, None)
        assert _bwd(L, prm, inp, grads) == -1 and "gradient pointers missing" in _err(L), f
        setattr(fg, f, D)
    # parameters without gradients, gradients without parameters
    for f in BG:
        setattr(fg, f, None)
    assert _bwd(L, prm, inp, grads) == -1 and "exactly when there are background" in _err(L)
    for f in BG:
        setattr(fg, f, D)
    fp.n_bg, prm.P = 0, 10
    assert _bwd(L, prm, inp, grads) == -1 and "exactly when there are background" in _err(L)
    del keep


def test_background_attribute_entry_points_reject_bad_arguments():
    L = _lib.lib()
    _, fp, _, fg, _ = keep = _frame()
    out = [D] * 5
    up = [D] * 5
    # the kernels store rotation rows as float4: a misaligned base is rejected, with and without background rows
    for n_bg in (5, 0):
        fp.n_bg = n_bg
        assert L.fb200_frosting_attributes(C.byref(fp), D, D, D, ODD, D, None) == -1 and \
            "rotations must be 16-byte aligned" in _err(L)
        fg_bg = [getattr(fg, f) for f in BG]
        for f in BG:
            setattr(fg, f, D if n_bg else None)
        assert L.fb200_frosting_attributes_backward(C.byref(fp), D, D, D, ODD, D, C.byref(fg), None) == -1 and \
            "dL/drotations must be 16-byte aligned" in _err(L)
        for f, v in zip(BG, fg_bg):
            setattr(fg, f, v)
    fp.n_bg = 5
    assert L.fb200_frosting_attributes(C.byref(fp), D, None, D, D, D, None) == -1 and \
        "missing output pointer" in _err(L)
    fp.d_bg_quats = ODD
    assert L.fb200_frosting_attributes(C.byref(fp), *out, None) == -1 and "quats must be" in _err(L)
    fp.d_bg_quats = D
    for f in BG:
        setattr(fg, f, None)
    assert L.fb200_frosting_attributes_backward(C.byref(fp), *up, C.byref(fg), None) == -1 and \
        "exactly when there are background" in _err(L)
    for f in BG:
        setattr(fg, f, D)
    fg.d_bg_sh_dc = None
    assert L.fb200_frosting_attributes_backward(C.byref(fp), *up, C.byref(fg), None) == -1 and \
        "gradient pointers missing" in _err(L)
    fg.d_bg_sh_dc = D
    fg.d_bg_quats = ODD
    assert L.fb200_frosting_attributes_backward(C.byref(fp), *up, C.byref(fg), None) == -1 and \
        "dL/dquats must be 16-byte aligned" in _err(L)
    fg.d_bg_quats = D
    assert L.fb200_frosting_attributes_backward(C.byref(fp), D, None, D, D, D, C.byref(fg), None) == -1 and \
        "upstream gradient" in _err(L)
    del keep


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



MESH_GRADS = ("d_bary_logits", "d_opacity_logits", "d_log_scales", "d_quats", "d_sh_dc", "d_sh_rest")


def test_attribute_entry_points_reject_bases_the_kernels_cannot_vector_access():
    """The attribute kernels move sh_rest, shs (sh_rest == 15) and the mesh parameter gradients with 128-bit accesses.
    Every call also carries a later argument error, so none of them can reach a launch."""
    L = _lib.lib()
    _, fp, _, fg, _ = keep = _frame()
    fp.d_sh_rest = ODD
    assert L.fb200_frosting_attributes(C.byref(fp), D, D, D, ODD, D, None) == -1 and \
        "sh_rest 16-byte aligned" in _err(L)
    fp.d_sh_rest = D
    assert L.fb200_frosting_attributes(C.byref(fp), D, D, D, ODD, ODD, None) == -1 and \
        "shs must be 16-byte aligned" in _err(L)
    assert L.fb200_frosting_attributes_backward(C.byref(fp), D, D, D, ODD, ODD, C.byref(fg), None) == -1 and \
        "dL/dshs must be 16-byte aligned" in _err(L)
    for f in MESH_GRADS:
        setattr(fg, f, ODD)
        assert L.fb200_frosting_attributes_backward(C.byref(fp), D, None, D, D, D, C.byref(fg), None) == -1 and \
            "mesh parameter gradients must be 16-byte aligned" in _err(L), f
        setattr(fg, f, D)
    del keep


def test_frosting_backward_checks_mesh_gradients_against_the_mesh_rows():
    """fb200_backward in frosting mode takes the attribute backward's gradient contract: with mesh rows their gradients
    are required and 16-byte aligned; without (background only, what frosting_render passes for an empty mesh block)
    they may be NULL.  The misaligned dL/drotations behind the frosting checks shows that a call got past them."""
    L = _lib.lib()
    prm, fp, inp, fg, grads = keep = _frame()
    grads.d_dL_drotations = ODD
    fg.d_sh_dc = ODD
    assert _bwd(L, prm, inp, grads) == -1 and "mesh parameter gradients must be 16-byte aligned" in _err(L)
    fg.d_sh_dc = D
    assert _bwd(L, prm, inp, grads) == -1 and "dL/drotations / dL/dsh rows must be 16-byte aligned" in _err(L)
    fp.P, prm.P = 0, 5
    for f in MESH_GRADS:
        setattr(fg, f, None)
    assert _bwd(L, prm, inp, grads) == -1 and "dL/drotations / dL/dsh rows must be 16-byte aligned" in _err(L)
    del keep
