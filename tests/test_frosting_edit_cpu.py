"""Edited-scene rendering (SURVEY.md row a21) without a GPU: the torch restatement against golden vectors made by the
reference's own source (tests/golden/make_frosting_edit_golden.py), the exported entry points, the argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frosting_edit.npz")
CASES = ("median_full_bg_d3", "triangle_partial_d1", "triangle_full_bg_d3", "median_partial_d1")


def golden_case(name):
    """The case's arrays over the shared scene: a case without background Gaussians takes the mesh rows only."""
    z = np.load(GOLD)
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith("scene/")}
    g.update({k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")})
    params = {k[len("param_"):]: torch.from_numpy(v) for k, v in g.items() if k.startswith("param_")}
    if not bool(g["background"]):
        params = {k: v for k, v in params.items() if not k.startswith("bg_")}
        g["orig_quats"] = g["orig_quats"][:params["quats"].shape[0]]
    return g, params


def restated(g, params, **kw):
    t = lambda k: torch.from_numpy(g[k])
    return scenes.edited_frosting_attributes(
        params, t("ref_verts"), t("faces"), t("cells"), t("inner_dist"), t("outer_dist"), t("verts"), t("campos"),
        int(g["sh_degree"]), edition_mask=t("edition_mask"), thickness_rescaling=str(g["rescaling"]),
        orig_quats=t("orig_quats"), deformation_threshold=2.0, **kw)


def rel_err(a, b):
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def check_against_golden(out, g):
    """shell / positions / scales 1e-5 relative, rotations as matrices 1e-5, dropped rows identical, colours 1e-5."""
    ref = {k[len("out_"):]: torch.from_numpy(v) for k, v in g.items() if k.startswith("out_")}
    for k in ("inner", "outer", "means3D", "scales"):
        assert rel_err(out[k].cpu(), ref[k]) <= 1e-5, k
    assert torch.equal(out["opacities"].cpu() == 0, ref["opacities"] == 0)
    assert (out["opacities"].cpu() - ref["opacities"]).abs().max() <= 1e-6
    m = scenes.quaternion_to_matrix(out["rotations"].cpu().double())
    mr = scenes.quaternion_to_matrix(ref["rotations"].double())
    assert (m - mr).abs().max() <= 1e-5
    assert (out["colors_precomp"].cpu() - ref["colors"]).abs().max() <= 1e-5


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_source(name):
    g, params = golden_case(name)
    out = restated(g, params)
    check_against_golden(out, g)
    ref_op = torch.from_numpy(g["out_opacities"])
    assert 0 < int((ref_op == 0).sum()) < ref_op.shape[0]        # the deformation drops some rows, not all


def test_golden_cases_cover_the_issue_matrix():
    seen = set()
    for name in CASES:
        g, params = golden_case(name)
        seen.add((str(g["rescaling"]), bool(g["edition_mask"].all()), "bg_points" in params, int(g["sh_degree"])))
        assert not np.allclose(g["orig_quats"][: len(params["quats"])],
                               torch.nn.functional.normalize(params["quats"], dim=-1).numpy(), atol=1e-3)
    assert {s[0] for s in seen} == {"median", "triangle"}
    assert {s[1] for s in seen} == {True, False}
    assert {s[2] for s in seen} == {True, False}
    assert {s[3] for s in seen} == {1, 3}


def test_quaternion_restatements_round_trip():
    q = torch.nn.functional.normalize(torch.randn(500, 4, generator=torch.Generator().manual_seed(0)), dim=-1)
    assert (scenes.matrix_to_quaternion(scenes.quaternion_to_matrix(q)) - scenes.standardize_quaternion(q)).abs().max() < 1e-6
    ident = scenes.quaternion_multiply(q, scenes.quaternion_invert(q))
    assert (ident - torch.tensor([1.0, 0, 0, 0])).abs().max() < 1e-6


def test_edit_entry_points_are_bound():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_frosting_edit_shell", "fb200_frosting_edit_attributes"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert callable(fb.frosting_render_edited) and fb.FrostingEdit is not None


def _edit_struct(**kw):
    d = C.c_void_p(0x1000)
    f = dict(n_verts=4, n_faces=2, rescaling=_lib.RESCALE_MEDIAN, n_edited=2, deformation_threshold=2.0)
    for n, _ in _lib.FrostingEdit._fields_[5:]:
        f[n] = d
    f.update(kw)
    return _lib.FrostingEdit(**f)


def test_edit_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    assert L.fb200_frosting_edit_shell(None, None) == -1 and b"null" in L.fb200_last_error()
    e = _edit_struct(rescaling=7)
    assert L.fb200_frosting_edit_shell(C.byref(e), None) == -1 and b"rescaling" in L.fb200_last_error()
    e = _edit_struct(d_rel_quats=None)
    assert L.fb200_frosting_edit_shell(C.byref(e), None) == -1 and b"missing face table" in L.fb200_last_error()
    e = _edit_struct(n_edited=0)
    assert L.fb200_frosting_edit_shell(C.byref(e), None) == -1 and b"at least one edited face" in L.fb200_last_error()
    e = _edit_struct(d_ref_median=None)
    assert L.fb200_frosting_edit_shell(C.byref(e), None) == -1 and b"reference table" in L.fb200_last_error()
    e = _edit_struct(n_edited=3)
    assert L.fb200_frosting_edit_shell(C.byref(e), None) == -1 and b"bad extents" in L.fb200_last_error()
    # attributes: the parameter block must describe the same mesh, and sh_degree must fit its SH rows
    d = C.c_void_p(0x1000)
    fp = _lib.FrostingParams(P=10, n_verts=4, n_faces=3, sh_rest=3, d_bary_logits=d, d_cells=d, d_faces=d,
                             d_inner_verts=d, d_outer_verts=d, d_opacity_logits=d, d_log_scales=d, d_quats=d, d_sh_dc=d,
                             d_sh_rest=d)
    e = _edit_struct()
    args = [d] * 7 + [None]
    assert L.fb200_frosting_edit_attributes(C.byref(e), C.byref(fp), 1, *args) == -1
    assert b"does not match" in L.fb200_last_error()
    fp.n_faces = 2
    assert L.fb200_frosting_edit_attributes(C.byref(e), C.byref(fp), 3, *args) == -1
    assert b"sh_degree" in L.fb200_last_error()


def test_python_surface_rejects_unsupported_options():
    from frosting_b200.edit import FrostingEdit
    v = torch.zeros(3, 3)
    f = torch.tensor([[0, 1, 2]])
    with pytest.raises(NotImplementedError, match="simple adaptation"):
        FrostingEdit(v, f, torch.zeros(1, dtype=torch.long), torch.zeros(3), torch.zeros(3), adaptation="complex")
    with pytest.raises(ValueError, match="not recognized"):
        FrostingEdit(v, f, torch.zeros(1, dtype=torch.long), torch.zeros(3), torch.zeros(3), thickness_rescaling="mean")
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        FrostingEdit(v, f, torch.zeros(1, dtype=torch.long), torch.zeros(3), torch.zeros(3))
