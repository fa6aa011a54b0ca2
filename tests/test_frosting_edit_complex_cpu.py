"""Edited-scene rendering with the complex adaptation (make_editable(use_simple_adapt=False), SURVEY.md row a21)
without a GPU: the torch restatement against golden vectors made by the reference's own source
(tests/golden/make_frosting_edit_complex_golden.py), the exported entry points and their argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frosting_edit_complex.npz")
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


def row_rel_err(a, b):
    """max over rows of max|a - b| / max|b| inside the row (rows: the leading dimension)."""
    a, b = a.reshape(a.shape[0], -1).double(), b.reshape(b.shape[0], -1).double()
    if a.shape[0] == 0:
        return 0.0
    return float(((a - b).abs().max(dim=1).values / b.abs().max(dim=1).values.clamp_min(1e-30)).max())


def check_against_golden(out, g, canonical=None, cell_T=None):
    """Scales 1e-5 relative per row, rotations as matrices 1e-5, canonical / cell transforms 1e-5 relative per matrix
    (edited rows); shell, positions, opacities and colours at the simple golden's bars."""
    ref = {k[len("out_"):]: torch.from_numpy(v) for k, v in g.items() if k.startswith("out_")}
    for k in ("inner", "outer", "means3D"):
        assert rel_err(out[k].cpu(), ref[k]) <= 1e-5, k
    assert row_rel_err(out["scales"].cpu(), ref["scales"]) <= 1e-5
    assert torch.equal(out["opacities"].cpu() == 0, ref["opacities"] == 0)
    assert (out["opacities"].cpu() - ref["opacities"]).abs().max() <= 1e-6
    m = scenes.quaternion_to_matrix(out["rotations"].cpu().double())
    mr = scenes.quaternion_to_matrix(ref["rotations"].double())
    assert (m - mr).abs().max() <= 1e-5
    assert (out["colors_precomp"].cpu() - ref["colors"]).abs().max() <= 1e-5
    em = torch.from_numpy(g["edition_mask"]).bool()
    gem = em[torch.from_numpy(g["cells"])]
    if canonical is not None:
        assert row_rel_err(canonical.cpu()[gem], ref["canonical"][gem]) <= 1e-5
    if cell_T is not None:
        assert row_rel_err(cell_T.cpu()[em], ref["cell_T"][em]) <= 1e-5


@pytest.mark.parametrize("name", CASES)
def test_restatement_matches_reference_source(name):
    g, params = golden_case(name)
    t = lambda k: torch.from_numpy(g[k])
    canonical, _ = scenes.complex_canonical_transforms(params, t("ref_verts"), t("faces"), t("cells"),
                                                       t("edition_mask"), str(g["rescaling"]))
    out = restated(g, params, adaptation="complex")
    check_against_golden(out, g, canonical=canonical, cell_T=out["cell_T"])
    assert torch.equal(restated(g, params, adaptation="complex", canonical=canonical)["scales"], out["scales"])
    # the complex rule is not the simple one on this deformed frame
    simple = restated(g, params)
    em = t("edition_mask").bool()
    gem = em[t("cells")]
    assert (simple["scales"][:gem.shape[0]][gem] - out["scales"][:gem.shape[0]][gem]).abs().max() > 1e-3
    ref_op = t("out_opacities")
    assert 0 < int((ref_op == 0).sum()) < ref_op.shape[0]


def test_golden_cases_cover_the_issue_matrix():
    seen = set()
    for name in CASES:
        g, params = golden_case(name)
        seen.add((str(g["rescaling"]), bool(g["edition_mask"].all()), "bg_points" in params, int(g["sh_degree"])))
        em = g["edition_mask"].astype(bool)
        gem = em[g["cells"]]
        assert np.abs(g["out_canonical"][gem]).max(axis=(1, 2)).min() > 0
        assert not np.any(g["out_canonical"][~gem]) and not np.any(g["out_cell_T"][~em])
    assert {s[0] for s in seen} == {"median", "triangle"}
    assert {s[1] for s in seen} == {True, False}
    assert {s[2] for s in seen} == {True, False}
    assert {s[3] for s in seen} == {1, 3}


def test_simple_adaptation_is_unchanged():
    from tests.test_frosting_edit_cpu import golden_case as simple_case
    for name in CASES:
        g, params = simple_case(name)
        a, b = restated(g, params), restated(g, params, adaptation="simple")
        assert a.keys() == b.keys() and "cell_T" not in a
        for k in a:
            assert torch.equal(a[k], b[k]), k
    with pytest.raises(ValueError, match="not recognized"):
        restated(g, params, adaptation="affine")


def test_unedited_frame_gives_back_the_gaussians():
    g, params = golden_case("median_full_bg_d3")
    t = lambda k: torch.from_numpy(g[k])
    g = dict(g, verts=g["ref_verts"])
    out = restated(g, params, adaptation="complex")
    P = params["quats"].shape[0]
    assert row_rel_err(out["scales"][:P], torch.exp(params["log_scales"])) <= 1e-5
    m = scenes.quaternion_to_matrix(out["rotations"][:P].double())
    mr = scenes.quaternion_to_matrix(torch.nn.functional.normalize(params["quats"], dim=-1).double())
    assert (m - mr).abs().max() <= 1e-5
    _, T_ref = scenes.complex_canonical_transforms(params, t("ref_verts"), t("faces"), t("cells"), t("edition_mask"))
    assert torch.equal(T_ref, out["cell_T"])


def test_degenerate_edited_face_is_singular():
    g, params = golden_case("triangle_partial_d1")
    t = lambda k: torch.from_numpy(g[k])
    verts, faces, cells = t("ref_verts").clone(), t("faces").long(), t("cells")
    em = t("edition_mask").bool()
    f = int(cells[em[cells]][0])
    # zero area: v1 onto v0.  Then a = 0, its orthogonalised copy and the normal are 0, and the fix-up's c1 x c2 is 0
    # too: T stays singular.  (A face collapsed to a point gives NaN axes in the reference, not a singular solve.)
    verts[faces[f, 1]] = verts[faces[f, 0]].clone()
    T = scenes.cell_transformations(verts, faces, em, "triangle", fix_singular=True)
    assert not torch.any(T[f][:, 0]) and not torch.any(T[f][:, 2]) and torch.any(T[f][:, 1])
    with pytest.raises(RuntimeError, match="singular"):
        scenes.complex_canonical_transforms(params, verts, faces, cells, em, "triangle")


def test_complex_entry_points_are_exported():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_frosting_edit_complex_capture", "fb200_frosting_edit_attributes_complex"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert fb.FrostingEditComplex is not None and issubclass(fb.FrostingEditComplex, fb.FrostingEdit)


def _edit_struct(**kw):
    d = C.c_void_p(0x1000)
    f = dict(n_verts=4, n_faces=2, rescaling=_lib.RESCALE_MEDIAN, n_edited=2, deformation_threshold=2.0)
    for n, _ in _lib.FrostingEdit._fields_[5:]:
        f[n] = d
    f.update(kw)
    return _lib.FrostingEdit(**f)


def _params_block(**kw):
    d = C.c_void_p(0x1000)
    f = dict(P=10, n_verts=4, n_faces=2, sh_rest=3, d_bary_logits=d, d_cells=d, d_faces=d, d_inner_verts=d,
             d_outer_verts=d, d_opacity_logits=d, d_log_scales=d, d_quats=d, d_sh_dc=d, d_sh_rest=d)
    f.update(kw)
    return _lib.FrostingParams(**f)


def test_complex_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    e, fp = _edit_struct(), _params_block()
    # capture
    assert L.fb200_frosting_edit_complex_capture(None, C.byref(fp), d, d, d, None) == -1
    assert b"null" in L.fb200_last_error()
    assert L.fb200_frosting_edit_complex_capture(C.byref(_edit_struct(rescaling=7)), C.byref(fp), d, d, d, None) == -1
    assert b"rescaling" in L.fb200_last_error()
    assert L.fb200_frosting_edit_complex_capture(C.byref(e), C.byref(_params_block(n_faces=3)), d, d, d, None) == -1
    assert b"does not match" in L.fb200_last_error()
    assert L.fb200_frosting_edit_complex_capture(C.byref(e), C.byref(fp), None, d, d, None) == -1
    assert b"missing cell transforms" in L.fb200_last_error()
    assert L.fb200_frosting_edit_complex_capture(C.byref(e), C.byref(fp), d, None, d, None) == -1
    assert b"missing canonical transforms" in L.fb200_last_error()
    assert L.fb200_frosting_edit_complex_capture(C.byref(e), C.byref(fp), d, d, None, None) == -1
    assert b"singular-cell counter" in L.fb200_last_error()
    # per frame: the simple entry point's checks, then the two tables
    outs = [d] * 5
    call = lambda e, fp, deg, canon, cell: L.fb200_frosting_edit_attributes_complex(
        C.byref(e), C.byref(fp), deg, d, None, canon, cell, *outs, None)
    assert call(e, _params_block(n_faces=3), 1, d, d) == -1 and b"does not match" in L.fb200_last_error()
    assert call(e, fp, 3, d, d) == -1 and b"sh_degree" in L.fb200_last_error()
    assert call(e, fp, 1, None, d) == -1 and b"missing canonical transforms" in L.fb200_last_error()
    assert call(e, fp, 1, d, None) == -1 and b"missing cell transforms" in L.fb200_last_error()
    assert L.fb200_frosting_edit_attributes_complex(C.byref(e), C.byref(fp), 1, d, None, d, d, d, d, d,
                                                    C.c_void_p(0x1004), d, None) == -1
    assert b"16-byte aligned" in L.fb200_last_error()


def test_python_surface_rejects_cpu_tensors():
    from frosting_b200.edit import FrostingEdit, FrostingEditComplex
    v = torch.zeros(3, 3)
    f = torch.tensor([[0, 1, 2]])
    with pytest.raises(NotImplementedError, match="FrostingEditComplex"):
        FrostingEdit(v, f, torch.zeros(1, dtype=torch.long), torch.zeros(3), torch.zeros(3), adaptation="complex")
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        FrostingEditComplex({}, v, f, torch.zeros(1, dtype=torch.long), torch.zeros(3), torch.zeros(3))
