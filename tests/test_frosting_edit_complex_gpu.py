"""Edited-scene rendering with the complex adaptation on the GPU (SURVEY.md row a21): csrc/frosting_edit.cu against the
reference's own source (golden vectors) and against the torch restatement + rasterizer at C3 size; unedited frames,
reproducibility, culling, singular cells, and the simple adaptation's outputs pinned from before the complex one."""
import hashlib

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import scenes
from tests.test_frosting_edit_complex_cpu import CASES, check_against_golden, golden_case, row_rel_err

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _edit_from_golden(g, params):
    t = lambda k: torch.from_numpy(g[k]).to(DEV)
    edit = fb.FrostingEditComplex(params, t("ref_verts"), t("faces"), t("cells"), t("inner_dist"), t("outer_dist"),
                                  edition_mask=t("edition_mask"), thickness_rescaling=str(g["rescaling"]))
    return edit, t


@pytest.mark.parametrize("name", CASES)
def test_cuda_attributes_match_reference_source(name):
    g, params = golden_case(name)
    params_d = {k: v.to(DEV) for k, v in params.items()}
    edit, t = _edit_from_golden(g, params_d)
    canonical = edit.canonical.clone()
    out = edit.attributes(params_d, t("verts"), t("campos"), int(g["sh_degree"]), orig_quats=t("orig_quats"))
    torch.cuda.synchronize()
    check_against_golden(out, g, canonical=canonical, cell_T=edit.cell_T)
    # the cell pass follows the reference's operation order: the CPU restatement's cell transforms to 1e-6
    tc = lambda k: torch.from_numpy(g[k])
    em = tc("edition_mask").bool()
    T = scenes.cell_transformations(tc("verts"), tc("faces"), em, str(g["rescaling"]))
    assert row_rel_err(edit.cell_T.cpu()[em], T[em]) <= 1e-6


def _c3_scene(n_bg=100_000):
    from tests.test_frosting_edit_gpu import c3_scene
    return c3_scene(n_bg)


def _render(a, rs, visibility=None):
    from tests.test_frosting_edit_gpu import _render_attrs
    return _render_attrs(a, rs, visibility)


def _qa_gap(M):
    """Relative gap between the two largest matrix_to_quaternion candidate magnitudes of M / column norms."""
    R = M / M.norm(dim=-2, keepdim=True).clamp_min(1e-10)
    m00, m11, m22 = R[:, 0, 0], R[:, 1, 1], R[:, 2, 2]
    qa = torch.stack([1 + m00 + m11 + m22, 1 + m00 - m11 - m22, 1 - m00 + m11 - m22, 1 - m00 - m11 + m22], -1)
    qa = qa.clamp_min(0).sqrt().sort(dim=-1, descending=True).values
    return (qa[:, 0] - qa[:, 1]) / qa[:, 0].clamp_min(1e-30)


@pytest.mark.parametrize("rescaling", ["median", "triangle"])
def test_c3_complex_frame_matches_restatement(rescaling):
    cam, rs, params, mesh, inner_dist, outer_dist = _c3_scene()
    F = mesh["faces"].shape[0]
    em = torch.rand(F, generator=torch.Generator().manual_seed(6)).to(DEV) < 0.7
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(quats + 0.2 * torch.randn_like(quats), dim=-1)
    verts = scenes.deform_base(mesh["verts"], 0.8)
    edit = fb.FrostingEditComplex(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist,
                                  edition_mask=em, thickness_rescaling=rescaling)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
        a = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
        C, _ = scenes.complex_canonical_transforms(params, mesh["verts"], mesh["faces"], mesh["cells"], em, rescaling)
        ref = scenes.edited_frosting_attributes(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist,
                                                outer_dist, verts, rs.campos, 3, edition_mask=em,
                                                thickness_rescaling=rescaling, orig_quats=orig, adaptation="complex",
                                                canonical=C)
        img_r, radii_r = _render(ref, rs)
    P = mesh["cells"].shape[0]
    gem = em[mesh["cells"]]
    n_edited = int(gem.sum())
    # shell and positions as the simple path; drop flags may differ on faces at the stretch threshold
    drop, drop_r = a["opacities"] == 0, ref["opacities"] == 0
    assert (drop != drop_r).float().mean().item() <= 1e-4
    same = (drop == drop_r)[:, 0]
    for k in ("inner", "outer", "means3D"):
        x, y = (a[k], ref[k]) if k in ("inner", "outer") else (a[k][same], ref[k][same])
        assert ((x - y).abs().max() / y.abs().max()).item() <= 1e-5, k
    # unedited rows: exp / normalize, as the simple path
    un = torch.cat([~gem, torch.ones(a["scales"].shape[0] - P, dtype=torch.bool, device=DEV)])
    assert row_rel_err(a["scales"][un], ref["scales"][un]) <= 1e-5
    # edited rows: scales per row and rotation matrices at 2e-3, save rows at a matrix_to_quaternion candidate tie or
    # on an ill-conditioned cell, which are counted
    s_err = ((a["scales"][:P][gem] - ref["scales"][:P][gem]).abs().max(dim=1).values
             / ref["scales"][:P][gem].abs().max(dim=1).values.clamp_min(1e-30))
    r_err = (scenes.quaternion_to_matrix(a["rotations"][:P][gem].double())
             - scenes.quaternion_to_matrix(ref["rotations"][:P][gem].double())).abs().amax(dim=(1, 2))
    bad = ((s_err > 2e-3) | (r_err > 2e-3)).nonzero()[:, 0]
    Tc = ref["cell_T"][mesh["cells"][gem][bad]]
    tie = _qa_gap(Tc @ C[gem][bad]) <= 1e-4
    ill = torch.linalg.cond(Tc.double()) > 1e4
    excluded = tie | ill
    print(f"\n{rescaling}: edited rows {n_edited}, scale max rel {s_err.max().item():.3g} "
          f"(p99.99 {s_err.sort().values[int(0.9999 * (n_edited - 1))].item():.3g}), "
          f"rotation max abs {r_err.max().item():.3g}, over 2e-3 {bad.numel()} (ties {int(tie.sum())}, "
          f"ill-conditioned {int(ill.sum())})")
    assert bool(excluded.all())
    assert bad.numel() <= 1e-4 * n_edited
    # colours: unedited rows as the simple path; edited rows follow their rotations (the image bars below)
    assert (a["colors_precomp"][un] - ref["colors_precomp"][un]).abs().max().item() <= 1e-5
    # the image bars of the simple path's C3 test
    assert int((radii > 0).sum()) > 100_000
    assert ((img - img_r).abs() > 1e-4).float().mean().item() <= 5e-3
    assert (radii == radii_r).float().mean().item() >= 0.999


def test_unedited_frame_gives_back_the_gaussians():
    g, params = golden_case("median_full_bg_d3")
    params = {k: v.to(DEV) for k, v in params.items()}
    edit, t = _edit_from_golden(g, params)
    T_ref = edit.cell_T.clone()
    out = edit.attributes(params, t("ref_verts"), t("campos"), int(g["sh_degree"]), orig_quats=t("orig_quats"))
    assert torch.equal(edit.cell_T, T_ref)
    P = params["quats"].shape[0]
    G = scenes.quaternion_to_matrix(torch.nn.functional.normalize(params["quats"], dim=-1))
    G = G * torch.exp(params["log_scales"])[:, None, :]
    assert row_rel_err(T_ref[edit.cells] @ edit.canonical, G) <= 1e-5
    assert row_rel_err(out["scales"][:P], torch.exp(params["log_scales"])) <= 1e-5
    m = scenes.quaternion_to_matrix(out["rotations"][:P].double())
    mr = scenes.quaternion_to_matrix(torch.nn.functional.normalize(params["quats"], dim=-1).double())
    assert (m - mr).abs().max().item() <= 1e-5


def test_c3_unedited_frame_reproduces_frosting_render():
    cam, rs, params, mesh, inner_dist, outer_dist = _c3_scene(n_bg=20_000)
    edit = fb.FrostingEditComplex(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist)
    orig = torch.nn.functional.normalize(torch.cat([params["quats"], params["bg_quats"]]), dim=-1)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, mesh["verts"], rs, orig_quats=orig)
        inner, outer = edit.shell(mesh["verts"])
        img_f, radii_f = fb.frosting_render(params, dict(mesh, inner=inner, outer=outer), rs)
    assert ((img - img_f).abs() > 1e-4).float().mean().item() <= 5e-3
    assert (radii == radii_f).float().mean().item() >= 0.999


def test_complex_frames_are_bit_reproducible():
    cam, rs, params, mesh, inner_dist, outer_dist = _c3_scene(n_bg=20_000)
    edit = fb.FrostingEditComplex(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist,
                                  thickness_rescaling="triangle")
    verts = scenes.deform_base(mesh["verts"], 0.5)
    orig = torch.nn.functional.normalize(torch.cat([params["quats"], params["bg_quats"]]) + 0.1, dim=-1)
    a1 = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
    a2 = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
    for k in a1:
        assert torch.equal(a1[k], a2[k]), k
    i1, r1 = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
    i2, r2 = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
    assert torch.equal(i1, i2) and torch.equal(r1, r2)


def test_face_visible_culling_matches_mask_route():
    cam, rs, params, mesh, inner_dist, outer_dist = _c3_scene(n_bg=20_000)
    edit = fb.FrostingEditComplex(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist)
    verts = scenes.deform_base(mesh["verts"], 0.7)
    F, P = mesh["faces"].shape[0], mesh["cells"].shape[0]
    fv = (torch.rand(F, generator=torch.Generator().manual_seed(8)) < 0.6).to(DEV)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, verts, rs, face_visible=fv)
        a = edit.attributes(params, verts, rs.campos, 3)
        mask = torch.cat([fv[mesh["cells"]], torch.ones(radii.shape[0] - P, dtype=torch.bool, device=DEV)])
        img_m, radii_m = _render(a, rs, visibility=mask.to(torch.uint8))
    culled = torch.cat([~fv[mesh["cells"]], torch.zeros(radii.shape[0] - P, dtype=torch.bool, device=DEV)])
    assert int(culled.sum()) > 0 and bool((radii[culled] == 0).all())
    assert torch.equal(radii, radii_m)
    assert torch.equal(img, img_m)


def test_zero_area_edited_face_raises():
    g, params = golden_case("triangle_partial_d1")
    params = {k: v.to(DEV) for k, v in params.items()}
    t = lambda k: torch.from_numpy(g[k]).to(DEV)
    verts, faces, cells = t("ref_verts").clone(), t("faces").long(), t("cells")
    em = t("edition_mask").bool()
    f = int(cells[em[cells]][0])
    verts[faces[f, 1]] = verts[faces[f, 0]].clone()     # v1 onto v0: T keeps two zero columns after the fix-up
    n_on_f = int((cells == f).sum())
    with pytest.raises(ValueError, match="singular"):
        fb.FrostingEditComplex(params, verts, faces, cells, t("inner_dist"), t("outer_dist"), edition_mask=em,
                               thickness_rescaling="triangle")
    assert n_on_f > 0


def simple_edit_digest():
    """SHA-256 of the simple FrostingEdit's outputs on a fixed seeded scene, median and triangle rescaling."""
    W, H = 640, 360
    cam = scenes.ring_cameras(8, W, H, radius=6.0, device=DEV)[0]
    rs = scenes.settings_for(cam, 3, device=DEV)
    params, mesh = scenes.frosting_layer(200_000, scenes.make_camera(W, H), 77, n_faces_target=100_000,
                                         n_background=5_000, device=DEV)
    g = torch.Generator().manual_seed(78)
    V, F = mesh["verts"].shape[0], mesh["faces"].shape[0]
    inner_dist = (-0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(DEV)
    outer_dist = (0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(DEV)
    em = (torch.rand(F, generator=g) < 0.7).to(DEV)
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(quats + 0.2 * torch.randn(quats.shape, generator=g).to(DEV), dim=-1)
    verts = scenes.deform_base(mesh["verts"], 0.6)
    h = hashlib.sha256()
    for rescaling in ("median", "triangle"):
        edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist, edition_mask=em,
                               thickness_rescaling=rescaling)
        a = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
        for k in sorted(a):
            h.update(a[k].contiguous().cpu().numpy().tobytes())
    return h.hexdigest()


# taken on an H100 from the commit before the complex adaptation
SIMPLE_EDIT_DIGEST = "da758fb014700342a6327de2b2443c4668cd744925e5afe76356843679b863df"


def test_simple_adaptation_outputs_are_unchanged():
    assert simple_edit_digest() == SIMPLE_EDIT_DIGEST
