"""Edited-scene rendering on the GPU (SURVEY.md row a21): csrc/frosting_edit.cu against the reference's own source
(golden vectors) and against the torch restatement + rasterizer at C3 size; no-op edits, reproducibility, culling."""
import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import rasterizer as R
from frosting_b200 import scenes
from tests.test_frosting_edit_cpu import CASES, check_against_golden, golden_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _edit_from_golden(g):
    t = lambda k: torch.from_numpy(g[k]).to(DEV)
    edit = fb.FrostingEdit(t("ref_verts"), t("faces"), t("cells"), t("inner_dist"), t("outer_dist"),
                           edition_mask=t("edition_mask"), thickness_rescaling=str(g["rescaling"]))
    return edit, t


@pytest.mark.parametrize("name", CASES)
def test_cuda_attributes_match_reference_source(name):
    g, params = golden_case(name)
    params = {k: v.to(DEV) for k, v in params.items()}
    edit, t = _edit_from_golden(g)
    out = edit.attributes(params, t("verts"), t("campos"), int(g["sh_degree"]), orig_quats=t("orig_quats"))
    torch.cuda.synchronize()
    check_against_golden(out, g)
    if str(g["rescaling"]) == "median":
        em = t("edition_mask").bool()
        # the radix select returns torch.median's element of the same distances, bit for bit
        assert edit.factor[0].item() == torch.median(edit.dists[em].reshape(-1)).item()
        assert edit.ref_median.item() == torch.median(edit.ref_dists[em].reshape(-1)).item()


def c3_scene(n_bg=100_000):
    W, H = 1920, 1080
    cam = scenes.ring_cameras(8, W, H, radius=6.0, device=DEV)[0]
    rs = scenes.settings_for(cam, 3, device=DEV)
    params, mesh = scenes.frosting_layer(2_000_000, scenes.make_camera(W, H), 1237, n_faces_target=1_000_000,
                                         n_background=n_bg, device=DEV)
    g = torch.Generator().manual_seed(4)
    V = mesh["verts"].shape[0]
    inner_dist = (-0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(DEV)
    outer_dist = (0.02 * (1 + 0.2 * torch.rand(V, generator=g))).to(DEV)
    return cam, rs, params, mesh, inner_dist, outer_dist


def _render_attrs(a, rs, visibility=None):
    e = torch.Tensor([])
    color, radii, _, _ = R._launch_forward(a["means3D"], e, a["colors_precomp"], a["opacities"], a["scales"],
                                           a["rotations"], e, rs, visibility)
    return color, radii


@pytest.mark.parametrize("rescaling", ["median", "triangle"])
def test_c3_edited_frame_matches_restatement(rescaling):
    cam, rs, params, mesh, inner_dist, outer_dist = c3_scene()
    F = mesh["faces"].shape[0]
    em = torch.rand(F, generator=torch.Generator().manual_seed(6)).to(DEV) < 0.7
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(quats + 0.2 * torch.randn_like(quats), dim=-1)
    verts = scenes.deform_base(mesh["verts"], 0.8)
    edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist, edition_mask=em,
                           thickness_rescaling=rescaling)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
        a = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
        ref = scenes.edited_frosting_attributes(params, mesh["verts"], mesh["faces"], mesh["cells"], inner_dist,
                                                outer_dist, verts, rs.campos, 3, edition_mask=em,
                                                thickness_rescaling=rescaling, orig_quats=orig)
        img_r, radii_r = _render_attrs(ref, rs)
    # attributes: the golden tolerances.  A face whose stretch ratio is within an ulp of the threshold may be kept by
    # one side and dropped by the other (distances differ in the last bit): such rows are counted, not compared
    drop, drop_r = a["opacities"] == 0, ref["opacities"] == 0
    assert (drop != drop_r).float().mean().item() <= 1e-4
    same = (drop == drop_r)[:, 0]
    for k in ("inner", "outer", "means3D", "scales"):
        x, y = (a[k], ref[k]) if k in ("inner", "outer") else (a[k][same], ref[k][same])
        assert ((x - y).abs().max() / y.abs().max()).item() <= 1e-5, k
    m = scenes.quaternion_to_matrix(a["rotations"].double())
    assert (m - scenes.quaternion_to_matrix(ref["rotations"].double())).abs().max().item() <= 1e-5
    assert (a["colors_precomp"] - ref["colors_precomp"]).abs().max().item() <= 1e-5
    # image: the same attributes up to ulps; a Gaussian whose alpha sits at the 1/255 cut-off, or whose drop flag
    # flips, changes a few pixels by more
    assert int((radii > 0).sum()) > 100_000
    d = (img - img_r).abs()
    assert (d > 1e-4).float().mean().item() <= 5e-3
    assert (radii == radii_r).float().mean().item() >= 0.999


@pytest.mark.parametrize("rescaling", ["median", "triangle"])
def test_noop_edit_reproduces_frosting_render(rescaling):
    cam, rs, params, mesh, inner_dist, outer_dist = c3_scene(n_bg=20_000)
    edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist,
                           thickness_rescaling=rescaling)
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(quats, dim=-1)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, mesh["verts"], rs, orig_quats=orig)
        inner, outer = edit.shell(mesh["verts"])
    if rescaling == "median":
        assert edit.factor[1].item() == 1.0
    assert bool((edit.face_factor == 1).all()) and bool((edit.face_keep == 1).all())
    with torch.no_grad():
        img_f, radii_f = fb.frosting_render(params, dict(mesh, inner=inner, outer=outer), rs)
    assert (img - img_f).abs().max().item() <= 1e-5
    assert (radii == radii_f).float().mean().item() >= 0.999


def test_edited_frames_are_bit_reproducible():
    cam, rs, params, mesh, inner_dist, outer_dist = c3_scene(n_bg=20_000)
    edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist)
    verts = scenes.deform_base(mesh["verts"], 0.5)
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(quats + 0.1, dim=-1)
    a1 = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
    a2 = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
    for k in a1:
        assert torch.equal(a1[k], a2[k]), k
    i1, r1 = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
    i2, r2 = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig)
    assert torch.equal(i1, i2) and torch.equal(r1, r2)


def test_face_visible_culling_matches_mask_route():
    cam, rs, params, mesh, inner_dist, outer_dist = c3_scene(n_bg=20_000)
    edit = fb.FrostingEdit(mesh["verts"], mesh["faces"], mesh["cells"], inner_dist, outer_dist,
                           thickness_rescaling="triangle")
    verts = scenes.deform_base(mesh["verts"], 0.7)
    F, P = mesh["faces"].shape[0], mesh["cells"].shape[0]
    fv = (torch.rand(F, generator=torch.Generator().manual_seed(8)) < 0.6).to(DEV)
    with torch.no_grad():
        img, radii = fb.frosting_render_edited(params, edit, verts, rs, face_visible=fv)
        a = edit.attributes(params, verts, rs.campos, 3)
        mask = torch.cat([fv[mesh["cells"]], torch.ones(radii.shape[0] - P, dtype=torch.bool, device=DEV)])
        img_m, radii_m = _render_attrs(a, rs, visibility=mask.to(torch.uint8))
    culled = torch.cat([~fv[mesh["cells"]], torch.zeros(radii.shape[0] - P, dtype=torch.bool, device=DEV)])
    assert int(culled.sum()) > 0 and bool((radii[culled] == 0).all())
    assert torch.equal(radii, radii_m)
    assert torch.equal(img, img_m)
