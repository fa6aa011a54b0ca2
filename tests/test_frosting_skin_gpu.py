"""Bone skinning on the GPU: csrc/frosting_skin.cu against the reference's own source (golden vectors), against the torch
restatement at C3 size (1 M-face sphere, 64 bones), the rest pose, and an animated frame end to end -- skin, edit,
render -- against the restated chain."""
from types import SimpleNamespace

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import scenes
from frosting_b200.mesh import rasterize_mesh
from tests.test_frosting_edit_gpu import _render_attrs, c3_scene
from tests.test_frosting_skin_cpu import NO_GROUP, UNRIGGED, close, golden

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
N_BONES, N_FRAMES = 64, 8


def test_cuda_matches_reference_source():
    z, package, ref_indices = golden()
    skin = fb.FrostingSkin(package, ref_indices, ref_indices[-1], DEV)
    init = torch.from_numpy(z["base_init"]).to(DEV)
    init[UNRIGGED[0]:UNRIGGED[1]] = float("nan")
    for k, f in enumerate(z["frames"]):
        base = init.clone()
        assert skin.pose(int(f), base) is base
        torch.cuda.synchronize()
        ref = torch.from_numpy(z["out_verts"][k]).to(DEV)
        rigged = torch.cat([torch.arange(0, UNRIGGED[0]), torch.arange(UNRIGGED[1], ref_indices[-1])]).to(DEV)
        assert close(base[rigged], ref[rigged]), int(f)
        assert torch.equal(base[list(NO_GROUP)], torch.zeros(len(NO_GROUP), 3, device=DEV))
        # the unrigged range is neither read nor written: its NaNs keep their bits
        assert torch.equal(base[UNRIGGED[0]:UNRIGGED[1]].view(torch.int32), init[UNRIGGED[0]:UNRIGGED[1]].view(torch.int32))


@pytest.fixture(scope="module")
def c3():
    cam, rs, params, mesh, inner_dist, outer_dist = c3_scene()
    package, ref_indices = scenes.skinned_rig(mesh["verts"], N_BONES, N_FRAMES)
    skin = fb.FrostingSkin(package, ref_indices, mesh["verts"].shape[0], DEV)
    return SimpleNamespace(cam=cam, rs=rs, params=params, mesh=mesh, inner_dist=inner_dist, outer_dist=outer_dist,
                           package=package, ref_indices=ref_indices, skin=skin)


def test_c3_matches_restatement_and_reproduces(c3):
    verts = c3.mesh["verts"]
    assert len(c3.skin.bone_names) == N_BONES
    for f in (1, 5, N_FRAMES + 2):
        out = c3.skin.pose(f, torch.empty_like(verts))
        ref = scenes.skin_vertices(c3.package, c3.ref_indices, f, verts.clone())
        assert close(out, ref), f
        assert (out - verts).abs().max().item() > 0.05
        assert torch.equal(c3.skin.pose(f, torch.empty_like(verts)), out)


def test_rest_pose_gives_back_the_tpose(c3):
    verts = c3.mesh["verts"]
    arm = c3.package["bones"][0]["armature"]
    rest = dict(c3.package["bones"][0], armature=dict(
        arm, pose_bones={n: m[None].expand(N_FRAMES, 4, 4) for n, m in arm["rest_bones"].items()}))
    skin = fb.FrostingSkin(dict(c3.package, bones=[rest]), c3.ref_indices, verts.shape[0], DEV)
    assert close(skin.pose(3, torch.empty_like(verts)), verts)


@pytest.mark.parametrize("adaptation,culling", [("simple", False), ("complex", False), ("simple", True)])
def test_animated_frame_end_to_end(c3, adaptation, culling):
    mesh, params, rs = c3.mesh, c3.params, c3.rs
    F = mesh["faces"].shape[0]
    em = torch.rand(F, generator=torch.Generator().manual_seed(6)).to(DEV) < 0.7
    quats = torch.cat([params["quats"], params["bg_quats"]])
    orig = torch.nn.functional.normalize(
        quats + 0.2 * torch.randn(quats.shape, generator=torch.Generator().manual_seed(7)).to(DEV), dim=-1)
    f = 3
    verts = c3.skin.pose(f, mesh["verts"].clone())
    verts_r = scenes.skin_vertices(c3.package, c3.ref_indices, f, mesh["verts"].clone())
    fv = mask = canonical = None
    if culling:
        _, fv, _ = rasterize_mesh(verts, mesh["faces"], c3.cam.full_proj_transform, c3.cam.image_height,
                                  c3.cam.image_width)
        mask = fb.gaussian_render_mask(fv, mesh["cells"], orig.shape[0])
        assert 0 < int(fv.sum()) < F
    args = (mesh["verts"], mesh["faces"], mesh["cells"], c3.inner_dist, c3.outer_dist)
    if adaptation == "simple":
        edit = fb.FrostingEdit(*args, edition_mask=em, thickness_rescaling="median")
    else:
        edit = fb.FrostingEditComplex(params, *args, edition_mask=em, thickness_rescaling="median")
    with torch.no_grad():
        if adaptation == "complex":
            canonical, _ = scenes.complex_canonical_transforms(params, mesh["verts"], mesh["faces"], mesh["cells"], em,
                                                               "median")
        img, radii = fb.frosting_render_edited(params, edit, verts, rs, orig_quats=orig, face_visible=fv)
        a = edit.attributes(params, verts, rs.campos, 3, orig_quats=orig)
        ref = scenes.edited_frosting_attributes(params, mesh["verts"], mesh["faces"], mesh["cells"], c3.inner_dist,
                                                c3.outer_dist, verts_r, rs.campos, 3, edition_mask=em,
                                                thickness_rescaling="median", orig_quats=orig, adaptation=adaptation,
                                                canonical=canonical)
        img_r, radii_r = _render_attrs(ref, rs, visibility=mask)
    drop, drop_r = a["opacities"] == 0, ref["opacities"] == 0
    assert (drop != drop_r).float().mean().item() <= 1e-4
    assert int((radii > 0).sum()) > 100_000
    assert ((img - img_r).abs() > 1e-4).float().mean().item() <= 5e-3
    assert (radii == radii_r).float().mean().item() >= 0.999
    if culling:
        assert bool((radii[:mesh["cells"].shape[0]][~fv[mesh["cells"]]] == 0).all())
