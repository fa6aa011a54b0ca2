"""Texture bake on the GPU (SURVEY.md row a22): csrc/texture.cu against the reference's own source (golden vectors), the
barycentric kernel against mesh._barycentrics, compute_textured_mesh against the torch restatement run on the CPU over
the same views, reproducibility, and a C3-size bake."""
import gc
from types import SimpleNamespace

import pytest
import torch

import frosting_b200 as fb
from frosting_b200 import scenes
from frosting_b200.frosting_render import MESH_KEYS, frosting_render
from frosting_b200.mesh import _barycentrics, rasterize_mesh
from frosting_b200.texture import _settings, render_view
from tests.test_texture_cpu import SQUARE_SIZES, golden, same

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.mark.parametrize("sq", SQUARE_SIZES)
def test_baker_matches_reference_source(sq):
    z, t = golden()
    baker = fb.TextureBaker(t("faces").to(DEV), t("cells").to(DEV), t("sh_dc").to(DEV), z["verts"].shape[0], sq)
    for v in range(z["images"].shape[0]):
        baker.add_view(t("images")[v].to(DEV), t("pix_to_face")[v].to(DEV), t("bary")[v].to(DEV))
    verts_uvs, faces_uvs, texture = baker.finish()
    torch.cuda.synchronize()
    assert same(texture.cpu(), t(f"texture_{sq}"))
    assert torch.equal(verts_uvs.cpu(), t(f"verts_uvs_{sq}")) and torch.equal(faces_uvs.cpu(), t(f"faces_uvs_{sq}"))
    # every view leaves the winner slots at -1
    assert bool((baker.face_winner == -1).all()) and bool((baker.texel_winner == -1).all())


@pytest.fixture(scope="module")
def small():
    W, H = 400, 300
    params, mesh = scenes.frosting_layer(40_000, scenes.make_camera(W, H), 77, n_faces_target=20_000,
                                         n_background=5_000, device=DEV)
    cams = scenes.ring_cameras(8, W, H, radius=6.0, device=DEV)
    return SimpleNamespace(params=params, mesh=mesh, cams=cams, mesh_params={k: params[k] for k in MESH_KEYS})


def test_uv_layout_on_the_device_divides_as_the_cpu():
    for F, sq in ((37, 3), (20_001, 8), (1_000_000, 8)):
        a, _, _, _ = scenes.texture_uv_layout(F, sq, DEV)
        b, _, _, _ = scenes.texture_uv_layout(F, sq)
        assert torch.equal(a.cpu(), b)


def test_mesh_bary_matches_torch_barycentrics(small):
    verts, faces = small.mesh["verts"], small.mesh["faces"]
    F = faces.shape[0]
    verts_uv, faces_uv, _, T = scenes.texture_uv_layout(F, 8, DEV)
    n_hit = n_same = 0
    worst = 0.0
    for cam in small.cams:
        H, W = cam.image_height, cam.image_width
        p2f, _, _ = rasterize_mesh(verts, faces, cam.full_proj_transform, H, W)
        bary = fb.mesh_bary(verts, faces, cam.full_proj_transform, p2f)
        uv, _ = _barycentrics(verts, faces, cam.full_proj_transform.float(), p2f, H, W)
        ref = torch.cat([uv, 1. - uv.sum(dim=-1, keepdim=True)], dim=-1)
        hit = p2f >= 0
        assert int(hit.sum()) > 20_000
        assert torch.equal(bary[~hit], torch.tensor([0., 0., 1.], device=DEV).expand(int((~hit).sum()), 3))
        worst = max(worst, (bary[hit] - ref[hit]).abs().max().item())
        f = p2f[hit].long()
        texel = lambda b: ((verts_uv[faces_uv[f]] * b[:, :, None]).sum(dim=1) * T).int()
        n_same += int((texel(bary[hit]) == texel(ref[hit])).all(dim=1).sum())
        n_hit += int(hit.sum())
    assert worst <= 1e-6, worst
    assert n_same >= 0.9999 * n_hit, (n_same, n_hit)


def _torch_bake_over_same_views(params, mesh, cams, sq, culling):
    """The views compute_textured_mesh makes, baked by scenes.bake_texture_torch on the CPU."""
    verts, faces = mesh["verts"], mesh["faces"]
    images, p2fs, barys = [], [], []
    bg = torch.zeros(3, device=DEV)
    with torch.no_grad():
        for cam in cams:
            H, W = cam.image_height, cam.image_width
            p2f, fv, _ = rasterize_mesh(verts, faces, cam.full_proj_transform, H, W)
            img = render_view(params, mesh, _settings(cam, 0, bg, DEV), face_visible=fv if culling else None)
            images.append(img.permute(1, 2, 0).cpu())
            p2fs.append(p2f.cpu())
            barys.append(fb.mesh_bary(verts, faces, cam.full_proj_transform, p2f).cpu())
    return scenes.bake_texture_torch(faces.shape[0], mesh["cells"].cpu(), params["sh_dc"].cpu(), sq, images, p2fs,
                                     barys)


@pytest.mark.parametrize("culling,background", [(False, False), (True, False), (False, True)])
def test_compute_textured_mesh_matches_torch_bake(small, culling, background):
    params = small.params if background else small.mesh_params
    out = fb.compute_textured_mesh(params, small.mesh, small.cams, square_size=8, use_occlusion_culling=culling)
    verts_uv, faces_uv, texture = _torch_bake_over_same_views(params, small.mesh, small.cams, 8, culling)
    assert out["verts"] is small.mesh["verts"] and out["texture_map"].shape == texture.shape
    assert same(out["texture_map"].cpu(), texture)
    assert torch.equal(out["verts_uvs"].cpu(), verts_uv) and torch.equal(out["faces_uvs"].cpu(), faces_uv)
    assert not bool(texture.isnan().any())                      # every face of this scene has Gaussians


def test_render_view_is_frosting_render(small):
    for culling in (False, True):
        cam = small.cams[3]
        _, fv, _ = rasterize_mesh(small.mesh["verts"], small.mesh["faces"], cam.full_proj_transform, cam.image_height,
                                  cam.image_width)
        fv = fv if culling else None
        rs = _settings(cam, 0, torch.tensor([0.2, 0.5, 0.1], device=DEV), DEV)
        with torch.no_grad():
            img, _ = frosting_render(small.params, small.mesh, rs, face_visible=fv)
        assert torch.equal(render_view(small.params, small.mesh, rs, face_visible=fv), img)


def test_culling_and_background_change_the_bake(small):
    a = fb.compute_textured_mesh(small.mesh_params, small.mesh, small.cams, square_size=8)["texture_map"]
    b = fb.compute_textured_mesh(small.mesh_params, small.mesh, small.cams, square_size=8,
                                 use_occlusion_culling=True)["texture_map"]
    c = fb.compute_textured_mesh(small.params, small.mesh, small.cams, square_size=8)["texture_map"]
    assert not torch.equal(a, b) and not torch.equal(a, c)


def test_two_bakes_are_bit_identical(small):
    a = fb.compute_textured_mesh(small.params, small.mesh, small.cams, square_size=10)
    b = fb.compute_textured_mesh(small.params, small.mesh, small.cams, square_size=10)
    assert same(a["texture_map"], b["texture_map"])


def test_c3_bake_completes_reproduces_and_frees_its_scratch():
    W, H = 1920, 1080
    params, mesh = scenes.frosting_layer(2_000_000, scenes.make_camera(W, H), 1237, n_faces_target=1_000_000,
                                         device=DEV)
    cams = scenes.ring_cameras(16, W, H, radius=6.0, device=DEV)
    a = fb.compute_textured_mesh(params, mesh, cams, square_size=8)
    T = a["texture_map"].shape[0]
    assert T == 5664 and a["texture_map"].shape == (T, T, 3)
    assert not bool(a["texture_map"].isnan().any())
    assert 0.0 <= float(a["texture_map"].min()) and float(a["texture_map"].max()) <= 1.0
    # the second bake: nothing but its outputs stays allocated (the first one has warmed the renderer's caches)
    gc.collect()
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(DEV)
    b = fb.compute_textured_mesh(params, mesh, cams, square_size=8)
    torch.cuda.synchronize()
    after = torch.cuda.memory_allocated(DEV)
    out_bytes = sum(b[k].numel() * b[k].element_size() for k in ("verts_uvs", "faces_uvs", "texture_map"))
    # the caching allocator may hand out a block up to 1 MB larger than asked; a scratch array left behind is >= 8 MB
    assert out_bytes <= after - before <= out_bytes + 3 * 2 ** 20, (after - before, out_bytes)
    assert same(a["texture_map"], b["texture_map"])
