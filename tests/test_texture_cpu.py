"""Texture bake on the CPU: the torch restatement against the reference's own source (golden vectors), the UV layout,
the new entry points' argument checks and the OBJ / MTL / PNG writer."""
import ctypes as C
import os
import struct
import zlib

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes
from frosting_b200.texture import TextureBaker, encode_png, write_textured_obj

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frosting_texture_bake.npz")
SQUARE_SIZES = (3, 8)


def golden():
    z = np.load(GOLDEN)
    return z, (lambda k: torch.from_numpy(z[k]))


def same(a, b):
    """Bit-for-bit equality, NaN positions included (a NaN's payload is not compared)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    nan = a.isnan()
    if not torch.equal(nan, b.isnan()):
        return False
    return torch.equal(a[~nan].view(torch.int32), b[~nan].view(torch.int32))


def bake_golden_torch(sq, device="cpu"):
    z, t = golden()
    return scenes.bake_texture_torch(z["faces"].shape[0], t("cells").to(device), t("sh_dc").to(device), sq,
                                     list(t("images").to(device)), list(t("pix_to_face").to(device)),
                                     list(t("bary").to(device)))


@pytest.mark.parametrize("sq", SQUARE_SIZES)
def test_restatement_matches_reference_source_bit_for_bit(sq):
    z, t = golden()
    verts_uv, faces_uv, texture = bake_golden_torch(sq)
    assert torch.equal(verts_uv, t(f"verts_uvs_{sq}")) and verts_uv.dtype == torch.float32
    assert torch.equal(faces_uv, t(f"faces_uvs_{sq}"))
    assert same(texture, t(f"texture_{sq}"))


def test_golden_covers_the_cases():
    z, t = golden()
    F = z["faces"].shape[0]
    p2f, cells = t("pix_to_face"), t("cells")
    assert F % 2 == 1
    seen = torch.zeros(F, dtype=torch.bool)
    seen[p2f[p2f >= 0].long()] = True
    has_g = torch.bincount(cells, minlength=F) > 0
    assert bool((~seen & has_g).any()) and bool((seen & ~has_g).any()) and bool((~seen & ~has_g).any())
    for v in range(p2f.shape[0]):                   # many pixels of a view share a face
        hits = p2f[v][p2f[v] >= 0]
        assert hits.numel() > 2 * hits.unique().numel()
    img = t("images")
    assert bool(img.isnan().any()) and bool(img.isinf().any()) and bool((img[img.isfinite()] < 0).any()) and \
        bool((img[img.isfinite()] > 1).any())
    # a face with neither hits nor Gaussians keeps the reference's 0 / 0
    for sq in SQUARE_SIZES:
        assert bool(t(f"texture_{sq}").isnan().any())


@pytest.mark.parametrize("sq", SQUARE_SIZES)
def test_the_last_pixel_of_a_view_wins(sq):
    """Reversing the pixel order of every view changes the bake: the rule is pinned by the golden vectors."""
    z, t = golden()
    rev = lambda x: x.flatten(0, 1).flip(0).reshape(x.shape)
    _, _, texture = scenes.bake_texture_torch(z["faces"].shape[0], t("cells"), t("sh_dc"), sq,
                                              [rev(x) for x in t("images")], [rev(x) for x in t("pix_to_face")],
                                              [rev(x) for x in t("bary")])
    assert not same(texture, t(f"texture_{sq}"))


@pytest.mark.parametrize("F,sq", [(1, 3), (2, 3), (37, 8), (1_000_000, 8)])
def test_uv_layout(F, sq):
    n = int(np.sqrt(F // 2 + 1) + 1)
    verts_uv, faces_uv, n2, T = scenes.texture_uv_layout(F, sq) if F < 10_000 else (None, None, *_layout(F, sq))
    assert n2 == n and T == sq * n and 2 * n * n >= F
    if F == 1_000_000:
        assert T == 5664
        return
    assert verts_uv.shape == (6 * n * n, 2) and torch.equal(faces_uv.reshape(-1), torch.arange(3 * F))
    # every face's corners lie in its own square (at square_size 3 one touches the far edge)
    corners = (verts_uv * T).round().long().view(n * n, 6, 2)
    ij = torch.cartesian_prod(torch.arange(n), torch.arange(n))
    rel = corners - (ij * sq)[:, None]
    assert int(rel.min()) >= 0 and int(rel.max()) <= sq


def _layout(F, sq):
    n = int(np.sqrt(F // 2 + 1) + 1)
    return n, sq * n


def test_texture_entry_points_are_bound():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_mesh_barycentrics", "fb200_texture_face_sh_colours", "fb200_texture_add_view",
              "fb200_texture_finish"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert fb.TextureBaker is TextureBaker and fb.write_textured_obj is write_textured_obj


def _texture_struct(**kw):
    d = C.c_void_p(0x1000)
    f = dict(n_faces=37, n_points=50, square_size=8, n_square_per_axis=5, texture_size=40)
    for n, _ in _lib.Texture._fields_[5:]:
        f[n] = d
    f.update(kw)
    return _lib.Texture(**f)


def test_texture_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    err = lambda: L.fb200_last_error()
    sh = lambda s: L.fb200_texture_face_sh_colours(C.byref(s) if s is not None else None, None)
    add = lambda s, img=d, p2f=d, bary=d, W=28, H=20: L.fb200_texture_add_view(
        C.byref(s) if s is not None else None, img, p2f, bary, W, H, None)
    fin = lambda s, out=d: L.fb200_texture_finish(C.byref(s) if s is not None else None, out, None)
    for call in (sh, add, fin):
        assert call(None) == -1 and b"null texture struct" in err()
        for bad in (dict(n_faces=0), dict(n_points=-1), dict(square_size=2, texture_size=10),
                    dict(n_square_per_axis=4), dict(texture_size=41), dict(n_square_per_axis=4, texture_size=32),
                    dict(n_square_per_axis=6000, texture_size=48000)):
            assert call(_texture_struct(**bad)) == -1 and b"bad extents" in err(), (call, bad)
        assert call(_texture_struct(d_cell_offsets=None)) == -1 and b"missing face table" in err()
        assert call(_texture_struct(d_sh_dc=None)) == -1 and b"missing face table" in err()
        assert call(_texture_struct(d_face_sh=None)) == -1 and b"missing face table" in err()
        assert call(_texture_struct(d_texel_winner=None)) == -1 and b"missing accumulator" in err()
        assert call(_texture_struct(d_face_acc=None)) == -1 and b"missing accumulator" in err()
        assert call(_texture_struct(d_texel_acc=C.c_void_p(0x1008))) == -1 and b"16-byte aligned" in err()
    for kw in (dict(img=None), dict(p2f=None), dict(bary=None), dict(W=0), dict(H=-1), dict(W=70000, H=70000)):
        assert add(_texture_struct(), **kw) == -1 and b"texture_add_view: bad arguments" in err(), kw
    assert fin(_texture_struct(), None) == -1 and b"missing output" in err()
    bary = lambda V=30, F=37, verts=d, faces=d, proj=d, W=28, H=20, p2f=d, out=d: L.fb200_mesh_barycentrics(
        V, F, verts, faces, proj, W, H, p2f, out, None)
    for kw in (dict(V=-1), dict(F=-1), dict(verts=None), dict(faces=None), dict(proj=None), dict(W=0), dict(H=0),
               dict(p2f=None), dict(out=None), dict(W=70000, H=70000)):
        assert bary(**kw) == -1 and b"mesh_barycentrics: bad arguments" in err(), kw


def test_python_surface_rejects_cpu_and_bad_arguments():
    z, t = golden()
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        TextureBaker(t("faces"), t("cells"), t("sh_dc"), z["verts"].shape[0], 8)
    with pytest.raises(ValueError, match="square_size"):
        TextureBaker(t("faces"), t("cells"), t("sh_dc"), z["verts"].shape[0], 2)


def _read_png(data):
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, chunks = 8, {}
    while pos < len(data):
        n, = struct.unpack(">I", data[pos:pos + 4])
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        crc, = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(kind + body) & 0xFFFFFFFF
        chunks.setdefault(kind, []).append(body)
        pos += 12 + n
    W, H, depth, colour, _, _, interlace = struct.unpack(">IIBBBBB", chunks[b"IHDR"][0])
    assert (depth, colour, interlace) == (8, 2, 0) and b"IEND" in chunks
    raw = np.frombuffer(zlib.decompress(b"".join(chunks[b"IDAT"])), np.uint8).reshape(H, 1 + 3 * W)
    assert (raw[:, 0] == 0).all()
    return raw[:, 1:].reshape(H, W, 3)


def test_encode_png_round_trips():
    rgb = np.random.default_rng(0).integers(0, 256, size=(7, 11, 3), dtype=np.uint8)
    assert np.array_equal(_read_png(encode_png(rgb)), rgb)


def test_write_textured_obj_round_trips(tmp_path):
    z, t = golden()
    verts, faces = t("verts"), t("faces")
    verts_uv, faces_uv, texture = bake_golden_torch(8)
    obj, mtl, png = write_textured_obj(str(tmp_path / "scene.obj"), verts, faces, verts_uv, faces_uv, texture)
    assert mtl == str(tmp_path / "scene.mtl") and png == str(tmp_path / "scene.png")
    v, vt, f, ft, heads = [], [], [], [], {}
    for line in open(obj):
        k, *rest = line.split()
        heads[k] = heads.get(k, 0) + 1
        if k == "v":
            v.append([float(x) for x in rest])
        elif k == "vt":
            vt.append([float(x) for x in rest])
        elif k == "f":
            pairs = [x.split("/") for x in rest]
            f.append([int(a) - 1 for a, _ in pairs])
            ft.append([int(b) - 1 for _, b in pairs])
        else:
            assert (k, rest) in (("mtllib", ["scene.mtl"]), ("usemtl", ["mesh"]))
    assert heads["mtllib"] == heads["usemtl"] == 1
    assert np.abs(np.array(v) - verts.numpy()).max() <= 5e-7 * max(1.0, float(verts.abs().max()))
    assert np.abs(np.array(vt) - verts_uv.numpy()).max() <= 5e-7
    assert np.array_equal(np.array(f), faces.numpy()) and np.array_equal(np.array(ft), faces_uv.numpy())
    lines = open(mtl).read().split("\n")
    assert "newmtl mesh" in lines and "map_Kd scene.png" in lines
    expect = (texture.nan_to_num(0.0).clamp(0, 1) * 255).to(torch.uint8).numpy()
    assert np.array_equal(_read_png(open(png, "rb").read()), expect)
