"""Textured base mesh of a trained Frosting model -- host side of csrc/texture.cu.

Frosting ends every default training run (refine.py's `export_obj`) and scripts/extract_frosting_textured_mesh.py with
`compute_textured_mesh_for_frosting_mesh` (frosting_utils/texture.py:11-181): render every training view at SH degree 0,
splat each pixel's colour onto the UV texel its barycentrics land on and average, then fill the untouched texels with
their face's colour.  The OBJ it writes is what a user opens in Blender to edit or rig the scene.  Here:

    baker = TextureBaker(faces, cells, sh_dc, n_verts, square_size)     # accumulators and winner slots, once
    baker.add_view(image, pix_to_face, bary)                            # per view: two launches
    verts_uvs, faces_uvs, texture_map = baker.finish()                  # one launch

or the whole function, `compute_textured_mesh(params, mesh, cameras, ...)`, and `write_textured_obj` for OBJ + MTL + PNG
without pytorch3d or PIL.  Per view the reference keeps ONE pixel per face and texel (`acc[idx] = acc[idx] + colors`
with duplicate indices); here it is the last hit pixel in row-major order, the CPU's outcome, so bakes are deterministic
and equal the reference run on the CPU bit for bit.  Forward only.
"""
import ctypes as C
import os
import struct
import zlib

import numpy as np
import torch

from . import _lib
from . import rasterizer as R
from ._lib import ptr, stream
from .frosting_render import FrostingBlock
from .mesh import rasterize_mesh
from .rasterizer import GaussianRasterizationSettings
from .scenes import texture_uv_layout


def mesh_bary(verts, faces, full_proj_transform, pix_to_face):
    """Perspective-correct barycentrics [H,W,3] of the faces `pix_to_face` [H,W] (rasterize_mesh's, same verts, faces
    and camera): what mesh._barycentrics and MeshRasterizer.forward give, (u, v, 1 - (u + v)), and (0, 0, 1) where no
    face is hit."""
    if not verts.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    dev = verts.device
    verts = verts.to(torch.float32).contiguous()
    faces = faces.to(device=dev, dtype=torch.int32).contiguous()
    proj = full_proj_transform.to(device=dev, dtype=torch.float32).contiguous()
    p2f = pix_to_face.to(device=dev, dtype=torch.int32).contiguous()
    if p2f.dim() != 2:
        raise ValueError("pix_to_face must be [H, W]")
    H, W = p2f.shape
    bary = torch.empty((H, W, 3), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().fb200_mesh_barycentrics(verts.shape[0], faces.shape[0], ptr(verts), ptr(faces), ptr(proj),
                                                      W, H, ptr(p2f), ptr(bary), stream(dev)))
    return bary


class TextureBaker:
    """One texture bake on the device.

    faces [F,3] (the base mesh, F >= 1), cells [P] (each mesh-bound Gaussian's face, Frosting's _point_cell_indices),
    sh_dc [P,1,3] or [P,3], n_verts (to check the faces), square_size >= 3 (texels per UV square side).  Holds the fp32
    accumulators (16 B per face and per texel) and the winner slots (4 B each); T = square_size * (int(sqrt(F//2+1)) + 1)
    -- at 1 M faces and square 8, T = 5664: 32 M texels, 640 MB."""

    def __init__(self, faces, cells, sh_dc, n_verts, square_size=10):
        if int(square_size) < 3:
            raise ValueError("square_size must be >= 3")
        if not faces.is_cuda:
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        dev = faces.device
        if faces.dim() != 2 or faces.shape[1] != 3 or faces.shape[0] < 1:
            raise ValueError("faces must be [F, 3] with F >= 1")
        F = faces.shape[0]
        if int(faces.min()) < 0 or int(faces.max()) >= int(n_verts):
            raise ValueError(f"faces index outside the {int(n_verts)} vertices")
        cells = cells.to(device=dev, dtype=torch.int64).reshape(-1)
        P = cells.shape[0]
        sh_dc = sh_dc.to(device=dev, dtype=torch.float32).reshape(-1, 3).contiguous()
        if sh_dc.shape[0] != P:
            raise ValueError("sh_dc must hold one row per entry of cells")
        if P and (int(cells.min()) < 0 or int(cells.max()) >= F):
            raise ValueError(f"cells index outside the {F} faces")
        self.device, self.n_faces, self.square_size = dev, F, int(square_size)
        self.faces = faces.to(torch.int32).contiguous()
        self.verts_uvs, self.faces_uvs, n, T = texture_uv_layout(F, self.square_size, dev)
        self.texture_size = T
        # face -> Gaussian CSR in ascending Gaussian order (the order the CPU index_add_ adds in)
        self.cell_points = torch.sort(cells, stable=True).indices.to(torch.int32)
        self.cell_offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev),
                                       torch.bincount(cells, minlength=F).cumsum(0)]).to(torch.int32)
        self.sh_dc = sh_dc
        self.face_sh = torch.empty((F, 3), dtype=torch.float32, device=dev)
        self.face_acc = torch.zeros((F, 4), dtype=torch.float32, device=dev)
        self.texel_acc = torch.zeros((T * T, 4), dtype=torch.float32, device=dev)
        self.face_winner = torch.full((F,), -1, dtype=torch.int32, device=dev)
        self.texel_winner = torch.full((T * T,), -1, dtype=torch.int32, device=dev)
        self._st = _lib.Texture(
            n_faces=F, n_points=P, square_size=self.square_size, n_square_per_axis=n, texture_size=T,
            d_cell_offsets=ptr(self.cell_offsets), d_cell_points=ptr(self.cell_points), d_sh_dc=ptr(self.sh_dc),
            d_face_sh=ptr(self.face_sh), d_face_acc=ptr(self.face_acc), d_texel_acc=ptr(self.texel_acc),
            d_face_winner=ptr(self.face_winner), d_texel_winner=ptr(self.texel_winner))
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_texture_face_sh_colours(C.byref(self._st), stream(dev)))

    def add_view(self, image, pix_to_face, bary):
        """One view: image [H,W,3] (the render; nan_to_num and clamp(0, 1) are applied in the kernel), pix_to_face
        [H,W] int32 (-1: background), bary [H,W,3] (mesh_bary's).  Stream-ordered, no host read-back."""
        dev = self.device
        p2f = pix_to_face.to(device=dev, dtype=torch.int32).contiguous()
        if p2f.dim() != 2:
            raise ValueError("pix_to_face must be [H, W]")
        H, W = p2f.shape
        image = image.to(device=dev, dtype=torch.float32).contiguous()
        bary = bary.to(device=dev, dtype=torch.float32).contiguous()
        if tuple(image.shape) != (H, W, 3) or tuple(bary.shape) != (H, W, 3):
            raise ValueError(f"image and bary must be [{H}, {W}, 3] like pix_to_face")
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_texture_add_view(C.byref(self._st), ptr(image), ptr(p2f), ptr(bary), W, H,
                                                         stream(dev)))

    def finish(self):
        """(verts_uvs [6n^2,2], faces_uvs [F,3], texture_map [T,T,3]) as TexturesUV receives them."""
        T = self.texture_size
        texture = torch.empty((T, T, 3), dtype=torch.float32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().fb200_texture_finish(C.byref(self._st), ptr(texture), stream(self.device)))
        return self.verts_uvs, self.faces_uvs, texture


def _camera_list(cameras):
    return list(cameras.gs_cameras) if hasattr(cameras, "gs_cameras") else list(cameras)


def _settings(cam, sh_degree, bg, dev):
    """GaussianRasterizationSettings of a GSCamera-like camera, as render_image_gaussian_rasterizer builds them."""
    tanfovx = getattr(cam, "tanfovx", None)
    tanfovy = getattr(cam, "tanfovy", None)
    if tanfovx is None:
        tanfovx, tanfovy = float(np.tan(cam.FoVx * 0.5)), float(np.tan(cam.FoVy * 0.5))
    return GaussianRasterizationSettings(
        image_height=int(cam.image_height), image_width=int(cam.image_width), tanfovx=tanfovx, tanfovy=tanfovy,
        bg=bg, scale_modifier=1.0, viewmatrix=cam.world_view_transform.to(dev),
        projmatrix=cam.full_proj_transform.to(dev), sh_degree=sh_degree, campos=cam.camera_center.to(dev),
        prefiltered=False, debug=False)


def render_view(params, mesh, raster_settings, face_visible=None):
    """frosting_render's image [3,H,W], forward only, with the binning buffer sized from this view's own tile-instance
    count (the two-phase forward: one host wait per view, where the reference's rasterizer blocks too).  The speculated
    capacity of frosting_render can overflow on one view of a camera ring and only reports it at the next call; a bake
    must never take such a frame."""
    color, _, _, _ = R._launch_forward(None, None, None, None, None, None, None, raster_settings, None, exact=True,
                                       frosting=FrostingBlock(params, mesh, face_visible))
    return color


@torch.no_grad()
def compute_textured_mesh(params, mesh, cameras, square_size=10, n_sh=0, bg_color=(0., 0., 0.),
                          use_occlusion_culling=False):
    """compute_textured_mesh_for_frosting_mesh (texture.py:11-181) on the device.

    params / mesh: the dicts of frosting_render (mesh["verts"] / ["faces"] the base mesh, ["cells"] the Gaussians'
    faces); background Gaussians are rendered when params has them.  cameras: a list of GSCamera-like cameras or a
    wrapper with .gs_cameras.  Per camera: one rasterize_mesh of the base mesh (pix_to_face and, with occlusion culling,
    the visible faces), the frosting render at SH degree n_sh over bg_color (render_view), mesh_bary, add_view.
    Returns dict(verts, faces, verts_uvs, faces_uvs, texture_map) -- write_textured_obj(path, **result) saves it."""
    if int(square_size) < 3:
        raise ValueError("square_size must be >= 3")
    verts, faces = mesh["verts"].float().contiguous(), mesh["faces"].int().contiguous()
    dev = verts.device
    baker = TextureBaker(faces, mesh["cells"], params["sh_dc"], verts.shape[0], square_size)
    bg = torch.tensor(bg_color, dtype=torch.float32, device=dev)
    for cam in _camera_list(cameras):
        H, W = int(cam.image_height), int(cam.image_width)
        p2f, face_visible, _ = rasterize_mesh(verts, faces, cam.full_proj_transform, H, W)
        img = render_view(params, mesh, _settings(cam, n_sh, bg, dev),
                          face_visible=face_visible if use_occlusion_culling else None)
        bary = mesh_bary(verts, faces, cam.full_proj_transform, p2f)
        baker.add_view(img.permute(1, 2, 0), p2f, bary)
    verts_uvs, faces_uvs, texture_map = baker.finish()
    return dict(verts=verts, faces=faces, verts_uvs=verts_uvs, faces_uvs=faces_uvs, texture_map=texture_map)


def _png_chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def encode_png(rgb):
    """8-bit RGB PNG bytes of a uint8 [H,W,3] array (filter 0 on every row, zlib-compressed)."""
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    H, W, _ = rgb.shape
    raw = np.concatenate([np.zeros((H, 1), np.uint8), rgb.reshape(H, W * 3)], axis=1)
    return (b"\x89PNG\r\n\x1a\n" + _png_chunk(b"IHDR", struct.pack(">IIBBBBB", W, H, 8, 2, 0, 0, 0)) +
            _png_chunk(b"IDAT", zlib.compress(raw.tobytes(), 6)) + _png_chunk(b"IEND", b""))


def write_textured_obj(path, verts, faces, verts_uvs, faces_uvs, texture_map):
    """Writes `path` (OBJ: mtllib / usemtl, v, vt, f v/vt), its .mtl (map_Kd) and its .png beside it.  The PNG holds
    uint8(clamp(x, 0, 1) * 255) of texture_map [T,T,3] (NaN as 0), rows as stored (row 0 at the top, v = 1).  Returns the
    three paths."""
    stem = os.path.splitext(path)[0]
    name = os.path.basename(stem)
    mtl_path, png_path = stem + ".mtl", stem + ".png"
    v = verts.detach().float().cpu().numpy().reshape(-1, 3)
    vt = verts_uvs.detach().float().cpu().numpy().reshape(-1, 2)
    f = faces.detach().cpu().numpy().astype(np.int64).reshape(-1, 3) + 1
    ft = faces_uvs.detach().cpu().numpy().astype(np.int64).reshape(-1, 3) + 1
    fi = np.stack([f, ft], axis=2).reshape(-1)
    with open(path, "w") as out:
        out.write(f"mtllib {name}.mtl\nusemtl mesh\n")
        out.write(("v %.6f %.6f %.6f\n" * v.shape[0]) % tuple(v.ravel().tolist()))
        out.write(("vt %.6f %.6f\n" * vt.shape[0]) % tuple(vt.ravel().tolist()))
        out.write(("f %d/%d %d/%d %d/%d\n" * f.shape[0]) % tuple(fi.tolist()))
    with open(mtl_path, "w") as out:
        out.write(f"newmtl mesh\nmap_Kd {name}.png\nKa 1.000 1.000 1.000\nKd 1.000 1.000 1.000\n"
                  "Ks 0.000 0.000 0.000\nNs 0.0\n")
    tex = texture_map.detach().float().nan_to_num(0.0).clamp(0, 1).mul(255).to(torch.uint8).cpu().numpy()
    with open(png_path, "wb") as out:
        out.write(encode_png(tex))
    return path, mtl_path, png_path
