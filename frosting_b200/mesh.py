"""Mesh occlusion-culling prepass -- host side.

Mirrors, for the GSCamera path Frosting uses on its render path:
  nvdiff_rasterization            frosting_utils/nvdiffrast.py:8-58
  nvdiff_rasterization_with_pix_to_face   frosting_utils/nvdiffrast.py:61-79
  MeshRasterizer / Fragments / RasterizationSettings   frosting_utils/mesh_rasterization.py:23-172
  the render_mask construction    frosting_scene/frosting_model.py:1564-1576
with the OpenGL rasteriser replaced by the CUDA kernels in csrc/mesh_vis.cu (C ABI
fb200_mesh_visibility / fb200_gaussian_mask_from_faces).

pytorch3d is not a dependency: `mesh` is anything with verts_list()/faces_list() (a pytorch3d Meshes
works) or a (verts, faces) pair; a camera is anything with .full_proj_transform, .image_height,
.image_width (GSCamera, frosting_scene/cameras.py:142-223) or a wrapper with .gs_cameras.
"""
from typing import Optional

import torch

from . import _lib
from ._lib import ptr, stream


def _verts_faces(mesh=None, verts=None, faces=None):
    if verts is None or faces is None:
        if mesh is None:
            raise ValueError('Either mesh or verts and faces must be provided')
        if isinstance(mesh, (tuple, list)):
            v, f = mesh
        else:
            v, f = mesh.verts_list()[0], mesh.faces_list()[0]
        verts = v if verts is None else verts
        faces = f if faces is None else faces
    return verts.float().contiguous(), faces.int().contiguous()


def rasterize_mesh(verts: torch.Tensor, faces: torch.Tensor, full_proj_transform: torch.Tensor,
                   image_height: int, image_width: int, mark_last_on_bg: bool = False, work_lists: bool = True):
    """Nearest-face id per pixel and per-face visibility.

    Returns (pix_to_face int32 [H,W] with -1 for background, face_visible bool [F], zkeys int64 [H,W]).
    """
    if not verts.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    device = verts.device
    H, W = int(image_height), int(image_width)
    F = faces.shape[0]
    proj = full_proj_transform.to(device=device, dtype=torch.float32).contiguous()
    with torch.cuda.device(device):
        zbuf = torch.empty((H, W), dtype=torch.int64, device=device)
        pix_to_face = torch.empty((H, W), dtype=torch.int32, device=device)
        face_visible = torch.empty((max(F, 1),), dtype=torch.uint8, device=device)
        scratch = torch.empty((2 * F + 4,), dtype=torch.int32, device=device) if (work_lists and F) else None
        _lib.check(_lib.lib().fb200_mesh_visibility(
            verts.shape[0], F, ptr(verts) if F else None, ptr(faces) if F else None, ptr(proj), W, H, ptr(zbuf),
            ptr(pix_to_face), ptr(face_visible), int(bool(mark_last_on_bg)), ptr(scratch), stream(device)))
    return pix_to_face, face_visible[:F].bool(), zbuf


def gaussian_render_mask(face_visible: torch.Tensor, point_cell_indices: torch.Tensor, n_total: int):
    """render_mask of frosting_model.py:1564-1576: face_visible[cell] for the mesh-bound Gaussians,
    True for the trailing (n_total - len(cells)) background Gaussians.  Returns uint8 [n_total]."""
    device = face_visible.device
    n_pts = point_cell_indices.shape[0]
    n_bg = int(n_total) - n_pts
    if n_bg < 0:
        raise ValueError("n_total smaller than the number of mesh-bound Gaussians")
    fv = face_visible.to(torch.uint8).contiguous()
    cells = point_cell_indices.to(device=device, dtype=torch.int64).contiguous()
    mask = torch.empty((n_total,), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        _lib.check(_lib.lib().fb200_gaussian_mask_from_faces(
            n_pts, ptr(cells), fv.shape[0], ptr(fv) if n_pts else None, n_bg, ptr(mask), stream(device)))
    return mask


def _barycentrics(verts, faces, proj, pix_to_face, H, W):
    """Perspective-correct barycentrics (u, v of vertices 0 and 1) and z/w per pixel, in torch.
    Off the hot path (only frosting_utils/texture.py consumes them)."""
    device = verts.device
    hit = pix_to_face >= 0
    uv = torch.zeros((H, W, 2), device=device)
    zw = torch.zeros((H, W), device=device)
    if hit.any():
        ys, xs = torch.nonzero(hit, as_tuple=True)
        f = faces[pix_to_face[ys, xs].long()].long()                        # [n,3]
        clip = torch.cat([verts, torch.ones_like(verts[:, :1])], 1) @ proj  # [V,4]
        c = clip[f]                                                         # [n,3,4]
        w = c[..., 3]
        sx = (c[..., 0] / w * 0.5 + 0.5) * W
        sy = (c[..., 1] / w * 0.5 + 0.5) * H
        px, py = xs.float() + 0.5, ys.float() + 0.5

        def edge(ax, ay, bx, by):
            return (bx - ax) * (py - ay) - (by - ay) * (px - ax)
        b0 = edge(sx[:, 1], sy[:, 1], sx[:, 2], sy[:, 2])
        b1 = edge(sx[:, 2], sy[:, 2], sx[:, 0], sy[:, 0])
        b2 = edge(sx[:, 0], sy[:, 0], sx[:, 1], sy[:, 1])
        area = b0 + b1 + b2
        b = torch.stack([b0, b1, b2], 1) / area[:, None]
        pc = b / w
        pc = pc / pc.sum(1, keepdim=True)
        uv[ys, xs] = pc[:, :2]
        zw[ys, xs] = (b * (c[..., 2] / w)).sum(1)
    return uv, zw


def nvdiff_rasterization(camera, image_height: int, image_width: int, mesh=None, verts=None, faces=None,
                         return_indices_only: bool = False, glctx=None):
    """Same contract as frosting_utils/nvdiffrast.py:8-58 for a GSCamera: pix_to_face is face id + 1
    with 0 for background (batch dim of 1)."""
    verts, faces = _verts_faces(mesh, verts, faces)
    proj = camera.full_proj_transform
    p2f, _, _ = rasterize_mesh(verts, faces, proj, image_height, image_width)
    pix_to_face = (p2f + 1)[None]
    if return_indices_only:
        return pix_to_face
    uv, zw = _barycentrics(verts, faces, proj.to(verts.device).float(), p2f, image_height, image_width)
    return uv[None], zw[None], pix_to_face


def nvdiff_rasterization_with_pix_to_face(mesh, cameras, cam_idx: int = 0, glctx=None):
    cam = cameras.gs_cameras[cam_idx]
    pix_to_face = nvdiff_rasterization(cam, cam.image_height, cam.image_width, mesh=mesh, return_indices_only=True)
    return pix_to_face.unique() - 1


class RasterizationSettings:
    def __init__(self, image_size=(1080, 1920), blur_radius=0.0, faces_per_pixel=1):
        self.image_size = image_size
        self.blur_radius = blur_radius
        self.faces_per_pixel = faces_per_pixel


class Fragments:
    def __init__(self, bary_coords, zbuf, pix_to_face):
        self.bary_coords = bary_coords   # (1, height, width, 1, 3)
        self.zbuf = zbuf                 # (1, height, width, 1)
        self.pix_to_face = pix_to_face   # (1, height, width, 1)


def _pick_camera(cameras, cam_idx):
    if hasattr(cameras, "gs_cameras"):
        return cameras.gs_cameras[cam_idx]
    if isinstance(cameras, (list, tuple)):
        return cameras[cam_idx]
    if hasattr(cameras, "full_proj_transform"):
        return cameras
    raise ValueError("cameras must be either CamerasWrapper, GSCamera or list of GSCamera")


class MeshRasterizer(torch.nn.Module):
    """Drop-in for frosting_utils/mesh_rasterization.py:42-172 (GSCamera path)."""

    def __init__(self, cameras=None, raster_settings: Optional[RasterizationSettings] = None,
                 use_nvdiffrast: bool = True):
        super().__init__()
        self.use_nvdiffrast = True   # there is one backend here: the CUDA prepass
        self.cameras = cameras
        if cameras is not None:
            cam0 = _pick_camera(cameras, 0)
            self.height, self.width = cam0.image_height, cam0.image_width
            self.raster_settings = RasterizationSettings(image_size=(self.height, self.width))
        else:
            self.raster_settings = raster_settings or RasterizationSettings()
            self.height, self.width = self.raster_settings.image_size

    def forward(self, mesh, cameras=None, cam_idx=0, return_only_pix_to_face=False):
        if cameras is None:
            if self.cameras is None:
                raise ValueError("cameras must be provided either in the constructor or in the forward method")
            cameras = self.cameras
        cam = _pick_camera(cameras, cam_idx)
        height, width = cam.image_height, cam.image_width
        if return_only_pix_to_face:
            p2f = nvdiff_rasterization(cam, height, width, mesh=mesh, return_indices_only=True) - 1
            return p2f.view(1, height, width, 1)
        bary, zbuf, p2f = nvdiff_rasterization(cam, height, width, mesh=mesh)
        p2f = p2f - 1
        bary = torch.cat([bary, 1. - bary.sum(dim=-1, keepdim=True)], dim=-1)
        return Fragments(bary.view(1, height, width, 1, 3), zbuf.view(1, height, width, 1),
                         p2f.view(1, height, width, 1))
