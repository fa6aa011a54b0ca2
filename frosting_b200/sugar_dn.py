"""SuGaR's depth-normal consistency of the coarse `dn_consistency` trainer (SURVEY.md row 17) -- host side of
csrc/sugar_dn.cu.

From iteration 9 001 on, frosting_trainers/coarse_density_and_dn_consistency.py:646-657 renders depth and camera-facing
normals in a second rasterizer call (frosting_scene/sugar_model.py:2343-2387) and adds 0.05 times the consistency
between the rendered normals and the normals of the rendered depth (:17-95).  Here the features ride in the colour
frame's traversal as the rasterizer's three extra channels (background 0), so the step renders once:

    feats = depth_normal_features(sugar.points, sugar.scaling, sugar.quaternions, raster_settings)
    rgb, radii, dn = rasterizer(..., extra_features=feats)
    loss = l1_dssim_loss(rgb, gt) + 0.05 * depth_normal_consistency(dn, raster_settings)

Both are autograd Functions over CUDA kernels with no host read-back.  `torch_reference_features` and
`torch_reference_loss` restate the reference's lines in torch for any dtype; they are the tests' oracle.
"""
import ctypes as C

import torch

from . import _lib, scenes
from ._lib import ptr, stream
from .sugar import _operand


def _camera(rs, dev, proj=False):
    view = _operand(rs.viewmatrix, "raster_settings.viewmatrix", (4, 4), dev)
    if proj:
        return view, _operand(rs.projmatrix, "raster_settings.projmatrix", (4, 4), dev)
    return view, _operand(rs.campos, "raster_settings.campos", (3,), dev)


class _DepthNormalFeatures(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, scaling, quaternions, view, campos):
        P, dev = points.shape[0], points.device
        feats = torch.empty(P, 3, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_sugar_dn_features(P, ptr(points), ptr(scaling), ptr(quaternions), ptr(view),
                                                          ptr(campos), ptr(feats), stream(dev)))
        ctx.save_for_backward(points, scaling, quaternions, view, campos)
        return feats

    @staticmethod
    def backward(ctx, g):
        points, scaling, quaternions, view, campos = ctx.saved_tensors
        P, dev = points.shape[0], points.device
        g = g.float().contiguous()
        d_points = torch.empty_like(points)
        d_quats = torch.empty_like(quaternions)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_sugar_dn_features_backward(
                P, ptr(points), ptr(scaling), ptr(quaternions), ptr(view), ptr(campos), ptr(g), ptr(d_points),
                ptr(d_quats), stream(dev)))
        # argmin is discrete: the scales get an explicit zero gradient, as autograd gives the reference's
        return d_points, torch.zeros_like(scaling), d_quats, None, None


def depth_normal_features(points, scaling, quaternions, raster_settings):
    """The [P,3] features render_depth_and_normal hands the rasterizer: view-space depth and the x, y of the
    camera-facing smallest-axis normal in pytorch3d's view frame, for the camera of `raster_settings` (its viewmatrix
    and campos).  Differentiable with respect to points [P,3] (through the depth) and quaternions [P,4] (raw, as SuGaR
    stores them); the scaling [P,3] only picks the axis and gets a zero gradient.  float32 CUDA tensors."""
    if not points.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    dev = points.device
    P = points.shape[0]
    args = [_operand(t, n, s, dev) for t, n, s in ((points, "points", (P, 3)), (scaling, "scaling", (P, 3)),
                                                   (quaternions, "quaternions", (P, 4)))]
    return _DepthNormalFeatures.apply(*args, *_camera(raster_settings, dev))


class _DepthNormalConsistency(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dn, view, proj):
        H, W, dev = dn.shape[1], dn.shape[2], dn.device
        L = _lib.lib()
        partials = torch.empty(L.fb200_sugar_dn_partials(H, W), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(L.fb200_sugar_dn_loss_forward(ptr(dn), H, W, ptr(view), ptr(proj), ptr(partials), ptr(loss),
                                                     stream(dev)))
        ctx.save_for_backward(dn, view, proj)
        return loss

    @staticmethod
    def backward(ctx, g):
        dn, view, proj = ctx.saved_tensors
        H, W, dev = dn.shape[1], dn.shape[2], dn.device
        g = g.float().reshape(1).contiguous()
        d_dn = torch.empty_like(dn)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_sugar_dn_loss_backward(ptr(dn), H, W, ptr(view), ptr(proj), ptr(g),
                                                               ptr(d_dn), stream(dev)))
        return d_dn, None, None


def depth_normal_consistency(dn, raster_settings):
    """depth_normal_consistency_loss of the image render_depth_and_normal makes, unweighted: `dn` [3,H,W] is the
    rasterizer's extra-channel output for depth_normal_features (background 0) at the camera of `raster_settings`
    (its viewmatrix and projmatrix).  Mean over the pixels of 1 - (rendered normal) . (normal of the rendered depth's
    points); border pixels count 1.  H < 3 or W < 3 gives 1 and a zero gradient.  A float32 CUDA scalar,
    differentiable with respect to dn."""
    if not dn.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    dev = dn.device
    H, W = int(raster_settings.image_height), int(raster_settings.image_width)
    dn = _operand(dn, "dn (3 extra channels)", (3, H, W), dev)
    return _DepthNormalConsistency.apply(dn, *_camera(raster_settings, dev, proj=True))


def torch_reference_features(points, scaling, quaternions, viewmatrix, campos):
    """render_depth_and_normal's features (sugar_model.py:2359-2367 with get_smallest_axis, :970-975) in torch, any
    dtype: pytorch3d's view frame is diag(-1, -1, 1) times the COLMAP view frame of `viewmatrix`
    (world_view_transform), so z is the COLMAP z and the normal's x, y are negated."""
    R = scenes.quaternion_to_matrix(quaternions)
    axis = scaling.min(dim=-1)[1][..., None, None].expand(-1, 3, -1)
    n = R.gather(2, axis).squeeze(dim=2)
    n = n * torch.sign((n * (campos - points)).sum(dim=-1, keepdim=True))
    z = points @ viewmatrix[:3, 2] + viewmatrix[3, 2]
    return torch.cat([z[:, None], -(n @ viewmatrix[:3, :2])], dim=-1)


def torch_reference_loss(dn, viewmatrix, projmatrix):
    """depth_normal_consistency_loss (coarse_density_and_dn_consistency.py:17-95, scale_rendered_normals=False) of the
    image `dn` [3,H,W] with render_depth_and_normal's normal (sugar_model.py:2378-2385), in torch, any dtype, for the
    camera's world_view_transform and full_proj_transform."""
    H, W = dn.shape[1], dn.shape[2]
    depth = dn[0:1]
    normal = torch.cat([-dn[1:], -torch.sqrt(1 - torch.sum(dn[1:] ** 2, dim=0, keepdim=True).clamp_max(1.0))], dim=0)
    c2w = viewmatrix.T.inverse()
    ndc2pix = torch.tensor([[W / 2, 0, 0, W / 2], [0, H / 2, 0, H / 2], [0, 0, 0, 1]], dtype=dn.dtype,
                           device=dn.device).T
    intrins = ((c2w.T @ projmatrix) @ ndc2pix)[:3, :3].T
    gx, gy = torch.meshgrid(torch.arange(W, device=dn.device).to(dn.dtype),
                            torch.arange(H, device=dn.device).to(dn.dtype), indexing="xy")
    pix = torch.stack([gx, gy, torch.ones_like(gx)], dim=-1).reshape(-1, 3)
    rays_d = pix @ intrins.inverse().T @ c2w[:3, :3].T
    points = (depth.reshape(-1, 1) * rays_d + c2w[:3, 3]).reshape(H, W, 3)
    out = torch.zeros_like(points)
    dx = points[2:, 1:-1] - points[:-2, 1:-1]
    dy = points[1:-1, 2:] - points[1:-1, :-2]
    out[1:-1, 1:-1, :] = torch.nn.functional.normalize(torch.cross(dx, dy, dim=-1), dim=-1)
    from_depth = (out @ viewmatrix[:3, :3]).permute(2, 0, 1)
    return (1 - (normal * from_depth).sum(dim=0)).mean()
