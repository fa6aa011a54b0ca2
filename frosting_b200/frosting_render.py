"""Frosting's whole render call as ONE differentiable op (SURVEY.md row f1).

`frosting_render(params, mesh, raster_settings, face_visible)` is what `Frosting.render_image_gaussian_rasterizer` does
between its learnable parameters and the image (frosting_scene/frosting_model.py:1470-1519 attribute properties :713-799,
:1564-1586 occlusion mask and boolean gathers, :1624 means2D sink, :1649-1657 rasterizer call), with everything that exists
only to glue torch ops together removed.  The rasterizer runs in FROSTING MODE (fb200_inputs.frosting):

  * preprocess reads the learnable parameters directly: softmax barycentrics -> position, sigmoid, exp, normalize, and
    the SH row from `dc | rest` in place.  No attribute tensor is materialised -- in particular no [P,16,3] SH copy (192 B
    per Gaussian each way in the reference's `cat`) -- and no attribute kernel runs;
  * occlusion culling is the lookup `face_visible[cell[i]]` at the top of preprocess: no `_index_mask`, no `render_mask`,
    no boolean gathers of five attribute tensors and no scatter in their backward;
  * the per-Gaussian backward kernel continues the chain rule through those maps and writes the PARAMETER gradients, for
    the rendered Gaussians only (radii > 0: ~10 % of a layer).  The other rows are zero by definition: a `grad_sink` that
    understands `row_radii` (FrostingAdam's) never reads them; otherwise they are zero-filled here.

Per frame at C3 that is: preprocess -> scan / scatter / sort -> blend -> [loss] -> blend bwd -> per-Gaussian bwd.  Two
fewer kernels and ~1 GB less HBM traffic than attribute kernel + rasterizer + attribute backward.

Background Gaussians (Frosting's default for real scenes, frosting_model.py:564-591, :801-876): the six `bg_*` keys of
`params` (BG_KEYS) add free Gaussians after the mesh-bound ones, in the same frame and the same kernels.  They skip the
occlusion lookup (`render_mask`'s trailing ones, :1571-1576); radii cover all n_mesh + n_bg Gaussians and the backward
returns the background parameters' gradients too.  `frosting_render_two_step` keeps the attribute-kernel route (tests
compare the two).
"""
import ctypes as C

import torch

from . import _lib
from . import rasterizer as R
from ._lib import FrostingParams, FrostingGrads

MESH_KEYS = ("bary_logits", "opacity_logits", "log_scales", "quats", "sh_dc", "sh_rest")
# Frosting's _bg_points, _bg_opacities, _bg_scales, _bg_quaternions, _bg_sh_coordinates_dc / _rest, in this order
BG_KEYS = ("bg_points", "bg_opacity_logits", "bg_log_scales", "bg_quats", "bg_sh_dc", "bg_sh_rest")


def _p(t):
    return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())


def background_params(params):
    """The six background tensors of `params` in BG_KEYS order, or None when it has none (all six or none)."""
    have = [k in params for k in BG_KEYS]
    if not any(have):
        return None
    if not all(have):
        raise ValueError(f"background Gaussians need all of {BG_KEYS}")
    return tuple(params[k] for k in BG_KEYS)


def _params_block(bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, face_visible,
                  bg, mask=None):
    """fb200_frosting_params over the whole model: the mesh parameters and shell, the optional culling inputs and the
    background parameters `bg` (BG_KEYS order; empty: none).  Returns it, the mesh-side tensors it points into
    (parameters, inner, outer, cells, faces, face_visible, mask), the background ones (None: none) and the device."""
    if not bary_logits.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    dev = bary_logits.device
    t = [R._f32c(x, dev, "frosting parameter") for x in (bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer)]
    bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer = t
    cells = cells.to(device=dev, dtype=torch.int64).contiguous()
    faces = faces.to(device=dev, dtype=torch.int32).contiguous()
    fv = None if face_visible is None else face_visible.to(device=dev, dtype=torch.uint8).contiguous()
    m = None if mask is None else mask.to(device=dev, dtype=torch.uint8).contiguous()
    P, Rn = bary_logits.shape[0], sh_rest.shape[1]
    bg_keep = tuple(R._f32c(x, dev, "background parameter") for x in bg) if bg else None
    b = bg_keep or (None,) * 6
    n_bg = 0 if bg_keep is None else b[0].shape[0]
    if bg_keep is not None and (b[0].shape != (n_bg, 3) or b[5].shape != (n_bg, Rn, 3) or
                                any(x.shape[0] != n_bg for x in b)):
        raise RuntimeError("background parameters must be [n,3], [n], [n,3], [n,4], [n,1,3], [n,M-1,3] with the mesh "
                           "block's M")
    fp = FrostingParams(P=P, n_verts=inner.shape[0], n_faces=faces.shape[0], sh_rest=Rn,
                        d_bary_logits=_p(bary_logits), d_cells=_p(cells), d_faces=_p(faces),
                        d_inner_verts=_p(inner), d_outer_verts=_p(outer), d_opacity_logits=_p(opacity_logits),
                        d_log_scales=_p(log_scales), d_quats=_p(quats), d_sh_dc=_p(sh_dc), d_sh_rest=_p(sh_rest),
                        d_mask=_p(m), d_face_visible=_p(fv), d_radii=None,
                        n_bg=n_bg, d_bg_points=_p(b[0]), d_bg_opacity_logits=_p(b[1]), d_bg_log_scales=_p(b[2]),
                        d_bg_quats=_p(b[3]), d_bg_sh_dc=_p(b[4]), d_bg_sh_rest=_p(b[5]))
    keep = (bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, fv, m)
    return fp, keep, bg_keep, dev


def _grads_block(d, d_in, d_out, bd):
    """fb200_frosting_grads over the six mesh parameter gradients, the shell vertices' and the background ones (bd:
    six tensors, or None without background Gaussians)."""
    b = bd or (None,) * 6
    return FrostingGrads(d_bary_logits=_p(d[0]), d_inner_verts=_p(d_in), d_outer_verts=_p(d_out),
                         d_opacity_logits=_p(d[1]), d_log_scales=_p(d[2]), d_quats=_p(d[3]), d_sh_dc=_p(d[4]),
                         d_sh_rest=_p(d[5]), d_bg_points=_p(b[0]), d_bg_opacity_logits=_p(b[1]),
                         d_bg_log_scales=_p(b[2]), d_bg_quats=_p(b[3]), d_bg_sh_dc=_p(b[4]), d_bg_sh_rest=_p(b[5]))


def _grad_targets(sink, keep, dev, radii, zero_rows, bg_keep=None):
    """The six parameter-gradient tensors -- and with background Gaussians their six -- : the caller's sink (the
    optimizer's slab) or fresh ones.  Returns (mesh list, background list or None)."""
    bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest = keep[:6]
    P, Rn = bary_logits.shape[0], sh_rest.shape[1]
    o = dict(dtype=torch.float32, device=dev)
    if sink is not None:
        if hasattr(sink, "sink_once"):
            sink.sink_once(MESH_KEYS + (BG_KEYS if bg_keep is not None else ()))
        out = [sink[n] for n in MESH_KEYS]
        bout = [sink[n] for n in BG_KEYS] if bg_keep is not None else None
        for tt, ref in zip(out + (bout or []), list(keep[:6]) + list(bg_keep or ())):
            if tt.numel() != ref.numel() or not tt.is_contiguous() or tt.dtype != torch.float32 or tt.device != dev:
                raise RuntimeError("grad_sink tensors must be contiguous fp32 CUDA tensors shaped like the parameters")
        if zero_rows:
            if getattr(sink, "accepts_row_radii", False):
                # rows with radii <= 0 stay unwritten; the consumer (FrostingAdam's step) treats them as zero rows.  The
                # background groups have no row structure there: they are zero-filled and stay dense
                sink.rows_from(radii if bout is None else radii[:P], MESH_KEYS)
                for tt in bout or ():
                    tt.zero_()
            else:
                for tt in out + (bout or []):
                    tt.zero_()
        return out, bout
    make = torch.zeros if zero_rows else torch.empty
    bout = None if bg_keep is None else [make(tuple(t.shape), **o) for t in bg_keep]
    return [make((P, 6), **o), make((P,), **o), make((P, 3), **o), make((P, 4), **o), make((P, 1, 3), **o),
            make((P, Rn, 3), **o)], bout


def _returned(ctx, keep, d, d_in, d_out, bg_keep, bd):
    """autograd's gradients for (mesh parameters, shell vertices, the five non-differentiable inputs -- cells, faces and
    three per-call arguments --, background parameters)."""
    tail = (None,) * 5
    if bg_keep is not None:
        tail += (None,) * 6 if ctx.sink is not None else (bd[0], bd[1].view_as(bg_keep[1])) + tuple(bd[2:])
    if ctx.sink is not None:
        return (None, None, None, None, None, None, d_in, d_out) + tail
    d_bary, d_op, d_ls, d_q, d_dc, d_rest = d
    return (d_bary, d_op.view_as(keep[1]), d_ls, d_q, d_dc, d_rest, d_in, d_out) + tail


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


class _FrostingRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces,
                face_visible, rs, sink, *bg):
        fp, keep, bg_keep, dev = _params_block(bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner,
                                               outer, cells, faces, face_visible, bg)
        color, radii, call, _ = R._launch_forward(None, None, None, None, None, None, None, rs, None,
                                                  want_backward=True, frosting=(fp, keep, dev))
        ctx.call, ctx.sink, ctx.keep, ctx.dev, ctx.bg_keep = call, sink, keep, dev, bg_keep
        ctx.vert_grad = inner.requires_grad or outer.requires_grad
        ctx.save_for_backward(radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _):
        (radii,) = ctx.saved_tensors
        keep, dev, bg_keep = ctx.keep, ctx.dev, ctx.bg_keep
        d, bd = _grad_targets(ctx.sink, keep, dev, radii, zero_rows=True, bg_keep=bg_keep)
        d_in = torch.empty_like(keep[6]) if ctx.vert_grad else None
        d_out = torch.empty_like(keep[7]) if ctx.vert_grad else None
        R._launch_backward(ctx.call, radii, g_color, frosting_grads=_grads_block(d, d_in, d_out, bd))
        return _returned(ctx, keep, d, d_in, d_out, bg_keep, bd)


class _FrostingRenderTwoStep(torch.autograd.Function):
    """Attribute kernel -> rasterizer -> attribute backward (round 2a's route; kept as the cross-check of frosting mode)."""

    @staticmethod
    def forward(ctx, bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces,
                face_visible, rs, sink, *bg):
        fp, keep, bg_keep, dev = _params_block(bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner,
                                               outer, cells, faces, face_visible, bg)
        fv = keep[10]
        P, Rn = fp.P + fp.n_bg, fp.sh_rest
        o = dict(dtype=torch.float32, device=dev)
        # rows of occluded Gaussians are never read by preprocess (same lookup): plain empty allocations
        means3D, opac = torch.empty((P, 3), **o), torch.empty((P, 1), **o)
        scales, rots, shs = torch.empty((P, 3), **o), torch.empty((P, 4), **o), torch.empty((P, Rn + 1, 3), **o)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_attributes(
                C.byref(fp), _p(means3D), _p(opac), _p(scales), _p(rots), _p(shs), _stream(dev)))
        e = torch.Tensor([])
        color, radii, call, _ = R._launch_forward(
            means3D, shs, e, opac, scales, rots, e, rs, None, want_backward=True,
            face_visibility=(fv, keep[8]) if fv is not None else None)
        ctx.fp, ctx.call, ctx.sink, ctx.keep, ctx.dev, ctx.bg_keep = fp, call, sink, keep, dev, bg_keep
        ctx.vert_grad = inner.requires_grad or outer.requires_grad
        ctx.save_for_backward(radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _):
        (radii,) = ctx.saved_tensors
        keep, dev, bg_keep = ctx.keep, ctx.dev, ctx.bg_keep
        (dL_dmeans2D, _c, dL_dopacity, dL_dmeans3D, _cov, dL_dsh, dL_dscales, dL_drotations, _e) = R._launch_backward(
            ctx.call, radii, g_color, sparse_rows=True)
        d, bd = _grad_targets(ctx.sink, keep, dev, radii, zero_rows=False, bg_keep=bg_keep)
        d_in = torch.empty_like(keep[6]) if ctx.vert_grad else None
        d_out = torch.empty_like(keep[7]) if ctx.vert_grad else None
        fp = ctx.fp
        fp.d_radii = _p(radii)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_attributes_backward(
                C.byref(fp), _p(dL_dmeans3D), _p(dL_dopacity), _p(dL_dscales), _p(dL_drotations), _p(dL_dsh),
                C.byref(_grads_block(d, d_in, d_out, bd)), _stream(dev)))
        return _returned(ctx, keep, d, d_in, d_out, bg_keep, bd)


def _apply(fn, params, mesh, raster_settings, face_visible, grad_sink):
    bg = background_params(params)
    return fn.apply(params["bary_logits"], params["opacity_logits"], params["log_scales"], params["quats"],
                    params["sh_dc"], params["sh_rest"], mesh["inner"], mesh["outer"], mesh["cells"],
                    mesh["faces"], face_visible, raster_settings, grad_sink, *(bg or ()))


def frosting_render(params, mesh, raster_settings, face_visible=None, grad_sink=None):
    """params / mesh: the dicts of `scenes.frosting_layer`; `face_visible` [F]: the prepass's visible-face marks for this
    camera (None: no occlusion culling).  Returns (color [3,H,W], radii [n_mesh + n_bg]); differentiable w.r.t. the
    parameters -- the background ones (BG_KEYS) included when `params` has them -- and the shell vertices.  `grad_sink`
    (FrostingAdam's `grads`, or a dict of tensors): the parameter gradients are written there instead."""
    return _apply(_FrostingRender, params, mesh, raster_settings, face_visible, grad_sink)


def frosting_render_two_step(params, mesh, raster_settings, face_visible=None, grad_sink=None):
    """The same call through the stand-alone attribute kernels (csrc/frosting_attr.cu)."""
    return _apply(_FrostingRenderTwoStep, params, mesh, raster_settings, face_visible, grad_sink)
