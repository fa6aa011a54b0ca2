"""Fused Frosting attribute construction (SURVEY.md row a20) -- host side.

`frosting_attributes_fused(params, mesh, mask=None)` returns the same dict as the torch restatement of
Frosting's properties (`scenes.frosting_attributes`, i.e. frosting_scene/frosting_model.py:713-799):
means3D, opacities, scales, rotations, shs -- from ONE kernel, with ONE backward kernel that returns the
gradients of the learnable parameters (bary logits, opacity logits, log-scales, raw quaternions, SH dc /
rest) and of the shell vertices (inner / outer, scatter-added).  Masked (occluded) Gaussians are skipped:
their outputs are left uninitialised -- the rasterizer never reads them when given the same
`visibility_mask` -- and their parameter gradients are zero.  With the six background keys in `params`
(frosting_render.BG_KEYS) the outputs have n_mesh + n_bg rows: the background rows (never masked) come from the
background attribute kernels, written in place behind the mesh rows.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import FrostingParams, FrostingGrads
from .frosting_render import BG_KEYS, background_params, _background_block, _background_grads


def _p(t):
    return None if t is None or t.numel() == 0 else C.c_void_p(t.data_ptr())


class _FrostingAttributes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, mask,
                sink=None, face_visible=None, *bg):
        if not bary_logits.is_cuda:
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        dev = bary_logits.device
        # contiguous, and copied if a view starts at an address the kernels' 64/128-bit row accesses cannot use
        t = [x.contiguous() if x.contiguous().data_ptr() % 16 == 0 else x.contiguous().clone()
             for x in (bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer)]
        bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer = t
        cells = cells.to(device=dev, dtype=torch.int64).contiguous()
        faces = faces.to(device=dev, dtype=torch.int32).contiguous()
        m = None if mask is None else mask.to(device=dev, dtype=torch.uint8).contiguous()
        fv = None if face_visible is None else face_visible.to(device=dev, dtype=torch.uint8).contiguous()
        n_mesh, R = bary_logits.shape[0], sh_rest.shape[1]
        fbg, bg_keep = _background_block(bg, dev, R)
        P = n_mesh + (fbg.n if fbg is not None else 0)
        fp = FrostingParams(P=n_mesh, n_verts=inner.shape[0], n_faces=faces.shape[0], sh_rest=R,
                            d_bary_logits=_p(bary_logits), d_cells=_p(cells), d_faces=_p(faces),
                            d_inner_verts=_p(inner), d_outer_verts=_p(outer), d_opacity_logits=_p(opacity_logits),
                            d_log_scales=_p(log_scales), d_quats=_p(quats), d_sh_dc=_p(sh_dc), d_sh_rest=_p(sh_rest),
                            d_mask=_p(m), d_face_visible=_p(fv))
        o = dict(dtype=torch.float32, device=dev)
        alloc = torch.empty if (m is None and fv is None) else torch.zeros    # masked rows stay finite for downstream torch code
        means3D, opac = alloc((P, 3), **o), alloc((P, 1), **o)
        scales, rots, shs = alloc((P, 3), **o), alloc((P, 4), **o), alloc((P, R + 1, 3), **o)
        with torch.cuda.device(dev):
            stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
            _lib.check(_lib.lib().fb200_frosting_attributes(
                C.byref(fp), _p(means3D), _p(opac), _p(scales), _p(rots), _p(shs), stream))
            if fbg is not None:
                _lib.check(_lib.lib().fb200_frosting_background_attributes(
                    C.byref(fbg), R, *[_p(t[n_mesh:]) for t in (means3D, opac, scales, rots, shs)], stream))
        ctx.fp, ctx.fbg, ctx.bg_keep = fp, fbg, bg_keep
        ctx.sink = sink
        ctx.keep = (bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, m, fv)
        ctx.vert_grad = inner.requires_grad or outer.requires_grad
        return means3D, opac, scales, rots, shs

    @staticmethod
    def backward(ctx, g_means3D, g_opac, g_scales, g_rots, g_shs):
        bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, m, fv = ctx.keep
        dev = bary_logits.device
        fbg, bg_keep = ctx.fbg, ctx.bg_keep
        n_mesh, R = bary_logits.shape[0], sh_rest.shape[1]
        P = n_mesh + (fbg.n if fbg is not None else 0)
        o = dict(dtype=torch.float32, device=dev)
        z = lambda g, shape: torch.zeros(shape, **o) if g is None else g.contiguous()
        g_means3D, g_opac, g_scales = z(g_means3D, (P, 3)), z(g_opac, (P, 1)), z(g_scales, (P, 3))
        g_rots, g_shs = z(g_rots, (P, 4)), z(g_shs, (P, R + 1, 3))
        if ctx.sink is not None:
            # gradients go straight into the optimizer's gradient slab (frosting_b200/optim.py); autograd gets None
            k = ctx.sink
            if hasattr(k, "sink_once"):
                k.sink_once(("bary_logits", "opacity_logits", "log_scales", "quats", "sh_dc", "sh_rest") +
                            (BG_KEYS if fbg is not None else ()))
            d_bary, d_op, d_ls = k["bary_logits"], k["opacity_logits"], k["log_scales"]
            d_q, d_dc, d_rest = k["quats"], k["sh_dc"], k["sh_rest"]
            for t, ref in ((d_bary, bary_logits), (d_op, opacity_logits), (d_ls, log_scales), (d_q, quats),
                           (d_dc, sh_dc), (d_rest, sh_rest)):
                if t.numel() != ref.numel() or not t.is_contiguous() or t.dtype != torch.float32 or t.device != dev:
                    raise RuntimeError("grad_sink tensors must be contiguous fp32 CUDA tensors shaped like the parameters")
            bd = None if fbg is None else [k[n] for n in BG_KEYS]
            for t, ref in zip(bd or (), bg_keep or ()):
                if t.numel() != ref.numel() or not t.is_contiguous() or t.dtype != torch.float32 or t.device != dev:
                    raise RuntimeError("grad_sink tensors must be contiguous fp32 CUDA tensors shaped like the parameters")
        else:
            d_bary, d_op, d_ls = torch.empty((n_mesh, 6), **o), torch.empty((n_mesh,), **o), torch.empty((n_mesh, 3), **o)
            d_q, d_dc = torch.empty((n_mesh, 4), **o), torch.empty((n_mesh, 1, 3), **o)
            d_rest = torch.empty((n_mesh, R, 3), **o)
            bd = None if fbg is None else [torch.empty(tuple(t.shape), **o) for t in bg_keep]
        d_in = torch.empty_like(inner) if ctx.vert_grad else None
        d_out = torch.empty_like(outer) if ctx.vert_grad else None
        grads = FrostingGrads(d_bary_logits=_p(d_bary), d_inner_verts=_p(d_in), d_outer_verts=_p(d_out),
                              d_opacity_logits=_p(d_op), d_log_scales=_p(d_ls), d_quats=_p(d_q), d_sh_dc=_p(d_dc),
                              d_sh_rest=_p(d_rest))
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_attributes_backward(
                C.byref(ctx.fp), _p(g_means3D), _p(g_opac), _p(g_scales), _p(g_rots), _p(g_shs), C.byref(grads),
                C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
            if fbg is not None:
                _lib.check(_lib.lib().fb200_frosting_background_attributes_backward(
                    C.byref(fbg), R, None, *[_p(t[n_mesh:]) for t in (g_means3D, g_opac, g_scales, g_rots, g_shs)],
                    C.byref(_background_grads(bd)), C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
        tail = ()
        if fbg is not None:
            tail = (None,) * 6 if ctx.sink is not None else (bd[0], bd[1].view_as(bg_keep[1])) + tuple(bd[2:])
        if ctx.sink is not None:
            return (None, None, None, None, None, None, d_in, d_out, None, None, None, None, None) + tail
        return (d_bary, d_op.view_as(opacity_logits), d_ls, d_q, d_dc, d_rest, d_in, d_out, None, None, None, None,
                None) + tail


def frosting_attributes_fused(params, mesh, mask=None, grad_sink=None, face_visible=None):
    """params / mesh: the dicts of `scenes.frosting_layer` (bary_logits, opacity_logits, log_scales, quats, sh_dc,
    sh_rest | inner, outer, cells, faces).  Returns the rasterizer inputs.  `grad_sink` (dict with the parameter
    names): the backward writes the parameter gradients there (overwriting) instead of returning them to autograd.
    `face_visible` [F]: cull by face_visible[cells[i]] inside the kernels (the mask without a mask tensor).  With the
    background keys (frosting_render.BG_KEYS) the outputs cover n_mesh + n_bg Gaussians, background rows last; mask /
    face_visible apply to the mesh rows only."""
    bg = background_params(params)
    means3D, opac, scales, rots, shs = _FrostingAttributes.apply(
        params["bary_logits"], params["opacity_logits"], params["log_scales"], params["quats"], params["sh_dc"],
        params["sh_rest"], mesh["inner"], mesh["outer"], mesh["cells"], mesh["faces"], mask, grad_sink, face_visible,
        *(bg or ()))
    return dict(means3D=means3D, opacities=opac, scales=scales, rotations=rots, shs=shs)
