"""Fused Frosting attribute construction (SURVEY.md row a20) -- host side.

`frosting_attributes_fused(params, mesh, mask=None)` returns the same dict as the torch restatement of
Frosting's properties (`scenes.frosting_attributes`, i.e. frosting_scene/frosting_model.py:713-799):
means3D, opacities, scales, rotations, shs -- from ONE kernel, with ONE backward kernel that returns the
gradients of the learnable parameters (bary logits, opacity logits, log-scales, raw quaternions, SH dc /
rest) and of the shell vertices (inner / outer, scatter-added).  Masked (occluded) Gaussians are skipped:
their outputs are left uninitialised -- the rasterizer never reads them when given the same
`visibility_mask` -- and their parameter gradients are zero.  With the six background keys in `params`
(frosting_render.BG_KEYS) the outputs have n_mesh + n_bg rows, the background rows (never masked) behind the mesh rows.
"""
import ctypes as C

import torch

from . import _lib
from .frosting_render import background_params, _p, _params_block, _grads_block, _grad_targets, _returned, _stream


class _FrostingAttributes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner, outer, cells, faces, mask,
                sink=None, face_visible=None, *bg):
        fp, keep, bg_keep, dev = _params_block(bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest, inner,
                                               outer, cells, faces, face_visible, bg, mask)
        P, R = fp.P + fp.n_bg, fp.sh_rest
        o = dict(dtype=torch.float32, device=dev)
        # masked rows stay finite for downstream torch code
        alloc = torch.empty if (mask is None and face_visible is None) else torch.zeros
        means3D, opac = alloc((P, 3), **o), alloc((P, 1), **o)
        scales, rots, shs = alloc((P, 3), **o), alloc((P, 4), **o), alloc((P, R + 1, 3), **o)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_attributes(
                C.byref(fp), _p(means3D), _p(opac), _p(scales), _p(rots), _p(shs), _stream(dev)))
        ctx.fp, ctx.sink, ctx.keep, ctx.bg_keep, ctx.dev = fp, sink, keep, bg_keep, dev
        ctx.vert_grad = inner.requires_grad or outer.requires_grad
        return means3D, opac, scales, rots, shs

    @staticmethod
    def backward(ctx, g_means3D, g_opac, g_scales, g_rots, g_shs):
        fp, keep, bg_keep, dev = ctx.fp, ctx.keep, ctx.bg_keep, ctx.dev
        P, R = fp.P + fp.n_bg, fp.sh_rest
        o = dict(dtype=torch.float32, device=dev)
        z = lambda g, shape: torch.zeros(shape, **o) if g is None else g.contiguous()
        g_means3D, g_opac, g_scales = z(g_means3D, (P, 3)), z(g_opac, (P, 1)), z(g_scales, (P, 3))
        g_rots, g_shs = z(g_rots, (P, 4)), z(g_shs, (P, R + 1, 3))
        # with a sink the gradients go straight into the optimizer's gradient slab (frosting_b200/optim.py) and autograd
        # gets None
        d, bd = _grad_targets(ctx.sink, keep, dev, None, zero_rows=False, bg_keep=bg_keep)
        d_in = torch.empty_like(keep[6]) if ctx.vert_grad else None
        d_out = torch.empty_like(keep[7]) if ctx.vert_grad else None
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_attributes_backward(
                C.byref(fp), _p(g_means3D), _p(g_opac), _p(g_scales), _p(g_rots), _p(g_shs),
                C.byref(_grads_block(d, d_in, d_out, bd)), _stream(dev)))
        return _returned(ctx, keep, d, d_in, d_out, bg_keep, bd)


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
