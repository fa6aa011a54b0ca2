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
returns the background parameters' gradients too.

The stand-alone attribute kernels (csrc/frosting_attr.cu, SURVEY.md row a20) serve `frosting_attributes_fused` -- the
rasterizer inputs of Frosting's properties from one kernel, the parameter gradients from one backward kernel -- and
`frosting_render_two_step`, which keeps the attribute-kernel route (tests compare the two).

`FrostingBlock` owns the parameter block (fb200_frosting_params) all of them, the edit and the texture bake launch with.
"""
import ctypes as C

import torch

from . import _lib
from . import rasterizer as R
from ._lib import FrostingParams, FrostingGrads, ptr, stream

MESH_KEYS = ("bary_logits", "opacity_logits", "log_scales", "quats", "sh_dc", "sh_rest")
# Frosting's _bg_points, _bg_opacities, _bg_scales, _bg_quaternions, _bg_sh_coordinates_dc / _rest, in this order
BG_KEYS = ("bg_points", "bg_opacity_logits", "bg_log_scales", "bg_quats", "bg_sh_dc", "bg_sh_rest")
SHELL_KEYS = ("inner", "outer", "cells", "faces")


def _has_background(params):
    """Whether `params` holds the six background tensors (all six or none)."""
    have = [k in params for k in BG_KEYS]
    if any(have) and not all(have):
        raise ValueError(f"background Gaussians need all of {BG_KEYS}")
    return all(have)


class FrostingBlock:
    """fb200_frosting_params over a whole model, and every tensor it points into.

    `params` / `mesh`: the dicts of `scenes.frosting_layer` (the background keys BG_KEYS optional); `face_visible` [F] and
    `mask` [n_mesh]: optional culling inputs.  The tensors are kept, converted for the kernels, in `tensors` under the
    struct's field names (without `d_`), so the struct `fp` and the memory it points to live and die together.  The frame
    has `rows` = `n_mesh` mesh-bound Gaussians and `n_bg` background ones after them.

    The autograd Functions below take the block's inputs as `leaves(params, mesh, *call)`: the six mesh parameters, the
    shell (inner, outer), cells, faces, the Function's N_CALL per-call arguments, then the six background parameters;
    `autograd_grads` returns the gradients in that order."""

    N_CALL = 3

    def __init__(self, params, mesh, face_visible=None, mask=None):
        self.has_bg = _has_background(params)
        if not params["bary_logits"].is_cuda:
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        dev = self.device = params["bary_logits"].device
        t = {k: R._f32c(params[k], dev, "frosting parameter") for k in MESH_KEYS}
        t["inner_verts"] = R._f32c(mesh["inner"], dev, "frosting parameter")
        t["outer_verts"] = R._f32c(mesh["outer"], dev, "frosting parameter")
        t["cells"] = mesh["cells"].to(device=dev, dtype=torch.int64).contiguous()
        t["faces"] = mesh["faces"].to(device=dev, dtype=torch.int32).contiguous()
        t["face_visible"] = None if face_visible is None else face_visible.to(device=dev, dtype=torch.uint8).contiguous()
        t["mask"] = None if mask is None else mask.to(device=dev, dtype=torch.uint8).contiguous()
        self.n_mesh, Rn = t["bary_logits"].shape[0], t["sh_rest"].shape[1]
        self.n_bg = 0
        if self.has_bg:
            t.update({k: R._f32c(params[k], dev, "background parameter") for k in BG_KEYS})
            n = self.n_bg = t["bg_points"].shape[0]
            if t["bg_points"].shape != (n, 3) or t["bg_sh_rest"].shape != (n, Rn, 3) or \
                    any(t[k].shape[0] != n for k in BG_KEYS):
                raise RuntimeError("background parameters must be [n,3], [n], [n,3], [n,4], [n,1,3], [n,M-1,3] with the "
                                   "mesh block's M")
        self.rows = self.n_mesh + self.n_bg
        self.tensors = t
        self.vert_grad = mesh["inner"].requires_grad or mesh["outer"].requires_grad
        self.fp = FrostingParams(P=self.n_mesh, n_verts=t["inner_verts"].shape[0], n_faces=t["faces"].shape[0],
                                 sh_rest=Rn, n_bg=self.n_bg, **{"d_" + k: ptr(v) for k, v in t.items()})

    @staticmethod
    def leaves(params, mesh, *call):
        """autograd's inputs for the block of `params` / `mesh` and a Function's N_CALL per-call arguments `call`."""
        bg = tuple(params[k] for k in BG_KEYS) if _has_background(params) else ()
        return tuple(params[k] for k in MESH_KEYS) + tuple(mesh[k] for k in SHELL_KEYS) + call + bg

    @staticmethod
    def split(leaves):
        """(params, mesh, call) of `leaves(params, mesh, *call)`."""
        n, s = len(MESH_KEYS), len(MESH_KEYS) + len(SHELL_KEYS)
        params = dict(zip(MESH_KEYS, leaves[:n]))
        params.update(zip(BG_KEYS, leaves[s + FrostingBlock.N_CALL:]))
        return params, dict(zip(SHELL_KEYS, leaves[n:s])), leaves[s:s + FrostingBlock.N_CALL]

    def grad_targets(self, sink, radii=None, zero_rows=False):
        """fb200_frosting_grads and the tensors it points into, by name: the parameter gradients -- the caller's sink (the
        optimizer's slab) or fresh tensors -- and the shell's (`inner_verts`, `outer_verts`: None unless the shell takes
        gradients).  `zero_rows`: the backward writes the rendered rows only (frosting mode) and the others are zero: a
        sink that understands `row_radii` is told so, anything else is zero-filled."""
        names = MESH_KEYS + (BG_KEYS if self.has_bg else ())
        if sink is not None:
            if hasattr(sink, "sink_once"):
                sink.sink_once(names)
            d = {k: sink[k] for k in names}
            for k in names:
                tt, ref = d[k], self.tensors[k]
                if tt.numel() != ref.numel() or not tt.is_contiguous() or tt.dtype != torch.float32 or \
                        tt.device != self.device or tt.data_ptr() % 16:
                    raise RuntimeError("grad_sink tensors must be contiguous, 16-byte aligned fp32 CUDA tensors shaped "
                                       "like the parameters")
            if zero_rows:
                if getattr(sink, "accepts_row_radii", False):
                    # rows with radii <= 0 stay unwritten; the consumer (FrostingAdam's step) treats them as zero rows.
                    # The background groups have no row structure there: they are zero-filled and stay dense
                    sink.rows_from(radii[:self.n_mesh] if self.has_bg else radii, MESH_KEYS)
                    for k in BG_KEYS if self.has_bg else ():
                        d[k].zero_()
                else:
                    for tt in d.values():
                        tt.zero_()
        else:
            make, o = torch.zeros if zero_rows else torch.empty, dict(dtype=torch.float32, device=self.device)
            P, Rn = self.n_mesh, self.fp.sh_rest
            d = {k: make(tuple(self.tensors[k].shape), **o) for k in BG_KEYS if self.has_bg}
            shapes = ((P, 6), (P,), (P, 3), (P, 4), (P, 1, 3), (P, Rn, 3))
            d.update((k, make(shape, **o)) for k, shape in zip(MESH_KEYS, shapes))
        d["inner_verts"] = torch.empty_like(self.tensors["inner_verts"]) if self.vert_grad else None
        d["outer_verts"] = torch.empty_like(self.tensors["outer_verts"]) if self.vert_grad else None
        return FrostingGrads(**{"d_" + k: ptr(v) for k, v in d.items()}), d

    def autograd_grads(self, d, sink):
        """autograd's gradients for `leaves`, from the tensors of `grad_targets`: the parameters' (None when they went to
        a sink), the shell's, None for cells, faces and the per-call arguments."""
        def g(k):
            if sink is not None:
                return None
            return d[k].view_as(self.tensors[k]) if k in ("opacity_logits", "bg_opacity_logits") else d[k]
        bg = tuple(g(k) for k in BG_KEYS) if self.has_bg else ()
        return tuple(g(k) for k in MESH_KEYS) + (d["inner_verts"], d["outer_verts"]) + (None,) * (2 + self.N_CALL) + bg

    def attributes(self, alloc):
        """fb200_frosting_attributes: means3D, opacities, scales, rotations, shs of the block's rows, in tensors made by
        `alloc` (torch.empty / torch.zeros)."""
        P, o = self.rows, dict(dtype=torch.float32, device=self.device)
        out = (alloc((P, 3), **o), alloc((P, 1), **o), alloc((P, 3), **o), alloc((P, 4), **o),
               alloc((P, self.fp.sh_rest + 1, 3), **o))
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().fb200_frosting_attributes(C.byref(self.fp), *(ptr(t) for t in out),
                                                            stream(self.device)))
        return out

    def attributes_backward(self, upstream, sink):
        """fb200_frosting_attributes_backward of the five upstream gradients; returns autograd's gradients."""
        fg, d = self.grad_targets(sink)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().fb200_frosting_attributes_backward(
                C.byref(self.fp), *(ptr(g) for g in upstream), C.byref(fg), stream(self.device)))
        return self.autograd_grads(d, sink)


class _FrostingRender(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *leaves):
        params, mesh, (face_visible, rs, sink) = FrostingBlock.split(leaves)
        blk = FrostingBlock(params, mesh, face_visible)
        color, radii, call, _ = R._launch_forward(None, None, None, None, None, None, None, rs, None,
                                                  want_backward=True, frosting=blk)
        ctx.blk, ctx.call, ctx.sink = blk, call, sink
        ctx.save_for_backward(radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _):
        (radii,) = ctx.saved_tensors
        fg, d = ctx.blk.grad_targets(ctx.sink, radii, zero_rows=True)
        R._launch_backward(ctx.call, radii, g_color, frosting_grads=fg)
        return ctx.blk.autograd_grads(d, ctx.sink)


class _FrostingRenderTwoStep(torch.autograd.Function):
    """Attribute kernel -> rasterizer -> attribute backward (round 2a's route; kept as the cross-check of frosting mode)."""

    @staticmethod
    def forward(ctx, *leaves):
        params, mesh, (face_visible, rs, sink) = FrostingBlock.split(leaves)
        blk = FrostingBlock(params, mesh, face_visible)
        # rows of occluded Gaussians are never read by preprocess (same lookup): plain empty allocations
        means3D, opac, scales, rots, shs = blk.attributes(torch.empty)
        fv = blk.tensors["face_visible"]
        e = torch.Tensor([])
        color, radii, call, _ = R._launch_forward(
            means3D, shs, e, opac, scales, rots, e, rs, None, want_backward=True,
            face_visibility=(fv, blk.tensors["cells"]) if fv is not None else None)
        ctx.blk, ctx.call, ctx.sink = blk, call, sink
        ctx.save_for_backward(radii)
        ctx.mark_non_differentiable(radii)
        return color, radii

    @staticmethod
    def backward(ctx, g_color, _):
        (radii,) = ctx.saved_tensors
        (dL_dmeans2D, _c, dL_dopacity, dL_dmeans3D, _cov, dL_dsh, dL_dscales, dL_drotations, _e) = R._launch_backward(
            ctx.call, radii, g_color, sparse_rows=True)
        ctx.blk.fp.d_radii = ptr(radii)
        return ctx.blk.attributes_backward((dL_dmeans3D, dL_dopacity, dL_dscales, dL_drotations, dL_dsh), ctx.sink)


class _FrostingAttributes(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *leaves):
        params, mesh, (face_visible, mask, sink) = FrostingBlock.split(leaves)
        blk = FrostingBlock(params, mesh, face_visible, mask)
        # masked rows stay finite for downstream torch code
        out = blk.attributes(torch.empty if (mask is None and face_visible is None) else torch.zeros)
        ctx.blk, ctx.sink = blk, sink
        return out

    @staticmethod
    def backward(ctx, *upstream):
        blk = ctx.blk
        P, o = blk.rows, dict(dtype=torch.float32, device=blk.device)
        shapes = ((P, 3), (P, 1), (P, 3), (P, 4), (P, blk.fp.sh_rest + 1, 3))
        upstream = [torch.zeros(s, **o) if g is None else g.contiguous() for g, s in zip(upstream, shapes)]
        # with a sink the gradients go straight into the optimizer's gradient slab (frosting_b200/optim.py) and autograd
        # gets None
        return blk.attributes_backward(upstream, ctx.sink)


def frosting_render(params, mesh, raster_settings, face_visible=None, grad_sink=None):
    """params / mesh: the dicts of `scenes.frosting_layer`; `face_visible` [F]: the prepass's visible-face marks for this
    camera (None: no occlusion culling).  Returns (color [3,H,W], radii [n_mesh + n_bg]); differentiable w.r.t. the
    parameters -- the background ones (BG_KEYS) included when `params` has them -- and the shell vertices.  `grad_sink`
    (FrostingAdam's `grads`, or a dict of tensors): the parameter gradients are written there instead."""
    return _FrostingRender.apply(*FrostingBlock.leaves(params, mesh, face_visible, raster_settings, grad_sink))


def frosting_render_two_step(params, mesh, raster_settings, face_visible=None, grad_sink=None):
    """The same call through the stand-alone attribute kernels (csrc/frosting_attr.cu)."""
    return _FrostingRenderTwoStep.apply(*FrostingBlock.leaves(params, mesh, face_visible, raster_settings, grad_sink))


def frosting_attributes_fused(params, mesh, mask=None, grad_sink=None, face_visible=None):
    """The rasterizer inputs of Frosting's properties (`scenes.frosting_attributes`, i.e. frosting_scene/
    frosting_model.py:713-799): dict(means3D, opacities, scales, rotations, shs), from ONE kernel, with ONE backward kernel
    that returns the gradients of the learnable parameters and of the shell vertices (inner / outer, scatter-added).

    params / mesh: the dicts of `scenes.frosting_layer` (bary_logits, opacity_logits, log_scales, quats, sh_dc, sh_rest |
    inner, outer, cells, faces).  `mask` [P] or `face_visible` [F] (cull by face_visible[cells[i]] inside the kernels):
    masked Gaussians are skipped -- their outputs are zero, their parameter gradients are zero.  `grad_sink` (dict with
    the parameter names): the backward writes the parameter gradients there (overwriting) instead of returning them to
    autograd.  With the background keys (BG_KEYS) the outputs cover n_mesh + n_bg Gaussians, background rows last;
    mask / face_visible apply to the mesh rows only."""
    means3D, opac, scales, rots, shs = _FrostingAttributes.apply(
        *FrostingBlock.leaves(params, mesh, face_visible, mask, grad_sink))
    return dict(means3D=means3D, opacities=opac, scales=scales, rotations=rots, shs=shs)
