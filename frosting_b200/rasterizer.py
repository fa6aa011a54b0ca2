"""Python surface of the rasterizer -- a drop-in for `diff_gaussian_rasterization`.

Mirrors DGR/diff_gaussian_rasterization/__init__.py (DGR = gaussian_splatting/submodules/
diff-gaussian-rasterization in the reference):
  GaussianRasterizationSettings  <- __init__.py:157-169 (same 12 fields, same order)
  GaussianRasterizer             <- __init__.py:171-220 (same forward signature, same exceptions,
                                    same (color[3,H,W], radii[P]) return, markVisible)
  _RasterizeGaussians            <- __init__.py:44-155  (same 8 gradients in the same order)
The native side is reached through the C ABI in include/frosting_b200.h via ctypes; torch only owns
the tensors and the stream.

One extension: `GaussianRasterizer.forward(..., visibility_mask=None)` takes the per-Gaussian
occlusion mask (frosting_model.py:1564-1576) and drops masked Gaussians inside the preprocess kernel
instead of boolean-gathering every attribute tensor (frosting_model.py:1578-1586).
"""
from typing import NamedTuple
import ctypes as C
import os
import threading

import torch
import torch.nn as nn

from . import _lib
from ._lib import Params, Inputs, Workspace, Grads, ptr


class GaussianRasterizationSettings(NamedTuple):
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: torch.Tensor
    scale_modifier: float
    viewmatrix: torch.Tensor
    projmatrix: torch.Tensor
    sh_degree: int
    campos: torch.Tensor
    prefiltered: bool
    debug: bool


NO_CULL = False   # test hook: disable sub-tile culling (debug bit 1) to prove it is output-neutral
# FB200_EXACT_BINNING=1: always size the binning buffer from this frame's own instance count (two-phase forward with a
# host wait, like the reference's blocking copy at rasterizer_impl.cu:280-281) instead of speculating from earlier frames
EXACT_BINNING = os.environ.get("FB200_EXACT_BINNING", "0") == "1"
# FB200_CHECK_BEFORE_BACKWARD=1: wait for a speculatively launched forward's status words before launching its backward
# (an overflow is then raised from backward()).  Default: no wait -- the backward is enqueued behind the forward at once
# (its kernels exit on the overflow word; the gradients of such a frame are zeros) and the overflow is raised by the next
# call on this host thread.  The wait cost the GPU an idle gap per frame: the host slept until the forward had finished
# and only then started enqueueing the loss / backward kernels.
CHECK_BEFORE_BACKWARD = os.environ.get("FB200_CHECK_BEFORE_BACKWARD", "0") == "1"
_HEADROOM = 2.0           # speculative capacity = _HEADROOM x (largest count seen for this problem size) + 64 Ki
_RING = 8                 # status mailboxes in flight per (thread, device)

_size_cache = {}


def _sizes(L, P, W, H):
    """Workspace sizes rounded up to 512 bytes (so the carved sub-buffers keep torch's base alignment)."""
    k = (P, W, H)
    v = _size_cache.get(k)
    if v is None:
        r = lambda n: (int(n) + 511) // 512 * 512
        v = (r(L.fb200_geom_bytes(P)), r(L.fb200_image_bytes(W, H)))
        if len(_size_cache) > 64:
            _size_cache.clear()
        _size_cache[k] = v
    return v


def _grow_hint(hint: int, num_rendered: int) -> int:
    """Capacity to launch the next frame of this size with.  It moves rarely and in coarse steps: every distinct capacity
    is a distinct allocation size for torch's caching allocator, and a fresh 100+ MB cudaMalloc stalls the stream for
    milliseconds (a training run whose instance count creeps upward would re-allocate every few frames).
    Grow only when less than 25 % of the headroom is left, then to `_HEADROOM` x the count, rounded up to 1/8 of its
    leading power of two."""
    n = max(int(num_rendered), 0)
    if hint > 0 and n * 1.25 <= hint:
        return hint
    want = int(n * _HEADROOM) + 65536
    step = 1 << max(want.bit_length() - 4, 16)
    return max(hint, (want + step - 1) // step * step)


class BinningOverflow(RuntimeError):
    """A frame's tile-instance count exceeded the capacity its binning buffer was launched with.  Nothing was rendered
    for that frame (the kernels see the overflow word and exit), its outputs are invalid; the capacity hint has been
    raised, re-running the frame succeeds."""


class _Pending:
    __slots__ = ("slot", "event", "capacity", "key", "done", "num_rendered", "overflow", "reported")


class _HostState:
    """Host-side state of ONE host thread on ONE device: capacity hints, the ring of pinned status mailboxes and
    the frames whose status words have not been looked at yet.  Per (thread, device), so one host thread per GPU --
    or several threads on one GPU -- never share a mailbox (SURVEY.md 8b: re-entrant, no globals across threads)."""

    def __init__(self, device):
        self.device = device
        self.hints = {}            # (P, W, H) -> capacity to launch the next frame of this size with
        self.slots = [torch.empty((_lib.FB200_STATUS_WORDS,), dtype=torch.int32, pin_memory=True) for _ in range(_RING)]
        self.events = [torch.cuda.Event() for _ in range(_RING)]
        self.next = 0
        self.pending = []          # oldest first
        self.overflowed = []       # resolved, overflowed, not yet reported
        self.last_num_rendered = 0

    def mailbox(self):
        """A free pinned mailbox; a frame still holding the next one is waited for first (it finished long ago)."""
        i = self.next
        self.next = (i + 1) % _RING
        for p in list(self.pending):
            if p.slot is self.slots[i]:
                try:
                    self.resolve(p)
                except BinningOverflow:
                    p.reported = False        # leave the report to the frame's own backward / the next poll
                    self.overflowed.append(p)
        return self.slots[i], self.events[i]

    def resolve(self, p, wait=True):
        """Read a frame's status words once its copy has landed; raises BinningOverflow (once) for an overflowed frame."""
        if not p.done:
            if not wait and not p.event.query():
                return False
            p.event.synchronize()
            p.num_rendered = int(p.slot[_lib.ST_NUM_RENDERED])
            p.overflow = bool(int(p.slot[_lib.ST_OVERFLOW])) or p.num_rendered > p.capacity or p.num_rendered < 0
            p.done = True
            if p in self.pending:
                self.pending.remove(p)
            self.last_num_rendered = p.num_rendered
            self.hints[p.key] = _grow_hint(self.hints.get(p.key, 0), p.num_rendered)
        if p.overflow and not p.reported:
            p.reported = True
            raise BinningOverflow(
                f"frosting_b200: a frame produced {p.num_rendered} tile instances but was launched with binning capacity "
                f"{p.capacity} (speculated from earlier frames of this size); that frame's outputs are invalid. The "
                "capacity has been raised -- re-run the frame, or set FB200_EXACT_BINNING=1 to size every frame exactly.")
        return True

    def poll(self):
        """Look at every earlier frame whose status copy has completed (no waiting)."""
        while self.overflowed:
            self.resolve(self.overflowed.pop(0))
        for p in list(self.pending):
            if not self.resolve(p, wait=False):
                break


_tls = threading.local()


def _host_state(device) -> _HostState:
    d = getattr(_tls, "states", None)
    if d is None:
        d = _tls.states = {}
    st = d.get(device.index)
    if st is None:
        st = d[device.index] = _HostState(device)
    return st


def _f32c(t: torch.Tensor, device, name: str) -> torch.Tensor:
    if t.numel() == 0:
        return t
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    if t.device != device:
        t = t.to(device)
    if not t.is_contiguous():
        t = t.contiguous()
    if t.data_ptr() % 16:
        # the kernels read rows with 128-bit loads; a contiguous VIEW at an odd storage offset is legal for the
        # reference (scalar loads) and must be legal here: copy it to an aligned allocation
        t = t.clone(memory_format=torch.contiguous_format)
    return t


class _Call:
    """Everything one forward needs again in backward (kept alive by the autograd ctx)."""
    __slots__ = ("prm", "inp", "ws", "tensors", "geom", "image", "binning", "status", "capacity",
                 "_num_rendered", "device", "extra", "pending", "host")

    @property
    def num_rendered(self) -> int:
        """R of this frame; for a speculatively launched frame this waits for its status copy (usually long done)."""
        if self._num_rendered is None:
            self.host.resolve(self.pending)
            self._num_rendered = self.pending.num_rendered
        return self._num_rendered

    def check(self):
        """Raise if this frame overflowed its binning capacity (waits for its status words; called before the backward is
        launched only under FB200_CHECK_BEFORE_BACKWARD=1)."""
        if self.pending is not None:
            self.host.resolve(self.pending)


def _prepare(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, visibility,
             extra_features, extra_bg, face_visibility=None):
    if means3D.dim() != 2 or means3D.size(1) != 3:
        raise RuntimeError("means3D must have dimensions (num_points, 3)")   # rasterize_points.cu:57-59
    if not means3D.is_cuda:
        raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
    device = means3D.device
    P = means3D.size(0)
    H, W = int(rs.image_height), int(rs.image_width)

    means3D = _f32c(means3D, device, "means3D")
    sh = _f32c(sh, device, "shs")
    colors_precomp = _f32c(colors_precomp, device, "colors_precomp")
    opacities = _f32c(opacities, device, "opacities")
    scales = _f32c(scales, device, "scales")
    rotations = _f32c(rotations, device, "rotations")
    cov3Ds_precomp = _f32c(cov3Ds_precomp, device, "cov3D_precomp")
    bg = _f32c(rs.bg, device, "bg")
    view = _f32c(rs.viewmatrix, device, "viewmatrix")
    proj = _f32c(rs.projmatrix, device, "projmatrix")
    campos = _f32c(rs.campos, device, "campos")
    vis = None
    if visibility is not None:
        vis = visibility.to(device=device, dtype=torch.uint8).contiguous() if visibility.dtype != torch.uint8 \
            else visibility.to(device).contiguous()
        if vis.numel() != P:
            raise RuntimeError("visibility_mask must have one entry per Gaussian")
    fvis = cells = None
    if face_visibility is not None:
        fvis, cells = face_visibility
        fvis = fvis.to(device=device, dtype=torch.uint8).contiguous()
        cells = cells.to(device=device, dtype=torch.int64).contiguous()
        if cells.numel() > P:
            raise RuntimeError("face_visibility: more cell indices than Gaussians")

    M = sh.size(1) if sh.numel() != 0 else 0   # rasterize_points.cu:84-87

    # row f4: extra feature channels blended in the same traversal
    if extra_features is not None:
        extra_features = _f32c(extra_features, device, "extra_features")
        if extra_features.dim() != 2 or extra_features.size(0) != P or not (1 <= extra_features.size(1) <= 3):
            raise RuntimeError("extra_features must have dimensions (num_points, 1..3)")
        E = extra_features.size(1)
        extra_bg = torch.zeros(E, dtype=torch.float32, device=device) if extra_bg is None \
            else _f32c(extra_bg.reshape(-1), device, "extra_background")
        if extra_bg.numel() != E:
            raise RuntimeError("extra_background must have one value per extra channel")

    prm = Params(P=P, sh_degree=int(rs.sh_degree), sh_coeffs=int(M), image_width=W, image_height=H,
                 tanfovx=float(rs.tanfovx), tanfovy=float(rs.tanfovy),
                 scale_modifier=float(rs.scale_modifier), prefiltered=int(bool(rs.prefiltered)),
                 debug=int(bool(rs.debug)) | (2 if NO_CULL else 0), extra=None)
    inp = Inputs(d_background=ptr(bg), d_means3D=ptr(means3D), d_shs=ptr(sh),
                 d_colors_precomp=ptr(colors_precomp), d_opacities=ptr(opacities), d_scales=ptr(scales),
                 d_rotations=ptr(rotations), d_cov3D_precomp=ptr(cov3Ds_precomp),
                 d_viewmatrix=ptr(view), d_projmatrix=ptr(proj), d_campos=ptr(campos), d_visibility=ptr(vis),
                 d_point_cells=ptr(cells) if fvis is not None and cells.numel() else None,
                 d_face_visible=ptr(fvis) if fvis is not None and cells.numel() else None,
                 n_cell_points=int(cells.numel()) if cells is not None else 0)
    tensors = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, bg, view, proj,
               campos, vis, extra_features, extra_bg, fvis, cells)
    return device, P, W, H, prm, inp, tensors, extra_features, extra_bg


def _prepare_frosting(block, rs):
    """Frosting mode (fb200_inputs.frosting): the rasterizer reads the parameter block itself; no attribute tensors.
    `block`: a frosting_render.FrostingBlock; the frame is its rows (mesh-bound Gaussians, then background ones)."""
    fp, device = block.fp, block.device
    P, M = block.rows, int(fp.sh_rest) + 1
    H, W = int(rs.image_height), int(rs.image_width)
    bg = _f32c(rs.bg, device, "bg")
    view = _f32c(rs.viewmatrix, device, "viewmatrix")
    proj = _f32c(rs.projmatrix, device, "projmatrix")
    campos = _f32c(rs.campos, device, "campos")
    prm = Params(P=P, sh_degree=int(rs.sh_degree), sh_coeffs=M, image_width=W, image_height=H,
                 tanfovx=float(rs.tanfovx), tanfovy=float(rs.tanfovy),
                 scale_modifier=float(rs.scale_modifier), prefiltered=int(bool(rs.prefiltered)),
                 debug=int(bool(rs.debug)) | (2 if NO_CULL else 0), extra=None)
    inp = Inputs(d_background=ptr(bg), d_viewmatrix=ptr(view), d_projmatrix=ptr(proj), d_campos=ptr(campos),
                 n_cell_points=0, frosting=C.addressof(fp))
    return device, P, W, H, prm, inp, (block, bg, view, proj, campos), None, None


def _launch_forward(means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                    rs: GaussianRasterizationSettings, visibility, extra_features=None, extra_bg=None,
                    want_backward=False, exact=False, geometry_only=False, face_visibility=None, frosting=None):
    """One forward through the C ABI.

    Default: ONE-PHASE, no host wait.  `fb200_forward` is launched with a binning capacity speculated from earlier frames
    of this problem size (2x the largest count seen); the frame's status words travel to a pinned mailbox behind the
    kernels and are looked at lazily -- by a later call on this thread, or before this frame's backward.  An overflow
    (never silently wrong: the kernels, the backward's included, exit on the overflow word) raises BinningOverflow from
    the next call on this thread and the next frame of this size is sized from the count that overflowed.  The FIRST frame of a problem size, `debug`, `exact=True` and
    FB200_EXACT_BINNING=1 take the two-phase path: preprocess + tile scan, host reads the exact count (the reference
    blocks at the same point, rasterizer_impl.cu:280-281), raster phase with an exactly sized buffer.
    """
    L = _lib.lib()
    if frosting is not None:
        device, P, W, H, prm, inp, tensors, extra_features, extra_bg = _prepare_frosting(frosting, rs)
    else:
        device, P, W, H, prm, inp, tensors, extra_features, extra_bg = _prepare(
            means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, rs, visibility, extra_features,
            extra_bg, face_visibility)
    host = _host_state(device)
    host.poll()
    extra = None

    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        out_color = torch.empty((3, H, W), dtype=torch.float32, device=device)
        radii = torch.empty((P,), dtype=torch.int32, device=device)
        out_extra = None
        if extra_features is not None:
            out_extra = torch.empty((extra_features.size(1), H, W), dtype=torch.float32, device=device)
            if P == 0:
                out_extra.copy_(extra_bg.view(-1, 1, 1).expand_as(out_extra))
            extra = _lib.Extra(channels=extra_features.size(1), d_features=ptr(extra_features),
                               d_background=ptr(extra_bg), d_out=ptr(out_extra), d_dL_dout=None, d_dL_dfeatures=None)
            prm.extra = C.addressof(extra)
        gb, ib = _sizes(L, P, W, H)
        slab = torch.empty((gb + ib + 128,), dtype=torch.uint8, device=device)   # one allocator call
        geom, image = slab[:gb], slab[gb:gb + ib]
        status = slab[gb + ib:gb + ib + 4 * _lib.FB200_STATUS_WORDS].view(torch.int32)
        ws = Workspace(d_geom=geom.data_ptr(), geom_bytes=geom.numel(),
                       d_image=image.data_ptr(), image_bytes=image.numel(),
                       d_binning=None, binning_bytes=0, binning_capacity=0, d_status=status.data_ptr(),
                       # a backward will follow: its accumulators are cleared inside the forward's launch sequence
                       acc_zeroed_by_forward=1 if want_backward else 0)
        rptr = C.c_void_p(radii.data_ptr()) if P > 0 else None
        sptr = C.c_void_p(stream.cuda_stream)
        key = (P, W, H)
        hint = host.hints.get(key, 0)
        mailbox, event = host.mailbox()
        pending = None
        if exact or geometry_only or EXACT_BINNING or rs.debug or hint == 0:
            # two-phase: exact count through the mailbox, then the raster phase
            _lib.check(L.fb200_forward_geometry(C.byref(prm), C.byref(inp), C.byref(ws), rptr, sptr))
            mailbox.copy_(status, non_blocking=True)
            stream.synchronize()
            num_rendered = int(mailbox[_lib.ST_NUM_RENDERED])
            capacity = max(num_rendered, 1)
            binning = None
            if not geometry_only:
                binning = torch.empty((L.fb200_binning_bytes(capacity),), dtype=torch.uint8, device=device)
                ws.d_binning, ws.binning_bytes, ws.binning_capacity = binning.data_ptr(), binning.numel(), capacity
                ws.h_status = mailbox.data_ptr()     # the host HAS this frame's status words: empty sort classes are skipped
                _lib.check(L.fb200_forward_raster(C.byref(prm), C.byref(inp), C.byref(ws),
                                                  C.c_void_p(out_color.data_ptr()), rptr, sptr))
                ws.h_status = None
            host.hints[key] = _grow_hint(hint, num_rendered)
            host.last_num_rendered = num_rendered
        else:
            capacity = hint
            binning = torch.empty((L.fb200_binning_bytes(capacity),), dtype=torch.uint8, device=device)
            ws.d_binning, ws.binning_bytes, ws.binning_capacity = binning.data_ptr(), binning.numel(), capacity
            _lib.check(L.fb200_forward(C.byref(prm), C.byref(inp), C.byref(ws), C.c_void_p(out_color.data_ptr()),
                                       rptr, sptr))
            mailbox.copy_(status, non_blocking=True)
            event.record(stream)
            pending = _Pending()
            pending.slot, pending.event, pending.capacity, pending.key = mailbox, event, capacity, key
            pending.done, pending.num_rendered, pending.overflow, pending.reported = False, None, False, False
            host.pending.append(pending)
            num_rendered = None

    call = _Call()
    call.prm, call.inp, call.ws = prm, inp, ws
    call.tensors = tensors
    call.extra = extra
    call.geom, call.image, call.binning, call.status = geom, image, binning, status
    call.capacity, call._num_rendered, call.device = capacity, num_rendered, device
    call.pending, call.host = pending, host
    return out_color, radii, call, out_extra


def _launch_backward(call: "_Call", radii, grad_out_color, grad_out_extra=None, sparse_rows=False,
                     frosting_grads=None):
    L = _lib.lib()
    if CHECK_BEFORE_BACKWARD:
        call.check()       # a speculatively launched forward that overflowed has no state to differentiate: raise here
    prm = call.prm
    P, M = prm.P, prm.sh_coeffs
    device = call.device
    with torch.cuda.device(device):
        stream = torch.cuda.current_stream(device)
        g = grad_out_color
        if g.dtype != torch.float32:
            g = g.float()
        g = g.contiguous()
        if frosting_grads is not None:
            # frosting mode: the per-Gaussian backward writes the parameter gradients (rendered rows only), background
            # rows -- if the forward had any -- into the block's d_bg_* gradients
            grads = Grads(sparse_rows=1, frosting=C.addressof(frosting_grads))
            _lib.check(L.fb200_backward(
                C.byref(prm), C.byref(call.inp), C.byref(call.ws), C.c_void_p(radii.data_ptr()) if P > 0 else None,
                C.c_void_p(g.data_ptr()), C.byref(grads), C.c_void_p(stream.cuda_stream)))
            call.ws.acc_zeroed_by_forward = 0
            return None
        # one allocation carved into the gradient tensors the caller can use (each offset a multiple of 4 floats);
        # dL/dcolors on the SH path, dL/dcov3D on the scale/rotation path and dL/dscales, dL/drotations on the
        # precomputed-covariance path are never returned (`backward` below) and are not materialised
        has_sh, has_col = call.inp.d_shs is not None, call.inp.d_colors_precomp is not None
        has_cov = call.inp.d_cov3D_precomp is not None
        n = [3 * P, 3 * P, 3 * P if has_col else 0, P, 6 * P if has_cov else 0, 3 * M * P if has_sh else 0,
             0 if has_cov else 3 * P, 0 if has_cov else 4 * P]
        offs, tot = [], 0
        for c in n:
            offs.append(tot)
            tot += (c + 3) // 4 * 4
        gslab = torch.empty((max(tot, 1),), dtype=torch.float32, device=device)
        cut = lambda k, shape: gslab[offs[k]:offs[k] + n[k]].view(shape) if n[k] or P == 0 else None
        dL_dmeans3D, dL_dmeans2D, dL_dcolors = cut(0, (P, 3)), cut(1, (P, 3)), cut(2, (P, 3))
        dL_dopacity, dL_dcov3D, dL_dsh = cut(3, (P, 1)), cut(4, (P, 6)), cut(5, (P, M, 3))
        dL_dscales, dL_drotations = cut(6, (P, 3)), cut(7, (P, 4))
        dL_dextra = None
        if call.extra is not None:
            E = call.extra.channels
            ge = grad_out_extra
            ge = torch.zeros((E, prm.image_height, prm.image_width), dtype=torch.float32, device=device) if ge is None \
                else ge.float().contiguous()
            dL_dextra = torch.empty((P, E), dtype=torch.float32, device=device)
            call.extra.d_dL_dout, call.extra.d_dL_dfeatures = ge.data_ptr(), dL_dextra.data_ptr()
            prm.extra = C.addressof(call.extra)
        grads = Grads(d_dL_dmeans2D=ptr(dL_dmeans2D), d_dL_dcolors=ptr(dL_dcolors),
                      d_dL_dopacity=ptr(dL_dopacity), d_dL_dmeans3D=ptr(dL_dmeans3D),
                      d_dL_dcov3D=ptr(dL_dcov3D), d_dL_dsh=ptr(dL_dsh), d_dL_dscales=ptr(dL_dscales),
                      d_dL_drotations=ptr(dL_drotations), sparse_rows=1 if sparse_rows else 0)
        _lib.check(L.fb200_backward(C.byref(prm), C.byref(call.inp), C.byref(call.ws),
                                    C.c_void_p(radii.data_ptr()) if P > 0 else None,
                                    C.c_void_p(g.data_ptr()), C.byref(grads),
                                    C.c_void_p(stream.cuda_stream)))
        call.ws.acc_zeroed_by_forward = 0      # a second backward over this forward must clear them itself
    return dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dcov3D, dL_dsh, dL_dscales, dL_drotations, dL_dextra


def last_num_rendered(device=None) -> int:
    """R (tile instances) of the most recent forward of this host thread on `device` (default: current device).
    Waits for that frame's status copy if it has not been looked at yet."""
    if device is None:
        device = torch.device("cuda", torch.cuda.current_device())
    host = _host_state(torch.device(device))
    for p in list(host.pending):
        host.resolve(p)
    return host.last_num_rendered


def cpu_deep_copy_tuple(input_tuple):
    return tuple(item.cpu().clone() if isinstance(item, torch.Tensor) else item for item in input_tuple)


def rasterize_gaussians(means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                        raster_settings, visibility_mask=None, extra_features=None, extra_background=None,
                        face_visibility=None, return_alpha=False):
    # autograd.Function.forward always runs with grad mode off: whether a backward can follow is decided HERE
    want_backward = torch.is_grad_enabled() and any(
        isinstance(t, torch.Tensor) and t.requires_grad
        for t in (means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, extra_features))
    out = _RasterizeGaussians.apply(means3D, means2D, sh, colors_precomp, opacities, scales, rotations,
                                    cov3Ds_precomp, raster_settings, visibility_mask, extra_features, extra_background,
                                    want_backward, face_visibility, return_alpha)
    res = out[:3] if extra_features is not None else out[:2]
    return res + (out[3],) if return_alpha else res


class _RasterizeGaussians(torch.autograd.Function):
    @staticmethod
    def forward(ctx, means3D, means2D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp,
                raster_settings, visibility_mask=None, extra_features=None, extra_background=None,
                want_backward=False, face_visibility=None, return_alpha=False):
        args = (means3D, sh, colors_precomp, opacities, scales, rotations, cov3Ds_precomp, raster_settings,
                visibility_mask, extra_features, extra_background, want_backward, False, False, face_visibility)
        if raster_settings.debug:
            cpu_args = cpu_deep_copy_tuple(args[:7])   # copy before they can be corrupted
            try:
                color, radii, call, extra = _launch_forward(*args)
            except Exception as ex:
                torch.save(cpu_args, "snapshot_fw.dump")
                print("\nAn error occured in forward. Please forward snapshot_fw.dump for debugging.")
                raise ex
        else:
            color, radii, call, extra = _launch_forward(*args)
        ctx.call = call          # call.num_rendered: the reference's ctx.num_rendered (__init__.py:96), resolved lazily
        ctx.raster_settings = raster_settings
        ctx.present = tuple(t.numel() != 0 for t in (sh, colors_precomp, scales, rotations, cov3Ds_precomp))
        ctx.save_for_backward(radii)
        ctx.mark_non_differentiable(radii)
        if extra is None:
            extra = color.new_empty(0)        # placeholder third output (autograd wants tensors)
        # alpha = 1 - final_T: the reference computes and keeps final_T (forward.cu:369, imgBuffer) but never returns it
        alpha = color.new_empty(0)
        if return_alpha:
            prm = call.prm
            alpha = 1.0 - _lib.workspace_views(None, call.image, None, prm.P, prm.image_width, prm.image_height, 0,
                                               0)["final_T"]
        ctx.mark_non_differentiable(alpha)
        return color, radii, extra, alpha

    @staticmethod
    def backward(ctx, grad_out_color, _, grad_out_extra=None, _alpha=None):
        (radii,) = ctx.saved_tensors
        call = ctx.call
        if ctx.raster_settings.debug:
            try:
                out = _launch_backward(call, radii, grad_out_color, grad_out_extra)
            except Exception as ex:
                torch.save(cpu_deep_copy_tuple(call.tensors[:7]) + (grad_out_color.cpu().clone(),), "snapshot_bw.dump")
                print("\nAn error occured in backward. Writing snapshot_bw.dump for debugging.\n")
                raise ex
        else:
            out = _launch_backward(call, radii, grad_out_color, grad_out_extra)
        (grad_means2D, grad_colors_precomp, grad_opacities, grad_means3D, grad_cov3Ds_precomp, grad_sh,
         grad_scales, grad_rotations, grad_extra) = out
        has_sh, has_col, has_s, has_r, has_cov = ctx.present
        # same order as DGR/diff_gaussian_rasterization/__init__.py:143-153
        return (
            grad_means3D,
            grad_means2D,
            grad_sh if has_sh else None,
            grad_colors_precomp if has_col else None,
            grad_opacities,
            grad_scales if has_s else None,
            grad_rotations if has_r else None,
            grad_cov3Ds_precomp if has_cov else None,
            None,
            None,
            grad_extra,
            None,
            None,
            None,
            None,
        )


class GaussianRasterizer(nn.Module):
    def __init__(self, raster_settings):
        super().__init__()
        self.raster_settings = raster_settings

    def markVisible(self, positions):
        """Boolean mask of points passing the near-plane test (checkFrustum, rasterizer_impl.cu:54-66)."""
        with torch.no_grad():
            rs = self.raster_settings
            if not positions.is_cuda:
                raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
            device = positions.device
            pos = _f32c(positions, device, "positions")
            view = _f32c(rs.viewmatrix, device, "viewmatrix")
            proj = _f32c(rs.projmatrix, device, "projmatrix")
            P = pos.size(0)
            present = torch.empty((P,), dtype=torch.bool, device=device)
            with torch.cuda.device(device):
                _lib.check(_lib.lib().fb200_mark_visible(
                    P, ptr(pos), ptr(view), ptr(proj), ptr(present), _lib.stream(device)))
        return present

    def forward(self, means3D, means2D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                cov3D_precomp=None, visibility_mask=None, extra_features=None, extra_background=None,
                face_visibility=None, return_alpha=False):
        """Reference surface (`__init__.py:187-220`) plus opt-in extensions: `visibility_mask` (row a19; per-Gaussian mask)
        or `face_visibility=(face_visible[F], point_cell_indices[n])` (row f1: the same occlusion culling looked up inside
        preprocess -- no mask tensor, no mask kernel; Gaussians beyond the n mesh-bound ones always render),
        `return_alpha=True` (appends the accumulated opacity 1 - final_T [H,W], detached -- the alpha of BASELINE's
        "RGB/depth/alpha"; a DIFFERENTIABLE alpha is `extra_features=ones[P,1]`, depth is `extra_features=view-space z`) and
        `extra_features` [P, 1..3] (row f4) -- blended with the colour's weights in the same traversal; when given, a
        third output `[E, H, W]` is returned (what a second call with `colors_precomp=extra_features` and
        `bg=extra_background` would return, sugar_model.py:2343-2387)."""
        raster_settings = self.raster_settings

        if (shs is None and colors_precomp is None) or (shs is not None and colors_precomp is not None):
            raise Exception('Please provide excatly one of either SHs or precomputed colors!')

        if ((scales is None or rotations is None) and cov3D_precomp is None) or \
                ((scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise Exception('Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!')

        if shs is None:
            shs = torch.Tensor([])
        if colors_precomp is None:
            colors_precomp = torch.Tensor([])
        if scales is None:
            scales = torch.Tensor([])
        if rotations is None:
            rotations = torch.Tensor([])
        if cov3D_precomp is None:
            cov3D_precomp = torch.Tensor([])

        return rasterize_gaussians(means3D, means2D, shs, colors_precomp, opacities, scales, rotations,
                                   cov3D_precomp, raster_settings, visibility_mask, extra_features, extra_background,
                                   face_visibility, return_alpha)


# ---- introspection for parity tests ----------------------------------------------------------------------
def forward_with_state(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
                       rotations=None, cov3D_precomp=None, visibility_mask=None):
    """Run the forward and expose the internal arrays (no autograd): used by tests to compare depth
    bits, rects, records, ranges and the sorted point list with the reference's buffers."""
    e = torch.Tensor([])
    with torch.no_grad():
        color, radii, call, _ = _launch_forward(
            means3D, e if shs is None else shs, e if colors_precomp is None else colors_precomp, opacities,
            e if scales is None else scales, e if rotations is None else rotations,
            e if cov3D_precomp is None else cov3D_precomp, raster_settings, visibility_mask, exact=True)
    prm, R = call.prm, call.num_rendered
    v = _lib.workspace_views(call.geom, call.image, call.binning, prm.P, prm.image_width, prm.image_height,
                             call.capacity, R)
    return dict(color=color, radii=radii, num_rendered=R, call=call,
                **{k: v[k] for k in ("rec", "depth", "rect", "clamped", "final_T", "n_contrib", "ranges", "tile_count",
                                     "point_list", "keys")})


def geometry_state(raster_settings, means3D, opacities, shs=None, colors_precomp=None, scales=None, rotations=None,
                   cov3D_precomp=None, visibility_mask=None):
    """Geometry phase only (preprocess + tile scan, `fb200_forward_geometry`): radii, depth bits, tile rects, per-tile
    counts and the instance count, without binning or blending -- the preprocess sweep of the parity tests."""
    e = torch.Tensor([])
    with torch.no_grad():
        _, radii, call, _ = _launch_forward(
            means3D, e if shs is None else shs, e if colors_precomp is None else colors_precomp, opacities,
            e if scales is None else scales, e if rotations is None else rotations,
            e if cov3D_precomp is None else cov3D_precomp, raster_settings, visibility_mask, geometry_only=True)
    prm = call.prm
    v = _lib.workspace_views(call.geom, call.image, None, prm.P, prm.image_width, prm.image_height, 0, 0)
    return dict(radii=radii, num_rendered=call.num_rendered, call=call,
                **{k: v[k] for k in ("depth", "rect", "rec", "tile_count")})
