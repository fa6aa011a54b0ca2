"""Rendering edited and animated Frosting scenes (SURVEY.md row a21) -- host side.

Frosting's headline use renders a scene whose base mesh has been edited or animated (render_blender_scene.py ->
blender/frosting_utils.py:551-588 render_composited_image) with the model made editable by
`make_editable(use_simple_adapt=True, ...)` (frosting_model.py:1013-1054).  Every frame then rebuilds the shell from the
deformed base mesh, rotates and rescales the Gaussians of edited faces, drops those of over-stretched faces and evaluates
the SH colours at view directions rotated back into each Gaussian's original frame -- dozens of torch kernels and
several host read-backs per frame in the reference.  Here:

    edit = FrostingEdit(ref_base_verts, faces, cells, inner_dist, outer_dist, edition_mask, thickness_rescaling="median")
    image, radii = frosting_render_edited(params, edit, frame_base_verts, raster_settings, orig_quats=...)

is two CUDA calls (csrc/frosting_edit.cu: shell + tables, then the per-Gaussian attributes) and the existing rasterizer
forward with precomputed colours.  The complex adaptation (`make_editable(use_simple_adapt=False)`, per-Gaussian
canonical transforms) is `FrostingEditComplex(params, ref_base_verts, faces, ...)`, used the same way.  Forward only.
"""
import ctypes as C

import torch

from . import _lib
from . import rasterizer as R
from ._lib import ptr, stream
from .frosting_render import FrostingBlock

RESCALING = {"median": _lib.RESCALE_MEDIAN, "triangle": _lib.RESCALE_TRIANGLE}


class FrostingEdit:
    """The reference state of `make_editable(use_simple_adapt=True, edition_mask, thickness_rescaling_method)`, captured on
    the device from the reference base vertices: face quaternions, vertex-to-centroid distances, their median (median
    method), the face / vertex edition masks and the vertex -> face adjacency.  `inner_dist` / `outer_dist` [V]: the
    shell offsets along the vertex normal (Frosting's _inner_dist / _outer_dist).  The tables of the last frame
    (`dists`, `rel_quats`, `face_factor`, `face_keep`, `factor`) stay readable on the object."""

    def __init__(self, base_verts, faces, cells, inner_dist, outer_dist, edition_mask=None, thickness_rescaling="median",
                 adaptation="simple"):
        if adaptation != "simple":
            raise NotImplementedError(f"adaptation {adaptation!r}: FrostingEdit is the simple adaptation "
                                      "(use_simple_adapt=True); the complex one is FrostingEditComplex")
        if thickness_rescaling not in RESCALING:
            raise ValueError(f"thickness rescaling method {thickness_rescaling!r} is not recognized "
                             f"(one of {sorted(RESCALING)})")
        if not base_verts.is_cuda:
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        dev = base_verts.device
        self.device, self.rescaling = dev, thickness_rescaling
        self.faces = faces.to(device=dev, dtype=torch.int32).contiguous()
        self.cells = cells.to(device=dev, dtype=torch.int64).contiguous()
        V, F = base_verts.shape[0], self.faces.shape[0]
        self.n_verts, self.n_faces = V, F
        f32 = lambda t, what: R._f32c(t, dev, what)
        self.inner_dist, self.outer_dist = f32(inner_dist.reshape(-1), "inner_dist"), f32(outer_dist.reshape(-1), "outer_dist")
        if self.inner_dist.numel() != V or self.outer_dist.numel() != V:
            raise ValueError("inner_dist / outer_dist need one value per base vertex")
        em = torch.ones(F, dtype=torch.bool, device=dev) if edition_mask is None else edition_mask.to(dev).bool()
        if em.numel() != F:
            raise ValueError("edition_mask needs one value per face")
        self.edition_mask = em.to(torch.uint8).contiguous()
        self.n_edited = int(em.sum())
        if thickness_rescaling == "median" and self.n_edited == 0:
            raise ValueError("median thickness rescaling needs at least one edited face")
        flat = self.faces.long().reshape(-1)
        vmask = torch.zeros(V, dtype=torch.uint8, device=dev)
        vmask[self.faces.long()[em].reshape(-1)] = 1
        self.verts_edition_mask = vmask
        # vertex -> face CSR, faces ascending per vertex: the vertex pass sums in this fixed order
        order = torch.sort(flat, stable=True).indices
        self.vf_faces = (order // 3).to(torch.int32).contiguous()
        self.vf_offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=dev),
                                     torch.bincount(flat, minlength=V).cumsum(0)]).to(torch.int32).contiguous()
        o = dict(dtype=torch.float32, device=dev)
        self.dists, self.face_normals = torch.empty((F, 3), **o), torch.empty((F, 3), **o)
        self.rel_quats, self.face_factor = torch.empty((F, 4), **o), torch.empty((F,), **o)
        self.face_keep = torch.empty((F,), dtype=torch.uint8, device=dev)
        self.factor = torch.ones((2,), **o)
        self._select = torch.empty((_lib.EDIT_SELECT_WORDS,), dtype=torch.int32, device=dev)
        self.ref_quats = self.ref_dists = self.ref_median = None
        self._capture(f32(base_verts, "base_verts"))

    def _capture(self, base_verts):
        """Reference capture: the same kernels over the reference vertices, so an unedited frame reproduces them bit for
        bit.  Returns the capture's struct and shell."""
        st, inner, outer = self._shell(base_verts, 2.0)
        self.ref_quats, self.ref_dists = self.rel_quats.clone(), self.dists.clone()
        self.ref_median = self.factor[:1].clone() if self.rescaling == "median" else None
        return st, inner, outer

    def _struct(self, base_verts, threshold, inner, outer):
        return _lib.FrostingEdit(
            n_verts=self.n_verts, n_faces=self.n_faces, rescaling=RESCALING[self.rescaling], n_edited=self.n_edited,
            deformation_threshold=float(threshold), d_base_verts=ptr(base_verts), d_faces=ptr(self.faces),
            d_inner_dist=ptr(self.inner_dist), d_outer_dist=ptr(self.outer_dist), d_edition_mask=ptr(self.edition_mask),
            d_verts_edition_mask=ptr(self.verts_edition_mask), d_vf_offsets=ptr(self.vf_offsets),
            d_vf_faces=ptr(self.vf_faces), d_ref_quats=ptr(self.ref_quats), d_ref_dists=ptr(self.ref_dists),
            d_ref_median=ptr(self.ref_median), d_dists=ptr(self.dists), d_face_normals=ptr(self.face_normals),
            d_rel_quats=ptr(self.rel_quats), d_face_factor=ptr(self.face_factor), d_face_keep=ptr(self.face_keep),
            d_factor=ptr(self.factor), d_select=ptr(self._select), d_inner_verts=ptr(inner), d_outer_verts=ptr(outer))

    def _shell(self, base_verts, threshold):
        if base_verts.shape != (self.n_verts, 3):
            raise ValueError(f"base_verts must be [{self.n_verts}, 3]")
        o = dict(dtype=torch.float32, device=self.device)
        inner, outer = torch.empty((self.n_verts, 3), **o), torch.empty((self.n_verts, 3), **o)
        st = self._struct(base_verts, threshold, inner, outer)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().fb200_frosting_edit_shell(C.byref(st), stream(self.device)))
        return st, inner, outer

    def shell(self, base_verts, deformation_threshold=2.0):
        """The frame's shell (inner, outer) [V,3] from its base vertices; updates the face tables."""
        _, inner, outer = self._shell(R._f32c(base_verts, self.device, "base_verts"), deformation_threshold)
        return inner, outer

    def _block(self, params, inner, outer, face_visible):
        blk = FrostingBlock(params, dict(inner=inner, outer=outer, cells=self.cells, faces=self.faces), face_visible)
        if blk.n_mesh != self.cells.numel():
            raise ValueError("params have a different number of mesh-bound Gaussians than the edit's cells")
        return blk

    def _launch_attributes(self, st, blk, sh_degree, cp, oq, outs):
        _lib.check(_lib.lib().fb200_frosting_edit_attributes(C.byref(st), C.byref(blk.fp), int(sh_degree), ptr(cp),
                                                              ptr(oq), *(ptr(t) for t in outs), stream(blk.device)))

    @torch.no_grad()
    def attributes(self, params, base_verts, campos, sh_degree, orig_quats=None, deformation_threshold=2.0,
                   face_visible=None):
        """Rasterizer inputs of one frame: means3D, opacities, scales, rotations, colors_precomp ([P + n_bg] rows,
        background rows last) and the frame's shell (inner, outer).  `params`: the keys of `frosting_render` (bg_*
        included).  `orig_quats` [P + n_bg, 4]: the rotations the SH were fitted in (Frosting's original_quaternions
        with original_bg_quaternions); None: SH evaluated at unrotated view directions.  `face_visible` [F]: mesh rows of
        culled faces are skipped (zero rows)."""
        base_verts = R._f32c(base_verts, self.device, "base_verts")
        st, inner, outer = self._shell(base_verts, deformation_threshold)
        blk = self._block(params, inner, outer, face_visible)
        dev, rows = blk.device, blk.rows
        oq = None
        if orig_quats is not None:
            oq = R._f32c(orig_quats, dev, "orig_quats")
            if oq.shape != (rows, 4):
                raise ValueError(f"orig_quats must be [{rows}, 4] (mesh rows, then background rows)")
        cp = R._f32c(campos.reshape(-1), dev, "campos")
        o = dict(dtype=torch.float32, device=dev)
        alloc = torch.empty if face_visible is None else torch.zeros
        means3D, opac, scales = alloc((rows, 3), **o), alloc((rows, 1), **o), alloc((rows, 3), **o)
        rots, colors = alloc((rows, 4), **o), alloc((rows, 3), **o)
        with torch.cuda.device(dev):
            self._launch_attributes(st, blk, sh_degree, cp, oq, (means3D, opac, scales, rots, colors))
        return dict(means3D=means3D, opacities=opac, scales=scales, rotations=rots, colors_precomp=colors,
                    inner=inner, outer=outer)


class FrostingEditComplex(FrostingEdit):
    """The reference state of `make_editable(use_simple_adapt=False, edition_mask, thickness_rescaling_method)` -- the
    complex adaptation, the default of make_editable and of Frosting's Blender pipeline.  On top of FrostingEdit's
    capture, each edited Gaussian keeps a canonical transform C = T_ref[cell]^-1 R(q) diag(exp(s)) from the `params`
    given here (`quats`, `log_scales`), where T maps a canonical cell to the world (two orthogonalised in-plane axes and
    the normal scaled by the median distance).  Per frame the scales are the column norms of T_frame[cell] C and the
    rotation is that matrix's; shell, positions, opacities, background rows and colours follow the simple path.
    `cell_T` [F,3,3] (the last frame's, edited faces) and `canonical` [P,3,3] (0 on unedited rows) stay readable.
    Raises ValueError when an edited Gaussian's reference cell is singular (a degenerate edited face), as the
    reference's solve does.  Rebuild it when the Gaussians' rotations or scales change."""

    def __init__(self, params, base_verts, faces, cells, inner_dist, outer_dist, edition_mask=None,
                 thickness_rescaling="median"):
        self._capture_params = params
        super().__init__(base_verts, faces, cells, inner_dist, outer_dist, edition_mask=edition_mask,
                         thickness_rescaling=thickness_rescaling)
        del self._capture_params

    def _capture(self, base_verts):
        # after the reference shell, d_dists / d_factor[0] hold the reference distances and median the cells scale by
        st, inner, outer = super()._capture(base_verts)
        blk = self._block(self._capture_params, inner, outer, None)
        dev = blk.device
        o = dict(dtype=torch.float32, device=dev)
        self.cell_T = torch.zeros((self.n_faces, 3, 3), **o)
        self.canonical = torch.empty((blk.n_mesh, 3, 3), **o)
        n_singular = torch.empty((1,), dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().fb200_frosting_edit_complex_capture(
                C.byref(st), C.byref(blk.fp), ptr(self.cell_T), ptr(self.canonical), ptr(n_singular), stream(dev)))
        n = int(n_singular.item())                      # the one host read-back, at capture only
        if n:
            raise ValueError(f"{n} edited Gaussian(s) sit on faces whose cell transformation is singular even after "
                             "the fix-up (degenerate edited faces): their canonical transforms are undefined")
        return st, inner, outer

    def _launch_attributes(self, st, blk, sh_degree, cp, oq, outs):
        _lib.check(_lib.lib().fb200_frosting_edit_attributes_complex(
            C.byref(st), C.byref(blk.fp), int(sh_degree), ptr(cp), ptr(oq), ptr(self.canonical), ptr(self.cell_T),
            *(ptr(t) for t in outs), stream(blk.device)))


@torch.no_grad()
def frosting_render_edited(params, edit, base_verts, raster_settings, orig_quats=None, deformation_threshold=2.0,
                           face_visible=None):
    """One frame of an edited / animated Frosting scene: `edit.attributes` then the rasterizer forward with precomputed
    colours (culling by `face_visible[cells[i]]` inside preprocess when given).  Returns (image [3,H,W], radii
    [P + n_bg])."""
    rs = raster_settings
    a = edit.attributes(params, base_verts, rs.campos, rs.sh_degree, orig_quats=orig_quats,
                        deformation_threshold=deformation_threshold, face_visible=face_visible)
    e = torch.Tensor([])
    color, radii, _, _ = R._launch_forward(
        a["means3D"], e, a["colors_precomp"], a["opacities"], a["scales"], a["rotations"], e, rs, None,
        face_visibility=(face_visible, edit.cells) if face_visible is not None else None)
    return color, radii
