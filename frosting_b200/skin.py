"""Posing Blender-animated Frosting scenes from their bone tracks -- host side of csrc/frosting_skin.cu.

Frosting's animated frame starts with `apply_poses_to_scene` (blender/frosting_utils.py:474-516): linear-blend skinning
of the rigged meshes' T-pose points into the base vertices, per bone a torch.inverse, two transform_points and an index
+= (hundreds of small kernels and one host synchronisation per bone, every frame).  Here:

    skin = FrostingSkin(package, ref_indices, n_verts, device)      # once: tables on the device
    skin.pose(i_frame, base_verts)                                  # per frame: one launch, in place

`package` is what load_blender_package returns (only the rig is read: `bones`, `bone_to_vertices`,
`bone_to_vertex_weights`, `camera.lens` for the frame count); `ref_indices` the composite mesh's per-mesh vertex starts
(build_composite_scene).  Forward only.
"""
import ctypes as C

import torch

from . import _lib
from .frosting_render import _p, _stream


def skin_tables(package, ref_indices, n_verts):
    """The rig of a processed package as flat tables (CPU tensors), in the reference's summation order.

    Rows are the rigged vertices, mesh by mesh (`vert_ids` int32: their base-vertex index; `tpose` [R,3]).  Row i's
    entries [offsets[i], offsets[i+1]) are its (bones int32, weights float64) pairs in rest_bones order.  Bones are those
    with vertices, numbered in package order (`bone_names`: (mesh, name)); `rest_t` [B,4,4] is rest^T and `pose`
    [B,n_frames,4,4] the tracks' first n_frames matrices transposed -- both as the reference hands them to Transform3d.
    Raises ValueError when a range disagrees with its tpose_points, or a used track is shorter than n_frames."""
    n_frames = len(package["camera"]["lens"])
    meshes = package["bones"]
    if len(ref_indices) < len(meshes) + 1:
        raise ValueError(f"ref_indices needs {len(meshes) + 1} entries (one start per mesh, then the end)")
    tpose, vert_ids, rows, bones, weights, rest_t, pose, names = [], [], [], [], [], [], [], []
    n_rows = 0
    for i, mesh_dict in enumerate(meshes):
        if not mesh_dict:
            continue
        start, end = int(ref_indices[i]), int(ref_indices[i + 1])
        tp = mesh_dict["vertex"]["tpose_points"].detach().float().cpu()
        if not 0 <= start <= end <= n_verts or end - start != tp.shape[0]:
            raise ValueError(f"mesh {i}: vertex range [{start}, {end}) does not hold its {tp.shape[0]} tpose_points "
                             f"within the {n_verts} base vertices")
        arm = mesh_dict["armature"]
        for name in arm["rest_bones"]:
            idx = package["bone_to_vertices"][i][name]
            if len(idx) == 0:
                continue
            track = arm["pose_bones"][name]
            if track.shape[0] < n_frames:
                raise ValueError(f"mesh {i}, bone {name!r}: pose track of {track.shape[0]} frames, the animation has "
                                 f"{n_frames}")
            idx = idx.detach().long().cpu()
            if int(idx.min()) < 0 or int(idx.max()) >= tp.shape[0]:
                raise ValueError(f"mesh {i}, bone {name!r}: vertex index outside its {tp.shape[0]} tpose_points")
            rows.append(idx + n_rows)
            bones.append(torch.full_like(idx, len(names)))
            weights.append(package["bone_to_vertex_weights"][i][name].detach().cpu().double().reshape(-1))
            rest_t.append(arm["rest_bones"][name].detach().float().cpu().transpose(-1, -2))
            pose.append(track[:n_frames].detach().float().cpu().transpose(-1, -2))
            names.append((i, name))
        tpose.append(tp)
        vert_ids.append(torch.arange(start, end))
        n_rows += tp.shape[0]
    cat = lambda ts, empty: torch.cat(ts) if ts else empty
    rows = cat(rows, torch.zeros(0, dtype=torch.long))
    order = torch.sort(rows, stable=True).indices           # per row, entries stay in bone order
    return dict(
        tpose=cat(tpose, torch.zeros(0, 3)).contiguous(),
        vert_ids=cat(vert_ids, torch.zeros(0, dtype=torch.long)).to(torch.int32),
        offsets=torch.cat([torch.zeros(1, dtype=torch.long),
                           torch.bincount(rows, minlength=n_rows).cumsum(0)]).to(torch.int32),
        bones=cat(bones, torch.zeros(0, dtype=torch.long))[order].to(torch.int32),
        weights=cat(weights, torch.zeros(0, dtype=torch.float64))[order],
        rest_t=cat([m[None] for m in rest_t], torch.zeros(0, 4, 4)).contiguous(),
        pose=cat([m[None] for m in pose], torch.zeros(0, n_frames, 4, 4)).contiguous(),
        bone_names=names, n_frames=n_frames)


class FrostingSkin:
    """The rig of a processed Blender package on the device: the tables of `skin_tables` (its `pose` as `tracks`) and
    the reset matrices inverse(rest^T), computed once with torch.linalg.inv (the function the reference calls for every
    bone and frame)."""

    def __init__(self, package, ref_indices, n_verts, device):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("frosting_b200 runs on CUDA tensors only (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        t = skin_tables(package, ref_indices, n_verts)
        self.n_verts, self.n_frames, self.bone_names = int(n_verts), t["n_frames"], t["bone_names"]
        for k in ("tpose", "vert_ids", "offsets", "bones", "weights"):
            setattr(self, k, t[k].to(self.device).contiguous())
        self.tracks = t["pose"].to(self.device).contiguous()
        self.reset = torch.linalg.inv(t["rest_t"].to(self.device)).contiguous()
        self._st = _lib.FrostingSkin(
            n_rows=self.vert_ids.numel(), n_verts=self.n_verts, n_bones=len(self.bone_names), n_frames=self.n_frames,
            d_tpose=_p(self.tpose), d_vert_ids=_p(self.vert_ids), d_offsets=_p(self.offsets), d_bones=_p(self.bones),
            d_weights=_p(self.weights), d_reset=_p(self.reset), d_pose=_p(self.tracks))

    @torch.no_grad()
    def pose(self, i_frame, base_verts):
        """Writes frame `i_frame` (wrapped: i_frame % n_frames) of every rigged range into `base_verts` [n_verts,3]
        (float32, contiguous, on the skin's device) in place and returns it; other ranges are untouched."""
        if base_verts.device != self.device or base_verts.dtype != torch.float32 or not base_verts.is_contiguous() \
                or tuple(base_verts.shape) != (self.n_verts, 3):
            raise ValueError(f"base_verts must be a contiguous float32 [{self.n_verts}, 3] tensor on {self.device}")
        if self.n_frames == 0:
            raise ValueError("the package has no frames")
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().fb200_frosting_skin_pose(C.byref(self._st), int(i_frame) % self.n_frames,
                                                           _p(base_verts), _stream(self.device)))
        return base_verts
