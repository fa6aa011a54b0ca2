"""Golden vectors for one frame of an EDITED Frosting scene, simple adaptation (SURVEY.md row a21), produced by EXECUTING
the reference's own source.

The per-frame chain of render_blender_scene.py is cut out of the reference with `ast` and compiled unmodified:
  frosting_scene/frosting_model.py   device, shell_base, shell_base_normals, outer_verts, inner_verts,
                                     shell_cells_verts, bary_coords, points, strengths, sh_coordinates, scaling,
                                     quaternions, bg_* properties, compute_face_quaternions, make_editable (its simple
                                     branch runs), get_points_rgb
  blender/frosting_utils.py          _get_edited_points_deformation_mask, get_frosting_sh_rotations
  frosting_utils/spherical_harmonics.py   eval_sh (the whole module: plain torch / numpy)
and driven as render_composited_image drives it (blender/frosting_utils.py:566-588, the directions of
frosting_model.py:1482).  pytorch3d is not installed: Meshes' normals and the quaternion helpers are supplied from
frosting_b200/scenes.py, which restates them from pytorch3d's documented maths -- those pieces are restated, not pinned.

    python tests/golden/make_frosting_edit_golden.py        # writes tests/golden/frosting_edit.npz

The checkout is found as oracle/build_ref.py finds it ($FROSTING_REFERENCE, else `reference/` beside the repository).
"""
import ast
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402
from frosting_b200 import scenes                 # noqa: E402

MODEL_WANT = ("device", "shell_base", "shell_base_normals", "outer_verts", "inner_verts", "shell_cells_verts",
              "bary_coords", "points", "strengths", "sh_coordinates", "scaling", "quaternions", "bg_points",
              "bg_strengths", "bg_sh_coordinates", "bg_scaling", "bg_quaternions", "compute_face_quaternions",
              "make_editable", "get_points_rgb")
BLENDER_WANT = ("_get_edited_points_deformation_mask", "get_frosting_sh_rotations")

# (name, thickness rescaling, partial edition mask, background Gaussians, sh_degree)
CASES = (("median_full_bg_d3", "median", False, True, 3),
         ("triangle_partial_d1", "triangle", True, False, 1),
         ("triangle_full_bg_d3", "triangle", False, True, 3),
         ("median_partial_d1", "median", True, False, 1))


class Meshes:
    """The two normals of pytorch3d's Meshes the chain reads (restated: scenes.p3d_*)."""

    def __init__(self, verts, faces):
        self._v, self._f = verts[0], faces[0]

    def verts_normals_list(self):
        return [scenes.p3d_verts_normals(self._v, self._f)]

    def faces_normals_list(self):
        return [scenes.p3d_faces_normals(self._v, self._f)]


def _cut(path, want, cls_name=None):
    src = open(path).read()
    tree = ast.parse(src)
    body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name).body if cls_name else tree.body
    lines = src.splitlines()
    chunks = []
    for n in body:
        if isinstance(n, ast.FunctionDef) and n.name in want:
            first = min([d.lineno for d in n.decorator_list] + [n.lineno])
            chunks.append("\n".join(lines[first - 1:n.end_lineno]))
    assert len(chunks) == len(want), (path, len(chunks))
    return chunks


def reference_namespace():
    ref = reference_dir()
    model = os.path.join(ref, "frosting_scene", "frosting_model.py")
    blender = os.path.join(ref, "blender", "frosting_utils.py")
    sh = os.path.join(ref, "frosting_utils", "spherical_harmonics.py")
    for p in (model, blender, sh):
        if not os.path.exists(p):
            raise SystemExit(f"{p} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    ns = {"torch": torch, "Meshes": Meshes, "torch_normalize": torch.nn.functional.normalize,
          "matrix_to_quaternion": scenes.matrix_to_quaternion, "quaternion_multiply": scenes.quaternion_multiply,
          "quaternion_invert": scenes.quaternion_invert, "quaternion_to_matrix": scenes.quaternion_to_matrix,
          "Frosting": object}
    exec(compile(open(sh).read(), sh, "exec"), ns)                     # eval_sh and its constants
    code = "class RefFrosting:\n" + "\n\n".join(_cut(model, MODEL_WANT, "Frosting")) + "\n"
    exec(compile(code, model, "exec"), ns)
    exec(compile("\n\n".join(_cut(blender, BLENDER_WANT)) + "\n", blender, "exec"), ns)
    return ns


N_BG = 48


def make_scene(seed=31):
    """One small layer (1000 mesh-bound Gaussians, 272 faces, N_BG background Gaussians), deformed; shared by every case
    (a case without background Gaussians uses the mesh rows only), so the parameters are stored once."""
    cam = scenes.make_camera(160, 96)
    params, mesh = scenes.frosting_layer(1000, cam, seed, n_faces_target=300, n_background=N_BG)
    thickness = 0.02
    V, F = mesh["verts"].shape[0], mesh["faces"].shape[0]
    g = torch.Generator().manual_seed(seed + 1)
    quats_all = torch.cat([params["quats"], params["bg_quats"]])
    return dict(params=params, ref_verts=mesh["verts"], verts=scenes.deform_base(mesh["verts"]), faces=mesh["faces"],
                cells=mesh["cells"], inner_dist=-thickness * (1.0 + 0.2 * torch.rand(V, generator=g)),
                outer_dist=thickness * (1.0 + 0.2 * torch.rand(V, generator=g)),
                partial_mask=torch.rand(F, generator=g) < 0.6,
                orig_quats=torch.nn.functional.normalize(quats_all + 0.3 * torch.randn(quats_all.shape, generator=g),
                                                         dim=-1),
                campos=torch.tensor([0.4, -0.3, 0.5]))


def scene_params(scene, with_bg):
    params = scene["params"]
    return params if with_bg else {k: v for k, v in params.items() if not k.startswith("bg_")}


def run_case(ns, scene, name, method, partial, with_bg, deg):
    params = scene_params(scene, with_bg)
    n_bg = N_BG if with_bg else 0
    ref_verts, verts, faces, cells = scene["ref_verts"], scene["verts"], scene["faces"], scene["cells"]
    inner_dist, outer_dist, campos = scene["inner_dist"], scene["outer_dist"], scene["campos"]
    F = faces.shape[0]
    em = scene["partial_mask"] if partial else torch.ones(F, dtype=torch.bool)
    P = params["quats"].shape[0]
    orig = scene["orig_quats"][:P + n_bg]

    m = ns["RefFrosting"]()
    m.editable, m.use_softmax_for_bary_coords, m.positions_are_absolute = False, True, False
    m.scale_activation, m.sh_levels = torch.exp, 4
    m.use_background_gaussians, m.use_background_sphere = n_bg > 0, False
    m._shell_base_verts, m._shell_base_faces, m._point_cell_indices = ref_verts.clone(), faces.long(), cells
    m._inner_dist, m._outer_dist = inner_dist, outer_dist
    m._bary_coords, m._opacities = params["bary_logits"], params["opacity_logits"]
    m._scales, m._quaternions = params["log_scales"], params["quats"]
    m._sh_coordinates_dc, m._sh_coordinates_rest = params["sh_dc"], params["sh_rest"]
    if n_bg:
        m._bg_points, m._bg_opacities = params["bg_points"], params["bg_opacity_logits"][:, None]
        m._bg_scales, m._bg_quaternions = params["bg_log_scales"], params["bg_quats"]
        m._bg_sh_coordinates_dc, m._bg_sh_coordinates_rest = params["bg_sh_dc"], params["bg_sh_rest"]
    P = params["quats"].shape[0]
    m.original_quaternions, m.original_bg_quaternions = orig[:P], orig[P:]
    m.make_editable(use_simple_adapt=True, edition_mask=em, thickness_rescaling_method=method)
    m._shell_base_verts = verts                                         # the frame's pose (apply_poses_to_scene)

    # render_composited_image (blender/frosting_utils.py:566-588) -> render_image_gaussian_rasterizer (:1470-1514)
    with torch.no_grad():
        keep = torch.ones(P, dtype=torch.bool)
        keep[m._gaussian_edition_mask] = ns["_get_edited_points_deformation_mask"](m, threshold=2.0)
        opac = m.strengths.view(-1, 1)
        opac[~keep] = 0.0
        pos, quats, scales = m.points, m.quaternions, m.scaling
        if n_bg:
            opac = torch.cat([opac, m.bg_strengths.view(-1, 1)])
            pos, quats, scales = torch.cat([pos, m.bg_points]), torch.cat([quats, m.bg_quaternions]), torch.cat([scales, m.bg_scaling])
        sh_rot = ns["get_frosting_sh_rotations"](m)
        dirs = (torch.nn.functional.normalize(pos - campos, dim=-1).unsqueeze(1) @ sh_rot)[..., 0, :]
        colors = m.get_points_rgb(positions=pos, camera_centers=None, directions=dirs, sh_levels=deg + 1)
        out = dict(inner=m.inner_verts, outer=m.outer_verts, means3D=pos, opacities=opac, scales=scales,
                   rotations=quats, colors=colors)
    save = {f"{name}/{k}": v for k, v in dict(
        edition_mask=em.numpy(), sh_degree=np.int32(deg), rescaling=np.array(method), background=np.bool_(with_bg)).items()}
    save.update({f"{name}/out_{k}": v.detach().numpy() for k, v in out.items()})
    return save


def main():
    ns = reference_namespace()
    scene = make_scene()
    save = {f"scene/param_{k}": v.numpy() for k, v in scene["params"].items()}
    save.update({f"scene/{k}": scene[k].numpy() for k in ("ref_verts", "verts", "faces", "cells", "inner_dist",
                                                         "outer_dist", "orig_quats", "campos")})
    for case in CASES:
        save.update(run_case(ns, scene, *case))
    np.savez_compressed(os.path.join(HERE, "frosting_edit.npz"), **save)
    print(sorted({k.split("/")[0] for k in save}), sum(v.nbytes for v in save.values()), "bytes")


if __name__ == "__main__":
    main()
