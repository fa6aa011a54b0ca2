"""Golden vectors for one frame of an EDITED Frosting scene, complex adaptation (make_editable(use_simple_adapt=False),
SURVEY.md row a21), produced by EXECUTING the reference's own source.

On top of what tests/golden/make_frosting_edit_golden.py cuts out of frosting_scene/frosting_model.py, this takes
compute_cell_transformations, get_edited_quaternions_and_scales and make_editable's complex branch, unmodified, and
supplies the module globals they read (`np`, `scale_activation = torch.exp`) and `faces_normals_packed` on the same
Meshes shim.  The scene, the four cases (median / triangle, full / partial edition mask, background Gaussians or none,
SH degree 3 / 1) and the driving of render_composited_image are those of the simple generator.  Besides the frame's
outputs each case stores the canonical transforms ([P,3,3], zero on unedited rows) and the frame's cell transforms
([F,3,3], zero on unedited faces).

    python tests/golden/make_frosting_edit_complex_golden.py    # writes tests/golden/frosting_edit_complex.npz
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_frosting_edit_golden as simple      # noqa: E402
from make_frosting_edit_golden import scenes     # noqa: E402

MODEL_WANT = simple.MODEL_WANT + ("compute_cell_transformations", "get_edited_quaternions_and_scales")


class Meshes(simple.Meshes):
    def faces_normals_packed(self):
        return scenes.p3d_faces_normals(self._v, self._f)


def reference_namespace():
    ref = simple.reference_dir()
    model = os.path.join(ref, "frosting_scene", "frosting_model.py")
    blender = os.path.join(ref, "blender", "frosting_utils.py")
    sh = os.path.join(ref, "frosting_utils", "spherical_harmonics.py")
    for p in (model, blender, sh):
        if not os.path.exists(p):
            raise SystemExit(f"{p} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    ns = {"torch": torch, "np": np, "Meshes": Meshes, "torch_normalize": torch.nn.functional.normalize,
          "scale_activation": torch.exp, "matrix_to_quaternion": scenes.matrix_to_quaternion,
          "quaternion_multiply": scenes.quaternion_multiply, "quaternion_invert": scenes.quaternion_invert,
          "quaternion_to_matrix": scenes.quaternion_to_matrix, "Frosting": object}
    exec(compile(open(sh).read(), sh, "exec"), ns)
    code = "class RefFrosting:\n" + "\n\n".join(simple._cut(model, MODEL_WANT, "Frosting")) + "\n"
    exec(compile(code, model, "exec"), ns)
    exec(compile("\n\n".join(simple._cut(blender, simple.BLENDER_WANT)) + "\n", blender, "exec"), ns)
    return ns


def run_case(ns, scene, name, method, partial, with_bg, deg):
    params = simple.scene_params(scene, with_bg)
    n_bg = simple.N_BG if with_bg else 0
    ref_verts, verts, faces, cells = scene["ref_verts"], scene["verts"], scene["faces"], scene["cells"]
    F = faces.shape[0]
    em = scene["partial_mask"] if partial else torch.ones(F, dtype=torch.bool)
    P = params["quats"].shape[0]
    orig = scene["orig_quats"][:P + n_bg]

    m = ns["RefFrosting"]()
    m.editable, m.use_softmax_for_bary_coords, m.positions_are_absolute = False, True, False
    m.scale_activation, m.sh_levels = torch.exp, 4
    m.use_background_gaussians, m.use_background_sphere = n_bg > 0, False
    m._shell_base_verts, m._shell_base_faces, m._point_cell_indices = ref_verts.clone(), faces.long(), cells
    m._inner_dist, m._outer_dist = scene["inner_dist"], scene["outer_dist"]
    m._bary_coords, m._opacities = params["bary_logits"], params["opacity_logits"]
    m._scales, m._quaternions = params["log_scales"], params["quats"]
    m._sh_coordinates_dc, m._sh_coordinates_rest = params["sh_dc"], params["sh_rest"]
    if n_bg:
        m._bg_points, m._bg_opacities = params["bg_points"], params["bg_opacity_logits"][:, None]
        m._bg_scales, m._bg_quaternions = params["bg_log_scales"], params["bg_quats"]
        m._bg_sh_coordinates_dc, m._bg_sh_coordinates_rest = params["bg_sh_dc"], params["bg_sh_rest"]
    m.original_quaternions, m.original_bg_quaternions = orig[:P], orig[P:]
    m.make_editable(use_simple_adapt=False, edition_mask=em, thickness_rescaling_method=method)
    m._shell_base_verts = verts                                         # the frame's pose (apply_poses_to_scene)

    with torch.no_grad():
        keep = torch.ones(P, dtype=torch.bool)
        keep[m._gaussian_edition_mask] = ns["_get_edited_points_deformation_mask"](m, threshold=2.0)
        opac = m.strengths.view(-1, 1)
        opac[~keep] = 0.0
        # quaternions then scaling: the second property call takes the first's edited_cache, as a frame does
        pos, quats, scales = m.points, m.quaternions, m.scaling
        if n_bg:
            opac = torch.cat([opac, m.bg_strengths.view(-1, 1)])
            pos, quats, scales = torch.cat([pos, m.bg_points]), torch.cat([quats, m.bg_quaternions]), torch.cat([scales, m.bg_scaling])
        sh_rot = ns["get_frosting_sh_rotations"](m)
        dirs = (torch.nn.functional.normalize(pos - scene["campos"], dim=-1).unsqueeze(1) @ sh_rot)[..., 0, :]
        colors = m.get_points_rgb(positions=pos, camera_centers=None, directions=dirs, sh_levels=deg + 1)
        gem = m._gaussian_edition_mask
        canonical = torch.zeros(P, 3, 3)
        canonical[gem] = m.canonical_gaussian_transformations
        cell_T = torch.where(em[:, None, None], m.compute_cell_transformations(faces_mask=em), torch.zeros(F, 3, 3))
        out = dict(inner=m.inner_verts, outer=m.outer_verts, means3D=pos, opacities=opac, scales=scales,
                   rotations=quats, colors=colors, canonical=canonical, cell_T=cell_T)
    save = {f"{name}/{k}": v for k, v in dict(
        edition_mask=em.numpy(), sh_degree=np.int32(deg), rescaling=np.array(method), background=np.bool_(with_bg)).items()}
    save.update({f"{name}/out_{k}": v.detach().numpy() for k, v in out.items()})
    return save


def main():
    ns = reference_namespace()
    scene = simple.make_scene()
    save = {f"scene/param_{k}": v.numpy() for k, v in scene["params"].items()}
    save.update({f"scene/{k}": scene[k].numpy() for k in ("ref_verts", "verts", "faces", "cells", "inner_dist",
                                                         "outer_dist", "orig_quats", "campos")})
    for case in simple.CASES:
        save.update(run_case(ns, scene, *case))
    np.savez_compressed(os.path.join(HERE, "frosting_edit_complex.npz"), **save)
    print(sorted({k.split("/")[0] for k in save}), sum(v.nbytes for v in save.values()), "bytes")


if __name__ == "__main__":
    main()
