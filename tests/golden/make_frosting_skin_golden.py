"""Golden vectors for the bone skinning of a Blender-animated Frosting scene, produced by EXECUTING the reference's own
source.

`load_blender_package` and `apply_poses_to_scene` are cut out of the reference's blender/frosting_utils.py with `ast`
and compiled unmodified.  The package JSON they read is written here to a temporary file:
  - three meshes: two rigged with different armatures (4 and 3 bones, one of them without vertices, one with a pose
    track longer than the animation) and one without a rig between them;
  - vertices with one to four groups of their armature, unnormalised weights, groups of the other armature and a
    non-bone group (filtered out by load_blender_package), and vertices with no group of their own armature;
  - affine rest and pose matrices (rotation, translation, a mild non-uniform scale in the poses);
  - three animation frames, posed at frames 0, 1, 2 and 4 (the last wraps to 1).
pytorch3d is not installed: its Transform3d is supplied from frosting_b200/scenes.py, which restates it from pytorch3d's
documented maths -- that piece is restated, not pinned.

    python tests/golden/make_frosting_skin_golden.py        # writes tests/golden/frosting_skin.npz

The npz stores the processed package (what load_blender_package returns, per rigged mesh: tpose points, bone names,
rest matrices, pose tracks, each bone's vertex indices and float64 weights), the JSON it came from, the base vertices
before posing (the unrigged range included) and the base vertices after each posed frame.
The checkout is found as oracle/build_ref.py finds it ($FROSTING_REFERENCE, else `reference/` beside the repository).
"""
import ast
import json
import math
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle.build_ref import reference_dir      # noqa: E402
from frosting_b200 import scenes                 # noqa: E402

WANT = ("load_blender_package", "apply_poses_to_scene")
N_FRAMES = 3
FRAMES = (0, 1, 2, 4)
SIZES = (40, 25, 30)                              # mesh 1 has no rig


def reference_namespace():
    path = os.path.join(reference_dir(), "blender", "frosting_utils.py")
    if not os.path.exists(path):
        raise SystemExit(f"{path} not found: set FROSTING_REFERENCE to a checkout of Anttwo/Frosting")
    src = open(path).read()
    lines = src.splitlines()
    chunks = ["\n".join(lines[n.lineno - 1:n.end_lineno]) for n in ast.parse(src).body
              if isinstance(n, ast.FunctionDef) and n.name in WANT]
    assert len(chunks) == len(WANT)
    ns = {"torch": torch, "np": np, "json": json, "Transform3d": scenes.Transform3d, "Frosting": object}
    exec(compile("\n\n".join(chunks) + "\n", path, "exec"), ns)
    return ns


def _rigid(rng, scale=(1.0, 1.0, 1.0), shift=2.0):
    """A column-convention 4x4 (Blender's matrices): rotation about a random axis, scale, translation."""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    a = rng.uniform(-math.pi, math.pi)
    K = np.array([[0, -axis[2], axis[1]], [axis[2], 0, -axis[0]], [-axis[1], axis[0], 0]])
    m = np.eye(4)
    m[:3, :3] = (np.eye(3) + math.sin(a) * K + (1 - math.cos(a)) * K @ K) @ np.diag(scale)
    m[:3, 3] = rng.uniform(-shift, shift, size=3)
    return m


def _mesh(rng, n, own, other, no_group):
    """One rigged mesh's JSON: groups mixing its own bones (1..4), a bone of the other armature and a non-bone group."""
    groups, weights = [], []
    for v in range(n):
        k = 1 + v % 4
        g = list(rng.choice(own, size=min(k, len(own)), replace=False))
        if v % 5 == 2:
            g.insert(int(rng.integers(0, len(g) + 1)), other[v % len(other)])
        if v % 7 == 3:
            g.append("Skin")
        if v in no_group:
            g = [other[0], "Skin"]
        groups.append([str(x) for x in g])
        weights.append([float(x) for x in rng.uniform(0.05, 1.7, size=len(g))])
    return {"matrix_world": np.eye(4).tolist(), "tpose_points": rng.uniform(-1.5, 1.5, size=(n, 3)).tolist(),
            "groups": groups, "weights": weights}


def _armature(rng, names, track_len):
    rest = {nm: _rigid(rng).tolist() for nm in names}
    pose = {nm: [_rigid(rng, scale=rng.uniform(0.9, 1.1, size=3)).tolist() for _ in range(track_len.get(nm, N_FRAMES))]
            for nm in names}
    return {"matrix_world": np.eye(4).tolist(), "rest_bones": rest, "pose_bones": pose}


def make_package(seed=5):
    rng = np.random.default_rng(seed)
    a_bones, b_bones = ["A_root", "A_spine", "A_arm", "A_hand"], ["B_hip", "B_unused", "B_leg"]
    mesh_a = _mesh(rng, SIZES[0], a_bones, b_bones, no_group={11})
    mesh_b = _mesh(rng, SIZES[2], ["B_hip", "B_leg"], a_bones, no_group={4, 17})
    return {"camera": {"lens": [50.0] * N_FRAMES},
            "bones": [{"vertex": mesh_a, "armature": _armature(rng, a_bones, {"A_arm": N_FRAMES + 2})},
                      None,
                      {"vertex": mesh_b, "armature": _armature(rng, b_bones, {})}]}


class _Mesh:
    def __init__(self, verts):
        self._v = verts

    def verts_list(self):
        return [self._v]


class _Composite:
    """The attributes of the Frosting model apply_poses_to_scene touches."""

    def __init__(self, base_verts, ref_indices):
        self.editable, self.use_simple_adapt, self.device = False, True, "cpu"
        self.ref_indices, self.shell_base = ref_indices, _Mesh(base_verts)


def main():
    ns = reference_namespace()
    text = json.dumps(make_package())
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "package.json")
        with open(path, "w") as f:
            f.write(text)
        package = ns["load_blender_package"](path, "cpu")
    ref_indices = [int(x) for x in np.cumsum((0,) + SIZES)]
    base = torch.from_numpy(np.random.default_rng(6).uniform(-3, 3, size=(ref_indices[-1], 3))).float()
    save = {"package_json": np.array(text), "n_frames": np.int32(N_FRAMES), "frames": np.array(FRAMES, np.int32),
            "ref_indices": np.array(ref_indices, np.int64), "base_init": base.numpy().copy(),
            "rigged": np.array([bool(m) for m in package["bones"]])}
    for i, mesh_dict in enumerate(package["bones"]):
        if not mesh_dict:
            continue
        arm = mesh_dict["armature"]
        names = list(arm["rest_bones"])
        save[f"mesh{i}/tpose"] = mesh_dict["vertex"]["tpose_points"].numpy()
        save[f"mesh{i}/bone_names"] = np.array(names)
        save[f"mesh{i}/rest"] = torch.stack([arm["rest_bones"][n] for n in names]).numpy()
        for n in names:
            save[f"mesh{i}/pose/{n}"] = arm["pose_bones"][n].numpy()
            idx, w = package["bone_to_vertices"][i][n], package["bone_to_vertex_weights"][i][n]
            save[f"mesh{i}/idx/{n}"] = idx.numpy() if len(idx) else np.zeros(0, np.int64)
            save[f"mesh{i}/w/{n}"] = w.numpy() if len(w) else np.zeros(0, np.float64)
            assert len(w) == 0 or w.dtype == torch.float64
    comp = _Composite(base.clone(), ref_indices)
    outs = []
    for f in FRAMES:
        ns["apply_poses_to_scene"](comp, f, package)
        outs.append(comp.shell_base.verts_list()[0].numpy().copy())
    save["out_verts"] = np.stack(outs)
    np.savez_compressed(os.path.join(HERE, "frosting_skin.npz"), **save)
    print(len(save), "arrays", sum(v.nbytes for v in save.values()), "bytes")


if __name__ == "__main__":
    main()
