"""Bone skinning of Blender-animated scenes without a GPU: the torch restatement of apply_poses_to_scene against golden
vectors made by the reference's own source (tests/golden/make_frosting_skin_golden.py), the flat tables of
`skin_tables`, the synthetic rig, and the exported entry point's argument checks."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, scenes
from frosting_b200.skin import FrostingSkin, skin_tables

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "frosting_skin.npz")
NO_GROUP = (11, 65 + 4, 65 + 17)       # base-vertex ids of rigged vertices with no group of their own armature
UNRIGGED = (40, 65)


def golden():
    """(npz, the processed package as load_blender_package returned it, ref_indices)."""
    z = np.load(GOLD)
    bones, idx_of, w_of = [], [], []
    for i, rigged in enumerate(z["rigged"]):
        if not rigged:
            bones.append(None)
            idx_of.append(None)
            w_of.append(None)
            continue
        names = [str(n) for n in z[f"mesh{i}/bone_names"]]
        rest = torch.from_numpy(z[f"mesh{i}/rest"])
        arm = {"rest_bones": {n: rest[k] for k, n in enumerate(names)},
               "pose_bones": {n: torch.from_numpy(z[f"mesh{i}/pose/{n}"]) for n in names}}
        bones.append({"vertex": {"tpose_points": torch.from_numpy(z[f"mesh{i}/tpose"])}, "armature": arm})
        idx = {n: torch.from_numpy(z[f"mesh{i}/idx/{n}"]) for n in names}
        w = {n: torch.from_numpy(z[f"mesh{i}/w/{n}"]) for n in names}
        idx_of.append({n: (v if len(v) else []) for n, v in idx.items()})
        w_of.append({n: (v if len(v) else []) for n, v in w.items()})
    package = {"camera": {"lens": torch.full((int(z["n_frames"]),), 50.0)}, "bones": bones,
               "bone_to_vertices": idx_of, "bone_to_vertex_weights": w_of}
    return z, package, [int(x) for x in z["ref_indices"]]


def replay_tables(t, frame, base_verts):
    """The kernel's arithmetic over skin_tables' output, in torch: per entry [p,1] @ reset, divide, [q,1] @ pose,
    divide; float64 product, accumulated and rounded to float32 entry by entry in the row's order."""
    reset = torch.linalg.inv(t["rest_t"])
    counts = (t["offsets"][1:] - t["offsets"][:-1]).long()
    acc = torch.zeros_like(t["tpose"])
    hom = lambda p: torch.cat([p, torch.ones(p.shape[0], 1)], 1)
    for k in range(int(counts.max()) if counts.numel() else 0):
        rows = torch.nonzero(counts > k)[:, 0]
        e = t["offsets"][rows].long() + k
        b = t["bones"][e].long()
        q = (hom(t["tpose"][rows])[:, None] @ reset[b])[:, 0]
        q = q[:, :3] / q[:, 3:]
        r = (hom(q)[:, None] @ t["pose"][b, frame])[:, 0]
        r = r[:, :3] / r[:, 3:]
        acc[rows] = (acc[rows].double() + t["weights"][e][:, None] * r.double()).float()
    base_verts[t["vert_ids"].long()] = acc
    return base_verts


def close(a, b, bar=1e-5):
    return bool(((a - b).abs() <= bar * (1 + b.abs())).all())


def test_restatement_matches_reference_source_bit_for_bit():
    z, package, ref_indices = golden()
    for k, f in enumerate(z["frames"]):
        base = torch.from_numpy(z["base_init"]).clone()
        scenes.skin_vertices(package, ref_indices, int(f), base)
        assert torch.equal(base, torch.from_numpy(z["out_verts"][k])), int(f)


def test_golden_covers_the_cases():
    z, package, ref_indices = golden()
    out, base = torch.from_numpy(z["out_verts"]), torch.from_numpy(z["base_init"])
    wrap = [k for k, f in enumerate(z["frames"]) if f >= z["n_frames"]]
    assert wrap and torch.equal(out[wrap[0]], out[list(z["frames"]).index(z["frames"][wrap[0]] % z["n_frames"])])
    assert torch.equal(out[:, UNRIGGED[0]:UNRIGGED[1]], base[None, UNRIGGED[0]:UNRIGGED[1]].expand(len(out), -1, -1))
    assert not torch.any(out[:, list(NO_GROUP)])
    # different frames pose differently; one bone has no vertices, one track is longer than the animation
    assert (out[0] - out[1]).abs().max() > 0.1
    assert len(package["bone_to_vertices"][2]["B_unused"]) == 0
    assert package["bones"][0]["armature"]["pose_bones"]["A_arm"].shape[0] > int(z["n_frames"])
    assert all(w.dtype == torch.float64 for m in package["bone_to_vertex_weights"] if m for w in m.values() if len(w))


def test_skin_tables_order_filtering_and_ranges():
    z, package, ref_indices = golden()
    t = skin_tables(package, ref_indices, ref_indices[-1])
    assert t["bone_names"] == [(0, "A_root"), (0, "A_spine"), (0, "A_arm"), (0, "A_hand"), (2, "B_hip"), (2, "B_leg")]
    assert t["n_frames"] == 3 and t["pose"].shape == (6, 3, 4, 4) and t["rest_t"].shape == (6, 4, 4)
    assert torch.equal(t["vert_ids"].long(), torch.cat([torch.arange(0, 40), torch.arange(65, 95)]))
    assert torch.equal(t["tpose"], torch.cat([torch.from_numpy(z["mesh0/tpose"]), torch.from_numpy(z["mesh2/tpose"])]))
    counts = (t["offsets"][1:] - t["offsets"][:-1]).tolist()
    rows_of = {int(v): r for r, v in enumerate(t["vert_ids"])}
    for v in NO_GROUP:
        assert counts[rows_of[v]] == 0
    assert sorted(set(counts) - {0}) == [1, 2, 3, 4]
    assert t["weights"].dtype == torch.float64 and t["bones"].dtype == torch.int32
    for r in range(len(counts)):
        e = slice(int(t["offsets"][r]), int(t["offsets"][r + 1]))
        b = t["bones"][e].tolist()
        assert b == sorted(b)                                   # rest_bones order
        if b:
            assert abs(float(t["weights"][e].sum()) - 1.0) < 1e-12
        i_mesh, local = (0, r) if r < 40 else (2, r - 40)
        for bb, w in zip(b, t["weights"][e].tolist()):
            name = t["bone_names"][bb][1]
            pos = (package["bone_to_vertices"][i_mesh][name] == local).nonzero()[:, 0]
            assert package["bone_to_vertex_weights"][i_mesh][name][pos].item() == w
    arm = package["bones"][0]["armature"]
    assert torch.equal(t["pose"][2], arm["pose_bones"]["A_arm"][:3].transpose(-1, -2))
    assert torch.equal(t["rest_t"][0], arm["rest_bones"]["A_root"].T)


def test_tables_replayed_match_reference_source():
    z, package, ref_indices = golden()
    t = skin_tables(package, ref_indices, ref_indices[-1])
    for k, f in enumerate(z["frames"]):
        base = torch.from_numpy(z["base_init"]).clone()
        replay_tables(t, int(f) % t["n_frames"], base)
        assert close(base, torch.from_numpy(z["out_verts"][k])), int(f)


def test_skin_tables_raise_on_short_track_or_range_mismatch():
    z, package, ref_indices = golden()
    arm = package["bones"][2]["armature"]
    # a short track on a bone without vertices is never read by the reference either
    arm["pose_bones"]["B_unused"] = arm["pose_bones"]["B_unused"][:1]
    skin_tables(package, ref_indices, ref_indices[-1])
    arm["pose_bones"]["B_leg"] = arm["pose_bones"]["B_leg"][:2]
    with pytest.raises(ValueError, match="pose track of 2 frames"):
        skin_tables(package, ref_indices, ref_indices[-1])
    z, package, ref_indices = golden()
    with pytest.raises(ValueError, match="does not hold its 40 tpose_points"):
        skin_tables(package, [0, 41, 65, 95], 95)
    with pytest.raises(ValueError, match="within the 90 base vertices"):
        skin_tables(package, ref_indices, 90)
    with pytest.raises(ValueError, match="ref_indices"):
        skin_tables(package, ref_indices[:3], 95)


@pytest.mark.parametrize("n_bones", [1, 8])
def test_synthetic_rig(n_bones):
    verts, _, _ = scenes.uv_sphere(24, 30)
    package, ref_indices = scenes.skinned_rig(verts, n_bones, 4)
    assert ref_indices == [0, verts.shape[0]]
    t = skin_tables(package, ref_indices, verts.shape[0])
    counts = (t["offsets"][1:] - t["offsets"][:-1])
    assert int(counts.min()) >= 1 and int(counts.max()) <= 4
    if n_bones == 8:
        assert set(counts.tolist()) == {1, 2, 3, 4} and len(t["bone_names"]) == 8
    sums = torch.zeros(verts.shape[0], dtype=torch.float64).index_add(
        0, torch.repeat_interleave(torch.arange(verts.shape[0]), counts.long()), t["weights"])
    assert (sums - 1).abs().max() < 1e-12
    frames = [scenes.skin_vertices(package, ref_indices, f, verts.clone()) for f in range(5)]
    assert torch.equal(frames[4], frames[0]) and (frames[1] - frames[0]).abs().max() > 1e-3
    replayed = replay_tables(t, 1, verts.clone())
    assert close(replayed, frames[1])
    # rest pose: the tracks are the rest bones, the vertices stay where they are
    arm = package["bones"][0]["armature"]
    arm["pose_bones"] = {n: m[None].expand(4, 4, 4) for n, m in arm["rest_bones"].items()}
    assert close(scenes.skin_vertices(package, ref_indices, 2, verts.clone()), verts)


def test_skin_entry_points_are_exported():
    import frosting_b200 as fb
    L = _lib.lib()
    for n in ("fb200_frosting_skin_pose", "fb200_frosting_skin_struct_size"):
        assert n in _lib.EXPORTED and hasattr(L, n)
    assert L.fb200_frosting_skin_struct_size() == C.sizeof(_lib.FrostingSkin)
    assert fb.FrostingSkin is FrostingSkin and fb.skin_tables is skin_tables


def _skin_struct(**kw):
    d = C.c_void_p(0x1000)
    f = dict(n_rows=4, n_verts=10, n_bones=2, n_frames=3)
    for n, _ in _lib.FrostingSkin._fields_[4:]:
        f[n] = d
    f.update(kw)
    return _lib.FrostingSkin(**f)


def test_skin_argument_errors_are_reported_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    call = lambda s, frame=0, out=d: L.fb200_frosting_skin_pose(C.byref(s) if s is not None else None, frame, out, None)
    assert call(None) == -1 and b"null skin struct" in L.fb200_last_error()
    for bad in (dict(n_rows=-1), dict(n_verts=-1), dict(n_bones=-1), dict(n_frames=-1), dict(n_rows=11)):
        assert call(_skin_struct(**bad)) == -1 and b"bad extents" in L.fb200_last_error(), bad
    for frame in (-1, 3, 7):
        assert call(_skin_struct(), frame) == -1 and b"frame outside [0, n_frames)" in L.fb200_last_error()
    assert call(_skin_struct(n_frames=0), 0) == -1 and b"frame outside" in L.fb200_last_error()
    assert call(_skin_struct(), 0, None) == -1 and b"missing vertex table pointer" in L.fb200_last_error()
    assert call(_skin_struct(d_offsets=None)) == -1 and b"missing vertex table pointer" in L.fb200_last_error()
    assert call(_skin_struct(d_weights=None)) == -1 and b"missing bone table pointer" in L.fb200_last_error()
    assert call(_skin_struct(d_pose=C.c_void_p(0x1004))) == -1 and b"16-byte aligned" in L.fb200_last_error()
    # nothing to do is not an error: no rows, no launch
    assert call(_skin_struct(n_rows=0, d_tpose=None, d_vert_ids=None, d_offsets=None), 2, None) == 0


def test_python_surface_rejects_cpu():
    z, package, ref_indices = golden()
    with pytest.raises(RuntimeError, match="CUDA tensors only"):
        FrostingSkin(package, ref_indices, ref_indices[-1], "cpu")
