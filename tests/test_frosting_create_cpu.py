"""Creating a Frosting layer, without a GPU: the float64 trimming and volume models against the float64 torch
restatements on hand-built meshes, torch's float32 scalar semantics the kernels follow, the cell counts, and the Python
and C argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, create_frosting, trim_shell
from frosting_b200.frosting_create import cell_counts, torch_cell_volumes, torch_trim_shell
from tests import frosting_create_oracle as oracle
from tests.knn_oracle import oracle_knn

EXTENT = 1.0


def sheets():
    """Two parallel square sheets, 4 x 4 vertices each, 18 faces each plus one zero-area face on A: A at z = 0 with
    normals +z and a shell of +-1, B at z = 0.2 above A's middle with normals -z and a shell of +-0.1, except B's
    vertex `STOP0` whose inner distance 3.4 puts its first trial (0.17 down) inside A's first-iteration shell.  A's outer
    side meets nothing and never stops; B's inner side meets A's inner shell in a few iterations."""
    g = np.linspace(0.0, 1.0, 4)
    xx, yy = np.meshgrid(g, g, indexing="ij")
    a = np.stack([xx.ravel(), yy.ravel(), np.zeros(16)], 1)
    b = np.stack([0.3 + 0.4 * xx.ravel(), 0.3 + 0.4 * yy.ravel(), np.full(16, 0.2)], 1)
    verts = np.concatenate([a, b]).astype(np.float32)
    q = []
    for i in range(3):
        for j in range(3):
            v = 4 * i + j
            q += [(v, v + 4, v + 1), (v + 1, v + 4, v + 5)]
    fa = np.array(q)
    faces = np.concatenate([fa, fa[:, ::-1] + 16, [[0, 1, 1]]]).astype(np.int32)
    normals = np.concatenate([np.tile([0, 0, 1.0], (16, 1)), np.tile([0, 0, -1.0], (16, 1))]).astype(np.float32)
    inner = np.concatenate([np.full(16, 1.0), np.full(16, 0.1)]).astype(np.float32)
    outer = -inner
    inner[16 + 5] = 3.4
    return dict(verts=verts, faces=faces, normals=normals, inner=inner, outer=outer, stop0=16 + 5)


def knn8(queries, centres):
    return oracle_knn(np.asarray(centres, np.float32), np.asarray(queries, np.float32), 8)[1]


def torch_knn(queries, centres, K):
    return torch.from_numpy(oracle_knn(centres.float().numpy(), queries.float().numpy(), K)[1])


def test_float32_scalar_semantics_of_the_reference():
    """is_inside_frosting's `proj > extent * proj_th` compares against the Python product rounded to float32, and the
    schedule's `1 / n * old` is a float32 multiply by float32(1 / n)."""
    s = 5.5 * 1e-6
    f = np.float32(s)
    assert float(f) > s                                   # a float64 comparison would call f32(s) > s true
    assert not bool(torch.tensor([float(f)]) > s)
    old = torch.tensor([0.3, 1.7, -0.9, 3.4])
    assert torch.equal(1 / 20 * old, torch.from_numpy(np.float32(0.05) * old.numpy()))


def test_cell_counts():
    assert cell_counts(10, 100) == (5, 100)
    assert cell_counts(10, 101) == (6, 101)
    assert cell_counts(10, 5) == (1, 10)                  # F * n_min > N raises N
    assert cell_counts(10, 100, 12) == (12, 120)
    assert cell_counts(10, 100, 3) == (3, 100)


def test_trimming_model_matches_the_float64_restatement():
    sc = sheets()
    t = {k: torch.from_numpy(np.asarray(sc[k])).double() for k in ("verts", "normals", "inner", "outer")}
    ref = torch_trim_shell(t["verts"], torch.from_numpy(sc["faces"]), t["normals"], t["inner"], t["outer"], EXTENT,
                           knn=torch_knn)
    th = float(np.float32(EXTENT * 1e-6))
    m = oracle.trim(sc["verts"], sc["faces"], sc["normals"], sc["inner"], sc["outer"], th, knn8, dtype=np.float64)
    assert (m["inner_stop"] == ref.inner_stop.numpy()).all() and (m["outer_stop"] == ref.outer_stop.numpy()).all()
    np.testing.assert_allclose(m["inner"], ref.inner_dist.numpy(), rtol=0, atol=1e-12)
    np.testing.assert_allclose(m["outer"], ref.outer_dist.numpy(), rtol=0, atol=1e-12)
    # the hand-built regimes: a side stopping at iteration 0, sides stopping later, sides never stopping
    assert m["inner_stop"][sc["stop0"]] == 0
    assert ((m["inner_stop"][16:] > 0) & (m["inner_stop"][16:] < 20)).any()
    assert (m["outer_stop"][:16] == 20).all()


def test_volume_model_matches_the_float64_restatement():
    sc = sheets()
    rng = np.random.default_rng(0)
    verts = (sc["verts"] * 4).astype(np.float32)
    inner, outer = (rng.random(32) * 0.2).astype(np.float32), (-rng.random(32) * 0.2).astype(np.float32)
    inner[:4] = outer[:4] = 0                                 # heights under the minimum
    cam = np.array([0.5, 0.5, 1.0], np.float32)
    for contract in (True, False):
        ref = torch_cell_volumes(*(torch.from_numpy(x).double() for x in (verts,)), torch.from_numpy(sc["faces"]),
                                 torch.from_numpy(inner).double(), torch.from_numpy(outer).double(), 3.0,
                                 torch.from_numpy(cam).double(), contract_points=contract)
        vol, _ = oracle.cell_volumes(verts, sc["faces"], inner, outer, 3.0, cam, 0.001 * 3.0, contract)
        np.testing.assert_allclose(vol.v, ref.numpy(), rtol=1e-12, atol=1e-15)
        assert vol.v[-1] == 0                                 # the zero-area face
    assert (np.linalg.norm(verts - cam, axis=1) > 3.0).any()  # some vertices contract


def test_fma_replay_rounds_once():
    a = np.float32([1 + 2 ** -12, 3.0])
    c = np.float32([-(1 + 2 ** -11), 2 ** -30])
    got = oracle.fma32(a, a, c)
    assert got[0] == np.float32(2.0 ** -24)                    # (1 + 2^-12)^2 - (1 + 2^-11), exact only when fused
    assert got[1] == np.float32(9.0)


def test_python_layer_rejects_bad_inputs_before_any_launch():
    sc = sheets()
    verts, faces = torch.from_numpy(sc["verts"]), torch.from_numpy(sc["faces"])
    n = torch.from_numpy(sc["normals"])
    d = torch.from_numpy(sc["inner"])
    with pytest.raises(ValueError, match="CUDA device"):
        trim_shell(verts, faces, n, d, -d, 1.0)
    with pytest.raises(ValueError, match="float32"):
        trim_shell(verts.double(), faces, n, d, -d, 1.0)
    with pytest.raises(ValueError, match="CUDA device"):
        create_frosting((verts, verts, verts, d), {}, verts, faces, spatial_extent=1.0, camera_center=verts[0])


def test_c_boundary_rejects_bad_extents_without_touching_cuda():
    L = _lib.lib()
    p = C.c_void_p(0x1000)
    base = dict(n_verts=4, n_faces=8, n_iterations=20, n_gaussians=8, n_gs=4, sh_rest=15, contract=1, step=0.05,
                inside_th=1e-6, extent=1.0, min_height=1e-3)
    ptrs = {f: p for f, t in _lib.FrostingCreate._fields_ if f.startswith("d_")}
    ok = dict(base, knn_workspace_bytes=0, **ptrs)
    cases = (("fb200_frosting_trim", dict(n_faces=7), b"F >= 8"), ("fb200_frosting_trim", dict(n_iterations=0), b"extents"),
             ("fb200_frosting_trim", dict(d_shell=None), b"missing output"),
             ("fb200_frosting_trim", dict(), b"workspace too small"),
             ("fb200_frosting_volumes", dict(d_camera_center=None), b"missing input"),
             ("fb200_frosting_volumes", dict(min_height=-1.0), b"min_height"),
             ("fb200_frosting_sample", dict(d_u=None), b"missing input"),
             ("fb200_frosting_sample", dict(n_gaussians=-1), b"extents"),
             ("fb200_frosting_finish", dict(n_gaussians=3), b"N >= 4"),
             ("fb200_frosting_finish", dict(d_sh_rest=None), b"missing output"))
    for fn, bad, msg in cases:
        st = _lib.FrostingCreate(**dict(ok, **bad))
        assert getattr(L, fn)(C.byref(st), None) == (-3 if b"workspace" in msg else -1), (fn, bad)
        assert msg in L.fb200_last_error(), (fn, bad, L.fb200_last_error())
    for fn in ("fb200_frosting_trim", "fb200_frosting_volumes", "fb200_frosting_sample", "fb200_frosting_finish"):
        assert getattr(L, fn)(None, None) == -1
    st = _lib.FrostingCreate(**dict(ok, n_verts=0, n_faces=0, n_gaussians=0))
    for fn in ("fb200_frosting_trim", "fb200_frosting_volumes", "fb200_frosting_sample", "fb200_frosting_finish"):
        assert getattr(L, fn)(C.byref(st), None) == 0        # nothing to do: no launch
