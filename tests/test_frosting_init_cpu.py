"""A Frosting layer's thickness without a GPU: the float64 model against the torch restatement in float64, the model's
branches on hand-built vertices (one branch each), and the argument checks of the Python layer and the C boundary."""
import ctypes as C

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, initial_shell, level_points_along_normals, scenes
from frosting_b200.frosting_init import torch_reference
from tests import frosting_init_oracle as oracle

LEVEL, N_SAMPLES, MIN_LAYER = 0.01, 21, 0.5
TINY = (20.0, 0.1, 1e-4)          # a Gaussian that adds nothing at the samples
# name -> the two Gaussians (offset along the normal, isotropic scale, strength) each vertex owns
CASES = {
    "all_under": [(0.0, 0.3, 1e-4), (0.0, 0.3, 1e-4)],
    "all_above": [(0.0, 100.0, 0.5), (0.0, 100.0, 0.5)],
    "one_crossing": [(1.5, 0.5, 1.0), TINY],
    "two_crossings": [(0.0, 0.2, 0.5), TINY],
    "saturated": [(0.0, 0.3, 0.9), (0.0, 0.3, 0.9)],
    "min_layer": [(0.0, 0.02, 0.02), TINY],
    "clamp_inner": [(0.0, 0.2, 0.5), TINY],
    "clamp_outer": [(0.0, 0.2, 0.5), TINY],
}


def edge_scene():
    """One vertex per case, 100 apart along x with normal +z and range [-1, 1], and a duplicate of the first vertex
    (the smoothing's tie rule).  Returns float32 CPU tensors and the float64 model's inputs."""
    names = list(CASES) + ["duplicate"]
    V = len(names)
    verts = torch.zeros(V, 3)
    verts[:len(CASES), 0] = 100.0 * torch.arange(len(CASES))
    normals = torch.tensor([0.0, 0.0, 1.0]).repeat(V, 1)
    pts, scl, strength = [], [], []
    for i, gs in enumerate(CASES.values()):
        for z, s, a in gs:
            pts.append([100.0 * i, 0.0, z])
            scl.append([s, s, s])
            strength.append([a])
    P = len(pts)
    gaussians = (torch.tensor(pts), torch.tensor(scl), torch.tensor([[1.0, 0.0, 0.0, 0.0]]).repeat(P, 1),
                 torch.tensor(strength))
    inner, outer = torch.ones(V), -torch.ones(V)
    clamp_inner, clamp_outer = torch.full((V,), -10.0), torch.full((V,), 10.0)
    clamp_inner[names.index("clamp_inner")] = 0.8
    clamp_outer[names.index("clamp_outer")] = -0.8
    knn_idx = np.stack([np.argsort(((np.asarray(pts) - verts[v].numpy()) ** 2).sum(1), kind="stable")[:2]
                        for v in range(V)])
    return dict(names=names, verts=verts, normals=normals, gaussians=gaussians, inner=inner, outer=outer,
                clamp_inner=clamp_inner, clamp_outer=clamp_outer, knn_idx=knn_idx)


def edge_oracle(sc, smooth_K=0):
    smooth_idx = oracle.self_knn(sc["verts"].numpy(), smooth_K) if smooth_K else None
    return oracle.level_points(tuple(t.numpy() for t in sc["gaussians"]), sc["verts"].numpy(), sc["normals"].numpy(),
                               sc["inner"].numpy(), sc["outer"].numpy(), sc["knn_idx"], n_samples=N_SAMPLES,
                               level=LEVEL, smooth_idx=smooth_idx, min_layer=MIN_LAYER,
                               min_clamp_inner=sc["clamp_inner"].numpy(), max_clamp_outer=sc["clamp_outer"].numpy())


def check_edge_values(names, outer, inner, atol):
    """The values each hand-built vertex must take before smoothing."""
    at = {n: i for i, n in enumerate(names)}
    # an empty range collapses to the centre, and then the min-layer widening applies to it as to any thin layer
    expect = {"all_under": (-0.25, 0.25), "all_above": (-1.0, 1.0), "min_layer": (-0.25, 0.25),
              "duplicate": (-0.25, 0.25)}
    for n, (o, i) in expect.items():
        assert abs(outer[at[n]] - o) <= atol and abs(inner[at[n]] - i) <= atol, (n, outer[at[n]], inner[at[n]])
    assert inner[at["one_crossing"]] == pytest.approx(1.0, abs=atol) and -0.1 < outer[at["one_crossing"]] < 0.0
    for n in ("two_crossings", "saturated"):
        assert -1.0 < outer[at[n]] < -0.5 and 0.5 < inner[at[n]] < 1.0, n
    # the clamps are float32 inputs
    assert inner[at["clamp_inner"]] == np.float32(0.8) and outer[at["clamp_inner"]] < -0.5
    assert outer[at["clamp_outer"]] == np.float32(-0.8) and inner[at["clamp_outer"]] > 0.5


def test_edge_branches_in_the_float64_model():
    sc = edge_scene()
    out = edge_oracle(sc)
    at = {n: i for i, n in enumerate(sc["names"])}
    assert out["empty"][at["all_under"]] and out["empty"][at["duplicate"]] and out["empty"].sum() == 2
    assert (out["first"][at["all_above"]], out["last"][at["all_above"]]) == (0, N_SAMPLES - 1)
    assert out["first"][at["one_crossing"]] > 0 and out["last"][at["one_crossing"]] == N_SAMPLES - 1
    assert out["d"][at["saturated"]].max() == pytest.approx(1.0, abs=1e-9)
    assert out["flat"][at["min_layer"]] and out["flat"].sum() == 1 + 2     # the two empty vertices have width 0 too
    check_edge_values(sc["names"], out["outer_raw"], out["inner_raw"], 1e-12)
    # every sample is decided: more than 1e-5 from the level
    assert (np.abs(out["d"] - LEVEL) > 1e-5).all()
    # smoothing over two vertices: the duplicate and its original are each other's neighbour (ties to the lower index)
    sm = edge_oracle(sc, smooth_K=2)
    assert sm["outer"][0] == sm["outer"][-1] == (out["outer_raw"][0] + out["outer_raw"][-1]) / 2


@pytest.mark.parametrize("smooth_K", [0, 2])
def test_torch_restatement_matches_the_float64_model_on_the_edge_scene(smooth_K):
    sc = edge_scene()
    ref = edge_oracle(sc, smooth_K)
    d64 = lambda t: t.double()
    smooth_idx = torch.from_numpy(oracle.self_knn(sc["verts"].numpy(), smooth_K)) if smooth_K else None
    out, dens = torch_reference(tuple(d64(t) for t in sc["gaussians"]), d64(sc["verts"]), d64(sc["normals"]),
                                d64(sc["inner"]), d64(sc["outer"]), n_samples=N_SAMPLES, K=2, level=LEVEL,
                                min_layer_size=MIN_LAYER, spatial_extent=1.0, min_clamp_inner=d64(sc["clamp_inner"]),
                                max_clamp_outer=d64(sc["clamp_outer"]), knn_idx=torch.from_numpy(sc["knn_idx"]),
                                smooth_idx=smooth_idx, return_densities=True)
    np.testing.assert_allclose(dens.numpy(), ref["d"], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(out.outer_dist.numpy(), ref["outer"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(out.inner_dist.numpy(), ref["inner"], rtol=0, atol=1e-12)


def test_torch_restatement_matches_the_float64_model_on_a_sphere():
    """Random scene, float64 both: the two restatements agree to rounding on every vertex."""
    sc = scenes.frosting_init_scene(600, 3000, 3000, 4)
    v, f = sc["verts"].double(), sc["faces"]
    n = scenes.p3d_verts_normals(v, f)
    g = tuple(t.double() for t in sc["gs"])
    knn = oracle_knn(sc["verts"].numpy(), sc["gs"][0].numpy(), 16)
    inner, outer = torch.full((len(v),), 0.6, dtype=torch.float64), torch.full((len(v),), -0.6, dtype=torch.float64)
    ref = oracle.level_points(tuple(t.numpy() for t in g), v.numpy(), n.numpy(), inner.numpy(), outer.numpy(), knn,
                              n_samples=N_SAMPLES, level=LEVEL, min_layer=0.004)
    out, dens = torch_reference(g, v, n, inner, outer, n_samples=N_SAMPLES, K=16, level=LEVEL, min_layer_size=0.001,
                                spatial_extent=4.0, knn_idx=torch.from_numpy(knn), n_points_per_pass=1000,
                                return_densities=True)
    np.testing.assert_allclose(dens.numpy(), ref["d"], rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(out.outer_dist.numpy(), ref["outer"], rtol=0, atol=1e-10)
    np.testing.assert_allclose(out.inner_dist.numpy(), ref["inner"], rtol=0, atol=1e-10)
    assert 0 < (ref["first"] > 0).sum() < len(v)


def oracle_knn(queries, points, K):
    d = ((np.asarray(queries, np.float64)[:, None] - np.asarray(points, np.float64)[None]) ** 2).sum(-1)
    return np.argsort(d, axis=1, kind="stable")[:, :K]


def _cpu_args():
    sc = edge_scene()
    return dict(gaussians=sc["gaussians"], verts=sc["verts"], normals=sc["normals"], inner_range=sc["inner"],
                outer_range=sc["outer"], level=LEVEL, spatial_extent=1.0)


def test_python_layer_rejects_bad_inputs_before_any_launch():
    a = _cpu_args()
    with pytest.raises(ValueError, match="CUDA device"):
        level_points_along_normals(**a)
    with pytest.raises(ValueError, match="float32"):
        level_points_along_normals(**dict(a, verts=a["verts"].double()))
    with pytest.raises(ValueError, match="CUDA device"):
        initial_shell(a["gaussians"], a["gaussians"], a["verts"], torch.zeros(1, 3, dtype=torch.int32), 1.0)


def test_c_boundary_rejects_bad_extents_without_touching_cuda():
    L = _lib.lib()
    d = C.c_void_p(0x1000)
    base = dict(n_verts=4, P=8, K=4, n_samples=21, smooth_K=4, std_K=0, level=0.01, d_verts=d, d_normals=d, d_points=d,
                d_scaling=d, d_quaternions=d, d_strengths=d, d_knn_idx=d, d_inner_range=d, d_outer_range=d,
                d_fractions=d, d_smooth_idx=d, d_level_outer=d, d_level_inner=d, d_outer_dist=d, d_inner_dist=d,
                d_outer_verts=d, d_inner_verts=d)
    for bad, msg in ((dict(n_samples=33), b"extents"), (dict(n_samples=0), b"extents"), (dict(K=9), b"extents"),
                     (dict(K=33, P=40), b"extents"), (dict(smooth_K=0), b"smoothing table"),
                     (dict(d_fractions=None), b"missing input"), (dict(d_outer_verts=None), b"missing output"),
                     (dict(d_faces=d), b"normals stage"), (dict(d_std_idx=d), b"proposal stage"),
                     (dict(min_layer=-1.0), b"min_layer")):
        st = _lib.FrostingInit(**dict(base, **bad))
        assert L.fb200_level_points(C.byref(st), None) == -1, bad
        assert msg in L.fb200_last_error(), (bad, L.fb200_last_error())
    assert L.fb200_level_points(None, None) == -1
    st = _lib.FrostingInit(**dict(base, n_verts=0))
    assert L.fb200_level_points(C.byref(st), None) == 0          # nothing to do: no launch
