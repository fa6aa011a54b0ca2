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
    "ends": [(-1.0, 0.02, 0.5), (1.0, 0.02, 0.5)],        # above only at samples 0 and n - 1: both crossings bound
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
    assert (out["first"][at["ends"]], out["last"][at["ends"]]) == (0, N_SAMPLES - 1) and not out["empty"][at["ends"]]
    assert (out["d"][at["ends"]] > LEVEL).sum() == 2
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


# ---------------------------------------------------------------------------------------------------------------------
# The staged model (normals, proposal, level stage with magnitudes) against the torch restatement in float64

FAN = 70                  # valence of the fan's centre vertex
ISOLATED, ZERO_AREA = FAN + 1, (FAN + 2, FAN + 3, FAN + 4)


def hand_mesh():
    """75 vertices (8 k + 3): a fan of FAN triangles around vertex 0 (its first five faces duplicated), an isolated
    vertex, and three vertices whose only faces have zero area (two of them coincide).  The Gaussians (SuGaR and 3DGS
    alike) have non-unit quaternions and some scales under the 1e-8 clamp; at the isolated vertex sits one of strength
    exactly the float32 level with scales (0, 1e-9, 1e-8) -- every sample of a zero-normal vertex is the vertex itself --
    and its other nearest Gaussians, a distance 1 away with scales <= 1e-7, underflow through the 1e8 clamp.
    Returns float32 CPU tensors."""
    g = torch.Generator().manual_seed(5)
    th = 2 * np.pi * torch.arange(FAN, dtype=torch.float64) / FAN
    ring = torch.stack([th.cos(), th.sin(), 0.05 * (3 * th).sin()], -1)
    verts = torch.cat([torch.zeros(1, 3, dtype=torch.float64), ring,
                       torch.tensor([[10.0, 0, 0], [20.0, 0, 0], [20.0, 1.0, 0], [20.0, 0, 0]], dtype=torch.float64)])
    fan = torch.stack([torch.zeros(FAN, dtype=torch.long), 1 + torch.arange(FAN), 1 + (torch.arange(FAN) + 1) % FAN], -1)
    z = ZERO_AREA
    faces = torch.cat([fan, fan[:5], torch.tensor([[z[0], z[0], z[1]], [z[1], z[2], z[0]]])]).to(torch.int32)
    n_fan = 48
    r, a = 1.1 * torch.rand(n_fan, generator=g).sqrt(), 2 * np.pi * torch.rand(n_fan, generator=g)
    pts = torch.cat([torch.stack([r * a.cos(), r * a.sin(), 0.03 * torch.randn(n_fan, generator=g)], -1),
                     torch.tensor([[10.0, 0, 0], [10.0, 1.0, 0], [10.0, -1.0, 0], [10.0, 0, 1.0], [20.0, 0.5, 0],
                                   [20.5, 1.0, 0]])])
    scl = torch.cat([torch.stack([0.3 * torch.exp(0.3 * torch.randn(n_fan, generator=g)),
                                  0.3 * torch.exp(0.3 * torch.randn(n_fan, generator=g)),
                                  0.02 * torch.exp(0.3 * torch.randn(n_fan, generator=g))], -1),
                     torch.tensor([[0.0, 1e-9, 1e-8], [1e-12, 1e-8, 1e-7], [1e-8, 1e-8, 1e-8], [1e-9, 1e-12, 1e-8],
                                   [0.5, 0.5, 0.5], [0.4, 0.3, 0.5]])])
    scl[:4, 0] = 1e-9                                 # a few fan Gaussians with one scale under the clamp
    tilt = torch.cat([torch.ones(n_fan, 1), 0.2 * torch.randn(n_fan, 3, generator=g)], -1)
    q = tilt / tilt.norm(dim=-1, keepdim=True) * torch.exp(0.7 * torch.randn(n_fan, 1, generator=g))
    q = torch.cat([q, torch.tensor([[1.0, 0, 0, 0], [0.5, 0.5, 0.5, 0.5], [2.0, 0, 0, 0], [0, 0.3, 0, 0],
                                    [1.5, 0.2, -0.4, 0.1], [0.7, 0, 0.7, 0]])])
    strength = torch.cat([0.8 * torch.ones(n_fan), torch.tensor([LEVEL, 0.9, 0.9, 0.9, 0.8, 0.6])])[:, None]
    gauss = (pts.float(), scl.float(), q.float(), strength.float())
    assert gauss[3][n_fan, 0].item() == np.float32(LEVEL)
    return dict(verts=verts.float(), faces=faces, gaussians=gauss, n_fan=n_fan)


def _sphere_inputs():
    sc = scenes.frosting_init_scene(600, 3000, 3000, 4)
    g = torch.Generator().manual_seed(9)
    q = sc["sugar"][2] * torch.exp(0.5 * torch.randn(len(sc["sugar"][2]), 1, generator=g))     # non-unit quaternions
    return sc, (sc["sugar"][0], sc["sugar"][1], q, sc["sugar"][3])


@pytest.mark.parametrize("mesh", ["sphere", "hand"])
def test_normals_model_matches_the_float64_restatement(mesh):
    m = hand_mesh() if mesh == "hand" else _sphere_inputs()[0]
    n, raw = oracle.vertex_normals(m["verts"].numpy(), m["faces"].numpy())
    want = scenes.p3d_verts_normals(m["verts"].double(), m["faces"]).numpy()
    np.testing.assert_allclose(n.v, want, rtol=0, atol=1e-12)
    assert np.isfinite(n.m).all() and (n.m > 0).any()
    if mesh == "hand":
        for v in (ISOLATED,) + ZERO_AREA:
            assert (raw[v] == 0).all() and (n.v[v] == 0).all(), v
        assert (n.v[0] == want[0]).all() and n.v[0, 2] > 0.99
    # the magnitude covers the float32 restatement's rounding
    n32 = scenes.p3d_verts_normals(m["verts"], m["faces"]).numpy()
    assert (np.abs(n32 - n.v) <= 4 * oracle.ULP * n.m + 1e-30).all()


@pytest.mark.parametrize("std_K", [1, 4, 32])
def test_proposal_model_matches_the_float64_restatement(std_K):
    """|s * (q^-1 (0, n) q)| averaged over the std_K nearest SuGaR Gaussians, q raw and not unit, as torch_initial_shell
    restates pytorch3d's quaternion_apply and quaternion_invert."""
    sc, sugar = _sphere_inputs()
    n32 = scenes.p3d_verts_normals(sc["verts"], sc["faces"])
    std_idx = oracle_knn(sc["verts"].numpy(), sugar[0].numpy(), std_K)
    inner, outer, _ = oracle.proposal(n32.numpy(), sugar[1].numpy(), sugar[2].numpy(), std_idx, 3.0)
    stds = lambda dt: (sugar[1].to(dt)[std_idx] * scenes.quaternion_apply(
        scenes.quaternion_invert(sugar[2].to(dt)[std_idx]), n32.to(dt)[:, None])).norm(dim=-1).mean(dim=-1)
    want = (3.0 * stds(torch.float64)).numpy()
    np.testing.assert_allclose(inner.v, want, rtol=1e-12, atol=0)
    np.testing.assert_allclose(outer.v, -want, rtol=1e-12, atol=0)
    got32 = (3.0 * stds(torch.float32)).numpy()
    assert (np.abs(got32 - inner.v) <= 4 * oracle.ULP * inner.m).all()


def _staged(g, verts, normals, inner, outer, knn, n_samples, **kw):
    fr = torch.linspace(0, 1, n_samples, dtype=torch.float64).numpy()
    return oracle.level_stage(tuple(t.numpy() for t in g), verts.numpy(), normals.numpy(), inner.numpy(),
                              outer.numpy(), knn, fr, **kw)


def test_staged_level_model_matches_the_float64_restatement_on_the_edge_scene():
    sc = edge_scene()
    ref = edge_oracle(sc)
    st = _staged(sc["gaussians"], sc["verts"], sc["normals"], sc["inner"], sc["outer"], sc["knn_idx"], N_SAMPLES,
                 level=LEVEL, min_layer=MIN_LAYER, half_layer=MIN_LAYER / 2, min_clamp_inner=sc["clamp_inner"].numpy(),
                 max_clamp_outer=sc["clamp_outer"].numpy())
    np.testing.assert_allclose(st["d"].v, ref["d"], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(st["outer"].v, ref["outer_raw"], rtol=0, atol=1e-12)
    np.testing.assert_allclose(st["inner"].v, ref["inner_raw"], rtol=0, atol=1e-12)
    at = {n: i for i, n in enumerate(sc["names"])}
    assert st["clamped_inner"][at["clamp_inner"]] and st["clamped_outer"][at["clamp_outer"]]
    assert st["clamped_inner"].sum() == st["clamped_outer"].sum() == 1
    assert (st["empty"] == ref["empty"]).all() and (st["flat"] == ref["flat"]).all() and st["saturated"].any()


def test_staged_model_matches_the_float64_restatement_on_a_sphere():
    """Normals, proposal and the first pass composed in float64 against torch_reference in float64, and the float32
    restatement inside the magnitudes."""
    sc, sugar = _sphere_inputs()
    v = sc["verts"]
    n, _ = oracle.vertex_normals(v.numpy(), sc["faces"].numpy())
    std_idx, knn = oracle_knn(v.numpy(), sugar[0].numpy(), 4), oracle_knn(v.numpy(), sugar[0].numpy(), 16)
    inner, outer, _ = oracle.proposal(n.v, sugar[1].numpy(), sugar[2].numpy(), std_idx, 3.0)
    d64 = lambda x: torch.from_numpy(np.asarray(x, np.float64))
    args = dict(n_samples=N_SAMPLES, K=16, level=LEVEL, min_layer_size=0.001, spatial_extent=4.0, knn_idx=d64(knn).long())
    ref, dens = torch_reference(tuple(t.double() for t in sugar), v.double(), d64(n.v), d64(inner.v), d64(outer.v),
                                return_densities=True, **args)
    st = _staged(sugar, v.double(), d64(n.v), d64(inner.v), d64(outer.v), knn, N_SAMPLES, level=LEVEL,
                 min_layer=0.004, half_layer=0.002)
    np.testing.assert_allclose(st["d"].v, dens.numpy(), rtol=1e-10, atol=1e-14)
    np.testing.assert_allclose(st["outer"].v, ref.outer_dist.numpy(), rtol=0, atol=1e-10)
    np.testing.assert_allclose(st["inner"].v, ref.inner_dist.numpy(), rtol=0, atol=1e-10)
    assert 0 < (st["first"] > 0).sum() < len(v)


def test_hand_mesh_exact_level_in_the_model():
    """At the isolated vertex every sample is the vertex and its density is exactly the level: not above, not under."""
    m = hand_mesh()
    g = m["gaussians"]
    n, _ = oracle.vertex_normals(m["verts"].numpy(), m["faces"].numpy())
    knn = oracle_knn(m["verts"].numpy(), g[0].numpy(), 4)
    inner, outer, _ = oracle.proposal(n.v, g[1].numpy(), g[2].numpy(), knn, 3.0)
    assert knn[ISOLATED, 0] == m["n_fan"] and inner.v[ISOLATED] == 0
    st = oracle.level_stage(tuple(t.numpy() for t in g), m["verts"].numpy(), n.v, inner.v, outer.v, knn,
                            torch.linspace(0, 1, N_SAMPLES).numpy(), level=oracle.f32(LEVEL),
                            min_layer=oracle.f32(0.004), half_layer=oracle.f32(0.002))
    assert (st["d"].v[ISOLATED] == oracle.f32(LEVEL)).all() and st["undecided"][ISOLATED].all()
    assert not st["empty"][ISOLATED] and st["flat"][ISOLATED]
