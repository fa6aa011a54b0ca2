"""A Frosting layer's thickness (csrc/frosting_init.cu) stage by stage against the float64 model with magnitudes
(tests/frosting_init_oracle.py: vertex_normals, proposal, level_stage, smooth).

Each pass runs through frosting_init._run twice, without and with smoothing, and reads back the vertex normals, the
proposal ranges, the sample densities, the raw and smoothed distances and the shell vertices.  Every stage is modelled
from the float32 values the kernel read -- the second pass from the first pass's float32 outputs, combined in torch as
initial_shell combines them -- and every element must satisfy

    |x32 - x64| <= TAU * m + 1e-30,

no fraction allowance and no excluded vertices.  Samples within K_BAND ULP m_d of the level take their side from the
kernel's own densities, which must then lie in that band; a decided sample on the wrong side fails.  Vertices without
a face or with only zero-area faces have exactly zero normals, the shell vertices are verts + dist * normals bit for
bit, and initial_shell is the step-by-step composition bit for bit.  Each test asserts minimum shares of the regimes
its scene is built for, so a scene change cannot drop one quietly.

TAU is more than ten times the largest |x32 - x64| / m observed on an H100 (sm_90a build) over every case of this file,
OBSERVED; both in units of ULP = 2^-24."""
import numpy as np
import pytest
import torch

from frosting_b200 import initial_shell, knn_points, scenes
from frosting_b200.frosting_init import MAX_SAMPLES, _fractions, _layer, _run
from tests import frosting_init_oracle as oracle
from tests.test_frosting_init_cpu import (FAN, ISOLATED, LEVEL, MIN_LAYER, N_SAMPLES, ZERO_AREA, edge_scene,
                                          hand_mesh)

pytestmark = pytest.mark.gpu

ULP, K_BAND = oracle.ULP, oracle.K_BAND
OBSERVED = 0.513       # largest |x32 - x64| / (ULP m) on an H100 80GB HBM3 over every case of this file: the smoothed
TAU = 6 * ULP          # outer distance, bench-size scene and the extent sweep
EXTENT = 4.0
WORST = {}             # stage -> largest |x32 - x64| / (ULP m) seen in this session


def cpu(t):
    return None if t is None else t.cpu().numpy()


def check(case, stage, x32, x):
    """Every element within TAU m + 1e-30 of the model; records the worst ratio per stage."""
    x32 = np.asarray(x32, np.float64).reshape(x.v.shape)
    err = np.abs(x32 - x.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err > 1e-30, (err - 1e-30) / (ULP * x.m), 0.0)     # beyond what underflow may lose
    if ratio.size:
        WORST[stage] = max(WORST.get(stage, 0.0), float(np.nan_to_num(ratio, nan=np.inf).max()))
    bad = ~(err <= TAU * x.m + 1e-30)
    if bad.any():
        i = int(np.flatnonzero(bad)[0])
        at = np.unravel_index(i, x.v.shape)
        pytest.fail(f"{case}: {stage}: {int(bad.sum())} of {bad.size} elements beyond TAU m, first at vertex {at[0]} "
                    f"{tuple(int(a) for a in at)}: kernel {x32.flat[i]!r}, model {x.v.flat[i]!r}, m {x.m.flat[i]!r}")


def regimes(st):
    n = st["d"].v.shape[1]
    rows = np.arange(len(st["first"]))
    return dict(undecided=int(st["undecided"].sum()), empty=st["empty"].mean(), widened=st["flat"].mean(),
                clamped_inner=st["clamped_inner"].mean(), clamped_outer=st["clamped_outer"].mean(),
                first_bound=((st["first"] == 0) & st["above"][:, 0]).mean(), first_interp=(st["first"] > 0).mean(),
                last_bound=((st["last"] == n - 1) & st["above"][rows, n - 1]).mean(),
                last_interp=(st["last"] < n - 1).mean(), saturated=st["saturated"].mean())


def level_pass(case, g, verts, normals, inner_range, outer_range, knn, n_samples, smooth_idx, layer, clamps=(None, None),
               faces=None, std_idx=None, std_range=0.0):
    """One pass without and with smoothing, checked stage by stage from the level stage on; returns (smoothed
    LevelPoints, the model's level-stage dict)."""
    dev, V = verts.device, verts.shape[0]
    dens = torch.empty(V, n_samples, device=dev)
    common = dict(faces=faces, std_idx=std_idx, std_range=std_range)
    raw = _run(dev, verts, normals, g, knn, inner_range, outer_range, n_samples, LEVEL, None, layer, *clamps,
               densities=dens, **common)
    sm = raw if smooth_idx is None else _run(dev, verts, normals, g, knn, inner_range, outer_range, n_samples, LEVEL,
                                             smooth_idx, layer, *clamps, **common)
    d32 = cpu(dens)
    st = oracle.level_stage(tuple(cpu(t) for t in g), cpu(verts), cpu(normals), cpu(inner_range), cpu(outer_range),
                            cpu(knn), cpu(_fractions(n_samples, dev)), level=oracle.f32(LEVEL),
                            min_layer=oracle.f32(layer[0]), half_layer=oracle.f32(layer[1]),
                            min_clamp_inner=cpu(clamps[0]), max_clamp_outer=cpu(clamps[1]), d32=d32,
                            raw32=(cpu(raw.outer_dist), cpu(raw.inner_dist)))
    if st["wrong"].any():
        v, j = np.argwhere(st["wrong"])[0]
        pytest.fail(f"{case}: densities: decided sample ({v}, {j}) on the wrong side of the level: kernel {d32[v, j]!r}, "
                    f"model {st['d'].v[v, j]!r} +- {K_BAND * ULP * st['d'].m[v, j]!r}")
    und = st["undecided"]
    assert (np.abs(d32 - oracle.f32(LEVEL))[und] <= 2 * K_BAND * ULP * st["d"].m[und]).all(), case
    check(case, "densities", d32, st["d"])
    check(case, "outer_raw", cpu(raw.outer_dist), st["outer"])
    check(case, "inner_raw", cpu(raw.inner_dist), st["inner"])
    if smooth_idx is not None:
        check(case, "outer_smoothed", cpu(sm.outer_dist), oracle.smooth(cpu(raw.outer_dist), cpu(smooth_idx)))
        check(case, "inner_smoothed", cpu(sm.inner_dist), oracle.smooth(cpu(raw.inner_dist), cpu(smooth_idx)))
    for out in (raw, sm):
        assert torch.equal(out.outer_verts, verts + out.outer_dist[:, None] * normals), case
        assert torch.equal(out.inner_verts, verts + out.inner_dist[:, None] * normals), case
    return sm, st


def stages(case, sugar, gs, verts, faces, *, n_samples=N_SAMPLES, K=16, smooth_K=4, std_K=4, extent=EXTENT):
    """initial_shell step by step: normals and proposal and the first pass over `sugar`, the second pass over `gs`
    inside the widened, clamped proposal.  Returns the two passes' level-stage dicts."""
    dev, V = verts.device, verts.shape[0]
    o = dict(dtype=torch.float32, device=dev)
    normals, inner_range, outer_range = torch.empty(V, 3, **o), torch.empty(V, **o), torch.empty(V, **o)
    std_idx = knn_points(verts, sugar[0], K=std_K).idx
    smooth_idx = knn_points(verts, K=smooth_K).idx if smooth_K else None
    layer = _layer(0.001, extent)
    s1, st1 = level_pass(case + " pass 1", sugar, verts, normals, inner_range, outer_range,
                         knn_points(verts, sugar[0], K=K).idx, n_samples, smooth_idx, layer, faces=faces,
                         std_idx=std_idx, std_range=3.0)
    nm, sums = oracle.vertex_normals(cpu(verts), cpu(faces))
    check(case, "normals", cpu(normals), nm)
    zero = (sums == 0).all(1)
    assert (cpu(normals)[zero] == 0).all(), (case, np.flatnonzero(zero))
    inner, outer, _ = oracle.proposal(cpu(normals), cpu(sugar[1]), cpu(sugar[2]), cpu(std_idx), 3.0)
    check(case, "inner_range", cpu(inner_range), inner)
    check(case, "outer_range", cpu(outer_range), outer)
    # the second pass's inputs, as initial_shell forms them
    centre = (s1.outer_dist + s1.inner_dist) / 2
    min_outer = centre + 3. * (s1.outer_dist - centre)
    max_inner = centre + 3. * (s1.inner_dist - centre)
    clamp_outer = centre + 0.1 * (s1.outer_dist - centre)
    clamp_inner = centre + 0.1 * (s1.inner_dist - centre)
    s2, st2 = level_pass(case + " pass 2", gs, verts, normals, max_inner, min_outer, knn_points(verts, gs[0], K=K).idx,
                         n_samples, smooth_idx, layer, (clamp_inner, clamp_outer))
    if smooth_K == std_K:        # initial_shell averages the proposal over smooth_K Gaussians
        ref = initial_shell(sugar, gs, verts, faces, extent, n_samples=n_samples, K=K, smooth_K=smooth_K)
        assert all(torch.equal(a, b) for a, b in zip(ref, s2)), case
    return st1, st2


def report(case, *sts):
    print(f"\n{case}: worst |x32 - x64| / (ULP m) so far: " + ", ".join(f"{k} {v:.3g}" for k, v in sorted(WORST.items())))
    for i, st in enumerate(sts):
        r = regimes(st)
        print(f"{case} pass {i + 1}: undecided samples resolved {r.pop('undecided')}; regime shares: "
              + ", ".join(f"{k} {v:.4g}" for k, v in r.items()))


def on(dev, sc):
    return (tuple(t.to(dev) for t in sc["sugar"]), tuple(t.to(dev) for t in sc["gs"]), sc["verts"].to(dev),
            sc["faces"].to(dev))


def assert_shares(case, st, minimum):
    r = regimes(st)
    for k, lo in minimum.items():
        assert r[k] >= lo, (case, k, r[k], lo)


# per scene and pass, the least share of vertices (samples for `saturated`, a count for `undecided`) in each regime: about
# half what the scenes give
MIN_SHARES = {
    "sphere_100k": (dict(undecided=1000, saturated=0.03, first_interp=0.02, last_interp=0.02, widened=0.4),
                    dict(undecided=1000, empty=0.1, widened=0.1, clamped_inner=0.005, clamped_outer=0.005,
                         first_bound=0.3, last_bound=0.3, first_interp=0.04, last_interp=0.04, saturated=2e-4)),
    "bench_1M": (dict(undecided=10_000, saturated=0.005, first_interp=0.05, last_interp=0.05, empty=0.01),
                 dict(undecided=10_000, empty=0.2, widened=0.2, clamped_inner=0.01, clamped_outer=0.01,
                      first_bound=0.1, last_bound=0.1, first_interp=0.1, last_interp=0.1, saturated=1e-5)),
}


@pytest.mark.parametrize("size", ["sphere_100k", "bench_1M"])
def test_initial_shell_stage_by_stage(cuda_device, size):
    """The existing 100 k-vertex sphere and the bench tool's scene (1 M vertices, 2 M + 2 M Gaussians)."""
    sc = (scenes.frosting_init_scene(100_000, 500_000, 200_000, 3) if size == "sphere_100k"
          else scenes.frosting_init_scene(1_000_000, 2_000_000, 2_000_000, 0))
    st1, st2 = stages(size, *on(cuda_device, sc))
    report(size, st1, st2)
    for i, st in enumerate((st1, st2)):
        assert_shares(f"{size} pass {i + 1}", st, MIN_SHARES[size][i])


@pytest.mark.parametrize("n_samples", [1, 2, 21, 31, 32])
@pytest.mark.parametrize("K", [1, 2, 16, 32])
def test_extents(cuda_device, n_samples, K):
    """Every n_samples against every K, smooth_K and std_K cycling through their edge values, V = 8 k + 3."""
    i = [1, 2, 21, 31, 32].index(n_samples) + [1, 2, 16, 32].index(K)
    smooth_K, std_K = (0, 1, 4, 32)[i % 4], (1, 4, 32)[i % 3]
    sc = scenes.frosting_init_scene(2000, 8000, 4000, 11)
    # one vertex without faces, just off the sphere, makes V = 8 k + 3: the last block's warps are not all used
    sc["verts"] = torch.cat([sc["verts"], torch.tensor([[2.02, 0.0, 6.0]])])
    V = sc["verts"].shape[0]
    assert V % 8 == 3, V
    case = f"n_samples={n_samples} K={K} smooth_K={smooth_K} std_K={std_K}"
    st1, st2 = stages(case, *on(cuda_device, sc), n_samples=n_samples, K=K, smooth_K=smooth_K, std_K=std_K)
    report(case, st1, st2)


def test_hand_built_mesh(cuda_device):
    """Isolated vertex, zero-area faces, a fan of valence > 64, duplicated faces, non-unit quaternions, scales at the
    1e-8 clamp, and a sample whose density is exactly the level."""
    m = hand_mesh()
    dev = cuda_device
    g = tuple(t.to(dev) for t in m["gaussians"])
    verts, faces = m["verts"].to(dev), m["faces"].to(dev)
    st1, st2 = stages("hand-built mesh", g, g, verts, faces, K=4, smooth_K=4, std_K=4, extent=1.0)
    report("hand-built mesh", st1, st2)
    normals = torch.empty(len(verts), 3, device=dev)
    ranges = torch.empty(len(verts), device=dev), torch.empty(len(verts), device=dev)
    dens = torch.empty(len(verts), N_SAMPLES, device=dev)
    _run(dev, verts, normals, g, knn_points(verts, g[0], K=4).idx, *ranges, N_SAMPLES, LEVEL, None, _layer(0.001, 1.0),
         faces=faces, std_idx=knn_points(verts, g[0], K=4).idx, std_range=3.0, densities=dens)
    for v in (ISOLATED,) + ZERO_AREA:
        assert (normals[v] == 0).all(), v
    assert normals[0, 2].item() > 0.99 and np.bincount(m["faces"].reshape(-1).numpy())[0] == FAN + 5
    # strength = level at the Gaussian's centre, the other neighbours underflow: d > level is false, d < level too
    assert (dens[ISOLATED] == np.float32(LEVEL)).all() and st1["undecided"][ISOLATED].all()
    assert not st1["empty"][ISOLATED] and st1["flat"][ISOLATED]


@pytest.mark.parametrize("smooth_K", [0, 2])
def test_hand_built_level_branches(cuda_device, smooth_K):
    """The edge scene's one vertex per branch (empty range, widening, both clamps, saturation, bound crossings at both
    ends, a duplicate vertex) through the level stage with given normals, ranges and clamps."""
    sc = edge_scene()
    dev = cuda_device
    g = tuple(t.to(dev) for t in sc["gaussians"])
    smooth_idx = knn_points(sc["verts"].to(dev), K=smooth_K).idx if smooth_K else None
    case = f"edge scene smooth_K={smooth_K}"
    _, st = level_pass(case, g, sc["verts"].to(dev), sc["normals"].to(dev), sc["inner"].to(dev), sc["outer"].to(dev),
                       torch.from_numpy(sc["knn_idx"]).to(dev), N_SAMPLES, smooth_idx, (MIN_LAYER, MIN_LAYER / 2),
                       (sc["clamp_inner"].to(dev), sc["clamp_outer"].to(dev)))
    report(case, st)
    at = {n: i for i, n in enumerate(sc["names"])}
    assert st["empty"][at["all_under"]] and st["flat"][at["min_layer"]] and st["saturated"][at["saturated"]].any()
    assert st["clamped_inner"][at["clamp_inner"]] and st["clamped_outer"][at["clamp_outer"]]
    assert (st["first"][at["ends"]], st["last"][at["ends"]]) == (0, N_SAMPLES - 1) and st["above"][at["ends"]].sum() == 2


def test_fractions_match_the_cpu_linspace(cuda_device):
    for n in range(1, MAX_SAMPLES + 1):
        assert torch.equal(_fractions(n, cuda_device).cpu(), torch.linspace(0., 1., n)), n


def test_tau_and_observed():
    assert 10 * OBSERVED * ULP < TAU < K_BAND * ULP
