"""A Frosting layer's thickness on the GPU: densities, crossings and distances held to the float64 model by the float32
torch restatement's own distance from it, bit-identical reruns, every hand-built branch, the end-to-end initial shell
against its torch restatement in float64, and the argument checks."""
import numpy as np
import pytest
import torch

from frosting_b200 import initial_shell, knn_points, level_points_along_normals, scenes
from frosting_b200.frosting_init import torch_initial_shell, torch_reference
from tests import frosting_init_oracle as oracle
from tests.test_frosting_init_cpu import LEVEL, MIN_LAYER, N_SAMPLES, check_edge_values, edge_oracle, edge_scene

pytestmark = pytest.mark.gpu

RANGE, EXTENT, MIN_SIZE = 0.5, 4.0, 0.001


@pytest.fixture(scope="module")
def sphere(cuda_device):
    """About 100 k base vertices, 500 k SuGaR and 200 k 3DGS Gaussians; the 3DGS pass over +-RANGE with float32 normals
    from the CPU, the float64 model and the float32 torch restatement over the same neighbour table."""
    sc = scenes.frosting_init_scene(100_000, 500_000, 200_000, 3)
    dev = cuda_device
    normals = scenes.p3d_verts_normals(sc["verts"], sc["faces"])
    V = len(sc["verts"])
    g = tuple(t.to(dev) for t in sc["gs"])
    verts, nrm = sc["verts"].to(dev), normals.to(dev)
    inner, outer = torch.full((V,), RANGE, device=dev), torch.full((V,), -RANGE, device=dev)
    args = dict(n_samples=N_SAMPLES, K=16, level=LEVEL, min_layer_size=MIN_SIZE, spatial_extent=EXTENT)
    out, dens = level_points_along_normals(g, verts, nrm, inner, outer, smooth_K=0, return_densities=True, **args)
    knn = knn_points(verts, g[0], K=16).idx
    t32, d32 = torch_reference(g, verts, nrm, inner, outer, knn_idx=knn, return_densities=True, **args)
    ref = oracle.level_points(tuple(t.numpy() for t in sc["gs"]), sc["verts"].numpy(), normals.numpy(),
                              inner.cpu().numpy(), outer.cpu().numpy(), knn.cpu().numpy(), n_samples=N_SAMPLES,
                              level=LEVEL, min_layer=np.float32(MIN_SIZE * EXTENT))
    decided = (np.abs(ref["d"] - LEVEL) > 1e-5).all(1)
    return dict(sc=sc, dev=dev, g=g, verts=verts, normals=nrm, inner=inner, outer=outer, args=args, out=out,
                dens=dens.cpu().numpy(), t32=t32, d32=d32.cpu().numpy(), ref=ref, decided=decided)


def _bar(ours, ref32, ref64):
    """max |ours - float64| and the bar: twice max |float32 torch - float64|, at least 1e-7."""
    err = np.abs(np.asarray(ours, np.float64) - ref64).max()
    return err, max(2 * np.abs(np.asarray(ref32, np.float64) - ref64).max(), 1e-7)


def test_densities_within_twice_the_float32_restatement(sphere):
    err, bar = _bar(sphere["dens"], sphere["d32"], sphere["ref"]["d"])
    assert err <= bar, (err, bar)


def test_crossings_identical_on_decided_vertices(sphere):
    d, ref, decided = sphere["dens"], sphere["ref"], sphere["decided"]
    first, last = oracle.crossings(d, LEVEL)
    assert (1 - decided.mean()) < 1e-3, f"{int((~decided).sum())} undecided vertices"
    assert (first[decided] == ref["first"][decided]).all() and (last[decided] == ref["last"][decided]).all()
    # the scene exercises both bound and interpolated crossings
    assert 0.1 < (ref["first"] > 0).mean() < 0.99 and 0.1 < (ref["last"] < N_SAMPLES - 1).mean() < 0.99


def test_distances_on_decided_vertices(sphere):
    out, t32, ref, dec = sphere["out"], sphere["t32"], sphere["ref"], sphere["decided"]
    for ours, r32, r64 in ((out.outer_dist, t32.outer_dist, ref["outer"]), (out.inner_dist, t32.inner_dist, ref["inner"])):
        err, bar = _bar(ours.cpu().numpy()[dec], r32.cpu().numpy()[dec], r64[dec])
        assert err <= bar, (err, bar)
    shell = sphere["verts"] + out.outer_dist[:, None] * sphere["normals"]
    assert torch.equal(shell, out.outer_verts)


def test_smoothing_over_the_vertex_table(sphere):
    """smooth_K = 4: the mean over knn_points' four nearest vertices of the unsmoothed distances."""
    s = sphere
    sm = level_points_along_normals(s["g"], s["verts"], s["normals"], s["inner"], s["outer"], smooth_K=4, **s["args"])
    idx = knn_points(s["verts"], K=4).idx
    raw = s["out"]
    for ours, r in ((sm.outer_dist, raw.outer_dist), (sm.inner_dist, raw.inner_dist)):
        want = r[idx].sum(1) / 4
        assert (ours - want).abs().max().item() <= 4 * torch.finfo(torch.float32).eps * r.abs().max().item()


def test_two_runs_are_bit_identical(sphere):
    sc, dev = sphere["sc"], sphere["dev"]
    args = (tuple(t.to(dev) for t in sc["sugar"]), sphere["g"], sphere["verts"], sc["faces"].to(dev), EXTENT)
    a, b = initial_shell(*args), initial_shell(*args)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_initial_shell_against_its_float64_restatement(sphere):
    """The whole initialisation (CUDA normals, proposal, both passes, smoothing) against torch_initial_shell in float64
    over the same neighbour tables: a vertex's result moves only when one of its samples sits within rounding of the
    level in either pass, so all but a few vertices agree to float32 rounding."""
    sc, dev = sphere["sc"], sphere["dev"]
    ours = initial_shell(tuple(t.to(dev) for t in sc["sugar"]), sphere["g"], sphere["verts"], sc["faces"].to(dev),
                         EXTENT)
    d64 = lambda ts: tuple(t.to(dev).double() for t in ts)
    ref = torch_initial_shell(d64(sc["sugar"]), d64(sc["gs"]), sc["verts"].to(dev).double(), sc["faces"].to(dev),
                              EXTENT)
    for a, b in ((ours.outer_dist, ref.outer_dist), (ours.inner_dist, ref.inner_dist)):
        off = ((a.double() - b).abs() > 1e-5).double().mean().item()
        assert off < 2e-3, off
    assert (ours.inner_dist >= ours.outer_dist).all()


@pytest.mark.parametrize("smooth_K", [0, 2])
def test_hand_built_branches(cuda_device, smooth_K):
    sc = edge_scene()
    dev = cuda_device
    out, dens = level_points_along_normals(
        tuple(t.to(dev) for t in sc["gaussians"]), sc["verts"].to(dev), sc["normals"].to(dev), sc["inner"].to(dev),
        sc["outer"].to(dev), n_samples=N_SAMPLES, K=2, level=LEVEL, smooth_K=smooth_K, min_layer_size=MIN_LAYER,
        spatial_extent=1.0, min_clamp_inner=sc["clamp_inner"].to(dev), max_clamp_outer=sc["clamp_outer"].to(dev),
        return_densities=True)
    ref = edge_oracle(sc, smooth_K)
    np.testing.assert_allclose(dens.cpu().numpy(), ref["d"], rtol=1e-5, atol=1e-7)
    o, i = out.outer_dist.cpu().numpy(), out.inner_dist.cpu().numpy()
    np.testing.assert_allclose(o, ref["outer"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(i, ref["inner"], rtol=0, atol=1e-5)
    if smooth_K == 0:
        check_edge_values(sc["names"], o, i, 1e-6)
        assert dens[4].max().item() == 1.0            # saturated: d / (d + 1e-12) rounds to 1
    else:
        assert o[0] == o[-1] and i[0] == i[-1]         # the duplicate and its original average the same pair


def test_argument_errors(cuda_device):
    sc = edge_scene()
    dev = cuda_device
    g = tuple(t.to(dev) for t in sc["gaussians"])
    a = dict(gaussians=g, verts=sc["verts"].to(dev), normals=sc["normals"].to(dev), inner_range=sc["inner"].to(dev),
             outer_range=sc["outer"].to(dev), level=LEVEL, spatial_extent=1.0, K=2, smooth_K=0)
    with pytest.raises(ValueError, match="K must be"):
        level_points_along_normals(**dict(a, K=len(g[0]) + 1))
    with pytest.raises(ValueError, match="n_samples"):
        level_points_along_normals(**dict(a, n_samples=33))
    with pytest.raises(ValueError, match="activated"):
        level_points_along_normals(**dict(a, gaussians=g[:3]))
    with pytest.raises(ValueError, match=r"\[n, 3\]"):
        level_points_along_normals(**dict(a, verts=a["verts"][:, :2]))
    with pytest.raises(ValueError, match="one row per vertex"):
        level_points_along_normals(**dict(a, inner_range=a["inner_range"][:-1]))
    bad = g[1].clone()
    bad[3, 1] = float("nan")
    with pytest.raises(ValueError, match="not finite"):
        level_points_along_normals(**dict(a, gaussians=(g[0], bad, g[2], g[3])))
    with pytest.raises(ValueError, match="not finite"):
        level_points_along_normals(**dict(a, normals=a["normals"] * float("inf")))
    with pytest.raises(ValueError, match="faces"):
        initial_shell(g, g, a["verts"], torch.full((1, 3), 99, dtype=torch.int32, device=dev), 1.0)
