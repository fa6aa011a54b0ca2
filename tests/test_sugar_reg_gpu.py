"""SuGaR's SDF regulariser on the GPU against float64.

Three results from the same float32 inputs: ours (`sdf_regularization`), R32 (`torch_reference` in float32 on the GPU:
the reference's own arithmetic) and R64 (`torch_reference` in float64).  The bar, as for the photometric loss: ours may
be at most twice as far from R64 as R32 is, plus 1e-6 of R64's size --
  - each term: |ours - R64| <= 2 |R32 - R64| + 1e-6 |R64|;
  - each gradient tensor, on the largest error and on the 99.9th percentile of the errors:
    err(ours) <= 2 err(R32) + 1e-6 max|R64|.
The gradients are those of est * a + nrm * b for the upstream pairs (a, b) below."""
import pytest
import torch

from frosting_b200 import scenes, sugar

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LEAVES = ("points", "scaling", "quaternions", "strengths")
UPSTREAM = ((1.0, 1.0), (0.2, 0.0), (0.0, 3.0), (-0.5, 1.0))
# K covers every lane-group width of the sample kernel: 1, 2, 4, 8, 16 and 32 lanes per sample
CASES = [(1, 1, 1), (1, 1, 1000), (1, 1, 1_000_000), (17, 2, 1000), (17, 5, 1000), (17, 16, 1), (17, 16, 1_000_000),
         (2000, 16, 1000), (2000, 3, 1_000_000), (2000, 5, 1_000_000), (2000, 1, 1000), (2000, 20, 1000),
         (200_000, 16, 1_000_000), (200_000, 5, 1000), (200_000, 32, 1_000_000), (1_000_000, 16, 1_000_000),
         (3_000_000, 16, 1_000_000)]


def _reference(sc, knn, idx, eps, dtype):
    leaves = [sc[k].to(dtype).requires_grad_(True) for k in LEAVES]
    est, nrm = sugar.torch_reference(*leaves, knn.long(), idx, eps.to(dtype))
    g_est = torch.autograd.grad(est, leaves, retain_graph=True, allow_unused=True)
    g_nrm = torch.autograd.grad(nrm, leaves, allow_unused=True)
    z = lambda g, l: torch.zeros_like(l) if g is None else g
    return (torch.stack([est, nrm]).detach().double(),
            [z(g, l).double() for g, l in zip(g_est, leaves)], [z(g, l).double() for g, l in zip(g_nrm, leaves)])


def _quantile(x, q):
    x = x.reshape(-1)
    return float(x.kthvalue(max(1, int(round(q * x.numel())))).values) if x.numel() else 0.0


def check(sc, knn, idx, eps, label):
    """Runs the three routes and asserts the bar for both terms and every upstream pair; returns the worst ratios."""
    leaves = {k: sc[k].clone().requires_grad_(True) for k in LEAVES}
    est, nrm = sugar.sdf_regularization(*leaves.values(), sugar.SugarNeighbours(knn), idx, eps)
    ours_t = torch.stack([est, nrm]).detach().double()
    t32, e32, n32 = _reference(sc, knn, idx, eps, torch.float32)
    t64, e64, n64 = _reference(sc, knn, idx, eps, torch.float64)
    bound = 2 * (t32 - t64).abs() + 1e-6 * t64.abs()
    assert bool(((ours_t - t64).abs() <= bound).all()), (label, ours_t.tolist(), t32.tolist(), t64.tolist())
    worst = 0.0
    for a, b in UPSTREAM:
        ours = torch.autograd.grad((est, nrm), list(leaves.values()),
                                   grad_outputs=(torch.tensor(a, device=DEV), torch.tensor(b, device=DEV)),
                                   retain_graph=True)
        for k, o, ge32, gn32, ge64, gn64 in zip(LEAVES, ours, e32, n32, e64, n64):
            r64 = a * ge64 + b * gn64
            err_o, err_r = (o.double() - r64).abs(), (a * ge32 + b * gn32 - r64).abs()
            floor = 1e-6 * float(r64.abs().max()) if r64.numel() else 0.0
            for stat in (lambda e: float(e.max()), lambda e: _quantile(e, 0.999)):
                lhs, rhs = stat(err_o), 2 * stat(err_r) + floor
                assert lhs <= rhs, (label, (a, b), k, lhs, stat(err_r), floor)
                worst = max(worst, lhs / rhs if rhs > 0 else 0.0)
    return worst


_SCENES = {}


def scene(P, K):
    if (P, K) not in _SCENES:
        sc = scenes.sugar_scene(P, P + K, K=K)
        _SCENES.clear()
        _SCENES[(P, K)] = ({k: v.to(DEV) for k, v in sc.items() if k != "knn_idx"}, sc["knn_idx"].to(DEV))
    return _SCENES[(P, K)]


@pytest.mark.parametrize("P,K,N", CASES)
def test_sweep_against_float64(P, K, N):
    sc, knn = scene(P, K)
    torch.manual_seed(P * 31 + K * 7 + N)
    mask = torch.rand(P, device=DEV) < 0.6
    mask[0] = True
    idx, eps = sugar.sample_in_gaussians(mask, N)
    check(sc, knn, idx, eps, (P, K, N))


def hand_built():
    """Eight Gaussians and 40 samples that reach every branch of the operation."""
    pts = torch.tensor([[0.0, 0.0, 0.0], [0.05, 0.0, 0.0], [100.0, 0.0, 0.0], [0.0, 0.05, 0.0], [-100.0, 0.0, 0.0],
                        [0.0, 0.0, 1.0], [0.01, 0.0, 1.0], [0.0, 0.01, 1.0]])
    scl = torch.tensor([[0.1, 0.1, 0.01], [0.01, 0.1, 0.1], [0.001, 0.002, 0.003], [1e-9, 0.05, 0.04],
                        [0.02, 0.03, 0.01], [0.2, 0.15, 0.05], [0.1, 0.02, 0.15], [0.12, 0.11, 0.03]])
    g = torch.Generator().manual_seed(3)
    q = torch.nn.functional.normalize(torch.randn(8, 4, generator=g), dim=-1)
    q[0] = q[1] = torch.tensor([1.0, 0.0, 0.0, 0.0])      # axis-aligned: normals e_z and e_x, exactly orthogonal
    # the 1e-9 axis: axis-aligned at x = 0, so that its samples' offsets along it (~1e-9) are exact in float32 (rotated,
    # or far from the origin, they would be below the rounding of the other coordinates, and every float32 evaluation,
    # the reference's included, would return noise there)
    q[3] = torch.tensor([1.0, 0.0, 0.0, 0.0])
    strengths = torch.tensor([[0.9], [0.8], [0.7], [0.6], [0.5], [0.95], [0.9], [0.99]])
    knn = torch.tensor([[0, 1, 2, 3, 5], [1, 0, 3, 2, 4], [2, 0, 1, 3, 4], [3, 0, 1, 2, 5], [4, 2, 0, 1, 3],
                        [5, 6, 7, 0, 3], [6, 5, 7, 0, 1], [7, 5, 6, 3, 0]])
    idx = torch.tensor([0, 0, 1, 1, 2, 3, 3, 4, 4] + [5] * 25 + [6, 6, 7, 7, 0, 3])
    eps = torch.randn(len(idx), 3, generator=g)
    eps[7] = torch.tensor([20.0, 0.0, 0.0])      # owner 4 far from all: every opacity underflows, d = 0
    eps[9:15] = 0.0                               # eps = 0 at the centre of overlapping Gaussians: d >= 1
    sc = dict(points=pts, scaling=scl, quaternions=q, strengths=strengths)
    return {k: v.to(DEV).contiguous() for k, v in sc.items()}, knn.to(DEV), idx.to(DEV), eps.to(DEV)


def test_hand_built_branches():
    sc, knn, idx, eps = hand_built()
    est, nrm, f = sugar.torch_reference(*(sc[k].double() for k in LEAVES), knn.long(), idx, eps.double(),
                                        return_fields=True)
    d = f["density"]
    assert float(d[7]) < 1e-30 and float(d[9:15].min()) >= 1.0
    assert float(sc["scaling"].min()) < 1e-8
    # the sign of e_z . e_x is 0; a neighbour 100 away has |w|^2 far above 1e8
    assert float(sc["points"][2, 0] / sc["scaling"][2].max()) ** 2 > 1e8
    check(sc, knn, idx, eps, "hand-built")


def test_terms_are_bit_reproducible_and_forward_only_agrees():
    sc, knn = scene(2000, 16)
    torch.manual_seed(0)
    idx, eps = sugar.sample_in_gaussians(torch.ones(2000, dtype=torch.bool, device=DEV), 100_000)
    nb = sugar.SugarNeighbours(knn)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    a = torch.stack(sugar.sdf_regularization(*leaves, nb, idx, eps)).detach()
    b = torch.stack(sugar.sdf_regularization(*leaves, nb, idx, eps)).detach()
    with torch.no_grad():
        c = torch.stack(sugar.sdf_regularization(*(sc[k] for k in LEAVES), nb, idx, eps))
    assert torch.equal(a, b)
    # the forward-only instance is compiled separately (its floating-point contractions may differ): same terms to 1e-6
    assert torch.allclose(a, c, rtol=1e-6, atol=0)


def test_empty_mask_gives_zero_terms_and_gradients():
    sc, knn = scene(2000, 16)
    idx, eps = sugar.sample_in_gaussians(torch.zeros(2000, dtype=torch.bool, device=DEV), 1_000_000)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    est, nrm = sugar.sdf_regularization(*leaves, sugar.SugarNeighbours(knn), idx, eps)
    assert float(est.detach()) == 0.0 and float(nrm.detach()) == 0.0
    (0.2 * est + 0.2 * nrm).backward()
    for l in leaves:
        assert l.grad is not None and l.grad.shape == l.shape and not l.grad.any()


def _peak_extra(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def test_peak_memory_is_independent_of_samples_times_neighbours():
    """Extra device memory of one forward + backward, above the inputs: at most 256 bytes per Gaussian (80-byte record,
    128-byte accumulator, 44 bytes of gradients) + 1 byte per sample (the block partials) + 64 KiB of small
    allocations, whatever K and N (below 2^18 Gaussians the accumulator replicas add up to 32 MiB; not here)."""
    P = 200_000
    sc, knn = scene(P, 16)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    for K in (4, 16):
        nb = sugar.SugarNeighbours(knn[:, :K])
        for N in (1000, 1_000_000):
            torch.manual_seed(1)
            idx, eps = sugar.sample_in_gaussians(torch.ones(P, dtype=torch.bool, device=DEV), N)

            def step():
                est, nrm = sugar.sdf_regularization(*leaves, nb, idx, eps)
                return torch.autograd.grad(0.2 * est + 0.2 * nrm, leaves)

            _, extra = _peak_extra(step)
            assert extra <= 256 * P + N + 65536, (K, N, extra)


def test_forward_under_no_grad_skips_the_gradient_pass():
    """Under torch.no_grad(), with inputs that require grad, the forward allocates no accumulators: only the records
    (80 B per Gaussian), the partials and the terms, plus up to 2 MiB of rounding (torch's caching allocator rounds
    blocks above 1 MiB up to a multiple of 2 MiB).  The accumulators would add 128 B per Gaussian, 25.6 MB here.  Its
    terms are those of the gradient pass to 1e-6."""
    P = 200_000
    sc, knn = scene(P, 16)
    nb = sugar.SugarNeighbours(knn)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    torch.manual_seed(2)
    idx, eps = sugar.sample_in_gaussians(torch.ones(P, dtype=torch.bool, device=DEV), 100_000)
    with torch.no_grad():
        terms, extra = _peak_extra(lambda: torch.stack(sugar.sdf_regularization(*leaves, nb, idx, eps)))
    assert not terms.requires_grad
    assert extra <= 80 * P + 100_000 + (2 << 20) + 65536, extra
    with_grad = torch.stack(sugar.sdf_regularization(*leaves, nb, idx, eps)).detach()
    assert torch.allclose(terms, with_grad, rtol=1e-6, atol=0)


def test_out_of_range_owner_makes_the_terms_nan():
    """Owner indices outside [0, P) (a sampling mask of another scene, say) are caught on the device: the samples are
    skipped and both terms are NaN; the gradients of the other samples are still finite."""
    P = 2000
    sc, knn = scene(P, 16)
    nb = sugar.SugarNeighbours(knn)
    leaves = [sc[k].clone().requires_grad_(True) for k in LEAVES]
    torch.manual_seed(3)
    idx, eps = sugar.sample_in_gaussians(torch.ones(P + 500, dtype=torch.bool, device=DEV), 10_000)
    assert int(idx.max()) >= P
    idx[0] = -1
    est, nrm = sugar.sdf_regularization(*leaves, nb, idx, eps)
    assert bool(torch.isnan(est.detach())) and bool(torch.isnan(nrm.detach()))
    grads = torch.autograd.grad(est + nrm, leaves)
    assert all(bool(torch.isfinite(g).all()) for g in grads)
