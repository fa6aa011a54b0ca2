"""knn_points on the GPU: bit-equal to the brute-force oracle (dists and idx) at every extent and on the hard scenes,
correct at scale, deterministic, on the caller's device and stream, and end to end into SuGaR's regulariser."""

import numpy as np
import pytest
import torch

from frosting_b200 import SugarNeighbours, _lib, camera_batch, knn_points, scenes, sdf_regularization
from tests.knn_oracle import check_against_tree, oracle_knn
from tests.test_sugar_reg_gpu import check as check_against_float64

pytestmark = pytest.mark.gpu

KS = (1, 2, 3, 5, 8, 16, 31, 32)


def _bits(d):
    return np.asarray(d, np.float32).view(np.int32)


def _check_prefixes(got_fn, points, queries, Ks):
    """knn_points(K) for each K against one oracle run at max(Ks): the (d, index) order makes every K-list the
    prefix of a longer one."""
    d_ref, i_ref = oracle_knn(points, queries, max(Ks))
    for K in Ks:
        d, i = got_fn(K)
        d, i = d.cpu().numpy(), i.cpu().numpy()
        assert d.shape == i.shape == (len(queries), K)
        bad = ~((_bits(d) == _bits(d_ref[:, :K])) & (i == i_ref[:, :K])).all(1)
        assert not bad.any(), f"K={K}: {int(bad.sum())} rows differ from the oracle, first {np.nonzero(bad)[0][:5]}"


@pytest.mark.parametrize("P", [1, 2, 31, 32, 33, 1023, 1024, 1025, 20000])
def test_bit_equal_to_oracle_at_every_extent(cuda_device, P):
    pts = scenes.knn_scene("cube", P, P)
    Ks = sorted({K for K in KS if K <= P} | ({P} if P <= 32 else set()))
    g = pts.to(cuda_device)
    _check_prefixes(lambda K: knn_points(g, K=K), pts.numpy(), pts.numpy(), Ks)
    # a separate query set, a third of it outside the points' box
    q = torch.rand(3000, 3, generator=torch.Generator().manual_seed(P)) * 1.5 - 0.25
    gq = q.to(cuda_device)
    _check_prefixes(lambda K: knn_points(gq, g, K=K), pts.numpy(), q.numpy(), Ks)


@pytest.mark.parametrize("kind", [k for k in scenes.KNN_SCENES if k != "lattice"])
def test_bit_equal_to_oracle_on_hard_scenes(cuda_device, kind):
    pts = scenes.knn_scene(kind, 20000, 7)
    g = pts.to(cuda_device)
    _check_prefixes(lambda K: knn_points(g, K=K), pts.numpy(), pts.numpy(), (1, 8, 16, 32))


def test_bit_equal_to_oracle_on_the_integer_lattice(cuda_device):
    pts = scenes.knn_scene("lattice", 64 ** 3, 3)
    g = pts.to(cuda_device)
    _check_prefixes(lambda K: knn_points(g, K=K), pts.numpy(), pts.numpy(), (7, 19))


def _c3_centres():
    P, W, H, D, kind, seed = camera_batch.WORKLOADS["c3"]
    threads = torch.get_num_threads()
    torch.set_num_threads(camera_batch.SCENE_THREADS)
    try:
        params, mesh = scenes.frosting_layer(P, scenes.make_camera(W, H), seed, n_faces_target=max(1000, P // 2),
                                             device="cpu")
        return scenes.frosting_attributes(params, mesh)["means3D"].contiguous()
    finally:
        torch.set_num_threads(threads)


@pytest.mark.parametrize("scene", ["sugar_1M", "sugar_3M", "c3_centres"])
def test_at_scale(cuda_device, scene):
    pts = _c3_centres() if scene == "c3_centres" else scenes.knn_scene("sugar", {"sugar_1M": 1_000_000,
                                                                                  "sugar_3M": 3_000_000}[scene], 21)
    K = 16
    g = pts.to(cuda_device)
    d, i = knn_points(g, K=K)
    d2, i2 = knn_points(g, K=K)
    assert torch.equal(d.view(torch.int32), d2.view(torch.int32)) and torch.equal(i, i2), "two runs differ"
    d, i = d.cpu().numpy(), i.cpu().numpy()
    rows = np.random.default_rng(5).choice(len(pts), 512, replace=False)
    d_ref, i_ref = oracle_knn(pts.numpy(), pts.numpy()[rows], K)
    assert (_bits(d[rows]) == _bits(d_ref)).all() and (i[rows] == i_ref).all()
    strict = check_against_tree(pts.numpy(), pts.numpy(), K, i)
    assert strict.mean() > 0.5


def test_empty_queries(cuda_device):
    pts = torch.rand(100, 3, device=cuda_device)
    d, i = knn_points(torch.zeros(0, 3, device=cuda_device), pts, K=4)
    assert d.shape == i.shape == (0, 4) and d.dtype == torch.float32 and i.dtype == torch.int64


def test_second_device_and_its_current_stream():
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    dev = torch.device("cuda:1")
    pts = scenes.knn_scene("cube", 5000, 1)
    g = pts.to(dev)
    s = torch.cuda.Stream(dev)
    with torch.cuda.stream(s):
        d, i = knn_points(g, K=8)
    s.synchronize()
    assert d.device == dev and i.device == dev
    d_ref, i_ref = oracle_knn(pts.numpy(), pts.numpy(), 8)
    assert (_bits(d.cpu().numpy()) == _bits(d_ref)).all() and (i.cpu().numpy() == i_ref).all()


def test_non_finite_inputs_terminate_with_valid_indices(cuda_device):
    pts = scenes.knn_scene("cube", 3000, 9)
    pts[::7, 0] = float("nan")
    pts[3::11, 1] = float("inf")
    pts[5::13, 2] = -float("inf")
    g = pts.to(cuda_device)
    with pytest.raises(ValueError, match="finite"):
        knn_points(g, K=16)
    # the C entry point itself: it terminates, raises the flag and writes indices in [0, P)
    P, K = len(pts), 16
    L = _lib.lib()
    ws = torch.zeros(L.fb200_knn_workspace_bytes(P, 0, K), dtype=torch.uint8, device=cuda_device)
    d = torch.empty(P, K, device=cuda_device)
    i = torch.full((P, K), -1, dtype=torch.int64, device=cuda_device)
    _lib.check(L.fb200_knn(_lib.ptr(g), P, None, P, K, _lib.ptr(ws), ws.numel(), _lib.ptr(d), _lib.ptr(i),
                           _lib.stream(cuda_device)))
    torch.cuda.synchronize()
    assert int(ws[:4].view(torch.int32).item()) != 0
    assert int(i.min()) >= 0 and int(i.max()) < P


def test_end_to_end_into_the_sdf_regulariser(cuda_device):
    """The table knn_points builds equals the scene's cKDTree table on every row rounding cannot reorder, and drives
    sdf_regularization like it.  On samples whose owners' rows agree, the two terms are bit-identical (the regulariser
    reads only the owners' rows, and its terms are reduced in a fixed order).  Its gradients cannot be: the backward
    accumulates them with atomics in no fixed order (csrc/sugar_reg.cu), so two runs over one table already differ in
    the last bits.  Each table's gradients are held to float64 by the regulariser's own bar instead."""
    sc = scenes.sugar_scene(200_000, 13, device=cuda_device)
    ours = knn_points(sc["points"], K=16).idx
    table = sc["knn_idx"]
    strict = check_against_tree(sc["points"].cpu().numpy(), sc["points"].cpu().numpy(), 16, ours.cpu().numpy())
    strict = torch.from_numpy(strict).to(cuda_device)
    assert torch.equal(ours[strict], table[strict])
    agree = (ours == table).all(1)
    assert agree.float().mean() > 0.9
    g = torch.Generator(device=cuda_device).manual_seed(3)
    owners = torch.nonzero(agree).squeeze(1)
    idx = owners[torch.randint(0, owners.numel(), (200_000,), generator=g, device=cuda_device)]
    eps = torch.randn(idx.numel(), 3, generator=g, device=cuda_device)
    leaves = [sc[k] for k in ("points", "scaling", "quaternions", "strengths")]
    with torch.no_grad():
        terms = [torch.stack(sdf_regularization(*leaves, SugarNeighbours(t), idx, eps)) for t in (ours, table)]
    assert torch.equal(terms[0].view(torch.int32), terms[1].view(torch.int32))
    for t, label in ((ours, "knn_points table"), (table, "cKDTree table")):
        check_against_float64(sc, t, idx, eps, label)
