"""Exact K nearest neighbours without a GPU: the brute-force oracle against scipy and a float64 ranking, the C boundary's
argument checks and workspace query, and the Python layer's input checks."""
import ctypes as C

import numpy as np
import pytest
import torch

from frosting_b200 import _lib, knn_points, scenes
from tests.knn_oracle import check_against_tree, oracle_knn

EINVAL, ENOSPC = -1, -3


@pytest.mark.parametrize("kind", scenes.KNN_SCENES + ("sugar_scene",))
def test_oracle_agrees_with_ckdtree(kind):
    if kind == "sugar_scene":
        pts = scenes.sugar_scene(3000, 5)["points"].numpy()
    else:
        pts = scenes.knn_scene(kind, 15 ** 3 if kind == "lattice" else 4000, 11).numpy()
    for K in (1, 7, 16, 32):
        d, i = oracle_knn(pts, pts, K)
        check_against_tree(pts, pts, K, i)
        assert (np.diff(d, axis=1) >= 0).all()


def test_oracle_lattice_matches_float64_ranking():
    pts = scenes.knn_scene("lattice", 12 ** 3, 2).numpy()
    q = np.concatenate([pts, pts[:50] + 0.5, pts[50:90] * 1.5 - 4.0]).astype(np.float32)
    K = 19
    d, i = oracle_knn(pts, q, K)
    d64 = ((q.astype(np.float64)[:, None, :] - pts.astype(np.float64)[None]) ** 2).sum(-1)
    order = np.lexsort((np.broadcast_to(np.arange(len(pts)), d64.shape), d64), axis=1)[:, :K]
    assert (i == order).all()
    assert (d == np.take_along_axis(d64, order, 1).astype(np.float32)).all()


def test_oracle_self_first_on_distinct_points():
    pts = scenes.knn_scene("cube", 2000, 4).numpy()
    d, i = oracle_knn(pts, pts, 4)
    assert (i[:, 0] == np.arange(len(pts))).all() and (d[:, 0] == 0).all()


# fake device addresses: every check below fails before anything touches CUDA
_A = 1 << 20


def _call(P=64, Q=64, K=8, points=_A, queries=None, ws=2 * _A, ws_bytes=None, dists=3 * _A, idx=4 * _A):
    L = _lib.lib()
    if ws_bytes is None:
        ws_bytes = 1 << 40
    return L.fb200_knn(points, P, queries, Q, K, ws, ws_bytes, dists, idx, None)


def test_c_boundary_rejects_bad_arguments():
    L = _lib.lib()
    cases = dict(k0=dict(K=0), k33=dict(K=33), k_over_p=dict(P=4, Q=4, K=5), neg_p=dict(P=-1), neg_q=dict(Q=-1, queries=_A),
                 self_q_mismatch=dict(Q=5), null_points=dict(points=None), null_ws=dict(ws=None),
                 null_dists=dict(dists=None), null_idx=dict(idx=None), misaligned_ws=dict(ws=2 * _A + 16))
    for name, kw in cases.items():
        assert _call(**kw) == EINVAL, name
        assert L.fb200_last_error().decode(), name
    short = L.fb200_knn_workspace_bytes(64, 0, 8) - 1
    assert _call(ws_bytes=short) == ENOSPC
    assert b"workspace" in L.fb200_last_error()
    sep = L.fb200_knn_workspace_bytes(64, 100, 8)
    assert _call(Q=100, queries=5 * _A, ws_bytes=sep - 1) == ENOSPC
    assert _call(Q=0, queries=5 * _A, points=None, ws=None, dists=None, idx=None) == 0     # empty: no launch


def test_workspace_query_is_host_only_linear_and_bounded():
    L = _lib.lib()
    for P, Q, K in ((0, 0, 1), (4, 0, 5), (10, 0, 0), (10, 0, 33), (10, -1, 1), (-5, 0, 1)):
        assert L.fb200_knn_workspace_bytes(P, Q, K) == 0, (P, Q, K)
    prev = 0
    for P in (1, 31, 32, 33, 1000, 2 ** 20, 3_000_000, 2 ** 31 - 1):
        b = L.fb200_knn_workspace_bytes(P, 0, min(16, P))
        assert 40 * P <= b <= 48 * P + 72 * 1024, (P, b)
        assert b >= prev
        prev = b
        assert L.fb200_knn_workspace_bytes(P, 0, 1) == b        # K does not size the workspace
        for Q in (1, 5000, 2 ** 20):
            bq = L.fb200_knn_workspace_bytes(P, Q, 1)
            assert 40 * Q <= bq - b <= 48 * Q + 72 * 1024, (P, Q)


def test_python_layer_rejects_bad_inputs():
    good = torch.zeros(8, 3)
    for bad in (good.double(), good.half(), torch.zeros(8, 4), torch.zeros(8), torch.zeros(2, 8, 3),
                torch.zeros(8, 3, dtype=torch.int32), good.numpy()):
        with pytest.raises(ValueError):
            knn_points(bad, K=1)
        with pytest.raises(ValueError):
            knn_points(good, bad, K=1)
    with pytest.raises(ValueError, match="CUDA|cuda"):
        knn_points(good, K=1)
