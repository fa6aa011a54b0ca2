"""Exact K nearest neighbours over Gaussian centres -- host side of csrc/knn.cu.

SuGaR's trainers rebuild the tracked-neighbour table with pytorch3d's `knn_points(points[None], points[None], K=16)`
(reset_neighbors, frosting_scene/sugar_model.py:1044-1061, and :249), once at iteration 7 001 and then every 500 steps.
Here, without pytorch3d:

    neighbours = SugarNeighbours(knn_points(sugar.points, K=16).idx)

The result is exact and deterministic: for each query the first K points in ascending (d, index) order, d the float32
squared distance of include/frosting_b200.h (fb200_knn).  pytorch3d leaves the order of tied distances unspecified;
here ties go to the lower index.
"""
from collections import namedtuple

import torch

from . import _lib
from ._lib import ptr, stream
from .sugar import MAX_K, _operand

KNN = namedtuple("KNN", "dists idx")


def _check_rows(t, name):
    if not isinstance(t, torch.Tensor) or t.dim() != 2 or t.shape[1] != 3 or t.dtype != torch.float32:
        raise ValueError(f"{name} must be a float32 [n, 3] tensor, got "
                         f"{t.dtype if isinstance(t, torch.Tensor) else type(t).__name__} "
                         f"{list(t.shape) if isinstance(t, torch.Tensor) else ''}")


def _rows(t, name, dev):
    """t as a contiguous, 16-byte aligned float32 [n,3] tensor on the CUDA device dev."""
    if not t.is_cuda or t.device != dev:
        raise ValueError(f"{name} must be on the CUDA device {dev if dev.type == 'cuda' else ''} (no CPU fallback), "
                         f"got {t.device}")
    return _operand(t.detach(), name, tuple(t.shape), dev)


def knn_points(p1, p2=None, K=1):
    """KNN(dists [Q,K] float32, idx [Q,K] int64) of the queries p1 [Q,3] among the points p2 [P,3] (None: p1 itself),
    float32 CUDA tensors on one device -- pytorch3d's knn_points(p1[None], p2[None], K) with norm = 2, unbatched, as
    `.dists[0]` / `.idx[0]`: squared distances, ascending.  1 <= K <= 32 and K <= P.  Runs without gradient (a
    parameter that requires grad is fine) on the device's current stream.  A non-finite coordinate raises ValueError
    after the call (one 4-byte read back)."""
    _check_rows(p1, "p1")
    if p2 is not None:
        _check_rows(p2, "p2")
    dev = p1.device
    with torch.no_grad():
        queries = _rows(p1, "p1", dev)
        points = queries if p2 is None else _rows(p2, "p2", dev)
        Q, P = queries.shape[0], points.shape[0]
        K = int(K)
        if not 1 <= K <= MAX_K or K > P:
            raise ValueError(f"K must be within [1, {MAX_K}] and at most the {P} points, got {K}")
        if P >= 2 ** 31 or Q >= 2 ** 31:
            raise ValueError("at most 2^31 - 1 points and queries")
        dists = torch.empty(Q, K, dtype=torch.float32, device=dev)
        idx = torch.empty(Q, K, dtype=torch.int64, device=dev)
        if Q == 0:
            return KNN(dists, idx)
        L = _lib.lib()
        nbytes = L.fb200_knn_workspace_bytes(P, 0 if p2 is None else Q, K)
        ws = torch.empty(nbytes + 256, dtype=torch.uint8, device=dev)
        ws = ws[(-ws.data_ptr()) % 256:]
        with torch.cuda.device(dev):
            _lib.check(L.fb200_knn(ptr(points), P, None if p2 is None else ptr(queries), Q, K, ptr(ws), nbytes,
                                   ptr(dists), ptr(idx), stream(dev)))
        if int(ws[:4].view(torch.int32).item()) != 0:
            raise ValueError("knn_points: a point or query coordinate is not finite")
        return KNN(dists, idx)
