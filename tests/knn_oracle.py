"""numpy wrapper of the brute-force K-nearest-neighbour oracle (tests/knn_oracle.c), and the float64 agreement
criterion the tests apply against scipy's cKDTree.

The C file is test-local: it is compiled on first use, so the tests need no build step, into a per-user temporary
directory named by a hash of the source, so an edited source is never served by a stale build.  Its flags are
oracle/Makefile's -ffp-contract=off -fno-fast-math, plus -O3 -march=native for speed: the 64^3 lattice test scans
7 * 10^10 pairs.  The explicit fmaf() calls round once at any vector width, so the flags cannot change a result.
Queries are split over host threads, each running its own ctypes call (ctypes releases the GIL).
"""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_SRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "knn_oracle.c")
_lib = None

# The index sets may differ only at points whose float64 distance lies within this relative margin of the float64 K-th
# distance: float32 rounding moves d by at most ~5 * 2^-24 relative, since fl(q - p) is exact to 2^-24.
MARGIN = 2.0 ** -20


def lib():
    global _lib
    if _lib is None:
        src = open(_SRC, "rb").read()
        out = os.path.join(tempfile.gettempdir(), f"fb200_knn_oracle_{os.getuid()}_{hashlib.sha1(src).hexdigest()[:12]}")
        so = os.path.join(out, "libknn_oracle.so")
        if not os.path.exists(so):
            os.makedirs(out, exist_ok=True)
            tmp = f"{so}.{os.getpid()}"
            cmd = ["gcc", "-O3", "-march=native", "-fPIC", "-shared", "-std=c11", "-ffp-contract=off", "-fno-fast-math",
                   "-o", tmp, _SRC, "-lm"]
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError("knn oracle build failed:\n" + r.stderr)
            os.replace(tmp, so)
        _lib = C.CDLL(so)
        _lib.oracle_knn.restype = None
        _lib.oracle_knn.argtypes = [C.c_void_p] * 3 + [C.c_int64, C.c_void_p, C.c_int64, C.c_int64, C.c_int32,
                                                        C.c_void_p, C.c_void_p]
    return _lib


def oracle_knn(points, queries, K, threads=None):
    """(dists [Q,K] float32, idx [Q,K] int64): brute force over all points, the library's expression and tie rule."""
    points = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    queries = np.ascontiguousarray(queries, dtype=np.float32).reshape(-1, 3)
    P, Q = points.shape[0], queries.shape[0]
    xyz = [np.ascontiguousarray(points[:, a]) for a in range(3)]
    assert 1 <= K <= min(32, P)
    dists = np.empty((Q, K), np.float32)
    idx = np.empty((Q, K), np.int64)
    L = lib()
    threads = threads or os.cpu_count() or 1
    step = max(1, -(-Q // (4 * threads)))

    def run(q0):
        q1 = min(Q, q0 + step)
        L.oracle_knn(*[a.ctypes.data for a in xyz], P, queries.ctypes.data, q0, q1, K, dists[q0:q1].ctypes.data,
                     idx[q0:q1].ctypes.data)

    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(run, range(0, Q, step)))
    return dists, idx


def check_against_tree(points, queries, K, idx, margin=MARGIN, chunk=1 << 16):
    """Check the index table idx [Q,K] against scipy's cKDTree in float64: per row, the index set may differ from the
    float64 K nearest only at indices whose float64 squared distance lies within a relative `margin` of the float64
    K-th one.  Returns the mask of rows whose K + 1 nearest float64 distances are all further apart than that (no
    rounding can reorder them), where the ordered rows must be equal, which is asserted too."""
    from scipy.spatial import cKDTree
    p64 = np.asarray(points, np.float64).reshape(-1, 3)
    q64 = np.asarray(queries, np.float64).reshape(-1, 3)
    idx = np.asarray(idx, np.int64).reshape(len(q64), K)
    kq = min(K + 1, len(p64))
    i_ref = cKDTree(p64).query(q64, k=kq, workers=-1)[1].reshape(len(q64), kq)
    strict = np.empty(len(q64), bool)
    for c0 in range(0, len(q64), chunk):
        c = slice(c0, c0 + chunk)
        q = q64[c, None, :]
        d_ref = ((q - p64[i_ref[c]]) ** 2).sum(-1)
        d_got = ((q - p64[idx[c]]) ** 2).sum(-1)
        dk = d_ref[:, K - 1:K]
        band = lambda d: np.abs(d - dk) <= margin * dk
        extra = ~(idx[c, :, None] == i_ref[c, None, :K]).any(-1)
        missing = ~(i_ref[c, :K, None] == idx[c, None, :]).any(-1)
        assert band(d_got)[extra].all(), "a returned neighbour lies outside the float64 K-th distance's band"
        assert band(d_ref[:, :K])[missing].all(), "a float64 neighbour clear of the band is missing"
        strict[c] = (d_ref[:, 1:] > d_ref[:, :-1] * (1 + margin)).all(1)
        rows = strict[c]
        assert (idx[c][rows] == i_ref[c][rows, :K]).all(), "a row with well-separated distances is ordered differently"
    return strict
