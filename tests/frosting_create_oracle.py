"""A model of a Frosting layer's creation after its thickness (frosting_model.py:398-554), in numpy, independent of the
package: the trimming schedule replayed in float32 or float64, the prism inside test in float64 with the magnitudes of
tests/frosting_init_oracle.py, the cell volumes, and distCUDA2's float32 sum over exactly rounded squared distances."""
import numpy as np

from tests.frosting_init_oracle import ULP, F, maximum, read, sqrt

TAU = 16.0              # an inside decision is undecided within TAU * ULP * m of the threshold


def _cross(a, b):
    return [a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]]


def _sub(a, b):
    return [x - y for x, y in zip(a, b)]


def _normalize(a, eps=1e-12):
    n = maximum(sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]), eps)
    return [x / n for x in a]


def projections(shell, faces, queries, idx):
    """F [Q,K,5]: the five projections of is_inside_frosting (:1681-1734) of each query against its K cells, in float64
    from the given shell [2V,3] (inner rows, then outer) with the first-order magnitudes of its float32 values."""
    V = len(shell) // 2
    f = np.asarray(faces, np.int64)[np.asarray(idx, np.int64)]                          # [Q,K,3]
    cv = [[[read(shell[s * V + f[..., k], c]) for c in range(3)] for k in range(3)] for s in range(2)]
    n = [_normalize(_cross(_sub(cv[0][1], cv[0][0]), _sub(cv[1][0], cv[0][0]))),
         _normalize(_cross(_sub(cv[0][2], cv[0][1]), _sub(cv[1][1], cv[0][1]))),
         _normalize(_cross(_sub(cv[1][0], cv[0][0]), _sub(cv[0][2], cv[0][0]))),
         _normalize(_cross(_sub(cv[0][2], cv[0][0]), _sub(cv[0][1], cv[0][0]))),
         _normalize(_cross(_sub(cv[1][1], cv[1][0]), _sub(cv[1][2], cv[1][0])))]
    fp = [cv[0][0], cv[0][1], cv[0][0], cv[0][0], cv[1][0]]
    x = [read(np.asarray(queries)[:, None, c]) for c in range(3)]
    out = []
    for j in range(5):
        d = _sub(x, fp[j])
        out.append(d[0] * n[j][0] + d[1] * n[j][1] + d[2] * n[j][2])
    return F(np.stack([p.v for p in out], -1), np.stack([p.m for p in out], -1))


def trim(verts, faces, normals, inner, outer, th, knn, *, n_iterations=20, dtype=np.float32, kernel_stops=None):
    """The trimming schedule (frosting_model.py:398-435).  Distances, shell and centres in `dtype` with the kernel's
    operation order (dist + step * init; vert + dist * normal; six vertices summed left to right, over 6); the inside
    test in float64 against `th` (float32 rounding of extent * proj_th).  knn(queries, centres) -> [Q,8] table.  With
    kernel_stops = (inner, outer), a decision within TAU * ULP * m of the threshold takes the kernel's side.  Returns
    dict(inner, outer, inner_stop, outer_stop, shell, centres, idx (last iteration), undecided, disagree, per_iter)."""
    t = dtype
    verts, normals = np.asarray(verts, t), np.asarray(normals, t)
    init = [np.asarray(inner, t), np.asarray(outer, t)]
    fl = np.asarray(faces, np.int64)
    V = len(verts)
    step = t(1 / n_iterations)
    dist = [np.zeros(V, t), np.zeros(V, t)]
    stop = [np.full(V, n_iterations, np.int64), np.full(V, n_iterations, np.int64)]
    undecided = disagree = 0
    for it in range(n_iterations):
        active = [s == n_iterations for s in stop]
        trial = [np.where(a, d + step * i, d).astype(t) for a, d, i in zip(active, dist, init)]
        shell = np.concatenate([verts + trial[0][:, None] * normals, verts + trial[1][:, None] * normals]).astype(t)
        cv = np.concatenate([shell[:V][fl], shell[V:][fl]], 1)                              # [F,6,3]
        s = cv[:, 0]
        for k in range(1, 6):
            s = (s + cv[:, k]).astype(t)
        centres = (s / t(6)).astype(t)
        q = np.nonzero(np.concatenate(active))[0]
        idx = np.zeros((2 * V, 8), np.int64)
        if len(q):
            idx[q] = knn(shell[q], centres)
            p = projections(shell.astype(np.float64), fl, shell[q], idx[q])
            above = p.v > th
            band = np.abs(p.v - th) <= TAU * ULP * p.m
            inside = (above & ~band).all(-1).any(-1)
            unsure = ~inside & (above | band).all(-1).any(-1)
            if kernel_stops is not None:
                ks = np.concatenate(kernel_stops)[q] == it
                disagree += int((ks != inside)[~unsure].sum())
                undecided += int(unsure.sum())
                inside = np.where(unsure, ks, inside)
            else:
                inside = (above.all(-1)).any(-1)
            for side in range(2):
                sel = (q >= side * V) & (q < (side + 1) * V)
                v = q[sel] - side * V
                ins = inside[sel]
                dist[side][v[~ins]] = trial[side][v[~ins]]
                stop[side][v[ins]] = it
    return dict(inner=dist[0], outer=dist[1], inner_stop=stop[0], outer_stop=stop[1], shell=shell, centres=centres,
                idx=idx, undecided=undecided, disagree=disagree)


def cell_volumes(verts, faces, inner, outer, extent, camera_center, min_height, contract=True):
    """F [F]: the prism cell volumes of frosting_model.py:441-472 from float32 inputs, float64 with magnitudes, and the
    faces' vertex contraction masks' distance to their threshold, relative (for the undecided band)."""
    fl = np.asarray(faces, np.int64)
    c = [read(np.full(len(verts), np.asarray(camera_center, np.float64).reshape(-1)[k])) for k in range(3)]
    p = [read(np.asarray(verts)[:, k]) for k in range(3)]
    r = _sub(p, c)
    d = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2])
    far = d.v > extent
    x = p
    if contract:
        a = extent * (2.0 - F(extent) / d)
        x = [F(np.where(far, (cc + a * rr / d).v, pp.v), np.where(far, (cc + a * rr / d).m, pp.m))
             for cc, rr, pp in zip(c, r, p)]
    h = maximum(F(np.abs(np.asarray(inner, np.float64) - np.asarray(outer, np.float64)),
                  np.abs(np.asarray(inner, np.float64)) + np.abs(np.asarray(outer, np.float64)) +
                  np.abs(np.asarray(inner, np.float64) - np.asarray(outer, np.float64))), min_height)
    if contract:
        q = F(extent) / d
        hq = h * (q * q)
        h = F(np.where(far, hq.v, h.v), np.where(far, hq.m, h.m))
    fx = [[x[k][fl[:, j]] for k in range(3)] for j in range(3)]
    ln = lambda u, w: sqrt(sum((a_ - b_) * (a_ - b_) for a_, b_ in zip(u, w)) + 0.0)
    A, B, E = ln(fx[0], fx[1]), ln(fx[1], fx[2]), ln(fx[2], fx[0])
    s = (A + B + E) / 2.0
    prod = s * (s - A) * (s - B) * (s - E)
    area = sqrt(maximum(prod, 0.0))
    hf = (h[fl[:, 0]] + h[fl[:, 1]] + h[fl[:, 2]]) / 3.0
    margin = np.abs(d.v - extent) / np.maximum(d.m, 1e-300)
    return area * hf, margin[fl].min(1)


def fma32(a, b, c):
    """fmaf(a, b, c) for float32 arrays, exactly rounded: a * b is exact in float64, the float64 sum is rounded once and
    only a float32 tie of it needs the sign of the sum's error."""
    a, b, c = (np.asarray(x, np.float32).astype(np.float64) for x in (a, b, c))
    p = a * b
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    g = 2 * s - r64                                             # the other float32 neighbour when s is their midpoint
    tie = (g.astype(np.float32).astype(np.float64) == g) & (g != r64) & (e != 0)
    towards = np.where(e > 0, np.maximum(r64, g), np.minimum(r64, g))
    return np.where(tie, towards, r64).astype(np.float32)


def dist_cuda2(points, nn_idx):
    """distCUDA2 over the neighbours nn_idx[:, 1:4]: simple-knn's fmaf(dz, dz, fmaf(dx, dx, dy * dy)) for sm_90a, sorted,
    ((b0 + b1) + b2) / 3 in float32."""
    p = np.asarray(points, np.float32)
    q = p[np.asarray(nn_idx)[:, 1:4]]
    d = (q - p[:, None]).astype(np.float32)
    d2 = fma32(d[..., 2], d[..., 2], fma32(d[..., 0], d[..., 0], (d[..., 1] * d[..., 1]).astype(np.float32)))
    d2 = np.sort(d2, axis=1)
    return (((d2[:, 0] + d2[:, 1]).astype(np.float32) + d2[:, 2]).astype(np.float32) / np.float32(3)).astype(np.float32)
