"""A float64 model of a Frosting layer's thickness, written from the reference's definition
(frosting_model.py compute_level_points_along_normals, :2078-2200, with use_last_intersection_as_inner_level_point=True)
in numpy, independent of the package: samples t_j = outer + (j / (n - 1)) (inner - outer) along the normal, densities
summed over the given neighbour table, the first and last samples above the level, linear interpolation, and the
reference's edge cases, widening, clamps and smoothing."""
import numpy as np


def quat_to_matrix(q):
    r, i, j, k = (q[:, c] for c in range(4))
    s = 2.0 / (q * q).sum(1)
    return np.stack([1 - s * (j * j + k * k), s * (i * j - k * r), s * (i * k + j * r),
                     s * (i * j + k * r), 1 - s * (i * i + k * k), s * (j * k - i * r),
                     s * (i * k - j * r), s * (j * k + i * r), 1 - s * (i * i + j * j)], 1).reshape(-1, 3, 3)


def densities(gaussians, verts, normals, inner_range, outer_range, knn_idx, n_samples, chunk=4096):
    """(t [V,n], d [V,n]) in float64."""
    pts, scaling, quats, strengths = (np.asarray(a, np.float64) for a in gaussians)
    strengths = strengths.reshape(-1)
    A = quat_to_matrix(quats) / np.maximum(scaling, 1e-8)[:, None, :]      # A[:, i, c] = R[i, c] / s_c
    verts, normals = np.asarray(verts, np.float64), np.asarray(normals, np.float64)
    lo, hi = np.asarray(outer_range, np.float64), np.asarray(inner_range, np.float64)
    frac = np.arange(n_samples) / max(n_samples - 1, 1)
    t = lo[:, None] + frac[None] * (hi - lo)[:, None]
    d = np.empty_like(t)
    for s in range(0, len(verts), chunk):
        e = min(len(verts), s + chunk)
        idx = np.asarray(knn_idx[s:e])
        x = verts[s:e, None] + t[s:e, :, None] * normals[s:e, None]                # [v,n,3]
        shift = x[:, :, None, :] - pts[idx][:, None]                              # [v,n,K,3]
        w = np.einsum("vkic,vnki->vnkc", A[idx], shift)
        m = np.clip((w * w).sum(-1), 0.0, 1e8)
        dd = (strengths[idx][:, None, :] * np.exp(-0.5 * m)).sum(-1)
        d[s:e] = np.where(dd >= 1.0, dd / (dd + 1e-12), dd)
    return t, d


def crossings(d, level):
    """(first, last): the first and last sample above the level; 0 and n - 1 when there is none."""
    above = d > level
    n = d.shape[1]
    anyv = above.any(1)
    first = np.where(anyv, above.argmax(1), 0)
    last = np.where(anyv, n - 1 - above[:, ::-1].argmax(1), n - 1)
    return first, last


def level_points(gaussians, verts, normals, inner_range, outer_range, knn_idx, *, n_samples, level, smooth_idx=None,
                 min_layer=0.0, min_clamp_inner=None, max_clamp_outer=None):
    """dict(t, d, first, last, outer_raw, inner_raw, outer, inner), float64.  min_layer: min_layer_size * extent."""
    t, d = densities(gaussians, verts, normals, inner_range, outer_range, knn_idx, n_samples)
    first, last = crossings(d, level)
    n, rows = d.shape[1], np.arange(len(d))
    fm, lp = np.maximum(first - 1, 0), np.minimum(last + 1, n - 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        outer = np.where(first > 0, (level - d[rows, fm]) / (d[rows, first] - d[rows, fm]) *
                         (t[rows, first] - t[rows, fm]) + t[rows, fm], t[:, 0])
        inner = np.where(last < n - 1, (level - d[rows, last]) / (d[rows, lp] - d[rows, last]) *
                         (t[rows, lp] - t[rows, last]) + t[rows, last], t[:, -1])
    centre = (np.asarray(inner_range, np.float64) + np.asarray(outer_range, np.float64)) / 2
    empty = (first == 0) & (last == n - 1) & (d[:, 0] < level)
    outer, inner = np.where(empty, centre, outer), np.where(empty, centre, inner)
    flat = np.abs(inner - outer) < min_layer
    outer, inner = np.where(flat, centre - min_layer / 2, outer), np.where(flat, centre + min_layer / 2, inner)
    if min_clamp_inner is not None:
        inner = np.maximum(inner, np.asarray(min_clamp_inner, np.float64))
    if max_clamp_outer is not None:
        outer = np.minimum(outer, np.asarray(max_clamp_outer, np.float64))
    out = dict(t=t, d=d, first=first, last=last, outer_raw=outer, inner_raw=inner, empty=empty, flat=flat)
    if smooth_idx is not None:
        outer, inner = outer[smooth_idx].mean(1), inner[smooth_idx].mean(1)
    out.update(outer=outer, inner=inner)
    return out


def self_knn(points, K):
    """Brute-force K nearest points of each point among them, ascending (d, index): ties go to the lower index."""
    p = np.asarray(points, np.float64)
    d = ((p[:, None] - p[None]) ** 2).sum(-1)
    return np.stack([np.lexsort((np.arange(len(p)), row))[:K] for row in d])
