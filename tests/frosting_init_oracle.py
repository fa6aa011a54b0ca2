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


# ---------------------------------------------------------------------------------------------------------------------
# The staged model with magnitudes (csrc/frosting_init.cu stage by stage).  Every stage takes the float32 values the
# kernel read and returns float64 values as F: the value and its magnitude m, the first-order change of the value when
# every float32 input and every float32 intermediate of the stage moves by its own relative rounding (each by |x|, in
# units of that rounding, as oracle/blend_f64.py counts its terms).  A float32 computation of the same expression, in
# any association the kernel may contract into FMAs, then sits within a small multiple of ULP * m of the value.

ULP = 2.0 ** -24        # float32 unit roundoff: half an ulp of 1
K_BAND = 16.0           # a decision is undecided within K_BAND * ULP * m of its threshold
EXPF_ULP = 4.0          # expf is within 2 ulp, at most 4 ULP of its value


def f32(x):
    """The float32 constant the kernel holds for x, as a float64."""
    return float(np.float32(x))


class F:
    """A float64 value and its magnitude (see above); operators follow numpy broadcasting and fancy indexing."""
    __slots__ = ("v", "m")

    def __init__(self, v, m=None):
        self.v = np.asarray(v, np.float64)
        self.m = np.zeros_like(self.v) if m is None else np.asarray(m, np.float64)

    def __getitem__(self, i):
        return F(self.v[i], self.m[i])

    def __radd__(self, a):
        return self + a

    def __rmul__(self, a):
        return self * a

    def __neg__(self):
        return F(-self.v, self.m)

    def __add__(self, b):
        b = _f(b)
        v = self.v + b.v
        return F(v, self.m + b.m + np.abs(v))

    def __sub__(self, b):
        return self + (-_f(b))

    def __rsub__(self, a):
        return _f(a) - self

    def __mul__(self, b):
        b = _f(b)
        with np.errstate(invalid="ignore"):
            v = self.v * b.v
            return F(v, self.m * np.abs(b.v) + b.m * np.abs(self.v) + np.abs(v))

    def __truediv__(self, b):
        b = _f(b)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / b.v
            return F(v, (self.m + b.m * np.abs(v)) / np.abs(b.v) + np.abs(v))


def _f(x):
    return x if isinstance(x, F) else F(x)


def read(x):
    """A float32 input as the kernel read it: exact, moving by its own rounding."""
    x = np.asarray(x, np.float64)
    return F(x, np.abs(x))


def sqrt(a):
    """A zero value keeps magnitude 0: the stages only take square roots of sums of squares, which are exactly 0 in
    float32 when every term is (checked separately)."""
    v = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        return F(v, np.where(v > 0, a.m / (2 * v), 0.0) + v)


def exp(a):
    v = np.exp(a.v)
    return F(v, v * (a.m + EXPF_ULP))


def maximum(a, b):
    """max / min move by at most the larger of their arguments' changes."""
    a, b = _f(a), _f(b)
    return F(np.maximum(a.v, b.v), np.maximum(a.m, b.m))


def minimum(a, b):
    a, b = _f(a), _f(b)
    return F(np.minimum(a.v, b.v), np.maximum(a.m, b.m))


def where(c, a, b):
    a, b = _f(a), _f(b)
    return F(np.where(c, a.v, b.v), np.where(c, a.m, b.m))


def stack(fs, axis=-1):
    return F(np.stack([f.v for f in fs], axis), np.stack([f.m for f in fs], axis))


def _sum(terms):
    """Left to right, as the kernel adds (the first add to 0 is exact)."""
    s = terms[0]
    for x in terms[1:]:
        s = s + x
    return s


def _norm(c):
    return sqrt(_sum([x * x for x in c]))


def vertex_normals(verts, faces):
    """Meshes.verts_normals_packed: per vertex the sum of cross(v2 - v1, v0 - v1) over its faces in ascending face order
    (a face naming the vertex twice counts twice), normalised by max(|.|, 1e-6).  Returns F [V,3] and the raw sums
    [V,3] (exactly 0 for a vertex without faces or with only zero-area faces)."""
    verts, faces = np.asarray(verts, np.float64), np.asarray(faces, np.int64).reshape(-1, 3)
    V = len(verts)
    p = [read(verts[faces[:, c]]) for c in range(3)]
    a, b = p[2] - p[1], p[0] - p[1]
    cr = [a[:, 1] * b[:, 2] - a[:, 2] * b[:, 1], a[:, 2] * b[:, 0] - a[:, 0] * b[:, 2],
          a[:, 0] * b[:, 1] - a[:, 1] * b[:, 0]]
    flat = faces.reshape(-1)
    order = np.argsort(flat, kind="stable")                 # per vertex its faces ascending
    vert, face = flat[order], order // 3
    start = np.concatenate([[0], np.cumsum(np.bincount(flat, minlength=V))])[vert]
    s = []
    for c in cr:
        val = c.v[face]
        run = np.cumsum(val)
        partial = run - np.concatenate([[0.0], run])[start]     # the running sum after each of the vertex's faces
        s.append(F(np.bincount(vert, val, V), np.bincount(vert, c.m[face] + np.abs(partial), V)))
    n = maximum(_norm(s), f32(1e-6))
    return stack([c / n for c in s]), np.stack([c.v for c in s], -1)


def _qmul(a, b):
    """quaternion_raw_multiply, (w, x, y, z) tuples of F, each component summed left to right."""
    return (a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3],
            a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
            a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1],
            a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0])


def proposal(normals, scaling, quats, std_idx, std_range):
    """The first pass's range: per vertex the mean over its std_K Gaussians of |s * (q^-1 (0, n) q)| with q raw
    (pytorch3d's quaternion_invert is the conjugate, so a non-unit q scales by |q|^2), times +-std_range.
    Returns (inner F [V], outer F [V], widths F [V, std_K])."""
    idx = np.asarray(std_idx)
    n = read(normals)
    q, s = read(np.asarray(quats, np.float64)[idx]), read(np.asarray(scaling, np.float64)[idx])
    qi = (q[..., 0], -q[..., 1], -q[..., 2], -q[..., 3])
    r = _qmul(_qmul(qi, (F(0.0), n[:, None, 0], n[:, None, 1], n[:, None, 2])), (q[..., 0], q[..., 1], q[..., 2], q[..., 3]))
    width = _norm([s[..., c] * r[c + 1] for c in range(3)])
    std = _sum([width[:, k] for k in range(idx.shape[1])]) / float(idx.shape[1])
    return F(f32(std_range)) * std, F(f32(-std_range)) * std, width


def _neighbours(gaussians, idx):
    """What the kernel stages per neighbour: A[r][c] = R[r][c] / max(s_c, 1e-8) (pytorch3d's quaternion_to_matrix of
    the raw q), the centre and the strength, gathered at idx."""
    pts, scaling, quats, strengths = (np.asarray(a, np.float64) for a in gaussians)
    q = read(quats[idx])
    r, i, j, k = (q[..., c] for c in range(4))
    two_s = F(2.0) / _sum([r * r, i * i, j * j, k * k])
    R = [[1.0 - two_s * (j * j + k * k), two_s * (i * j - k * r), two_s * (i * k + j * r)],
         [two_s * (i * j + k * r), 1.0 - two_s * (i * i + k * k), two_s * (j * k - i * r)],
         [two_s * (i * k - j * r), two_s * (j * k + i * r), 1.0 - two_s * (i * i + j * j)]]
    s = read(scaling[idx])
    inv = [F(1.0) / maximum(s[..., c], f32(1e-8)) for c in range(3)]
    A = [[R[a][c] * inv[c] for c in range(3)] for a in range(3)]
    return A, read(pts[idx]), read(strengths.reshape(-1)[idx])


def stage_densities(gaussians, verts, normals, inner_range, outer_range, knn_idx, fractions, chunk=1024):
    """(t F [V,n], d F [V,n], saturated [V,n]): t_j = frac_j (inner - outer) + outer, x = p + t n, and
    d = sum_k strength_k exp(-min(|A_k^T (x - mu_k)|^2, 1e8) / 2) over the table in order, d / (d + 1e-12) when d >= 1."""
    verts, normals = np.asarray(verts, np.float64), np.asarray(normals, np.float64)
    knn_idx = np.asarray(knn_idx)
    lo = read(outer_range)
    t = read(fractions)[None] * (read(inner_range) - lo)[:, None] + lo[:, None]
    V, n = t.v.shape
    dv, dm, sat = np.empty((V, n)), np.empty((V, n)), np.empty((V, n), bool)
    for s0 in range(0, V, chunk):
        e = slice(s0, min(V, s0 + chunk))
        A, mu, st = _neighbours(gaussians, knn_idx[e])                     # [v,K]
        A = [[x[:, None] for x in row] for row in A]
        mu, st = mu[:, None], st[:, None]
        p, nn = read(verts[e]), read(normals[e])
        x = [p[:, c][:, None] + t[e] * nn[:, c][:, None] for c in range(3)]   # [v,n]
        sh = [x[c][:, :, None] - mu[..., c] for c in range(3)]                  # [v,n,K]
        w = [_sum([A[0][c] * sh[0], A[1][c] * sh[1], A[2][c] * sh[2]]) for c in range(3)]
        m = minimum(maximum(_sum([w[c] * w[c] for c in range(3)]), 0.0), f32(1e8))
        term = st * exp(F(-0.5) * m)
        d = _sum([term[..., k] for k in range(knn_idx.shape[1])])
        sat[e] = d.v >= 1.0
        d = where(sat[e], d / (d + f32(1e-12)), d)
        dv[e], dm[e] = d.v, d.m
    return t, F(dv, dm), sat


def _first_last(above):
    n = above.shape[1]
    anyv = above.any(1)
    return (np.where(anyv, above.argmax(1), 0), np.where(anyv, n - 1 - above[:, ::-1].argmax(1), n - 1))


def level_stage(gaussians, verts, normals, inner_range, outer_range, knn_idx, fractions, *, level, min_layer=0.0,
                half_layer=0.0, min_clamp_inner=None, max_clamp_outer=None, d32=None, raw32=None):
    """One pass of the level kernel before smoothing, from the float32 values it read (level, min_layer and half_layer
    as the float32 constants it holds).  Decisions: a sample is undecided when |d - level| <= K_BAND ULP m_d; its
    above / below bits come from the kernel's own densities d32 [V,n] when given, the rest from float64 (`wrong`: decided
    samples the kernel put on the other side).  The min-layer test |inner - outer| < min_layer is undecided within
    K_BAND ULP of its magnitude; the kernel's choice is read from its raw distances raw32 = (outer, inner) when given.
    With the decisions fixed, the interpolations, empty range, widening and clamps are evaluated with magnitudes.
    Returns a dict of F (t, d, outer, inner, clamps not yet applied: outer_pre, inner_pre) and masks."""
    t, d, saturated = stage_densities(gaussians, verts, normals, inner_range, outer_range, knn_idx, fractions)
    V, n = d.v.shape
    gap = d.v - level
    undecided = np.abs(gap) <= K_BAND * ULP * d.m
    above, under = gap > 0, gap < 0
    wrong = np.zeros_like(undecided)
    if d32 is not None:
        d32 = np.asarray(d32, np.float64)
        wrong = ~undecided & ((d32 > level) != above)
        above, under = np.where(undecided, d32 > level, above), np.where(undecided, d32 < level, under)
    first, last = _first_last(above)
    rows, lev = np.arange(V), read(level)
    fm, la = np.maximum(first - 1, 0), np.minimum(last + 1, n - 1)
    lerp = lambda a, b: (lev - d[rows, a]) / (d[rows, b] - d[rows, a]) * (t[rows, b] - t[rows, a]) + t[rows, a]
    outer = where(first > 0, lerp(fm, first), t[:, 0])
    inner = where(last < n - 1, lerp(last, la), t[:, n - 1])
    centre = (read(inner_range) + read(outer_range)) / 2.0
    empty = (first == 0) & (last == n - 1) & under[:, 0]
    outer, inner = where(empty, centre, outer), where(empty, centre, inner)
    width = inner - outer
    flat = np.abs(width.v) < min_layer
    flat_undecided = (min_layer > 0) & (np.abs(np.abs(width.v) - min_layer) <= K_BAND * ULP * (width.m + min_layer))
    half = read(half_layer)
    wide = (centre - half, centre + half)

    def clamp(o, i):
        ci = None if min_clamp_inner is None else read(min_clamp_inner)
        co = None if max_clamp_outer is None else read(max_clamp_outer)
        return (o if co is None else minimum(o, co)), (i if ci is None else maximum(i, ci))

    if raw32 is not None and flat_undecided.any():
        o32, i32 = (np.asarray(x, np.float64) for x in raw32)
        miss = lambda o, i: np.maximum(np.abs(o32 - o.v) / (o.m + 1e-300), np.abs(i32 - i.v) / (i.m + 1e-300))
        flat = np.where(flat_undecided, miss(*clamp(*wide)) <= miss(*clamp(outer, inner)), flat)
    outer_pre, inner_pre = where(flat, wide[0], outer), where(flat, wide[1], inner)
    outer, inner = clamp(outer_pre, inner_pre)
    return dict(t=t, d=d, undecided=undecided, wrong=wrong, above=above, first=first, last=last, empty=empty,
                flat=flat, flat_undecided=flat_undecided, outer_pre=outer_pre, inner_pre=inner_pre, outer=outer,
                inner=inner, saturated=saturated,
                clamped_inner=np.zeros(V, bool) if min_clamp_inner is None else inner.v > inner_pre.v,
                clamped_outer=np.zeros(V, bool) if max_clamp_outer is None else outer.v < outer_pre.v)


def smooth(values32, smooth_idx):
    """The smoothing kernel from the float32 values it read: the sum over the table in order, over smooth_K."""
    x, idx = read(values32), np.asarray(smooth_idx)
    return _sum([x[idx[:, k]] for k in range(idx.shape[1])]) / float(idx.shape[1])
