// frosting_init.cu -- the thickness of a new Frosting layer (include/frosting_b200.h: fb200_level_points over fb200_frosting_init).
//
// Replaces compute_level_points_along_normals (frosting_model.py:2016-2208), which Frosting.__init__ (:296-369) runs
// twice over every base-mesh vertex: against the coarse SuGaR model with a +-3 sigma proposal, then against the 3DGS
// model inside the widened proposal.  The reference evaluates n_samples x K Gaussians per vertex through [2M,16,3,3]
// torch temporaries, pass after pass; here two kernels:
//   level kernel   one warp per vertex, lane = sample.  Lane 0 sums the vertex normal over its faces (normals stage),
//                  lanes < std_K give the proposal's per-Gaussian widths; lanes < K stage the vertex's neighbour
//                  Gaussians (centre, R diag(1 / s), strength) in shared memory once; every lane then sums its sample's
//                  density over them in table order, and one ballot gives the first and last samples above the level;
//   smooth kernel  one thread per vertex: the mean over its nearest vertices, and the shell vertices.
// Nothing of size samples x K exists, no atomics, no host read-back.
//
// The rest of the constructor (:398-554), over fb200_frosting_create:
//   trimming   n_iterations x (shell kernel: trial shell and cell centres; fb200_knn: 8 nearest centres of all 2V shell
//              vertices; inside kernel: the prism test, advance or freeze), stream-ordered, no read-back;
//   volumes    one thread per face: contracted Heron area times the mean clamped, contracted height;
//   sample     one thread per Gaussian: sorted-uniform barycentrics, their logits, the position in the untrimmed cell and
//              the cell's longest edge;
//   finish     one thread per Gaussian: distCUDA2's mean of the 3 nearest squared distances, the scales, constant
//              rotation and opacity, and the SH rows of the nearest 3DGS Gaussian.
#include "common.cuh"
#include "sugar_common.cuh"
#include "vec3.cuh"

namespace fb200 {

namespace {

constexpr int kInitWarps = 8;
constexpr int kSmoothThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

// a neighbour Gaussian as the density reads it: A = R diag(1 / clamp(s, 1e-8)) row-major, centre, strength
struct Nbr { float A[9]; float mu[3]; float strength; };

// quaternion_raw_multiply (w, x, y, z), each component summed left to right as pytorch3d writes it
__device__ __forceinline__ float4 q_raw_mul(float4 a, float4 b) {
    return make_float4(fadd(fadd(fadd(fmul(a.x, b.x), -fmul(a.y, b.y)), -fmul(a.z, b.z)), -fmul(a.w, b.w)),
                       fadd(fadd(fadd(fmul(a.x, b.y), fmul(a.y, b.x)), fmul(a.z, b.w)), -fmul(a.w, b.z)),
                       fadd(fadd(fadd(fmul(a.x, b.z), -fmul(a.y, b.w)), fmul(a.z, b.x)), fmul(a.w, b.y)),
                       fadd(fadd(fadd(fmul(a.x, b.w), fmul(a.y, b.z)), -fmul(a.z, b.y)), fmul(a.w, b.x)));
}

__device__ __forceinline__ float4 ld_quat(const float* q, int64_t g) {
    return make_float4(__ldg(q + 4 * g), __ldg(q + 4 * g + 1), __ldg(q + 4 * g + 2), __ldg(q + 4 * g + 3));
}

// (level - v0) / (v1 - v0) * (t1 - t0) + t0, the reference's operation order
__device__ __forceinline__ float lerp_level(float level, float v0, float v1, float t0, float t1) {
    return fadd(fmul(__fdiv_rn(fadd(level, -v0), fadd(v1, -v0)), fadd(t1, -t0)), t0);
}

__global__ void __launch_bounds__(32 * kInitWarps)
level_points_kernel(fb200_frosting_init lp) {
    __shared__ Nbr nbrs[kInitWarps][32];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int v = blockIdx.x * kInitWarps + w;
    if (v >= lp.n_verts) return;                     // whole warps leave together
    const V3 p = ld3(lp.d_verts + 3 * (size_t)v);

    // normals stage: lane 0 over the vertex's faces in CSR order
    V3 n = {0.f, 0.f, 0.f};
    if (lp.d_faces) {
        if (lane == 0) {
            float nx = 0.f, ny = 0.f, nz = 0.f;
            const int lo = __ldg(lp.d_vf_offsets + v), hi = __ldg(lp.d_vf_offsets + v + 1);
            for (int j = lo; j < hi; ++j) {
                const int f = __ldg(lp.d_vf_faces + j);
                const V3 an = area_normal(ld3(lp.d_verts + 3 * (size_t)__ldg(lp.d_faces + 3 * f)),
                                          ld3(lp.d_verts + 3 * (size_t)__ldg(lp.d_faces + 3 * f + 1)),
                                          ld3(lp.d_verts + 3 * (size_t)__ldg(lp.d_faces + 3 * f + 2)));
                nx = fadd(nx, an.x); ny = fadd(ny, an.y); nz = fadd(nz, an.z);
            }
            n = normalize_eps({nx, ny, nz}, 1e-6f);
            lp.d_normals[3 * (size_t)v] = n.x; lp.d_normals[3 * (size_t)v + 1] = n.y; lp.d_normals[3 * (size_t)v + 2] = n.z;
        }
        n.x = __shfl_sync(kFull, n.x, 0); n.y = __shfl_sync(kFull, n.y, 0); n.z = __shfl_sync(kFull, n.z, 0);
    } else {
        n = ld3(lp.d_normals + 3 * (size_t)v);
    }

    // proposal stage: lane k < std_K the width of Gaussian k along the normal, lane 0 their mean in table order
    float inner_range, outer_range;
    if (lp.d_std_idx) {
        float width = 0.f;
        if (lane < lp.std_K) {
            const int64_t g = __ldg(lp.d_std_idx + (size_t)v * lp.std_K + lane);
            const float4 q = ld_quat(lp.d_quaternions, g);
            const float4 qi = make_float4(q.x, -q.y, -q.z, -q.w);
            const float4 r = q_raw_mul(q_raw_mul(qi, make_float4(0.f, n.x, n.y, n.z)),
                                       make_float4(qi.x, -qi.y, -qi.z, -qi.w));
            const V3 a = {fmul(__ldg(lp.d_scaling + 3 * g), r.y), fmul(__ldg(lp.d_scaling + 3 * g + 1), r.z),
                          fmul(__ldg(lp.d_scaling + 3 * g + 2), r.w)};
            width = norm3(a);
        }
        float sum = 0.f;
        for (int k = 0; k < lp.std_K; ++k) sum = fadd(sum, __shfl_sync(kFull, width, k));
        const float std = __fdiv_rn(sum, (float)lp.std_K);
        inner_range = fmul(lp.std_range, std);
        outer_range = fmul(-lp.std_range, std);
        if (lane == 0) { lp.d_inner_range[v] = inner_range; lp.d_outer_range[v] = outer_range; }
    } else {
        inner_range = __ldg(lp.d_inner_range + v);
        outer_range = __ldg(lp.d_outer_range + v);
    }

    // stage the neighbours
    Nbr* nb = nbrs[w];
    if (lane < lp.K) {
        const int64_t g = __ldg(lp.d_knn_idx + (size_t)v * lp.K + lane);
        const float4 q = ld_quat(lp.d_quaternions, g);
        float R[9];
        quat_to_matrix(q.x, q.y, q.z, q.w, R);
        float inv[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) inv[c] = __fdiv_rn(1.f, fmaxf(__ldg(lp.d_scaling + 3 * g + c), 1e-8f));
#pragma unroll
        for (int e = 0; e < 9; ++e) nb[lane].A[e] = fmul(R[e], inv[e % 3]);
#pragma unroll
        for (int c = 0; c < 3; ++c) nb[lane].mu[c] = __ldg(lp.d_points + 3 * g + c);
        nb[lane].strength = __ldg(lp.d_strengths + g);
    }
    __syncwarp();

    // this lane's sample and its density
    const int ns = lp.n_samples;
    const int j = min(lane, ns - 1);
    const float t = fadd(fmul(__ldg(lp.d_fractions + j), fadd(inner_range, -outer_range)), outer_range);
    const V3 x = {fadd(p.x, fmul(t, n.x)), fadd(p.y, fmul(t, n.y)), fadd(p.z, fmul(t, n.z))};
    float d = 0.f;
    for (int k = 0; k < lp.K; ++k) {
        const Nbr& g = nb[k];
        const float sx = x.x - g.mu[0], sy = x.y - g.mu[1], sz = x.z - g.mu[2];
        const float w0 = g.A[0] * sx + g.A[3] * sy + g.A[6] * sz;
        const float w1 = g.A[1] * sx + g.A[4] * sy + g.A[7] * sz;
        const float w2 = g.A[2] * sx + g.A[5] * sy + g.A[8] * sz;
        const float m = fminf(fmaxf(w0 * w0 + w1 * w1 + w2 * w2, 0.f), 1e8f);
        d = fadd(d, fmul(g.strength, expf(-0.5f * m)));
    }
    if (d >= 1.f) d = __fdiv_rn(d, fadd(d, 1e-12f));
    if (lp.d_densities && lane < ns) lp.d_densities[(size_t)v * ns + lane] = d;

    // first / last sample above the level
    const float level = lp.level;
    const unsigned above = __ballot_sync(kFull, lane < ns && d > level);
    const int first = above ? __ffs(above) - 1 : 0;
    const int last = above ? 31 - __clz(above) : ns - 1;
    const float d_first = __shfl_sync(kFull, d, first), d_before = __shfl_sync(kFull, d, max(first - 1, 0));
    const float t_first = __shfl_sync(kFull, t, first), t_before = __shfl_sync(kFull, t, max(first - 1, 0));
    const float d_last = __shfl_sync(kFull, d, last), d_after = __shfl_sync(kFull, d, min(last + 1, ns - 1));
    const float t_last = __shfl_sync(kFull, t, last), t_after = __shfl_sync(kFull, t, min(last + 1, ns - 1));
    const float d0 = __shfl_sync(kFull, d, 0), t0 = __shfl_sync(kFull, t, 0), tn = __shfl_sync(kFull, t, ns - 1);
    if (lane != 0) return;

    float outer = first > 0 ? lerp_level(level, d_before, d_first, t_before, t_first) : t0;
    float inner = last < ns - 1 ? lerp_level(level, d_last, d_after, t_last, t_after) : tn;
    const float centre = __fdiv_rn(fadd(inner_range, outer_range), 2.f);
    if (first == 0 && last == ns - 1 && d0 < level) outer = inner = centre;     // nothing above the level
    if (fabsf(fadd(inner, -outer)) < lp.min_layer) {
        outer = fadd(centre, -lp.half_layer);
        inner = fadd(centre, lp.half_layer);
    }
    if (lp.d_min_clamp_inner) inner = fmaxf(inner, __ldg(lp.d_min_clamp_inner + v));
    if (lp.d_max_clamp_outer) outer = fminf(outer, __ldg(lp.d_max_clamp_outer + v));
    lp.d_level_outer[v] = outer;
    lp.d_level_inner[v] = inner;
}

__global__ void __launch_bounds__(kSmoothThreads)
level_smooth_kernel(fb200_frosting_init lp) {
    const int v = blockIdx.x * kSmoothThreads + threadIdx.x;
    if (v >= lp.n_verts) return;
    float outer, inner;
    if (lp.smooth_K > 0) {
        float so = 0.f, si = 0.f;
        for (int k = 0; k < lp.smooth_K; ++k) {
            const int64_t u = __ldg(lp.d_smooth_idx + (size_t)v * lp.smooth_K + k);
            so = fadd(so, lp.d_level_outer[u]);
            si = fadd(si, lp.d_level_inner[u]);
        }
        outer = __fdiv_rn(so, (float)lp.smooth_K);
        inner = __fdiv_rn(si, (float)lp.smooth_K);
    } else {
        outer = lp.d_level_outer[v];
        inner = lp.d_level_inner[v];
    }
    lp.d_outer_dist[v] = outer;
    lp.d_inner_dist[v] = inner;
    const V3 p = ld3(lp.d_verts + 3 * (size_t)v), n = ld3(lp.d_normals + 3 * (size_t)v);
    lp.d_outer_verts[3 * (size_t)v] = fadd(p.x, fmul(outer, n.x));
    lp.d_outer_verts[3 * (size_t)v + 1] = fadd(p.y, fmul(outer, n.y));
    lp.d_outer_verts[3 * (size_t)v + 2] = fadd(p.z, fmul(outer, n.z));
    lp.d_inner_verts[3 * (size_t)v] = fadd(p.x, fmul(inner, n.x));
    lp.d_inner_verts[3 * (size_t)v + 1] = fadd(p.y, fmul(inner, n.y));
    lp.d_inner_verts[3 * (size_t)v + 2] = fadd(p.z, fmul(inner, n.z));
}

constexpr int kCreateThreads = 256;

// the shell vertex of side `side` (0 inner, 1 outer) of vertex v at iteration `it`: an active vertex (it == 0, or never
// stopped so far) at its trial distance dist + step * init, a frozen one where it stopped
__device__ __forceinline__ float trial_dist(const fb200_frosting_create& c, int side, int v, int it, bool* active) {
    const float* dist = side ? c.d_outer_dist : c.d_inner_dist;
    const int32_t* stop = side ? c.d_outer_stop : c.d_inner_stop;
    const float* init = side ? c.d_outer_init : c.d_inner_init;
    *active = it == 0 || stop[v] == c.n_iterations;
    const float d = it == 0 ? 0.f : dist[v];
    return *active ? fadd(d, fmul(c.step, __ldg(init + v))) : d;
}

__device__ __forceinline__ V3 along(const V3& p, float d, const V3& n) {
    return {fadd(p.x, fmul(d, n.x)), fadd(p.y, fmul(d, n.y)), fadd(p.z, fmul(d, n.z))};
}

__device__ __forceinline__ V3 add3(V3 a, V3 b) { return {fadd(a.x, b.x), fadd(a.y, b.y), fadd(a.z, b.z)}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z)); }

__global__ void __launch_bounds__(kCreateThreads)
trim_shell_kernel(fb200_frosting_create c, int it) {
    const int t = blockIdx.x * kCreateThreads + threadIdx.x;
    bool active;
    if (t < c.n_verts) {
        const V3 p = ld3(c.d_verts + 3 * (size_t)t), n = ld3(c.d_normals + 3 * (size_t)t);
        for (int side = 0; side < 2; ++side) {
            const V3 x = along(p, trial_dist(c, side, t, it, &active), n);
            float* o = c.d_shell + 3 * ((size_t)side * c.n_verts + t);
            o[0] = x.x; o[1] = x.y; o[2] = x.z;
        }
    }
    if (t < c.n_faces) {
        // the same six vertices, recomputed from the distances: inner corners 0..2, then outer, summed left to right
        V3 s = {0.f, 0.f, 0.f};
        for (int side = 0; side < 2; ++side)
            for (int k = 0; k < 3; ++k) {
                const int v = __ldg(c.d_faces + 3 * (size_t)t + k);
                s = add3(s, along(ld3(c.d_verts + 3 * (size_t)v), trial_dist(c, side, v, it, &active),
                                  ld3(c.d_normals + 3 * (size_t)v)));
            }
        float* o = c.d_centres + 3 * (size_t)t;
        o[0] = __fdiv_rn(s.x, 6.f); o[1] = __fdiv_rn(s.y, 6.f); o[2] = __fdiv_rn(s.z, 6.f);
    }
}

// is_inside_frosting (frosting_model.py:1675-1737) for one point against one cell of the current shell: every one of the
// five face projections above the threshold.  cv[s][k]: side s (0 inner, 1 outer), corner k.
__device__ bool inside_cell(const fb200_frosting_create& c, const V3& x, int f) {
    V3 cv[2][3];
    for (int s = 0; s < 2; ++s)
        for (int k = 0; k < 3; ++k)
            cv[s][k] = ld3(c.d_shell + 3 * ((size_t)s * c.n_verts + __ldg(c.d_faces + 3 * (size_t)f + k)));
    const float eps = 1e-12f;                                          // F.normalize's
    const V3 n[5] = {normalize_eps(cross(sub(cv[0][1], cv[0][0]), sub(cv[1][0], cv[0][0])), eps),
                     normalize_eps(cross(sub(cv[0][2], cv[0][1]), sub(cv[1][1], cv[0][1])), eps),
                     normalize_eps(cross(sub(cv[1][0], cv[0][0]), sub(cv[0][2], cv[0][0])), eps),
                     normalize_eps(cross(sub(cv[0][2], cv[0][0]), sub(cv[0][1], cv[0][0])), eps),
                     normalize_eps(cross(sub(cv[1][1], cv[1][0]), sub(cv[1][2], cv[1][0])), eps)};
    const V3 fp[5] = {cv[0][0], cv[0][1], cv[0][0], cv[0][0], cv[1][0]};
    for (int j = 0; j < 5; ++j)
        if (!(dot3(sub(x, fp[j]), n[j]) > c.inside_th)) return false;
    return true;
}

__global__ void __launch_bounds__(kCreateThreads)
trim_inside_kernel(fb200_frosting_create c, int it) {
    const int q = blockIdx.x * kCreateThreads + threadIdx.x;
    if (q >= 2 * c.n_verts) return;
    const int side = q >= c.n_verts, v = q - side * c.n_verts;
    bool active;
    const float nd = trial_dist(c, side, v, it, &active);
    if (!active) return;
    const V3 x = ld3(c.d_shell + 3 * (size_t)q);
    bool inside = false;
    for (int k = 0; k < FB200_TRIM_K && !inside; ++k)
        inside = inside_cell(c, x, (int)__ldg(c.d_knn_idx + (size_t)q * FB200_TRIM_K + k));
    float* dist = side ? c.d_outer_dist : c.d_inner_dist;
    int32_t* stop = side ? c.d_outer_stop : c.d_inner_stop;
    if (inside) {
        dist[v] = it == 0 ? 0.f : dist[v];                               // back to the previous iteration's value
        stop[v] = it;
    } else {
        dist[v] = nd;
        stop[v] = c.n_iterations;
    }
}

// contract(x, c, L) (frosting_model.py:36-48): x beyond L from c moves to c + L (2 - L / d) (x - c) / d
__device__ __forceinline__ V3 contract(V3 x, V3 cc, float L) {
    const V3 r = sub(x, cc);
    const float d = norm3(r);
    if (!(d > L)) return x;
    const float a = fmul(L, fadd(2.f, -__fdiv_rn(L, d)));
    return {fadd(cc.x, fmul(a, __fdiv_rn(r.x, d))), fadd(cc.y, fmul(a, __fdiv_rn(r.y, d))),
            fadd(cc.z, fmul(a, __fdiv_rn(r.z, d)))};
}

__global__ void __launch_bounds__(kCreateThreads)
cell_volumes_kernel(fb200_frosting_create c) {
    const int f = blockIdx.x * kCreateThreads + threadIdx.x;
    if (f >= c.n_faces) return;
    const V3 cc = ld3(c.d_camera_center);
    V3 x[3];
    float h = 0.f;
    for (int k = 0; k < 3; ++k) {
        const int v = __ldg(c.d_faces + 3 * (size_t)f + k);
        const V3 p = ld3(c.d_verts + 3 * (size_t)v);
        x[k] = c.contract ? contract(p, cc, c.extent) : p;
        float hv = fmaxf(fabsf(fadd(c.d_inner_dist[v], -c.d_outer_dist[v])), c.min_height);
        if (c.contract) {
            const float d = norm3(sub(p, cc));
            if (d > c.extent) {
                const float r = __fdiv_rn(c.extent, d);
                hv = fmul(hv, fmul(r, r));
            }
        }
        h = fadd(h, hv);
    }
    h = __fdiv_rn(h, 3.f);
    const float a = norm3(sub(x[0], x[1])), b = norm3(sub(x[1], x[2])), e = norm3(sub(x[2], x[0]));
    const float s = __fdiv_rn(fadd(fadd(a, b), e), 2.f);
    const float area = __fsqrt_rn(fmaxf(fmul(fmul(fmul(s, fadd(s, -a)), fadd(s, -b)), fadd(s, -e)), 0.f));
    c.d_volumes[f] = fmul(area, h);
}

__global__ void __launch_bounds__(kCreateThreads)
sample_gaussians_kernel(fb200_frosting_create c) {
    const int i = blockIdx.x * kCreateThreads + threadIdx.x;
    if (i >= c.n_gaussians) return;
    float u[6];
    for (int k = 0; k < 5; ++k) u[k] = __ldg(c.d_u + 6 * (size_t)i + k);
    u[5] = 1.f;
#pragma unroll
    for (int a = 0; a < 5; ++a)                                          // ascending: the sorted values, ties immaterial
#pragma unroll
        for (int b = 0; b < 5 - a; ++b) {
            const float lo = fminf(u[b], u[b + 1]), hi = fmaxf(u[b], u[b + 1]);
            u[b] = lo; u[b + 1] = hi;
        }
    const int64_t f = __ldg(c.d_cells + i);
    V3 cv[6];
    for (int k = 0; k < 3; ++k) {
        const int v = __ldg(c.d_faces + 3 * f + k);
        cv[k] = ld3(c.d_inner_verts + 3 * (size_t)v);
        cv[3 + k] = ld3(c.d_outer_verts + 3 * (size_t)v);
    }
    V3 p = {0.f, 0.f, 0.f};
    for (int k = 0; k < 6; ++k) {
        const float b = k == 0 ? u[0] : fadd(u[k], -u[k - 1]);
        c.d_bary_logits[6 * (size_t)i + k] = logf(fmaxf(b, 1e-8f));
        p = add3(p, {fmul(b, cv[k].x), fmul(b, cv[k].y), fmul(b, cv[k].z)});
    }
    c.d_points[3 * (size_t)i] = p.x; c.d_points[3 * (size_t)i + 1] = p.y; c.d_points[3 * (size_t)i + 2] = p.z;
    // the cell's 9 edges: 3 sides, then each side's base edges k -> k + 1
    float m = 0.f;
    for (int k = 0; k < 3; ++k) m = fmaxf(m, norm3(sub(cv[3 + k], cv[k])));
    for (int s = 0; s < 2; ++s)
        for (int k = 0; k < 3; ++k) m = fmaxf(m, norm3(sub(cv[3 * s + k], cv[3 * s + (k + 1) % 3])));
    c.d_max_scales[i] = m;
}

// simple-knn's squared distance as nvcc contracts `d.x*d.x + d.y*d.y + d.z*d.z` for sm_90a (its SASS: FMUL on y, then
// FFMA x, FFMA z) -- not fb200_knn's order, so the neighbours' distances are recomputed here
__device__ __forceinline__ float sknn_dist2(V3 a, V3 b) {
    const float dx = fadd(b.x, -a.x), dy = fadd(b.y, -a.y), dz = fadd(b.z, -a.z);
    return __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, fmul(dy, dy)));
}

__global__ void __launch_bounds__(kCreateThreads)
finish_gaussians_kernel(fb200_frosting_create c) {
    const int i = blockIdx.x * kCreateThreads + threadIdx.x;
    if (i >= c.n_gaussians) return;
    const V3 p = ld3(c.d_points + 3 * (size_t)i);
    float d[3];
    for (int k = 0; k < 3; ++k) d[k] = sknn_dist2(p, ld3(c.d_points + 3 * __ldg(c.d_nn_idx + 4 * (size_t)i + 1 + k)));
    const float lo = fminf(d[0], d[1]), hi = fmaxf(d[0], d[1]);        // ascending, as updateKBest keeps them
    const float b0 = fminf(lo, d[2]), b2 = fmaxf(hi, d[2]), b1 = fmaxf(lo, fminf(hi, d[2]));
    const float dist2 = __fdiv_rn(fadd(fadd(b0, b1), b2), 3.f);
    c.d_dist2[i] = dist2;
    const float ms = c.d_max_scales[i];
    const float s = logf(__fsqrt_rn(fmaxf(fminf(dist2, fmul(ms, ms)), 1e-7f)));
    for (int k = 0; k < 3; ++k) c.d_log_scales[3 * (size_t)i + k] = s;
    c.d_quats[4 * (size_t)i] = 1.f;
    for (int k = 1; k < 4; ++k) c.d_quats[4 * (size_t)i + k] = 0.f;
    c.d_opacity_logits[i] = logf(__fdiv_rn(0.1f, fadd(1.f, -0.1f)));    // inverse_sigmoid(0.1) in float32
    const int64_t g = __ldg(c.d_sh_idx + i);
    for (int k = 0; k < 3; ++k) c.d_sh_dc[3 * (size_t)i + k] = __ldg(c.d_gs_sh_dc + 3 * g + k);
    const int w = 3 * c.sh_rest;
    for (int k = 0; k < w; ++k) c.d_sh_rest[(size_t)w * i + k] = __ldg(c.d_gs_sh_rest + w * g + k);
}

int blocks(int n) { return (n + kCreateThreads - 1) / kCreateThreads; }

}  // namespace

cudaError_t launch_frosting_trim(const fb200_frosting_create& c, cudaStream_t s) {
    for (int it = 0; it < c.n_iterations; ++it) {
        trim_shell_kernel<<<blocks(max(c.n_verts, c.n_faces)), kCreateThreads, 0, s>>>(c, it);
        count_launch();
        cudaError_t e = launch_knn(c.d_centres, c.n_faces, c.d_shell, 2 * c.n_verts, FB200_TRIM_K, c.d_knn_workspace,
                                   c.d_knn_dists, c.d_knn_idx, s);
        if (e != cudaSuccess) return e;
        trim_inside_kernel<<<blocks(2 * c.n_verts), kCreateThreads, 0, s>>>(c, it);
        count_launch();
    }
    return cudaGetLastError();
}

cudaError_t launch_frosting_volumes(const fb200_frosting_create& c, cudaStream_t s) {
    cell_volumes_kernel<<<blocks(c.n_faces), kCreateThreads, 0, s>>>(c);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_frosting_sample(const fb200_frosting_create& c, cudaStream_t s) {
    sample_gaussians_kernel<<<blocks(c.n_gaussians), kCreateThreads, 0, s>>>(c);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_frosting_finish(const fb200_frosting_create& c, cudaStream_t s) {
    finish_gaussians_kernel<<<blocks(c.n_gaussians), kCreateThreads, 0, s>>>(c);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_level_points(const fb200_frosting_init& lp, cudaStream_t s) {
    if (lp.n_verts == 0) return cudaSuccess;
    level_points_kernel<<<(lp.n_verts + kInitWarps - 1) / kInitWarps, 32 * kInitWarps, 0, s>>>(lp);
    count_launch();
    level_smooth_kernel<<<(lp.n_verts + kSmoothThreads - 1) / kSmoothThreads, kSmoothThreads, 0, s>>>(lp);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
