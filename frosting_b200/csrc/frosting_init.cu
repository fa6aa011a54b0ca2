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

}  // namespace

cudaError_t launch_level_points(const fb200_frosting_init& lp, cudaStream_t s) {
    if (lp.n_verts == 0) return cudaSuccess;
    level_points_kernel<<<(lp.n_verts + kInitWarps - 1) / kInitWarps, 32 * kInitWarps, 0, s>>>(lp);
    count_launch();
    level_smooth_kernel<<<(lp.n_verts + kSmoothThreads - 1) / kSmoothThreads, kSmoothThreads, 0, s>>>(lp);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
