// frosting_attr.cuh -- Frosting's parameter -> attribute maps as device functions.
//
// Shared by the stand-alone attribute kernels (frosting_attr.cu) and by the frosting mode of preprocess / geom_bwd
// (SURVEY.md row f1: attributes built inside the rasterizer's own per-Gaussian kernels, nothing materialised), so the
// two paths produce the same values bit for bit: every rounding is explicit, nothing is left to FMA contraction.
//   bary_coords  frosting_scene/frosting_model.py:713-719  softmax over the 6 prism-cell logits
//   points       :721-726   sum_k bary_k * shell_cells_verts[cell][k]   (inner v0..v2, outer v0..v2, :705-710)
//   strengths    :729-730   sigmoid
//   scaling      :765       exp
//   quaternions  :798       F.normalize (eps 1e-12)
#pragma once

#include "common.cuh"

namespace fb200 {

__device__ __forceinline__ void frost_softmax6(const float* __restrict__ logits, float* w) {
    // rows of 6 floats are 8-byte aligned (16-byte aligned tensor base): three 64-bit loads
    const float2* l2 = reinterpret_cast<const float2*>(logits);
    const float2 l01 = __ldg(l2), l23 = __ldg(l2 + 1), l45 = __ldg(l2 + 2);
    const float l[6] = {l01.x, l01.y, l23.x, l23.y, l45.x, l45.y};
    float m = l[0];
#pragma unroll
    for (int k = 1; k < 6; ++k) m = fmaxf(m, l[k]);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) { w[k] = expf(fadd(l[k], -m)); s = fadd(s, w[k]); }
    const float inv = __fdiv_rn(1.0f, s);
#pragma unroll
    for (int k = 0; k < 6; ++k) w[k] = fmul(w[k], inv);
}

// softmax weights, the cell's three vertex ids, and the point itself
__device__ __forceinline__ void frost_point(const fb200_frosting_params& p, size_t i, float* w, int* vid,
                                            float& px, float& py, float& pz) {
    frost_softmax6(p.d_bary_logits + 6 * i, w);
    const long long cell = __ldg(p.d_cells + i);
#pragma unroll
    for (int k = 0; k < 3; ++k) vid[k] = __ldg(p.d_faces + 3 * cell + k);
    px = 0.f; py = 0.f; pz = 0.f;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float* vi = p.d_inner_verts + 3 * (size_t)vid[k];
        const float* vo = p.d_outer_verts + 3 * (size_t)vid[k];
        px = ffma(w[k], __ldg(vi), px);     px = ffma(w[3 + k], __ldg(vo), px);
        py = ffma(w[k], __ldg(vi + 1), py); py = ffma(w[3 + k], __ldg(vo + 1), py);
        pz = ffma(w[k], __ldg(vi + 2), pz); pz = ffma(w[3 + k], __ldg(vo + 2), pz);
    }
}

__device__ __forceinline__ float frost_sigmoid(float x) { return __fdiv_rn(1.0f, fadd(1.0f, expf(-x))); }

// F.normalize: q / max(|q|, 1e-12); returns the norm used
__device__ __forceinline__ float4 frost_normalize(float4 q, float& nrm) {
    nrm = fmaxf(__fsqrt_rn(ffma(q.w, q.w, ffma(q.z, q.z, ffma(q.y, q.y, fmul(q.x, q.x))))), 1e-12f);
    return make_float4(__fdiv_rn(q.x, nrm), __fdiv_rn(q.y, nrm), __fdiv_rn(q.z, nrm), __fdiv_rn(q.w, nrm));
}

// the chain rule back through the maps above, for one Gaussian:
//   g_mean (dL/dpoint) -> bary logits (softmax backward) and the six shell vertices (scatter-add)
__device__ __forceinline__ void frost_point_backward(const fb200_frosting_params& p, const float* w, const int* vid,
                                                     float gx, float gy, float gz, float* g_inner, float* g_outer,
                                                     float* gb) {
    float dw[6];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float* vi = p.d_inner_verts + 3 * (size_t)vid[k];
        const float* vo = p.d_outer_verts + 3 * (size_t)vid[k];
        dw[k] = gx * __ldg(vi) + gy * __ldg(vi + 1) + gz * __ldg(vi + 2);
        dw[3 + k] = gx * __ldg(vo) + gy * __ldg(vo + 1) + gz * __ldg(vo + 2);
        if (g_inner != nullptr && (gx != 0.f || gy != 0.f || gz != 0.f)) {
            float* di = g_inner + 3 * (size_t)vid[k];
            float* dout = g_outer + 3 * (size_t)vid[k];
            atomicAdd(di, w[k] * gx); atomicAdd(di + 1, w[k] * gy); atomicAdd(di + 2, w[k] * gz);
            atomicAdd(dout, w[3 + k] * gx); atomicAdd(dout + 1, w[3 + k] * gy); atomicAdd(dout + 2, w[3 + k] * gz);
        }
    }
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < 6; ++k) dot += w[k] * dw[k];
#pragma unroll
    for (int k = 0; k < 6; ++k) gb[k] = w[k] * (dw[k] - dot);
}

// d/dq of normalize: (g - n <n, g>) / |q|
__device__ __forceinline__ float4 frost_normalize_backward(float4 n, float nrm, float4 g) {
    const float ng = n.x * g.x + n.y * g.y + n.z * g.z + n.w * g.w;
    return make_float4((g.x - n.x * ng) / nrm, (g.y - n.y * ng) / nrm, (g.z - n.z * ng) / nrm, (g.w - n.w * ng) / nrm);
}

// Background Gaussians (frosting_model.py:801-876): row i of a frosting-mode frame is mesh row i of the parameter block
// for i < P and background row i - P (its d_bg_* rows) after them.  Both go through the maps above (sigmoid, exp,
// normalize, dc | rest); only the position differs: a background row stores it (bg_points), a mesh row builds it in its
// prism cell.  The rows are chosen at run time: they are contiguous, so only the warp that straddles P mixes the two.
template <typename T>
struct FrostRowT {
    T* opacity_logits; T* log_scales; T* quats; T* sh_dc; T* sh_rest;   // row pointers into the mesh or background rows
    size_t r;                                                           // row among those
    bool bg;
};

__device__ __forceinline__ FrostRowT<const float> frost_row(const fb200_frosting_params& p, size_t i) {
    FrostRowT<const float> s;
    s.bg = i >= (size_t)p.P;
    s.r = s.bg ? i - (size_t)p.P : i;
    s.opacity_logits = (s.bg ? p.d_bg_opacity_logits : p.d_opacity_logits) + s.r;
    s.log_scales = (s.bg ? p.d_bg_log_scales : p.d_log_scales) + 3 * s.r;
    s.quats = (s.bg ? p.d_bg_quats : p.d_quats) + 4 * s.r;
    s.sh_dc = (s.bg ? p.d_bg_sh_dc : p.d_sh_dc) + 3 * s.r;
    s.sh_rest = (s.bg ? p.d_bg_sh_rest : p.d_sh_rest) + s.r * (size_t)p.sh_rest * 3;
    return s;
}

__device__ __forceinline__ FrostRowT<float> frost_grad_row(const fb200_frosting_params& p, const fb200_frosting_grads& g,
                                                           size_t i) {
    FrostRowT<float> s;
    s.bg = i >= (size_t)p.P;
    s.r = s.bg ? i - (size_t)p.P : i;
    s.opacity_logits = (s.bg ? g.d_bg_opacity_logits : g.d_opacity_logits) + s.r;
    s.log_scales = (s.bg ? g.d_bg_log_scales : g.d_log_scales) + 3 * s.r;
    s.quats = (s.bg ? g.d_bg_quats : g.d_quats) + 4 * s.r;
    s.sh_dc = (s.bg ? g.d_bg_sh_dc : g.d_sh_dc) + 3 * s.r;
    s.sh_rest = (s.bg ? g.d_bg_sh_rest : g.d_sh_rest) + s.r * (size_t)p.sh_rest * 3;
    return s;
}

}  // namespace fb200
