// frosting_attr.cu -- Frosting's per-frame attribute construction, fused (SURVEY.md row a20).
//
// Replaces the chain of torch ops behind Frosting's properties
//   bary_coords  frosting_scene/frosting_model.py:713-719  softmax over the 6 prism-cell logits
//   points       :721-726   sum_k bary_k * shell_cells_verts[cell][k]   (inner v0..v2, outer v0..v2, :705-710)
//   strengths    :729-730   sigmoid
//   sh_coordinates :733-734 cat(dc[P,1,3], rest[P,M-1,3])
//   scaling      :765       exp
//   quaternions  :798       normalize
// (softmax, index, mul, sum, sigmoid, exp, normalize, cat and their ~10 backward kernels; the cat alone
// copies 192 B per Gaussian each way) by one forward and one backward kernel.  An optional occlusion mask
// skips the Gaussians the rasterizer will drop anyway.  Values are tolerance-level (torch's own softmax /
// normalize roundings are not part of the reference rasterizer's bit-exact contract): 1e-6 relative.
#include "common.cuh"
#include "frosting_attr.cuh"

namespace fb200 {

namespace {

struct AttrArgs {
    fb200_frosting_params p;
    float* means3D; float* opacities; float* scales; float* rotations; float* shs;
};

struct AttrBwdArgs {
    fb200_frosting_params p;
    const float* g_means3D; const float* g_opacities; const float* g_scales; const float* g_rotations; const float* g_shs;
    float* g_bary; float* g_inner; float* g_outer; float* g_opacity_logits; float* g_log_scales; float* g_quats;
    float* g_sh_dc; float* g_sh_rest;
};

constexpr int kAttrThreads = 128;
constexpr int kMaxRest = 15;                       // SH degree 3: 15 "rest" coefficients -> 45 floats per row

// The `rest` rows are 3*R floats (180 B for R = 15): only 4-byte aligned per row, but a warp's 32 rows are one
// contiguous, 16-byte aligned block.  Full warps therefore move the block with coalesced 128-bit accesses
// through shared memory (row stride 3R words is odd -> conflict-free scalar LDS/STS per lane); per-lane scalar
// accesses at a 180-byte stride cost 32 LSU wavefronts per instruction and dominated the first version.
__global__ void __launch_bounds__(kAttrThreads)
frosting_attr_fwd_kernel(AttrArgs a) {
    __shared__ __align__(16) float stage[kAttrThreads / 32][32 * 3 * kMaxRest];
    const unsigned full = 0xffffffffu;
    const int P = a.p.P, R = a.p.sh_rest;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g0 = idx - lane;
    const bool in_range = idx < P;
    const bool live = in_range && !(a.p.d_mask != nullptr && a.p.d_mask[idx] == 0) &&
                      !(a.p.d_face_visible != nullptr && a.p.d_face_visible[a.p.d_cells[idx]] == 0);
    const unsigned live_mask = __ballot_sync(full, live);
    if (live_mask == 0) return;
    // stage the warp's rest block when the warp is full and at least half of its rows are needed
    const bool staged = (g0 + 31 < P) && R > 0 && R <= kMaxRest && ((3 * R * 32) % 4 == 0) && __popc(live_mask) >= 16;
    float* srow = stage[warp];
    if (staged) {
        const float4* src = reinterpret_cast<const float4*>(a.p.d_sh_rest + (size_t)g0 * R * 3);
        float4* dst = reinterpret_cast<float4*>(srow);
        const int n4 = 3 * R * 32 / 4;
        for (int f = lane; f < n4; f += 32) dst[f] = __ldg(src + f);
        __syncwarp();
    }
    if (!live) return;
    const size_t i = (size_t)idx;
    // position
    float w[6], px, py, pz;
    int vid[3];
    frost_point(a.p, i, w, vid, px, py, pz);
    a.means3D[3 * i] = px; a.means3D[3 * i + 1] = py; a.means3D[3 * i + 2] = pz;
    // opacity, scale, rotation
    a.opacities[i] = frost_sigmoid(__ldg(a.p.d_opacity_logits + i));
#pragma unroll
    for (int k = 0; k < 3; ++k) a.scales[3 * i + k] = expf(__ldg(a.p.d_log_scales + 3 * i + k));
    float nrm;
    reinterpret_cast<float4*>(a.rotations)[i] = frost_normalize(__ldg(reinterpret_cast<const float4*>(a.p.d_quats) + i), nrm);
    // SH: dc | rest -> [M,3]
    float* sh = a.shs + i * (size_t)(R + 1) * 3;
    const float d0 = __ldg(a.p.d_sh_dc + 3 * i), d1 = __ldg(a.p.d_sh_dc + 3 * i + 1), d2 = __ldg(a.p.d_sh_dc + 3 * i + 2);
    if (R == kMaxRest) {
        // 48 output floats = twelve aligned 128-bit stores
        const float* rest = staged ? srow + lane * 45 : a.p.d_sh_rest + i * 45;
        float o[48];
        o[0] = d0; o[1] = d1; o[2] = d2;
#pragma unroll
        for (int k = 0; k < 45; ++k) o[3 + k] = staged ? rest[k] : __ldg(rest + k);
        float4* sh4 = reinterpret_cast<float4*>(sh);
#pragma unroll
        for (int q4 = 0; q4 < 12; ++q4) sh4[q4] = make_float4(o[4 * q4], o[4 * q4 + 1], o[4 * q4 + 2], o[4 * q4 + 3]);
    } else {
        sh[0] = d0; sh[1] = d1; sh[2] = d2;
        const float* rest = a.p.d_sh_rest + i * (size_t)R * 3;
        for (int k = 0; k < 3 * R; ++k) sh[3 + k] = staged ? srow[lane * 3 * R + k] : __ldg(rest + k);
    }
}

__global__ void __launch_bounds__(kAttrThreads)
frosting_attr_bwd_kernel(AttrBwdArgs a) {
    __shared__ __align__(16) float stage[kAttrThreads / 32][32 * 3 * kMaxRest];
    const unsigned full = 0xffffffffu;
    const int P = a.p.P, R = a.p.sh_rest;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g0 = idx - lane;
    const bool full_warp = g0 + 31 < P;
    const bool in_range = idx < P;
    // with d_radii the test is "was rendered": upstream rows of unrendered Gaussians are zero by definition and may be
    // unwritten (fb200_grads.sparse_rows), so they are not read
    const bool live = in_range && (a.p.d_radii != nullptr
        ? a.p.d_radii[idx] > 0
        : (!(a.p.d_mask != nullptr && a.p.d_mask[idx] == 0) &&
           !(a.p.d_face_visible != nullptr && a.p.d_face_visible[a.p.d_cells[idx]] == 0)));
    const unsigned live_mask = __ballot_sync(full, live);
    const size_t i = (size_t)(in_range ? idx : 0);
    float* srow = stage[warp];
    const bool vec_rest = full_warp && R > 0 && R <= kMaxRest && ((3 * R * 32) % 4 == 0);

    if (full_warp && live_mask == 0) {
        // every Gaussian of the warp is occluded: coalesced zero fill of all parameter gradients
        const size_t g = (size_t)g0;
        float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
        float4* p;
        p = reinterpret_cast<float4*>(a.g_bary + 6 * g);           for (int f = lane; f < 48; f += 32) p[f] = z4;
        p = reinterpret_cast<float4*>(a.g_opacity_logits + g);     if (lane < 8) p[lane] = z4;
        p = reinterpret_cast<float4*>(a.g_log_scales + 3 * g);     if (lane < 24) p[lane] = z4;
        p = reinterpret_cast<float4*>(a.g_quats + 4 * g);          p[lane] = z4;
        p = reinterpret_cast<float4*>(a.g_sh_dc + 3 * g);          if (lane < 24) p[lane] = z4;
        if (vec_rest) {
            p = reinterpret_cast<float4*>(a.g_sh_rest + (size_t)R * 3 * g);
            for (int f = lane; f < 3 * R * 8; f += 32) p[f] = z4;
        } else {
            for (int k = lane; k < 3 * R * 32; k += 32) a.g_sh_rest[(size_t)R * 3 * g + k] = 0.f;
        }
        return;
    }

    float gb[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    float g_op = 0.f, g_ls[3] = {0.f, 0.f, 0.f}, g_dc[3] = {0.f, 0.f, 0.f};
    float4 g_q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
        // position: d/dw_k = <g, vert_k>, softmax backward, vertices get w_k * g (scatter-add)
        float w[6], px, py, pz;
        int vid[3];
        frost_point(a.p, i, w, vid, px, py, pz);
        frost_point_backward(a.p, w, vid, a.g_means3D[3 * i], a.g_means3D[3 * i + 1], a.g_means3D[3 * i + 2],
                             a.g_inner, a.g_outer, gb);
        // sigmoid, exp
        const float sg = frost_sigmoid(__ldg(a.p.d_opacity_logits + i));
        g_op = a.g_opacities[i] * sg * (1.0f - sg);
#pragma unroll
        for (int k = 0; k < 3; ++k) g_ls[k] = a.g_scales[3 * i + k] * expf(__ldg(a.p.d_log_scales + 3 * i + k));
        float nrm;
        const float4 n = frost_normalize(__ldg(reinterpret_cast<const float4*>(a.p.d_quats) + i), nrm);
        g_q = frost_normalize_backward(n, nrm, reinterpret_cast<const float4*>(a.g_rotations)[i]);
    }
    // SH split: dc gradient to registers, rest gradient rows to the staging block (or straight to memory)
    const float* gsh = a.g_shs + i * (size_t)(R + 1) * 3;
    if (live && R == kMaxRest) {
        const float4* g4 = reinterpret_cast<const float4*>(gsh);
        float o[48];
#pragma unroll
        for (int q4 = 0; q4 < 12; ++q4) { const float4 t = g4[q4]; o[4 * q4] = t.x; o[4 * q4 + 1] = t.y; o[4 * q4 + 2] = t.z; o[4 * q4 + 3] = t.w; }
        g_dc[0] = o[0]; g_dc[1] = o[1]; g_dc[2] = o[2];
        float* dst = vec_rest ? srow + lane * 45 : a.g_sh_rest + i * 45;
#pragma unroll
        for (int k = 0; k < 45; ++k) dst[k] = o[3 + k];
    } else if (in_range) {
        if (live) { g_dc[0] = gsh[0]; g_dc[1] = gsh[1]; g_dc[2] = gsh[2]; }
        float* dst = vec_rest ? srow + lane * 3 * R : a.g_sh_rest + i * (size_t)R * 3;
        for (int k = 0; k < 3 * R; ++k) dst[k] = live ? gsh[3 + k] : 0.f;
    }
    if (vec_rest) {
        __syncwarp();
        const float4* src = reinterpret_cast<const float4*>(srow);
        float4* dst = reinterpret_cast<float4*>(a.g_sh_rest + (size_t)g0 * R * 3);
        const int n4 = 3 * R * 32 / 4;
        for (int f = lane; f < n4; f += 32) dst[f] = src[f];
    }
    if (!in_range) return;
#pragma unroll
    for (int k = 0; k < 6; ++k) a.g_bary[6 * i + k] = gb[k];
    a.g_opacity_logits[i] = g_op;
#pragma unroll
    for (int k = 0; k < 3; ++k) { a.g_log_scales[3 * i + k] = g_ls[k]; a.g_sh_dc[3 * i + k] = g_dc[k]; }
    reinterpret_cast<float4*>(a.g_quats)[i] = g_q;
}

// Background Gaussians (frosting_model.py:801-876): position as stored, then the same maps as a mesh row.  One thread per
// row with plain per-row accesses: this is the cross-check of frosting mode, not a hot path.  The output / upstream
// gradient pointers (and `radii`) start at the first background row, row p.P of the [P + n_bg, ...] tensors.
struct BgAttrBwdArgs {
    fb200_frosting_params p;
    const int32_t* radii;
    const float* g_means3D; const float* g_opacities; const float* g_scales; const float* g_rotations; const float* g_shs;
    fb200_frosting_grads g;
};

__global__ void __launch_bounds__(kAttrThreads)
frosting_bg_attr_fwd_kernel(AttrArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.p.n_bg) return;
    const size_t i = (size_t)idx;
    const int R = a.p.sh_rest;
#pragma unroll
    for (int k = 0; k < 3; ++k) a.means3D[3 * i + k] = __ldg(a.p.d_bg_points + 3 * i + k);
    a.opacities[i] = frost_sigmoid(__ldg(a.p.d_bg_opacity_logits + i));
#pragma unroll
    for (int k = 0; k < 3; ++k) a.scales[3 * i + k] = expf(__ldg(a.p.d_bg_log_scales + 3 * i + k));
    float nrm;
    reinterpret_cast<float4*>(a.rotations)[i] = frost_normalize(__ldg(reinterpret_cast<const float4*>(a.p.d_bg_quats) + i), nrm);
    // the output rows start at row P of a [P + n_bg, M, 3] tensor: 4-byte alignment only, scalar stores
    float* sh = a.shs + i * (size_t)(R + 1) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) sh[k] = __ldg(a.p.d_bg_sh_dc + 3 * i + k);
    const float* rest = a.p.d_bg_sh_rest + i * (size_t)R * 3;
    for (int k = 0; k < 3 * R; ++k) sh[3 + k] = __ldg(rest + k);
}

__global__ void __launch_bounds__(kAttrThreads)
frosting_bg_attr_bwd_kernel(BgAttrBwdArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= a.p.n_bg) return;
    const size_t i = (size_t)idx;
    const int R = a.p.sh_rest;
    // with radii: an unrendered row's upstream gradients are zero by definition and may be unwritten -- not read
    const bool live = a.radii == nullptr || a.radii[idx] > 0;
    float gp[3] = {0.f, 0.f, 0.f}, g_ls[3] = {0.f, 0.f, 0.f}, g_op = 0.f;
    float4 g_q = make_float4(0.f, 0.f, 0.f, 0.f);
    if (live) {
#pragma unroll
        for (int k = 0; k < 3; ++k) gp[k] = a.g_means3D[3 * i + k];
        const float sg = frost_sigmoid(__ldg(a.p.d_bg_opacity_logits + i));
        g_op = a.g_opacities[i] * sg * (1.0f - sg);
#pragma unroll
        for (int k = 0; k < 3; ++k) g_ls[k] = a.g_scales[3 * i + k] * expf(__ldg(a.p.d_bg_log_scales + 3 * i + k));
        float nrm;
        const float4 n = frost_normalize(__ldg(reinterpret_cast<const float4*>(a.p.d_bg_quats) + i), nrm);
        g_q = frost_normalize_backward(n, nrm, reinterpret_cast<const float4*>(a.g_rotations)[i]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) { a.g.d_bg_points[3 * i + k] = gp[k]; a.g.d_bg_log_scales[3 * i + k] = g_ls[k]; }
    a.g.d_bg_opacity_logits[i] = g_op;
    reinterpret_cast<float4*>(a.g.d_bg_quats)[i] = g_q;
    const float* gsh = a.g_shs + i * (size_t)(R + 1) * 3;
#pragma unroll
    for (int k = 0; k < 3; ++k) a.g.d_bg_sh_dc[3 * i + k] = live ? gsh[k] : 0.f;
    float* grest = a.g.d_bg_sh_rest + i * (size_t)R * 3;
    for (int k = 0; k < 3 * R; ++k) grest[k] = live ? gsh[3 + k] : 0.f;
}

}  // namespace

cudaError_t launch_frosting_attr_fwd(const fb200_frosting_params& p, float* means3D, float* opacities, float* scales,
                                     float* rotations, float* shs, cudaStream_t s) {
    AttrArgs a; a.p = p; a.means3D = means3D; a.opacities = opacities; a.scales = scales; a.rotations = rotations; a.shs = shs;
    if (p.P > 0) {
        frosting_attr_fwd_kernel<<<(p.P + kAttrThreads - 1) / kAttrThreads, kAttrThreads, 0, s>>>(a);
        count_launch();
    }
    if (p.n_bg > 0) {
        const size_t P = (size_t)p.P;
        a.means3D += 3 * P; a.opacities += P; a.scales += 3 * P; a.rotations += 4 * P; a.shs += P * (p.sh_rest + 1) * 3;
        frosting_bg_attr_fwd_kernel<<<(p.n_bg + kAttrThreads - 1) / kAttrThreads, kAttrThreads, 0, s>>>(a);
        count_launch();
    }
    return cudaGetLastError();
}

cudaError_t launch_frosting_attr_bwd(const fb200_frosting_params& p, const float* g_means3D, const float* g_opacities,
                                     const float* g_scales, const float* g_rotations, const float* g_shs,
                                     const fb200_frosting_grads& g, cudaStream_t s) {
    if (g.d_inner_verts != nullptr && p.n_verts > 0) {
        cudaError_t e = cudaMemsetAsync(g.d_inner_verts, 0, sizeof(float) * 3 * (size_t)p.n_verts, s);
        if (e != cudaSuccess) return e;
        e = cudaMemsetAsync(g.d_outer_verts, 0, sizeof(float) * 3 * (size_t)p.n_verts, s);
        if (e != cudaSuccess) return e;
    }
    if (p.P > 0) {
        AttrBwdArgs a; a.p = p;
        a.g_means3D = g_means3D; a.g_opacities = g_opacities; a.g_scales = g_scales; a.g_rotations = g_rotations; a.g_shs = g_shs;
        a.g_bary = g.d_bary_logits; a.g_inner = g.d_inner_verts; a.g_outer = g.d_outer_verts;
        a.g_opacity_logits = g.d_opacity_logits; a.g_log_scales = g.d_log_scales; a.g_quats = g.d_quats;
        a.g_sh_dc = g.d_sh_dc; a.g_sh_rest = g.d_sh_rest;
        frosting_attr_bwd_kernel<<<(p.P + kAttrThreads - 1) / kAttrThreads, kAttrThreads, 0, s>>>(a);
        count_launch();
    }
    if (p.n_bg > 0) {
        const size_t P = (size_t)p.P;
        BgAttrBwdArgs b; b.p = p; b.radii = p.d_radii != nullptr ? p.d_radii + P : nullptr;
        b.g_means3D = g_means3D + 3 * P; b.g_opacities = g_opacities + P; b.g_scales = g_scales + 3 * P;
        b.g_rotations = g_rotations + 4 * P; b.g_shs = g_shs + P * (p.sh_rest + 1) * 3; b.g = g;
        frosting_bg_attr_bwd_kernel<<<(p.n_bg + kAttrThreads - 1) / kAttrThreads, kAttrThreads, 0, s>>>(b);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace fb200
