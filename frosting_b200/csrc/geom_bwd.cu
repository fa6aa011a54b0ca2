// geom_bwd.cu -- per-Gaussian backward: conic -> cov2D -> (cov3D, mean), projected mean -> mean,
// colour -> SH (+ view direction -> mean), cov3D -> scale / quaternion.
//
// One fused kernel replaces computeCov2DCUDA (DGR/cuda_rasterizer/backward.cu:144-274) and
// preprocessCUDA backward (backward.cu:346-396 with computeColorFromSH backward :20-139 and
// computeCov3D backward :278-341), and removes the nine zero-filled gradient tensors of
// DGR/rasterize_points.cu:151-159: every output element is written exactly once here (zeros for
// Gaussians with radii == 0), so the caller allocates with torch.empty.
//
// Gradients are tolerance-level quantities (the reference accumulates them with unordered float
// atomics), so this file is written in plain C++ from the maths, not from the reference's op order:
//   cov2D = M S M^T with M = J * W (2x3),  conic = cov2D^-1,
//   S = R^T diag(s)^2 R,  colour = clamp(sum_k b_k(dir) sh_k + 0.5).
// Quirks of the reference that ARE reproduced because they change the values:
//   * d(scale) omits the chain factor scale_modifier (backward.cu:318-321),
//   * the quaternion gradient is w.r.t. the un-normalised input (backward.cu:340),
//   * denom2inv = 1 / (det^2 + 1e-7) (backward.cu:203) and its == 0 guard,
//   * the 1.3*tanfov clamp masks on d/dt.x, d/dt.y (backward.cu:175-176).
#include "common.cuh"
#include "frosting_attr.cuh"

namespace fb200 {

namespace {

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }

// symmetric 3x3 times vector, S = (c0 c1 c2; c1 c3 c4; c2 c4 c5)
__device__ __forceinline__ V3 symv(const float* c, V3 t) {
    return v3(c[0] * t.x + c[1] * t.y + c[2] * t.z,
              c[1] * t.x + c[3] * t.y + c[4] * t.z,
              c[2] * t.x + c[4] * t.y + c[5] * t.z);
}

constexpr int kGeomThreads = 128;

// coalesced zero fill of `n4` float4 starting at a 16-byte aligned address, by one warp
__device__ __forceinline__ void warp_zero4(float* base, int n4, int lane) {
    float4* p = reinterpret_cast<float4*>(base);
    for (int i = lane; i < n4; i += 32) p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// all gradient rows of the 32 Gaussians starting at g: fully coalesced 128-bit zero stores
__device__ __forceinline__ void zero_warp_rows(const BwdArgs& a, size_t g, int M, int lane) {
    warp_zero4(a.g.d_dL_dmeans2D + 3 * g, 24, lane);
    if (a.g.d_dL_dcolors) warp_zero4(a.g.d_dL_dcolors + 3 * g, 24, lane);
    warp_zero4(a.g.d_dL_dopacity + g, 8, lane);
    warp_zero4(a.g.d_dL_dmeans3D + 3 * g, 24, lane);
    if (a.g.d_dL_dcov3D) warp_zero4(a.g.d_dL_dcov3D + 6 * g, 48, lane);
    if (a.g.d_dL_dscales) warp_zero4(a.g.d_dL_dscales + 3 * g, 24, lane);
    if (a.g.d_dL_drotations) warp_zero4(a.g.d_dL_drotations + 4 * g, 32, lane);
    if (a.g.d_dL_dsh != nullptr && M > 0 && ((M * 3) & 3) == 0) warp_zero4(a.g.d_dL_dsh + (size_t)M * 3 * g, M * 24, lane);
    else if (a.g.d_dL_dsh != nullptr && M > 0)
        for (int k = lane; k < M * 3 * 32; k += 32) a.g.d_dL_dsh[(size_t)M * 3 * g + k] = 0.f;
}

// ---- one row per lane <-> shared staging block, moved by the whole warp ----
// A lane reading ITS row straight from global memory (12 x 128-bit at a 192-byte stride, or 45 scalars at 180 bytes
// for Frosting's `rest` rows) costs 32 LSU wavefronts per instruction -- two to seven times the sectors the rows
// occupy -- and that, not arithmetic, bounded this kernel.  Here the warp walks the rows together: each instruction
// touches one or two rows contiguously (<= 12 sectors); the lanes then work on their rows in shared memory.  Every SH
// row -- M == 16, any other width, Frosting's dc | rest -- is staged in one layout: coefficient-major, RGB innermost, at
// most 48 floats, 13 float4 apart so that the lanes' per-row LDS.128 / STS.128 are conflict-free (the scalar movers
// write one row per instruction, lane = float: their banks do not depend on the stride).  `rows` <= 32 rows are live;
// lane r holds row r's pointer.
constexpr int kStageStride4 = 13;                    // float4 per staged row (12 used)
constexpr int kStageStride = 4 * kStageStride4;      // floats per staged row: 52

// The loads of a batch are all issued before the first one is consumed (a plain loop would pay one memory round trip
// per row: load -> store to shared -> next load).
__device__ __forceinline__ void warp_gather_rows4(const float* my_row, float4* stage4, int rows, int lane) {
    const int half = lane / 12, k4 = lane - 12 * half;          // lanes 0-11: row 2t, 12-23: row 2t+1, 24-31: idle
#pragma unroll
    for (int t0 = 0; t0 < 16; t0 += 8) {
        if (2 * t0 >= rows) break;
        float4 v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int r = 2 * (t0 + u) + half;
            const float4* p = reinterpret_cast<const float4*>(__shfl_sync(0xffffffffu, (unsigned long long)my_row, r & 31));
            v[u] = (half < 2 && r < rows) ? __ldg(p + k4) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int r = 2 * (t0 + u) + half;
            if (half < 2 && r < rows) stage4[r * kStageStride4 + k4] = v[u];
        }
    }
    __syncwarp();
}

__device__ __forceinline__ void warp_scatter_rows4(float* my_row, const float4* stage4, int rows, int lane) {
    __syncwarp();
    const int half = lane / 12, k4 = lane - 12 * half;
    for (int t = 0; t < (rows + 1) / 2; ++t) {
        const int r = 2 * t + half;
        float4* p = reinterpret_cast<float4*>(__shfl_sync(0xffffffffu, (unsigned long long)my_row, r & 31));
        if (half < 2 && r < rows) p[k4] = stage4[r * kStageStride4 + k4];
    }
    __syncwarp();
}

// 32 CONSECUTIVE rows of 12 float4 (the in-place walk): the block is one contiguous 6 KB span
__device__ __forceinline__ void warp_gather_block4(const float* block, float4* stage4, int lane) {
    const float4* src = reinterpret_cast<const float4*>(block);
    float4 v[12];
#pragma unroll
    for (int t = 0; t < 12; ++t) v[t] = __ldg(src + t * 32 + lane);
#pragma unroll
    for (int t = 0; t < 12; ++t) { const int f = t * 32 + lane; stage4[(f / 12) * kStageStride4 + (f % 12)] = v[t]; }
    __syncwarp();
}

__device__ __forceinline__ void warp_scatter_block4(float* block, const float4* stage4, int lane) {
    __syncwarp();
    float4* dst = reinterpret_cast<float4*>(block);
#pragma unroll
    for (int t = 0; t < 12; ++t) { const int f = t * 32 + lane; dst[f] = stage4[(f / 12) * kStageStride4 + (f % 12)]; }
    __syncwarp();
}

__device__ __forceinline__ void warp_gather_rows(const float* my_row, int nf, float* stage, int stride, int rows, int lane) {
    // nf <= 64 floats per row: two loads per lane and row, sixteen rows in flight
#pragma unroll
    for (int r0 = 0; r0 < 32; r0 += 16) {
        if (r0 >= rows) break;
        float v0[16], v1[16];
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const int r = r0 + u;
            const float* p = reinterpret_cast<const float*>(__shfl_sync(0xffffffffu, (unsigned long long)my_row, r));
            v0[u] = (r < rows && lane < nf) ? __ldg(p + lane) : 0.f;
            v1[u] = (r < rows && lane + 32 < nf) ? __ldg(p + lane + 32) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 16; ++u) {
            const int r = r0 + u;
            if (r < rows && lane < nf) stage[r * stride + lane] = v0[u];
            if (r < rows && lane + 32 < nf) stage[r * stride + lane + 32] = v1[u];
        }
    }
    __syncwarp();
}

// rows of nf floats of which the first n_staged are staged: the others go out as zeros
__device__ __forceinline__ void warp_scatter_rows(float* my_row, int nf, int n_staged, const float* stage, int stride,
                                                  int rows, int lane) {
    __syncwarp();
    for (int r = 0; r < rows; ++r) {
        float* p = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, (unsigned long long)my_row, r));
        for (int k = lane; k < nf; k += 32) p[k] = k < n_staged ? stage[r * stride + k] : 0.f;
    }
    __syncwarp();
}

// One kernel, two walks over the Gaussians (32 per warp and step):
//   kList  -- the RENDERED Gaussians only, over the list preprocess appended them to (vis_list, no particular order,
//             FB200_ST_NUM_VISIBLE entries): full warps whatever the visibility pattern; unrendered rows are never
//             touched.  The sparse-row contract and frosting mode: ~10 % of a Frosting layer is rendered per camera.
//   !kList -- in place over all P rows, for the reference's dense contract (zeros for unrendered rows): runs of 32
//             unrendered rows are zero-filled with coalesced 128-bit stores, the others computed with the unrendered lanes
//             writing zeros in the same store instructions.  (List walk + a separate zero-fill kernel was measured for
//             this contract too and lost where many rows are rendered (C5, C2): a list step costs one more dependent
//             memory round trip than an in-place step, which only pays off when most rows are skipped.)
// SH rows (192 B in, 192 B out per Gaussian) always travel through a per-warp staging block: see the movers above.
// kFrost (row f1): attributes are rebuilt from Frosting's parameters and the chain rule continues through
// frosting_attr.cuh to the PARAMETER gradients.
template <bool kFrost, bool kList>
__global__ void __launch_bounds__(kGeomThreads, 4)
geom_bwd_kernel(BwdArgs a) {
    __shared__ float view[16], proj[16], campos[3];
    __shared__ __align__(16) float stage_all[kGeomThreads / 32][32 * kStageStride];
    if (threadIdx.x < 16) {
        view[threadIdx.x] = a.in.d_viewmatrix[threadIdx.x];
        proj[threadIdx.x] = a.in.d_projmatrix[threadIdx.x];
    }
    if (threadIdx.x < 3) campos[threadIdx.x] = a.in.d_campos[threadIdx.x];
    __syncthreads();

    const unsigned full = 0xffffffffu;
    const int M = a.prm.sh_coeffs, D = a.prm.sh_degree;
    const fb200_frosting_params& fr = a.fr;
    const int n = kList ? a.status[FB200_ST_NUM_VISIBLE] : a.prm.P;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* const stage = stage_all[warp];
    float4* const stage4 = reinterpret_cast<float4*>(stage);
    constexpr int kWarps = kGeomThreads / 32;
    // a warp takes 32 consecutive entries at a time; the lanes behind the end shadow entry `jb` (valid memory, results
    // discarded) so that the cooperative row moves stay warp-uniform
    for (int jb = (blockIdx.x * kWarps + warp) * 32; jb < n; jb += gridDim.x * kWarps * 32) {
        const int rows = min(32, n - jb);
        const bool in_rows = lane < rows;
        int idx;
        bool active;             // this lane computes a gradient row
        if (kList) {
            idx = (int)a.vis_list[jb + (in_rows ? lane : 0)];
            active = in_rows;
        } else {
            idx = jb + (in_rows ? lane : 0);
            active = in_rows && a.radii[idx] > 0;
            if (rows == 32 && !__any_sync(full, active)) {
                // nothing rendered in this run (the common case under occlusion culling): zeros, coalesced.  The final,
                // shorter run goes through the compute path below, whose unrendered lanes store zeros.
                zero_warp_rows(a, (size_t)jb, M, lane);
                continue;
            }
        }
        const bool write = kList ? active : in_rows;      // this lane owns an output row (zeros if it computed none)
        const size_t i = (size_t)idx;
        // frosting mode: the row's parameters and gradient rows are the mesh rows or (idx >= fr.P) the d_bg_* rows of
        // the blocks; a warp may mix the two (the row movers below take one row pointer per lane).  The row pointers are
        // re-derived where they are used (frost_row: a select between kernel parameters) rather than kept live.
        const bool bg_row = kFrost && idx >= fr.P;

        float* dsh = (!kFrost && a.g.d_dL_dsh != nullptr && M > 0) ? a.g.d_dL_dsh + i * M * 3 : nullptr;
        const bool has_sh = kFrost || (a.in.d_shs != nullptr && M > 0 && dsh != nullptr);
        // the rows every lane reads for itself further down: start them moving now, beside the staged SH rows
        auto touch = [](const void* p) { asm volatile("prefetch.global.L1 [%0];" ::"l"(p)); };
        touch(a.acc + i * 12);
        if (kFrost) {
            const FrostRowT<const float> src = frost_row(fr, i);
            if (bg_row) touch(fr.d_bg_points + 3 * src.r);
            else { touch(fr.d_bary_logits + 6 * i); touch(fr.d_cells + i); }
            touch(src.log_scales); touch(src.quats); touch(src.opacity_logits);
        } else {
            touch(a.in.d_means3D + 3 * i);
            if (a.in.d_scales) { touch(a.in.d_scales + 3 * i); touch(a.in.d_rotations + 4 * i); }
        }
        if (kFrost) {
            // dc | rest rows into the staging block: [0..2] dc, [3..] rest
            const FrostRowT<const float> src = frost_row(fr, i);
            warp_gather_rows(src.sh_rest, fr.sh_rest * 3, stage + 3, kStageStride, rows, lane);
            stage[lane * kStageStride + 0] = __ldg(src.sh_dc);
            stage[lane * kStageStride + 1] = __ldg(src.sh_dc + 1);
            stage[lane * kStageStride + 2] = __ldg(src.sh_dc + 2);
        } else if (has_sh && M == 16) {
            if (!kList && rows == 32) warp_gather_block4(a.in.d_shs + (size_t)jb * 48, stage4, lane);
            else warp_gather_rows4(a.in.d_shs + i * 48, stage4, rows, lane);
        } else if (has_sh) {
            // coefficients beyond degree 3 (M > 16) are not read: their gradients are zero
            warp_gather_rows(a.in.d_shs + i * M * 3, min(3 * M, 48), stage, kStageStride, rows, lane);
        }

        float g_mean2d_x, g_mean2d_y, g_op;
        V3 g_col, g_mean;
        float g_cov[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        V3 g_scale = v3(0.f, 0.f, 0.f);
        float4 g_rot = make_float4(0.f, 0.f, 0.f, 0.f);

        const float4* accp = reinterpret_cast<const float4*>(a.acc + i * 12);
        const float4 a0 = accp[0], a1 = accp[1];
        const float a2x = a.acc[i * 12 + 8];
        g_mean2d_x = a0.x; g_mean2d_y = a0.y;
        const float dLc_x = a0.z, dLc_y = a0.w, dLc_w = a1.x;   // dL/dconic (x, y, w)
        g_op = a1.y;
        g_col = v3(a1.z, a1.w, a2x);

        // frosting mode: position, scale, rotation from the parameters (bit-identical to the forward's)
        float fw[6], q_nrm = 1.f, raw_s[3] = {0.f, 0.f, 0.f};
        int fvid[3];
        float mx, my, mz;
        if (bg_row) {
            const float* pt = fr.d_bg_points + 3 * (i - (size_t)fr.P);
            mx = __ldg(pt); my = __ldg(pt + 1); mz = __ldg(pt + 2);
        } else if (kFrost) {
            frost_point(fr, i, fw, fvid, mx, my, mz);
        } else { mx = a.in.d_means3D[3 * i]; my = a.in.d_means3D[3 * i + 1]; mz = a.in.d_means3D[3 * i + 2]; }

        // ---- 3D covariance (recomputed from scale/rotation, or the precomputed input) ----
        float S[6];
        float sx = 0.f, sy = 0.f, sz = 0.f, qr = 0.f, qx = 0.f, qy = 0.f, qz = 0.f;
        float Rm[3][3];   // Rm[row][col], maths convention: Sigma = Rm^T diag(s)^2 Rm
        const bool from_sr = kFrost || a.in.d_cov3D_precomp == nullptr;
        if (from_sr) {
            const float mod = a.prm.scale_modifier;
            float4 q;
            if (kFrost) {
                const FrostRowT<const float> src = frost_row(fr, i);
#pragma unroll
                for (int k = 0; k < 3; ++k) raw_s[k] = expf(__ldg(src.log_scales + k));
                q = frost_normalize(__ldg(reinterpret_cast<const float4*>(src.quats)), q_nrm);
            } else {
                raw_s[0] = a.in.d_scales[3 * i]; raw_s[1] = a.in.d_scales[3 * i + 1]; raw_s[2] = a.in.d_scales[3 * i + 2];
                q = reinterpret_cast<const float4*>(a.in.d_rotations)[i];
            }
            sx = mod * raw_s[0]; sy = mod * raw_s[1]; sz = mod * raw_s[2];
            qr = q.x; qx = q.y; qy = q.z; qz = q.w;
            Rm[0][0] = 1.f - 2.f * (qy * qy + qz * qz); Rm[0][1] = 2.f * (qx * qy + qr * qz); Rm[0][2] = 2.f * (qx * qz - qr * qy);
            Rm[1][0] = 2.f * (qx * qy - qr * qz); Rm[1][1] = 1.f - 2.f * (qx * qx + qz * qz); Rm[1][2] = 2.f * (qy * qz + qr * qx);
            Rm[2][0] = 2.f * (qx * qz + qr * qy); Rm[2][1] = 2.f * (qy * qz - qr * qx); Rm[2][2] = 1.f - 2.f * (qx * qx + qy * qy);
            const float s2[3] = {sx * sx, sy * sy, sz * sz};
            int k = 0;
            for (int r = 0; r < 3; ++r)
                for (int c = r; c < 3; ++c, ++k)
                    S[k] = s2[0] * Rm[0][r] * Rm[0][c] + s2[1] * Rm[1][r] * Rm[1][c] + s2[2] * Rm[2][r] * Rm[2][c];
        } else {
            for (int k = 0; k < 6; ++k) S[k] = a.in.d_cov3D_precomp[6 * i + k];
        }

        // ---- conic -> cov2D -> cov3D and view-space mean ----
        const float tx_raw = view[0] * mx + view[4] * my + view[8] * mz + view[12];
        const float ty_raw = view[1] * mx + view[5] * my + view[9] * mz + view[13];
        const float tz = view[2] * mx + view[6] * my + view[10] * mz + view[14];
        const float limx = 1.3f * a.prm.tanfovx, limy = 1.3f * a.prm.tanfovy;
        const float txtz = tx_raw / tz, tytz = ty_raw / tz;
        const float tx = fminf(limx, fmaxf(-limx, txtz)) * tz;
        const float ty = fminf(limy, fmaxf(-limy, tytz)) * tz;
        const float x_grad_mul = (txtz < -limx || txtz > limx) ? 0.f : 1.f;
        const float y_grad_mul = (tytz < -limy || tytz > limy) ? 0.f : 1.f;
        const float fx = a.focal_x, fy = a.focal_y;
        const float J00 = fx / tz, J02 = -(fx * tx) / (tz * tz), J11 = fy / tz, J12 = -(fy * ty) / (tz * tz);
        // rows of M = J * W, W[i][j] = view[4*j + i]
        const V3 T0 = v3(J00 * view[0] + J02 * view[2], J00 * view[4] + J02 * view[6], J00 * view[8] + J02 * view[10]);
        const V3 T1 = v3(J11 * view[1] + J12 * view[2], J11 * view[5] + J12 * view[6], J11 * view[9] + J12 * view[10]);
        const V3 ST0 = symv(S, T0), ST1 = symv(S, T1);
        const float ca = dot(T0, ST0) + 0.3f, cb = dot(T0, ST1), cc = dot(T1, ST1) + 0.3f;
        const float denom = ca * cc - cb * cb;
        const float denom2inv = 1.0f / (denom * denom + 0.0000001f);
        float dL_da = 0.f, dL_db = 0.f, dL_dc = 0.f;
        if (denom2inv != 0.f) {
            dL_da = denom2inv * (-cc * cc * dLc_x + 2.f * cb * cc * dLc_y + (denom - ca * cc) * dLc_w);
            dL_dc = denom2inv * (-ca * ca * dLc_w + 2.f * ca * cb * dLc_y + (denom - ca * cc) * dLc_x);
            dL_db = denom2inv * 2.f * (cb * cc * dLc_x - (denom + 2.f * cb * cb) * dLc_y + ca * cb * dLc_w);
            // d cov2D / d Sigma (off-diagonals appear twice)
            g_cov[0] = T0.x * T0.x * dL_da + T0.x * T1.x * dL_db + T1.x * T1.x * dL_dc;
            g_cov[3] = T0.y * T0.y * dL_da + T0.y * T1.y * dL_db + T1.y * T1.y * dL_dc;
            g_cov[5] = T0.z * T0.z * dL_da + T0.z * T1.z * dL_db + T1.z * T1.z * dL_dc;
            g_cov[1] = 2.f * T0.x * T0.y * dL_da + (T0.x * T1.y + T0.y * T1.x) * dL_db + 2.f * T1.x * T1.y * dL_dc;
            g_cov[2] = 2.f * T0.x * T0.z * dL_da + (T0.x * T1.z + T0.z * T1.x) * dL_db + 2.f * T1.x * T1.z * dL_dc;
            g_cov[4] = 2.f * T0.z * T0.y * dL_da + (T0.y * T1.z + T0.z * T1.y) * dL_db + 2.f * T1.y * T1.z * dL_dc;
        }
        // d/dT rows, then d/dJ, then d/dt
        const V3 dT0 = v3(2.f * ST0.x * dL_da + ST1.x * dL_db, 2.f * ST0.y * dL_da + ST1.y * dL_db, 2.f * ST0.z * dL_da + ST1.z * dL_db);
        const V3 dT1 = v3(2.f * ST1.x * dL_dc + ST0.x * dL_db, 2.f * ST1.y * dL_dc + ST0.y * dL_db, 2.f * ST1.z * dL_dc + ST0.z * dL_db);
        const float dJ00 = view[0] * dT0.x + view[4] * dT0.y + view[8] * dT0.z;
        const float dJ02 = view[2] * dT0.x + view[6] * dT0.y + view[10] * dT0.z;
        const float dJ11 = view[1] * dT1.x + view[5] * dT1.y + view[9] * dT1.z;
        const float dJ12 = view[2] * dT1.x + view[6] * dT1.y + view[10] * dT1.z;
        const float itz = 1.f / tz, itz2 = itz * itz, itz3 = itz2 * itz;
        const float dtx = x_grad_mul * -fx * itz2 * dJ02;
        const float dty = y_grad_mul * -fy * itz2 * dJ12;
        const float dtz = -fx * itz2 * dJ00 - fy * itz2 * dJ11 + (2.f * fx * tx) * itz3 * dJ02 + (2.f * fy * ty) * itz3 * dJ12;
        g_mean = v3(view[0] * dtx + view[1] * dty + view[2] * dtz,
                    view[4] * dtx + view[5] * dty + view[6] * dtz,
                    view[8] * dtx + view[9] * dty + view[10] * dtz);

        // ---- projected mean -> mean ----
        {
            const float hx = proj[0] * mx + proj[4] * my + proj[8] * mz + proj[12];
            const float hy = proj[1] * mx + proj[5] * my + proj[9] * mz + proj[13];
            const float hw = proj[3] * mx + proj[7] * my + proj[11] * mz + proj[15];
            const float m_w = 1.0f / (hw + 0.0000001f);
            const float mul1 = hx * m_w * m_w, mul2 = hy * m_w * m_w;
            g_mean.x += (proj[0] * m_w - proj[3] * mul1) * g_mean2d_x + (proj[1] * m_w - proj[3] * mul2) * g_mean2d_y;
            g_mean.y += (proj[4] * m_w - proj[7] * mul1) * g_mean2d_x + (proj[5] * m_w - proj[7] * mul2) * g_mean2d_y;
            g_mean.z += (proj[8] * m_w - proj[11] * mul1) * g_mean2d_x + (proj[9] * m_w - proj[11] * mul2) * g_mean2d_y;
        }

        // ---- colour -> SH coefficients and view direction ----
        if (has_sh) {
            const uint8_t cl = a.clamped[idx];
            const V3 dRGB = v3((cl & 1) ? 0.f : g_col.x, (cl & 2) ? 0.f : g_col.y, (cl & 4) ? 0.f : g_col.z);
            const V3 dorig = v3(mx - campos[0], my - campos[1], mz - campos[2]);
            const float len = sqrtf(dot(dorig, dorig));
            const float x = dorig.x / len, y = dorig.y / len, z = dorig.z / len;
            // basis value and gradient per coefficient
            float bv[16], bx[16], by[16], bz[16];
#pragma unroll
            for (int k = 0; k < 16; ++k) { bv[k] = 0.f; bx[k] = 0.f; by[k] = 0.f; bz[k] = 0.f; }
            bv[0] = kC0;
            if (D > 0) {
                bv[1] = -kC1 * y; by[1] = -kC1;
                bv[2] = kC1 * z;  bz[2] = kC1;
                bv[3] = -kC1 * x; bx[3] = -kC1;
                if (D > 1) {
                    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                    bv[4] = kC2_0 * xy;                 bx[4] = kC2_0 * y;        by[4] = kC2_0 * x;
                    bv[5] = kC2_1 * yz;                 by[5] = kC2_1 * z;        bz[5] = kC2_1 * y;
                    bv[6] = kC2_2 * (2.f * zz - xx - yy); bx[6] = kC2_2 * 2.f * -x; by[6] = kC2_2 * 2.f * -y; bz[6] = kC2_2 * 4.f * z;
                    bv[7] = kC2_3 * xz;                 bx[7] = kC2_3 * z;        bz[7] = kC2_3 * x;
                    bv[8] = kC2_4 * (xx - yy);          bx[8] = kC2_4 * 2.f * x;  by[8] = kC2_4 * 2.f * -y;
                    if (D > 2) {
                        bv[9] = kC3_0 * y * (3.f * xx - yy);            bx[9] = kC3_0 * 6.f * xy;  by[9] = kC3_0 * 3.f * (xx - yy);
                        bv[10] = kC3_1 * xy * z;                        bx[10] = kC3_1 * yz;      by[10] = kC3_1 * xz;   bz[10] = kC3_1 * xy;
                        bv[11] = kC3_2 * y * (4.f * zz - xx - yy);      bx[11] = kC3_2 * -2.f * xy; by[11] = kC3_2 * (-3.f * yy + 4.f * zz - xx); bz[11] = kC3_2 * 8.f * yz;
                        bv[12] = kC3_3 * z * (2.f * zz - 3.f * xx - 3.f * yy); bx[12] = kC3_3 * -6.f * xz; by[12] = kC3_3 * -6.f * yz; bz[12] = kC3_3 * 3.f * (2.f * zz - xx - yy);
                        bv[13] = kC3_4 * x * (4.f * zz - xx - yy);      bx[13] = kC3_4 * (-3.f * xx + 4.f * zz - yy); by[13] = kC3_4 * -2.f * xy; bz[13] = kC3_4 * 8.f * xz;
                        bv[14] = kC3_5 * z * (xx - yy);                 bx[14] = kC3_5 * 2.f * xz; by[14] = kC3_5 * -2.f * yz; bz[14] = kC3_5 * (xx - yy);
                        bv[15] = kC3_6 * x * (xx - 3.f * yy);           bx[15] = kC3_6 * 3.f * (xx - yy); by[15] = kC3_6 * -6.f * xy;
                    }
                }
            }
            const int ncoef = (D + 1) * (D + 1);
            const float dR[3] = {dRGB.x, dRGB.y, dRGB.z};
            float ax[3] = {0.f, 0.f, 0.f}, ay[3] = {0.f, 0.f, 0.f}, az[3] = {0.f, 0.f, 0.f};
            // the staged row's values; their gradients overwrite them there (zeros past the degree's coefficients)
            float4* srow4 = stage4 + lane * kStageStride4;
#pragma unroll
            for (int q = 0; q < 12; ++q) {
                float o[4] = {0.f, 0.f, 0.f, 0.f};
                if (4 * q < 3 * ncoef) {
                    const float4 s4 = srow4[q];
                    const float sv[4] = {s4.x, s4.y, s4.z, s4.w};
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const int k = (4 * q + e) / 3, c = (4 * q + e) % 3;
                        if (k < ncoef) {
                            o[e] = bv[k] * dR[c];
                            ax[c] += bx[k] * sv[e]; ay[c] += by[k] * sv[e]; az[c] += bz[k] * sv[e];
                        }
                    }
                }
                srow4[q] = make_float4(o[0], o[1], o[2], o[3]);
            }
            const V3 dcdx = v3(ax[0], ax[1], ax[2]), dcdy = v3(ay[0], ay[1], ay[2]), dcdz = v3(az[0], az[1], az[2]);
            // through dir = dorig / |dorig|:  d/dv = (dv |v|^2 - v (v . dv)) / |v|^3
            const V3 ddir = v3(dot(dcdx, dRGB), dot(dcdy, dRGB), dot(dcdz, dRGB));
            const float sum2 = dot(dorig, dorig);
            const float inv32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
            const float vd = dot(dorig, ddir);
            g_mean.x += (ddir.x * sum2 - dorig.x * vd) * inv32;
            g_mean.y += (ddir.y * sum2 - dorig.y * vd) * inv32;
            g_mean.z += (ddir.z * sum2 - dorig.z * vd) * inv32;
        } else if (dsh != nullptr && write) {
            for (int k = 0; k < M * 3; ++k) dsh[k] = 0.f;
        }
        // SH gradient rows back to memory, by the whole warp (has_sh and M are warp-uniform)
        if (!kList && has_sh && !active) {
            // in-place walk: an unrendered lane's staged row holds whatever the garbage inputs produced: zeros go out
#pragma unroll
            for (int q = 0; q < 12; ++q) stage4[lane * kStageStride4 + q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (kFrost) {
            const int nf = fr.sh_rest * 3;
            const FrostRowT<float> dst = frost_grad_row(fr, a.fg, i);
            warp_scatter_rows(dst.sh_rest, nf, nf, stage + 3, kStageStride, rows, lane);
            if (active) {
                dst.sh_dc[0] = stage[lane * kStageStride]; dst.sh_dc[1] = stage[lane * kStageStride + 1];
                dst.sh_dc[2] = stage[lane * kStageStride + 2];
            }
            __syncwarp();
        } else if (has_sh && M == 16) {
            if (!kList && rows == 32) warp_scatter_block4(a.g.d_dL_dsh + (size_t)jb * 48, stage4, lane);
            else warp_scatter_rows4(dsh, stage4, rows, lane);
        } else if (has_sh) {
            warp_scatter_rows(dsh, 3 * M, 48, stage, kStageStride, rows, lane);
        }
        if (!write) continue;

        // ---- cov3D -> scale, quaternion ----
        if (from_sr) {
            // dL/dSigma as a symmetric matrix (off-diagonals halved), dL/dMm = 2 * Mm * dL/dSigma,
            // Mm[r][c] = s_r * Rm[r][c]
            const float dS[3][3] = {{g_cov[0], 0.5f * g_cov[1], 0.5f * g_cov[2]},
                                    {0.5f * g_cov[1], g_cov[3], 0.5f * g_cov[4]},
                                    {0.5f * g_cov[2], 0.5f * g_cov[4], g_cov[5]}};
            const float sv[3] = {sx, sy, sz};
            float Gm[3][3];   // dL/dRm[r][c] = s_r * dL/dMm[r][c]
            float gs[3];
            for (int r = 0; r < 3; ++r) {
                float acc_s = 0.f;
                for (int c = 0; c < 3; ++c) {
                    const float dMm = 2.f * sv[r] * (Rm[r][0] * dS[0][c] + Rm[r][1] * dS[1][c] + Rm[r][2] * dS[2][c]);
                    acc_s += Rm[r][c] * dMm;
                    Gm[r][c] = sv[r] * dMm;
                }
                gs[r] = acc_s;
            }
            g_scale = v3(gs[0], gs[1], gs[2]);
            // Hm[a][b] = dL/dRm[a][b]; the four sums below are dRm/dq contracted with it.
            const float (&Hm)[3][3] = Gm;
            g_rot.x = 2.f * qz * (Hm[0][1] - Hm[1][0]) + 2.f * qy * (Hm[2][0] - Hm[0][2]) + 2.f * qx * (Hm[1][2] - Hm[2][1]);
            g_rot.y = 2.f * qy * (Hm[1][0] + Hm[0][1]) + 2.f * qz * (Hm[2][0] + Hm[0][2]) + 2.f * qr * (Hm[1][2] - Hm[2][1]) - 4.f * qx * (Hm[2][2] + Hm[1][1]);
            g_rot.z = 2.f * qx * (Hm[1][0] + Hm[0][1]) + 2.f * qr * (Hm[2][0] - Hm[0][2]) + 2.f * qz * (Hm[1][2] + Hm[2][1]) - 4.f * qy * (Hm[2][2] + Hm[0][0]);
            g_rot.w = 2.f * qr * (Hm[0][1] - Hm[1][0]) + 2.f * qx * (Hm[2][0] + Hm[0][2]) + 2.f * qy * (Hm[1][2] + Hm[2][1]) - 4.f * qz * (Hm[1][1] + Hm[0][0]);
        }

        if (!kList && !active) {
            // in-place walk, unrendered row inside a run that has rendered ones: whatever its garbage inputs produced is
            // dropped, zeros go out through the same stores
            g_mean2d_x = 0.f; g_mean2d_y = 0.f; g_op = 0.f;
            g_col = v3(0.f, 0.f, 0.f); g_mean = v3(0.f, 0.f, 0.f); g_scale = v3(0.f, 0.f, 0.f);
            g_rot = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int k = 0; k < 6; ++k) g_cov[k] = 0.f;
        }
        if (a.g.d_dL_dmeans2D) {
            a.g.d_dL_dmeans2D[3 * i] = g_mean2d_x; a.g.d_dL_dmeans2D[3 * i + 1] = g_mean2d_y; a.g.d_dL_dmeans2D[3 * i + 2] = 0.f;
        }
        if (kFrost) {
            // the chain rule through the attribute maps (fb200_frosting_attributes_backward, same formulas)
            const FrostRowT<const float> src = frost_row(fr, i);
            const FrostRowT<float> dst = frost_grad_row(fr, a.fg, i);
            if (bg_row) {
                // a background position is a parameter itself: dL/dbg_points = dL/dmean3D
                float* gp = a.fg.d_bg_points + 3 * src.r;
                gp[0] = g_mean.x; gp[1] = g_mean.y; gp[2] = g_mean.z;
            } else {
                float gb[6];
                frost_point_backward(fr, fw, fvid, g_mean.x, g_mean.y, g_mean.z, a.fg.d_inner_verts, a.fg.d_outer_verts, gb);
                float2* gb2 = reinterpret_cast<float2*>(a.fg.d_bary_logits + 6 * i);
                gb2[0] = make_float2(gb[0], gb[1]); gb2[1] = make_float2(gb[2], gb[3]); gb2[2] = make_float2(gb[4], gb[5]);
            }
            const float sg = frost_sigmoid(__ldg(src.opacity_logits));
            dst.opacity_logits[0] = g_op * sg * (1.0f - sg);
            dst.log_scales[0] = g_scale.x * raw_s[0];
            dst.log_scales[1] = g_scale.y * raw_s[1];
            dst.log_scales[2] = g_scale.z * raw_s[2];
            *reinterpret_cast<float4*>(dst.quats) = frost_normalize_backward(make_float4(qr, qx, qy, qz), q_nrm, g_rot);
        } else {
            if (a.g.d_dL_dcolors) { a.g.d_dL_dcolors[3 * i] = g_col.x; a.g.d_dL_dcolors[3 * i + 1] = g_col.y; a.g.d_dL_dcolors[3 * i + 2] = g_col.z; }
            a.g.d_dL_dopacity[i] = g_op;
            a.g.d_dL_dmeans3D[3 * i] = g_mean.x; a.g.d_dL_dmeans3D[3 * i + 1] = g_mean.y; a.g.d_dL_dmeans3D[3 * i + 2] = g_mean.z;
            if (a.g.d_dL_dcov3D)
                for (int k = 0; k < 6; ++k) a.g.d_dL_dcov3D[6 * i + k] = g_cov[k];
            if (a.g.d_dL_dscales) { a.g.d_dL_dscales[3 * i] = g_scale.x; a.g.d_dL_dscales[3 * i + 1] = g_scale.y; a.g.d_dL_dscales[3 * i + 2] = g_scale.z; }
            if (a.g.d_dL_drotations) reinterpret_cast<float4*>(a.g.d_dL_drotations)[i] = g_rot;
        }
    }
}

}  // namespace

cudaError_t launch_geom_bwd(const BwdArgs& a, cudaStream_t s) {
    if (a.prm.P > 0) {
        // grid-stride, four resident CTAs per SM (the visible list's length is known to the device only)
        const int want = (a.prm.P + kGeomThreads - 1) / kGeomThreads;
        const int cap = sm_count() * 4;
        const int blocks = want < cap ? want : cap;
        if (a.frosting) {
            if (a.fg.d_inner_verts != nullptr && a.fr.n_verts > 0) {
                cudaError_t e = cudaMemsetAsync(a.fg.d_inner_verts, 0, sizeof(float) * 3 * (size_t)a.fr.n_verts, s);
                if (e != cudaSuccess) return e;
                e = cudaMemsetAsync(a.fg.d_outer_verts, 0, sizeof(float) * 3 * (size_t)a.fr.n_verts, s);
                if (e != cudaSuccess) return e;
            }
            geom_bwd_kernel<true, true><<<blocks, kGeomThreads, 0, s>>>(a);
        } else if (a.g.sparse_rows) {
            geom_bwd_kernel<false, true><<<blocks, kGeomThreads, 0, s>>>(a);
        } else {
            geom_bwd_kernel<false, false><<<blocks, kGeomThreads, 0, s>>>(a);
        }
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace fb200
