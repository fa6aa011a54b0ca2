// loss.cu -- fused photometric loss  (1 - lambda) * L1 + lambda * (1 - SSIM), forward and backward.
//
// Replaces, for the loss every Frosting trainer applies to the rasterizer's output
// (frosting_trainers/refine.py:407-409, coarse_*.py), the torch implementation in
// frosting_utils/loss_utils.py:17-63: l1_loss = mean|x - y|; ssim = mean of the SSIM map built from five
// depthwise 11x11 Gaussian (sigma 1.5) convolutions with zero padding (mu1, mu2, E[x^2], E[y^2], E[xy]),
// C1 = 0.01^2, C2 = 0.03^2.  That is 5 convolutions + ~15 elementwise kernels forward and as many backward at
// 1080p; here: one forward kernel (separable convolution in shared memory, SSIM map, L1 term, per-block loss
// partials, three derivative maps), one tiny deterministic reduction, one backward kernel (separable
// convolution of the derivative maps + the L1 sign term).  Tolerance-level arithmetic (the reference convolves
// with the 2-D outer-product window; the separable form differs by float rounding): tests/test_loss_f64_gpu.py holds
// it to no worse than the reference's float32 arithmetic, both measured against float64.
#include "common.cuh"

namespace fb200 {

namespace {

constexpr int kLossTile = 16;
constexpr int kHalo = 5;
constexpr int kPadded = kLossTile + 2 * kHalo;   // 26

struct GaussW { float g[11]; };

__device__ __forceinline__ float img_at(const float* __restrict__ img, int H, int W, int y, int x) {
    return (x >= 0 && x < W && y >= 0 && y < H) ? __ldg(img + (size_t)y * W + x) : 0.0f;   // zero padding
}

__global__ void __launch_bounds__(kLossTile * kLossTile)
l1_dssim_fwd_kernel(const float* __restrict__ pred, const float* __restrict__ gt, int C, int H, int W, float lambda,
                    GaussW gw, float* __restrict__ maps /* [3,C,H,W] */, float* __restrict__ partials) {
    __shared__ float sx[kPadded][kPadded + 1], sy[kPadded][kPadded + 1];
    __shared__ float hz[5][kPadded][kLossTile + 1];
    __shared__ float red[kLossTile * kLossTile / 32];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kLossTile + tx;
    const int c = blockIdx.z;
    const int x0 = blockIdx.x * kLossTile, y0 = blockIdx.y * kLossTile;
    const float* p = pred + (size_t)c * H * W;
    const float* g = gt + (size_t)c * H * W;
    for (int i = tid; i < kPadded * kPadded; i += kLossTile * kLossTile) {
        const int r = i / kPadded, col = i % kPadded;
        sx[r][col] = img_at(p, H, W, y0 + r - kHalo, x0 + col - kHalo);
        sy[r][col] = img_at(g, H, W, y0 + r - kHalo, x0 + col - kHalo);
    }
    __syncthreads();
    // horizontal pass: rows 0..25, columns tx
    for (int r = ty; r < kPadded; r += kLossTile) {
        float a = 0.f, b = 0.f, aa = 0.f, bb = 0.f, ab = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float xv = sx[r][tx + k], yv = sy[r][tx + k], w = gw.g[k];
            a += w * xv; b += w * yv; aa += w * xv * xv; bb += w * yv * yv; ab += w * xv * yv;
        }
        hz[0][r][tx] = a; hz[1][r][tx] = b; hz[2][r][tx] = aa; hz[3][r][tx] = bb; hz[4][r][tx] = ab;
    }
    __syncthreads();
    float mu1 = 0.f, mu2 = 0.f, exx = 0.f, eyy = 0.f, exy = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
        const float w = gw.g[k];
        mu1 += w * hz[0][ty + k][tx]; mu2 += w * hz[1][ty + k][tx];
        exx += w * hz[2][ty + k][tx]; eyy += w * hz[3][ty + k][tx]; exy += w * hz[4][ty + k][tx];
    }
    const int x = x0 + tx, y = y0 + ty;
    float term = 0.f;
    if (x < W && y < H) {
        const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
        // Rounded products, as the reference's separate torch ops.  In flat regions sigma^2 = E[x^2] - mu^2 cancels
        // down to ~C2, and a contraction of s1 and s2 into FMAs but not s12 (mu12 is also needed for A) would make
        // B != D for identical images: SSIM off 1 by up to ulp(mu^2) / C2 ~ 7e-5 over a whole white background.
        const float mu1_sq = __fmul_rn(mu1, mu1), mu2_sq = __fmul_rn(mu2, mu2), mu12 = __fmul_rn(mu1, mu2);
        const float s1 = exx - mu1_sq, s2 = eyy - mu2_sq, s12 = exy - mu12;
        const float A = 2.f * mu12 + C1, B = 2.f * s12 + C2, Cc = mu1_sq + mu2_sq + C1, D = s1 + s2 + C2;
        const float inv = 1.0f / (Cc * D);
        // divided, as the reference does: identical windows give exactly 1 (A * B * inv can miss it by an ulp, a bias
        // that sums over every pixel where the prediction matches the ground truth)
        const float ssim = (A * B) / (Cc * D);
        // derivatives of the SSIM value w.r.t. mu1, E[x^2], E[xy] (E[.] held independent)
        const float dA = 2.f * mu2, dB = -2.f * mu2, dC = 2.f * mu1, dD = -2.f * mu1;
        const float d_mu1 = (dA * B + A * dB) * inv - ssim * (dC * D + Cc * dD) * inv;
        const float d_exx = -ssim / D;
        const float d_exy = 2.f * A * inv;
        const size_t o = ((size_t)c * H + y) * W + x, plane = (size_t)C * H * W;
        maps[o] = d_mu1; maps[plane + o] = d_exx; maps[2 * plane + o] = d_exy;
        const float xv = sx[ty + kHalo][tx + kHalo], yv = sy[ty + kHalo][tx + kHalo];
        term = (1.f - lambda) * fabsf(xv - yv) + lambda * (1.f - ssim);
    }
    // block sum -> one partial per block (fixed order => deterministic)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) term += __shfl_xor_sync(0xffffffffu, term, o);
    if ((tid & 31) == 0) red[tid >> 5] = term;
    __syncthreads();
    if (tid == 0) {
        float s = 0.f;
        for (int i = 0; i < kLossTile * kLossTile / 32; ++i) s += red[i];
        partials[((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(1024)
loss_reduce_kernel(const float* __restrict__ partials, int n, float scale, float* __restrict__ out) {
    __shared__ double sh[32];
    double s = 0.0;
    for (int i = threadIdx.x; i < n; i += 1024) s += (double)partials[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int i = 0; i < 32; ++i) t += sh[i];
        out[0] = (float)(t * (double)scale);
    }
}

__global__ void __launch_bounds__(kLossTile * kLossTile)
l1_dssim_bwd_kernel(const float* __restrict__ pred, const float* __restrict__ gt, const float* __restrict__ maps,
                    int C, int H, int W, float lambda, GaussW gw, const float* __restrict__ dL_dloss,
                    float* __restrict__ dpred) {
    __shared__ float sm[3][kPadded][kPadded + 1];
    __shared__ float hz[3][kPadded][kLossTile + 1];
    const int tx = threadIdx.x, ty = threadIdx.y, tid = ty * kLossTile + tx;
    const int c = blockIdx.z;
    const int x0 = blockIdx.x * kLossTile, y0 = blockIdx.y * kLossTile;
    const size_t plane = (size_t)C * H * W;
    for (int q = 0; q < 3; ++q) {
        const float* m = maps + q * plane + (size_t)c * H * W;
        for (int i = tid; i < kPadded * kPadded; i += kLossTile * kLossTile) {
            const int r = i / kPadded, col = i % kPadded;
            sm[q][r][col] = img_at(m, H, W, y0 + r - kHalo, x0 + col - kHalo);
        }
    }
    __syncthreads();
    for (int r = ty; r < kPadded; r += kLossTile) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
        for (int k = 0; k < 11; ++k) {
            const float w = gw.g[k];
            a0 += w * sm[0][r][tx + k]; a1 += w * sm[1][r][tx + k]; a2 += w * sm[2][r][tx + k];
        }
        hz[0][r][tx] = a0; hz[1][r][tx] = a1; hz[2][r][tx] = a2;
    }
    __syncthreads();
    float c0 = 0.f, c1 = 0.f, c2 = 0.f;
#pragma unroll
    for (int k = 0; k < 11; ++k) {
        const float w = gw.g[k];
        c0 += w * hz[0][ty + k][tx]; c1 += w * hz[1][ty + k][tx]; c2 += w * hz[2][ty + k][tx];
    }
    const int x = x0 + tx, y = y0 + ty;
    if (x < W && y < H) {
        const size_t o = ((size_t)c * H + y) * W + x;
        const float xv = __ldg(pred + o), yv = __ldg(gt + o);
        const float inv_n = 1.0f / (float)((double)C * H * W);
        const float d_ssim = c0 + 2.f * xv * c1 + yv * c2;           // d(sum of SSIM map)/dx
        const float diff = xv - yv;
        const float sgn = (diff > 0.f) ? 1.f : ((diff < 0.f) ? -1.f : 0.f);   // torch.abs backward: sign, 0 at 0
        dpred[o] = dL_dloss[0] * inv_n * ((1.f - lambda) * sgn - lambda * d_ssim);
    }
}

GaussW make_window() {
    // frosting_utils/loss_utils.py:23-25: float32 exp values, normalised in float32
    GaussW w;
    float v[11], s = 0.f;
    for (int i = 0; i < 11; ++i) { v[i] = (float)exp(-(double)((i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5)); s += v[i]; }
    for (int i = 0; i < 11; ++i) w.g[i] = v[i] / s;
    return w;
}

}  // namespace

size_t l1_dssim_num_partials(int C, int H, int W) {
    return (size_t)C * ((H + kLossTile - 1) / kLossTile) * ((W + kLossTile - 1) / kLossTile);
}

cudaError_t launch_l1_dssim_fwd(const float* pred, const float* gt, int C, int H, int W, float lambda, float* maps,
                                float* partials, float* loss, cudaStream_t s) {
    const dim3 grid((W + kLossTile - 1) / kLossTile, (H + kLossTile - 1) / kLossTile, C), block(kLossTile, kLossTile);
    l1_dssim_fwd_kernel<<<grid, block, 0, s>>>(pred, gt, C, H, W, lambda, make_window(), maps, partials);
    const int n = (int)l1_dssim_num_partials(C, H, W);
    loss_reduce_kernel<<<1, 1024, 0, s>>>(partials, n, 1.0f / (float)((double)C * H * W), loss);
    count_launch(2);
    return cudaGetLastError();
}

cudaError_t launch_l1_dssim_bwd(const float* pred, const float* gt, const float* maps, int C, int H, int W, float lambda,
                                const float* dL_dloss, float* dpred, cudaStream_t s) {
    const dim3 grid((W + kLossTile - 1) / kLossTile, (H + kLossTile - 1) / kLossTile, C), block(kLossTile, kLossTile);
    l1_dssim_bwd_kernel<<<grid, block, 0, s>>>(pred, gt, maps, C, H, W, lambda, make_window(), dL_dloss, dpred);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
