// sugar_reg.cu -- SuGaR's SDF regulariser of the coarse stage (density-mode estimation term + "better normal" term),
// forward and backward, over a neighbour table that is an input (SURVEY.md row a23).
//
// Replaces, for the default trainer settings (`sdf_estimation_mode = 'density'`, `beta_mode = 'average'`,
// `sdf_better_normal_gradient_through_normal_only = True`), frosting_trainers/coarse_density_and_dn_consistency.py:745-833
// with frosting_scene/sugar_model.py:755-761 (get_covariance), :961-975 (get_smallest_axis), :1223-1226 (get_beta) and
// :1278-1347 (get_field_values): about a hundred torch kernels over [N,K,3,3] gathers, and index-put scatters backward.
// Here no N x K tensor exists:
//   1. sugar_record_kernel (P threads): per Gaussian j one 80-byte record {mu, sigma}, A = R(q) diag(1/clamp(s, 1e-8)),
//      {min s, nrm = the column of R at argmin s}, so that a neighbour costs one gathered record.
//   2. sugar_sample_kernel<G, grad> (G lanes per sample, one neighbour per lane, G = the power of two >= K): the
//      sample x = mu_i + q_i (f s_i * eps) q_i^-1, the field, beta, both terms per sample, shuffle reductions, and one
//      partial pair per block.  With `grad` the same pass also differentiates both terms at unit upstream (they are
//      linear in their upstream scalars) into a [P,32] float accumulator per Gaussian, with sm_90 vector reductions
//      (red.global.add.v4.f32): five per (sample, neighbour) pair and five per sample for the owner.  Small scenes get
//      R = 2^18 / P (a power of two, at most 1024) replicas of the accumulators, sample n adding into replica n % R:
//      at P = 17 and a million samples a float32 sum would otherwise take ~10^6 terms per address, and its rounding
//      exceeds the reference's own by 60x.
//   3. sugar_terms_kernel: the two means from the partials, in double, in a fixed order (deterministic).
//   4. sugar_chain_kernel (P threads, the backward): the replicas summed in double, x upstream -> d(points, scaling, quaternions,
//      strengths), through 1/clamp(s), argmin s and pytorch3d's quaternion_to_matrix (two_s = 2/|q|^2 kept, so the
//      radial parts autograd gives at the op's raw quaternions are kept too).
// The gradients are autograd's of the reference's expressions: |0| and sign(0) give 0, clamp passes its bounds
// inclusively, min / argmin route to the first minimal axis.  Accumulation order of the atomics is not fixed, so the
// gradients are reproducible to float rounding only; the two terms are bit-reproducible.
#include "common.cuh"
#include "sugar_common.cuh"

namespace fb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kRec = 5;       // float4 per Gaussian record
constexpr int kAcc = 8;       // float4 per Gaussian accumulator

// accumulator slots (float4 each): what a (sample, neighbour) pair adds to the neighbour j, what a sample adds to its
// owner i.  "e": estimation term, "n": normal term; the chain pass scales them by their own upstream.
enum : int {
    kAccMuSigma = 0,    // e: dmu.xyz, dsigma           (pair: -dshift, dsigma; owner: sum of dshift)
    kAccA0 = 1,         // e: dA[0..3]                  (pair)
    kAccA1 = 2,         // e: dA[4..7]                  (pair)
    kAccA2 = 3,         // e: dA[8], dmin_s, -, -       (pair)
    kAccNrmN = 4,       // n: dnrm.xyz, -               (pair: -w_k sign_k dr; owner: dr)
    kAccNrmE = 5,       // e: dnrm.xyz, -               (owner: dsdf * v)
    kAccQuat = 6,       // e: dq (w, x, y, z)           (owner, through the sample's rotation)
    kAccScale = 7,      // e: ds.xyz, -                 (owner, through the sample's scale)
};

__global__ void __launch_bounds__(kThreads)
sugar_record_kernel(int P, const float* __restrict__ points, const float* __restrict__ scaling,
                    const float4* __restrict__ quats, const float* __restrict__ strengths, float4* __restrict__ rec) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= P) return;
    const float4 q = __ldg(quats + p);
    float R[9];
    quat_to_matrix(q.x, q.y, q.z, q.w, R);
    const size_t p3 = (size_t)3 * p;
    const float s[3] = {__ldg(scaling + p3), __ldg(scaling + p3 + 1), __ldg(scaling + p3 + 2)};
    const float inv[3] = {1.f / fmaxf(s[0], 1e-8f), 1.f / fmaxf(s[1], 1e-8f), 1.f / fmaxf(s[2], 1e-8f)};
    const int c = argmin3(s[0], s[1], s[2]);
    float A[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) A[e] = R[e] * inv[e % 3];
    float4* o = rec + (size_t)kRec * p;
    o[0] = make_float4(__ldg(points + p3), __ldg(points + p3 + 1), __ldg(points + p3 + 2), __ldg(strengths + p));
    o[1] = make_float4(A[0], A[1], A[2], A[3]);
    o[2] = make_float4(A[4], A[5], A[6], A[7]);
    o[3] = make_float4(A[8], s[c], R[c], R[3 + c]);
    o[4] = make_float4(R[6 + c], 0.f, 0.f, 0.f);
}

template <int G>
__device__ __forceinline__ float group_sum(float v) {
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o, G);
    return v;
}

__device__ __forceinline__ void red4(float4* a, float x, float y, float z, float w) {
    atomicAdd(a, make_float4(x, y, z, w));     // red.global.add.v4.f32 (sm_90+): the result is unused
}

struct SampleArgs {
    int P, K, N;
    int rep_mask;        // R - 1
    float f;             // sampling scale factor
    float inv_n;         // 1 / N: d(mean)/d(term_n)
    const float* scaling;
    const float4* quats;
    const int32_t* knn;
    const long long* idx;
    const float* eps;
    const float4* rec;
    float4* acc;         // [R, P, kAcc] (grad instances only)
    float* partials;     // [2, gridDim.x]
};

template <int G, bool kGrad>
__global__ void __launch_bounds__(kThreads)
sugar_sample_kernel(SampleArgs a) {
    constexpr int kPerBlock = kThreads / G;
    __shared__ float red[2][kThreads / 32];
    const int lane = threadIdx.x & (G - 1);
    const int n = blockIdx.x * kPerBlock + threadIdx.x / G;
    const bool in_range = n < a.N;          // uniform over the group: every lane runs the shuffles
    const int nn = in_range ? n : a.N - 1;
    // an owner outside [0, P) is never dereferenced: the sample is skipped and makes both terms NaN
    const long long owner = __ldg(a.idx + nn);
    const bool valid = owner >= 0 && owner < a.P;
    const bool live = in_range && valid;
    const int i = valid ? (int)owner : 0;
    const float* si = a.scaling + (size_t)3 * i;
    const float* en = a.eps + (size_t)3 * nn;

    // the sample: v = quaternion_apply(q_i, (f s_i) * eps), x = mu_i + v
    const float4 q = __ldg(a.quats + i);
    const float u[3] = {a.f * __ldg(si) * __ldg(en), a.f * __ldg(si + 1) * __ldg(en + 1),
                        a.f * __ldg(si + 2) * __ldg(en + 2)};
    // (q * (0, u)) * conj(q), pytorch3d's quaternion_raw_multiply twice
    const float pw = -q.y * u[0] - q.z * u[1] - q.w * u[2];
    const float px = q.x * u[0] + q.z * u[2] - q.w * u[1];
    const float py = q.x * u[1] - q.y * u[2] + q.w * u[0];
    const float pz = q.x * u[2] + q.y * u[1] - q.z * u[0];
    const float v[3] = {-pw * q.y + px * q.x - py * q.w + pz * q.z,
                        -pw * q.z + px * q.w + py * q.x - pz * q.y,
                        -pw * q.w - px * q.z + py * q.y + pz * q.x};
    const float4* ri = a.rec + (size_t)kRec * i;
    const float4 ri0 = __ldg(ri), ri3 = __ldg(ri + 3), ri4 = __ldg(ri + 4);
    const float nrm_i[3] = {ri3.z, ri3.w, ri4.x};

    // this lane's neighbour
    const bool has = lane < a.K;
    float4 r0 = make_float4(0.f, 0.f, 0.f, 0.f), r1 = r0, r2 = r0, r3 = r0, r4 = r0;
    int j = 0;
    if (has) {
        j = __ldg(a.knn + (size_t)i * a.K + lane);
        const float4* rj = a.rec + (size_t)kRec * j;
        r0 = __ldg(rj); r1 = __ldg(rj + 1); r2 = __ldg(rj + 2); r3 = __ldg(rj + 3); r4 = __ldg(rj + 4);
    }
    const float A[9] = {r1.x, r1.y, r1.z, r1.w, r2.x, r2.y, r2.z, r2.w, r3.x};
    const float nrm_j[3] = {r3.z, r3.w, r4.x};
    const float min_s = r3.y, sigma = r0.w;
    // x - mu_j, formed as (mu_i - mu_j) + v: the offset is not lost to the rounding of x
    const float sh[3] = {(ri0.x - r0.x) + v[0], (ri0.y - r0.y) + v[1], (ri0.z - r0.z) + v[2]};
    float w[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) w[c] = A[c] * sh[0] + A[3 + c] * sh[1] + A[6 + c] * sh[2];
    const float q2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
    const float ex = expf(-0.5f * fminf(fmaxf(q2, 0.f), 1e8f));
    const float o = has ? sigma * ex : 0.f;
    // normal weights, without gradient
    const float sg = sign_of(nrm_j[0] * nrm_i[0] + nrm_j[1] * nrm_i[1] + nrm_j[2] * nrm_i[2]);
    const float m[3] = {nrm_j[0] * sg, nrm_j[1] * sg, nrm_j[2] * sg};
    const float cm = fmaxf(min_s, 1e-6f);
    const float om = has ? o * fabsf(sh[0] * m[0] + sh[1] * m[1] + sh[2] * m[2]) / (cm * cm) : 0.f;

    const float d = group_sum<G>(o);
    const float beta = group_sum<G>(has ? min_s : 0.f) / (float)a.K;
    const float wsum = fmaxf(group_sum<G>(om), 1e-6f);
    const float wk = om / wsum;
    const float S[3] = {group_sum<G>(wk * m[0]), group_sum<G>(wk * m[1]), group_sum<G>(wk * m[2])};
    const float sdf = v[0] * nrm_i[0] + v[1] * nrm_i[1] + v[2] * nrm_i[2];
    const float b2 = beta * beta;
    const float ce = -0.5f * (sdf * sdf) / b2;
    const float t = expf(ce);
    const float res[3] = {nrm_i[0] - S[0], nrm_i[1] - S[1], nrm_i[2] - S[2]};

    if (kGrad) {
        // estimation term: |d - t| / N
        const float gd = sign_of(d - t) * a.inv_n;
        const float dce = -gd * t;
        const float dsdf = dce * (-0.5f / b2) * 2.f * sdf;
        const float dbeta = -dce * ce / b2 * 2.f * beta;
        // per pair: o = sigma exp(-q2 / 2) (q2 clamped to [0, 1e8])
        const float dq2 = (q2 <= 1e8f) ? gd * sigma * ex * -0.5f : 0.f;
        float dw[3], dsh[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) dw[c] = 2.f * w[c] * dq2;
#pragma unroll
        for (int r = 0; r < 3; ++r) dsh[r] = A[3 * r] * dw[0] + A[3 * r + 1] * dw[1] + A[3 * r + 2] * dw[2];
        // normal term: |nrm_i - sum_k w_k m_k|^2 / N
        const float dr[3] = {2.f * res[0] * a.inv_n, 2.f * res[1] * a.inv_n, 2.f * res[2] * a.inv_n};
        if (live && has) {
            float4* aj = a.acc + (size_t)kAcc * ((size_t)(n & a.rep_mask) * a.P + j);
            red4(aj + kAccMuSigma, -dsh[0], -dsh[1], -dsh[2], gd * ex);
            red4(aj + kAccA0, sh[0] * dw[0], sh[0] * dw[1], sh[0] * dw[2], sh[1] * dw[0]);
            red4(aj + kAccA1, sh[1] * dw[1], sh[1] * dw[2], sh[2] * dw[0], sh[2] * dw[1]);
            red4(aj + kAccA2, sh[2] * dw[2], dbeta / (float)a.K, 0.f, 0.f);
            const float cn = -wk * sg;
            red4(aj + kAccNrmN, cn * dr[0], cn * dr[1], cn * dr[2], 0.f);
        }
        // owner: x = mu_i + v, sdf = v . nrm_i
        const float dmu[3] = {group_sum<G>(dsh[0]), group_sum<G>(dsh[1]), group_sum<G>(dsh[2])};
        // five owner slots, spread over the group's lanes
        float4* ai = a.acc + (size_t)kAcc * ((size_t)(n & a.rep_mask) * a.P + i);
        const float g[3] = {dmu[0] + dsdf * nrm_i[0], dmu[1] + dsdf * nrm_i[1], dmu[2] + dsdf * nrm_i[2]};   // dL/dv
        const float b[3] = {q.y, q.z, q.w};
        for (int slot = lane; live && slot < 5; slot += G) {
            if (slot == 0) {
                red4(ai + kAccMuSigma, dmu[0], dmu[1], dmu[2], 0.f);
            } else if (slot == 1) {
                red4(ai + kAccNrmN, dr[0], dr[1], dr[2], 0.f);
            } else if (slot == 2) {
                red4(ai + kAccNrmE, dsdf * v[0], dsdf * v[1], dsdf * v[2], 0.f);
            } else if (slot == 3) {
                // v = (w^2 - |b|^2) u + 2 (b.u) b + 2 w (b x u) for q = (w, b): d/dw and d/db
                const float ug = u[0] * g[0] + u[1] * g[1] + u[2] * g[2];
                const float bg = b[0] * g[0] + b[1] * g[1] + b[2] * g[2];
                const float bu = b[0] * u[0] + b[1] * u[1] + b[2] * u[2];
                const float bxu[3] = {b[1] * u[2] - b[2] * u[1], b[2] * u[0] - b[0] * u[2], b[0] * u[1] - b[1] * u[0]};
                const float uxg[3] = {u[1] * g[2] - u[2] * g[1], u[2] * g[0] - u[0] * g[2], u[0] * g[1] - u[1] * g[0]};
                float db[3];
#pragma unroll
                for (int c = 0; c < 3; ++c) db[c] = -2.f * ug * b[c] + 2.f * bg * u[c] + 2.f * bu * g[c] + 2.f * q.x * uxg[c];
                red4(ai + kAccQuat, 2.f * q.x * ug + 2.f * (bxu[0] * g[0] + bxu[1] * g[1] + bxu[2] * g[2]), db[0], db[1],
                     db[2]);
            } else {
                // du = (w^2 - |b|^2) g + 2 (b.g) b + 2 w (g x b); u = (f s) * eps
                const float bg = b[0] * g[0] + b[1] * g[1] + b[2] * g[2];
                const float a0 = q.x * q.x - (b[0] * b[0] + b[1] * b[1] + b[2] * b[2]);
                const float gxb[3] = {g[1] * b[2] - g[2] * b[1], g[2] * b[0] - g[0] * b[2], g[0] * b[1] - g[1] * b[0]};
                float ds[3];
#pragma unroll
                for (int c = 0; c < 3; ++c)
                    ds[c] = a.f * ((a0 * g[c] + 2.f * bg * b[c] + 2.f * q.x * gxb[c]) * __ldg(en + c));
                red4(ai + kAccScale, ds[0], ds[1], ds[2], 0.f);
            }
        }
    }

    // the two terms: one partial pair per block, in a fixed order
    float te = 0.f, tn = 0.f;
    if (in_range && lane == 0) {
        const float nan = __int_as_float(0x7fc00000);
        te = valid ? fabsf(d - t) : nan;
        tn = valid ? res[0] * res[0] + res[1] * res[1] + res[2] * res[2] : nan;
    }
#pragma unroll
    for (int o2 = 16; o2 > 0; o2 >>= 1) {
        te += __shfl_xor_sync(0xffffffffu, te, o2);
        tn += __shfl_xor_sync(0xffffffffu, tn, o2);
    }
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = te; red[1][threadIdx.x >> 5] = tn; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float se = 0.f, sn = 0.f;
        for (int k = 0; k < kThreads / 32; ++k) { se += red[0][k]; sn += red[1][k]; }
        a.partials[blockIdx.x] = se;
        a.partials[gridDim.x + blockIdx.x] = sn;
    }
}

__global__ void __launch_bounds__(1024)
sugar_terms_kernel(const float* __restrict__ partials, int n_blocks, double inv_n, float* __restrict__ terms) {
    __shared__ double sh[2][32];
    double se = 0.0, sn = 0.0;
    for (int b = threadIdx.x; b < n_blocks; b += 1024) {
        se += (double)partials[b];
        sn += (double)partials[n_blocks + b];
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        se += __shfl_xor_sync(0xffffffffu, se, o);
        sn += __shfl_xor_sync(0xffffffffu, sn, o);
    }
    if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = se; sh[1][threadIdx.x >> 5] = sn; }
    __syncthreads();
    if (threadIdx.x < 2) {
        double tot = 0.0;
        for (int w = 0; w < 32; ++w) tot += sh[threadIdx.x][w];
        terms[threadIdx.x] = (float)(tot * inv_n);
    }
}

// accumulator x upstream (d_up[0]: estimation, d_up[1]: normal) -> the four input gradients
__global__ void __launch_bounds__(kThreads)
sugar_chain_kernel(int P, int reps, const float* __restrict__ scaling, const float4* __restrict__ quats,
                   const float4* __restrict__ acc, const float* __restrict__ up, float* __restrict__ d_points,
                   float* __restrict__ d_scaling, float4* __restrict__ d_quats, float* __restrict__ d_strengths) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= P) return;
    const float ge = __ldg(up), gn = __ldg(up + 1);
    float4 sum[kAcc];
    if (reps == 1) {
#pragma unroll
        for (int k = 0; k < kAcc; ++k) sum[k] = acc[(size_t)kAcc * p + k];
    } else {
        double t[4 * kAcc] = {};
        for (int r = 0; r < reps; ++r) {
            const float4* ap = acc + (size_t)kAcc * ((size_t)r * P + p);
#pragma unroll
            for (int k = 0; k < kAcc; ++k) {
                const float4 v = ap[k];
                t[4 * k] += v.x; t[4 * k + 1] += v.y; t[4 * k + 2] += v.z; t[4 * k + 3] += v.w;
            }
        }
#pragma unroll
        for (int k = 0; k < kAcc; ++k)
            sum[k] = make_float4((float)t[4 * k], (float)t[4 * k + 1], (float)t[4 * k + 2], (float)t[4 * k + 3]);
    }
    const float4 a0 = sum[kAccMuSigma], a1 = sum[kAccA0], a2 = sum[kAccA1], a3 = sum[kAccA2], a4 = sum[kAccNrmN],
                 a5 = sum[kAccNrmE], a6 = sum[kAccQuat], a7 = sum[kAccScale];
    const size_t p3 = (size_t)3 * p;
    d_points[p3] = ge * a0.x; d_points[p3 + 1] = ge * a0.y; d_points[p3 + 2] = ge * a0.z;
    d_strengths[p] = ge * a0.w;

    const float4 q = __ldg(quats + p);
    float R[9];
    quat_to_matrix(q.x, q.y, q.z, q.w, R);
    const float s[3] = {__ldg(scaling + p3), __ldg(scaling + p3 + 1), __ldg(scaling + p3 + 2)};
    const float cs[3] = {fmaxf(s[0], 1e-8f), fmaxf(s[1], 1e-8f), fmaxf(s[2], 1e-8f)};
    const float inv[3] = {1.f / cs[0], 1.f / cs[1], 1.f / cs[2]};
    const float dA[9] = {ge * a1.x, ge * a1.y, ge * a1.z, ge * a1.w, ge * a2.x, ge * a2.y, ge * a2.z, ge * a2.w,
                         ge * a3.x};
    // A = R diag(inv): dR = dA diag(inv), dinv_c = sum_r dA[r][c] R[r][c]; d(1/clamp(s))/ds = -1/clamp(s)^2 for s >= 1e-8
    float dR[9], ds[3];
#pragma unroll
    for (int e = 0; e < 9; ++e) dR[e] = dA[e] * inv[e % 3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float dinv = dA[c] * R[c] + dA[3 + c] * R[3 + c] + dA[6 + c] * R[6 + c];
        ds[c] = (s[c] >= 1e-8f) ? -dinv / (cs[c] * cs[c]) : 0.f;
    }
    ds[0] += ge * a7.x; ds[1] += ge * a7.y; ds[2] += ge * a7.z;
    // min s (beta) and the normal: the column at argmin s
    const int c = argmin3(s[0], s[1], s[2]);
    ds[c] += ge * a3.y;
    dR[c] += ge * a5.x + gn * a4.x;
    dR[3 + c] += ge * a5.y + gn * a4.y;
    dR[6 + c] += ge * a5.z + gn * a4.z;
    d_scaling[p3] = ds[0]; d_scaling[p3 + 1] = ds[1]; d_scaling[p3 + 2] = ds[2];

    const float4 dq = quat_to_matrix_bwd(q.x, q.y, q.z, q.w, dR);
    d_quats[p] = make_float4(dq.x + ge * a6.x, dq.y + ge * a6.y, dq.z + ge * a6.z, dq.w + ge * a6.w);
}

int group_width(int K) {
    int g = 1;
    while (g < K) g <<= 1;
    return g;
}

template <bool kGrad>
void launch_samples(const SampleArgs& a, int G, int blocks, cudaStream_t s) {
    switch (G) {
        case 1: sugar_sample_kernel<1, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
        case 2: sugar_sample_kernel<2, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
        case 4: sugar_sample_kernel<4, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
        case 8: sugar_sample_kernel<8, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
        case 16: sugar_sample_kernel<16, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
        default: sugar_sample_kernel<32, kGrad><<<blocks, kThreads, 0, s>>>(a); break;
    }
}

// accumulator replicas: R * P <= max(P, 2^18), R a power of two <= 1024
int replicas(int P) {
    int r = 1;
    while (r < 1024 && (int64_t)2 * r * P <= (1 << 18)) r <<= 1;
    return r;
}

// workspace: records [P,5] float4 | partials [2, blocks] float | (gradient pass only) accumulators [R,P,8] float4
struct SugarLayout {
    size_t rec, partials, acc, acc_bytes, forward_bytes, total;
    int blocks, reps;
    SugarLayout(int P, int K, int N) {
        blocks = (int)(((int64_t)N + kThreads / group_width(K) - 1) / (kThreads / group_width(K)));
        reps = replicas(P);
        rec = 0;
        partials = rec + sizeof(float4) * kRec * (size_t)P;
        forward_bytes = partials + sizeof(float) * 2 * (size_t)blocks;
        acc = (forward_bytes + 15) & ~size_t(15);
        acc_bytes = sizeof(float4) * kAcc * (size_t)P * reps;
        total = acc + acc_bytes;
    }
};

}  // namespace

size_t sugar_reg_workspace_bytes(int P, int K, int N, bool grad) {
    const SugarLayout L(P, K, N);
    return grad ? L.total : L.forward_bytes;
}

cudaError_t launch_sugar_reg_fwd(const fb200_sugar_reg& r, bool grad, float* terms, cudaStream_t s) {
    const SugarLayout L(r.P, r.K, r.N);
    char* ws = static_cast<char*>(r.d_workspace);
    if (r.N == 0) {
        cudaError_t e = cudaMemsetAsync(terms, 0, 2 * sizeof(float), s);
        if (e == cudaSuccess && grad && r.P > 0) e = cudaMemsetAsync(ws + L.acc, 0, L.acc_bytes, s);
        return e;
    }
    float4* rec = reinterpret_cast<float4*>(ws + L.rec);
    sugar_record_kernel<<<(r.P + kThreads - 1) / kThreads, kThreads, 0, s>>>(
        r.P, r.d_points, r.d_scaling, reinterpret_cast<const float4*>(r.d_quaternions), r.d_strengths, rec);
    if (grad) {
        cudaError_t e = cudaMemsetAsync(ws + L.acc, 0, L.acc_bytes, s);
        if (e != cudaSuccess) return e;
    }
    SampleArgs a;
    a.P = r.P; a.K = r.K; a.N = r.N;
    a.rep_mask = L.reps - 1;
    a.f = r.sampling_scale_factor;
    a.inv_n = (float)(1.0 / (double)r.N);
    a.scaling = r.d_scaling;
    a.quats = reinterpret_cast<const float4*>(r.d_quaternions);
    a.knn = r.d_knn_idx;
    a.idx = reinterpret_cast<const long long*>(r.d_idx);
    a.eps = r.d_eps;
    a.rec = rec;
    a.acc = reinterpret_cast<float4*>(ws + L.acc);
    a.partials = reinterpret_cast<float*>(ws + L.partials);
    const int G = group_width(r.K);
    if (grad) launch_samples<true>(a, G, L.blocks, s);
    else launch_samples<false>(a, G, L.blocks, s);
    sugar_terms_kernel<<<1, 1024, 0, s>>>(a.partials, L.blocks, 1.0 / (double)r.N, terms);
    count_launch(3);
    return cudaGetLastError();
}

cudaError_t launch_sugar_reg_bwd(const fb200_sugar_reg& r, const float* up, float* d_points, float* d_scaling,
                                 float* d_quaternions, float* d_strengths, cudaStream_t s) {
    const SugarLayout L(r.P, r.K, r.N);
    const float4* acc = reinterpret_cast<const float4*>(static_cast<const char*>(r.d_workspace) + L.acc);
    sugar_chain_kernel<<<(r.P + kThreads - 1) / kThreads, kThreads, 0, s>>>(
        r.P, L.reps, r.d_scaling, reinterpret_cast<const float4*>(r.d_quaternions), acc, up, d_points, d_scaling,
        reinterpret_cast<float4*>(d_quaternions), d_strengths);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
