// sh.cuh -- spherical-harmonics colour evaluation, shared by preprocess (the rasterizer's own SH -> RGB) and the
// edited-frame attribute kernel (frosting_edit.cu: SH evaluated at rotated view directions).  One definition, so the
// two produce the same colour bit for bit from the same coefficients and direction.
#pragma once

#include "common.cuh"

namespace fb200 {

// The SH row of one Gaussian into registers: 3*M floats, coefficient-major, RGB innermost.
template <bool kAligned>
__device__ __forceinline__ void load_sh(int deg, const float* __restrict__ sh, float* c) {
    const int ncoef = (deg + 1) * (deg + 1);
    if (kAligned) {
        const float4* s4 = reinterpret_cast<const float4*>(sh);
        const int nq = (ncoef * 3 + 3) >> 2;
#pragma unroll
        for (int i = 0; i < 12; ++i) {
            if (i < nq) {
                float4 t = __ldg(s4 + i);
                c[4 * i + 0] = t.x; c[4 * i + 1] = t.y; c[4 * i + 2] = t.z; c[4 * i + 3] = t.w;
            }
        }
    } else {
#pragma unroll
        for (int i = 0; i < 48; ++i)
            if (i < ncoef * 3) c[i] = __ldg(sh + i);
    }
}

// frosting mode: the same row read in place from its two parameter tensors, dc [P,1,3] | rest [P,M-1,3]
// (sh_coordinates = cat(dc, rest), frosting_model.py:733-734); rest rows are 12*(M-1) bytes apart: scalar loads
__device__ __forceinline__ void load_sh_split(int deg, const float* __restrict__ dc, const float* __restrict__ rest,
                                              float* c) {
    const int ncoef = (deg + 1) * (deg + 1);
    c[0] = __ldg(dc); c[1] = __ldg(dc + 1); c[2] = __ldg(dc + 2);
#pragma unroll
    for (int i = 3; i < 48; ++i)
        if (i < ncoef * 3) c[i] = __ldg(rest + i - 3);
}

// computeColorFromSH, forward.cu:20-71.  Returns result before the +0.5 / clamp.
__device__ __forceinline__ void eval_sh(int deg, const float* c, float x, float y, float z,
                                        float& o0, float& o1, float& o2) {
    float r0 = fmul(c[0], kC0), r1 = fmul(c[1], kC0), r2 = fmul(c[2], kC0);
    if (deg > 0) {
        float k;
        k = fmul(y, kC1);
        r0 = ffma(-k, c[3], r0); r1 = ffma(-k, c[4], r1); r2 = ffma(-k, c[5], r2);
        k = fmul(z, kC1);
        r0 = ffma(k, c[6], r0); r1 = ffma(k, c[7], r1); r2 = ffma(k, c[8], r2);
        k = fmul(x, kC1);
        r0 = ffma(-k, c[9], r0); r1 = ffma(-k, c[10], r1); r2 = ffma(-k, c[11], r2);
        if (deg > 1) {
            const float xx = fmul(x, x), yy = fmul(y, y), zz = fmul(z, z);
            const float xy = fmul(y, x), yz = fmul(z, y), xz = fmul(z, x);
            k = fmul(xy, kC2_0);
            r0 = ffma(k, c[12], r0); r1 = ffma(k, c[13], r1); r2 = ffma(k, c[14], r2);
            k = fmul(yz, kC2_1);
            r0 = ffma(k, c[15], r0); r1 = ffma(k, c[16], r1); r2 = ffma(k, c[17], r2);
            const float zz2 = fadd(zz, zz);
            k = fmul(fadd(-yy, fadd(-xx, zz2)), kC2_2);
            r0 = ffma(k, c[18], r0); r1 = ffma(k, c[19], r1); r2 = ffma(k, c[20], r2);
            k = fmul(xz, kC2_3);
            r0 = ffma(k, c[21], r0); r1 = ffma(k, c[22], r1); r2 = ffma(k, c[23], r2);
            const float xx_yy = fadd(xx, -yy);
            k = fmul(xx_yy, kC2_4);
            r0 = ffma(k, c[24], r0); r1 = ffma(k, c[25], r1); r2 = ffma(k, c[26], r2);
            if (deg > 2) {
                k = fmul(fmul(y, kC3_0), ffma(xx, 3.0f, -yy));
                r0 = ffma(k, c[27], r0); r1 = ffma(k, c[28], r1); r2 = ffma(k, c[29], r2);
                k = fmul(fmul(xy, kC3_1), z);
                r0 = ffma(k, c[30], r0); r1 = ffma(k, c[31], r1); r2 = ffma(k, c[32], r2);
                const float f4 = fadd(-yy, ffma(zz, 4.0f, -xx));   // 4zz - xx - yy
                k = fmul(fmul(y, kC3_2), f4);
                r0 = ffma(k, c[33], r0); r1 = ffma(k, c[34], r1); r2 = ffma(k, c[35], r2);
                k = fmul(fmul(z, kC3_3), ffma(yy, -3.0f, ffma(xx, -3.0f, zz2)));
                r0 = ffma(k, c[36], r0); r1 = ffma(k, c[37], r1); r2 = ffma(k, c[38], r2);
                k = fmul(f4, fmul(x, kC3_4));
                r0 = ffma(k, c[39], r0); r1 = ffma(k, c[40], r1); r2 = ffma(k, c[41], r2);
                k = fmul(xx_yy, fmul(z, kC3_5));
                r0 = ffma(k, c[42], r0); r1 = ffma(k, c[43], r1); r2 = ffma(k, c[44], r2);
                k = fmul(fmul(x, kC3_6), ffma(yy, -3.0f, xx));
                r0 = ffma(k, c[45], r0); r1 = ffma(k, c[46], r1); r2 = ffma(k, c[47], r2);
            }
        }
    }
    o0 = r0; o1 = r1; o2 = r2;
}

}  // namespace fb200
