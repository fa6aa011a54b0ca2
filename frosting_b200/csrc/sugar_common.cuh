// sugar_common.cuh -- per-Gaussian helpers shared by SuGaR's regularisers (sugar_reg.cu, sugar_dn.cu): pytorch3d's
// quaternion_to_matrix on raw quaternions and its backward, the smallest-axis choice and torch.sign.
#pragma once

namespace fb200 {

// pytorch3d quaternion_to_matrix, row-major: R[3 r + c]
__device__ __forceinline__ void quat_to_matrix(float r, float i, float j, float k, float R[9]) {
    const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
    R[0] = 1.f - two_s * (j * j + k * k); R[1] = two_s * (i * j - k * r); R[2] = two_s * (i * k + j * r);
    R[3] = two_s * (i * j + k * r); R[4] = 1.f - two_s * (i * i + k * k); R[5] = two_s * (j * k - i * r);
    R[6] = two_s * (i * k - j * r); R[7] = two_s * (j * k + i * r); R[8] = 1.f - two_s * (i * i + j * j);
}

// quaternion_to_matrix backward at the raw quaternion q = (r, i, j, k): dL/dq from dL/dR, two_s = 2 / |q|^2 included,
// so the radial part autograd gives through d(two_s)/dq = -two_s^2 q is kept
__device__ __forceinline__ float4 quat_to_matrix_bwd(float r, float i, float j, float k, const float dR[9]) {
    const float two_s = 2.0f / (r * r + i * i + j * j + k * k);
    const float dts = -dR[0] * (j * j + k * k) + dR[1] * (i * j - k * r) + dR[2] * (i * k + j * r) +
                      dR[3] * (i * j + k * r) - dR[4] * (i * i + k * k) + dR[5] * (j * k - i * r) +
                      dR[6] * (i * k - j * r) + dR[7] * (j * k + i * r) - dR[8] * (i * i + j * j);
    const float dr_ = two_s * (-dR[1] * k + dR[2] * j + dR[3] * k - dR[5] * i - dR[6] * j + dR[7] * i);
    const float di = two_s * (dR[1] * j + dR[2] * k + dR[3] * j - 2.f * dR[4] * i - dR[5] * r + dR[6] * k + dR[7] * r -
                              2.f * dR[8] * i);
    const float dj = two_s * (-2.f * dR[0] * j + dR[1] * i + dR[2] * r + dR[3] * i + dR[5] * k - dR[6] * r + dR[7] * k -
                              2.f * dR[8] * j);
    const float dk = two_s * (-2.f * dR[0] * k - dR[1] * r + dR[2] * i + dR[3] * r - 2.f * dR[4] * k + dR[5] * j +
                              dR[6] * i + dR[7] * j);
    const float rad = -two_s * two_s * dts;      // d(two_s)/dq = -two_s^2 q
    return make_float4(dr_ + rad * r, di + rad * i, dj + rad * j, dk + rad * k);
}

// torch.min(dim=-1): the first minimal axis
__device__ __forceinline__ int argmin3(float a, float b, float c) {
    int m = 0;
    float v = a;
    if (b < v) { m = 1; v = b; }
    if (c < v) m = 2;
    return m;
}

__device__ __forceinline__ float sign_of(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

}  // namespace fb200
