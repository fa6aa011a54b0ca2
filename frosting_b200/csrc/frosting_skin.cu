// frosting_skin.cu -- linear-blend skinning of the base mesh of a Blender-animated Frosting scene.
//
// Replaces the per-frame bone loop of blender/frosting_utils.py:474-516 apply_poses_to_scene: for every rigged mesh and
// every bone with vertices, two pytorch3d Transform3d's (a torch.inverse with its host-side status check, two
// transform_points), a float64 multiply and an index += -- hundreds of small kernels and one host synchronisation per
// bone.  Here one thread per rigged vertex walks its CSR entries (bone, float64 weight) in the reference's bone order:
//   q = [p_tpose, 1] @ reset[bone];          q = q.xyz / q.w      reset = inverse(rest^T), computed once by the caller
//   r = [q, 1]       @ pose[bone][frame];    r = r.xyz / r.w      pose  = the track's matrix transposed
//   acc = float(double(acc) + w * double(r))                      the float64 product, then the float32 index +=
// and writes acc into the caller's base-vertex buffer.  A vertex without a bone of its armature is written 0 (the
// reference starts from zeros).  Summation follows the bone order per vertex, so no atomics and frames reproduce bit
// for bit.  No allocation, no host read-back; the frame index is a by-value argument.
#include "common.cuh"

namespace fb200 {

namespace {

constexpr int kSkinThreads = 128;

// [x, y, z, 1] @ m (row-major 4x4, row-vector convention as Transform3d.transform_points), then the homogeneous divide
__device__ __forceinline__ float3 transform_point(const float4* __restrict__ m, float3 p) {
    const float4 r0 = __ldg(m), r1 = __ldg(m + 1), r2 = __ldg(m + 2), r3 = __ldg(m + 3);
    const float x = p.x * r0.x + p.y * r1.x + p.z * r2.x + r3.x;
    const float y = p.x * r0.y + p.y * r1.y + p.z * r2.y + r3.y;
    const float z = p.x * r0.z + p.y * r1.z + p.z * r2.z + r3.z;
    const float w = p.x * r0.w + p.y * r1.w + p.z * r2.w + r3.w;
    return make_float3(__fdiv_rn(x, w), __fdiv_rn(y, w), __fdiv_rn(z, w));
}

__global__ void __launch_bounds__(kSkinThreads)
skin_kernel(fb200_frosting_skin s, int frame, float* __restrict__ base_verts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s.n_rows) return;
    const float3 p = make_float3(__ldg(s.d_tpose + 3 * i), __ldg(s.d_tpose + 3 * i + 1), __ldg(s.d_tpose + 3 * i + 2));
    const float4* reset = reinterpret_cast<const float4*>(s.d_reset);
    const float4* pose = reinterpret_cast<const float4*>(s.d_pose);
    float ax = 0.f, ay = 0.f, az = 0.f;
    const int end = __ldg(s.d_offsets + i + 1);
    for (int k = __ldg(s.d_offsets + i); k < end; ++k) {
        const int b = __ldg(s.d_bones + k);
        const double w = __ldg(s.d_weights + k);
        const float3 q = transform_point(reset + 4 * (size_t)b, p);
        const float3 r = transform_point(pose + 4 * ((size_t)b * s.n_frames + frame), q);
        ax = __double2float_rn(__dadd_rn((double)ax, __dmul_rn(w, (double)r.x)));
        ay = __double2float_rn(__dadd_rn((double)ay, __dmul_rn(w, (double)r.y)));
        az = __double2float_rn(__dadd_rn((double)az, __dmul_rn(w, (double)r.z)));
    }
    const int v = __ldg(s.d_vert_ids + i);
    base_verts[3 * (size_t)v] = ax;
    base_verts[3 * (size_t)v + 1] = ay;
    base_verts[3 * (size_t)v + 2] = az;
}

}  // namespace

cudaError_t launch_frosting_skin(const fb200_frosting_skin& s, int frame, float* base_verts, cudaStream_t st) {
    if (s.n_rows > 0) {
        skin_kernel<<<(s.n_rows + kSkinThreads - 1) / kSkinThreads, kSkinThreads, 0, st>>>(s, frame, base_verts);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace fb200
