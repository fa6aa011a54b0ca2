// vec3.cuh -- float3 arithmetic in explicit round-to-nearest steps, shared by the mesh passes (frosting_edit.cu,
// frosting_init.cu): pytorch3d's normal computations are restated with it, so both give the same bits.
#pragma once

#include "common.cuh"

namespace fb200 {

struct V3 { float x, y, z; };

__device__ __forceinline__ V3 ld3(const float* p) { return {__ldg(p), __ldg(p + 1), __ldg(p + 2)}; }
__device__ __forceinline__ V3 sub(V3 a, V3 b) { return {fadd(a.x, -b.x), fadd(a.y, -b.y), fadd(a.z, -b.z)}; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) {
    return {fadd(fmul(a.y, b.z), -fmul(a.z, b.y)), fadd(fmul(a.z, b.x), -fmul(a.x, b.z)),
            fadd(fmul(a.x, b.y), -fmul(a.y, b.x))};
}
__device__ __forceinline__ float norm3(V3 a) { return __fsqrt_rn(fadd(fadd(fmul(a.x, a.x), fmul(a.y, a.y)), fmul(a.z, a.z))); }
// x / max(|x|, eps): F.normalize and pytorch3d's normal normalisations
__device__ __forceinline__ V3 normalize_eps(V3 a, float eps) {
    const float n = fmaxf(norm3(a), eps);
    return {__fdiv_rn(a.x, n), __fdiv_rn(a.y, n), __fdiv_rn(a.z, n)};
}
// a face's contribution to its vertices' normals (Meshes._compute_vertex_normals): cross(v2 - v1, v0 - v1), |.| = twice
// the area
__device__ __forceinline__ V3 area_normal(V3 v0, V3 v1, V3 v2) { return cross(sub(v2, v1), sub(v0, v1)); }

}  // namespace fb200
