// frosting_edit.cu -- per-frame attributes of an EDITED / ANIMATED Frosting scene (SURVEY.md row a21), simple and
// complex adaptation.
//
// Replaces the torch chain Frosting runs on every frame of a deformed base mesh (render_blender_scene.py ->
// blender/frosting_utils.py:551-588 render_composited_image, with make_editable(use_simple_adapt=True)):
//   shell        frosting_model.py:649-705   pytorch3d vertex normals, thickness factor (median: .median().item(),
//                                             host read-backs; triangle: per-face factor averaged over the vertex)
//   scaling      :736-756    exp * factor on edited Gaussians
//   quaternions  :768-789    face_q * ref_q^-1 * normalize(q) on edited Gaussians (compute_face_quaternions :886-898)
//   opacity drop blender/frosting_utils.py:537-548, 566-571   faces stretched beyond the threshold
//   colours      frosting_model.py:1479-1484, 1304-1352 with blender/frosting_utils.py:519-534   SH evaluated at view
//                directions rotated by R(q' * q_orig^-1), +0.5, clamp_min 0 -- in Python (eval_sh) in the reference
// by three passes over the faces / vertices and one over the Gaussians:
//   face pass    one thread per face: normal, face quaternion, relative rotation, centroid distances, triangle factor,
//                deformation keep flag;
//   median       (median method) the lower median of the edited faces' 3*F_e distances, torch.median's element, by a
//                radix select over the float bits (non-negative floats order as their bits) -- on the device, no
//                host read-back;
//   vertex pass  one thread per vertex: area-weighted normal summed over a vertex -> face CSR in a fixed order (no
//                atomics: frames are reproducible bit for bit), thickness factor, inner / outer shell vertices;
//   attributes   one thread per Gaussian (mesh rows, then background rows): position in the new shell, sigmoid
//                opacity (0 on dropped faces), exp scale * factor, rotated quaternion, SH colour.
// The complex adaptation (make_editable(use_simple_adapt=False), frosting_model.py:900-967, :1055-1119, :1149-1183) adds
//   cell pass    one thread per edited face: the cell transform T (after the shell passes: the median is on the device);
//   capture      once, one thread per mesh Gaussian: the canonical transform C = T_ref[cell]^-1 R(q) diag(exp s);
// and an attribute-kernel instance whose edited rows take scales and rotation from M = T_frame[cell] C.
// pytorch3d's maths (Meshes normals, matrix_to_quaternion, quaternion_multiply / invert / to_matrix) is restated from
// its documented definitions; see DESIGN.md.
#include <cfloat>

#include "common.cuh"
#include "frosting_attr.cuh"
#include "sh.cuh"

namespace fb200 {

namespace {

constexpr int kEditThreads = 128;
constexpr int kSelectBins = 2048;                     // 11-bit digits: passes over bits 31..21, 20..10, 9..0
constexpr int kSelBelow = kSelectBins;                // d_select words after the histogram
constexpr int kSelPrefix = kSelectBins + 1;
constexpr int kSelMask = kSelectBins + 2;

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
__device__ __forceinline__ float median3(float a, float b, float c) { return fmaxf(fminf(a, b), fminf(fmaxf(a, b), c)); }

// quaternions (w, x, y, z) as float4 (x = w)
__device__ __forceinline__ float4 q_standardize(float4 q) {
    return q.x < 0.f ? make_float4(-q.x, -q.y, -q.z, -q.w) : q;
}
__device__ __forceinline__ float4 q_invert(float4 q) { return make_float4(q.x, -q.y, -q.z, -q.w); }
// quaternion_multiply: raw Hamilton product, then the real part made non-negative.  The terms are summed in pairs that
// cancel exactly for q * q^-1, so an unmoved face's relative rotation has an exactly zero vector part
__device__ __forceinline__ float4 q_mul(float4 a, float4 b) {
    const float w = fadd(fadd(fmul(a.x, b.x), -fmul(a.y, b.y)), -fadd(fmul(a.z, b.z), fmul(a.w, b.w)));
    const float x = fadd(fadd(fmul(a.x, b.y), fmul(a.y, b.x)), fadd(fmul(a.z, b.w), -fmul(a.w, b.z)));
    const float y = fadd(fadd(fmul(a.x, b.z), fmul(a.z, b.x)), fadd(fmul(a.w, b.y), -fmul(a.y, b.w)));
    const float z = fadd(fadd(fmul(a.x, b.w), fmul(a.w, b.x)), fadd(fmul(a.y, b.z), -fmul(a.z, b.y)));
    return q_standardize(make_float4(w, x, y, z));
}
// quaternion_to_matrix (row-major m[3*r + c]); two_s = 2 / |q|^2
__device__ __forceinline__ void q_to_matrix(float4 q, float* m) {
    const float r = q.x, i = q.y, j = q.z, k = q.w;
    const float two_s = __fdiv_rn(2.0f, fadd(fadd(fadd(fmul(r, r), fmul(i, i)), fmul(j, j)), fmul(k, k)));
    m[0] = fadd(1.0f, -fmul(two_s, fadd(fmul(j, j), fmul(k, k))));
    m[1] = fmul(two_s, fadd(fmul(i, j), -fmul(k, r)));
    m[2] = fmul(two_s, fadd(fmul(i, k), fmul(j, r)));
    m[3] = fmul(two_s, fadd(fmul(i, j), fmul(k, r)));
    m[4] = fadd(1.0f, -fmul(two_s, fadd(fmul(i, i), fmul(k, k))));
    m[5] = fmul(two_s, fadd(fmul(j, k), -fmul(i, r)));
    m[6] = fmul(two_s, fadd(fmul(i, k), -fmul(j, r)));
    m[7] = fmul(two_s, fadd(fmul(j, k), fmul(i, r)));
    m[8] = fadd(1.0f, -fmul(two_s, fadd(fmul(i, i), fmul(j, j))));
}
__device__ __forceinline__ float sqrt_pos(float x) { return x > 0.f ? __fsqrt_rn(x) : 0.f; }
// matrix_to_quaternion: the candidate of the largest |q_c| (first on ties), divided by 2 max(|q_c|, 0.1); standardised
__device__ __forceinline__ float4 matrix_to_q(const float* m) {
    const float m00 = m[0], m01 = m[1], m02 = m[2], m10 = m[3], m11 = m[4], m12 = m[5], m20 = m[6], m21 = m[7], m22 = m[8];
    float qa[4] = {sqrt_pos(fadd(fadd(fadd(1.0f, m00), m11), m22)), sqrt_pos(fadd(fadd(fadd(1.0f, m00), -m11), -m22)),
                   sqrt_pos(fadd(fadd(fadd(1.0f, -m00), m11), -m22)), sqrt_pos(fadd(fadd(fadd(1.0f, -m00), -m11), m22))};
    int c = 0;
#pragma unroll
    for (int t = 1; t < 4; ++t) if (qa[t] > qa[c]) c = t;
    float4 v;
    if (c == 0)      v = make_float4(fmul(qa[0], qa[0]), fadd(m21, -m12), fadd(m02, -m20), fadd(m10, -m01));
    else if (c == 1) v = make_float4(fadd(m21, -m12), fmul(qa[1], qa[1]), fadd(m10, m01), fadd(m02, m20));
    else if (c == 2) v = make_float4(fadd(m02, -m20), fadd(m10, m01), fmul(qa[2], qa[2]), fadd(m12, m21));
    else             v = make_float4(fadd(m10, -m01), fadd(m20, m02), fadd(m21, m12), fmul(qa[3], qa[3]));
    const float d = fmul(2.0f, fmaxf(qa[c], 0.1f));
    return q_standardize(make_float4(__fdiv_rn(v.x, d), __fdiv_rn(v.y, d), __fdiv_rn(v.z, d), __fdiv_rn(v.w, d)));
}

__device__ __forceinline__ float nan_to_num(float x) {
    if (isnan(x)) return 0.f;
    if (isinf(x)) return x > 0.f ? FLT_MAX : -FLT_MAX;
    return x;
}

// ---- face pass ----
__global__ void __launch_bounds__(kEditThreads)
edit_face_kernel(fb200_frosting_edit e) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= e.n_faces) return;
    int vid[3];
    V3 v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { vid[k] = __ldg(e.d_faces + 3 * f + k); v[k] = ld3(e.d_base_verts + 3 * (size_t)vid[k]); }
    // vertex-normal contribution (Meshes._compute_vertex_normals): cross(v2 - v1, v0 - v1), |.| = twice the area
    const V3 an = cross(sub(v[2], v[1]), sub(v[0], v[1]));
    e.d_face_normals[3 * f] = an.x; e.d_face_normals[3 * f + 1] = an.y; e.d_face_normals[3 * f + 2] = an.z;
    // face frame [n, normalize(v0 - v1), normalize(n x R1)] -> quaternion (compute_face_quaternions)
    const V3 r0 = normalize_eps(normalize_eps(cross(sub(v[1], v[0]), sub(v[2], v[0])), 1e-6f), 1e-12f);
    const V3 r1 = normalize_eps(sub(v[0], v[1]), 1e-12f);
    const V3 r2 = normalize_eps(cross(r0, r1), 1e-12f);
    const float m[9] = {r0.x, r1.x, r2.x, r0.y, r1.y, r2.y, r0.z, r1.z, r2.z};
    float4 q = matrix_to_q(m);
    float nrm;
    q = frost_normalize(q, nrm);
    // vertex-to-centroid distances
    const float third = 1.0f / 3.0f;
    const V3 ctr = {fmul(fadd(fadd(v[0].x, v[1].x), v[2].x), third), fmul(fadd(fadd(v[0].y, v[1].y), v[2].y), third),
                    fmul(fadd(fadd(v[0].z, v[1].z), v[2].z), third)};
    float d[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) { d[k] = norm3(sub(v[k], ctr)); e.d_dists[3 * f + k] = d[k]; }
    const bool edited = __ldg(e.d_edition_mask + f) != 0;
    if (e.d_ref_quats == nullptr) {
        // reference capture: the face quaternions themselves, nothing dropped or rescaled
        reinterpret_cast<float4*>(e.d_rel_quats)[f] = q;
        e.d_face_factor[f] = 1.0f;
        e.d_face_keep[f] = 1;
        return;
    }
    // renormalised (a product of unit quaternions, up to rounding): an unmoved face gets the identity exactly, so an
    // unedited frame reproduces the unedited rotations bit for bit
    reinterpret_cast<float4*>(e.d_rel_quats)[f] =
        edited ? frost_normalize(q_mul(q, q_invert(__ldg(reinterpret_cast<const float4*>(e.d_ref_quats) + f))), nrm)
               : make_float4(1.f, 0.f, 0.f, 0.f);
    const V3 rd = ld3(e.d_ref_dists + 3 * f);
    e.d_face_factor[f] = edited ? nan_to_num(__fdiv_rn(median3(d[0], d[1], d[2]), median3(rd.x, rd.y, rd.z))) : 1.0f;
    // max_k(new_k / ref_k) <= threshold, a NaN ratio drops the face
    const float t = e.deformation_threshold;
    e.d_face_keep[f] = (__fdiv_rn(d[0], rd.x) <= t) && (__fdiv_rn(d[1], rd.y) <= t) && (__fdiv_rn(d[2], rd.z) <= t);
}

// ---- median: radix select over the float bits of the edited faces' distances ----
__global__ void __launch_bounds__(256)
edit_select_hist_kernel(fb200_frosting_edit e, int shift) {
    __shared__ uint32_t h[kSelectBins];
    for (int b = threadIdx.x; b < kSelectBins; b += blockDim.x) h[b] = 0;
    __syncthreads();
    const uint32_t prefix = e.d_select[kSelPrefix], mask = e.d_select[kSelMask];
    for (int f = blockIdx.x * blockDim.x + threadIdx.x; f < e.n_faces; f += gridDim.x * blockDim.x) {
        if (__ldg(e.d_edition_mask + f) == 0) continue;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const uint32_t u = __float_as_uint(e.d_dists[3 * f + k]);
            if ((u & mask) == prefix) atomicAdd(&h[(u >> shift) & (kSelectBins - 1)], 1u);
        }
    }
    __syncthreads();
    for (int b = threadIdx.x; b < kSelectBins; b += blockDim.x)
        if (h[b]) atomicAdd(e.d_select + b, h[b]);
}

// one warp: the bin holding rank k among the values still selected; the last pass writes the median and the factor
__global__ void __launch_bounds__(32)
edit_select_pick_kernel(fb200_frosting_edit e, int shift, int bits, uint32_t k, int last) {
    const unsigned full = 0xffffffffu;
    const int lane = threadIdx.x;
    constexpr int kPer = kSelectBins / 32;
    uint32_t* hist = e.d_select;
    uint32_t s = 0;
    for (int b = 0; b < kPer; ++b) s += hist[lane * kPer + b];
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(full, incl, o); if (lane >= o) incl += t; }
    const uint32_t below = hist[kSelBelow];
    const uint32_t r = k - below;                      // rank inside the selected values
    const uint32_t excl = incl - s;
    const bool mine = r >= excl && r < incl;
    __syncwarp();
    if (mine) {
        uint32_t acc = excl;
        int bin = lane * kPer;
        for (int b = 0; b < kPer; ++b) {
            const uint32_t c = hist[lane * kPer + b];
            if (r < acc + c) { bin = lane * kPer + b; break; }
            acc += c;
        }
        const uint32_t prefix = hist[kSelPrefix] | ((uint32_t)bin << shift);
        hist[kSelPrefix] = prefix;
        hist[kSelMask] |= ((1u << bits) - 1u) << shift;
        hist[kSelBelow] = below + acc;
        if (last) {
            const float med = __uint_as_float(prefix);
            e.d_factor[0] = med;
            // (current / reference) formed in double like the reference's two Python floats, stored as fp32
            e.d_factor[1] = e.d_ref_median == nullptr ? 1.0f : (float)((double)med / (double)__ldg(e.d_ref_median));
        }
    }
    __syncwarp();
    // clear the histogram for the next pass
    for (int b = 0; b < kPer; ++b) hist[lane * kPer + b] = 0;
}

// ---- vertex pass ----
__global__ void __launch_bounds__(kEditThreads)
edit_vertex_kernel(fb200_frosting_edit e) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= e.n_verts) return;
    const int lo = __ldg(e.d_vf_offsets + v), hi = __ldg(e.d_vf_offsets + v + 1);
    float nx = 0.f, ny = 0.f, nz = 0.f, fsum = 0.f;
    for (int j = lo; j < hi; ++j) {
        const int f = __ldg(e.d_vf_faces + j);
        nx = fadd(nx, e.d_face_normals[3 * f]); ny = fadd(ny, e.d_face_normals[3 * f + 1]); nz = fadd(nz, e.d_face_normals[3 * f + 2]);
        fsum = fadd(fsum, e.d_face_factor[f]);
    }
    const V3 n = normalize_eps({nx, ny, nz}, 1e-6f);
    float factor;
    if (e.rescaling == FB200_RESCALE_MEDIAN) factor = __ldg(e.d_verts_edition_mask + v) ? e.d_factor[1] : 1.0f;
    else factor = __fdiv_rn(fsum, fmaxf((float)(hi - lo), 1.0f));
    const V3 b = ld3(e.d_base_verts + 3 * (size_t)v);
    const float di = fmul(factor, __ldg(e.d_inner_dist + v)), dout = fmul(factor, __ldg(e.d_outer_dist + v));
    e.d_inner_verts[3 * v] = fadd(b.x, fmul(di, n.x)); e.d_inner_verts[3 * v + 1] = fadd(b.y, fmul(di, n.y));
    e.d_inner_verts[3 * v + 2] = fadd(b.z, fmul(di, n.z));
    e.d_outer_verts[3 * v] = fadd(b.x, fmul(dout, n.x)); e.d_outer_verts[3 * v + 1] = fadd(b.y, fmul(dout, n.y));
    e.d_outer_verts[3 * v + 2] = fadd(b.z, fmul(dout, n.z));
}

// ---- complex adaptation: cell transforms, canonical transforms ----
// axis_bary_shifts of compute_cell_transformations: float64 constants rounded to fp32, as torch.tensor(..., float32) does
constexpr float kShiftA = (float)(1.4142135623730951 / 2.0);          // np.sqrt(2) / 2
constexpr float kShiftB = (float)(1.0 / 2.449489742783178);           // 1 / np.sqrt(6)
constexpr float kShiftB2 = (float)(2.0 / 2.449489742783178);          // 2 / np.sqrt(6)

__device__ __forceinline__ V3 scale3(V3 a, float s) { return {fmul(a.x, s), fmul(a.y, s), fmul(a.z, s)}; }
__device__ __forceinline__ float dot3(V3 a, V3 b) { return fadd(fadd(fmul(a.x, b.x), fmul(a.y, b.y)), fmul(a.z, b.z)); }
__device__ __forceinline__ bool is_zero3(V3 a) { return a.x == 0.f && a.y == 0.f && a.z == 0.f; }

// compute_cell_transformations(faces_mask=edition_mask), one thread per face: T = [a', b', normalize(n) * d] (columns,
// row-major T[3r + c]) on edited faces.  a, b: the axis_bary_shifts products summed in v0, v1, v2 order; the shorter one
// Gram-Schmidt-orthogonalised against the longer as written at :943-946, both in their own slots.  d: the median of the
// edited faces' distances (median method, d_factor[0]) or the face's own median distance, 0 -> 1 (triangle).  capture:
// make_editable's fix-up of singular cells -- a zero column 0 becomes c1 x c2, then a zero column 1 becomes c2 x c0 (a
// zero column is the only way torch.det is exactly 0 that the fix-up changes)
__global__ void __launch_bounds__(kEditThreads)
edit_cell_kernel(fb200_frosting_edit e, float* cell_T, int capture) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= e.n_faces || __ldg(e.d_edition_mask + f) == 0) return;
    V3 v[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) v[k] = ld3(e.d_base_verts + 3 * (size_t)__ldg(e.d_faces + 3 * f + k));
    V3 a, b;
    a.x = fadd(fadd(fmul(-kShiftA, v[0].x), fmul(kShiftA, v[1].x)), fmul(0.f, v[2].x));
    a.y = fadd(fadd(fmul(-kShiftA, v[0].y), fmul(kShiftA, v[1].y)), fmul(0.f, v[2].y));
    a.z = fadd(fadd(fmul(-kShiftA, v[0].z), fmul(kShiftA, v[1].z)), fmul(0.f, v[2].z));
    b.x = fadd(fadd(fmul(-kShiftB, v[0].x), fmul(-kShiftB, v[1].x)), fmul(kShiftB2, v[2].x));
    b.y = fadd(fadd(fmul(-kShiftB, v[0].y), fmul(-kShiftB, v[1].y)), fmul(kShiftB2, v[2].y));
    b.z = fadd(fadd(fmul(-kShiftB, v[0].z), fmul(-kShiftB, v[1].z)), fmul(kShiftB2, v[2].z));
    const bool swap = norm3(b) > norm3(a);                // the longer axis first; a first on ties
    const V3 first = swap ? b : a, second = swap ? a : b;
    const float dt = dot3(second, first), sq = dot3(first, first);
    const V3 ortho = {fadd(second.x, -__fdiv_rn(fmul(dt, first.x), sq)), fadd(second.y, -__fdiv_rn(fmul(dt, first.y), sq)),
                      fadd(second.z, -__fdiv_rn(fmul(dt, first.z), sq))};
    V3 c0 = swap ? ortho : first, c1 = swap ? first : ortho;
    float d;
    if (e.rescaling == FB200_RESCALE_MEDIAN) {
        d = e.d_factor[0];
    } else {
        d = median3(e.d_dists[3 * f], e.d_dists[3 * f + 1], e.d_dists[3 * f + 2]);
        if (d == 0.f) d = 1.0f;
    }
    const V3 n = normalize_eps(normalize_eps(cross(sub(v[1], v[0]), sub(v[2], v[0])), 1e-6f), 1e-12f);
    const V3 c2 = scale3(n, d);
    if (capture) {
        if (is_zero3(c0)) c0 = cross(c1, c2);
        if (is_zero3(c1)) c1 = cross(c2, c0);
    }
    float* T = cell_T + 9 * (size_t)f;
    T[0] = c0.x; T[1] = c1.x; T[2] = c2.x;
    T[3] = c0.y; T[4] = c1.y; T[5] = c2.y;
    T[6] = c0.z; T[7] = c1.z; T[8] = c2.z;
}

__device__ __forceinline__ void swap_rows(float* m, int r0, int r1) {
#pragma unroll
    for (int c = 0; c < 3; ++c) { const float t = m[3 * r0 + c]; m[3 * r0 + c] = m[3 * r1 + c]; m[3 * r1 + c] = t; }
}

// make_editable(use_simple_adapt=False), one thread per mesh Gaussian: C = T_ref[cell]^-1 G, G = R(normalize(q)) diag(exp(s)),
// by a 3x3 LU with partial pivoting (getrf's rule: the first largest |a|), then getrs' two triangular solves.  An exact
// zero pivot is a singular cell (torch.linalg.solve raises): the Gaussian is counted into n_singular, its C set to zero.
// Unedited rows get C = 0.
__global__ void __launch_bounds__(kEditThreads)
edit_capture_kernel(fb200_frosting_edit e, fb200_frosting_params p, const float* cell_T, float* canonical,
                    uint32_t* n_singular) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= p.P) return;
    const size_t i = (size_t)idx;
    float* out = canonical + 9 * i;
    const long long cell = __ldg(p.d_cells + i);
    if (__ldg(e.d_edition_mask + cell) == 0) {
#pragma unroll
        for (int k = 0; k < 9; ++k) out[k] = 0.f;
        return;
    }
    float nrm;
    const float4 q = frost_normalize(__ldg(reinterpret_cast<const float4*>(p.d_quats) + i), nrm);
    float B[9], A[9];
    q_to_matrix(q, B);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float s = expf(__ldg(p.d_log_scales + 3 * i + c));
#pragma unroll
        for (int r = 0; r < 3; ++r) B[3 * r + c] = fmul(B[3 * r + c], s);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) A[k] = __ldg(cell_T + 9 * (size_t)cell + k);
    bool singular = false;
#pragma unroll
    for (int j = 0; j < 3; ++j) {
        int piv = j;
#pragma unroll
        for (int r = j + 1; r < 3; ++r) if (fabsf(A[3 * r + j]) > fabsf(A[3 * piv + j])) piv = r;
        if (piv == 1) { swap_rows(A, j, 1); swap_rows(B, j, 1); }
        else if (piv == 2) { swap_rows(A, j, 2); swap_rows(B, j, 2); }
        if (A[3 * j + j] == 0.f) { singular = true; continue; }
#pragma unroll
        for (int r = j + 1; r < 3; ++r) {
            const float l = __fdiv_rn(A[3 * r + j], A[3 * j + j]);
            A[3 * r + j] = l;
#pragma unroll
            for (int c = j + 1; c < 3; ++c) A[3 * r + c] = fadd(A[3 * r + c], -fmul(l, A[3 * j + c]));
        }
    }
    if (singular) {
        atomicAdd(n_singular, 1u);
#pragma unroll
        for (int k = 0; k < 9; ++k) out[k] = 0.f;
        return;
    }
    // L (unit lower) then U, column by column of B as trsm does
#pragma unroll
    for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int k = 0; k < 3; ++k)
#pragma unroll
            for (int r = k + 1; r < 3; ++r) B[3 * r + c] = fadd(B[3 * r + c], -fmul(B[3 * k + c], A[3 * r + k]));
#pragma unroll
        for (int k = 2; k >= 0; --k) {
            B[3 * k + c] = __fdiv_rn(B[3 * k + c], A[3 * k + k]);
#pragma unroll
            for (int r = 0; r < k; ++r) B[3 * r + c] = fadd(B[3 * r + c], -fmul(B[3 * k + c], A[3 * r + k]));
        }
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) out[k] = B[k];
}

// get_edited_quaternions_and_scales for one edited Gaussian: M = T_frame[cell] C, scales = column norms (nan_to_num),
// q = normalize(matrix_to_quaternion(M / max(scales, 1e-10)))
__device__ __forceinline__ float4 complex_edit(const float* T, const float* Cm, float* scales) {
    float t[9], c[9], m[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) { t[k] = __ldg(T + k); c[k] = __ldg(Cm + k); }
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int col = 0; col < 3; ++col)
            m[3 * r + col] = fadd(fadd(fmul(t[3 * r], c[col]), fmul(t[3 * r + 1], c[3 + col])), fmul(t[3 * r + 2], c[6 + col]));
#pragma unroll
    for (int col = 0; col < 3; ++col) {
        const float s = norm3({m[col], m[3 + col], m[6 + col]});
        scales[col] = nan_to_num(s);
        const float dv = fmaxf(s, 1e-10f);
#pragma unroll
        for (int r = 0; r < 3; ++r) m[3 * r + col] = __fdiv_rn(m[3 * r + col], dv);
    }
    float nrm;
    return frost_normalize(matrix_to_q(m), nrm);
}

// ---- per-Gaussian attributes ----
struct EditAttrArgs {
    fb200_frosting_edit e;
    fb200_frosting_params p;
    int sh_degree;
    const float* campos;
    const float* orig_quats;       // [P + n_bg, 4] or NULL
    float* means3D; float* opacities; float* scales; float* rotations; float* colors;
    const float* cell_T;           // complex adaptation: [F,9] this frame's cell transforms
    const float* canonical;        // complex adaptation: [P,9] canonical transforms
};

// Complex = false: the simple adaptation (rotate by the face's relative rotation, rescale by the thickness factor);
// true: edited rows from T_frame[cell] C[i], and every mesh row's NaN quaternion -> identity, scales nan_to_num'd
template <bool Complex>
__global__ void __launch_bounds__(kEditThreads)
edit_attr_kernel(EditAttrArgs a) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const fb200_frosting_params& p = a.p;
    if (idx >= p.P + p.n_bg) return;
    const size_t i = (size_t)idx;
    const bool bg = idx >= p.P;
    long long cell = 0;
    if (!bg) {
        cell = __ldg(p.d_cells + i);
        if (p.d_face_visible != nullptr && p.d_face_visible[cell] == 0) return;
    }
    const FrostRowT<const float> src = frost_row(p, i);
    float px, py, pz;
    if (bg) {
        px = __ldg(p.d_bg_points + 3 * src.r); py = __ldg(p.d_bg_points + 3 * src.r + 1); pz = __ldg(p.d_bg_points + 3 * src.r + 2);
    } else {
        float w[6];
        int vid[3];
        frost_point(p, i, w, vid, px, py, pz);
    }
    const bool edited = !bg && __ldg(a.e.d_edition_mask + cell) != 0;
    float opacity = frost_sigmoid(__ldg(src.opacity_logits));
    if (edited && a.e.d_face_keep[cell] == 0) opacity = 0.f;
    float4 q;
    float sc[3];
    float factor = 1.0f;
    if (Complex && edited) {
        q = complex_edit(a.cell_T + 9 * cell, a.canonical + 9 * i, sc);
    } else {
        if (edited) factor = a.e.rescaling == FB200_RESCALE_MEDIAN ? a.e.d_factor[1] : a.e.d_face_factor[cell];
        float nrm;
        q = frost_normalize(__ldg(reinterpret_cast<const float4*>(src.quats)), nrm);
        if (edited) q = q_mul(reinterpret_cast<const float4*>(a.e.d_rel_quats)[cell], q);
    }
    if (Complex && !bg && (isnan(q.x) || isnan(q.y) || isnan(q.z) || isnan(q.w))) q = make_float4(1.f, 0.f, 0.f, 0.f);
    a.means3D[3 * i] = px; a.means3D[3 * i + 1] = py; a.means3D[3 * i + 2] = pz;
    a.opacities[i] = opacity;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (Complex && edited) { a.scales[3 * i + k] = sc[k]; continue; }
        const float s = expf(__ldg(src.log_scales + k));
        // complex: the reference nan_to_num's every mesh row's scale
        a.scales[3 * i + k] = Complex ? (bg ? s : nan_to_num(s)) : edited ? fmul(s, factor) : s;
    }
    reinterpret_cast<float4*>(a.rotations)[i] = q;
    // colour: SH at the view direction, rotated into the Gaussian's original frame (row vector times R)
    const V3 dir = normalize_eps({fadd(px, -__ldg(a.campos)), fadd(py, -__ldg(a.campos + 1)), fadd(pz, -__ldg(a.campos + 2))},
                                 1e-12f);
    float x = dir.x, y = dir.y, z = dir.z;
    if (a.orig_quats != nullptr) {
        float m[9];
        q_to_matrix(q_mul(q, q_invert(__ldg(reinterpret_cast<const float4*>(a.orig_quats) + i))), m);
        x = fadd(fadd(fmul(dir.x, m[0]), fmul(dir.y, m[3])), fmul(dir.z, m[6]));
        y = fadd(fadd(fmul(dir.x, m[1]), fmul(dir.y, m[4])), fmul(dir.z, m[7]));
        z = fadd(fadd(fmul(dir.x, m[2]), fmul(dir.y, m[5])), fmul(dir.z, m[8]));
    }
    float c[48];
    load_sh_split(a.sh_degree, src.sh_dc, src.sh_rest, c);
    float r0, r1, r2;
    eval_sh(a.sh_degree, c, x, y, z, r0, r1, r2);
    a.colors[3 * i] = fmaxf(fadd(r0, 0.5f), 0.f);
    a.colors[3 * i + 1] = fmaxf(fadd(r1, 0.5f), 0.f);
    a.colors[3 * i + 2] = fmaxf(fadd(r2, 0.5f), 0.f);
}

}  // namespace

cudaError_t launch_frosting_edit_shell(const fb200_frosting_edit& e, cudaStream_t s) {
    const int F = e.n_faces, V = e.n_verts;
    if (F > 0) {
        edit_face_kernel<<<(F + kEditThreads - 1) / kEditThreads, kEditThreads, 0, s>>>(e);
        count_launch();
    }
    if (e.rescaling == FB200_RESCALE_MEDIAN && e.n_edited > 0) {
        cudaError_t err = cudaMemsetAsync(e.d_select, 0, sizeof(uint32_t) * FB200_EDIT_SELECT_WORDS, s);
        if (err != cudaSuccess) return err;
        const uint32_t k = (uint32_t)((3 * (int64_t)e.n_edited - 1) / 2);   // torch.median: the lower median
        const int grid = min((F + 255) / 256, 4 * 132);
        const int shifts[3] = {21, 10, 0}, bits[3] = {11, 11, 10};
        for (int pass = 0; pass < 3; ++pass) {
            edit_select_hist_kernel<<<grid, 256, 0, s>>>(e, shifts[pass]);
            edit_select_pick_kernel<<<1, 32, 0, s>>>(e, shifts[pass], bits[pass], k, pass == 2);
            count_launch(2);
        }
    }
    if (V > 0) {
        edit_vertex_kernel<<<(V + kEditThreads - 1) / kEditThreads, kEditThreads, 0, s>>>(e);
        count_launch();
    }
    return cudaGetLastError();
}

namespace {

void launch_cells(const fb200_frosting_edit& e, float* cell_T, int capture, cudaStream_t s) {
    if (e.n_faces > 0 && e.n_edited > 0) {
        edit_cell_kernel<<<(e.n_faces + kEditThreads - 1) / kEditThreads, kEditThreads, 0, s>>>(e, cell_T, capture);
        count_launch();
    }
}

cudaError_t launch_attr(bool complex, const fb200_frosting_edit& e, const fb200_frosting_params& p, int sh_degree,
                        const float* campos, const float* orig_quats, const float* canonical, const float* cell_T,
                        float* means3D, float* opacities, float* scales, float* rotations, float* colors,
                        cudaStream_t s) {
    const int rows = p.P + p.n_bg;
    if (rows > 0) {
        EditAttrArgs a;
        a.e = e; a.p = p; a.sh_degree = sh_degree; a.campos = campos; a.orig_quats = orig_quats;
        a.means3D = means3D; a.opacities = opacities; a.scales = scales; a.rotations = rotations; a.colors = colors;
        a.cell_T = cell_T; a.canonical = canonical;
        const auto kernel = complex ? edit_attr_kernel<true> : edit_attr_kernel<false>;
        kernel<<<(rows + kEditThreads - 1) / kEditThreads, kEditThreads, 0, s>>>(a);
        count_launch();
    }
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_frosting_edit_attr(const fb200_frosting_edit& e, const fb200_frosting_params& p, int sh_degree,
                                      const float* campos, const float* orig_quats, float* means3D, float* opacities,
                                      float* scales, float* rotations, float* colors, cudaStream_t s) {
    return launch_attr(false, e, p, sh_degree, campos, orig_quats, nullptr, nullptr, means3D, opacities, scales, rotations,
                       colors, s);
}

cudaError_t launch_frosting_edit_complex_capture(const fb200_frosting_edit& e, const fb200_frosting_params& p,
                                                 float* cell_T, float* canonical, uint32_t* n_singular,
                                                 cudaStream_t s) {
    cudaError_t err = cudaMemsetAsync(n_singular, 0, sizeof(uint32_t), s);
    if (err != cudaSuccess) return err;
    launch_cells(e, cell_T, 1, s);
    if (p.P > 0) {
        edit_capture_kernel<<<(p.P + kEditThreads - 1) / kEditThreads, kEditThreads, 0, s>>>(e, p, cell_T, canonical,
                                                                                              n_singular);
        count_launch();
    }
    return cudaGetLastError();
}

cudaError_t launch_frosting_edit_attr_complex(const fb200_frosting_edit& e, const fb200_frosting_params& p,
                                              int sh_degree, const float* campos, const float* orig_quats,
                                              const float* canonical, float* cell_T, float* means3D,
                                              float* opacities, float* scales, float* rotations, float* colors,
                                              cudaStream_t s) {
    launch_cells(e, cell_T, 0, s);
    return launch_attr(true, e, p, sh_degree, campos, orig_quats, canonical, cell_T, means3D, opacities, scales, rotations,
                       colors, s);
}

}  // namespace fb200
