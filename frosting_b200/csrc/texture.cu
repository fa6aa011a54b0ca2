// texture.cu -- baking the textured base mesh of a trained Frosting model (frosting_utils/texture.py:11-181
// compute_textured_mesh_for_frosting_mesh, the default end of refine.py and scripts/extract_frosting_textured_mesh.py).
//
// The UV layout is implicit: face f owns half f % 2 of square f / 2 (square s = i * n + j sits at texels
// [i sq, (i+1) sq) x [j sq, (j+1) sq)), with the six inset corners of texture.py:55-69.  Nothing of it is stored; every
// kernel derives corners and faces from indices.
//
//   mesh_bary_kernel         per pixel: perspective-correct barycentrics of the prepass's face (mesh.py _barycentrics
//                            plus MeshRasterizer.forward's third weight), the same operations in the same order.
//   face_sh_colour_kernel    per face, once per bake: mean of clamp(SH2RGB(dc), 0, 1) over the face's Gaussians, summed
//                            in ascending Gaussian order over a CSR (the CPU index_add_ order).  The reference drops the
//                            result of its count clamp, so a face without Gaussians gets 0 / 0 = NaN, as there.
//   texture_claim_kernel     per pixel, pass 1 of a view: atomicMax of the pixel index into the face's and the texel's
//   texture_add_kernel       winner slot; pass 2: the winner adds its colour and 1 to the fp32 accumulators and resets its
//                            slots to -1.  `acc[idx] = acc[idx] + colors` with duplicate indices keeps ONE pixel per slot
//                            and view; on the CPU the last in row-major order, which is the rule stated here, so bakes
//                            are deterministic and match the reference run on the CPU bit for bit.
//   texture_fill_kernel      per texel: sum / count where filled, else its face's colour (view mean, or SH colour for an
//                            unseen face), written to the flipped row.
// No allocation, no host read-back; the accumulators are zeroed and the winner slots set to -1 once by the caller.
#include "common.cuh"

namespace fb200 {

namespace {

constexpr int kTexThreads = 256;

__device__ __forceinline__ float fsub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }

// nan_to_num().clamp(0, 1) of the render (texture.py:132): NaN -> 0, +-inf -> +-FLT_MAX -> 1 / 0
__device__ __forceinline__ float sanitize(float x) { return isnan(x) ? 0.f : fminf(fmaxf(x, 0.f), 1.f); }

// Texel of a pixel of face f with barycentrics b (texture.py:148):
//   int(sum_k(verts_uv[3f+k] * b_k) * T)     verts_uv = float(corner) / T,   sum left to right (the CPU reduction)
// as row * T + col (row from v, col from u, texture.py:149), or -1 when it falls outside the texture.
__device__ __forceinline__ int texel_of(int f, float b0, float b1, float b2, int sq, int n, int T) {
    const int s = f >> 1, i = s / n, j = s - i * n;
    const int u0 = i * sq, v0 = j * sq;
    int cu0, cv0, cu1, cv1, cu2, cv2;
    if (f & 1) {            // top half: (i, j+1) + (1, -1), (i, j) + (1, 3), (i+1, j+1) + (-3, -1)
        cu0 = u0 + 1;       cv0 = v0 + sq - 1;
        cu1 = u0 + 1;       cv1 = v0 + 3;
        cu2 = u0 + sq - 3;  cv2 = v0 + sq - 1;
    } else {                // bottom half: (i+1, j) + (-2, 1), (i, j) + (2, 1), (i+1, j+1) + (-2, -3)
        cu0 = u0 + sq - 2;  cv0 = v0 + 1;
        cu1 = u0 + 2;       cv1 = v0 + 1;
        cu2 = u0 + sq - 2;  cv2 = v0 + sq - 3;
    }
    const float Tf = (float)T;
    const float su = fadd(fadd(fmul(fdiv((float)cu0, Tf), b0), fmul(fdiv((float)cu1, Tf), b1)), fmul(fdiv((float)cu2, Tf), b2));
    const float sv = fadd(fadd(fmul(fdiv((float)cv0, Tf), b0), fmul(fdiv((float)cv1, Tf), b1)), fmul(fdiv((float)cv2, Tf), b2));
    const float x = fmul(su, Tf), y = fmul(sv, Tf);
    // .int() truncates toward zero: (-1, T) maps into [0, T).  Outside it the reference wraps or raises; with the inset
    // corners and the barycentrics of a hit that cannot happen, and such a pixel is dropped here.
    if (!(x > -1.f && x < Tf && y > -1.f && y < Tf)) return -1;
    return __float2int_rz(y) * T + __float2int_rz(x);
}

__global__ void __launch_bounds__(kTexThreads)
mesh_bary_kernel(int F, const float* __restrict__ verts, const int32_t* __restrict__ faces,
                 const float* __restrict__ proj, int W, int H, const int32_t* __restrict__ pix_to_face,
                 float* __restrict__ bary) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= W * H) return;
    const int f = __ldg(pix_to_face + p);
    float* out = bary + 3 * (size_t)p;
    if (f < 0 || f >= F) {                    // no hit: uv = 0, third weight 1 - 0
        out[0] = 0.f; out[1] = 0.f; out[2] = 1.f;
        return;
    }
    // clip = [v, 1] @ proj, then screen coordinates (c / w * 0.5 + 0.5) * size
    float sx[3], sy[3], w[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const int v = __ldg(faces + 3 * f + k);
        const float x = __ldg(verts + 3 * v), y = __ldg(verts + 3 * v + 1), z = __ldg(verts + 3 * v + 2);
        float c[4];
#pragma unroll
        for (int r = 0; r < 4; ++r)
            c[r] = fadd(ffma(z, __ldg(proj + 8 + r), ffma(y, __ldg(proj + 4 + r), fmul(x, __ldg(proj + r)))),
                        __ldg(proj + 12 + r));
        w[k] = c[3];
        sx[k] = fmul(fadd(fmul(fdiv(c[0], c[3]), 0.5f), 0.5f), (float)W);
        sy[k] = fmul(fadd(fmul(fdiv(c[1], c[3]), 0.5f), 0.5f), (float)H);
    }
    const int py_i = p / W;
    const float px = fadd((float)(p - py_i * W), 0.5f), py = fadd((float)py_i, 0.5f);
    auto edge = [&](int a, int b) {
        return fsub(fmul(fsub(sx[b], sx[a]), fsub(py, sy[a])), fmul(fsub(sy[b], sy[a]), fsub(px, sx[a])));
    };
    float b0 = edge(1, 2), b1 = edge(2, 0), b2 = edge(0, 1);
    const float area = fadd(fadd(b0, b1), b2);
    b0 = fdiv(fdiv(b0, area), w[0]);
    b1 = fdiv(fdiv(b1, area), w[1]);
    b2 = fdiv(fdiv(b2, area), w[2]);
    const float s = fadd(fadd(b0, b1), b2);
    const float u = fdiv(b0, s), v = fdiv(b1, s);
    out[0] = u; out[1] = v; out[2] = fsub(1.f, fadd(u, v));
}

__global__ void __launch_bounds__(kTexThreads)
face_sh_colour_kernel(fb200_texture t) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= t.n_faces) return;
    const int beg = __ldg(t.d_cell_offsets + f), end = __ldg(t.d_cell_offsets + f + 1);
    float r = 0.f, g = 0.f, b = 0.f;
    for (int k = beg; k < end; ++k) {
        const float* dc = t.d_sh_dc + 3 * (size_t)__ldg(t.d_cell_points + k);
        // SH2RGB: sh * C0 + 0.5 (two roundings), then clamp(0, 1)
        r = fadd(r, fminf(fmaxf(fadd(fmul(__ldg(dc), kC0), 0.5f), 0.f), 1.f));
        g = fadd(g, fminf(fmaxf(fadd(fmul(__ldg(dc + 1), kC0), 0.5f), 0.f), 1.f));
        b = fadd(b, fminf(fmaxf(fadd(fmul(__ldg(dc + 2), kC0), 0.5f), 0.f), 1.f));
    }
    const float n = (float)(end - beg);       // not clamped: 0 / 0 = NaN without Gaussians, as the reference
    t.d_face_sh[3 * (size_t)f] = fdiv(r, n);
    t.d_face_sh[3 * (size_t)f + 1] = fdiv(g, n);
    t.d_face_sh[3 * (size_t)f + 2] = fdiv(b, n);
}

__device__ __forceinline__ int texel_of_pixel(const fb200_texture& t, int f, const float* __restrict__ bary, int p) {
    return texel_of(f, __ldg(bary + 3 * (size_t)p), __ldg(bary + 3 * (size_t)p + 1), __ldg(bary + 3 * (size_t)p + 2),
                    t.square_size, t.n_square_per_axis, t.texture_size);
}

__global__ void __launch_bounds__(kTexThreads)
texture_claim_kernel(fb200_texture t, const int32_t* __restrict__ pix_to_face, const float* __restrict__ bary, int n_pix) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pix) return;
    const int f = __ldg(pix_to_face + p);
    if (f < 0 || f >= t.n_faces) return;
    atomicMax(t.d_face_winner + f, p);
    const int x = texel_of_pixel(t, f, bary, p);
    if (x >= 0) atomicMax(t.d_texel_winner + x, p);
}

__device__ __forceinline__ void add_colour(float* __restrict__ acc, float r, float g, float b) {
    float4 a = *reinterpret_cast<float4*>(acc);
    a.x = fadd(a.x, r); a.y = fadd(a.y, g); a.z = fadd(a.z, b); a.w = fadd(a.w, 1.f);
    *reinterpret_cast<float4*>(acc) = a;
}

__global__ void __launch_bounds__(kTexThreads)
texture_add_kernel(fb200_texture t, const float* __restrict__ image, const int32_t* __restrict__ pix_to_face,
                   const float* __restrict__ bary, int n_pix) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pix) return;
    const int f = __ldg(pix_to_face + p);
    if (f < 0 || f >= t.n_faces) return;
    const int x = texel_of_pixel(t, f, bary, p);
    // a slot read here holds this view's winner or, once the winner has reset it, -1: only the winner matches
    const bool face_win = t.d_face_winner[f] == p;
    const bool texel_win = x >= 0 && t.d_texel_winner[x] == p;
    if (!face_win && !texel_win) return;
    const float r = sanitize(__ldg(image + 3 * (size_t)p)), g = sanitize(__ldg(image + 3 * (size_t)p + 1)),
                b = sanitize(__ldg(image + 3 * (size_t)p + 2));
    if (face_win) {
        add_colour(t.d_face_acc + 4 * (size_t)f, r, g, b);
        t.d_face_winner[f] = -1;
    }
    if (texel_win) {
        add_colour(t.d_texel_acc + 4 * (size_t)x, r, g, b);
        t.d_texel_winner[x] = -1;
    }
}

__global__ void __launch_bounds__(kTexThreads)
texture_fill_kernel(fb200_texture t, float* __restrict__ texture) {
    const int T = t.texture_size;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= T * T) return;
    const int r = x / T, c = x - r * T;
    const float4 a = *reinterpret_cast<const float4*>(t.d_texel_acc + 4 * (size_t)x);
    float o0, o1, o2;
    if (a.w > 0.f) {
        o0 = fdiv(a.x, a.w); o1 = fdiv(a.y, a.w); o2 = fdiv(a.z, a.w);
    } else {
        // uv_to_faces transposed (texture.py:75-87): column c is the first coordinate, row r the second
        const int sq = t.square_size;
        const int f = min(2 * ((c / sq) * t.n_square_per_axis + r / sq) + ((c % sq) < (r % sq) ? 1 : 0), t.n_faces - 1);
        const float4 fa = *reinterpret_cast<const float4*>(t.d_face_acc + 4 * (size_t)f);
        if (fa.w > 0.f) {
            o0 = fdiv(fa.x, fa.w); o1 = fdiv(fa.y, fa.w); o2 = fdiv(fa.z, fa.w);
        } else {
            o0 = t.d_face_sh[3 * (size_t)f]; o1 = t.d_face_sh[3 * (size_t)f + 1]; o2 = t.d_face_sh[3 * (size_t)f + 2];
        }
    }
    float* out = texture + 3 * ((size_t)(T - 1 - r) * T + c);     // flip(0)
    out[0] = o0; out[1] = o1; out[2] = o2;
}

inline int blocks(long long n) { return (int)((n + kTexThreads - 1) / kTexThreads); }

}  // namespace

cudaError_t launch_mesh_bary(int F, const float* verts, const int32_t* faces, const float* proj, int W, int H,
                             const int32_t* pix_to_face, float* bary, cudaStream_t s) {
    mesh_bary_kernel<<<blocks((long long)W * H), kTexThreads, 0, s>>>(F, verts, faces, proj, W, H, pix_to_face, bary);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_texture_face_sh(const fb200_texture& t, cudaStream_t s) {
    face_sh_colour_kernel<<<blocks(t.n_faces), kTexThreads, 0, s>>>(t);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_texture_add_view(const fb200_texture& t, const float* image, const int32_t* pix_to_face,
                                    const float* bary, int n_pix, cudaStream_t s) {
    texture_claim_kernel<<<blocks(n_pix), kTexThreads, 0, s>>>(t, pix_to_face, bary, n_pix);
    texture_add_kernel<<<blocks(n_pix), kTexThreads, 0, s>>>(t, image, pix_to_face, bary, n_pix);
    count_launch(2);
    return cudaGetLastError();
}

cudaError_t launch_texture_fill(const fb200_texture& t, float* texture, cudaStream_t s) {
    texture_fill_kernel<<<blocks((long long)t.texture_size * t.texture_size), kTexThreads, 0, s>>>(t, texture);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
