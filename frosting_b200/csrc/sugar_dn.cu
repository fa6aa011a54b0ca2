// sugar_dn.cu -- SuGaR's depth-normal consistency of the coarse `dn_consistency` trainer, forward and backward
// (SURVEY.md row 17).
//
// Replaces frosting_scene/sugar_model.py:2343-2387 (render_depth_and_normal) and
// frosting_trainers/coarse_density_and_dn_consistency.py:17-95 (depths_to_points, depth2normal_2dgs,
// depth_normal_consistency_loss), which the reference runs as a second rasterizer call plus ~30 torch kernels.  The
// render itself is the rasterizer's extra channels (fb200_extra, row f4): one traversal blends these features with the
// colour's weights.  Here:
//   1. dn_features_kernel (P threads): n = the column of quaternion_to_matrix(q) at argmin s (raw q, two_s = 2/|q|^2),
//      flipped by sign(n . (campos - p)) (0 gives a zero normal); features = {z, (R n).x, (R n).y} in pytorch3d's view
//      frame, which is diag(-1, -1, 1) times the COLMAP view frame of `viewmatrix` (z equal, x and y negated).
//   2. dn_features_bwd_kernel (P threads): dL/dfeatures -> dL/dpoints (through z only) and dL/dquaternions (through the
//      selected column, radial part kept); argmin and sign are discrete and get no gradient.
//   3. dn_loss_fwd_kernel (16 x 16 pixel tiles): the blended image dn [3,H,W] gives depth dn[0] and the normal
//      (-dn[1], -dn[2], -sqrt(1 - min(dn[1]^2 + dn[2]^2, 1))); the depth's points d * ray(x, y), the central differences
//      dx (rows) and dy (columns) at interior pixels, n_d = normalize(dx x dy) (eps 1e-12), rotated into the COLMAP view
//      frame; per pixel 1 - normal . n_d (border pixels: 1), one partial per tile, loss.cu's fixed-order reduction.
//   4. dn_loss_bwd_kernel (same tiles): a pixel's depth enters dx of its vertical neighbours and dy of its horizontal
//      ones, so each tile recomputes dL/ddx and dL/ddy over itself plus a one-pixel halo into shared memory (the depths
//      with a two-pixel halo) and gathers them: no atomics, bit-reproducible.  Normal channels are local.
// Arithmetic: the rays are c2w[:3,:3] K^-1 (x, y, 1) at integer pixel coordinates, with c2w = (viewmatrix^T)^-1 and
// K^-1 from ((c2w^T projmatrix) ndc2pix)[:3,:3]^T, derived by each block in double from the two device 4x4s (no host
// read-back, no extra launch).  dx and dy are formed in double as d_a ray_a - d_b ray_b: the camera origin, which the
// reference adds to every point before subtracting neighbours ~1e-3 apart, cancels and is never added.  From dx and dy
// on the arithmetic is float32 in the reference's operation order, so the branches of normalize (|v| < eps) and of
// clamp_max / sqrt are decided as torch decides them; at exactly |xy|^2 = 1 the normal channels' gradient is torch's
// infinite (or NaN) one.
#include "common.cuh"
#include "sugar_common.cuh"

namespace fb200 {

namespace {

constexpr int kThreads = 256;
constexpr int kT = 16;                  // tile edge (pixels)
constexpr int kG = kT + 2;              // tile + one-pixel halo: where the backward needs dL/ddx, dL/ddy
constexpr int kD = kT + 4;              // tile + two-pixel halo: the depths those need
constexpr float kEps = 1e-12f;          // F.normalize

// ---- features ------------------------------------------------------------------------------------------------------

struct DnGauss {
    float n[3];     // the column of R(q) at the smallest axis
    int c;          // that axis
    float sg;       // sign(n . (campos - p))
};

__device__ __forceinline__ DnGauss dn_gauss(int p, const float* __restrict__ points, const float* __restrict__ scaling,
                                            const float4* __restrict__ quats, const float* __restrict__ campos) {
    DnGauss g;
    const float4 q = __ldg(quats + p);
    float R[9];
    quat_to_matrix(q.x, q.y, q.z, q.w, R);
    const size_t p3 = (size_t)3 * p;
    g.c = argmin3(__ldg(scaling + p3), __ldg(scaling + p3 + 1), __ldg(scaling + p3 + 2));
#pragma unroll
    for (int r = 0; r < 3; ++r) g.n[r] = g.c == 0 ? R[3 * r] : (g.c == 1 ? R[3 * r + 1] : R[3 * r + 2]);
    // decided in double (exact differences, a 3-term dot product rounded once): the sign of the exact value at the
    // float32 inputs, except within ~1e-16 relative of zero
    const double to[3] = {(double)__ldg(campos) - __ldg(points + p3), (double)__ldg(campos + 1) - __ldg(points + p3 + 1),
                          (double)__ldg(campos + 2) - __ldg(points + p3 + 2)};
    const double dot = (double)g.n[0] * to[0] + (double)g.n[1] * to[1] + (double)g.n[2] * to[2];
    g.sg = dot > 0.0 ? 1.f : (dot < 0.0 ? -1.f : 0.f);
    return g;
}

// viewmatrix: world_view_transform (row-vector convention, row-major [4,4]): COLMAP view = [p, 1] @ V
__global__ void __launch_bounds__(kThreads)
dn_features_kernel(int P, const float* __restrict__ points, const float* __restrict__ scaling,
                   const float4* __restrict__ quats, const float* __restrict__ view, const float* __restrict__ campos,
                   float* __restrict__ feat) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= P) return;
    const DnGauss g = dn_gauss(p, points, scaling, quats, campos);
    const size_t p3 = (size_t)3 * p;
    const float x = __ldg(points + p3), y = __ldg(points + p3 + 1), z = __ldg(points + p3 + 2);
    const float n[3] = {g.n[0] * g.sg, g.n[1] * g.sg, g.n[2] * g.sg};
    feat[p3] = x * __ldg(view + 2) + y * __ldg(view + 6) + z * __ldg(view + 10) + __ldg(view + 14);
    feat[p3 + 1] = -(n[0] * __ldg(view + 0) + n[1] * __ldg(view + 4) + n[2] * __ldg(view + 8));
    feat[p3 + 2] = -(n[0] * __ldg(view + 1) + n[1] * __ldg(view + 5) + n[2] * __ldg(view + 9));
}

__global__ void __launch_bounds__(kThreads)
dn_features_bwd_kernel(int P, const float* __restrict__ points, const float* __restrict__ scaling,
                       const float4* __restrict__ quats, const float* __restrict__ view,
                       const float* __restrict__ campos, const float* __restrict__ d_feat,
                       float* __restrict__ d_points, float4* __restrict__ d_quats) {
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= P) return;
    const DnGauss g = dn_gauss(p, points, scaling, quats, campos);
    const size_t p3 = (size_t)3 * p;
    const float gz = __ldg(d_feat + p3), gx = __ldg(d_feat + p3 + 1), gy = __ldg(d_feat + p3 + 2);
    d_points[p3] = gz * __ldg(view + 2);
    d_points[p3 + 1] = gz * __ldg(view + 6);
    d_points[p3 + 2] = gz * __ldg(view + 10);
    // feature 1 = -(n . V[:,0]), feature 2 = -(n . V[:,1]), n = sg R[:, c]
    float dR[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        const float dn = -g.sg * (gx * __ldg(view + 4 * r) + gy * __ldg(view + 4 * r + 1));
#pragma unroll
        for (int c = 0; c < 3; ++c) dR[3 * r + c] = (c == g.c) ? dn : 0.f;
    }
    const float4 q = __ldg(quats + p);
    d_quats[p] = quat_to_matrix_bwd(q.x, q.y, q.z, q.w, dR);
}

// ---- consistency loss ----------------------------------------------------------------------------------------------

// inverse of a row-major [4,4] by cofactors (2x2 sub-determinants of rows 0-1 and 2-3), in double
__host__ __device__ inline void invert4(const double* a, double* b) {
    const double s0 = a[0] * a[5] - a[4] * a[1], s1 = a[0] * a[6] - a[4] * a[2], s2 = a[0] * a[7] - a[4] * a[3];
    const double s3 = a[1] * a[6] - a[5] * a[2], s4 = a[1] * a[7] - a[5] * a[3], s5 = a[2] * a[7] - a[6] * a[3];
    const double c5 = a[10] * a[15] - a[14] * a[11], c4 = a[9] * a[15] - a[13] * a[11], c3 = a[9] * a[14] - a[13] * a[10];
    const double c2 = a[8] * a[15] - a[12] * a[11], c1 = a[8] * a[14] - a[12] * a[10], c0 = a[8] * a[13] - a[12] * a[9];
    const double id = 1.0 / (s0 * c5 - s1 * c4 + s2 * c3 + s3 * c2 - s4 * c1 + s5 * c0);
    b[0] = (a[5] * c5 - a[6] * c4 + a[7] * c3) * id;
    b[1] = (-a[1] * c5 + a[2] * c4 - a[3] * c3) * id;
    b[2] = (a[13] * s5 - a[14] * s4 + a[15] * s3) * id;
    b[3] = (-a[9] * s5 + a[10] * s4 - a[11] * s3) * id;
    b[4] = (-a[4] * c5 + a[6] * c2 - a[7] * c1) * id;
    b[5] = (a[0] * c5 - a[2] * c2 + a[3] * c1) * id;
    b[6] = (-a[12] * s5 + a[14] * s2 - a[15] * s1) * id;
    b[7] = (a[8] * s5 - a[10] * s2 + a[11] * s1) * id;
    b[8] = (a[4] * c4 - a[5] * c2 + a[7] * c0) * id;
    b[9] = (-a[0] * c4 + a[1] * c2 - a[3] * c0) * id;
    b[10] = (a[12] * s4 - a[13] * s2 + a[15] * s0) * id;
    b[11] = (-a[8] * s4 + a[9] * s2 - a[11] * s0) * id;
    b[12] = (-a[4] * c3 + a[5] * c1 - a[6] * c0) * id;
    b[13] = (a[0] * c3 - a[1] * c1 + a[2] * c0) * id;
    b[14] = (-a[12] * s3 + a[13] * s1 - a[14] * s0) * id;
    b[15] = (a[8] * s3 - a[9] * s1 + a[10] * s0) * id;
}

// inverse of a row-major [3,3] by its adjugate, in double
__host__ __device__ inline void invert3(const double* a, double* b) {
    const double c0 = a[4] * a[8] - a[5] * a[7], c1 = a[5] * a[6] - a[3] * a[8], c2 = a[3] * a[7] - a[4] * a[6];
    const double id = 1.0 / (a[0] * c0 + a[1] * c1 + a[2] * c2);
    b[0] = c0 * id; b[1] = (a[2] * a[7] - a[1] * a[8]) * id; b[2] = (a[1] * a[5] - a[2] * a[4]) * id;
    b[3] = c1 * id; b[4] = (a[0] * a[8] - a[2] * a[6]) * id; b[5] = (a[2] * a[3] - a[0] * a[5]) * id;
    b[6] = c2 * id; b[7] = (a[1] * a[6] - a[0] * a[7]) * id; b[8] = (a[0] * a[4] - a[1] * a[3]) * id;
}

// What every pixel of a frame shares: the ray matrix M (ray(x, y) = M (x, y, 1), row-major) and the view rotation
// V[:3,:3].  Derived by one thread of each block.
struct DnCam {
    double M[9];
    float V[9];
};

__host__ __device__ inline void dn_camera(const float* view, const float* proj, int H, int W, DnCam& cam) {
    double A[16], c2w[16];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) A[r * 4 + c] = view[c * 4 + r];
    invert4(A, c2w);                                            // c2w = (V^T)^-1
    // intrins = ((c2w^T F) ndc2pix)[:3,:3]^T with ndc2pix [4,3] = {{W/2,0,0}, {0,H/2,0}, {0,0,0}, {W/2,H/2,1}}:
    // row c of intrins is row r of c2w^T F, columns 0..2, times ndc2pix
    double PF[12];                                              // (c2w^T F)[:3, :]
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            double s = 0.0;
#pragma unroll
            for (int k = 0; k < 4; ++k) s += c2w[k * 4 + r] * (double)proj[k * 4 + c];
            PF[r * 4 + c] = s;
        }
    const double hw = 0.5 * W, hh = 0.5 * H;
    double K[9], Kinv[9];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
        K[0 * 3 + r] = PF[r * 4 + 0] * hw + PF[r * 4 + 3] * hw;
        K[1 * 3 + r] = PF[r * 4 + 1] * hh + PF[r * 4 + 3] * hh;
        K[2 * 3 + r] = PF[r * 4 + 3];
    }
    invert3(K, Kinv);
    // rays_d = pix @ K^-T @ c2w[:3,:3]^T, i.e. ray = c2w[:3,:3] K^-1 pix
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c)
            cam.M[r * 3 + c] = c2w[r * 4] * Kinv[c] + c2w[r * 4 + 1] * Kinv[3 + c] + c2w[r * 4 + 2] * Kinv[6 + c];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) cam.V[r * 3 + c] = view[r * 4 + c];
}

__device__ __forceinline__ float3 cross3(float3 a, float3 b) {
    return make_float3(a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x);
}

// ray(x, y) = M (x, y, 1) in double
__device__ __forceinline__ double3 ray_at(const DnCam& cam, int x, int y) {
    const double X = x, Y = y;
    return make_double3(fma(cam.M[0], X, fma(cam.M[1], Y, cam.M[2])), fma(cam.M[3], X, fma(cam.M[4], Y, cam.M[5])),
                        fma(cam.M[6], X, fma(cam.M[7], Y, cam.M[8])));
}

// d_b ray(p + e) - d_a ray(p - e) = (d_b - d_a) ray(p) + (d_b + d_a) m, m = M e the ray's step: in double (d_b - d_a
// and d_b + d_a of two floats are exact there), rounded once to float
__device__ __forceinline__ float3 central_diff(double3 ray, float da, float db, double mx, double my, double mz) {
    const double s = (double)db - (double)da, t = (double)db + (double)da;
    return make_float3((float)fma(s, ray.x, t * mx), (float)fma(s, ray.y, t * my), (float)fma(s, ray.z, t * mz));
}

// the view-frame normal n_d at an interior pixel from its four neighbours' depths (u, d: rows y -+ 1; l, r: columns)
struct DnStencil {
    float3 dx, dy, v;
    float nrm, den;
    float nv[3];
};

__device__ __forceinline__ DnStencil stencil(const DnCam& cam, int x, int y, float du, float dd, float dl, float dr) {
    DnStencil s;
    const double3 ray = ray_at(cam, x, y);
    s.dx = central_diff(ray, du, dd, cam.M[1], cam.M[4], cam.M[7]);
    s.dy = central_diff(ray, dl, dr, cam.M[0], cam.M[3], cam.M[6]);
    s.v = cross3(s.dx, s.dy);
    s.nrm = sqrtf(s.v.x * s.v.x + s.v.y * s.v.y + s.v.z * s.v.z);
    s.den = fmaxf(s.nrm, kEps);
    const float n[3] = {s.v.x / s.den, s.v.y / s.den, s.v.z / s.den};
#pragma unroll
    for (int j = 0; j < 3; ++j) s.nv[j] = n[0] * cam.V[j] + n[1] * cam.V[3 + j] + n[2] * cam.V[6 + j];
    return s;
}

struct DnNormal {
    float a, b, q, s;
};

__device__ __forceinline__ DnNormal rendered_normal(const float* __restrict__ dn, size_t plane, size_t o) {
    DnNormal n;
    n.a = __ldg(dn + plane + o);
    n.b = __ldg(dn + 2 * plane + o);
    n.q = __fadd_rn(__fmul_rn(n.a, n.a), __fmul_rn(n.b, n.b));     // rounded as torch's pow and sum: no FMA
    n.s = sqrtf(1.f - fminf(n.q, 1.f));
    return n;
}

__device__ __forceinline__ bool interior(int x, int y, int H, int W) { return x >= 1 && x <= W - 2 && y >= 1 && y <= H - 2; }

__global__ void __launch_bounds__(kThreads, 2)
dn_loss_fwd_kernel(const float* __restrict__ dn, int H, int W, const float* __restrict__ view,
                   const float* __restrict__ proj, float* __restrict__ partials) {
    __shared__ DnCam cam;
    __shared__ float red[kThreads / 32];
    if (threadIdx.x == 0) dn_camera(view, proj, H, W, cam);
    __syncthreads();
    const int tiles_x = (W + kT - 1) / kT, n_tiles = tiles_x * ((H + kT - 1) / kT);
    const size_t plane = (size_t)H * W;
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int x = (t % tiles_x) * kT + threadIdx.x % kT, y = (t / tiles_x) * kT + threadIdx.x / kT;
        float e = 0.f;
        if (x < W && y < H) {
            const size_t o = (size_t)y * W + x;
            float nv[3] = {0.f, 0.f, 0.f};
            if (interior(x, y, H, W)) {
                const DnStencil s = stencil(cam, x, y, __ldg(dn + o - W), __ldg(dn + o + W), __ldg(dn + o - 1),
                                            __ldg(dn + o + 1));
                nv[0] = s.nv[0]; nv[1] = s.nv[1]; nv[2] = s.nv[2];
            }
            const DnNormal n = rendered_normal(dn, plane, o);
            e = 1.f - ((-n.a) * nv[0] + (-n.b) * nv[1] + (-n.s) * nv[2]);
        }
#pragma unroll
        for (int k = 16; k > 0; k >>= 1) e += __shfl_xor_sync(0xffffffffu, e, k);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = e;
        __syncthreads();
        if (threadIdx.x == 0) {
            float s = 0.f;
            for (int i = 0; i < kThreads / 32; ++i) s += red[i];
            partials[t] = s;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads, 2)
dn_loss_bwd_kernel(const float* __restrict__ dn, int H, int W, const float* __restrict__ view,
                   const float* __restrict__ proj, const float* __restrict__ dL_dloss, float* __restrict__ d_dn) {
    __shared__ DnCam cam;
    __shared__ float sd[kD][kD + 1];            // depths, two-pixel halo (0 outside the image)
    __shared__ float sg[6][kG][kG + 1];         // dL/ddx, dL/ddy, one-pixel halo (0 where not interior)
    __shared__ float snv[3][kT][kT];            // the tile's n_d in the view frame (0 at border pixels)
    if (threadIdx.x == 0) dn_camera(view, proj, H, W, cam);
    const int tiles_x = (W + kT - 1) / kT, n_tiles = tiles_x * ((H + kT - 1) / kT);
    const size_t plane = (size_t)H * W;
    // torch's mean backward: the upstream scalar divided by the element count
    const float ge = __ldg(dL_dloss) / (float)((double)H * W);
    for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        const int x0 = (t % tiles_x) * kT, y0 = (t / tiles_x) * kT;
        for (int i = threadIdx.x; i < kD * kD; i += kThreads) {
            const int x = x0 - 2 + i % kD, y = y0 - 2 + i / kD;
            sd[i / kD][i % kD] = (x >= 0 && x < W && y >= 0 && y < H) ? __ldg(dn + (size_t)y * W + x) : 0.f;
        }
        __syncthreads();
        for (int i = threadIdx.x; i < kG * kG; i += kThreads) {
            const int gx = i % kG, gy = i / kG, x = x0 - 1 + gx, y = y0 - 1 + gy;
            float3 gdx = make_float3(0.f, 0.f, 0.f), gdy = gdx, nv = gdx;
            if (interior(x, y, H, W)) {
                const int lx = gx + 1, ly = gy + 1;     // position in sd
                const DnStencil s = stencil(cam, x, y, sd[ly - 1][lx], sd[ly + 1][lx], sd[ly][lx - 1], sd[ly][lx + 1]);
                const DnNormal n = rendered_normal(dn, plane, (size_t)y * W + x);
                // e = 1 - normal . nv: dL/dnv = -ge normal; nv = n_d @ V[:3,:3]: dL/dn_d = V[:3,:3] dL/dnv
                const float gnv[3] = {ge * n.a, ge * n.b, ge * n.s};
                float gn[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) gn[r] = cam.V[3 * r] * gnv[0] + cam.V[3 * r + 1] * gnv[1] + cam.V[3 * r + 2] * gnv[2];
                // n_d = v / max(|v|, eps): the quotient's part, plus the norm's where |v| >= eps (clamp_min's mask)
                float3 gv = make_float3(gn[0] / s.den, gn[1] / s.den, gn[2] / s.den);
                if (s.nrm >= kEps) {
                    const float gden = -(gn[0] * s.v.x + gn[1] * s.v.y + gn[2] * s.v.z) / (s.den * s.den);
                    const float k = gden / s.nrm;
                    gv.x += s.v.x * k; gv.y += s.v.y * k; gv.z += s.v.z * k;
                }
                gdx = cross3(s.dy, gv);                 // v = dx x dy
                gdy = cross3(gv, s.dx);
                nv = make_float3(s.nv[0], s.nv[1], s.nv[2]);
            }
            if (gx >= 1 && gx <= kT && gy >= 1 && gy <= kT) {
                snv[0][gy - 1][gx - 1] = nv.x; snv[1][gy - 1][gx - 1] = nv.y; snv[2][gy - 1][gx - 1] = nv.z;
            }
            sg[0][gy][gx] = gdx.x; sg[1][gy][gx] = gdx.y; sg[2][gy][gx] = gdx.z;
            sg[3][gy][gx] = gdy.x; sg[4][gy][gx] = gdy.y; sg[5][gy][gx] = gdy.z;
        }
        __syncthreads();
        const int tx = threadIdx.x % kT, ty = threadIdx.x / kT, x = x0 + tx, y = y0 + ty;
        if (x < W && y < H) {
            const size_t o = (size_t)y * W + x;
            // dx(r, c) = P(r+1, c) - P(r-1, c), dy(r, c) = P(r, c+1) - P(r, c-1); P = d ray (+ the origin, cancelled)
            const int gx = tx + 1, gy = ty + 1;
            float gp[3];
#pragma unroll
            for (int k = 0; k < 3; ++k)
                gp[k] = (sg[k][gy - 1][gx] - sg[k][gy + 1][gx]) + (sg[3 + k][gy][gx - 1] - sg[3 + k][gy][gx + 1]);
            const double3 ray = ray_at(cam, x, y);
            d_dn[o] = (float)(ray.x * gp[0] + ray.y * gp[1] + ray.z * gp[2]);
            // normal = (-a, -b, -sqrt(1 - clamp_max(a^2 + b^2, 1))); nv = 0 at border pixels
            const float nv[3] = {snv[0][ty][tx], snv[1][ty][tx], snv[2][ty][tx]};
            const DnNormal n = rendered_normal(dn, plane, o);
            const float g_s = ge * nv[2];                   // dL/ds = -dL/dnormal_z = ge nv_z
            const float g_u = g_s / (2.f * n.s);            // sqrt backward: inf (or NaN) at s = 0
            const float g_q = (n.q <= 1.f) ? -g_u : 0.f;    // u = 1 - clamp_max(q, 1): clamp passes q <= 1
            d_dn[plane + o] = ge * nv[0] + g_q * (2.f * n.a);
            d_dn[2 * plane + o] = ge * nv[1] + g_q * (2.f * n.b);
        }
        __syncthreads();
    }
}

// resident blocks only (two per SM): each derives the camera once and walks its tiles
int dn_grid(int H, int W) {
    const int tiles = ((W + kT - 1) / kT) * ((H + kT - 1) / kT);
    return tiles < 2 * sm_count() ? tiles : 2 * sm_count();
}

}  // namespace

cudaError_t launch_sugar_dn_features(int P, const float* points, const float* scaling, const float* quats,
                                     const float* view, const float* campos, float* feat, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    dn_features_kernel<<<(P + kThreads - 1) / kThreads, kThreads, 0, s>>>(
        P, points, scaling, reinterpret_cast<const float4*>(quats), view, campos, feat);
    count_launch();
    return cudaGetLastError();
}

cudaError_t launch_sugar_dn_features_bwd(int P, const float* points, const float* scaling, const float* quats,
                                         const float* view, const float* campos, const float* d_feat, float* d_points,
                                         float* d_quats, cudaStream_t s) {
    if (P == 0) return cudaSuccess;
    dn_features_bwd_kernel<<<(P + kThreads - 1) / kThreads, kThreads, 0, s>>>(
        P, points, scaling, reinterpret_cast<const float4*>(quats), view, campos, d_feat, d_points,
        reinterpret_cast<float4*>(d_quats));
    count_launch();
    return cudaGetLastError();
}

size_t sugar_dn_num_partials(int H, int W) { return (size_t)((W + kT - 1) / kT) * ((H + kT - 1) / kT); }

cudaError_t launch_sugar_dn_loss_fwd(const float* dn, int H, int W, const float* view, const float* proj,
                                     float* partials, float* loss, cudaStream_t s) {
    if (H < 3 || W < 3) {
        // every pixel is a border pixel: the mean of ones, without the stencil
        static const float kOne = 1.0f;
        return cudaMemcpyAsync(loss, &kOne, sizeof(float), cudaMemcpyHostToDevice, s);
    }
    dn_loss_fwd_kernel<<<dn_grid(H, W), kThreads, 0, s>>>(dn, H, W, view, proj, partials);
    count_launch();
    return launch_loss_reduce(partials, (int)sugar_dn_num_partials(H, W), 1.0f / (float)((double)H * W), loss, s);
}

cudaError_t launch_sugar_dn_loss_bwd(const float* dn, int H, int W, const float* view, const float* proj,
                                     const float* dL_dloss, float* d_dn, cudaStream_t s) {
    if (H < 3 || W < 3) return cudaMemsetAsync(d_dn, 0, sizeof(float) * 3 * (size_t)H * W, s);
    dn_loss_bwd_kernel<<<dn_grid(H, W), kThreads, 0, s>>>(dn, H, W, view, proj, dL_dloss, d_dn);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
