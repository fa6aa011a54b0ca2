// render_bwd.cu -- backward of the alpha compositing, warp-autonomous: one warp per 8x4-pixel sub-tile, no CTA barrier
// (staging 256-instance batches cooperatively was dominated by barrier stalls).
//
// Replaces renderCUDA<3> backward (DGR/cuda_rasterizer/backward.cu:399-557): back-to-front traversal from each
// pixel's last contributor, T recovered by division, gradients w.r.t. the per-Gaussian 2D mean, conic, opacity and
// colour.  Same formulas.  The reference issues 9 global float atomics per contributing PIXEL-Gaussian pair (its
// dominant cost); here a warp sums its 32 pixels' contributions before it touches the accumulators.  One kernel,
// render_bwd_t16_kernel, instruction-issue bound: it walks the sub-tile hit list the forward blend wrote, in blocks of
// 16 Gaussians, lane = Gaussian for the per-pair math, lane = pixel for the recurrences (kernel comment below).  Extra
// feature channels (fb200_extra) are its kExtra instance: they widen the per-pair dot product with dL/dpixel by the
// features' dot product with dL/dextra, and add one gradient sum per channel.
#include "common.cuh"

namespace fb200 {

namespace {

__device__ __forceinline__ P2 ldp(const float* a, int k) { return *reinterpret_cast<const float2*>(a + k); }

// ---- v4: transposed blocks -- lane = Gaussian for the per-pair math, lane = pixel for the recurrences --------------------
// A kernel that keeps lane = pixel throughout must sum every Gaussian's 9 partial gradients over the warp: a third of
// such a pair loop is the transposing butterfly (20 SHFL + 36 FSEL per two Gaussians; DESIGN.md §3.2).  Here the hits of
// a warp's 8x4 sub-tile are processed in blocks of 16 Gaussians and the work is split by what each part needs:
//   phase 1  lane = (Gaussian g, pixel half h): the lane evaluates ITS Gaussian at its 16 pixels, two pixels at a time on
//            pair operations -- same op order as the forward (power / libdevice exp / alpha tests, bit-identical decisions) --
//            and leaves three values per (Gaussian, pixel) in a padded shared-memory matrix: the masked opacity*G, the
//            1/(1-alpha) of the pair and alpha * (colour . dL/dpixel);
//   phase 2  lane = pixel: the only sequential part, the back-to-front recurrences, walks the 16 Gaussians of the block
//            for the lane's own pixel -- T <- T/(1-alpha), E <- E + alpha T (c . dL/dpix) -- two loads, four flops and two
//            stores per pair; the per-pixel state (T, E) lives in registers across blocks.  It leaves T_g and
//            U = (K - E_g)/(1-alpha) in place of the inputs, so that dL/dalpha = T_g (c . dL/dpix) + U
//            (backward.cu:509-534 with accum_rec kept un-normalised: T_g * accum_rec = E_g / (1 - alpha_g));
//   phase 3  lane = (g, h) again: gradient algebra for its Gaussian, accumulated over its 16 pixels IN REGISTERS as five
//            image moments of S = dL/dG * G (sum S dx, S dy, S dx^2, S dx dy, S dy^2), sum S / opacity-side and the three
//            colour sums; no cross-lane reduction except one xor-16 add per block.  9 red.global.add per Gaussian, as before.
// With extra channels (kExtra) c . dL/dpix becomes c . dL/dpix + e . dL/dextra throughout, K gains -T_final (bg_e .
// dL/dextra), and phase 3 adds one sum per channel (dL/de_c, accumulator slots 9..11).
// No shuffle and no select in the inner loops; the matrix rows are padded to 34 floats so that the 64-bit row accesses of
// phases 1/3 (lane stride = one row) and the 32-bit column accesses of phase 2 (lane stride = one word) are both
// bank-conflict free.
constexpr int kBlk = 16;            // Gaussians per block
constexpr int kRow = 34;            // padded row length (floats) of the [kBlk][32 pixels] matrices

struct __align__(16) BwdWarpSmem {
    float m0[kBlk * kRow];          // masked opacity * G                       (phase 1 -> phase 3)
    float m1[kBlk * kRow];          // 1 / (1 - alpha)  -> T_g                  (phase 1 -> 2 -> 3)
    float m2[kBlk * kRow];          // alpha * (c . dL/dpix)  -> U              (phase 1 -> 2 -> 3)
    float dp0[32], dp1[32], dp2[32], K[32];     // per pixel: dL/dpixel, K = -T_final * (bg . dL/dpixel)
    uint32_t last[32];                          // per pixel: entries of the hit list up to its last contributor
};
struct __align__(16) BwdWarpSmemX {            // kExtra only
    float de0[32], de1[32], de2[32];            // per pixel: dL/dextra (zero beyond ex.ch)
};

// The list a warp walks is its sub-tile's HIT LIST, written by the forward blend (render_fwd.cu): the Gaussian ids
// that passed the sub-tile test, in tile-list order, and per pixel the number of entries up to its last contributor.
// The backward therefore touches no instance the forward did not blend into this sub-tile: no re-test, no walk over
// the other 7/8 of the tile list, and the per-pixel "before my last contributor" test is a compare of entry numbers.
// Colour only: 20 resident warps per SM, 96 registers, no spills (24 warps at 80 registers measured slower).
// Extra channels: 16 resident warps per SM, which leaves room for the extra registers without spills.
template <int kWarps, bool kExtra>
__global__ void __launch_bounds__(32 * kWarps, (kExtra ? 16 : 20) / kWarps)
render_bwd_t16_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ sub_hits,
                      const SplatRec* __restrict__ rec, int W, int H, int tiles_x,
                      const float* __restrict__ bg, const float* __restrict__ final_T,
                      const uint32_t* __restrict__ last_entry, const float* __restrict__ dL_dpix,
                      float* __restrict__ acc, const int32_t* __restrict__ status, const ExtraArgs ex,
                      const uint32_t* __restrict__ tile_order) {
    __shared__ BwdWarpSmem smem[kWarps];
    __shared__ BwdWarpSmemX smem_x[kExtra ? kWarps : 1];
    if (status[FB200_ST_OVERFLOW]) return;

    const unsigned full = 0xffffffffu;
    constexpr int kSplit = kWarpsPerTile / kWarps;
    const int tile = (int)tile_order[blockIdx.x / kSplit];       // longest lists first (binning.cu)
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const int wslot = threadIdx.x >> 5;
    const int warp = (blockIdx.x % kSplit) * kWarps + wslot;      // sub-tile index inside the tile
    int lane;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(lane));
    BwdWarpSmem& sm = smem[wslot];
    BwdWarpSmemX& smx = smem_x[kExtra ? wslot : 0];
    const int sub_x0 = tile_x * kTile + (warp & 1) * kSubW;
    const int sub_y0 = tile_y * kTile + (warp >> 1) * kSubH;
    const uint2 range = ranges[tile];
    const uint32_t* const sub = sub_hits + (size_t)kWarpsPerTile * range.x + (size_t)warp * (range.y - range.x);

    // ---- lane = pixel: the lane's own pixel, its recurrence state and its row of the per-pixel constants ----
    float T, E = 0.f, Kp;
    int top;                        // entries [0, top) of the hit list are still to be processed
    {
        const int pix_x = sub_x0 + (lane & 7), pix_y = sub_y0 + (lane >> 3);
        const bool inside = pix_x < W && pix_y < H;
        const size_t pix_id = (size_t)pix_y * W + pix_x;
        const size_t HW = (size_t)H * W;
        const float T_final = inside ? final_T[pix_id] : 0.f;
        const uint32_t le = inside ? last_entry[pix_id] : 0u;
        float dp0 = 0.f, dp1 = 0.f, dp2 = 0.f;
        if (inside) {
            dp0 = dL_dpix[pix_id];
            dp1 = dL_dpix[HW + pix_id];
            dp2 = dL_dpix[2 * HW + pix_id];
        }
        float bg_dot = bg[0] * dp0 + bg[1] * dp1 + bg[2] * dp2;
        if (kExtra) {
            float de0 = 0.f, de1 = 0.f, de2 = 0.f;
            if (inside) {
                de0 = ex.dL_dout[pix_id];
                if (ex.ch > 1) de1 = ex.dL_dout[HW + pix_id];
                if (ex.ch > 2) de2 = ex.dL_dout[2 * HW + pix_id];
            }
            bg_dot += ex.bg[0] * de0;
            if (ex.ch > 1) bg_dot += ex.bg[1] * de1;
            if (ex.ch > 2) bg_dot += ex.bg[2] * de2;
            smx.de0[lane] = de0; smx.de1[lane] = de1; smx.de2[lane] = de2;
        }
        Kp = -T_final * bg_dot;
        T = T_final;
        sm.dp0[lane] = dp0; sm.dp1[lane] = dp1; sm.dp2[lane] = dp2; sm.K[lane] = Kp; sm.last[lane] = le;
        top = (int)__reduce_max_sync(full, le);
    }
    if (top == 0) return;
    __syncwarp();
    // Pixel-pair slot k (0..7) of phases 1 / 3 covers pixels {2k, 2k+1} of the upper half and {16+2k, 16+2k+1} of the
    // lower half at once.  pair_last[k] = the largest "last entry" among those four pixels: a block whose entries all lie
    // at or beyond it has nothing to do in slot k.  Deep in a list only the few pixels that never saturated are still
    // live, so most slots are skipped there (C2 / C5: most of the walk).
    uint32_t pair_last;
    {
        const int k = lane & 7;
        pair_last = max(max(sm.last[2 * k], sm.last[2 * k + 1]), max(sm.last[16 + 2 * k], sm.last[17 + 2 * k]));
    }

    // ---- lane = (Gaussian g, pixel half h): rows 2h, 2h+1 of the 8x4 sub-tile ----
    const int g = lane & (kBlk - 1), h = lane >> 4;
    const float ddelx_dx = 0.5f * W, ddely_dy = 0.5f * H;
    const float px0 = (float)sub_x0;
    const float py0 = (float)(sub_y0 + 2 * h);
    float* const row0 = sm.m0 + g * kRow + 16 * h;
    float* const row1 = sm.m1 + g * kRow + 16 * h;
    float* const row2 = sm.m2 + g * kRow + 16 * h;
    const float* const pdp0 = sm.dp0 + 16 * h;
    const float* const pdp1 = sm.dp1 + 16 * h;
    const float* const pdp2 = sm.dp2 + 16 * h;
    const uint32_t* const plast = sm.last + 16 * h;
    const float* const pde0 = smx.de0 + 16 * h;
    const float* const pde1 = smx.de1 + 16 * h;
    const float* const pde2 = smx.de2 + 16 * h;

    // Register prefetch, two stages deep: the Gaussian ids of block k+2 and the records of block k+1 are requested while
    // block k is processed, so neither hop of the dependent chain id -> record is waited for (without it, the id load
    // at the top of every block was the largest stall).  Staging the records with one 48-byte cp.async.bulk each into a
    // 4-deep shared-memory ring, 3 blocks ahead, was slower: 16 small bulk copies per block per warp exceed what the
    // SM's TMA unit issues and the warps spin on the mbarriers.
    auto load_id = [&](int t) -> uint32_t {       // entry t-1-g of the list, 0 if beyond its start
        const int e = t - 1 - g;
        return e >= 0 ? __ldg(sub + e) : 0u;
    };
    uint32_t nid = load_id(top), nnid = load_id(top - kBlk);
    float4 n0, n1, n2;
    n0 = n1 = n2 = make_float4(0.f, 0.f, 0.f, 0.f);
    float nf0 = 0.f, nf1 = 0.f, nf2 = 0.f;        // extra features, prefetched with the record
    auto fetch_rec = [&](uint32_t id, int t) {    // records of the block whose top is t
        if (t - 1 - g >= 0) {
            const float4* p = reinterpret_cast<const float4*>(rec + id);
            n0 = __ldg(p); n1 = __ldg(p + 1); n2 = __ldg(p + 2);
            if (kExtra) {
                const float* f = ex.feat + (size_t)id * ex.ch;
                nf0 = __ldg(f);
                if (ex.ch > 1) nf1 = __ldg(f + 1);
                if (ex.ch > 2) nf2 = __ldg(f + 2);
            }
        }
    };
    fetch_rec(nid, top);

    while (top > 0) {
        const int cnt = min(kBlk, top);
        const bool valid = g < cnt;
        const uint32_t entry = (uint32_t)(top - 1 - g);          // this Gaussian's entry number (valid lanes)
        const float X = n0.x, Y = n0.y, A = n0.z, B = n0.w, Cc = n1.x;
        const float op = valid ? n1.y : 0.f;
        const float cr = valid ? n1.z : 0.f, cg = valid ? n1.w : 0.f, cb = valid ? n2.x : 0.f;
        const float f0 = valid ? nf0 : 0.f, f1 = valid ? nf1 : 0.f, f2 = valid ? nf2 : 0.f;
        const uint32_t gid = nid;
        top -= cnt;
        nid = nnid;
        fetch_rec(nid, top);                  // next block's records (its ids arrived a block ago)
        nnid = load_id(top - kBlk);           // ids of the block after that
        // ---- phase 1: alpha of (Gaussian g) x (up to 16 pixels), the forward's op order ----
        // slots that can hold a contributing pixel for some entry of this block (entries [top, top + cnt) after the update)
        const unsigned slots = __ballot_sync(full, pair_last > (uint32_t)top) & 0xffu;
        bool any_act = false;
        unsigned my_slots = 0;          // slots where THIS lane found a contributing pixel
        auto phase1 = [&](int r, int c) {
            const float dy = fadd(Y, -(py0 + (float)r));
            const float dyC = fmul(dy, fmul(dy, Cc));
            const int k = 8 * r + 2 * c;                                   // pixel pair (k, k+1) of this half
            const P2 dx = add2(bc(X), p2(-(px0 + (float)(2 * c)), -(px0 + (float)(2 * c + 1))));
            const P2 q = fma2(dx, mul2(dx, bc(A)), bc(dyC));
            const P2 u = mul2(bc(dy), mul2(dx, bc(B)));
            const P2 power = fma2(q, bc(-0.5f), neg2(u));
            const P2 og = mul2(bc(op), exp_pair(power));
            const uint2 lastp = *reinterpret_cast<const uint2*>(plast + k);
            // contributes iff the forward blended it: not beyond the pixel's last contributor, power <= 0,
            // alpha >= 1/255 (min(0.99, og) < 1/255  <=>  og < 1/255)
            const bool a0 = valid && (entry < lastp.x) && !(power.x > 0.0f) && !(og.x < 1.0f / 255.0f);
            const bool a1 = valid && (entry < lastp.y) && !(power.y > 0.0f) && !(og.y < 1.0f / 255.0f);
            any_act |= a0 | a1;
            my_slots |= (a0 | a1) ? (1u << (4 * r + c)) : 0u;
            const P2 ogm = p2(a0 ? og.x : 0.f, a1 ? og.y : 0.f);
            const P2 am = p2(fminf(0.99f, ogm.x), fminf(0.99f, ogm.y));
            const P2 om = add2(bc(1.0f), neg2(am));                        // 1 - alpha in [0.01, 1]
            P2 inv;
            {
                float i0, i1;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(i0) : "f"(om.x));
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(i1) : "f"(om.y));
                const P2 rr = p2(i0, i1);
                inv = fma2(rr, fma2(neg2(om), rr, bc(1.0f)), rr);          // one Newton step
            }
            P2 cd = fma2(ldp(pdp0, k), bc(cr), fma2(ldp(pdp1, k), bc(cg), mul2(ldp(pdp2, k), bc(cb))));
            if (kExtra) cd = fma2(ldp(pde0, k), bc(f0), fma2(ldp(pde1, k), bc(f1), fma2(ldp(pde2, k), bc(f2), cd)));
            *reinterpret_cast<float2*>(row0 + k) = ogm;
            *reinterpret_cast<float2*>(row1 + k) = inv;
            *reinterpret_cast<float2*>(row2 + k) = mul2(am, cd);
        };
        if (slots == 0xffu) {
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) phase1(r, c);
        } else {
            // skipped slots keep whatever an earlier block left in the matrices: make them identities for phase 2
            for (unsigned todo = ~slots & 0xffu; todo; todo &= todo - 1) {
                const int sl = __ffs(todo) - 1, k = 8 * (sl >> 2) + 2 * (sl & 3);
                *reinterpret_cast<float2*>(row1 + k) = make_float2(1.f, 1.f);
                *reinterpret_cast<float2*>(row2 + k) = make_float2(0.f, 0.f);
            }
            for (unsigned todo = slots; todo; todo &= todo - 1) {
                const int sl = __ffs(todo) - 1;
                phase1(sl >> 2, sl & 3);
            }
        }
        // Gaussians of the block with at least one contributing pixel (either half); the others are identities for the
        // recurrences and add nothing to any sum
        const unsigned act_bits = __ballot_sync(full, any_act);
        const unsigned act16 = (act_bits | (act_bits >> 16)) & 0xffffu;
        if (act16 == 0) continue;
        __syncwarp();                  // phase 1's stores before phase 2's loads
        // ---- phase 2: lane = pixel, back-to-front recurrences over the block's Gaussians ----
        {
            float* c1 = sm.m1 + lane;
            float* c2 = sm.m2 + lane;
            if (__popc(act16) + 2 >= cnt) {
                // dense block: walk every row (inactive rows are identities: inv = 1, bb = 0), loads four deep
#pragma unroll 4
                for (int i = 0; i < cnt; ++i) {
                    const float inv = c1[i * kRow], bb = c2[i * kRow];
                    const float Tg = T * inv;                  // transmittance in front of Gaussian i at this pixel
                    c1[i * kRow] = Tg;
                    c2[i * kRow] = (Kp - E) * inv;             // U: everything behind it (and the background) seen through it
                    E = fmaf(bb, Tg, E);
                    T = Tg;
                }
            } else {
                for (unsigned todo = act16; todo; todo &= todo - 1) {
                    const int i = __ffs(todo) - 1;
                    const float inv = c1[i * kRow], bb = c2[i * kRow];
                    const float Tg = T * inv;
                    c1[i * kRow] = Tg;
                    c2[i * kRow] = (Kp - E) * inv;
                    E = fmaf(bb, Tg, E);
                    T = Tg;
                }
            }
        }
        __syncwarp();
        // ---- phase 3: gradient sums of Gaussian g over its 16 pixels ----
        const float rop = op > 0.f ? __frcp_rn(op) : 0.f;
        P2 sR = bc(0.f), sG = bc(0.f), sB = bc(0.f), sO = bc(0.f);
        P2 M10 = bc(0.f), M01 = bc(0.f), M20 = bc(0.f), M11 = bc(0.f), M02 = bc(0.f);
        P2 sE0 = bc(0.f), sE1 = bc(0.f), sE2 = bc(0.f);                    // kExtra: dL/d(extra feature c)
        auto phase3 = [&](int r, int c) {
            const float dy = fadd(Y, -(py0 + (float)r));
            const int k = 8 * r + 2 * c;
            const P2 dx = add2(bc(X), p2(-(px0 + (float)(2 * c)), -(px0 + (float)(2 * c + 1))));
            const P2 ogm = ldp(row0, k), Tg = ldp(row1, k), U = ldp(row2, k);
            const P2 d0 = ldp(pdp0, k), d1 = ldp(pdp1, k), d2 = ldp(pdp2, k);
            const P2 am = p2(fminf(0.99f, ogm.x), fminf(0.99f, ogm.y));
            const P2 Gm = mul2(ogm, bc(rop));                               // G (0 where the pair does not contribute)
            P2 cd = fma2(d0, bc(cr), fma2(d1, bc(cg), mul2(d2, bc(cb))));
            const P2 dch = mul2(am, Tg);                                   // d(pixel channel)/d(colour)
            sR = fma2(dch, d0, sR); sG = fma2(dch, d1, sG); sB = fma2(dch, d2, sB);
            if (kExtra) {
                const P2 e0 = ldp(pde0, k), e1 = ldp(pde1, k), e2 = ldp(pde2, k);
                cd = fma2(e0, bc(f0), fma2(e1, bc(f1), fma2(e2, bc(f2), cd)));
                sE0 = fma2(dch, e0, sE0); sE1 = fma2(dch, e1, sE1); sE2 = fma2(dch, e2, sE2);
            }
            const P2 dLa = fma2(Tg, cd, U);                                // dL/dalpha
            const P2 S = mul2(dLa, Gm);                                    // dL/dopacity contribution
            sO = add2(sO, S);
            const P2 SG = mul2(S, bc(op));                                 // dL/dG * G
            const P2 sx = mul2(SG, dx), sy = mul2(SG, bc(dy));
            M10 = add2(M10, sx); M01 = add2(M01, sy);
            M20 = fma2(sx, dx, M20); M11 = fma2(sx, bc(dy), M11); M02 = fma2(sy, bc(dy), M02);
        };
        // only the slots where some lane found a contributing pixel carry anything
        const unsigned live_slots = __reduce_or_sync(full, my_slots);
        if (live_slots == 0xffu) {
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) phase3(r, c);
        } else {
            for (unsigned todo = live_slots; todo; todo &= todo - 1) {
                const int sl = __ffs(todo) - 1;
                phase3(sl >> 2, sl & 3);
            }
        }
        constexpr int kSums = kExtra ? 12 : 9;
        float v[kSums] = {M10.x + M10.y, M01.x + M01.y, M20.x + M20.y, M11.x + M11.y, M02.x + M02.y,
                          sO.x + sO.y, sR.x + sR.y, sG.x + sG.y, sB.x + sB.y};
        if constexpr (kExtra) { v[9] = sE0.x + sE0.y; v[10] = sE1.x + sE1.y; v[11] = sE2.x + sE2.y; }
#pragma unroll
        for (int i = 0; i < kSums; ++i) v[i] += __shfl_xor_sync(full, v[i], 16);
        if (h == 0 && ((act16 >> g) & 1u)) {
            float* a = acc + (size_t)gid * 12;
            // dG/ddelx = -G (dx A + dy B), dG/ddely = -G (dy C + dx B)   (backward.cu:536-546)
            // two 128-bit vector reductions + one scalar (red.global.add.v4.f32, sm_90+): a third of the L2 atomic
            // transactions of nine scalar ones -- neighbouring sub-tiles hit the same 48-byte accumulator records
            atomicAdd(reinterpret_cast<float4*>(a),
                      make_float4(-ddelx_dx * fmaf(A, v[0], B * v[1]), -ddely_dy * fmaf(Cc, v[1], B * v[0]),
                                  -0.5f * v[2], -0.5f * v[3]));
            atomicAdd(reinterpret_cast<float4*>(a) + 1, make_float4(-0.5f * v[4], v[5], v[6], v[7]));
            if constexpr (kExtra)     // slots 8..11: {db, dL/dextra}, 16-byte aligned like the other two
                atomicAdd(reinterpret_cast<float4*>(a) + 2, make_float4(v[8], v[9], v[10], v[11]));
            else
                atomicAdd(a + 8, v[8]);
        }
        __syncwarp();      // the matrices are rewritten by the next block
    }
}

}  // namespace

cudaError_t launch_render_bwd_clear(const BwdArgs& a, cudaStream_t s) {
    return cudaMemsetAsync(a.acc, 0, sizeof(float) * 12 * (size_t)a.prm.P, s);
}

cudaError_t launch_render_bwd(const BwdArgs& a, cudaStream_t s) {
    const int T = a.tiles_x * a.tiles_y;
    constexpr int kWarps = 4;   // 4-warp CTAs (half tiles): a CTA slot frees as soon as its half is done; beat 8 and 2 on C3
    const int grid = T * (kWarpsPerTile / kWarps);
    count_launch();
    const auto kernel = a.ex.ch > 0 ? render_bwd_t16_kernel<kWarps, true> : render_bwd_t16_kernel<kWarps, false>;
    kernel<<<grid, 32 * kWarps, 0, s>>>(
        a.ranges, a.sub_hits, a.rec, a.prm.image_width, a.prm.image_height, a.tiles_x, a.in.d_background,
        a.final_T, a.last_entry, a.dL_dpix, a.acc, a.status, a.ex, a.tile_order);
    return cudaGetLastError();
}

namespace {
// dL/d(extra features): slots 9..11 of the accumulator record, zero for Gaussians that were not rendered
__global__ void __launch_bounds__(256)
extra_grad_kernel(int P, int ch, const int32_t* __restrict__ radii, const float* __restrict__ acc,
                  float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const bool vis = radii[i] > 0;
    for (int c = 0; c < ch; ++c) out[(size_t)i * ch + c] = vis ? acc[(size_t)i * 12 + 9 + c] : 0.f;
}
}  // namespace

cudaError_t launch_extra_grad(const BwdArgs& a, cudaStream_t s) {
    if (a.ex.ch <= 0 || a.prm.P <= 0) return cudaSuccess;
    extra_grad_kernel<<<(a.prm.P + 255) / 256, 256, 0, s>>>(a.prm.P, a.ex.ch, a.radii, a.acc, a.ex.dL_dfeat);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
