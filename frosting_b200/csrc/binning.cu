// binning.cu -- per-tile binning and depth sort.
//
// Replaces, with identical results, the reference's
//   cub::DeviceScan::InclusiveSum + D2H copy   (DGR/cuda_rasterizer/rasterizer_impl.cu:277-281)
//   duplicateWithKeys                          (rasterizer_impl.cu:70-111)
//   cub::DeviceRadixSort::SortPairs on 32+bit  (rasterizer_impl.cu:300-308)
//   identifyTileRanges                         (rasterizer_impl.cu:116-138)
//
// The reference sorts R 64-bit (tile | depth_bits) keys globally with a stable LSD radix sort, so
// within a tile instances are ordered by depth bits and, for equal depths, by emission order =
// ascending Gaussian index.  Here the per-tile instance counts are already known from preprocess,
// so the tile ranges come from one scan over T tiles, instances are scattered straight into their
// tile's segment, and each segment is sorted in shared memory by the 64-bit key
// (depth_bits << 32 | gaussian_index) -- a total order that equals the reference's stable order.
// Global traffic: 8 B written + 8 B read + 4 B written per instance instead of ~150 B/instance for
// a 6-pass global radix sort.
#include <mutex>

#include "common.cuh"

namespace fb200 {

namespace {

typedef unsigned long long u64;

// ---- tile scan: counts -> ranges, cursors, sort work lists, status ---------------------------------
// One CTA (the host is waiting for the instance count this kernel produces, so it is latency that matters):
// the counts are staged in shared memory with coalesced loads, each thread then owns a contiguous run of tiles.
constexpr int kScanStage = 10240;   // tiles staged in shared memory (40 KB); larger grids read global memory twice

__global__ void __launch_bounds__(1024)
tile_scan_kernel(int T, const uint32_t* __restrict__ tile_count, uint2* __restrict__ ranges,
                 uint32_t* __restrict__ cursor, uint32_t* __restrict__ list_tiny, uint32_t* __restrict__ list_small,
                 uint32_t* __restrict__ list_large, uint32_t* __restrict__ list_huge,
                 uint32_t* __restrict__ counters, long long capacity, int32_t* __restrict__ status,
                 uint32_t* __restrict__ order) {
    __shared__ uint32_t staged[kScanStage];
    __shared__ uint32_t s_bucket[40];
    __shared__ uint32_t warp_sums[32];
    __shared__ u64 cls_sums[2][32];
    __shared__ u64 cls_total[2];
    __shared__ uint32_t s_max;
    const int tid = threadIdx.x;
    if (tid == 0) s_max = 0;
    const bool use_stage = T <= kScanStage;
    if (use_stage)
        for (int t = tid; t < T; t += 1024) staged[t] = tile_count[t];
    __syncthreads();
    const uint32_t* cnt = use_stage ? staged : tile_count;
    const int per = (T + 1023) / 1024;
    const int begin = min(T, tid * per), end = min(T, begin + per);
    uint32_t local = 0, lmax = 0;
    for (int t = begin; t < end; ++t) {
        uint32_t c = cnt[t];
        local += c;
        lmax = max(lmax, c);
    }
    // block exclusive scan of `local`
    const uint32_t incl = warp_inclusive_scan(local, tid & 31);
    if ((tid & 31) == 31) warp_sums[tid >> 5] = incl;
    __syncthreads();
    if (tid < 32) {
        const uint32_t w = warp_sums[tid];
        warp_sums[tid] = warp_inclusive_scan(w, tid) - w;   // exclusive
    }
    __syncthreads();
    uint32_t run = warp_sums[tid >> 5] + incl - local;
    // work-list slots come from a second block scan (per-thread counts of the four classes, two per 64-bit word)
    // instead of shared-memory atomics: 8 k returning atomics on four addresses serialise to ~30 k cycles
    u64 cls_a = 0, cls_b = 0;     // (tiny | small << 32), (large | huge << 32)
    for (int t = begin; t < end; ++t) {
        const uint32_t c = cnt[t];
        if (c >= 1) {
            if (c <= (uint32_t)kSortTinyMax) cls_a += 1ull;
            else if (c <= (uint32_t)kSortSmallMax) cls_a += 1ull << 32;
            else if (c <= (uint32_t)kSortMediumMax) cls_b += 1ull;
            else cls_b += 1ull << 32;
        }
    }
    const u64 inc_a = warp_inclusive_scan(cls_a, tid & 31), inc_b = warp_inclusive_scan(cls_b, tid & 31);
    __syncthreads();                 // warp_sums is reused below
    if ((tid & 31) == 31) { cls_sums[0][tid >> 5] = inc_a; cls_sums[1][tid >> 5] = inc_b; }
    __syncthreads();
    if (tid < 32) {
        const u64 wa = cls_sums[0][tid], wb = cls_sums[1][tid];
        const u64 ia = warp_inclusive_scan(wa, tid), ib = warp_inclusive_scan(wb, tid);
        cls_sums[0][tid] = ia - wa;
        cls_sums[1][tid] = ib - wb;
        if (tid == 31) { cls_total[0] = ia; cls_total[1] = ib; }
    }
    __syncthreads();
    const u64 ex_a = cls_sums[0][tid >> 5] + inc_a - cls_a, ex_b = cls_sums[1][tid >> 5] + inc_b - cls_b;
    uint32_t at_tiny = (uint32_t)ex_a, at_small = (uint32_t)(ex_a >> 32);
    uint32_t at_large = (uint32_t)ex_b, at_huge = (uint32_t)(ex_b >> 32);
    for (int t = begin; t < end; ++t) {
        uint32_t c = cnt[t];
        // untouched tiles keep (0,0) exactly like the reference's memset + identifyTileRanges
        ranges[t] = c ? make_uint2(run, run + c) : make_uint2(0u, 0u);
        cursor[t] = run;
        if (c >= 1) {
            if (c <= (uint32_t)kSortTinyMax) list_tiny[at_tiny++] = t;
            else if (c <= (uint32_t)kSortSmallMax) list_small[at_small++] = t;
            else if (c <= (uint32_t)kSortMediumMax) list_large[at_large++] = t;
            else list_huge[at_huge++] = t;
        }
        run += c;
    }
    atomicMax(&s_max, lmax);
    // ---- launch order of the blend kernels: longest lists first ----
    // A tile's blend time grows with its list length and tiles differ by 10-100x; CTAs are dispatched in blockIdx order,
    // so raster order leaves the SMs that drew a long tile late running alone at the end.  order[] lists the tiles by
    // descending size class (power-of-two buckets of the instance count; empty tiles last): the classic longest-
    // processing-time-first heuristic, at the cost of one warp-aggregated counting pass here.
    if (tid < 40) s_bucket[tid] = 0;
    __syncthreads();
    auto bucket_of = [](uint32_t c) { return c ? 31 - (32 - __clz(c)) : 32; };       // big lists -> small bucket index
    // one tile per lane; lanes of a warp that share a bucket are counted / placed with ONE shared-memory atomic
    // (8 k atomics on ~6 addresses serialise to tens of microseconds otherwise)
    const unsigned lanemask_lt = (1u << (tid & 31)) - 1u;
    for (int t0 = tid; t0 < ((T + 31) & ~31); t0 += 1024) {
        const bool have = t0 < T;
        const int b = have ? bucket_of(cnt[t0]) : 33;
        const unsigned peers = __match_any_sync(0xffffffffu, b);
        if (have && (peers & lanemask_lt) == 0) atomicAdd(&s_bucket[b], (uint32_t)__popc(peers));
    }
    __syncthreads();
    if (tid == 0) {
        uint32_t run_b = 0;
        for (int b = 0; b <= 32; ++b) { const uint32_t c = s_bucket[b]; s_bucket[b] = run_b; run_b += c; }
    }
    __syncthreads();
    // Inside a size class the tiles are emitted in a SCATTERED order (index * odd constant mod 2^k): neighbouring tiles
    // share Gaussians, and running them at the same moment makes the backward's gradient atomics collide
    int kbits = 0;
    while ((1 << kbits) < T) ++kbits;
    const uint32_t kmask = (1u << kbits) - 1u;
    for (uint32_t i = (uint32_t)tid; i < (1u << kbits) || (i & ~31u) < (1u << kbits); i += 1024) {
        const uint32_t t0 = (i * 0x9E3779B1u) & kmask;
        const bool have = i < (1u << kbits) && t0 < (uint32_t)T;
        const int b = have ? bucket_of(cnt[t0]) : 33;
        const unsigned peers = __match_any_sync(0xffffffffu, b);
        uint32_t base_b = 0;
        const int leader = __ffs(peers) - 1;
        if (have && (peers & lanemask_lt) == 0) base_b = atomicAdd(&s_bucket[b], (uint32_t)__popc(peers));
        base_b = __shfl_sync(0xffffffffu, base_b, leader);
        if (have) order[base_b + __popc(peers & lanemask_lt)] = t0;
    }
    __syncthreads();
    if (tid == 1023) {
        // the instance count is reported as a non-negative int32: anything beyond that is an overflow whatever the capacity
        status[FB200_ST_NUM_RENDERED] = run > 0x7fffffffu ? 0x7fffffff : (int32_t)run;
        status[FB200_ST_OVERFLOW] = ((long long)run > capacity || run > 0x7fffffffu) ? 1 : 0;
        status[FB200_ST_MAX_TILE] = (int32_t)s_max;
        status[FB200_ST_NUM_VISIBLE] = (int32_t)counters[3];   // counted by preprocess (Gaussians with radii > 0)
    }
    if (tid == 0) {
        counters[4] = (uint32_t)cls_total[0];            // tiny
        counters[0] = (uint32_t)(cls_total[0] >> 32);    // small
        counters[1] = (uint32_t)cls_total[1];            // large
        counters[2] = (uint32_t)(cls_total[1] >> 32);    // huge
    }
}

// ---- scatter: one (depth_bits<<32 | idx) key per (Gaussian, tile) into the tile's segment ----------
// Warp-balanced expansion: a warp owns 32 consecutive Gaussians, scans their tile counts and then walks
// the concatenated instance list 32 instances at a time, so a splat covering 1000 tiles costs the warp
// 32 steps instead of stalling one lane for 1000 dependent atomic round trips (the reference's
// duplicateWithKeys has the same per-thread double loop, rasterizer_impl.cu:98-108).
__global__ void __launch_bounds__(256)
scatter_kernel(int P, int tiles_x, const uint2* __restrict__ rect, const float* __restrict__ depth,
               uint32_t* __restrict__ cursor, u64* __restrict__ keys, const int32_t* __restrict__ status) {
    if (status[FB200_ST_OVERFLOW]) return;
    const unsigned full = 0xffffffffu;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    uint32_t minx = 0, miny = 0, w = 0, n = 0, dbits = 0;
    if (idx < P) {
        const uint2 r = rect[idx];
        minx = r.x & 0xffffu; miny = r.x >> 16;
        const uint32_t maxx = r.y & 0xffffu, maxy = r.y >> 16;
        if (maxx > minx && maxy > miny) {
            w = maxx - minx;
            n = w * (maxy - miny);
            dbits = __float_as_uint(depth[idx]);
        }
    }
    const uint32_t incl = warp_inclusive_scan(n, lane);
    const uint32_t excl = incl - n;
    const uint32_t total = __shfl_sync(full, incl, 31);
    for (uint32_t base = 0; base < total; base += 32) {
        const uint32_t item = base + lane;
        const int owner = warp_expand_owner(incl, item);
        const uint32_t o_excl = __shfl_sync(full, excl, owner);
        const uint32_t o_minx = __shfl_sync(full, minx, owner);
        const uint32_t o_miny = __shfl_sync(full, miny, owner);
        const uint32_t o_w = __shfl_sync(full, w, owner);
        const uint32_t o_d = __shfl_sync(full, dbits, owner);
        if (item < total) {
            const uint32_t k = item - o_excl;
            const uint32_t ty = o_miny + k / o_w, tx = o_minx + k % o_w;
            const uint32_t gidx = (uint32_t)(idx - lane + owner);
            const uint32_t slot = atomicAdd(cursor + ty * tiles_x + tx, 1u);
            keys[slot] = ((u64)o_d << 32) | gidx;
        }
    }
}

// ---- per-tile sort ----------------------------------------------------------------------------------
// Each tile's list is sorted by the 64-bit key (depth_bits << 32 | gaussian_idx).  The keys of a tile are unique, so
// every correct sort gives the same bits: the reference's stable order.  The shared-memory classes run the bucket sort
// and fall back to the radix sort when a bucket is too full; the global-memory class runs the radix sort alone.  Both
// sorts are written once for a warp (kThreads = 32, __syncwarp only) and for a CTA; t is the thread's index in it.
template <int kThreads>
__device__ __forceinline__ void scope_sync() {
    if (kThreads == 32) __syncwarp(); else __syncthreads();
}

// insertion sort of b[lo, hi) on the full key
__device__ __forceinline__ void insertion_sort(u64* b, int lo, int hi) {
    for (int x = lo + 1; x < hi; ++x) {
        const u64 kx = b[x];
        int y = x - 1;
        while (y >= lo && b[y] > kx) { b[y + 1] = b[y]; --y; }
        b[y + 1] = kx;
    }
}

// Lanes holding the same 8-bit digit as this lane, among the lanes with `have` set: eight ballots and eight
// LOP3s at fixed latency.  (__match_any_sync does the same in one instruction, but its latency grows with
// the number of distinct values -- with 32 near-random digits it dominated this kernel: ~98 k cycles per
// 1.5 k-key tile.)
__device__ __forceinline__ unsigned digit_peers(uint32_t d, bool have) {
    const unsigned full = 0xffffffffu;
    unsigned peers = __ballot_sync(full, have);
#pragma unroll
    for (int b = 0; b < 8; ++b) {
        const bool bit = (d >> b) & 1u;
        const unsigned bal = __ballot_sync(full, bit);
        peers &= bit ? bal : ~bal;
    }
    return peers;
}

// ---- radix sort -----------------------------------------------------------------------------------------------------
// Stable LSD radix sort of one tile's keys on the 32 depth bits (4 passes of 8 bits; a pass whose digit
// is the same for every key is skipped), followed by a fix-up that orders runs of EQUAL depth by
// Gaussian index -- together the total order (depth_bits, idx) of the reference's stable global sort.
// Ranking is warp-synchronous: each warp owns a contiguous slice of the list, walks it 32 keys at a
// time and ranks equal digits with ballots (digit_peers), so no per-key shared-memory atomics are needed.
// Sorts src[0, n) with dst as the other ping-pong buffer, both in shared memory or, for lists of any length, in global
// memory (L2); returns the buffer holding the result.
// counters: (kThreads / 32) * 256 words, one digit histogram per warp; s_misc: 1 + min(kThreads, 256) / 32 words.
template <int kThreads>
// NOTE: no __restrict__ on any of these pointers -- they are written by other threads of the CTA and
// re-read after barriers; with __restrict__ nvcc forwards a thread's own stale store across
// __syncthreads() (observed: s_misc[0] kept in a register, threads disagreeing on `skip`, deadlock).
__device__ __forceinline__ u64* radix_sort(u64* src, u64* dst, int n, uint32_t* counters, volatile uint32_t* s_misc,
                                           int t) {
    constexpr int kWarps = kThreads / 32;
    constexpr int kOwners = kThreads < 256 ? kThreads : 256;    // step 2: thread t < kOwners owns kPer digits
    constexpr int kPer = 256 / kOwners;
    const int warp = t >> 5, lane = t & 31;
    // contiguous slice per warp, multiple of 32; the whole list at warp scope, spelled out (with the general bounds,
    // ptxas re-reads the shared-memory window base for every key of the tiny kernel's bucket insertion loop)
    const int seg = (((n + kWarps - 1) / kWarps) + 31) & ~31;
    const int seg_lo = kWarps == 1 ? 0 : min(n, warp * seg), seg_hi = kWarps == 1 ? n : min(n, seg_lo + seg);
    for (int shift = 32; shift < 64; shift += 8) {
        for (int i = t; i < kWarps * 256; i += kThreads) counters[i] = 0;
        if (t == 0) s_misc[0] = 0;
        scope_sync<kThreads>();
        // 1. per-warp digit histogram of its slice
        for (int i0 = seg_lo; i0 < seg_hi; i0 += 32) {
            const int i = i0 + lane;
            const bool have = i < seg_hi;
            const uint32_t d = have ? (uint32_t)(src[i] >> shift) & 0xffu : 0u;
            const unsigned peers = digit_peers(d, have);
            if (have && (__ffs(peers) - 1) == lane) counters[warp * 256 + d] += __popc(peers);
            __syncwarp();
        }
        scope_sync<kThreads>();
        // 2. digit totals, uniform-digit test, exclusive offsets per (digit, warp)
        uint32_t tot = 0;
        if (t < kOwners) {
#pragma unroll
            for (int k = 0; k < kPer; ++k) {
                uint32_t c = 0;
#pragma unroll
                for (int w = 0; w < kWarps; ++w) c += counters[w * 256 + kPer * t + k];
                if (c == (uint32_t)n) s_misc[0] = 1;   // every key has this digit: pass is the identity
                tot += c;
            }
        }
        scope_sync<kThreads>();
        const bool skip = s_misc[0] != 0;
        if (!skip) {
            // exclusive scan of tot over the owners
            uint32_t incl = 0;
            if (t < kOwners) {
                incl = warp_inclusive_scan(tot, lane);
                if (lane == 31) s_misc[1 + warp] = incl;
            }
            scope_sync<kThreads>();
            if (t < kOwners) {
                uint32_t base = incl - tot;
                for (int w = 0; w < warp; ++w) base += s_misc[1 + w];
#pragma unroll
                for (int k = 0; k < kPer; ++k) {
#pragma unroll
                    for (int w = 0; w < kWarps; ++w) {
                        const uint32_t c = counters[w * 256 + kPer * t + k];
                        counters[w * 256 + kPer * t + k] = base;
                        base += c;
                    }
                }
            }
            scope_sync<kThreads>();
            // 3. stable scatter
            for (int i0 = seg_lo; i0 < seg_hi; i0 += 32) {
                const int i = i0 + lane;
                const bool have = i < seg_hi;
                const u64 k = have ? src[i] : 0ull;
                const uint32_t d = have ? (uint32_t)(k >> shift) & 0xffu : 0u;
                const unsigned peers = digit_peers(d, have);
                uint32_t off = 0;
                if (have) off = counters[warp * 256 + d] + __popc(peers & ((1u << lane) - 1u));
                __syncwarp();
                if (have) {
                    dst[off] = k;
                    if ((__ffs(peers) - 1) == lane) counters[warp * 256 + d] += __popc(peers);
                }
                __syncwarp();
            }
            u64* tmp = src; src = dst; dst = tmp;
        }
        scope_sync<kThreads>();
    }
    // 4. order runs of equal depth by Gaussian index (rare: exact float ties)
    for (int i = t; i < n; i += kThreads) {
        const uint32_t d = (uint32_t)(src[i] >> 32);
        const bool run_start = (i == 0 || (uint32_t)(src[i - 1] >> 32) != d) && (i + 1 < n) &&
                               (uint32_t)(src[i + 1] >> 32) == d;
        if (run_start) {
            int e = i + 1;
            while (e < n && (uint32_t)(src[e] >> 32) == d) ++e;
            insertion_sort(src, i, e);
        }
    }
    scope_sync<kThreads>();
    return src;
}

// ---- bucket sort: the common case of every shared-memory class ------------------------------------------------------
// A tile's depths are a few hundred to a few thousand floats inside one narrow interval, close to uniform in it.  Instead
// of four 8-bit LSD passes (two ballot-ranked sweeps each: ~10 warp-instructions per key), the
// keys are dropped into kBuckets >= n equal-width buckets over the tile's own [min, max] of depth bits -- one histogram
// sweep and one scatter sweep with native shared-memory integer atomics -- and each bucket (1-2 keys on average) is put
// in order by an insertion sort on the full 64-bit key (depth_bits, gaussian_idx): the same total order as the
// reference's stable sort.  A tile whose fullest bucket exceeds kInsertMax (depths piled on a few values) takes the radix
// sort instead, decided per tile on the device.
constexpr int kInsertMax = 24;

// Sorts a[0, n) into b[0, n); returns false (uniformly, b unspecified, a intact) when a bucket is too full.
// cnt: kBuckets words; s_misc: words {min, max, maxcnt}; warp_tot: 32 words (CTA scope only).
template <int kThreads, int kBuckets>
__device__ __forceinline__ bool bucket_sort_tile(const u64* a, u64* b, int n, uint32_t* cnt, uint32_t* s_misc,
                                                 uint32_t* warp_tot, int t) {
    const unsigned full = 0xffffffffu;
    if (t == 0) { s_misc[0] = 0xffffffffu; s_misc[1] = 0u; s_misc[2] = 0u; }
    for (int i = t; i < kBuckets; i += kThreads) cnt[i] = 0;
    scope_sync<kThreads>();
    uint32_t lmin = 0xffffffffu, lmax = 0u;
    for (int i = t; i < n; i += kThreads) {
        const uint32_t d = (uint32_t)(a[i] >> 32);
        lmin = min(lmin, d); lmax = max(lmax, d);
    }
    lmin = __reduce_min_sync(full, lmin);
    lmax = __reduce_max_sync(full, lmax);
    if ((t & 31) == 0) { atomicMin(&s_misc[0], lmin); atomicMax(&s_misc[1], lmax); }
    scope_sync<kThreads>();
    const uint32_t dmin = *(volatile uint32_t*)&s_misc[0], range = *(volatile uint32_t*)&s_misc[1] - dmin;
    constexpr int kLog = 31 - __builtin_clz((unsigned)kBuckets);
    const int bits = range ? 32 - __clz(range) : 0;
    const int shift = max(0, bits - kLog);
    // 1. histogram
    for (int i = t; i < n; i += kThreads) atomicAdd(cnt + (((uint32_t)(a[i] >> 32) - dmin) >> shift), 1u);
    scope_sync<kThreads>();
    // 2. exclusive scan of the bucket counts (each thread owns kBuckets / kThreads consecutive buckets) + fullest bucket
    constexpr int kPer = kBuckets / kThreads;
    static_assert(kBuckets % kThreads == 0, "buckets per thread");
    uint32_t local = 0, lmaxc = 0;
#pragma unroll 4
    for (int k = 0; k < kPer; ++k) {
        const uint32_t c = cnt[t * kPer + k];
        local += c; lmaxc = max(lmaxc, c);
    }
    const uint32_t incl = warp_inclusive_scan(local, t & 31);
    lmaxc = __reduce_max_sync(full, lmaxc);
    uint32_t warp_base = 0;
    if (kThreads > 32) {
        if ((t & 31) == 31) warp_tot[t >> 5] = incl;
        if ((t & 31) == 0) atomicMax(&s_misc[2], lmaxc);
        __syncthreads();
        for (int w = 0; w < (t >> 5); ++w) warp_base += warp_tot[w];
        lmaxc = *(volatile uint32_t*)&s_misc[2];
    }
    if (lmaxc > (uint32_t)kInsertMax) return false;          // uniform over the scope
    uint32_t run = warp_base + incl - local;
#pragma unroll 4
    for (int k = 0; k < kPer; ++k) {
        const uint32_t c = cnt[t * kPer + k];
        cnt[t * kPer + k] = run;
        run += c;
    }
    scope_sync<kThreads>();
    // 3. scatter (the order inside a bucket is whatever the atomics make it; step 4 fixes it)
    for (int i = t; i < n; i += kThreads) {
        const u64 k = a[i];
        b[atomicAdd(cnt + (((uint32_t)(k >> 32) - dmin) >> shift), 1u)] = k;
    }
    scope_sync<kThreads>();
    // 4. insertion sort inside each bucket; cnt[j] is now the END of bucket j
    for (int j = t; j < kBuckets; j += kThreads) insertion_sort(b, j ? (int)cnt[j - 1] : 0, (int)cnt[j]);
    scope_sync<kThreads>();
    return true;
}

// Sorts the keys of the tile with range rg in shared memory -- the bucket sort, else the radix sort -- and writes them
// back, with their Gaussian indices to point_list.  buf_a, buf_b: kMaxN keys each; counters: kMaxN bucket words, whose
// first (kThreads / 32) * 256 double as the radix sort's per-warp digit counters; s_misc: 3 words at warp scope, 9 at
// CTA scope; warp_tot: 32 words (CTA scope only).
template <int kThreads, int kMaxN>
__device__ __forceinline__ void sort_tile_shared(u64* keys, uint32_t* point_list, uint2 rg, u64* buf_a, u64* buf_b,
                                                 uint32_t* counters, uint32_t* s_misc, uint32_t* warp_tot, int t) {
    static_assert(kMaxN >= (kThreads / 32) * 256, "counter aliasing");
    const int n = (int)(rg.y - rg.x);
    u64* g = keys + rg.x;
    for (int i = t; i < n; i += kThreads) buf_a[i] = g[i];
    scope_sync<kThreads>();
    const u64* res = buf_b;
    if (!bucket_sort_tile<kThreads, kMaxN>(buf_a, buf_b, n, counters, s_misc, warp_tot, t)) {
        scope_sync<kThreads>();
        res = radix_sort<kThreads>(buf_a, buf_b, n, counters, s_misc, t);
    }
    for (int i = t; i < n; i += kThreads) {
        const u64 k = res[i];
        g[i] = k;
        point_list[rg.x + i] = (uint32_t)k;
    }
    scope_sync<kThreads>();
}

template <int kThreads, int kMaxN, bool kDynamic>
__global__ void __launch_bounds__(kThreads)
tile_sort_shared_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                        const uint2* __restrict__ ranges, u64* __restrict__ keys,
                        uint32_t* __restrict__ point_list, const int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char dyn_smem[];
    __shared__ u64 stat_a[kDynamic ? 1 : kMaxN];
    __shared__ u64 stat_b[kDynamic ? 1 : kMaxN];
    __shared__ uint32_t stat_counters[kDynamic ? 1 : kMaxN];
    __shared__ uint32_t s_misc[40];
    __shared__ uint32_t s_warp_tot[32];
    u64* buf_a = kDynamic ? reinterpret_cast<u64*>(dyn_smem) : stat_a;
    u64* buf_b = kDynamic ? reinterpret_cast<u64*>(dyn_smem) + kMaxN : stat_b;
    uint32_t* counters = kDynamic ? reinterpret_cast<uint32_t*>(dyn_smem + 2 * sizeof(u64) * kMaxN) : stat_counters;
    if (status[FB200_ST_OVERFLOW]) return;
    const uint32_t count = *n_list;
    for (uint32_t w = blockIdx.x; w < count; w += gridDim.x)
        sort_tile_shared<kThreads, kMaxN>(keys, point_list, ranges[list[w]], buf_a, buf_b, counters, s_misc, s_warp_tot,
                                          threadIdx.x);
}

// ---- tiny lists: one WARP per tile ---------------------------------------------------------------------
// Most tiles of a real frame hold a few hundred instances.  Spreading such a list over the 8 warps of a CTA leaves each
// warp one or two 32-key steps per pass between CTA barriers (barrier stalls dominate).  Here a
// warp sorts a whole tile by itself (__syncwarp only), so an SM runs dozens of independent tile sorts.
template <int kWarps>
__global__ void __launch_bounds__(32 * kWarps)
tile_sort_warp_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                      const uint2* __restrict__ ranges, u64* __restrict__ keys, uint32_t* __restrict__ point_list,
                      const int32_t* __restrict__ status) {
    __shared__ u64 s_a[kWarps][kSortTinyMax];
    __shared__ u64 s_b[kWarps][kSortTinyMax];
    __shared__ uint32_t s_cnt[kWarps][kSortTinyMax];
    __shared__ uint32_t s_misc[kWarps][4];
    if (status[FB200_ST_OVERFLOW]) return;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t count = *n_list;
    for (uint32_t w = blockIdx.x * kWarps + warp; w < count; w += gridDim.x * kWarps) {
        const uint2 rg = ranges[list[w]];
        const int n = (int)(rg.y - rg.x);
        u64* g = keys + rg.x;
        if (n == 1) {                                   // nothing to sort, only the point_list entry
            if (lane == 0) point_list[rg.x] = (uint32_t)g[0];
            continue;
        }
        sort_tile_shared<32, kSortTinyMax>(keys, point_list, rg, s_a[warp], s_b[warp], s_cnt[warp], s_misc[warp], nullptr,
                                           lane);
    }
}

// Lists longer than the shared-memory classes: the radix sort alone, ping-pong between the key array and a
// scratch array in global memory (L2-resident for any realistic tile).
template <int kThreads>
__global__ void __launch_bounds__(kThreads)
tile_sort_global_kernel(const uint32_t* __restrict__ list, const uint32_t* __restrict__ n_list,
                        const uint2* __restrict__ ranges, u64* __restrict__ keys, u64* __restrict__ scratch,
                        uint32_t* __restrict__ point_list, const int32_t* __restrict__ status) {
    __shared__ uint32_t counters[(kThreads / 32) * 256];
    __shared__ uint32_t s_misc[40];
    if (status[FB200_ST_OVERFLOW]) return;
    const uint32_t count = *n_list;
    for (uint32_t w = blockIdx.x; w < count; w += gridDim.x) {
        const uint2 rg = ranges[list[w]];
        const int n = (int)(rg.y - rg.x);
        u64* g = keys + rg.x;
        const u64* res = radix_sort<kThreads>(g, scratch + rg.x, n, counters, s_misc, threadIdx.x);
        for (int i = threadIdx.x; i < n; i += kThreads) {
            const u64 k = res[i];
            if (res != g) g[i] = k;
            point_list[rg.x + i] = (uint32_t)k;
        }
        __syncthreads();
    }
}

}  // namespace

cudaError_t launch_tile_scan(const FwdArgs& a, cudaStream_t s) {
    const int T = a.tiles_x * a.tiles_y;
    tile_scan_kernel<<<1, 1024, 0, s>>>(T, a.tile_count, a.ranges, a.cursor, a.list_tiny, a.list_small, a.list_large,
                                        a.list_huge, a.counters, a.capacity, a.status, a.tile_order);
    count_launch();
    return cudaGetLastError();
}

// set the overflow word for a raster phase launched with its own capacity
__global__ void check_capacity_kernel(long long capacity, int32_t* __restrict__ status) {
    const int32_t r = status[FB200_ST_NUM_RENDERED];
    status[FB200_ST_OVERFLOW] = ((long long)r > capacity || r == 0x7fffffff) ? 1 : 0;
}

// The tiny-list and small-list sorts are independent and each ends in a long tail (a few long lists on a few SMs);
// the small-list kernel therefore runs on a side stream, forked after the scatter and joined before the blend.
SideStream* side_stream() {
    static SideStream pool[64];
    static std::mutex mu;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    std::lock_guard<std::mutex> lk(mu);
    SideStream& a = pool[dev];
    if (!a.ready) {
        if (cudaStreamCreateWithFlags(&a.stream, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
        if (cudaEventCreateWithFlags(&a.fork, cudaEventDisableTiming) != cudaSuccess) return nullptr;
        if (cudaEventCreateWithFlags(&a.join, cudaEventDisableTiming) != cudaSuccess) return nullptr;
        a.ready = true;
    }
    return &a;
}

// h_status: the status words of the geometry phase as the HOST has read them (or NULL).  With them the launches
// that would find an empty work list are skipped (the lists live on the device, so without them every class is
// launched for the worst case and exits at once).
cudaError_t launch_binning(const FwdArgs& a, cudaStream_t s, const int32_t* h_status) {
    const int T = a.tiles_x * a.tiles_y;
    const int max_tile = h_status ? h_status[FB200_ST_MAX_TILE] : 0x7fffffff;
    const bool capacity_known_ok = h_status && (long long)h_status[FB200_ST_NUM_RENDERED] <= a.capacity &&
                                   h_status[FB200_ST_OVERFLOW] == 0;
    if (!capacity_known_ok) {
        check_capacity_kernel<<<1, 1, 0, s>>>(a.capacity, a.status);
        count_launch();
    }
    if (a.prm.P > 0) {
        // (CTA-private counting / scattering through shared-memory tables was slower at C5: shared-memory atomics retire
        // ~2 cycles per lane; the direct global atomics stay)
        scatter_kernel<<<(a.prm.P + 255) / 256, 256, 0, s>>>(a.prm.P, a.tiles_x, a.rect, a.depth, a.cursor,
                                                             a.keys, a.status);
        count_launch();
    }
    // The work lists live on the device: launch enough CTAs for the worst case, each CTA strides over its list.
    SideStream* side = (max_tile > kSortTinyMax) ? side_stream() : nullptr;
    std::unique_lock<std::mutex> side_use;
    if (side) side_use = std::unique_lock<std::mutex>(side->use);
    cudaStream_t s2 = s;
    if (side) {
        cudaError_t e = cudaEventRecord(side->fork, s);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(side->stream, side->fork, 0);
        if (e != cudaSuccess) return e;
        s2 = side->stream;
    }
    {
        constexpr int kWarps = 4;                        // 4 x 10 KB of shared memory per CTA
        const int grid = min((T + kWarps - 1) / kWarps, sm_count() * 6);
        tile_sort_warp_kernel<kWarps><<<grid, 32 * kWarps, 0, s>>>(a.list_tiny, a.counters + 4, a.ranges, a.keys,
                                                                   a.point_list, a.status);
        count_launch();
    }
    if (max_tile > kSortTinyMax) {
        const int grid = min(T, sm_count() * 5);
        tile_sort_shared_kernel<256, kSortSmallMax, false><<<grid, 256, 0, s2>>>(
            a.list_small, a.counters + 0, a.ranges, a.keys, a.point_list, a.status);
        count_launch();
    }
    if (max_tile > kSortSmallMax) {
        // medium lists (2048 < n <= 8192): 1024 threads, ping-pong buffers + per-warp counters in 160 KB of
        // dynamic shared memory, one CTA per SM
        const int smem = 2 * 8 * kSortMediumMax + 4 * kSortMediumMax;     // two key buffers + one counter word per bucket
        // per call, not once per process: the attribute is per device
        const cudaError_t attr = cudaFuncSetAttribute(tile_sort_shared_kernel<1024, kSortMediumMax, true>,
                                                      cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (attr != cudaSuccess) return attr;
        const int grid = min(T, sm_count());
        tile_sort_shared_kernel<1024, kSortMediumMax, true><<<grid, 1024, smem, s2>>>(
            a.list_large, a.counters + 1, a.ranges, a.keys, a.point_list, a.status);
        count_launch();
    }
    if (max_tile > kSortMediumMax) {
        const int grid = min(T, sm_count() * 2);
        tile_sort_global_kernel<1024><<<grid, 1024, 0, s2>>>(a.list_huge, a.counters + 2, a.ranges, a.keys,
                                                             a.keys_scratch, a.point_list, a.status);
        count_launch();
    }
    if (side) {
        cudaError_t e = cudaEventRecord(side->join, side->stream);
        if (e == cudaSuccess) e = cudaStreamWaitEvent(s, side->join, 0);
        if (e != cudaSuccess) return e;
    }
    return cudaGetLastError();
}

}  // namespace fb200
