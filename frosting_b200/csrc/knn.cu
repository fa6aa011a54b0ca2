// knn.cu -- exact K nearest neighbours over a point set (pytorch3d's knn_points with norm = 2, unbatched), the
// neighbour table of SuGaR's coarse regulariser (reset_neighbors, frosting_scene/sugar_model.py:1044-1061).
//
// Contract (include/frosting_b200.h, fb200_knn): for each query, the first K points in ascending (d, index) order, with
// d = fmaf(dz, dz, fmaf(dy, dy, dx * dx)) and dx = q.x - p.x rounded to float32.  The result is a function of the input
// bits alone.  Both are carried as one 64-bit key, float bits of d (d >= +0, so its bits order like its value) above
// the point index, so one unsigned compare is the lexicographic (d, index) compare.
//
//   1. knn_box_kernel (one block): a robust quantisation box from a strided sample of at most 8192 points, the 1/64 and
//      63/64 quantiles per axis widened by 1/8 of their span.  Far outliers (background Gaussians) then no longer
//      stretch the Morton grid; they fall into the end cells.  The box only shapes the tree, never the result.
//   2. knn_key_kernel: 63-bit Morton keys (21 bits per axis) over that box, index as value; raises the non-finite flag.
//   3. CUB DeviceRadixSort::SortPairs (stable, so equal keys stay in index order): deterministic.
//   4. knn_leaf_kernel (one warp per leaf of 32 consecutive sorted points): gathers the points as float4 {x, y, z,
//      index} and writes the leaf's AABB and minimum index.  knn_level_kernel then builds an implicit balanced binary
//      tree over the leaves, bottom up, one launch per level (heap order: node n has children 2n, 2n + 1; leaf l is node
//      N2 + l for N2 = the power of two >= the leaf count; padding leaves are empty boxes).
//   5. knn_query_kernel (one warp per query, queries in Morton order): the K-list is one entry per lane, sorted by key,
//      seeded with K points around the query's place in the sorted points, then a nearest-first walk with a per-lane
//      stack (lane s holds stack entry s).  A leaf is evaluated 32 points at once, candidates merged by ballot and
//      shuffle.  A node is pruned when its key (lower bound of d, minimum index) exceeds the K-th key: the bound is
//      formed with round-down intrinsics, so it is <= the round-to-nearest d of every point in the box, and the index
//      clause keeps a large set of coincident points from degrading to a full walk.
#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"

namespace fb200 {

namespace {

constexpr int kKnnThreads = 256;
constexpr int kBoxSample = 8192;     // points sampled for the robust box
constexpr int kMortonBits = 21;

struct KnnNode {
    float4 lo;   // xyz: box minimum; w: minimum point index (int bits)
    float4 hi;   // xyz: box maximum
};

// Workspace sections, each 256-byte aligned, the non-finite flag first (header: fb200_knn).  Self queries (no query
// set) need no query sections.
struct KnnLayout {
    size_t flag, box, pkeys[2], pvals[2], qkeys[2], qvals[2], pts, qpts, nodes, cub, cub_bytes, total;
    int n_leaves, n2;
    KnnLayout(int P, int Q) {
        n_leaves = (int)(((int64_t)P + 31) / 32);
        n2 = 1;
        while (n2 < n_leaves) n2 <<= 1;
        const size_t n = (size_t)(P > Q ? P : Q);
        // CUB 2.8.2 (the CCCL of CUDA 12.9) asks ~1 byte per item for 64-bit keys with 32-bit values (onesweep
        // lookback and bins); fb200_knn compares CUB's own size query with this before it launches (knn_sort_scratch)
        cub_bytes = 2 * n + (64 << 10);
        size_t o = 0;
        auto take = [&](size_t bytes) { size_t at = o; o = (o + bytes + 255) & ~size_t(255); return at; };
        flag = take(sizeof(int));
        box = take(2 * sizeof(float4));
        for (int b = 0; b < 2; ++b) pkeys[b] = take(sizeof(uint64_t) * (size_t)P);
        for (int b = 0; b < 2; ++b) pvals[b] = take(sizeof(uint32_t) * (size_t)P);
        for (int b = 0; b < 2; ++b) qkeys[b] = take(sizeof(uint64_t) * (size_t)Q);
        for (int b = 0; b < 2; ++b) qvals[b] = take(sizeof(uint32_t) * (size_t)Q);
        pts = take(sizeof(float4) * (size_t)P);
        qpts = take(sizeof(float4) * (size_t)Q);
        nodes = take(sizeof(KnnNode) * 2 * (size_t)n2);
        cub = take(cub_bytes);
        total = o;
    }
};

// float <-> unsigned with the same order (NaNs sort to the ends)
__device__ __forceinline__ uint32_t ordered_bits(float v) {
    const uint32_t u = __float_as_uint(v);
    return u ^ ((u >> 31) ? 0xffffffffu : 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(uint32_t u) {
    return __uint_as_float(u ^ ((u >> 31) ? 0x80000000u : 0xffffffffu));
}

__global__ void __launch_bounds__(1024) knn_box_kernel(const float* __restrict__ points, int P, float4* box) {
    __shared__ uint32_t s[kBoxSample];
    const int S = P < kBoxSample ? P : kBoxSample;
    int n2 = 1;
    while (n2 < S) n2 <<= 1;
    float lo[3], hi[3];
    for (int axis = 0; axis < 3; ++axis) {
        for (int i = threadIdx.x; i < n2; i += blockDim.x)
            s[i] = i < S ? ordered_bits(points[3 * (((int64_t)i * P) / S) + axis]) : 0xffffffffu;
        __syncthreads();
        for (int k = 2; k <= n2; k <<= 1)          // bitonic sort, ascending
            for (int j = k >> 1; j > 0; j >>= 1) {
                for (int i = threadIdx.x; i < n2; i += blockDim.x) {
                    const int o = i ^ j;
                    if (o > i) {
                        const uint32_t a = s[i], b = s[o];
                        if ((a > b) == ((i & k) == 0)) { s[i] = b; s[o] = a; }
                    }
                }
                __syncthreads();
            }
        const float a = from_ordered_bits(s[S / 64]), b = from_ordered_bits(s[S - 1 - S / 64]);
        const float m = 0.125f * (b - a);
        lo[axis] = a - m;
        hi[axis] = b + m;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        float4 l, sc;
        float* lp = &l.x;
        float* sp = &sc.x;
        for (int axis = 0; axis < 3; ++axis) {
            const float span = hi[axis] - lo[axis];
            const bool ok = isfinite(lo[axis]) && isfinite(span) && span > 0.f;
            lp[axis] = ok ? lo[axis] : 0.f;
            sp[axis] = ok ? (float)((1 << kMortonBits) - 1) / span : 0.f;   // degenerate axis: one cell
            if (!isfinite(sp[axis])) sp[axis] = 0.f;
        }
        l.w = sc.w = 0.f;
        box[0] = l;
        box[1] = sc;
    }
}

__device__ __forceinline__ uint64_t spread21(uint32_t v) {
    uint64_t x = v & 0x1fffffu;
    x = (x | x << 32) & 0x1f00000000ffffull;
    x = (x | x << 16) & 0x1f0000ff0000ffull;
    x = (x | x << 8) & 0x100f00f00f00f00full;
    x = (x | x << 4) & 0x10c30c30c30c30c3ull;
    x = (x | x << 2) & 0x1249249249249249ull;
    return x;
}

__device__ __forceinline__ uint32_t cell(float v, float lo, float scale) {
    // fmaxf drops a NaN, so any bits give a cell in range
    return (uint32_t)fminf(fmaxf((v - lo) * scale, 0.f), (float)((1 << kMortonBits) - 1));
}

__global__ void knn_key_kernel(const float* __restrict__ xyz, int n, const float4* __restrict__ box,
                               uint64_t* __restrict__ keys, uint32_t* __restrict__ vals, int* flag) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    if (!isfinite(x) || !isfinite(y) || !isfinite(z)) atomicOr(flag, 1);
    const float4 lo = box[0], sc = box[1];
    keys[i] = spread21(cell(x, lo.x, sc.x)) << 2 | spread21(cell(y, lo.y, sc.y)) << 1 | spread21(cell(z, lo.z, sc.z));
    vals[i] = (uint32_t)i;
}

// one warp per sorted slot range of 32: the gathered rows {x, y, z, index} (also the sorted queries, with leaves = NULL)
__global__ void knn_leaf_kernel(const float* __restrict__ xyz, int n, const uint32_t* __restrict__ order,
                                float4* __restrict__ rows, KnnNode* __restrict__ leaves, int n_slots) {
    const int leaf = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (leaf >= n_slots) return;
    const int64_t i = (int64_t)leaf * 32 + lane;
    float3 lo = make_float3(INFINITY, INFINITY, INFINITY), hi = make_float3(-INFINITY, -INFINITY, -INFINITY);
    uint32_t mi = 0x7fffffffu;
    if (i < n) {
        const uint32_t j = order[i];
        const float x = xyz[3 * (int64_t)j], y = xyz[3 * (int64_t)j + 1], z = xyz[3 * (int64_t)j + 2];
        rows[i] = make_float4(x, y, z, __uint_as_float(j));
        lo = hi = make_float3(x, y, z);
        mi = j;
    }
    if (!leaves) return;
    for (int o = 16; o > 0; o >>= 1) {
        lo.x = fminf(lo.x, __shfl_xor_sync(0xffffffffu, lo.x, o));
        lo.y = fminf(lo.y, __shfl_xor_sync(0xffffffffu, lo.y, o));
        lo.z = fminf(lo.z, __shfl_xor_sync(0xffffffffu, lo.z, o));
        hi.x = fmaxf(hi.x, __shfl_xor_sync(0xffffffffu, hi.x, o));
        hi.y = fmaxf(hi.y, __shfl_xor_sync(0xffffffffu, hi.y, o));
        hi.z = fmaxf(hi.z, __shfl_xor_sync(0xffffffffu, hi.z, o));
        mi = min(mi, __shfl_xor_sync(0xffffffffu, mi, o));
    }
    if (lane == 0) leaves[leaf] = KnnNode{make_float4(lo.x, lo.y, lo.z, __uint_as_float(mi)),
                                          make_float4(hi.x, hi.y, hi.z, 0.f)};
}

// nodes [first, 2 first) from their children
__global__ void knn_level_kernel(KnnNode* __restrict__ nodes, int first) {
    const int n = first + (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (n >= 2 * first) return;
    const KnnNode a = nodes[2 * n], b = nodes[2 * n + 1];
    nodes[n] = KnnNode{make_float4(fminf(a.lo.x, b.lo.x), fminf(a.lo.y, b.lo.y), fminf(a.lo.z, b.lo.z),
                                   __uint_as_float(min(__float_as_uint(a.lo.w), __float_as_uint(b.lo.w)))),
                       make_float4(fmaxf(a.hi.x, b.hi.x), fmaxf(a.hi.y, b.hi.y), fmaxf(a.hi.z, b.hi.z), 0.f)};
}

__device__ __forceinline__ uint64_t point_key(float qx, float qy, float qz, float4 p) {
    const float dx = __fsub_rn(qx, p.x), dy = __fsub_rn(qy, p.y), dz = __fsub_rn(qz, p.z);
    const float d = __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
    return (uint64_t)__float_as_uint(d) << 32 | __float_as_uint(p.w);
}

// (lower bound of d over the box, minimum index): <= the key of every point in the box
__device__ __forceinline__ uint64_t node_key(float qx, float qy, float qz, const KnnNode& n) {
    const float gx = fmaxf(fmaxf(__fsub_rd(n.lo.x, qx), __fsub_rd(qx, n.hi.x)), 0.f);
    const float gy = fmaxf(fmaxf(__fsub_rd(n.lo.y, qy), __fsub_rd(qy, n.hi.y)), 0.f);
    const float gz = fmaxf(fmaxf(__fsub_rd(n.lo.z, qz), __fsub_rd(qz, n.hi.z)), 0.f);
    const float b = __fadd_rd(__fadd_rd(__fmul_rd(gx, gx), __fmul_rd(gy, gy)), __fmul_rd(gz, gz));
    return (uint64_t)__float_as_uint(b) << 32 | __float_as_uint(n.lo.w);
}

struct QueryArgs {
    int P, Q, K, n2;
    const float4* rows;        // sorted points
    const KnnNode* nodes;
    const float4* qrows;       // sorted queries (rows for self queries)
    const uint64_t* pkeys;     // sorted point keys (separate queries: placing the seed)
    const uint64_t* qkeys;     // sorted query keys, or NULL for self queries
    float* dists;
    int64_t* idx;
};

__global__ void __launch_bounds__(kKnnThreads) knn_query_kernel(QueryArgs a) {
    const int w = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= a.Q) return;
    const float4 q = a.qrows[w];
    const int K = a.K;

    // seed: K consecutive sorted points around the query's place in Morton order
    int home = w;
    if (a.qkeys) {
        const uint64_t qk = a.qkeys[w];
        int lo = 0, hi = a.P;
        while (lo < hi) {
            const int mid = (int)(((unsigned)lo + (unsigned)hi) >> 1);
            if (a.pkeys[mid] < qk) lo = mid + 1; else hi = mid;
        }
        home = lo;
    }
    const int s0 = max(0, min(home - (K - 1) / 2, a.P - K));
    uint64_t key = lane < K ? point_key(q.x, q.y, q.z, a.rows[s0 + lane]) : ~0ull;
    for (int k = 2; k <= 32; k <<= 1)                // bitonic sort across lanes, ascending
        for (int j = k >> 1; j > 0; j >>= 1) {
            const uint64_t o = __shfl_xor_sync(0xffffffffu, key, j);
            const bool take_min = ((lane & j) == 0) == ((lane & k) == 0);
            key = take_min ? (o < key ? o : key) : (o > key ? o : key);
        }
    uint64_t worst = __shfl_sync(0xffffffffu, key, K - 1);

    int stack = 0, sp = 0;      // lane s holds entry s
    int node = 1;
    bool have = node_key(q.x, q.y, q.z, a.nodes[1]) <= worst;
    while (have) {
        if (node >= a.n2) {
            const int64_t i = (int64_t)(node - a.n2) * 32 + lane;
            const uint64_t c = i < a.P ? point_key(q.x, q.y, q.z, a.rows[i]) : ~0ull;
            unsigned cand = __ballot_sync(0xffffffffu, c < worst);
            while (cand) {
                const int src = __ffs(cand) - 1;
                cand &= cand - 1;
                const uint64_t ck = __shfl_sync(0xffffffffu, c, src);
                if (ck >= worst) continue;                                    // the list tightened meanwhile
                if (__ballot_sync(0xffffffffu, key == ck)) continue;          // a seed point already listed
                const int pos = __popc(__ballot_sync(0xffffffffu, key < ck));
                const uint64_t up = __shfl_up_sync(0xffffffffu, key, 1);
                key = lane < pos ? key : (lane == pos ? ck : up);
                worst = __shfl_sync(0xffffffffu, key, K - 1);
            }
        } else {
            const uint64_t kl = node_key(q.x, q.y, q.z, a.nodes[2 * node]);
            const uint64_t kr = node_key(q.x, q.y, q.z, a.nodes[2 * node + 1]);
            const bool left_first = kl <= kr;
            const uint64_t kn = left_first ? kl : kr, kf = left_first ? kr : kl;
            if (kn <= worst) {
                if (kf <= worst) {
                    if (lane == sp) stack = 2 * node + (left_first ? 1 : 0);
                    ++sp;
                }
                node = 2 * node + (left_first ? 0 : 1);
                continue;
            }
        }
        have = false;
        while (sp > 0) {
            --sp;
            node = __shfl_sync(0xffffffffu, stack, sp);
            if (node_key(q.x, q.y, q.z, a.nodes[node]) <= worst) { have = true; break; }
        }
    }
    if (lane < K) {
        const int64_t out = (int64_t)__float_as_uint(q.w) * K + lane;
        a.dists[out] = __uint_as_float((uint32_t)(key >> 32));
        a.idx[out] = (int64_t)(uint32_t)key;
    }
}

unsigned blocks(int64_t n, int per_block) { return (unsigned)((n + per_block - 1) / per_block); }

// CUB's scratch bytes for sorting n (key, index) pairs (a host query; needs the current device)
cudaError_t sort_scratch(int n, size_t* bytes) {
    cub::DoubleBuffer<uint64_t> k(nullptr, nullptr);
    cub::DoubleBuffer<uint32_t> v(nullptr, nullptr);
    *bytes = 0;
    return cub::DeviceRadixSort::SortPairs(nullptr, *bytes, k, v, n, 0, 3 * kMortonBits);
}

// stable (key, index) sort in the workspace's double buffers, with the layout's scratch reservation
cudaError_t sort_pairs(const KnnLayout& L, char* ws, const size_t kb[2], const size_t vb[2], int n,
                       const uint64_t** sorted_keys, const uint32_t** sorted_vals, cudaStream_t s) {
    cub::DoubleBuffer<uint64_t> k(reinterpret_cast<uint64_t*>(ws + kb[0]), reinterpret_cast<uint64_t*>(ws + kb[1]));
    cub::DoubleBuffer<uint32_t> v(reinterpret_cast<uint32_t*>(ws + vb[0]), reinterpret_cast<uint32_t*>(ws + vb[1]));
    size_t bytes = L.cub_bytes;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(ws + L.cub, bytes, k, v, n, 0, 3 * kMortonBits, s);
    *sorted_keys = k.Current();
    *sorted_vals = v.Current();
    return e;
}

}  // namespace

size_t knn_workspace_bytes(int P, int Q) { return KnnLayout(P, Q).total; }

cudaError_t knn_sort_scratch(int P, int Q, size_t* need, size_t* reserved) {
    size_t np = 0, nq = 0;
    cudaError_t e = sort_scratch(P, &np);
    if (e == cudaSuccess && Q > 0) e = sort_scratch(Q, &nq);
    *need = np > nq ? np : nq;
    *reserved = KnnLayout(P, Q).cub_bytes;
    return e;
}

cudaError_t launch_knn(const float* points, int P, const float* queries, int Q, int K, void* workspace, float* dists,
                       int64_t* idx, cudaStream_t s) {
    const KnnLayout L(P, queries ? Q : 0);
    char* ws = static_cast<char*>(workspace);
    int* flag = reinterpret_cast<int*>(ws + L.flag);
    float4* box = reinterpret_cast<float4*>(ws + L.box);
    cudaError_t e = cudaMemsetAsync(flag, 0, sizeof(int), s);
    if (e != cudaSuccess) return e;
    knn_box_kernel<<<1, 1024, 0, s>>>(points, P, box);
    knn_key_kernel<<<blocks(P, kKnnThreads), kKnnThreads, 0, s>>>(
        points, P, box, reinterpret_cast<uint64_t*>(ws + L.pkeys[0]), reinterpret_cast<uint32_t*>(ws + L.pvals[0]), flag);
    count_launch(2);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    const uint64_t* pkeys;
    const uint32_t* porder;
    if ((e = sort_pairs(L, ws, L.pkeys, L.pvals, P, &pkeys, &porder, s)) != cudaSuccess) return e;
    float4* rows = reinterpret_cast<float4*>(ws + L.pts);
    KnnNode* nodes = reinterpret_cast<KnnNode*>(ws + L.nodes);
    const int warps_per_block = kKnnThreads / 32;
    knn_leaf_kernel<<<blocks(L.n2, warps_per_block), kKnnThreads, 0, s>>>(points, P, porder, rows,
                                                                                          nodes + L.n2, L.n2);
    count_launch();
    for (int first = L.n2 / 2; first >= 1; first /= 2) {
        knn_level_kernel<<<blocks(first, kKnnThreads), kKnnThreads, 0, s>>>(nodes, first);
        count_launch();
    }
    QueryArgs a;
    a.P = P; a.Q = Q; a.K = K; a.n2 = L.n2;
    a.rows = rows; a.nodes = nodes; a.pkeys = pkeys;
    a.qrows = rows; a.qkeys = nullptr;
    a.dists = dists; a.idx = idx;
    if (queries) {
        knn_key_kernel<<<blocks(Q, kKnnThreads), kKnnThreads, 0, s>>>(
            queries, Q, box, reinterpret_cast<uint64_t*>(ws + L.qkeys[0]), reinterpret_cast<uint32_t*>(ws + L.qvals[0]),
            flag);
        count_launch();
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
        const uint32_t* qorder;
        if ((e = sort_pairs(L, ws, L.qkeys, L.qvals, Q, &a.qkeys, &qorder, s)) != cudaSuccess) return e;
        float4* qrows = reinterpret_cast<float4*>(ws + L.qpts);
        const int slots = (int)(((int64_t)Q + 31) / 32);
        knn_leaf_kernel<<<blocks(slots, warps_per_block), kKnnThreads, 0, s>>>(queries, Q, qorder,
                                                                                               qrows, nullptr, slots);
        count_launch();
        a.qrows = qrows;
    }
    knn_query_kernel<<<blocks(Q, warps_per_block), kKnnThreads, 0, s>>>(a);
    count_launch();
    return cudaGetLastError();
}

}  // namespace fb200
