/* Brute-force K nearest neighbours, the oracle of fb200_knn (test infrastructure, built with -ffp-contract=off so that
 * only the explicit fmaf() calls fuse).  For each query q in [q0, q1): the first K points in ascending (d, index) order,
 * d = fmaf(dz, dz, fmaf(dy, dy, dx * dx)) with dx = q.x - p.x in float32 -- the library's expression and tie rule. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define BLOCK 1024

static uint64_t key_of(float d, int64_t i) {
    uint32_t u;
    memcpy(&u, &d, sizeof(u));
    return ((uint64_t)u << 32) | (uint64_t)(uint32_t)i;
}

/* points as three coordinate arrays (px, py, pz), queries as [Q,3] rows */
void oracle_knn(const float* px, const float* py, const float* pz, int64_t P, const float* queries, int64_t q0,
                int64_t q1, int32_t K, float* dists, int64_t* idx) {
    float d[BLOCK];
    uint64_t best[32];
    for (int64_t q = q0; q < q1; ++q) {
        const float qx = queries[3 * q], qy = queries[3 * q + 1], qz = queries[3 * q + 2];
        int n = 0;
        float worst = INFINITY;    /* d of best[K - 1] once the list is full: a cheap first filter */
        for (int64_t b = 0; b < P; b += BLOCK) {
            const int m = (int)(P - b < BLOCK ? P - b : BLOCK);
            for (int j = 0; j < m; ++j) {
                const float dx = qx - px[b + j], dy = qy - py[b + j], dz = qz - pz[b + j];
                d[j] = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
            }
            for (int j = 0; j < m; ++j) {
                if (n == K && !(d[j] <= worst)) continue;
                const uint64_t k = key_of(d[j], b + j);
                if (n == K && k >= best[K - 1]) continue;
                int at = n < K ? n++ : K - 1;
                while (at > 0 && best[at - 1] > k) { best[at] = best[at - 1]; --at; }
                best[at] = k;
                if (n == K) {
                    const uint32_t u = (uint32_t)(best[K - 1] >> 32);
                    memcpy(&worst, &u, sizeof(u));
                }
            }
        }
        for (int k = 0; k < K; ++k) {
            const uint32_t u = (uint32_t)(best[k] >> 32);
            memcpy(&dists[(q - q0) * K + k], &u, sizeof(u));
            idx[(q - q0) * K + k] = (int64_t)(uint32_t)best[k];
        }
    }
}
