/* Host replay of the PF / MCL estimate (include/pf_moments.h) in the device's reduction order, bit for bit: the same merge
 * routine compiled without contraction, the same particle-to-thread assignment, the same shuffle and warp trees.
 *
 *   form 0  pf_moments_kernel (`blocks` CTAs, thread t takes particles t, t + blocks * NT, ...) + pf_moments_reduce_kernel
 *           (thread t takes block partials t, t + NT, ...); a sharded engine does this per rank on its contiguous n / shards
 *           slots and merges the ranks' results in rank order (pf_moments_final_kernel)
 *   form 1  pf3_post_kernel (`blocks` tiles, thread tid of tile b takes particles b * NT * K + tid * K + 0 .. K - 1; the last
 *           CTA's thread t takes tile t)
 */
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/pf_moments.h"

#define NT 256

static const PfMom EMPTY = { 0.0, { 0.0, 0.0, 0.0, 0.0 }, { 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 } };

/* pf_mom_block_merge: __shfl_down_sync by 16, 8, 4, 2, 1 (lane l merges lane l + o; only lanes below o feed lane 0 later),
 * then thread 0 merges the warps' lane 0 in warp order */
static PfMom block_merge(PfMom* v /* [NT] */) {
    for (int w = 0; w < NT / 32; ++w)
        for (int o = 16; o > 0; o >>= 1)
            for (int l = 0; l < o; ++l) pf_mom_merge(&v[32 * w + l], &v[32 * w + l + o]);
    PfMom r = v[0];
    for (int w = 1; w < NT / 32; ++w) pf_mom_merge(&r, &v[32 * w]);
    return r;
}

static void add(PfMom* v, const double* a5, size_t i) { pf_mom_add(v, a5[5 * i + 4], a5[5 * i], a5[5 * i + 1], a5[5 * i + 2], a5[5 * i + 3]); }

static PfMom form0(const double* a5, size_t n, unsigned blocks, PfMom* th, PfMom* part) {
    for (unsigned b = 0; b < blocks; ++b) {
        for (unsigned t = 0; t < NT; ++t) {
            th[t] = EMPTY;
            for (size_t i = (size_t)b * NT + t; i < n; i += (size_t)blocks * NT) add(&th[t], a5, i);
        }
        part[b] = block_merge(th);
    }
    for (unsigned t = 0; t < NT; ++t) {
        th[t] = EMPTY;
        for (unsigned b = t; b < blocks; b += NT) pf_mom_merge(&th[t], &part[b]);
    }
    return block_merge(th);
}

static PfMom form1(const double* a5, size_t n, unsigned tiles, unsigned K, PfMom* th, PfMom* part) {
    const size_t T = (size_t)NT * K;
    for (unsigned b = 0; b < tiles; ++b) {
        for (unsigned t = 0; t < NT; ++t) {
            th[t] = EMPTY;
            const size_t g0 = (size_t)b * T + (size_t)t * K;
            for (unsigned k = 0; k < K && g0 + k < n; ++k) add(&th[t], a5, g0 + k);
        }
        part[b] = block_merge(th);
    }
    for (unsigned t = 0; t < NT; ++t) th[t] = t < tiles ? part[t] : EMPTY;
    return block_merge(th);
}

/* aos5: n rows (x, y, yaw, v, w).  Returns 0, or -1 on a bad shape (form 1 holds at most NT tiles). */
int pf_moments_replay(const double* aos5, size_t n, int form, unsigned blocks, unsigned K, unsigned shards, double est[4], double cov[16]) {
    if (blocks < 1 || shards < 1 || n % shards != 0 || (form == 1 && (blocks > NT || shards != 1 || K < 1))) return -1;
    PfMom* th = (PfMom*)malloc(NT * sizeof(PfMom));
    PfMom* part = (PfMom*)malloc((size_t)(blocks > NT ? blocks : NT) * sizeof(PfMom));
    PfMom r;
    if (form == 1) r = form1(aos5, n, blocks, K, th, part);
    else {
        const size_t nl = n / shards;
        for (unsigned s = 0; s < shards; ++s) {
            const PfMom m = form0(aos5 + 5 * nl * s, nl, blocks, th, part);
            if (s == 0) r = m; else pf_mom_merge(&r, &m);
        }
    }
    free(th); free(part);
    pf_mom_final(&r, est, cov);
    return 0;
}
