/*
 * pf_tail_oracle.c — the PF / MCL step tail (normalise, N_eff gate, resample, refresh_cache) from raw weights.  TEST
 * INFRASTRUCTURE ONLY.  Includes oracle/pf_oracle.c unchanged and adds:
 *   orc_tail_normalize          normalize_weights + refresh_cache (pf.rs:331-332) on the particles' weights as raw likelihoods;
 *                               after orc_pf_set_particles, this and orc_pf_resample are a step's tail
 *   orc_tail_resample_runmax    orc_pf_resample of a fixed-size filter (MCL: n_particles == max_particles), every draw looked
 *                               up by a lower bound on the running maximum of the cumulative weights with NaN entries skipped
 *                               (-inf while none is finite).  r <= c_i first holds where that maximum first reaches r, so the
 *                               index is the linear scan's (pf.rs:459-465, mcl.rs:387-392) on any CDF, one that goes down or
 *                               turns NaN included, in O(log n) per draw.  tests/test_pf_tail_cases_oracle.py pins the two.
 */
#include "../../oracle/pf_oracle.c"

void orc_tail_normalize(orc_pf* f) {
    normalize_weights(f);
    refresh_cache(f);
}

int orc_tail_resample_runmax(orc_pf* f) {
    const size_t n = f->n;
    if (n == 0 || n != f->cfg.n_particles) return -1;
    if (f->cfg.mode == 0 && !(orc_pf_neff(f) < (double)f->cfg.n_particles * f->cfg.resample_threshold)) return 0;   /* pf.rs:337-345 */
    double* cum = (double*)malloc(sizeof(double) * n);
    double* mx = (double*)malloc(sizeof(double) * n);
    double cum_sum = 0.0, m = -INFINITY;
    for (size_t i = 0; i < n; ++i) { cum_sum += f->p[i].w; cum[i] = cum_sum; }
    if (f->cfg.mode == 1) cum[n - 1] = 1.0;                                         /* mcl.rs:334-336 */
    for (size_t i = 0; i < n; ++i) { if (cum[i] > m) m = cum[i]; mx[i] = m; }
    const size_t fallback = f->cfg.mode == 1 ? n - 1 : 0;                           /* pf.rs:459, mcl.rs:387-392 */
    for (size_t t = 0; t < n; ++t) {
        const double r = pfc_u01_53(pfc_blk_u64(pfc_rng_block(f->seed, PFC_STREAM_PF_RESAMPLE, f->n_resample, t), 0));
        size_t lo = 0, hi = n;
        while (lo < hi) { const size_t mid = lo + (hi - lo) / 2; if (!(r <= mx[mid])) lo = mid + 1; else hi = mid; }
        const size_t index = lo < n ? lo : fallback;
        f->scratch[t] = f->p[index];
        f->scratch[t].w = 1.0 / (double)n;
        f->last_idx[t] = (uint32_t)index;
    }
    orc_particle* tmp = f->p; f->p = f->scratch; f->scratch = tmp;
    f->last_idx_n = n;
    f->n_resample++;
    free(cum); free(mx);
    refresh_cache(f);
    return 1;
}
