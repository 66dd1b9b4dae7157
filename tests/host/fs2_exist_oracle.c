/*
 * fs2_exist_oracle.c — CPU oracle of the landmark existence counters (DESIGN §3.7) on the unknown-association step of
 * fs2_assoc_oracle.c, which it includes unchanged (association, update and the library's proposal / normalise / resample).
 * TEST INFRASTRUCTURE ONLY.  Per slot an int tau, cloned with the particle on resample: a match sets tau += 1, a birth tau = 1;
 * then every initialised slot no observation of the step went to, within `range` of the sampled pose (sqrt(dx*dx + dy*dy) <=
 * range, get_observations' test fs2.rs:400-406), gets tau -= 1, and below 0 it is removed (create_particles' fresh landmark).
 * k = 0 steps run the same pass after the motion step.  Built twice by tests/_exist_oracle.py, like fs2_assoc_oracle.c.
 */
#include "fs2_assoc_oracle.c"
#include <stdlib.h>
#include <string.h>

typedef struct { int32_t* tau; size_t n, m; double range; uint64_t removed; } orc_ex;   /* tau [n][m] */

static void particle_exist(orc_fs* f, size_t i, const double u[2], const double* z2, size_t k, double gate_d2, const double nz[3],
                           uint64_t cnt[3], int32_t* tau, double range, uint64_t* rem) {
    const double pose[3] = { f->x[i], f->y[i], f->yaw[i] };                  /* the pose: particle_unknown's, restated */
    double np[3];
    if (k > 0) {
        const double xp0 = pose[0] + u[0] * f->cfg.dt * M_COS(pose[2]), xp1 = pose[1] + u[0] * f->cfg.dt * M_SIN(pose[2]);
        const double xp2 = orc_fs_normalize_angle(pose[2] + u[1] * f->cfg.dt);
        const long l = associate(f, i, xp0, xp1, xp2, z2[0], z2[1], gate_d2);
        const lm_t fresh = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
        const lm_t* L = l >= 0 ? &f->lm[i * f->m + (size_t)l] : &fresh;
        const double lm6[6] = { L->x, L->y, L->c00, L->c01, L->c10, L->c11 };
        double mean[3], cov[9];
        orc_fs2_compute_proposal(&f->cfg, pose, u, z2[0], z2[1], lm6, mean, cov);
        orc_fs2_sample_pose(mean, cov, nz, np);
    } else {                                                                  /* fs2.rs:347-356 */
        const double un0 = u[0] + nz[0] * sqrt(f->cfg.q00), un1 = u[1] + nz[1] * sqrt(f->cfg.q11);
        np[0] = pose[0] + un0 * f->cfg.dt * M_COS(pose[2]);
        np[1] = pose[1] + un0 * f->cfg.dt * M_SIN(pose[2]);
        np[2] = orc_fs_normalize_angle(pose[2] + un1 * f->cfg.dt);
    }
    f->x[i] = np[0]; f->y[i] = np[1]; f->yaw[i] = orc_fs_normalize_angle(np[2]);
    unsigned char* seen = calloc(f->m ? f->m : 1, 1);
    for (size_t j = 0; j < k; ++j) {
        const double z0 = z2[2 * j], z1 = z2[2 * j + 1];
        long l = associate(f, i, f->x[i], f->y[i], f->yaw[i], z0, z1, gate_d2);
        if (l >= 0) { cnt[0]++; tau[l] += 1; }
        else {
            for (size_t e = 0; e < f->m && l < 0; ++e) if (!(f->lm[i * f->m + e].c00 < 100.0)) l = (long)e;
            if (l < 0) { cnt[2]++; continue; }                                /* map full: dropped */
            cnt[1]++; tau[l] = 1;
        }
        seen[l] = 1;
        f->w[i] *= update_landmark_and_weight(f, i, z0, z1, (size_t)l);
    }
    for (size_t l = 0; l < f->m; ++l) {                                       /* negative evidence at the sampled pose */
        lm_t* L = &f->lm[i * f->m + l];
        if (seen[l] || !(L->c00 < 100.0)) continue;
        const double dx = L->x - f->x[i], dy = L->y - f->y[i];
        if (sqrt(dx * dx + dy * dy) <= range && --tau[l] < 0) {
            const lm_t fresh = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
            *L = fresh;
            (*rem)++;
        }
    }
    free(seen);
}

/* step_unknown with counters; nz0 == NULL: the Philox draws, else injected (nz0[i], nz1[i], nz1[n + i]) and u01 */
static int step_exist(orc_fs* f, orc_ex* e, const double u[2], const double* z2, size_t k, double gate_d2, const double* nz0,
                      const double* nz1, const double* r01, uint64_t counts[3], uint64_t* removed) {
    const long n = (long)f->n;
    const uint32_t call = f->n_step;
    uint64_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1) reduction(+ : c0, c1, c2, c3)
    for (long i = 0; i < n; ++i) {
        double a[3], dummy;
        if (nz0) { a[0] = nz0[i]; a[1] = nz1[i]; a[2] = nz1[n + i]; }
        else {
            pfc_normal_pair(pfc_rng_block(f->seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)i), &a[0], &a[1]);
            pfc_normal_pair(pfc_rng_block(f->seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)i), &a[2], &dummy);
        }
        uint64_t c[3] = { 0, 0, 0 }, r = 0;
        particle_exist(f, (size_t)i, u, z2, k, gate_d2, a, c, e->tau + (size_t)i * f->m, e->range, &r);
        c0 += c[0]; c1 += c[1]; c2 += c[2]; c3 += r;
    }
    counts[0] = c0; counts[1] = c1; counts[2] = c2;
    *removed = e->removed = c3;
    orc_fs_normalize_weights_(f);
    const double neff = orc_fs_compute_neff_(f);
    f->last_neff = neff;
    f->n_step++;
    if (!(neff < f->cfg.nth)) { f->last_idx_n = 0; return 0; }
    orc_fs_resample_(f, r01 ? *r01 : pfc_u01_52(pfc_blk_u64(pfc_rng_block(f->seed, PFC_STREAM_FS_RESAMPLE, f->n_resample, 0), 0)));
    f->n_resample++;
    if (f->m) {                                                               /* tau is cloned with its particle */
        int32_t* t2 = malloc(f->n * f->m * sizeof(int32_t));
        for (size_t i = 0; i < f->n; ++i) memcpy(t2 + i * f->m, e->tau + (size_t)f->last_idx[i] * f->m, f->m * sizeof(int32_t));
        memcpy(e->tau, t2, f->n * f->m * sizeof(int32_t));
        free(t2);
    }
    return 1;
}

/* a counter set for f's shape, every tau = 1 (enable; orc_fs2_ex_reset: what upload / seed_map do) */
orc_ex* orc_fs2_ex_new(const orc_fs* f, double range) {
    orc_ex* e = calloc(1, sizeof(orc_ex));
    e->n = f->n; e->m = f->m; e->range = range;
    e->tau = malloc((f->n * f->m > 0 ? f->n * f->m : 1) * sizeof(int32_t));
    for (size_t j = 0; j < f->n * f->m; ++j) e->tau[j] = 1;
    return e;
}
void orc_fs2_ex_free(orc_ex* e) { if (e) { free(e->tau); free(e); } }
void orc_fs2_ex_reset(orc_ex* e) { for (size_t j = 0; j < e->n * e->m; ++j) e->tau[j] = 1; e->removed = 0; }
int orc_fs2_step_unknown_ex(orc_fs* f, orc_ex* e, const double u[2], const double* z2, size_t k, double gate_d2, const double* nz0,
                            const double* nz1, double u01, uint64_t counts[3], uint64_t* removed) {
    return step_exist(f, e, u, z2, k, gate_d2, nz0, nz1, nz0 ? &u01 : NULL, counts, removed);
}
/* out [n][m]: tau, 0 for an empty slot */
void orc_fs2_ex_counts(const orc_fs* f, const orc_ex* e, int32_t* out) {
    for (size_t j = 0; j < f->n * f->m; ++j) out[j] = f->lm[j].c00 < 100.0 ? e->tau[j] : 0;
}
