/*
 * fs2_assoc_oracle.c — CPU oracle of the FastSLAM 2.0 step with UNKNOWN data association (DESIGN §3.5).  TEST INFRASTRUCTURE
 * ONLY, like oracle/ (see oracle/oracle.h), and built against it: the particle set is oracle/fs_state.h's, the proposal, the pose
 * sample, normalise, N_eff and resample are liboracle's own exported routines.  What this file restates is the new part:
 *
 *   association  A(pose, z) = argmin over the slots with cov00 < 100 (fs2.rs:49-51), in ascending index, of the squared
 *                Mahalanobis distance y^T S^-1 y, y and S formed as update_landmark_and_weight forms them (fs2.rs:258-262); a
 *                slot whose det S == 0 is skipped (try_inverse fails, ekf_slam.rs:293); strict `<` against a best that starts
 *                at f64::MAX, so the first minimum wins and NaN / inf / f64::MAX never do; the winner only if best < gate_d2
 *                (the rule of search_correspond_landmark_id, ekf_slam.rs:284-308, with M_DIST_TH^2 = 16 by default)
 *   proposal     compute_proposal (fs2.rs:173-216) with the landmark A(x_pred, z[0]) picks at the noise-free prediction x_pred,
 *                or its uninitialised branch (the motion prior) when there is none
 *   updates      for each observation in order: A at the sampled pose against the map as the earlier observations left it;
 *                matched -> update_landmark_and_weight on that slot; else a birth in the lowest slot with !(cov00 < 100);
 *                no such slot -> the observation is dropped (weight and map unchanged)
 *
 * Built twice by tests/_assoc_oracle.py, like liboracle: contract math (linked to liboracle.so) and glibc libm
 * (-DPF_ORACLE_LIBM, linked to liboracle_libm.so).
 */
#include "../../oracle/fs_state.h"
#include <float.h>

/* update_landmark_and_weight fs2.rs:242-280 for slot l of particle i; returns the weight factor */
static double update_landmark_and_weight(orc_fs* f, size_t i, double z0, double z1, size_t l) {
    lm_t* L = &f->lm[i * f->m + l];
    const double px = f->x[i], py = f->y[i], pyaw = f->yaw[i];
    if (!(L->c00 < 100.0)) {                                                  /* fs2.rs:250-256 */
        L->x = px + z0 * M_COS(pyaw + z1);
        L->y = py + z0 * M_SIN(pyaw + z1);
        L->c00 = 10.0; L->c01 = 0.0; L->c10 = 0.0; L->c11 = 10.0;
        return 1.0;
    }
    const double dx = L->x - px, dy = L->y - py;
    const double d = sqrt(dx * dx + dy * dy);
    const double y0 = z0 - d, y1 = orc_fs_normalize_angle(z1 - orc_fs_normalize_angle(M_ATAN2(dy, dx) - pyaw));
    const double d2 = dx * dx + dy * dy, dd = sqrt(d2);
    const double h00 = dx / dd, h01 = dy / dd, h10 = -dy / d2, h11 = dx / d2;
    const double p00 = L->c00, p01 = L->c01, p10 = L->c10, p11 = L->c11;
    const double a00 = h00 * p00 + h01 * p10, a01 = h00 * p01 + h01 * p11;
    const double a10 = h10 * p00 + h11 * p10, a11 = h10 * p01 + h11 * p11;
    const double s00 = (a00 * h00 + a01 * h01) + f->cfg.r00, s01 = (a00 * h10 + a01 * h11) + 0.0;
    const double s10 = (a10 * h00 + a11 * h01) + 0.0, s11 = (a10 * h10 + a11 * h11) + f->cfg.r11;
    const double det = s00 * s11 - s10 * s01;
    double i00 = 1.0, i01 = 0.0, i10 = 0.0, i11 = 1.0;
    if (det != 0.0) { i00 = s11 / det; i01 = -s01 / det; i10 = -s10 / det; i11 = s00 / det; }
    const double b00 = p00 * h00 + p01 * h01, b01 = p00 * h10 + p01 * h11;
    const double b10 = p10 * h00 + p11 * h01, b11 = p10 * h10 + p11 * h11;
    const double k00 = b00 * i00 + b01 * i10, k01 = b00 * i01 + b01 * i11;
    const double k10 = b10 * i00 + b11 * i10, k11 = b10 * i01 + b11 * i11;
    L->x += k00 * y0 + k01 * y1;
    L->y += k10 * y0 + k11 * y1;
    const double m00 = 1.0 - (k00 * h00 + k01 * h10), m01 = 0.0 - (k00 * h01 + k01 * h11);
    const double m10 = 0.0 - (k10 * h00 + k11 * h10), m11 = 1.0 - (k10 * h01 + k11 * h11);
    L->c00 = m00 * p00 + m01 * p10; L->c01 = m00 * p01 + m01 * p11;
    L->c10 = m10 * p00 + m11 * p10; L->c11 = m10 * p01 + m11 * p11;
    if (det > 0.0) {                                                          /* fs2.rs:273-279 (det_s is det) */
        const double t0 = y0 * i00 + y1 * i10, t1 = y0 * i01 + y1 * i11;
        return M_EXP(-0.5 * (t0 * y0 + t1 * y1)) / (2.0 * PFC_PI * sqrt(det));
    }
    return 1e-10;
}

/* the metric: 0 when det S == 0 (skip), else 1 and y^T S^-1 y */
static int assoc_d2(const orc_fs_config* c, const lm_t* L, double px, double py, double pyaw, double z0, double z1, double* out) {
    const double dx = L->x - px, dy = L->y - py;
    const double d = sqrt(dx * dx + dy * dy);
    const double y0 = z0 - d, y1 = orc_fs_normalize_angle(z1 - orc_fs_normalize_angle(M_ATAN2(dy, dx) - pyaw));
    const double d2 = dx * dx + dy * dy, dd = sqrt(d2);
    const double h00 = dx / dd, h01 = dy / dd, h10 = -dy / d2, h11 = dx / d2;
    const double a00 = h00 * L->c00 + h01 * L->c10, a01 = h00 * L->c01 + h01 * L->c11;
    const double a10 = h10 * L->c00 + h11 * L->c10, a11 = h10 * L->c01 + h11 * L->c11;
    const double s00 = (a00 * h00 + a01 * h01) + c->r00, s01 = (a00 * h10 + a01 * h11) + 0.0;
    const double s10 = (a10 * h00 + a11 * h01) + 0.0, s11 = (a10 * h10 + a11 * h11) + c->r11;
    const double det = s00 * s11 - s10 * s01;
    if (det == 0.0) return 0;
    const double i00 = s11 / det, i01 = -s01 / det, i10 = -s10 / det, i11 = s00 / det;
    const double t0 = y0 * i00 + y1 * i10, t1 = y0 * i01 + y1 * i11;
    *out = t0 * y0 + t1 * y1;
    return 1;
}

/* A(pose, z) over particle i's map: the slot, or -1 for none */
static long associate(const orc_fs* f, size_t i, double px, double py, double pyaw, double z0, double z1, double gate_d2) {
    double best = DBL_MAX;
    long bl = -1;
    for (size_t l = 0; l < f->m; ++l) {
        const lm_t* L = &f->lm[i * f->m + l];
        double q;
        if (!(L->c00 < 100.0) || !assoc_d2(&f->cfg, L, px, py, pyaw, z0, z1, &q)) continue;
        if (q < best) { best = q; bl = (long)l; }
    }
    return bl >= 0 && best < gate_d2 ? bl : -1;
}

static void particle_unknown(orc_fs* f, size_t i, const double u[2], const double* z2, size_t k, double gate_d2,
                             double n0, double n1, double n2, uint64_t cnt[3]) {
    const double pose[3] = { f->x[i], f->y[i], f->yaw[i] };
    double np[3];
    if (k > 0) {
        const double yaw = pose[2];                                           /* motion_model fs2.rs:95-102: x_pred */
        const double xp0 = pose[0] + u[0] * f->cfg.dt * M_COS(yaw), xp1 = pose[1] + u[0] * f->cfg.dt * M_SIN(yaw);
        const double xp2 = orc_fs_normalize_angle(pose[2] + u[1] * f->cfg.dt);
        const long l = associate(f, i, xp0, xp1, xp2, z2[0], z2[1], gate_d2);
        const lm_t fresh = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
        const lm_t* L = l >= 0 ? &f->lm[i * f->m + (size_t)l] : &fresh;
        const double lm6[6] = { L->x, L->y, L->c00, L->c01, L->c10, L->c11 }, n3[3] = { n0, n1, n2 };
        double mean[3], cov[9];
        orc_fs2_compute_proposal(&f->cfg, pose, u, z2[0], z2[1], lm6, mean, cov);
        orc_fs2_sample_pose(mean, cov, n3, np);
    } else {                                                                  /* fs2.rs:347-356 */
        const double un0 = u[0] + n0 * sqrt(f->cfg.q00), un1 = u[1] + n1 * sqrt(f->cfg.q11);
        np[0] = pose[0] + un0 * f->cfg.dt * M_COS(pose[2]);
        np[1] = pose[1] + un0 * f->cfg.dt * M_SIN(pose[2]);
        np[2] = orc_fs_normalize_angle(pose[2] + un1 * f->cfg.dt);
    }
    f->x[i] = np[0]; f->y[i] = np[1]; f->yaw[i] = orc_fs_normalize_angle(np[2]);   /* set_pose fs2.rs:77-81 */
    for (size_t j = 0; j < k; ++j) {
        const double z0 = z2[2 * j], z1 = z2[2 * j + 1];
        long l = associate(f, i, f->x[i], f->y[i], f->yaw[i], z0, z1, gate_d2);
        if (l >= 0) cnt[0]++;
        else {
            for (size_t e = 0; e < f->m && l < 0; ++e) if (!(f->lm[i * f->m + e].c00 < 100.0)) l = (long)e;
            if (l < 0) { cnt[2]++; continue; }                                /* map full: dropped */
            cnt[1]++;
        }
        f->w[i] *= update_landmark_and_weight(f, i, z0, z1, (size_t)l);
    }
}

static int step_unknown(orc_fs* f, const double u[2], const double* z2, size_t k, double gate_d2, const double* nz0,
                        const double* nz1, const double* r01, uint64_t counts[3]) {
    const long n = (long)f->n;
    const uint64_t seed = f->seed;
    const uint32_t call = f->n_step;
    uint64_t c0 = 0, c1 = 0, c2 = 0;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1) reduction(+ : c0, c1, c2)
    for (long i = 0; i < n; ++i) {
        double a0, a1, a2, dummy;
        if (nz0) { a0 = nz0[i]; a1 = nz1[i]; a2 = nz1[n + i]; }
        else {
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)i), &a0, &a1);
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)i), &a2, &dummy);
        }
        uint64_t c[3] = { 0, 0, 0 };
        particle_unknown(f, (size_t)i, u, z2, k, gate_d2, a0, a1, a2, c);
        c0 += c[0]; c1 += c[1]; c2 += c[2];
    }
    if (counts) { counts[0] = c0; counts[1] = c1; counts[2] = c2; }
    orc_fs_normalize_weights_(f);                                             /* fs2.rs:368-373 */
    const double neff = orc_fs_compute_neff_(f);
    f->last_neff = neff;
    f->n_step++;
    if (neff < f->cfg.nth) {
        const double u01 = r01 ? *r01 : pfc_u01_52(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_FS_RESAMPLE, f->n_resample, 0), 0));
        orc_fs_resample_(f, u01);
        f->n_resample++;
        return 1;
    }
    f->last_idx_n = 0;
    return 0;
}

/* one step; z2 = k (d, angle) pairs; counts = (matched, born, dropped) summed over the particles; returns 1 if it resampled */
int orc_fs2_step_unknown(orc_fs* f, const double u[2], const double* z2, size_t k, double gate_d2, uint64_t counts[3]) {
    return step_unknown(f, u, z2, k, gate_d2, NULL, NULL, NULL, counts);
}
/* the same with injected draws: nz0[i], nz1[i] and nz1[n + i] are particle i's three N(0,1), u01 the resample's uniform */
int orc_fs2_step_unknown_with_noise(orc_fs* f, const double u[2], const double* z2, size_t k, double gate_d2, const double* nz0,
                                    const double* nz1, double u01, uint64_t counts[3]) {
    return step_unknown(f, u, z2, k, gate_d2, nz0, nz1, &u01, counts);
}
/* probe of the metric (lm6 = x, y, c00, c01, c10, c11): 0 = skipped (det S == 0) */
int orc_fs2_assoc_d2(const orc_fs_config* c, const double lm6[6], const double pose3[3], double z0, double z1, double* d2) {
    const lm_t L = { lm6[0], lm6[1], lm6[2], lm6[3], lm6[4], lm6[5] };
    return assoc_d2(c, &L, pose3[0], pose3[1], pose3[2], z0, z1, d2);
}
