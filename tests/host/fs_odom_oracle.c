/*
 * fs_odom_oracle.c — CPU oracle of FastSLAM's odometry motion model (DESIGN §3.15, the rule of include/fs_odom_math.h and
 * include/pfgpu.h pfgpu_fs_*_odom).  TEST INFRASTRUCTURE ONLY.  Includes tests/host/fs2_exist_oracle.c (and through it
 * fs2_assoc_oracle.c) unchanged for the association, update_landmark_and_weight and the existence counters, links liboracle for
 * normalise / N_eff / resample and sample_pose, and restates the rest in the header's operation order:
 *   the move      pf_odom_move (include/pf_odom_math.h, as the PF oracle uses it), then yaw wrapped
 *   the prior     mu = the move with zero normals; Sigma = (V D) V^T + eps I, V and D as the header writes them
 *   the proposal  compute_proposal's fusion (fs2.rs:188-216) from N(mu, Sigma + eps I), then sample_pose and set_pose
 *   the cases     every sigma 0: mu; the landmark not initialised (or no match): the move; else the proposal
 *   FastSLAM 1.0  the move, then update_landmark (fs1.rs:140-183) per observation
 * Draws: Philox (the FS_PREDICT pair; the third normal from FS_ODOM for the move, FS2_POSE3 for the proposal), or injected
 * (nz3: n x 3, the third column being whichever third normal the particle's case takes) so that
 * tests/golden/make_fs_odom_golden.py pins the arithmetic without Philox.  Built twice by tests/_fs_odom_oracle.py (contract math;
 * glibc libm with -DPF_ORACLE_LIBM, as Python's math module).
 */
#include "fs2_exist_oracle.c"

#ifdef PF_ORACLE_LIBM
#define PF_ODOM_ATAN2(y, x) atan2((y), (x))
#define PF_ODOM_SINCOS(a, s, c) (*(s) = sin(a), *(c) = cos(a))
#endif
#include "../../include/pf_odom_math.h"

#define FO_EPS 1e-8
enum { FO_STILL = 0, FO_MOVE = 1, FO_PROPOSE = 2 };

static void fo_move(const PfOdom* m, double za, double zb, double zc, double* x, double* y, double* yaw) {
    pf_odom_move(m, za, zb, zc, x, y, yaw);
    *yaw = orc_fs_normalize_angle(*yaw);
}

/* mean3 = mu, cov9 = Sigma + eps I (row-major) at pose3 */
static void fo_prior(const PfOdom* m, const double pose3[3], double mean3[3], double cov9[9]) {
    const double s = M_SIN(pose3[2] + m->rot1), c = M_COS(pose3[2] + m->rot1), t = m->trans;
    mean3[0] = pose3[0]; mean3[1] = pose3[1]; mean3[2] = pose3[2];
    fo_move(m, 0.0, 0.0, 0.0, &mean3[0], &mean3[1], &mean3[2]);
    const double V[3][3] = { { -(t * s), c, 0.0 }, { t * c, s, 0.0 }, { 1.0, 0.0, 1.0 } };
    const double D[3] = { m->s_rot1 * m->s_rot1, m->s_trans * m->s_trans, m->s_rot2 * m->s_rot2 };
    double VD[3][3];
    for (int i = 0; i < 3; ++i)                      /* (V D): the zero entries of D take part, as in a full 3x3 product */
        for (int j = 0; j < 3; ++j) {
            double acc = V[i][0] * (j == 0 ? D[0] : 0.0);
            acc = V[i][1] * (j == 1 ? D[1] : 0.0) + acc;
            acc = V[i][2] * (j == 2 ? D[2] : 0.0) + acc;
            VD[i][j] = acc;
        }
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double acc = VD[i][0] * V[j][0];
            acc = VD[i][1] * V[j][1] + acc;
            acc = VD[i][2] * V[j][2] + acc;
            cov9[3 * i + j] = acc;
        }
    cov9[0] = cov9[0] + FO_EPS; cov9[4] = cov9[4] + FO_EPS; cov9[8] = cov9[8] + FO_EPS;
}

static int fo_case(const PfOdom* m, const lm_t* L) {
    if (m->s_rot1 == 0.0 && m->s_trans == 0.0 && m->s_rot2 == 0.0) return FO_STILL;
    return L->c00 < 100.0 ? FO_PROPOSE : FO_MOVE;
}

/* Matrix3::try_inverse (fs2_oracle.c's m3_try_inverse, restated on row-major arrays): 1 on success */
static int fo_inv33(const double* a, double* o) {
    const double mi0 = a[4] * a[8] - a[7] * a[5], mi1 = a[3] * a[8] - a[6] * a[5], mi2 = a[3] * a[7] - a[6] * a[4];
    const double det = a[0] * mi0 - a[1] * mi1 + a[2] * mi2;
    if (det == 0.0) return 0;
    o[0] = mi0 / det; o[1] = (a[2] * a[7] - a[8] * a[1]) / det; o[2] = (a[1] * a[5] - a[4] * a[2]) / det;
    o[3] = -mi1 / det; o[4] = (a[0] * a[8] - a[6] * a[2]) / det; o[5] = (a[2] * a[3] - a[5] * a[0]) / det;
    o[6] = mi2 / det; o[7] = (a[1] * a[6] - a[7] * a[0]) / det; o[8] = (a[0] * a[4] - a[3] * a[1]) / det;
    return 1;
}

/* compute_proposal fs2.rs:188-216 from the prior (mean, cov): mean and cov become the posterior's */
static void fo_fuse(const orc_fs_config* cf, const lm_t* lm, double z0, double z1, double mean[3], double cov[9]) {
    const double dx = lm->x - mean[0], dy = lm->y - mean[1];
    const double d2 = dx * dx + dy * dy;
    const double d = sqrt(d2);
    const double hp[2][3] = { { -dx / d, -dy / d, 0.0 }, { dy / d2, -dx / d2, -1.0 } };
    const double hl[2][2] = { { dx / d, dy / d }, { -dy / d2, dx / d2 } };
    const double p00 = lm->c00, p01 = lm->c01, p10 = lm->c10, p11 = lm->c11;
    const double a00 = hl[0][0] * p00 + hl[0][1] * p10, a01 = hl[0][0] * p01 + hl[0][1] * p11;
    const double a10 = hl[1][0] * p00 + hl[1][1] * p10, a11 = hl[1][0] * p01 + hl[1][1] * p11;
    const double q00 = (a00 * hl[0][0] + a01 * hl[0][1]) + cf->r00;
    const double q01 = (a00 * hl[1][0] + a01 * hl[1][1]) + 0.0;
    const double q10 = (a10 * hl[0][0] + a11 * hl[0][1]) + 0.0;
    const double q11 = (a10 * hl[1][0] + a11 * hl[1][1]) + cf->r11;
    const double qdet = q00 * q11 - q10 * q01;
    double qi[2][2];
    if (qdet == 0.0) { qi[0][0] = 1.0; qi[0][1] = 0.0; qi[1][0] = 0.0; qi[1][1] = 1.0; }
    else { qi[0][0] = q11 / qdet; qi[0][1] = -q01 / qdet; qi[1][0] = -q10 / qdet; qi[1][1] = q00 / qdet; }
    double ppi[9], pinv[9], post[9];
    if (!fo_inv33(cov, ppi))
        for (int e = 0; e < 9; ++e) ppi[e] = (e % 4 == 0 ? 1.0 : 0.0) * 1e-6;
    double hq[3][2];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 2; ++j) hq[i][j] = hp[0][i] * qi[0][j] + hp[1][i] * qi[1][j];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) pinv[3 * i + j] = ppi[3 * i + j] + (hq[i][0] * hp[0][j] + hq[i][1] * hp[1][j]);
    if (!fo_inv33(pinv, post)) for (int e = 0; e < 9; ++e) post[e] = cov[e];
    const double zp1 = orc_fs_normalize_angle(M_ATAN2(dy, dx) - mean[2]);
    const double in0 = z0 - d, in1 = orc_fs_normalize_angle(z1 - zp1);
    for (int i = 0; i < 3; ++i) {
        double ph0 = post[3 * i] * hp[0][0], ph1 = post[3 * i] * hp[1][0];
        ph0 = post[3 * i + 1] * hp[0][1] + ph0; ph1 = post[3 * i + 1] * hp[1][1] + ph1;
        ph0 = post[3 * i + 2] * hp[0][2] + ph0; ph1 = post[3 * i + 2] * hp[1][2] + ph1;
        const double k0 = ph0 * qi[0][0] + ph1 * qi[1][0], k1 = ph0 * qi[0][1] + ph1 * qi[1][1];
        mean[i] = mean[i] + (k0 * in0 + k1 * in1);
    }
    for (int e = 0; e < 9; ++e) cov[e] = post[e];
}

/* FastSLAM 2.0's pose of one particle: pose3 in/out, n3 = (FS_PREDICT pair, the third normal of the case) */
static void fo_pose2(const orc_fs_config* cf, const PfOdom* m, int kase, const lm_t* L, double z0, double z1, const double n3[3], double pose3[3]) {
    if (kase == FO_STILL) { fo_move(m, 0.0, 0.0, 0.0, &pose3[0], &pose3[1], &pose3[2]); return; }
    if (kase == FO_MOVE) { fo_move(m, n3[0], n3[1], n3[2], &pose3[0], &pose3[1], &pose3[2]); return; }
    double mean[3], cov[9], out[3];
    fo_prior(m, pose3, mean, cov);
    fo_fuse(cf, L, z0, z1, mean, cov);
    orc_fs2_sample_pose(mean, cov, n3, out);
    pose3[0] = out[0]; pose3[1] = out[1]; pose3[2] = orc_fs_normalize_angle(out[2]);    /* set_pose fs2.rs:77-81 */
}

/* update_landmark fs1.rs:140-183 (fs1_oracle.c's, restated: it is static there) */
static void fo_update_fs1(orc_fs* f, size_t i, double z0, double z1, size_t lm_id) {
    lm_t* L = &f->lm[i * f->m + lm_id];
    const double px = f->x[i], py = f->y[i], pyaw = f->yaw[i];
    if (L->c00 > 100.0) {
        L->x = px + z0 * M_COS(pyaw + z1);
        L->y = py + z0 * M_SIN(pyaw + z1);
        return;
    }
    const double dx = L->x - px, dy = L->y - py;
    const double d = sqrt(dx * dx + dy * dy);
    const double zp1 = orc_fs_normalize_angle(M_ATAN2(dy, dx) - pyaw);
    const double y0 = z0 - d, y1 = orc_fs_normalize_angle(z1 - zp1);
    const double d2 = dx * dx + dy * dy, dd = sqrt(d2);
    const double h00 = dx / dd, h01 = dy / dd, h10 = -dy / d2, h11 = dx / d2;
    const double p00 = L->c00, p01 = L->c01, p10 = L->c10, p11 = L->c11;
    const double a00 = h00 * p00 + h01 * p10, a01 = h00 * p01 + h01 * p11;
    const double a10 = h10 * p00 + h11 * p10, a11 = h10 * p01 + h11 * p11;
    const double s00 = (a00 * h00 + a01 * h01) + f->cfg.r00, s01 = (a00 * h10 + a01 * h11) + 0.0;
    const double s10 = (a10 * h00 + a11 * h01) + 0.0, s11 = (a10 * h10 + a11 * h11) + f->cfg.r11;
    const double det = s00 * s11 - s10 * s01;
    double i00, i01, i10, i11;
    if (det == 0.0) { i00 = 1.0; i01 = 0.0; i10 = 0.0; i11 = 1.0; }
    else { i00 = s11 / det; i01 = -s01 / det; i10 = -s10 / det; i11 = s00 / det; }
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
    if (det > 0.0) {
        const double t0 = y0 * i00 + y1 * i10, t1 = y0 * i01 + y1 * i11;
        f->w[i] *= M_EXP(-0.5 * (t0 * y0 + t1 * y1)) / (2.0 * PFC_PI * sqrt(det));
    }
}

/* the three normals of particle i for a case: injected, or Philox */
static void fo_draws(const orc_fs* f, size_t i, int kase, const double* nz3, double n3[3]) {
    if (nz3) { n3[0] = nz3[3 * i]; n3[1] = nz3[3 * i + 1]; n3[2] = nz3[3 * i + 2]; return; }
    double unused;
    pfc_normal_pair(pfc_rng_block(f->seed, PFC_STREAM_FS_PREDICT, f->n_step, (uint64_t)i), &n3[0], &n3[1]);
    pfc_normal_pair(pfc_rng_block(f->seed, kase == FO_PROPOSE ? PFC_STREAM_FS2_POSE3 : PFC_STREAM_FS_ODOM, f->n_step, (uint64_t)i), &n3[2], &unused);
}

/* normalise, N_eff, gate and resample (the tail of every step), tau cloned with its particle when e != NULL */
static int fo_tail(orc_fs* f, orc_ex* e, const double* u01) {
    orc_fs_normalize_weights_(f);
    const double neff = orc_fs_compute_neff_(f);
    f->last_neff = neff;
    f->n_step++;
    if (!(neff < f->cfg.nth)) { f->last_idx_n = 0; return 0; }
    orc_fs_resample_(f, u01 ? *u01 : pfc_u01_52(pfc_blk_u64(pfc_rng_block(f->seed, PFC_STREAM_FS_RESAMPLE, f->n_resample, 0), 0)));
    f->n_resample++;
    if (e && f->m) {
        int32_t* t2 = malloc(f->n * f->m * sizeof(int32_t));
        for (size_t i = 0; i < f->n; ++i) memcpy(t2 + i * f->m, e->tau + (size_t)f->last_idx[i] * f->m, f->m * sizeof(int32_t));
        memcpy(e->tau, t2, f->n * f->m * sizeof(int32_t));
        free(t2);
    }
    return 1;
}

/* ------------------------------------------------ exported ------------------------------------------------ */
int orc_fo_increment(const double odom6[6], const double alpha4[4], double out6[6]) {
    PfOdom m;
    if (!pf_odom_alpha_ok(alpha4) || pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    out6[0] = m.rot1; out6[1] = m.trans; out6[2] = m.rot2; out6[3] = m.s_rot1; out6[4] = m.s_trans; out6[5] = m.s_rot2;
    return 0;
}
/* the prior at pose3: mean3, cov9 */
int orc_fo_prior(const double odom6[6], const double alpha4[4], const double pose3[3], double mean3[3], double cov9[9]) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    fo_prior(&m, pose3, mean3, cov9);
    return 0;
}
/* FastSLAM 1.0's move of pose3 (in/out) under n3 */
int orc_fo_move(const double odom6[6], const double alpha4[4], const double n3[3], double pose3[3]) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    fo_move(&m, n3[0], n3[1], n3[2], &pose3[0], &pose3[1], &pose3[2]);
    return 0;
}
/* FastSLAM 2.0's pose of one particle (pose3 in/out) against landmark lm6 and observation (z0, z1); returns the case */
int orc_fo_pose2(const orc_fs_config* cf, const double odom6[6], const double alpha4[4], const double lm6[6], double z0, double z1,
                 const double n3[3], double pose3[3]) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    const lm_t L = { lm6[0], lm6[1], lm6[2], lm6[3], lm6[4], lm6[5] };
    const int kase = fo_case(&m, &L);
    fo_pose2(cf, &m, kase, &L, z0, z1, n3, pose3);
    return kase;
}

/* pfgpu_fs_step_odom: known ids; nz3 NULL = Philox (u01 unused), else injected; returns 1 if it resampled, -1 when refused */
int orc_fo_step(orc_fs* f, const double odom6[6], const double alpha4[4], const orc_fs_obs* z, size_t k, const double* nz3, double u01) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    const long n = (long)f->n;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1)
    for (long i = 0; i < n; ++i) {
        double pose[3] = { f->x[i], f->y[i], f->yaw[i] }, n3[3];
        if (f->variant == 2 && k > 0) {
            const lm_t* L = &f->lm[(size_t)i * f->m + (size_t)z[0].lm_id];
            const int kase = fo_case(&m, L);
            fo_draws(f, (size_t)i, kase, nz3, n3);
            fo_pose2(&f->cfg, &m, kase, L, z[0].d, z[0].angle, n3, pose);
        } else {
            fo_draws(f, (size_t)i, FO_MOVE, nz3, n3);
            fo_move(&m, n3[0], n3[1], n3[2], &pose[0], &pose[1], &pose[2]);
        }
        f->x[i] = pose[0]; f->y[i] = pose[1]; f->yaw[i] = pose[2];
        for (size_t j = 0; j < k; ++j) {
            if (z[j].lm_id >= f->m) continue;
            if (f->variant == 2) f->w[i] *= update_landmark_and_weight(f, (size_t)i, z[j].d, z[j].angle, (size_t)z[j].lm_id);
            else fo_update_fs1(f, (size_t)i, z[j].d, z[j].angle, (size_t)z[j].lm_id);
        }
    }
    return fo_tail(f, NULL, nz3 ? &u01 : NULL);
}

/* pfgpu_fs_step_unknown_odom (variant 2); e NULL: no existence counters.  counts = (matched, born, dropped), *removed = copies removed */
int orc_fo_step_unknown(orc_fs* f, orc_ex* e, const double odom6[6], const double alpha4[4], const double* z2, size_t k, double gate_d2,
                        const double* nz3, double u01, uint64_t counts[3], uint64_t* removed) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    if (k == 0 && !e) {                                     /* the known-id step with k = 0 */
        counts[0] = counts[1] = counts[2] = 0; *removed = 0;
        return orc_fo_step(f, odom6, alpha4, NULL, 0, nz3, u01);
    }
    const long n = (long)f->n;
    uint64_t c0 = 0, c1 = 0, c2 = 0, c3 = 0;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1) reduction(+ : c0, c1, c2, c3)
    for (long i = 0; i < n; ++i) {
        double pose[3] = { f->x[i], f->y[i], f->yaw[i] }, n3[3];
        if (k > 0) {
            double mu[3] = { pose[0], pose[1], pose[2] };
            fo_move(&m, 0.0, 0.0, 0.0, &mu[0], &mu[1], &mu[2]);
            const long l = associate(f, (size_t)i, mu[0], mu[1], mu[2], z2[0], z2[1], gate_d2);
            const lm_t fresh = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
            const lm_t* L = l >= 0 ? &f->lm[(size_t)i * f->m + (size_t)l] : &fresh;
            const int kase = fo_case(&m, L);
            fo_draws(f, (size_t)i, kase, nz3, n3);
            fo_pose2(&f->cfg, &m, kase, L, z2[0], z2[1], n3, pose);
        } else {
            fo_draws(f, (size_t)i, FO_MOVE, nz3, n3);
            fo_move(&m, n3[0], n3[1], n3[2], &pose[0], &pose[1], &pose[2]);
        }
        f->x[i] = pose[0]; f->y[i] = pose[1]; f->yaw[i] = pose[2];
        int32_t* tau = e ? e->tau + (size_t)i * f->m : NULL;
        unsigned char* seen = calloc(f->m ? f->m : 1, 1);
        for (size_t j = 0; j < k; ++j) {
            const double z0 = z2[2 * j], z1 = z2[2 * j + 1];
            long l = associate(f, (size_t)i, f->x[i], f->y[i], f->yaw[i], z0, z1, gate_d2);
            if (l >= 0) { c0++; if (tau) tau[l] += 1; }
            else {
                for (size_t q = 0; q < f->m && l < 0; ++q) if (!(f->lm[(size_t)i * f->m + q].c00 < 100.0)) l = (long)q;
                if (l < 0) { c2++; continue; }
                c1++;
                if (tau) tau[l] = 1;
            }
            seen[l] = 1;
            f->w[i] *= update_landmark_and_weight(f, (size_t)i, z0, z1, (size_t)l);
        }
        if (tau)
            for (size_t l = 0; l < f->m; ++l) {                 /* negative evidence at the sampled pose (fs2_exist_oracle.c's rule) */
                lm_t* L = &f->lm[(size_t)i * f->m + l];
                if (seen[l] || !(L->c00 < 100.0)) continue;
                const double dx = L->x - f->x[i], dy = L->y - f->y[i];
                if (sqrt(dx * dx + dy * dy) <= e->range && --tau[l] < 0) {
                    const lm_t fresh = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
                    *L = fresh;
                    c3++;
                }
            }
        free(seen);
    }
    counts[0] = c0; counts[1] = c1; counts[2] = c2;
    *removed = c3;
    if (e) e->removed = c3;
    return fo_tail(f, e, nz3 ? &u01 : NULL);
}
