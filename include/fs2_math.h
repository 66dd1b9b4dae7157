/*
 * fs2_math.h — the pose proposal of FastSLAM 2.0 for one particle: compute_proposal (fs2.rs:173-216) followed by
 * sample_pose_with_rng (fs2.rs:219-239) and set_pose (fs2.rs:77-81).  fs2.rs = crates/rust_robotics_slam/src/fastslam2.rs.
 * Shared by the CUDA kernel (fs2_propose_kernel, rust_robotics_b200/csrc/fs3.cuh) and a host test; every operation in the
 * reference's order, IEEE f64, the libm of pf_contract_math.h — bit-identical to oracle/fs2_oracle.c (the tests compare them).
 *
 * nalgebra 0.33 conventions (restated from upstream, SURVEY.md §8c): a product of static matrices accumulates each entry left
 * to right, ((a_i0 b_0j) + a_i1 b_1j) + a_i2 b_2j; try_inverse divides the adjugate by the determinant (None when it is
 * exactly 0); Cholesky works on the lower triangle, column by column, and fails on a zero / negative / NaN pivot.
 */
#ifndef FS2_MATH_H
#define FS2_MATH_H

#include "fs_ekf_math.h"

/* c = a b for 3x3 row-major arrays */
PFC_HD void fs2_mul33(const double* a, const double* b, double* c) {
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            double t = a[3 * i] * b[j];
            t = a[3 * i + 1] * b[3 + j] + t;
            t = a[3 * i + 2] * b[6 + j] + t;
            c[3 * i + j] = t;
        }
}
/* Matrix3::try_inverse: 1 on success */
PFC_HD int fs2_inv33(const double* m, double* o) {
    const double mi0 = m[4] * m[8] - m[7] * m[5];               /* minors of the first row */
    const double mi1 = m[3] * m[8] - m[6] * m[5];
    const double mi2 = m[3] * m[7] - m[6] * m[4];
    const double det = m[0] * mi0 - m[1] * mi1 + m[2] * mi2;
    if (det == 0.0) return 0;
    const pfc_rcp_t rd = pfc_rcp_make(det);                     /* nine IEEE quotients over one denominator */
    o[0] = pfc_div_by(mi0, rd);
    o[1] = pfc_div_by(m[2] * m[7] - m[8] * m[1], rd);
    o[2] = pfc_div_by(m[1] * m[5] - m[4] * m[2], rd);
    o[3] = pfc_div_by(-mi1, rd);
    o[4] = pfc_div_by(m[0] * m[8] - m[6] * m[2], rd);
    o[5] = pfc_div_by(m[2] * m[3] - m[5] * m[0], rd);
    o[6] = pfc_div_by(mi2, rd);
    o[7] = pfc_div_by(m[1] * m[6] - m[7] * m[0], rd);
    o[8] = pfc_div_by(m[0] * m[4] - m[3] * m[1], rd);
    return 1;
}

/* proposal + sample for one particle.  pose = (x, y, yaw) in/out; L = the landmark of the step's FIRST observation (z0, z1) as it
 * stands before this step's updates; (n0, n1, n2) = the three N(0,1) draws in the order sample_pose takes them (fs2.rs:234);
 * mc = the 3x3 MOTION_COV (fs2.rs:31). */
PFC_HD void fs2_propose_pose(double* px, double* py, double* pyaw, const FsLm* L, double u0, double u1, double dt, double z0, double z1,
                             double r00, double r11, const double* mc, double n0, double n1, double n2) {
    const double x = *px, y = *py, yaw = *pyaw;
    double sn, cs;
    pfc_sincos(yaw, &sn, &cs);
    /* motion_model fs2.rs:95-102 */
    const double xp0 = x + u0 * dt * cs, xp1 = y + u0 * dt * sn, xp2 = fs_normalize_angle(yaw + u1 * dt);
    /* p_pred = g * motion_cov * g^T  fs2.rs:184-186, g = motion_jacobian fs2.rs:105-120 */
    const double g[9] = { 1.0, 0.0, -u0 * dt * sn, 0.0, 1.0, u0 * dt * cs, 0.0, 0.0, 1.0 };
    const double gt[9] = { g[0], g[3], g[6], g[1], g[4], g[7], g[2], g[5], g[8] };
    double gm[9], cov[9], mean[3];
    fs2_mul33(g, mc, gm);
    fs2_mul33(gm, gt, cov);
    mean[0] = xp0; mean[1] = xp1; mean[2] = xp2;
    if (L->c00 < 100.0) {                                       /* is_initialized fs2.rs:49-51; otherwise the motion prior alone */
        const double dx = L->x - xp0, dy = L->y - xp1;
        const double d2 = dx * dx + dy * dy;
        const double d = sqrt(d2);
        /* h_pose = obs_jacobian_pose fs2.rs:141-148 (2x3), h_lm = obs_jacobian_landmark fs2.rs:132-138 (2x2) */
        const pfc_rcp_t rd = pfc_rcp_make(d), rd2 = pfc_rcp_make(d2);
        const double hp[6] = { pfc_div_by(-dx, rd), pfc_div_by(-dy, rd), 0.0, pfc_div_by(dy, rd2), pfc_div_by(-dx, rd2), -1.0 };
        const double h00 = pfc_div_by(dx, rd), h01 = pfc_div_by(dy, rd), h10 = pfc_div_by(-dy, rd2), h11 = pfc_div_by(dx, rd2);
        /* q_obs = h_lm * cov_lm * h_lm^T + r  fs2.rs:198 */
        const double a00 = h00 * L->c00 + h01 * L->c10, a01 = h00 * L->c01 + h01 * L->c11;
        const double a10 = h10 * L->c00 + h11 * L->c10, a11 = h10 * L->c01 + h11 * L->c11;
        const double q00 = (a00 * h00 + a01 * h01) + r00, q01 = (a00 * h10 + a01 * h11) + 0.0;
        const double q10 = (a10 * h00 + a11 * h01) + 0.0, q11 = (a10 * h10 + a11 * h11) + r11;
        const double qdet = q00 * q11 - q10 * q01;              /* try_inverse().unwrap_or(identity) fs2.rs:203 */
        double i00 = 1.0, i01 = 0.0, i10 = 0.0, i11 = 1.0;
        if (qdet != 0.0) {
            const pfc_rcp_t rq = pfc_rcp_make(qdet);
            i00 = pfc_div_by(q11, rq); i01 = pfc_div_by(-q01, rq); i10 = pfc_div_by(-q10, rq); i11 = pfc_div_by(q00, rq);
        }
        double ppi[9], ppost_inv[9], ppost[9];
        if (!fs2_inv33(cov, ppi)) {                             /* unwrap_or(identity * 1e-6) fs2.rs:205 */
            for (int e = 0; e < 9; ++e) ppi[e] = 0.0 * 1e-6;
            ppi[0] = ppi[4] = ppi[8] = 1.0 * 1e-6;
        }
        double hq[6];                                           /* h_pose^T * q_obs_inv: 3x2 */
        for (int i = 0; i < 3; ++i) {
            hq[2 * i] = hp[i] * i00 + hp[3 + i] * i10;
            hq[2 * i + 1] = hp[i] * i01 + hp[3 + i] * i11;
        }
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) ppost_inv[3 * i + j] = ppi[3 * i + j] + (hq[2 * i] * hp[j] + hq[2 * i + 1] * hp[3 + j]);   /* fs2.rs:206 */
        const int inv_ok = fs2_inv33(ppost_inv, ppost);         /* unwrap_or(p_pred) fs2.rs:207 */
        /* innovation at the predicted pose fs2.rs:210-211 */
        const double zp1 = fs_normalize_angle(pfc_atan2(dy, dx) - xp2);
        const double in0 = z0 - d, in1 = fs_normalize_angle(z1 - zp1);
        if (inv_ok) for (int e = 0; e < 9; ++e) cov[e] = ppost[e];
        /* x_post = x_pred + ((p_post * h_pose^T) * q_obs_inv) * innovation  fs2.rs:213 */
        for (int i = 0; i < 3; ++i) {
            double ph0 = cov[3 * i] * hp[0], ph1 = cov[3 * i] * hp[3];
            ph0 = cov[3 * i + 1] * hp[1] + ph0; ph1 = cov[3 * i + 1] * hp[4] + ph1;
            ph0 = cov[3 * i + 2] * hp[2] + ph0; ph1 = cov[3 * i + 2] * hp[5] + ph1;
            const double k0 = ph0 * i00 + ph1 * i10, k1 = ph0 * i01 + ph1 * i11;
            mean[i] = mean[i] + (k0 * in0 + k1 * in1);
        }
    }
    /* sample_pose: Cholesky factor of cov (lower triangle), or the square roots of its diagonal  fs2.rs:226-233 */
    double w[9], l[9];
    for (int e = 0; e < 9; ++e) { w[e] = cov[e]; l[e] = 0.0; }
    int ok = 1;
    for (int j = 0; j < 3 && ok; ++j) {
        for (int k = 0; k < j; ++k) {
            const double f = -w[3 * j + k];
            for (int i = j; i < 3; ++i) w[3 * i + j] = f * w[3 * i + k] + w[3 * i + j];
        }
        const double dg = w[3 * j + j];
        if (dg == 0.0 || !(dg >= 0.0)) { ok = 0; break; }
        const double den = sqrt(dg);
        w[3 * j + j] = den;
        const pfc_rcp_t rden = pfc_rcp_make(den);
        for (int i = j + 1; i < 3; ++i) w[3 * i + j] = pfc_div_by(w[3 * i + j], rden);
    }
    if (ok) { l[0] = w[0]; l[3] = w[3]; l[4] = w[4]; l[6] = w[6]; l[7] = w[7]; l[8] = w[8]; }
    else for (int i = 0; i < 3; ++i) { const double c = cov[4 * i]; l[4 * i] = sqrt(c > 0.0 ? c : 0.0); }
    double out[3];
    for (int i = 0; i < 3; ++i) {                               /* mean + l * noise  fs2.rs:236 */
        double t = l[3 * i] * n0;
        t = l[3 * i + 1] * n1 + t;
        t = l[3 * i + 2] * n2 + t;
        out[i] = mean[i] + t;
    }
    *px = out[0]; *py = out[1]; *pyaw = fs_normalize_angle(out[2]);   /* set_pose fs2.rs:77-81 */
}

/* The association metric of the unknown-correspondence step (DESIGN §3.5): the squared Mahalanobis distance y^T S^-1 y of
 * observation (z0, z1) from landmark L seen at pose (px, py, pyaw).  y and S are formed exactly as update_landmark_and_weight
 * forms them (fs2.rs:258-262), S^-1 as try_inverse forms it and the quadratic form in fs2.rs:275's order (the rule itself is
 * search_correspond_landmark_id of ekf_slam.rs:284-308).  Returns 0 when det S == 0 (try_inverse fails: the slot is skipped,
 * ekf_slam.rs:293), else 1 with the distance in *d2 (NaN / inf pass through).  The caller tests `cov00 < 100` first. */
PFC_HD int fs_assoc_d2(const FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11, double* d2out) {
    const double dx = L->x - px, dy = L->y - py;
    const double d2 = dx * dx + dy * dy;
    const double d = sqrt(d2);
    const double zp1 = fs_normalize_angle(pfc_atan2(dy, dx) - pyaw);
    const double y0 = z0 - d, y1 = fs_normalize_angle(z1 - zp1);
    const pfc_rcp_t rd = pfc_rcp_make(d), rd2 = pfc_rcp_make(d2);
    const double h00 = pfc_div_by(dx, rd), h01 = pfc_div_by(dy, rd), h10 = pfc_div_by(-dy, rd2), h11 = pfc_div_by(dx, rd2);
    const double p00 = L->c00, p01 = L->c01, p10 = L->c10, p11 = L->c11;
    const double a00 = h00 * p00 + h01 * p10, a01 = h00 * p01 + h01 * p11;
    const double a10 = h10 * p00 + h11 * p10, a11 = h10 * p01 + h11 * p11;
    const double s00 = (a00 * h00 + a01 * h01) + r00;
    const double s01 = (a00 * h10 + a01 * h11) + 0.0;
    const double s10 = (a10 * h00 + a11 * h01) + 0.0;
    const double s11 = (a10 * h10 + a11 * h11) + r11;
    const double det = s00 * s11 - s10 * s01;
    if (det == 0.0) return 0;
    const pfc_rcp_t rdet = pfc_rcp_make(det);
    const double i00 = pfc_div_by(s11, rdet), i01 = pfc_div_by(-s01, rdet), i10 = pfc_div_by(-s10, rdet), i11 = pfc_div_by(s00, rdet);
    const double t0 = y0 * i00 + y1 * i10, t1 = y0 * i01 + y1 * i11;
    *d2out = t0 * y0 + t1 * y1;
    return 1;
}

#endif
