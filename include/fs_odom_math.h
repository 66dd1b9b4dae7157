/*
 * fs_odom_math.h — the odometry motion model of every FastSLAM step path (DESIGN §3.15), shared by the library's host code, the
 * CUDA kernels (fs3.cuh, fs3_assoc.cuh) and the test oracle (tests/host/fs_odom_oracle.c).  Not in the reference, whose FastSLAM
 * modules only have the velocity model (fs1.rs:123-137, fs2.rs:95-120).  It is include/pf_odom_math.h's model (Probabilistic
 * Robotics Table 5.6, ROS AMCL's diff-corrected noise) applied to FastSLAM's particles, plus the prior FastSLAM 2.0's proposal
 * fuses with the first observation.  Arithmetic as in pf_odom_math.h: one IEEE f64 operation each, in the order written.
 *
 * Once per call (host): m = pf_odom_increment(odom6, alpha), unchanged.
 *
 * The move (FastSLAM 1.0, FastSLAM 2.0 without observations, and FastSLAM 2.0 when the first observation's landmark is not
 * initialised, i.e. the proposal has nothing to fuse): pf_odom_move(m, za, zb, zc, x, y, yaw), then yaw = normalize(yaw).  FastSLAM
 * poses stay wrapped (fs1.rs:76, set_pose fs2.rs:77-81).  (za, zb) = the pair of Philox block (seed, PFC_STREAM_FS_PREDICT, call,
 * global slot), the pair the velocity model draws; zc = the first normal of block (seed, PFC_STREAM_FS_ODOM, call, global slot).
 * Standing still (odom' == odom) every sigma is 0, every guarded term is 0 and the pose comes back as it was.
 *
 * The proposal (FastSLAM 2.0 with observations, known or unknown association): fs2_propose_pose's fusion with the first
 * observation, Cholesky, sample and set_pose, in its order, from the prior N(mu, Sigma + eps I) (see fs2_odom_pose):
 *   mu     = the move with za = zb = zc = 0, yaw wrapped
 *   (s, c) = sincos(yaw + rot1)            (the particle's yaw before the move; the same argument the move passes to sincos)
 *   V      = [ -t*s  c  0 ]                 d(x, y, yaw) / d(rot1, trans, rot2) at the particle, t = trans
 *            [  t*c  s  0 ]                 (-t*s and t*c: one product each, the negation applied to t*s)
 *            [  1    0  1 ]
 *   D      = diag(s_rot1 * s_rot1, s_trans * s_trans, s_rot2 * s_rot2)
 *   Sigma  = (V D) V^T, both products in fs2_mul33's order; then each diagonal entry + eps
 * with the three normals of the velocity proposal: the FS_PREDICT pair and the first normal of PFC_STREAM_FS2_POSE3.
 *   - Every sigma 0 (standing still, or all alphas 0): the pose takes mu.  No proposal, no sampling, no draw.
 *   - eps = FS_ODOM_EPS = 1e-8 (a standard deviation of 0.1 mm / 0.1 mrad).  A turn in place (t = 0) leaves V of rank 2, and
 *     the reference's fallback for a singular prior (try_inverse().unwrap_or(I * 1e-6), fs2.rs:205) is a prior PRECISION of 1e-6,
 *     i.e. a standard deviation of 1 km: the floor keeps the prior invertible and its null direction a tenth of a millimetre wide.
 *   - The first observation's landmark not initialised (cov00 >= 100; for unknown association: no slot matched): the move above,
 *     with zc from FS_ODOM: the prior alone is the motion model, and the move is its exact sample.
 *
 * Which case a particle takes depends on m and on the landmark only; fs2_odom_case says which, and which third normal it draws.
 */
#ifndef FS_ODOM_MATH_H
#define FS_ODOM_MATH_H

#include "pf_odom_math.h"
#include "fs2_math.h"

/* the diagonal floor of the proposal's prior covariance (see above) */
#define FS_ODOM_EPS 1e-8

/* FastSLAM 1.0's odometry move (and FastSLAM 2.0's without a landmark to fuse): pf_odom_move, yaw wrapped */
PFC_HD void fs_odom_move(const PfOdom* m, double za, double zb, double zc, double* x, double* y, double* yaw) {
    pf_odom_move(m, za, zb, zc, x, y, yaw);
    *yaw = fs_normalize_angle(*yaw);
}

/* the prior of the proposal at pose (x, y, yaw): mean[3] = mu, cov[9] = Sigma + eps I (row-major) */
PFC_HD void fs_odom_prior(const PfOdom* m, double x, double y, double yaw, double* mean, double* cov) {
    double s, c;
    PF_ODOM_SINCOS(yaw + m->rot1, &s, &c);
    mean[0] = x; mean[1] = y; mean[2] = yaw;
    fs_odom_move(m, 0.0, 0.0, 0.0, &mean[0], &mean[1], &mean[2]);
    const double t = m->trans;
    const double v[9] = { -(t * s), c, 0.0, t * c, s, 0.0, 1.0, 0.0, 1.0 };
    const double vt[9] = { v[0], v[3], v[6], v[1], v[4], v[7], v[2], v[5], v[8] };
    const double dg[9] = { m->s_rot1 * m->s_rot1, 0.0, 0.0, 0.0, m->s_trans * m->s_trans, 0.0, 0.0, 0.0, m->s_rot2 * m->s_rot2 };
    double vd[9];
    fs2_mul33(v, dg, vd);
    fs2_mul33(vd, vt, cov);
    cov[0] = cov[0] + FS_ODOM_EPS;
    cov[4] = cov[4] + FS_ODOM_EPS;
    cov[8] = cov[8] + FS_ODOM_EPS;
}

/* the FastSLAM 2.0 cases: STILL takes mu (no draw), MOVE is fs_odom_move (third normal from PFC_STREAM_FS_ODOM), PROPOSE samples the
 * proposal (third normal from PFC_STREAM_FS2_POSE3) */
enum { FS_ODOM_STILL = 0, FS_ODOM_MOVE = 1, FS_ODOM_PROPOSE = 2 };
PFC_HD int fs2_odom_case(const PfOdom* m, const FsLm* L) {
    if (m->s_rot1 == 0.0 && m->s_trans == 0.0 && m->s_rot2 == 0.0) return FS_ODOM_STILL;
    return L->c00 < 100.0 ? FS_ODOM_PROPOSE : FS_ODOM_MOVE;   /* is_initialized fs2.rs:49-51 */
}

/* FastSLAM 2.0's pose with odometry: pose in/out; L, (z0, z1) as fs2_propose_pose; kase = fs2_odom_case(m, L); (n0, n1) = the
 * FS_PREDICT pair, n2 = the first normal of the stream kase names (unused for STILL).  PROPOSE is fs2_propose_pose itself, from mu
 * with u = (0, 0), dt = 0 and MOTION_COV := Sigma + eps I: its motion model is then the identity (mu + 0, normalize(yaw + 0)) and its
 * jacobian G = I, so its prior is N(mu, Sigma + eps I) exactly (up to the sign of a zero) and the fusion, the Cholesky factor, the
 * sample and set_pose are its own, in its order. */
PFC_HD void fs2_odom_pose(int kase, const PfOdom* m, double* px, double* py, double* pyaw, const FsLm* L, double z0, double z1,
                          double r00, double r11, double n0, double n1, double n2) {
    if (kase == FS_ODOM_STILL) { fs_odom_move(m, 0.0, 0.0, 0.0, px, py, pyaw); return; }
    if (kase == FS_ODOM_MOVE) { fs_odom_move(m, n0, n1, n2, px, py, pyaw); return; }
    double mean[3], cov[9];
    fs_odom_prior(m, *px, *py, *pyaw, mean, cov);
    *px = mean[0]; *py = mean[1]; *pyaw = mean[2];
    fs2_propose_pose(px, py, pyaw, L, 0.0, 0.0, 0.0, z0, z1, r00, r11, cov, n0, n1, n2);
}

#endif /* FS_ODOM_MATH_H */
