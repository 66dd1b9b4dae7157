/*
 * pf_odom_math.h — the odometry motion model of the PF / MCL predict (DESIGN §3.14), shared by the library's host code, the CUDA
 * kernel (pf_kernels.cuh) and the test oracle (tests/host/pf_odom_oracle.c).  Not in the reference, whose filters only have the
 * velocity model (pf.rs:279-296, mcl.rs:236-253).  This is sample_motion_model_odometry (Thrun, Burgard and Fox, Probabilistic
 * Robotics, Table 5.6) in the form ROS AMCL ships as `diff-corrected`: the rotation noise uses the smaller of |rot| and
 * |rot - pi| (so reversing is not a half turn), and each sigma is the square root of Table 5.6's variance.
 *
 * Input: the previous and the current odometry pose o = (x, y, yaw), o' = (x', y', yaw') as odom6 = (o, o'), and alpha[4].
 * normalize = fs_normalize_angle, atan2 / sincos = the contract libm (pfc_atan2, pfc_sincos), sqrt = IEEE.  Every operation below
 * is one IEEE f64 operation in the order written (no contraction: nvcc --fmad=false, gcc -ffp-contract=off); a sum of three
 * terms is evaluated left to right.
 *
 * Once per call (pf_odom_increment), common to all particles:
 *   dx = x' - x, dy = y' - y, trans = sqrt(dx * dx + dy * dy)
 *   rot1 = trans < 0.01 ? 0 : normalize(atan2(dy, dx) - yaw)               AMCL's guard: no heading from a tiny translation
 *   rot2 = normalize(normalize(yaw' - yaw) - rot1)
 *   n1 = min(|normalize(rot1)|, |normalize(rot1 - pi)|), n2 likewise for rot2
 *   s_rot1  = sqrt(a1 * (n1 * n1) + a2 * (trans * trans))
 *   s_trans = sqrt((a3 * (trans * trans) + a4 * (n1 * n1)) + a4 * (n2 * n2))
 *   s_rot2  = sqrt(a1 * (n2 * n2) + a2 * (trans * trans))
 *
 * Per particle (pf_odom_move), with za, zb the pair of Philox block (seed, PFC_STREAM_PF_PREDICT, call, slot) and zc the first
 * normal of block (seed, PFC_STREAM_PF_ODOM, call, slot), call = the handle's predict counter, slot = the global slot:
 *   r1 = normalize(rot1 - (s_rot1 > 0 ? s_rot1 * za : 0))
 *   t  = trans - (s_trans > 0 ? s_trans * zb : 0)
 *   r2 = normalize(rot2 - (s_rot2 > 0 ? s_rot2 * zc : 0))
 *   (s, c) = sincos(yaw + r1);  x = x + t * c;  y = y + t * s;  yaw = yaw + normalize(r1 + r2)
 * The particle's yaw is not wrapped (as pf.rs:294 does not wrap it) and v is left as it was: odometry carries no velocity.  The
 * turn r1 + r2 is normalised before it is added: r1 and r2 are each wrapped into [-pi, pi], so when the robot reverses (rot1 near
 * +-pi) the noise flips some particles' r1 across the wrap and their plain sum is 2 pi off the others'.  Table 5.6 leaves that to
 * an estimate that averages yaw on the circle; this engine's estimate is the weighted linear mean of the unwrapped yaws (pf.rs:382-396),
 * so unnormalised, the cloud would split into copies 2 pi apart and the estimated heading would be wrong after every reverse.
 *
 * PF_ODOM_ATAN2 and PF_ODOM_SINCOS may be defined before inclusion (the oracle's glibc build does); the library never does.
 */
#ifndef PF_ODOM_MATH_H
#define PF_ODOM_MATH_H

#include "pf_contract_math.h"
#include "fs_ekf_math.h"                 /* fs_normalize_angle */

#ifndef PF_ODOM_ATAN2
#define PF_ODOM_ATAN2(y, x) pfc_atan2((y), (x))
#endif
#ifndef PF_ODOM_SINCOS
#define PF_ODOM_SINCOS(a, s, c) pfc_sincos((a), (s), (c))
#endif

/* below this translation the heading of the increment is not used (rot1 = 0) */
#define PF_ODOM_MIN_TRANS 0.01
/* the alphas a handle starts with: AMCL's odom_alpha1..4 defaults */
#define PF_ODOM_ALPHA_DEFAULT 0.2

/* what a predict needs of one odometry increment: the same for every particle */
typedef struct { double rot1, trans, rot2, s_rot1, s_trans, s_rot2; } PfOdom;

/* min(|normalize(a)|, |normalize(a - pi)|): the rotation a counts for in the noise, whether driving forward or reversing */
PFC_HD double pf_odom_rot_noise(double a) {
    const double d1 = fabs(fs_normalize_angle(a)), d2 = fabs(fs_normalize_angle(a - PFC_PI));
    return d2 < d1 ? d2 : d1;
}

/* 1 when every alpha is finite and >= 0 */
PFC_HD int pf_odom_alpha_ok(const double alpha[4]) {
    for (int j = 0; j < 4; ++j)
        if (!(alpha[j] >= 0.0 && alpha[j] <= 1.7976931348623157e308)) return 0;
    return 1;
}

/* the increment of odom6 = (x, y, yaw, x', y', yaw') under alpha; 0, or -1 when an odometry component is not finite */
PFC_HD int pf_odom_increment(const double odom6[6], const double alpha[4], PfOdom* m) {
    for (int j = 0; j < 6; ++j)
        if (!(fabs(odom6[j]) <= 1.7976931348623157e308)) return -1;
    const double dx = odom6[3] - odom6[0], dy = odom6[4] - odom6[1];
    const double trans = sqrt(dx * dx + dy * dy);
    const double rot1 = trans < PF_ODOM_MIN_TRANS ? 0.0 : fs_normalize_angle(PF_ODOM_ATAN2(dy, dx) - odom6[2]);
    const double rot2 = fs_normalize_angle(fs_normalize_angle(odom6[5] - odom6[2]) - rot1);
    const double n1 = pf_odom_rot_noise(rot1), n2 = pf_odom_rot_noise(rot2);
    const double tt = trans * trans, q1 = n1 * n1, q2 = n2 * n2;
    m->rot1 = rot1; m->trans = trans; m->rot2 = rot2;
    m->s_rot1 = sqrt(alpha[0] * q1 + alpha[1] * tt);
    m->s_trans = sqrt((alpha[2] * tt + alpha[3] * q1) + alpha[3] * q2);
    m->s_rot2 = sqrt(alpha[0] * q2 + alpha[1] * tt);
    return 0;
}

/* one particle's move by the increment m under the normals (za, zb, zc) */
PFC_HD void pf_odom_move(const PfOdom* m, double za, double zb, double zc, double* x, double* y, double* yaw) {
    const double r1 = fs_normalize_angle(m->rot1 - (m->s_rot1 > 0.0 ? m->s_rot1 * za : 0.0));
    const double t = m->trans - (m->s_trans > 0.0 ? m->s_trans * zb : 0.0);
    const double r2 = fs_normalize_angle(m->rot2 - (m->s_rot2 > 0.0 ? m->s_rot2 * zc : 0.0));
    double s, c;
    PF_ODOM_SINCOS(*yaw + r1, &s, &c);
    *x = *x + t * c;
    *y = *y + t * s;
    *yaw = *yaw + fs_normalize_angle(r1 + r2);
}

#endif /* PF_ODOM_MATH_H */
