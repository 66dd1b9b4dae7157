/*
 * gs_prop_math.h — the arithmetic of grid FastSLAM's scan-matched proposal (GMapping's improved proposal, Grisetti, Stachniss and
 * Burgard, IEEE T-RO 23(1), 2007; DESIGN §3.17; the rule is stated at pfgpu_gs_proposal in include/pfgpu.h).  Shared by the CUDA
 * kernel (gs_propose_kernel, rust_robotics_b200/csrc/gslam.cuh), the library's host code and the test oracle
 * (tests/host/gs_prop_oracle.c).  Not in the reference.  Every operation is one IEEE f64 operation in the order written (nvcc
 * --fmad=false, gcc -ffp-contract=off); a sum runs left to right from 0.
 *
 * What is here: the still test, the normaliser c of eta, the lattice offsets, the quadratic form of the prior, and the lattice
 * moments with the sample.  The sample is fs2_propose_pose itself with a landmark that is not initialised (c00 = 100) and a zero
 * control: its motion model is then the identity and nothing is fused, so it is FastSLAM 2.0's Cholesky factor (with its diagonal
 * fallback), its sample mean + L n and set_pose's yaw wrap, in its order, of the lattice's N(x^ + m_o, C).
 */
#ifndef GS_PROP_MATH_H
#define GS_PROP_MATH_H

#include "fs_odom_math.h"

/* the exp of pi_j: the contract exp (the oracle's glibc build defines it as exp before inclusion) */
#ifndef GS_PROP_EXP
#define GS_PROP_EXP(x) pfc_exp(x)
#endif

/* the lattice covariance's diagonal floor: the prior's (FS_ODOM_EPS) */
#define GS_PROP_EPS FS_ODOM_EPS
/* the largest lattice half-width k: (2k + 1)^3 = 343 points */
#define GS_PROP_MAX_K 3
/* the most match candidates (2 n_l + 1)^2 (2 n_a + 1) a particle may have, and the most yaws (2 n_a + 1) */
#define GS_PROP_MAX_CAND 2048
#define GS_PROP_MAX_YAWS 1024

/* m stands still: every sigma 0 (fs2_odom_case's FS_ODOM_STILL) */
PFC_HD int gs_prop_still(const PfOdom* m) { return m->s_rot1 == 0.0 && m->s_trans == 0.0 && m->s_rot2 == 0.0; }

/* c = (kl * kl * ka) / sqrt((2 pi)^3 det Sigma_0), Sigma_0 = fs_odom_prior's covariance with (s, c) = (0, 1), i.e. at yaw + rot1 = 0,
 * and its determinant expanded along the first row as fs2_inv33 expands it.  Computed once per step (host). */
PFC_HD double gs_prop_norm(const PfOdom* m, double kl, double ka) {
    const double t = m->trans;
    const double v[9] = { -(t * 0.0), 1.0, 0.0, t * 1.0, 0.0, 0.0, 1.0, 0.0, 1.0 };
    const double vt[9] = { v[0], v[3], v[6], v[1], v[4], v[7], v[2], v[5], v[8] };
    const double dg[9] = { m->s_rot1 * m->s_rot1, 0.0, 0.0, 0.0, m->s_trans * m->s_trans, 0.0, 0.0, 0.0, m->s_rot2 * m->s_rot2 };
    double vd[9], s[9];
    fs2_mul33(v, dg, vd);
    fs2_mul33(vd, vt, s);
    s[0] = s[0] + FS_ODOM_EPS;
    s[4] = s[4] + FS_ODOM_EPS;
    s[8] = s[8] + FS_ODOM_EPS;
    const double mi0 = s[4] * s[8] - s[7] * s[5], mi1 = s[3] * s[8] - s[6] * s[5], mi2 = s[3] * s[7] - s[6] * s[4];
    const double det = s[0] * mi0 - s[1] * mi1 + s[2] * mi2;
    const double tp = 2.0 * PFC_PI;
    return ((kl * kl) * ka) / sqrt(((tp * tp) * tp) * det);
}

/* offsets (a, b, e) of point j of a window with half-widths (nl, nl, na), loop order a, b, e (e fastest, CSM's order) */
PFC_HD void gs_prop_index(int j, int nl, int na, int* a, int* b, int* e) {
    const int NL = 2 * nl + 1, NA = 2 * na + 1;
    *e = j % NA - na;
    *b = (j / NA) % NL - nl;
    *a = j / (NA * NL) - nl;
}

/* d^T A d: t_i = (A[3i] d0 + A[3i+1] d1) + A[3i+2] d2 (fs2_mul33's order), then (d0 t0 + d1 t1) + d2 t2 */
PFC_HD double gs_prop_quad(const double* A, const double* d) {
    double t[3];
    for (int i = 0; i < 3; ++i) {
        double u = A[3 * i] * d[0];
        u = A[3 * i + 1] * d[1] + u;
        u = A[3 * i + 2] * d[2] + u;
        t[i] = u;
    }
    double q = d[0] * t[0];
    q = d[1] * t[1] + q;
    q = d[2] * t[2] + q;
    return q;
}

/* tau_j of lattice point j: x_j = (xh0 + a kl, xh1 + b kl, normalize(xh2 + e ka)), d_j = x_j - mu (yaw difference normalised),
 * tau_j = L_j * exp(-0.5 * d_j^T A d_j) (contract exp) */
PFC_HD double gs_prop_tau(int j, int k, double kl, double ka, const double* xh, const double* mu, const double* A, double Lj) {
    int a, b, e;
    gs_prop_index(j, k, k, &a, &b, &e);
    const double x = xh[0] + (double)a * kl, y = xh[1] + (double)b * kl, yaw = fs_normalize_angle(xh[2] + (double)e * ka);
    const double d[3] = { x - mu[0], y - mu[1], fs_normalize_angle(yaw - mu[2]) };
    return Lj * GS_PROP_EXP(-0.5 * gs_prop_quad(A, d));
}

/* Steps 3 and 4 of the rule from tau[0 .. K-1] (lattice order): T = sum tau_j, *eta = c * T.  0 (the fallback) when eta is not a
 * normal number; else 1 with the sampled pose in pose[3]:
 *   m_o = (sum tau_j o_j) / T;  C = (sum tau_j (o_j - m_o)(o_j - m_o)^T) / T + eps I, upper triangle accumulated as (tau u_i) u_k
 *   pose = fs2_propose_pose from (xh0 + m_o0, xh1 + m_o1, normalize(xh2 + m_o2)) with covariance C and normals (n0, n1, n2) */
PFC_HD int gs_prop_sample(const double* tau, int k, double kl, double ka, const double* xh, double c, double n0, double n1, double n2,
                          double* pose, double* eta) {
    const int S = 2 * k + 1, K = S * S * S;
    double T = 0.0;
    for (int j = 0; j < K; ++j) T = T + tau[j];
    *eta = c * T;
    if (!(*eta >= 2.2250738585072014e-308 && *eta <= 1.7976931348623157e308)) return 0;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0;
    for (int j = 0; j < K; ++j) {
        int a, b, e;
        gs_prop_index(j, k, k, &a, &b, &e);
        s0 = s0 + tau[j] * ((double)a * kl);
        s1 = s1 + tau[j] * ((double)b * kl);
        s2 = s2 + tau[j] * ((double)e * ka);
    }
    const double m0 = s0 / T, m1 = s1 / T, m2 = s2 / T;
    double c00 = 0.0, c01 = 0.0, c02 = 0.0, c11 = 0.0, c12 = 0.0, c22 = 0.0;
    for (int j = 0; j < K; ++j) {
        int a, b, e;
        gs_prop_index(j, k, k, &a, &b, &e);
        const double u0 = (double)a * kl - m0, u1 = (double)b * kl - m1, u2 = (double)e * ka - m2;
        const double v0 = tau[j] * u0, v1 = tau[j] * u1, v2 = tau[j] * u2;
        c00 = c00 + v0 * u0; c01 = c01 + v0 * u1; c02 = c02 + v0 * u2;
        c11 = c11 + v1 * u1; c12 = c12 + v1 * u2; c22 = c22 + v2 * u2;
    }
    const double C01 = c01 / T, C02 = c02 / T, C12 = c12 / T;
    const double C[9] = { c00 / T + GS_PROP_EPS, C01, C02, C01, c11 / T + GS_PROP_EPS, C12, C02, C12, c22 / T + GS_PROP_EPS };
    const FsLm none = { 0.0, 0.0, 100.0, 0.0, 0.0, 100.0 };
    pose[0] = xh[0] + m0;
    pose[1] = xh[1] + m1;
    pose[2] = fs_normalize_angle(xh[2] + m2);
    fs2_propose_pose(&pose[0], &pose[1], &pose[2], &none, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, C, n0, n1, n2);
    return 1;
}

#endif /* GS_PROP_MATH_H */
