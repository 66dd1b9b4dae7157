/*
 * pf_moments.h — the PF / MCL estimate and covariance (compute_estimate + compute_covariance, pf.rs:382-413), shared by the
 * CUDA kernels (pf_kernels.cuh, pf3.cuh) and by a host test (tests/host/pf_moments_test.c).
 *
 * The reference makes two passes: est = sum w p (not divided by sum w), then cov = sum w (p - est)(p - est)^T.  The device
 * makes one pass of weighted central moments (total weight W, weighted mean m, m2 = sum w (p - m)(p - m)^T), built with the
 * pairwise (Chan / West) update: one particle at a time within a thread, then partial against partial in a fixed tree.  Every
 * term that update adds is a product of deviations from a mean of the points merged so far, so nothing cancels however far
 * the cloud lies from the origin or from the previous estimate.  The result is then
 *
 *     est = W m,     cov = m2 + W (m - est)(m - est)^T        (sum w (p - m) = 0, so the cross terms vanish)
 *
 * which is the reference's definition for any total weight (W = n for weights all 1 gives its n * mean).
 *
 * Edges, as in the reference's sums:
 *   - a zero weight adds nothing, except that a non-finite coordinate of that pose turns the coordinate's mean (and so its
 *     estimate, covariance row and column) into NaN, like 0 * inf in sum w p;
 *   - all weights zero: est = 0, cov = 0;
 *   - a non-finite coordinate of a weighted pose leaves non-finite exactly that coordinate's estimate, row and column.
 * The update divides by the running total weight; it is meant for non-negative weights (a running total of exactly 0 after a
 * non-zero weight drops that weight's share of the mean).
 *
 * Compiled without contraction on both sides (nvcc --fmad=false, gcc -ffp-contract=off), so the host test replays the
 * device's reduction order bit for bit.
 */
#ifndef PF_MOMENTS_H
#define PF_MOMENTS_H

#include "pf_contract_math.h"

/* total weight, weighted mean of (x, y, yaw, v), sum w (p - m)(p - m)^T as the upper triangle (xx, xy, xyaw, xv, yy, yyaw,
 * yv, yawyaw, yawv, vv).  15 doubles, the layout of the per-block partials in device memory. */
typedef struct { double w, m[4], q[10]; } PfMom;
#define PF_MOM 15

/* a <- a (+) b.  An empty side (w == 0, m == 0, q == 0) is the identity for finite values. */
PFC_HD void pf_mom_merge(PfMom* a, const PfMom* b) {
    const double W = a->w + b->w;
    const double f = W != 0.0 ? b->w / W : 0.0, g = a->w * f;
    double d[4];
    for (int k = 0; k < 4; ++k) { d[k] = b->m[k] - a->m[k]; a->m[k] = a->m[k] + d[k] * f; }
    int q = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j) { a->q[q] = a->q[q] + b->q[q] + d[i] * d[j] * g; ++q; }
    a->w = W;
}

/* a <- a (+) one particle of weight w */
PFC_HD void pf_mom_add(PfMom* a, double w, double x, double y, double yaw, double v) {
    const PfMom b = { w, { x, y, yaw, v }, { 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 } };
    pf_mom_merge(a, &b);
}

/* est[4] = sum w p, cov[16] (row-major, symmetric) = sum w (p - est)(p - est)^T */
PFC_HD void pf_mom_final(const PfMom* a, double est[4], double cov[16]) {
    double dl[4];
    for (int k = 0; k < 4; ++k) { est[k] = a->w * a->m[k]; dl[k] = a->m[k] - est[k]; }
    int q = 0;
    for (int i = 0; i < 4; ++i)
        for (int j = i; j < 4; ++j) { const double c = a->q[q] + dl[i] * dl[j] * a->w; cov[i * 4 + j] = c; cov[j * 4 + i] = c; ++q; }
}

#endif
