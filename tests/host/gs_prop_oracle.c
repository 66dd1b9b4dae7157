/*
 * gs_prop_oracle.c — CPU oracle of grid FastSLAM's scan-matched proposal (DESIGN §3.17, the rule at pfgpu_gs_proposal in
 * include/pfgpu.h).  TEST INFRASTRUCTURE ONLY.  The sequential statement: gs_oracle.c, included unchanged, for the state, the
 * weight, the normalise, the fuse and the resample; per particle the prior, the match (every candidate in loop order, the winner
 * kept by CSM's total order), the lattice and the sample of include/gs_prop_math.h, or the fallback (gs_oracle.c's move and
 * weight).  Draws: Philox, or injected per slot (za, zb, zc, n2): (za, zb) the FS_PREDICT pair, zc the FS_ODOM normal of the
 * fallback, n2 the FS2_POSE3 normal of the proposal.  Built twice by tests/_gs_prop_oracle.py (contract math; glibc with
 * -DPF_ORACLE_LIBM).
 */
#include "gs_oracle.c"

#ifdef PF_ORACLE_LIBM
#define GS_PROP_EXP(x) exp(x)
#endif
#include "../../include/gs_prop_math.h"

/* the proposal: match range / step, lattice k, kl, ka, min_hits */
enum { P_LR, P_LS, P_AR, P_AS, P_K, P_KL, P_KA, P_MINH };

/* w_raw of one pose (orc_gs_weight's arithmetic) and its hits: used beams whose window has a cell inside with l* > 0 */
static double prop_weight(const orc_gs* g, const double* grid, double x, double y, double yaw, const double* pairs, size_t k,
                          double angle_min, int* hits) {
    const double q_out = g->model[G_ZRAND] / g->model[G_MAXR];
    const int R = (int)g->model[G_R];
    double wr = 1.0;
    int h = 0;
    for (size_t j = 0; j < k; ++j) {
        const double r = pairs[2 * j], angle = (yaw + angle_min) + pairs[2 * j + 1];
        const double ex = x + r * M_COS(angle), ey = y + r * M_SIN(angle);
        const int64_t cx = sat_i32(floor(ex / g->cfg[C_RES] + (double)g->W / 2.0)), cy = sat_i32(floor(ey / g->cfg[C_RES] + (double)g->H / 2.0));
        int any = 0;
        double best = -INFINITY;
        for (int64_t ix = cx - R; ix <= cx + R; ++ix)
            for (int64_t iy = cy - R; iy <= cy + R; ++iy) {
                if (ix < 0 || ix >= (int64_t)g->W || iy < 0 || iy >= (int64_t)g->H) continue;
                any = 1;
                const double l = grid[ix * (int64_t)g->H + iy];
                if (l > best) best = l;
            }
        wr = wr * (any ? g->model[G_ZHIT] * (1.0 - 1.0 / (1.0 + M_EXP(best))) + q_out : q_out);
        h += (any && best > 0.0) ? 1 : 0;
    }
    *hits = h;
    return wr;
}

/* slot i's move and weight under the proposal; xh[3] and *eta NaN unless computed; returns took */
static int prop_particle(orc_gs* g, size_t i, const PfOdom* m, const double* P, double c, const double* pairs, size_t k,
                         double angle_min, const double* z4, double* xh, double* eta) {
    const double* grid = g->grid + i * g->cells;
    xh[0] = xh[1] = xh[2] = *eta = NAN;
    double mu[3], cov[9], A[9];
    fs_odom_prior(m, g->x[i], g->y[i], g->yaw[i], mu, cov);
    if (!gs_prop_still(m) && fs2_inv33(cov, A)) {
        const int nl = (int)round(P[P_LR] / P[P_LS]), na = (int)round(P[P_AR] / P[P_AS]);
        const int n = (2 * nl + 1) * (2 * nl + 1) * (2 * na + 1);
        double bs = -1.0, bp = INFINITY;
        int bh = 0;
        for (int j = 0; j < n; ++j) {                           /* loop order: the first of equals stays */
            int a, b, e, h;
            gs_prop_index(j, nl, na, &a, &b, &e);
            const double x = mu[0] + (double)a * P[P_LS], y = mu[1] + (double)b * P[P_LS];
            const double yaw = fs_normalize_angle(mu[2] + (double)e * P[P_AS]);
            const double s = prop_weight(g, grid, x, y, yaw, pairs, k, angle_min, &h);
            const double dx = (double)a * P[P_LS], dy = (double)b * P[P_LS], dyaw = (double)e * P[P_AS];
            const double pen = (dx * dx + dy * dy) + dyaw * dyaw;
            if (s > bs || (s == bs && pen < bp)) { bs = s; bp = pen; bh = h; xh[0] = x; xh[1] = y; xh[2] = yaw; }
        }
        if (bh >= (int)P[P_MINH]) {
            const int kk = (int)P[P_K], K = (2 * kk + 1) * (2 * kk + 1) * (2 * kk + 1);
            double tau[343], pose[3];
            for (int j = 0; j < K; ++j) {
                int a, b, e, h;
                gs_prop_index(j, kk, kk, &a, &b, &e);
                const double x = xh[0] + (double)a * P[P_KL], y = xh[1] + (double)b * P[P_KL];
                const double yaw = fs_normalize_angle(xh[2] + (double)e * P[P_KA]);
                tau[j] = gs_prop_tau(j, kk, P[P_KL], P[P_KA], xh, mu, A, prop_weight(g, grid, x, y, yaw, pairs, k, angle_min, &h));
            }
            if (gs_prop_sample(tau, kk, P[P_KL], P[P_KA], xh, c, z4[0], z4[1], z4[3], pose, eta)) {
                g->x[i] = pose[0]; g->y[i] = pose[1]; g->yaw[i] = pose[2];
                g->w[i] = g->w[i] * *eta;
                return 1;
            }
        }
    }
    pf_odom_move(m, z4[0], z4[1], z4[2], &g->x[i], &g->y[i], &g->yaw[i]);
    g->yaw[i] = fs_normalize_angle(g->yaw[i]);
    g->w[i] = g->w[i] * orc_gs_weight(grid, g->cfg, g->W, g->H, g->model, g->x[i], g->y[i], g->yaw[i], pairs, k, angle_min);
    return 0;
}

/* c of the step (gs_prop_norm) */
double orc_gsp_norm(const double* odom6, const double* alpha, double kl, double ka) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha, &m) != 0) return NAN;
    return gs_prop_norm(&m, kl, ka);
}

/* one step under the proposal P[8]; nz (nullable) = n x 4 injected (za, zb, zc, n2), u01 (nullable) the resample draw; xh (n x 3),
 * eta (n) and took (n) out.  -1: refused, nothing changed; else whether it resampled.  The rest is orc_gs_step's. */
int orc_gsp_step(orc_gs* g, const double* odom6, const double* alpha, const double* ranges, size_t B, double angle_min, double angle_inc,
                 const double* P, const double* nz, const double* u01, double* xh, double* eta, uint8_t* took) {
    PfOdom m;
    if (!isfinite(angle_min) || !isfinite(angle_inc) || pf_odom_increment(odom6, alpha, &m) != 0) return -1;
    double* pairs = (double*)malloc((B + 1) * 2 * sizeof(double));
    const size_t k = orc_gs_used(g->model, ranges, B, angle_inc, pairs);
    if (k > g->L) { free(pairs); return -1; }
    const double c = gs_prop_norm(&m, P[P_KL], P[P_KA]);
    if (!gs_prop_still(&m)) {                                   /* the high side of eta's bound: c K q_hi^k <= DBL_MAX */
        const double S = 2.0 * P[P_K] + 1.0, q_hi = g->model[G_ZHIT] + g->model[G_ZRAND] / g->model[G_MAXR];
        double hi = c * ((S * S) * S);
        for (size_t j = 0; j < k; ++j) hi = hi * q_hi;
        if (!(hi <= 1.7976931348623157e308)) { free(pairs); return -1; }
    }
    const size_t n = g->n, cells = g->cells;
    for (size_t i = 0; i < n; ++i) {
        double z4[4], unused;
        if (nz) memcpy(z4, nz + 4 * i, sizeof(z4));
        else {
            pfc_normal_pair(pfc_rng_block(g->seed, PFC_STREAM_FS_PREDICT, g->step, (uint64_t)i), &z4[0], &z4[1]);
            pfc_normal_pair(pfc_rng_block(g->seed, PFC_STREAM_FS_ODOM, g->step, (uint64_t)i), &z4[2], &unused);
            pfc_normal_pair(pfc_rng_block(g->seed, PFC_STREAM_FS2_POSE3, g->step, (uint64_t)i), &z4[3], &unused);
        }
        took[i] = (uint8_t)prop_particle(g, i, &m, P, c, pairs, k, angle_min, z4, xh + 3 * i, eta + i);
    }
    free(pairs);
    g->used = k;
    normalize_w(g);
    double s2 = 0.0;
    for (size_t i = 0; i < n; ++i) s2 += g->w[i] * g->w[i];
    g->neff = s2 > 0.0 ? 1.0 / s2 : 0.0;
    uint64_t* ev = (uint64_t*)calloc(n, sizeof(uint64_t));
    for (size_t i = 0; i < n; ++i) {
        ev[i] = scan_events(g->cfg, g->W, g->H, g->x[i], g->y[i], g->yaw[i], ranges, B, angle_min, angle_inc);
        orc_ogm_update_scan(g->grid + i * cells, g->cfg, g->W, g->H, g->x[i], g->y[i], g->yaw[i], ranges, B, angle_min, angle_inc);
    }
    g->step++;
    g->resampled = g->neff < g->model[G_NTH];
    g->copies = 0;
    g->events = 0;
    if (!g->resampled) {
        for (size_t i = 0; i < n; ++i) g->events += ev[i];
        g->last_n = 0;
        free(ev);
        return 0;
    }
    normalize_w(g);
    double* cum = (double*)malloc(sizeof(double) * (n + 1));
    cum[0] = 0.0;
    for (size_t i = 0; i < n; ++i) cum[i + 1] = cum[i] + g->w[i];
    const double u = u01 ? *u01 : pfc_u01_52(pfc_blk_u64(pfc_rng_block(g->seed, PFC_STREAM_FS_RESAMPLE, g->n_resample, 0), 0));
    double r = u * (1.0 / (double)n - 0.0) + 0.0;
    size_t j = 0;
    for (size_t t = 0; t < n; ++t) {
        while (r > cum[j + 1] && j < n - 1) j++;
        g->idx[t] = (uint32_t)j;
        r += 1.0 / (double)n;
    }
    free(cum);
    for (size_t t = 0; t < n; ++t) {
        const size_t a = g->idx[t];
        g->x2[t] = g->x[a]; g->y2[t] = g->y[a]; g->yaw2[t] = g->yaw[a];
        memcpy(g->grid2 + t * cells, g->grid + a * cells, cells * sizeof(double));
        g->w[t] = 1.0 / (double)n;
        if (t == 0 || g->idx[t] != g->idx[t - 1]) g->events += ev[a];
        else g->copies++;
    }
    double* s;
    s = g->x; g->x = g->x2; g->x2 = s; s = g->y; g->y = g->y2; g->y2 = s; s = g->yaw; g->yaw = g->yaw2; g->yaw2 = s;
    s = g->grid; g->grid = g->grid2; g->grid2 = s;
    g->n_resample++;
    g->last_n = n;
    free(ev);
    return 1;
}

/* one particle on one grid (W x H, cells ix * H + iy): pose3 in / out; returns the factor its weight is multiplied by */
double orc_gsp_one(const double* grid, const double* cfg6, size_t W, size_t H, const double* model6, double* pose3, const double* odom6,
                   const double* alpha, const double* ranges, size_t B, double angle_min, double angle_inc, const double* P,
                   const double* z4, double* xh, double* eta, uint8_t* took) {
    PfOdom m;
    if (pf_odom_increment(odom6, alpha, &m) != 0) return NAN;
    orc_gs* g = orc_gs_new(cfg6, W, H, model6, 1, 0, pose3);
    memcpy(g->grid, grid, W * H * sizeof(double));
    g->w[0] = 1.0;
    double* pairs = (double*)malloc((B + 1) * 2 * sizeof(double));
    const size_t k = orc_gs_used(g->model, ranges, B, angle_inc, pairs);
    *took = (uint8_t)prop_particle(g, 0, &m, P, gs_prop_norm(&m, P[P_KL], P[P_KA]), pairs, k, angle_min, z4, xh, eta);
    pose3[0] = g->x[0]; pose3[1] = g->y[0]; pose3[2] = g->yaw[0];
    const double f = g->w[0];
    free(pairs);
    orc_gs_free(g);
    return f;
}
