/*
 * gs_oracle.c — CPU oracle of grid-based FastSLAM (DESIGN §3.16, the rule of include/pfgpu.h pfgpu_gs_*).  TEST INFRASTRUCTURE
 * ONLY.  The sequential statement, with a full grid per slot and no buffer sharing (the device's inheritance is what it checks):
 *   move       include/pf_odom_math.h's increment and move, yaw wrapped (include/fs_odom_math.h's FastSLAM 1.0 move)
 *   weigh      the endpoint model: per used beam the window maximum of the grid before the scan, q, w_raw = 1 * q_0 * q_1 * ..
 *   normalise  fs1.rs's normalize_weights / compute_neff / resample, written as oracle/fs1_oracle.c writes them
 *   fuse       OccupancyGridMap::update_with_scan of every slot, before the resample: tests/host/ogm_oracle.c, included unchanged
 * Draws: Philox (the header's streams), or injected (za, zb, zc per slot and the resample's u) so that tests/golden/make_gs_golden.py
 * pins the arithmetic without Philox.  Built twice by tests/_gs_oracle.py (contract math; glibc libm with -DPF_ORACLE_LIBM).
 */
#include "ogm_oracle.c"

#ifdef PF_ORACLE_LIBM
#define PF_ODOM_ATAN2(y, x) atan2((y), (x))
#define PF_ODOM_SINCOS(a, s, c) (*(s) = sin(a), *(c) = cos(a))
#endif
#include "../../include/pf_odom_math.h"

/* model: z_hit, z_rand, max_range, max_beams, R, nth */
enum { G_ZHIT, G_ZRAND, G_MAXR, G_BEAMS, G_R, G_NTH };

typedef struct {
    size_t n, W, H, cells;
    double cfg[6], model[6];
    uint64_t seed, L;
    uint32_t step, n_resample;
    double *x, *y, *yaw, *w, *grid;         /* grid: n * cells, slot i at i * cells */
    double *x2, *y2, *yaw2, *grid2;
    uint32_t* idx;
    size_t last_n;
    double neff;
    uint64_t copies, events, used;
    int resampled;
} orc_gs;

/* the likelihood field's L rule with q_lo = q_out and q_hi = z_hit + q_out */
uint64_t orc_gs_limit(double q_out, double q_hi) {
    double pmin = 1.0, pmax = 1.0;
    uint64_t L = 0;
    for (uint64_t m = 1; m <= 4097; ++m) {
        pmin = pmin * q_out;
        pmax = pmax * q_hi;
        if (!(pmin >= 2.2250738585072014e-308) || !(pmax <= 1.7976931348623157e308)) break;
        L = m - 1;
    }
    return L;
}

orc_gs* orc_gs_new(const double* cfg6, size_t W, size_t H, const double* model6, size_t n, uint64_t seed, const double* start3) {
    orc_gs* g = (orc_gs*)calloc(1, sizeof(orc_gs));
    g->n = n; g->W = W; g->H = H; g->cells = W * H; g->seed = seed;
    memcpy(g->cfg, cfg6, sizeof(g->cfg));
    memcpy(g->model, model6, sizeof(g->model));
    const double q_out = model6[G_ZRAND] / model6[G_MAXR];
    g->L = orc_gs_limit(q_out, model6[G_ZHIT] + q_out);
    g->x = (double*)malloc(n * 8); g->y = (double*)malloc(n * 8); g->yaw = (double*)malloc(n * 8); g->w = (double*)malloc(n * 8);
    g->x2 = (double*)malloc(n * 8); g->y2 = (double*)malloc(n * 8); g->yaw2 = (double*)malloc(n * 8);
    g->grid = (double*)malloc(n * g->cells * 8); g->grid2 = (double*)malloc(n * g->cells * 8);
    g->idx = (uint32_t*)calloc(n, 4);
    for (size_t i = 0; i < n; ++i) { g->x[i] = start3[0]; g->y[i] = start3[1]; g->yaw[i] = start3[2]; g->w[i] = 1.0 / (double)n; }
    for (size_t c = 0; c < n * g->cells; ++c) g->grid[c] = cfg6[C_PRIOR];
    return g;
}
void orc_gs_free(orc_gs* g) {
    if (!g) return;
    free(g->x); free(g->y); free(g->yaw); free(g->w); free(g->x2); free(g->y2); free(g->yaw2); free(g->grid); free(g->grid2); free(g->idx);
    free(g);
}

/* the used beams of a scan: (r, i as f64 * angle_inc) into pairs (room for B pairs); returns their count */
size_t orc_gs_used(const double* model, const double* ranges, size_t B, double angle_inc, double* pairs) {
    size_t k = 0;
    if (B == 0) return 0;
    const size_t beams = (size_t)model[G_BEAMS];
    size_t s = (B - 1) / (beams - 1);
    if (s < 1) s = 1;
    for (size_t i = 0; i < B; i += s) {
        const double r = ranges[i];
        if (r <= 0.0 || !isfinite(r) || r >= model[G_MAXR]) continue;
        pairs[2 * k] = r; pairs[2 * k + 1] = (double)i * angle_inc;
        k++;
    }
    return k;
}

/* w_raw of pose (x, y, yaw) against one grid over k used beams */
double orc_gs_weight(const double* grid, const double* cfg, size_t W, size_t H, const double* model, double x, double y, double yaw,
                     const double* pairs, size_t k, double angle_min) {
    const double q_out = model[G_ZRAND] / model[G_MAXR];
    const int R = (int)model[G_R];
    double wr = 1.0;
    for (size_t j = 0; j < k; ++j) {
        const double r = pairs[2 * j], angle = (yaw + angle_min) + pairs[2 * j + 1];
        const double ex = x + r * M_COS(angle), ey = y + r * M_SIN(angle);
        const int64_t cx = sat_i32(floor(ex / cfg[C_RES] + (double)W / 2.0)), cy = sat_i32(floor(ey / cfg[C_RES] + (double)H / 2.0));
        int any = 0;
        double best = -INFINITY;
        for (int64_t ix = cx - R; ix <= cx + R; ++ix)
            for (int64_t iy = cy - R; iy <= cy + R; ++iy) {
                if (ix < 0 || ix >= (int64_t)W || iy < 0 || iy >= (int64_t)H) continue;
                any = 1;
                const double l = grid[ix * (int64_t)H + iy];
                if (l > best) best = l;
            }
        const double q = any ? model[G_ZHIT] * (1.0 - 1.0 / (1.0 + M_EXP(best))) + q_out : q_out;
        wr = wr * q;
    }
    return wr;
}

/* the cell updates update_with_scan applies for one pose */
static uint64_t scan_events(const double* cfg, size_t W, size_t H, double x, double y, double yaw, const double* ranges, size_t B,
                            double angle_min, double angle_inc) {
    int32_t ox, oy;
    if (!world_to_grid(cfg, W, H, x, y, &ox, &oy)) return 0;
    cells_t ray = {0};
    uint64_t e = 0;
    for (size_t i = 0; i < B; ++i) {
        int inside;
        int32_t ex, ey;
        if (!beam_ray(cfg, W, H, ox, oy, x, y, yaw, ranges[i], i, angle_min, angle_inc, &ray, &inside, &ex, &ey)) continue;
        e += (uint64_t)(ray.n - 1) + (uint64_t)inside;
    }
    free(ray.xy);
    return e;
}

static void normalize_w(orc_gs* g) {                          /* normalize_weights fs1.rs:196-203 */
    double sum_w = 0.0;
    for (size_t i = 0; i < g->n; ++i) sum_w += g->w[i];
    if (sum_w > 0.0) for (size_t i = 0; i < g->n; ++i) g->w[i] /= sum_w;
}

/* one step; nz (nullable) = n x 3 injected (za, zb, zc), u01 (nullable) the injected resample draw.  -1: refused, nothing changed;
 * else whether it resampled */
int orc_gs_step(orc_gs* g, const double* odom6, const double* alpha, const double* ranges, size_t B, double angle_min, double angle_inc,
                const double* nz, const double* u01) {
    PfOdom m;
    if (!isfinite(angle_min) || !isfinite(angle_inc) || pf_odom_increment(odom6, alpha, &m) != 0) return -1;
    double* pairs = (double*)malloc((B + 1) * 2 * sizeof(double));
    const size_t k = orc_gs_used(g->model, ranges, B, angle_inc, pairs);
    if (k > g->L) { free(pairs); return -1; }
    const size_t n = g->n, cells = g->cells;
    for (size_t i = 0; i < n; ++i) {
        double za, zb, zc, unused;
        if (nz) { za = nz[3 * i]; zb = nz[3 * i + 1]; zc = nz[3 * i + 2]; }
        else {
            pfc_normal_pair(pfc_rng_block(g->seed, PFC_STREAM_FS_PREDICT, g->step, (uint64_t)i), &za, &zb);
            pfc_normal_pair(pfc_rng_block(g->seed, PFC_STREAM_FS_ODOM, g->step, (uint64_t)i), &zc, &unused);
        }
        pf_odom_move(&m, za, zb, zc, &g->x[i], &g->y[i], &g->yaw[i]);
        g->yaw[i] = fs_normalize_angle(g->yaw[i]);
        const double wr = orc_gs_weight(g->grid + i * cells, g->cfg, g->W, g->H, g->model, g->x[i], g->y[i], g->yaw[i], pairs, k, angle_min);
        g->w[i] = g->w[i] * wr;
    }
    free(pairs);
    g->used = k;
    normalize_w(g);
    double s2 = 0.0;                                            /* compute_neff fs1.rs:186-193 */
    for (size_t i = 0; i < n; ++i) s2 += g->w[i] * g->w[i];
    g->neff = s2 > 0.0 ? 1.0 / s2 : 0.0;
    uint64_t* ev = (uint64_t*)calloc(n, sizeof(uint64_t));
    for (size_t i = 0; i < n; ++i) {                            /* the fuse: every slot, its own grid */
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
    /* resample fs1.rs:206-234 */
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

void orc_gs_state(const orc_gs* g, double* poses3, double* w) {
    for (size_t i = 0; i < g->n; ++i) {
        if (poses3) { poses3[3 * i] = g->x[i]; poses3[3 * i + 1] = g->y[i]; poses3[3 * i + 2] = g->yaw[i]; }
        if (w) w[i] = g->w[i];
    }
}
void orc_gs_grid(const orc_gs* g, size_t slot, double* out) { memcpy(out, g->grid + slot * g->cells, g->cells * sizeof(double)); }
size_t orc_gs_last_indices(const orc_gs* g, uint32_t* idx) {
    for (size_t i = 0; i < g->last_n; ++i) idx[i] = g->idx[i];
    return g->last_n;
}
/* out: neff, resampled, copies, events, used beams, L, steps */
void orc_gs_info(const orc_gs* g, double* out7) {
    out7[0] = g->neff; out7[1] = g->resampled; out7[2] = (double)g->copies; out7[3] = (double)g->events; out7[4] = (double)g->used;
    out7[5] = (double)g->L; out7[6] = g->step;
}
int orc_gs_is_libm(void) {
#ifdef PF_ORACLE_LIBM
    return 1;
#else
    return 0;
#endif
}
