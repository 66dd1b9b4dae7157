/*
 * pf_lfield_oracle.c — CPU oracle of the likelihood-field scan model (DESIGN §3.9, the rule of include/pfgpu.h pfgpu_pf_lfield_* /
 * pfgpu_pf_*_scan).  TEST INFRASTRUCTURE ONLY.  Includes tests/host/pf_recovery_oracle.c (and so oracle/pf_oracle.c) unchanged
 * and adds compute_udf, the factor table and the scan update in the engine's operation order.  Built twice by
 * tests/_lfield_oracle.py (contract math; glibc libm with -DPF_ORACLE_LIBM).
 */
#include "pf_recovery_oracle.c"
#include <float.h>

#define LF_INF 1e20           /* distance_map.rs:10 */
#define LF_MAX_L 4096

typedef struct {
    orc_rec* r;
    int on;
    size_t W, H;
    double res, sigma, z_hit, z_rand, max_range, q_out;
    uint32_t max_beams;
    uint64_t L;
    double* D;
    double* q;
} orc_lf;

orc_lf* orc_lf_new(const orc_pf_config* cfg, uint64_t seed) {
    orc_rec* r = orc_rec_new(cfg, seed);
    if (!r) return NULL;
    orc_lf* l = (orc_lf*)calloc(1, sizeof(orc_lf));
    l->r = r;
    return l;
}
static void lf_clear(orc_lf* l) { free(l->D); free(l->q); l->D = l->q = NULL; l->on = 0; l->W = l->H = 0; l->L = 0; }
void orc_lf_free(orc_lf* l) { if (l) { lf_clear(l); orc_rec_free(l->r); free(l); } }
orc_rec* orc_lf_rec(orc_lf* l) { return l->r; }
void orc_lf_clear(orc_lf* l) { lf_clear(l); }

/* dt_1d (distance_map.rs:15-53) over in[q * stride] -> out[q * stride]; the final loop reads the input line (DESIGN §3.9) */
static void dt_1d(const double* in, double* out, size_t stride, size_t n, size_t* v, double* z) {
    if (n == 0) return;
    size_t k = 0;
    v[0] = 0;
    z[0] = -LF_INF;
    z[1] = LF_INF;
    for (size_t q = 1; q < n; ++q) {
        size_t vk = v[k];
        double s = ((in[q * stride] + (double)(q * q)) - (in[vk * stride] + (double)(vk * vk))) / (2.0 * (double)q - 2.0 * (double)vk);
        while (s <= z[k]) {
            k -= 1;
            size_t vk2 = v[k];
            s = ((in[q * stride] + (double)(q * q)) - (in[vk2 * stride] + (double)(vk2 * vk2))) / (2.0 * (double)q - 2.0 * (double)vk2);
        }
        k += 1;
        v[k] = q;
        z[k] = s;
        if (k + 1 < n + 1) z[k + 1] = LF_INF;
    }
    k = 0;
    for (size_t q = 0; q < n; ++q) {
        while (k + 1 < n + 1 && z[k + 1] < (double)q) k += 1;
        double dx = (double)q - (double)v[k];
        out[q * stride] = dx * dx + in[v[k] * stride];
    }
}

/* compute_udf (distance_map.rs:63-100), nrows = W (row = ix), ncols = H: D[ix * H + iy] */
void orc_lf_compute_udf(const uint8_t* mask, size_t W, size_t H, double* D) {
    const size_t cells = W * H, m = (W > H ? W : H) + 1;
    double* a = (double*)malloc(sizeof(double) * cells);
    size_t* v = (size_t*)malloc(sizeof(size_t) * m);
    double* z = (double*)malloc(sizeof(double) * m);
    for (size_t i = 0; i < cells; ++i) D[i] = mask[i] ? 0.0 : LF_INF;
    for (size_t r = 0; r < W; ++r) dt_1d(D + r * H, a + r * H, 1, H, v, z);
    for (size_t c = 0; c < H; ++c) dt_1d(a + c, D + c, H, W, v, z);
    for (size_t i = 0; i < cells; ++i) D[i] = sqrt(D[i]);
    free(a); free(v); free(z);
}

static uint64_t lf_limit(double q_lo, double q_hi) {
    double pmin = 1.0, pmax = 1.0;
    uint64_t L = 0;
    for (uint64_t m = 1; m <= LF_MAX_L + 1; ++m) {
        pmin = pmin * q_lo;
        pmax = pmax * q_hi;
        if (!(pmin >= DBL_MIN) || !(pmax <= DBL_MAX)) break;
        L = m - 1;
    }
    return L;
}

/* pfgpu_pf_lfield_set; cfg6 = (res, sigma_hit, z_hit, z_rand, max_range, max_beams) */
int orc_lf_set(orc_lf* l, const uint8_t* mask, size_t W, size_t H, const double* cfg6) {
    const double res = cfg6[0], sigma = cfg6[1], z_hit = cfg6[2], z_rand = cfg6[3], max_range = cfg6[4], mb = cfg6[5];
    if (!mask || W < 1 || H < 1 || W > 65536 || H > 65536 || W * H > ((size_t)1 << 28)) return -1;
    if (!(finite_(res) && res > 0.0) || !(finite_(sigma) && sigma > 0.0) || !(finite_(z_rand) && z_rand > 0.0) ||
        !(finite_(max_range) && max_range > 0.0) || !finite_(z_hit) || z_hit < 0.0 || !(mb >= 2.0) || mb > 4294967295.0) return -1;
    const double q_out = z_rand / max_range;
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (sigma * sigma));
    const uint64_t L = lf_limit(q_out, z_hit * coeff + q_out);
    if (L < 1) return -1;
    lf_clear(l);
    const size_t cells = W * H;
    l->D = (double*)malloc(sizeof(double) * cells);
    l->q = (double*)malloc(sizeof(double) * cells);
    orc_lf_compute_udf(mask, W, H, l->D);
    for (size_t i = 0; i < cells; ++i) {                 /* gauss_likelihood mcl.rs:408-411 */
        const double t = l->D[i] * res;
        const double g = coeff * M_EXP(-(t * t) / (2.0 * (sigma * sigma)));
        l->q[i] = z_hit * g + q_out;
    }
    l->W = W; l->H = H; l->res = res; l->sigma = sigma; l->z_hit = z_hit; l->z_rand = z_rand; l->max_range = max_range;
    l->max_beams = (uint32_t)mb; l->q_out = q_out; l->L = L; l->on = 1;
    return 0;
}
void orc_lf_info(const orc_lf* l, uint64_t out3[3]) { out3[0] = l->W; out3[1] = l->H; out3[2] = l->L; }
void orc_lf_tables(const orc_lf* l, double* D, double* q) {
    for (size_t i = 0; i < l->W * l->H; ++i) { D[i] = l->D[i]; q[i] = l->q[i]; }
}

/* the used beams: pairs2 = (r_i, a_i) with room for B pairs; returns their count, or -1 (refused) */
long orc_lf_beams(const orc_lf* l, const double* ranges, size_t B, double angle_min, double angle_inc, double* pairs2) {
    if (!l->on || (B && !ranges) || !finite_(angle_min) || !finite_(angle_inc)) return -1;
    size_t k = 0;
    if (B) {
        size_t s = (B - 1) / (size_t)(l->max_beams - 1);
        if (s < 1) s = 1;
        for (size_t i = 0; i < B; i += s) {
            const double r = ranges[i];
            if (r <= 0.0 || !finite_(r) || r >= l->max_range) continue;
            pairs2[2 * k] = r;
            pairs2[2 * k + 1] = (double)i * angle_inc;
            k++;
        }
    }
    return k > l->L ? -1 : (long)k;
}

static double lf_factor(const orc_lf* l, double ex, double ey) {
    const int32_t ix = sat_i32(floor(ex / l->res + (double)l->W / 2.0));
    const int32_t iy = sat_i32(floor(ey / l->res + (double)l->H / 2.0));
    if (ix < 0 || ix >= (int32_t)l->W || iy < 0 || iy >= (int32_t)l->H) return l->q_out;
    return l->q[(size_t)ix * l->H + (size_t)iy];
}
static double lf_weight(const orc_lf* l, double x, double y, double yaw, double angle_min, const double* pairs2, size_t k) {
    double w = 1.0;
    for (size_t j = 0; j < k; ++j) {
        const double angle = (yaw + angle_min) + pairs2[2 * j + 1];
        const double r = pairs2[2 * j];
        const double ex = x + r * M_COS(angle), ey = y + r * M_SIN(angle);
        w = w * lf_factor(l, ex, ey);
    }
    return w;
}
/* raw weights of n poses (x, y, yaw) under one scan, without touching the filter; returns the used beams or -1 */
long orc_lf_weights(const orc_lf* l, const double* pose3, size_t n, const double* ranges, size_t B, double angle_min, double angle_inc,
                    double* w) {
    double* pr = (double*)malloc(sizeof(double) * 2 * (B ? B : 1));
    const long k = orc_lf_beams(l, ranges, B, angle_min, angle_inc, pr);
    if (k >= 0)
        for (size_t i = 0; i < n; ++i) w[i] = lf_weight(l, pose3[3 * i], pose3[3 * i + 1], pose3[3 * i + 2], angle_min, pr, (size_t)k);
    free(pr);
    return k;
}

/* pfgpu_pf_update_scan: the weights, then orc_rec_update's S, filter, normalisation and refresh */
int orc_lf_update_scan(orc_lf* l, const double* ranges, size_t B, double angle_min, double angle_inc) {
    orc_rec* r = l->r;
    orc_pf* f = r->f;
    double* pr = (double*)malloc(sizeof(double) * 2 * (B ? B : 1));
    const long k = orc_lf_beams(l, ranges, B, angle_min, angle_inc, pr);
    if (k < 0) { free(pr); return -1; }
    long n = (long)f->n;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1)
    for (long i = 0; i < n; ++i) {
        orc_particle* q = &f->p[i];
        q->w = lf_weight(l, q->x, q->y, q->yaw, angle_min, pr, (size_t)k);
    }
    free(pr);
    double S = 0.0;
    for (size_t i = 0; i < f->n; ++i) S += f->p[i].w;
    rec_filter(r, S, f->n);
    normalize_weights(f);
    refresh_cache(f);
    r->armed = 0;
    return 0;
}
