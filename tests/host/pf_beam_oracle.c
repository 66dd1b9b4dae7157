/*
 * pf_beam_oracle.c — CPU oracle of the beam measurement model (DESIGN §3.11, the rule of include/pfgpu.h pfgpu_pf_beam_* /
 * pfgpu_pf_*_beam).  TEST INFRASTRUCTURE ONLY.  Includes tests/host/pf_lfield_oracle.c (and so the recovery and PF oracles)
 * unchanged, so one handle holds a likelihood field and a beam map.  The ray cast is a literal transcription of bresenham_line's
 * loop (rust_robotics_mapping/src/occupancy_grid_map.rs:164-193) over the obstacle mask: no clearance, no skipping, no closed form.
 * The clearance table is a plain two-pass chessboard chamfer.  Built twice by tests/_beam_oracle.py (contract math; glibc libm with
 * -DPF_ORACLE_LIBM).
 */
#include "pf_lfield_oracle.c"

typedef struct {
    orc_lf* lf;
    int on;
    size_t W, H;
    double res, sigma, z_hit, z_short, z_max, z_rand, lambda, max_range;
    uint32_t max_beams;
    uint64_t L;
    uint8_t* occ;
    uint8_t* clr;
} orc_bm;

orc_bm* orc_bm_new(const orc_pf_config* cfg, uint64_t seed) {
    orc_lf* lf = orc_lf_new(cfg, seed);
    if (!lf) return NULL;
    orc_bm* b = (orc_bm*)calloc(1, sizeof(orc_bm));
    b->lf = lf;
    return b;
}
static void bm_clear(orc_bm* b) { free(b->occ); free(b->clr); b->occ = b->clr = NULL; b->on = 0; b->W = b->H = 0; b->L = 0; }
void orc_bm_free(orc_bm* b) { if (b) { bm_clear(b); orc_lf_free(b->lf); free(b); } }
orc_lf* orc_bm_lf(orc_bm* b) { return b->lf; }
void orc_bm_clear(orc_bm* b) { bm_clear(b); }

/* the chessboard distance of every cell to the nearest obstacle or the ring of obstacles around the grid, capped at 255:
 * forward and backward chamfer passes over the padded (W + 2) x (H + 2) grid */
void orc_bm_chessboard(const uint8_t* mask, size_t W, size_t H, uint8_t* out) {
    const size_t PW = W + 2, PH = H + 2;
    int64_t* d = (int64_t*)malloc(sizeof(int64_t) * PW * PH);
    for (size_t i = 0; i < PW; ++i)
        for (size_t j = 0; j < PH; ++j) {
            const int ring = i == 0 || j == 0 || i == PW - 1 || j == PH - 1;
            d[i * PH + j] = (ring || mask[(i - 1) * H + (j - 1)]) ? 0 : INT32_MAX;
        }
#define D_(i, j) d[(size_t)(i) * PH + (size_t)(j)]
#define RELAX(i, j, a, b) do { if (D_(a, b) + 1 < D_(i, j)) D_(i, j) = D_(a, b) + 1; } while (0)
    for (size_t i = 1; i + 1 < PW; ++i)
        for (size_t j = 1; j + 1 < PH; ++j) {
            RELAX(i, j, i - 1, j - 1); RELAX(i, j, i - 1, j); RELAX(i, j, i - 1, j + 1); RELAX(i, j, i, j - 1);
        }
    for (size_t i = PW - 2; i >= 1; --i)
        for (size_t j = PH - 2; j >= 1; --j) {
            RELAX(i, j, i + 1, j + 1); RELAX(i, j, i + 1, j); RELAX(i, j, i + 1, j - 1); RELAX(i, j, i, j + 1);
        }
#undef RELAX
    for (size_t i = 0; i < W; ++i)
        for (size_t j = 0; j < H; ++j) {
            const int64_t v = D_(i + 1, j + 1);
            out[i * H + j] = (uint8_t)(v > 255 ? 255 : v);
        }
#undef D_
    free(d);
}

/* pfgpu_pf_beam_set; cfg9 = (res, sigma_hit, z_hit, z_short, z_max, z_rand, lambda_short, max_range, max_beams) */
int orc_bm_set(orc_bm* b, const uint8_t* mask, size_t W, size_t H, const double* cfg9) {
    const double res = cfg9[0], sigma = cfg9[1], z_hit = cfg9[2], z_short = cfg9[3], z_max = cfg9[4], z_rand = cfg9[5],
                 lambda = cfg9[6], max_range = cfg9[7], mb = cfg9[8];
    if (!mask || W < 1 || H < 1 || W > 65536 || H > 65536 || W * H > ((size_t)1 << 28)) return -1;
    if (!(finite_(res) && res > 0.0) || !(finite_(sigma) && sigma > 0.0) || !(finite_(z_rand) && z_rand > 0.0) ||
        !(finite_(max_range) && max_range > 0.0) || !(finite_(lambda) && lambda > 0.0) || !finite_(z_hit) || z_hit < 0.0 ||
        !finite_(z_short) || z_short < 0.0 || !finite_(z_max) || z_max < 0.0 || !(mb >= 2.0) || mb > 4294967295.0 ||
        !(max_range / res <= 1048576.0))
        return -1;
    const double q_rand = z_rand / max_range;
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (sigma * sigma));
    const double q_lo = z_max > 0.0 ? (z_max < q_rand ? z_max : q_rand) : q_rand;
    const double q_hi = z_hit * coeff + z_short * lambda + (z_max > q_rand ? z_max : q_rand);
    const uint64_t L = lf_limit(q_lo, q_hi);
    if (L < 1) return -1;
    bm_clear(b);
    const size_t cells = W * H;
    b->occ = (uint8_t*)malloc(cells);
    b->clr = (uint8_t*)malloc(cells);
    for (size_t i = 0; i < cells; ++i) b->occ[i] = mask[i] ? 1 : 0;
    orc_bm_chessboard(b->occ, W, H, b->clr);
    b->W = W; b->H = H; b->res = res; b->sigma = sigma; b->z_hit = z_hit; b->z_short = z_short; b->z_max = z_max; b->z_rand = z_rand;
    b->lambda = lambda; b->max_range = max_range; b->max_beams = (uint32_t)mb; b->L = L; b->on = 1;
    return 0;
}
void orc_bm_info(const orc_bm* b, uint64_t out3[3]) { out3[0] = b->W; out3[1] = b->H; out3[2] = b->L; }
void orc_bm_clearance(const orc_bm* b, uint8_t* out) { for (size_t i = 0; i < b->W * b->H; ++i) out[i] = b->clr[i]; }

/* world_to_grid (occupancy_grid_map.rs:144-153) without the inside test */
static void bm_cell(const orc_bm* b, double x, double y, int64_t* ix, int64_t* iy) {
    *ix = sat_i32(floor(x / b->res + (double)b->W / 2.0));
    *iy = sat_i32(floor(y / b->res + (double)b->H / 2.0));
}
static int bm_blocked(const orc_bm* b, int64_t x, int64_t y) {
    return x < 0 || x >= (int64_t)b->W || y < 0 || y >= (int64_t)b->H || b->occ[(size_t)x * b->H + (size_t)y];
}
/* the expected range of one beam: bresenham_line(c0, c1)'s loop, stopping at the first occupied or outside cell */
double orc_bm_cast(const orc_bm* b, double px, double py, double angle) {
    int64_t x0, y0, x1, y1;
    bm_cell(b, px, py, &x0, &y0);
    if (bm_blocked(b, x0, y0)) return 0.0;
    bm_cell(b, px + b->max_range * M_COS(angle), py + b->max_range * M_SIN(angle), &x1, &y1);
    const int64_t dx = x1 - x0 < 0 ? x0 - x1 : x1 - x0;
    const int64_t dy = y1 - y0 < 0 ? y0 - y1 : y1 - y0;
    const int64_t sx = x0 < x1 ? 1 : -1;
    const int64_t sy = y0 < y1 ? 1 : -1;
    int64_t x = x0, y = y0, err = dx - dy;
    for (;;) {
        if (bm_blocked(b, x, y)) {
            const int64_t ox = x - x0, oy = y - y0;
            return b->res * sqrt((double)(ox * ox + oy * oy));
        }
        if (x == x1 && y == y1) break;
        const int64_t e2 = 2 * err;
        if (e2 > -dy) { err -= dy; x += sx; }
        if (e2 < dx) { err += dx; y += sy; }
    }
    return b->max_range;
}
/* pfgpu_pf_beam_raycast */
void orc_bm_raycast(const orc_bm* b, const double* pose3, size_t n, size_t B, double angle_min, double angle_inc, double* out) {
    for (size_t p = 0; p < n; ++p)
        for (size_t j = 0; j < B; ++j)
            out[p * B + j] = orc_bm_cast(b, pose3[3 * p], pose3[3 * p + 1], (pose3[3 * p + 2] + angle_min) + (double)j * angle_inc);
}

/* the used beams: pairs2 = (r_i, a_i) with room for B pairs (a max reading as r = max_range); their count, or -1 (refused) */
long orc_bm_beams(const orc_bm* b, const double* ranges, size_t B, double angle_min, double angle_inc, double* pairs2) {
    if (!b->on || (B && !ranges) || !finite_(angle_min) || !finite_(angle_inc)) return -1;
    size_t k = 0;
    if (B) {
        size_t s = (B - 1) / (size_t)(b->max_beams - 1);
        if (s < 1) s = 1;
        for (size_t i = 0; i < B; i += s) {
            double r = ranges[i];
            if (r != r || r <= 0.0) continue;
            if (r >= b->max_range) {
                if (!(b->z_max > 0.0)) continue;
                r = b->max_range;
            }
            pairs2[2 * k] = r;
            pairs2[2 * k + 1] = (double)i * angle_inc;
            k++;
        }
    }
    return k > b->L ? -1 : (long)k;
}
static double bm_weight(const orc_bm* b, double x, double y, double yaw, double angle_min, const double* pairs2, size_t k) {
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (b->sigma * b->sigma));
    double w = 1.0;
    for (size_t j = 0; j < k; ++j) {
        const double r = pairs2[2 * j];
        const double rhat = orc_bm_cast(b, x, y, (yaw + angle_min) + pairs2[2 * j + 1]);
        const double z = r - rhat;
        double q = b->z_hit * coeff * M_EXP(-(z * z) / (2.0 * (b->sigma * b->sigma)));
        if (z < 0.0) q = q + b->z_short * b->lambda * M_EXP(-(b->lambda * r));
        q = q + (r >= b->max_range ? b->z_max : b->z_rand / b->max_range);
        w = w * q;
    }
    return w;
}
/* raw weights of n poses (x, y, yaw) under one scan, without touching the filter; returns the used beams or -1 */
long orc_bm_weights(const orc_bm* b, const double* pose3, size_t n, const double* ranges, size_t B, double angle_min, double angle_inc,
                    double* w) {
    double* pr = (double*)malloc(sizeof(double) * 2 * (B ? B : 1));
    const long k = orc_bm_beams(b, ranges, B, angle_min, angle_inc, pr);
    if (k >= 0)
        for (size_t i = 0; i < n; ++i) w[i] = bm_weight(b, pose3[3 * i], pose3[3 * i + 1], pose3[3 * i + 2], angle_min, pr, (size_t)k);
    free(pr);
    return k;
}

/* pfgpu_pf_update_beam: the weights, then orc_rec_update's S, filter, normalisation and refresh */
int orc_bm_update_beam(orc_bm* b, const double* ranges, size_t B, double angle_min, double angle_inc) {
    orc_rec* r = b->lf->r;
    orc_pf* f = r->f;
    double* pr = (double*)malloc(sizeof(double) * 2 * (B ? B : 1));
    const long k = orc_bm_beams(b, ranges, B, angle_min, angle_inc, pr);
    if (k < 0) { free(pr); return -1; }
    long n = (long)f->n;
#pragma omp parallel for num_threads(f->threads) schedule(dynamic, 64) if (f->threads > 1)
    for (long i = 0; i < n; ++i) {
        orc_particle* q = &f->p[i];
        q->w = bm_weight(b, q->x, q->y, q->yaw, angle_min, pr, (size_t)k);
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
