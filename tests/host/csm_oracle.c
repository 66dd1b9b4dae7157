/*
 * csm_oracle.c — CPU oracle of correlative scan matching (DESIGN §3.13, the rule of include/pfgpu.h pfgpu_csm_*).  TEST
 * INFRASTRUCTURE ONLY.  A literal restatement of correlative_scan_match (rust_robotics_slam/src/correlative_scan_matching.rs:55-197):
 * the lookup table is a hash map from (ix, iy) to the maximum weight, filled point by point and window cell by window cell; the
 * search is the triple loop dx, dy, dyaw with the `>` / `==`-and-`<` update; each candidate's score is a sequential sum of hash
 * lookups.  No dense table, no cell-index arrays, no reduction.  Built twice by tests/_csm_oracle.py (contract math; glibc libm
 * with -DPF_ORACLE_LIBM).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include "../../include/pf_contract_math.h"

#ifdef PF_ORACLE_LIBM
#define M_EXP(x) exp(x)
#define M_SIN(x) sin(x)
#define M_COS(x) cos(x)
#else
#define M_EXP(x) pfc_exp(x)
#define M_SIN(x) pfc_sin(x)
#define M_COS(x) pfc_cos(x)
#endif

#define RS_PI 3.14159265358979323846

int orc_csm_is_libm(void) {
#ifdef PF_ORACLE_LIBM
    return 1;
#else
    return 0;
#endif
}

/* cfg: CorrelativeScanMatcherConfig's five fields */
enum { C_LR, C_AR, C_LS, C_AS, C_RES };

/* Rust's `as i32`: saturating, NaN -> 0 */
static int32_t sat_i32(double v) {
    if (v != v) return 0;
    if (v >= 2147483647.0) return 2147483647;
    if (v <= -2147483648.0) return INT32_MIN;
    return (int32_t)v;
}
/* normalize_angle (:189-197), with fs1.rs's cap of 2^22 turns (DESIGN §8 deviation 2) */
static double normalize_angle(double a) {
    int guard = 0;
    while (a > RS_PI && guard < (1 << 22)) { a -= 2.0 * RS_PI; ++guard; }
    while (a < -RS_PI && guard < (1 << 23)) { a += 2.0 * RS_PI; ++guard; }
    return a;
}

/* the HashMap<(i32, i32), f64>: open addressing on the packed key */
typedef struct { uint64_t* key; double* val; uint8_t* used; size_t cap, n; } map_t;
static uint64_t pack(int32_t ix, int32_t iy) { return ((uint64_t)(uint32_t)ix << 32) | (uint32_t)iy; }
static size_t slot_of(uint64_t k, size_t cap) {
    k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
    return (size_t)(k & (cap - 1));
}
static void map_init(map_t* m, size_t cap) {
    m->cap = cap; m->n = 0;
    m->key = (uint64_t*)malloc(cap * sizeof(uint64_t));
    m->val = (double*)malloc(cap * sizeof(double));
    m->used = (uint8_t*)calloc(cap, 1);
}
static void map_free(map_t* m) { free(m->key); free(m->val); free(m->used); }
static double* map_find(const map_t* m, uint64_t k) {
    for (size_t s = slot_of(k, m->cap);; s = (s + 1) & (m->cap - 1)) {
        if (!m->used[s]) return NULL;
        if (m->key[s] == k) return &m->val[s];
    }
}
static void map_grow(map_t* m);
/* grid.entry((ix, iy)).and_modify(|s| *s = s.max(w)).or_insert(w) */
static void map_entry_max(map_t* m, uint64_t k, double w) {
    if (2 * (m->n + 1) > m->cap) map_grow(m);
    size_t s = slot_of(k, m->cap);
    for (; m->used[s]; s = (s + 1) & (m->cap - 1))
        if (m->key[s] == k) { m->val[s] = fmax(m->val[s], w); return; }
    m->used[s] = 1; m->key[s] = k; m->val[s] = w; m->n++;
}
static void map_grow(map_t* m) {
    map_t b;
    map_init(&b, m->cap * 2);
    for (size_t s = 0; s < m->cap; ++s)
        if (m->used[s]) {
            size_t t = slot_of(m->key[s], b.cap);
            while (b.used[t]) t = (t + 1) & (b.cap - 1);
            b.used[t] = 1; b.key[t] = m->key[s]; b.val[t] = m->val[s]; b.n++;
        }
    map_free(m);
    *m = b;
}

/* cell_index (:182-187) */
static void cell_index(double x, double y, double res, int32_t* cx, int32_t* cy) {
    *cx = sat_i32(round(x / res));
    *cy = sat_i32(round(y / res));
}
/* build_lookup_table (:129-159); *R_out = the cutoff radius */
static void build_lookup_table(const double* rx, const double* ry, size_t n, double res, map_t* grid, int32_t* R_out) {
    map_init(grid, 1024);
    const double sigma = res;
    const int32_t R = sat_i32(ceil(3.0 * sigma / res));
    const double inv_two_sigma_sq = 0.5 / (sigma * sigma);
    *R_out = R;
    for (size_t i = 0; i < n; ++i) {
        const double x = rx[i], y = ry[i];
        int32_t cx, cy;
        cell_index(x, y, res, &cx, &cy);
        for (int32_t ix = cx - R; ix <= cx + R; ++ix)
            for (int32_t iy = cy - R; iy <= cy + R; ++iy) {
                const double gx = (double)ix * res, gy = (double)iy * res;
                const double squared_distance = (gx - x) * (gx - x) + (gy - y) * (gy - y);
                const double weight = M_EXP(-squared_distance * inv_two_sigma_sq);
                if (weight < 1.0e-6) continue;
                map_entry_max(grid, pack(ix, iy), weight);
            }
    }
}
/* score_candidate (:161-180) */
static double score_candidate(const map_t* grid, const double* qx, const double* qy, size_t n, double px, double py, double pyaw,
                              double res) {
    const double cos_yaw = M_COS(pyaw), sin_yaw = M_SIN(pyaw);
    double score = 0.0;
    for (size_t i = 0; i < n; ++i) {
        const double x = qx[i], y = qy[i];
        const double world_x = cos_yaw * x - sin_yaw * y + px;
        const double world_y = sin_yaw * x + cos_yaw * y + py;
        int32_t cx, cy;
        cell_index(world_x, world_y, res, &cx, &cy);
        const double* v = map_find(grid, pack(cx, cy));
        score += v ? *v : 0.0;
    }
    return score;
}

/* correlative_scan_match (:55-120): out = x, y, yaw, score, converged; the number of candidates in *n_cand */
void orc_csm_match(const double* rx, const double* ry, size_t nr, const double* qx, const double* qy, size_t nq, const double* pose,
                   const double* cfg, double* out, uint64_t* n_cand) {
    *n_cand = 0;
    if (nr == 0 || nq == 0 || cfg[C_LS] <= 0.0 || cfg[C_AS] <= 0.0 || cfg[C_RES] <= 0.0) {
        out[0] = pose[0]; out[1] = pose[1]; out[2] = pose[2]; out[3] = 0.0; out[4] = 0.0;
        return;
    }
    map_t grid;
    int32_t R;
    build_lookup_table(rx, ry, nr, cfg[C_RES], &grid, &R);
    const int32_t nl = sat_i32(round(cfg[C_LR] / cfg[C_LS])), na = sat_i32(round(cfg[C_AR] / cfg[C_AS]));
    double best_x = pose[0], best_y = pose[1], best_yaw = normalize_angle(pose[2]), best_score = -1.0, best_penalty = INFINITY;
    int converged = 0;
    for (int64_t i = -(int64_t)nl; i <= nl; ++i) {
        const double dx = (double)i * cfg[C_LS];
        for (int64_t j = -(int64_t)nl; j <= nl; ++j) {
            const double dy = (double)j * cfg[C_LS];
            for (int64_t k = -(int64_t)na; k <= na; ++k) {
                const double dyaw = (double)k * cfg[C_AS];
                const double cx = pose[0] + dx, cy = pose[1] + dy, cyaw = normalize_angle(pose[2] + dyaw);
                const double score = score_candidate(&grid, qx, qy, nq, cx, cy, cyaw, cfg[C_RES]);
                const double penalty = dx * dx + dy * dy + dyaw * dyaw;
                (*n_cand)++;
                if (score > best_score || (score == best_score && penalty < best_penalty)) {
                    best_x = cx; best_y = cy; best_yaw = cyaw; best_score = score; converged = score > 0.0;
                    best_penalty = penalty;
                }
            }
        }
    }
    map_free(&grid);
    out[0] = best_x; out[1] = best_y; out[2] = best_yaw; out[3] = best_score; out[4] = converged ? 1.0 : 0.0;
}

/* the lookup table's entries: up to cap (ix, iy) keys and weights in slot order; returns the number of entries and the radius */
size_t orc_csm_table(const double* rx, const double* ry, size_t nr, double res, int32_t* keys, double* vals, size_t cap, int32_t* R) {
    map_t grid;
    build_lookup_table(rx, ry, nr, res, &grid, R);
    size_t k = 0;
    for (size_t s = 0; s < grid.cap; ++s)
        if (grid.used[s]) {
            if (k < cap) { keys[2 * k] = (int32_t)(grid.key[s] >> 32); keys[2 * k + 1] = (int32_t)(uint32_t)grid.key[s]; vals[k] = grid.val[s]; }
            ++k;
        }
    map_free(&grid);
    return k;
}

/* score_candidate on its own (the reference's lookup-table test, :315-345) */
double orc_csm_score(const double* rx, const double* ry, size_t nr, const double* qx, const double* qy, size_t nq, const double* pose,
                     double res) {
    map_t grid;
    int32_t R;
    build_lookup_table(rx, ry, nr, res, &grid, &R);
    const double s = score_candidate(&grid, qx, qy, nq, pose[0], pose[1], pose[2], res);
    map_free(&grid);
    return s;
}
