/*
 * ogm_oracle.c — CPU oracle of occupancy grid mapping (DESIGN §3.12, the rule of include/pfgpu.h pfgpu_ogm_*).  TEST INFRASTRUCTURE
 * ONLY.  A literal restatement of OccupancyGridMap::update_with_scan (rust_robotics_mapping/src/occupancy_grid_map.rs:69-131): per
 * beam the cells of bresenham_line's loop (:164-193) are collected in a vector, then the free loop and the occupied update run over
 * the grid in place.  No closed form, no events, no sorting.  Built twice by tests/_ogm_oracle.py (contract math; glibc libm with
 * -DPF_ORACLE_LIBM).
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

/* cfg: resolution, prior, occupied, free, max, min (OccupancyGridConfig's log-odds fields) */
enum { C_RES, C_PRIOR, C_OCC, C_FREE, C_MAX, C_MIN };

/* Rust's `as i32`: saturating, NaN -> 0 */
static int32_t sat_i32(double v) {
    if (v != v) return 0;
    if (v >= 2147483647.0) return 2147483647;
    if (v <= -2147483648.0) return INT32_MIN;
    return (int32_t)v;
}
static double clamp_rs(double l, double lo, double hi) {
    if (l < lo) l = lo;
    if (l > hi) l = hi;
    return l;
}
/* world_to_grid (:144-153): 1 and (ix, iy) when inside */
static int world_to_grid(const double* cfg, size_t W, size_t H, double x, double y, int32_t* ix, int32_t* iy) {
    *ix = sat_i32(floor(x / cfg[C_RES] + (double)W / 2.0));
    *iy = sat_i32(floor(y / cfg[C_RES] + (double)H / 2.0));
    return *ix >= 0 && *ix < (int32_t)W && *iy >= 0 && *iy < (int32_t)H;
}

typedef struct { int32_t* xy; size_t n, cap; } cells_t;
static void push(cells_t* c, int32_t x, int32_t y) {
    if (c->n == c->cap) { c->cap = c->cap ? 2 * c->cap : 64; c->xy = (int32_t*)realloc(c->xy, 2 * c->cap * sizeof(int32_t)); }
    c->xy[2 * c->n] = x; c->xy[2 * c->n + 1] = y; c->n++;
}
/* bresenham_line (:164-193), both ends included */
static void bresenham(int32_t x0, int32_t y0, int32_t x1, int32_t y1, cells_t* c) {
    c->n = 0;
    const int32_t dx = abs(x1 - x0), dy = abs(y1 - y0);
    const int32_t sx = x0 < x1 ? 1 : -1, sy = y0 < y1 ? 1 : -1;
    int32_t x = x0, y = y0, err = dx - dy;
    for (;;) {
        push(c, x, y);
        if (x == x1 && y == y1) break;
        const int32_t e2 = 2 * err;
        if (e2 > -dy) { err -= dy; x += sx; }
        if (e2 < dx) { err += dx; y += sy; }
    }
}

/* one beam's cells and end flag: 0 when skipped (the scan's origin is given) */
static int beam_ray(const double* cfg, size_t W, size_t H, int32_t ox, int32_t oy, double x, double y, double yaw, double r, size_t i,
                    double angle_min, double angle_inc, cells_t* ray, int* end_inside, int32_t* ex, int32_t* ey) {
    if (r <= 0.0 || !isfinite(r)) return 0;
    const double angle = yaw + angle_min + (double)i * angle_inc;
    const double end_x = x + r * M_COS(angle), end_y = y + r * M_SIN(angle);
    int32_t ix, iy;
    *end_inside = world_to_grid(cfg, W, H, end_x, end_y, &ix, &iy);
    if (!*end_inside) {
        ix = sat_i32(round(end_x / cfg[C_RES] + (double)W / 2.0));
        if (ix < 0) ix = 0;
        if (ix > (int32_t)W - 1) ix = (int32_t)W - 1;
        iy = sat_i32(round(end_y / cfg[C_RES] + (double)H / 2.0));
        if (iy < 0) iy = 0;
        if (iy > (int32_t)H - 1) iy = (int32_t)H - 1;
    }
    *ex = ix; *ey = iy;
    bresenham(ox, oy, ix, iy, ray);
    return 1;
}

/* update_with_scan on grid[ix * H + iy] */
void orc_ogm_update_scan(double* grid, const double* cfg, size_t W, size_t H, double x, double y, double yaw, const double* ranges,
                         size_t B, double angle_min, double angle_inc) {
    int32_t ox, oy;
    if (!world_to_grid(cfg, W, H, x, y, &ox, &oy)) return;
    cells_t ray = {0};
    for (size_t i = 0; i < B; ++i) {
        int inside;
        int32_t ex, ey;
        if (!beam_ray(cfg, W, H, ox, oy, x, y, yaw, ranges[i], i, angle_min, angle_inc, &ray, &inside, &ex, &ey)) continue;
        for (size_t k = 0; k + 1 < ray.n; ++k) {                 /* every cell but the last */
            const int32_t cx = ray.xy[2 * k], cy = ray.xy[2 * k + 1];
            if (cx >= 0 && cx < (int32_t)W && cy >= 0 && cy < (int32_t)H) {
                double* l = grid + (size_t)cx * H + (size_t)cy;
                *l = clamp_rs(*l + cfg[C_FREE], cfg[C_MIN], cfg[C_MAX]);
            }
        }
        if (inside) {
            double* l = grid + (size_t)ex * H + (size_t)ey;
            *l = clamp_rs(*l + cfg[C_OCC], cfg[C_MIN], cfg[C_MAX]);
        }
    }
    free(ray.xy);
}

/* the batch: S single-scan updates in order (poses3 S x 3, ranges S x B) */
void orc_ogm_update_scans(double* grid, const double* cfg, size_t W, size_t H, const double* poses3, size_t S, const double* ranges,
                          size_t B, double angle_min, double angle_inc) {
    for (size_t s = 0; s < S; ++s)
        orc_ogm_update_scan(grid, cfg, W, H, poses3[3 * s], poses3[3 * s + 1], poses3[3 * s + 2], ranges + s * B, B, angle_min, angle_inc);
}

/* What a batch does to each cell, without changing any: out[0] = cell updates (events), out[1] = the most updates one cell takes,
 * out[2] = beams in which some cell would be updated twice (the property the device's ordering by cell relies on: always 0),
 * out[3] = the longest ray in cells. */
void orc_ogm_census(const double* cfg, size_t W, size_t H, const double* poses3, size_t S, const double* ranges, size_t B,
                    double angle_min, double angle_inc, uint64_t* out) {
    uint32_t* per = (uint32_t*)calloc(W * H, sizeof(uint32_t));
    uint64_t* seen = (uint64_t*)calloc(W * H, sizeof(uint64_t));   /* 1 + the global beam index that last touched the cell */
    cells_t ray = {0};
    memset(out, 0, 4 * sizeof(uint64_t));
    for (size_t s = 0; s < S; ++s) {
        int32_t ox, oy;
        const double x = poses3[3 * s], y = poses3[3 * s + 1], yaw = poses3[3 * s + 2];
        if (!world_to_grid(cfg, W, H, x, y, &ox, &oy)) continue;
        for (size_t i = 0; i < B; ++i) {
            int inside;
            int32_t ex, ey;
            if (!beam_ray(cfg, W, H, ox, oy, x, y, yaw, ranges[s * B + i], i, angle_min, angle_inc, &ray, &inside, &ex, &ey)) continue;
            const uint64_t tag = (uint64_t)(s * B + i) + 1;
            int repeat = 0;
            if (ray.n > out[3]) out[3] = ray.n;
            for (size_t k = 0; k < ray.n; ++k) {
                if (k + 1 == ray.n && !inside) break;
                const size_t c = (size_t)ray.xy[2 * k] * H + (size_t)ray.xy[2 * k + 1];
                if (seen[c] == tag) repeat = 1;
                seen[c] = tag;
                per[c]++;
                out[0]++;
            }
            out[2] += (uint64_t)repeat;
        }
    }
    for (size_t c = 0; c < W * H; ++c)
        if (per[c] > out[1]) out[1] = per[c];
    free(ray.xy); free(per); free(seen);
}

/* is_occupied (:136-159) of every cell */
void orc_ogm_obstacles(const double* grid, size_t cells, double threshold, uint8_t* mask) {
    for (size_t c = 0; c < cells; ++c) mask[c] = (1.0 - 1.0 / (1.0 + M_EXP(grid[c]))) > threshold ? 1 : 0;
}

/* bresenham_line's cells, for tests: up to cap (x, y) pairs, returns the count */
size_t orc_ogm_line(int32_t x0, int32_t y0, int32_t x1, int32_t y1, int32_t* out, size_t cap) {
    cells_t c = {0};
    bresenham(x0, y0, x1, y1, &c);
    for (size_t k = 0; k < c.n && k < cap; ++k) { out[2 * k] = c.xy[2 * k]; out[2 * k + 1] = c.xy[2 * k + 1]; }
    const size_t n = c.n;
    free(c.xy);
    return n;
}

int orc_ogm_is_libm(void) {
#ifdef PF_ORACLE_LIBM
    return 1;
#else
    return 0;
#endif
}
