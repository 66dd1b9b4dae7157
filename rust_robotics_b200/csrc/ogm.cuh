// ogm.cuh — occupancy grid mapping (DESIGN §3.12): laser scans fused into a log-odds grid with OccupancyGridMap::update_with_scan's
// sequential result bit for bit (rust_robotics_mapping/src/occupancy_grid_map.rs:69-131), and the grid's obstacle mask.
//
// Layout: cell (ix, iy) of a W x H grid at ix * H + iy, like the scan models' tables.  One update runs in chunks of whole beams:
//   count  one thread per beam: origin, end cell and the beam's event count (its cell updates)
//   scan   inclusive sum of the counts (CUB), one f64-free integer pass
//   emit   one warp per beam: its events (cell | kind << 31) at the beam's offset, in global beam order g = s * B + i
//   sort   stable radix sort on the cell bits alone (CUB), so each cell's events stay in g order
//   fold   one thread per run of equal cells: the run's additions in order, the cell written once
// A cell occurs at most once per beam (bresenham_line's cells are distinct and the end cell is not in the free run), so a cell's
// updates in g order are the sequential order.  No floating-point atomics.
#pragma once
#include "common.cuh"
#include "pf_kernels.cuh"           // pf_lf_sat_i32
#include <cub/cub.cuh>

#define PF_OGM_EVENT_CAP (1u << 24)     // events per chunk (a beam has at most 65536)
#define PF_OGM_BEAM_CAP (1u << 20)      // beams per window of the count / scan workspace
#define PF_OGM_OCC 0x80000000u          // the event's kind bit: the occupied update of a beam's end cell

struct PfOgmGeom {
    double res = 1.0, half_w = 0.0, half_h = 0.0;     // half_w = W as f64 / 2.0
    int W = 0, H = 0;
};

// The minor-axis offset of step k of bresenham_line's closed form, floor((2 k dm + dM - 1) / den) with den = 2 dM and dm > 0: the
// same arithmetic as pf_beam_cast's loop (pf_beam.cuh).  A twin rather than a shared routine: factoring it out of pf_beam_cast
// reorders the instructions nvcc emits for the beam kernels, and their SASS is kept as it was.  num < 2^44, so the f64 estimate is
// within one and corrected in integers.
__device__ __forceinline__ long long pf_ogm_bres_minor(long long k, long long dm, long long dM, long long den, double rden) {
    const long long num = 2 * k * dm + dM - 1;
    long long mi = (long long)((double)num * rden);
    if (mi * den > num) mi -= 1;
    else if ((mi + 1) * den <= num) mi += 1;
    return mi;
}

// world_to_grid's value before the floor: v / res + W / 2
__device__ __forceinline__ double pf_ogm_pre(double v, const pfc_rcp_t& rres, double half) { return pfc_div_by(v, rres) + half; }

// one thread per beam g = g0 + t of the window: the beam's (origin, end cell) and its event count max(|dx|, |dy|) + 1, less one
// when the end is outside the grid (its clamped end cell takes no update).  Skipped beams and scans from outside count 0.
__global__ void __launch_bounds__(256) pf_ogm_count_kernel(PfOgmGeom gm, const double* pose3, const double* ranges, size_t B, size_t g0,
                                                           size_t nb, double angle_min, double angle_inc, int4* geo,
                                                           unsigned long long* cnt) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= nb) return;
    const size_t g = g0 + t, s = g / B, i = g - s * B;
    const double x = pose3[3 * s], y = pose3[3 * s + 1], yaw = pose3[3 * s + 2];
    const pfc_rcp_t rres = pfc_rcp_make(gm.res);
    const int ox = pf_lf_sat_i32(floor(pf_ogm_pre(x, rres, gm.half_w))), oy = pf_lf_sat_i32(floor(pf_ogm_pre(y, rres, gm.half_h)));
    const double r = ranges[g];
    if (ox < 0 || ox >= gm.W || oy < 0 || oy >= gm.H || r <= 0.0 || !isfinite(r)) { cnt[t] = 0; geo[t] = make_int4(0, 0, 0, 0); return; }
    double sn, cs;
    pfc_sincos((yaw + angle_min) + (double)i * angle_inc, &sn, &cs);
    const double vx = pf_ogm_pre(x + r * cs, rres, gm.half_w), vy = pf_ogm_pre(y + r * sn, rres, gm.half_h);
    int ex = pf_lf_sat_i32(floor(vx)), ey = pf_lf_sat_i32(floor(vy));
    const bool inside = ex >= 0 && ex < gm.W && ey >= 0 && ey < gm.H;
    if (!inside) {                  // both coordinates from round-and-clamp, even one that was inside (:93-101)
        ex = min(max(pf_lf_sat_i32(round(vx)), 0), gm.W - 1);
        ey = min(max(pf_lf_sat_i32(round(vy)), 0), gm.H - 1);
    }
    const int adx = abs(ex - ox), ady = abs(ey - oy);
    cnt[t] = (unsigned long long)max(adx, ady) + (inside ? 1ull : 0ull);
    geo[t] = make_int4(ox, oy, ex, ey);
}

// one thread: the chunk from beam b of the window: e = the largest index <= nb with incl[e - 1] - base <= cap (at least b + 1, since
// a beam has at most 65536 <= cap events).  out[0] = e, out[1] = the chunk's events.
__global__ void pf_ogm_chunk_kernel(const unsigned long long* incl, size_t b, size_t nb, unsigned long long base, unsigned long long cap,
                                    unsigned long long* out) {
    size_t lo = b + 1, hi = nb;                                          // incl[lo - 1] - base <= cap holds; find the last such
    while (lo < hi) {
        const size_t mid = lo + (hi - lo + 1) / 2;
        if (incl[mid - 1] - base <= cap) lo = mid;
        else hi = mid - 1;
    }
    out[0] = lo;
    out[1] = incl[lo - 1] - base;
}

// one warp per beam j in [b, e): its events at offset incl[j - 1] - base, k = 0 .. cnt - 1 along bresenham_line(origin, end);
// step k == dM (the end cell, reached only when the end is inside) is the occupied update, every other step a free one
__global__ void __launch_bounds__(256) pf_ogm_emit_kernel(const int4* geo, const unsigned long long* incl, size_t b, size_t e,
                                                          unsigned long long base, int H, unsigned int* keys) {
    const size_t j = b + ((size_t)blockIdx.x * 256 + threadIdx.x) / 32;
    const int lane = threadIdx.x & 31;
    if (j >= e) return;
    const unsigned long long o = (j ? incl[j - 1] : 0ull), n = incl[j] - o;
    if (n == 0) return;
    const int4 q = geo[j];
    const long long dx = (long long)q.z - q.x, dy = (long long)q.w - q.y;
    const long long adx = dx < 0 ? -dx : dx, ady = dy < 0 ? -dy : dy;
    const bool xmaj = adx >= ady;
    const long long dM = xmaj ? adx : ady, dm = xmaj ? ady : adx;
    const int sx = q.x < q.z ? 1 : -1, sy = q.y < q.w ? 1 : -1;
    const long long den = 2 * dM;
    const double rden = dm ? 1.0 / (double)den : 0.0;
    unsigned int* out = keys + (o - base);
    for (long long k = lane; k < (long long)n; k += 32) {
        const long long mi = dm ? pf_ogm_bres_minor(k, dm, dM, den, rden) : 0;
        const long long ox = xmaj ? k : mi, oy = xmaj ? mi : k;
        const unsigned int cell = (unsigned int)((q.x + (int)(sx * ox)) * H + (q.y + (int)(sy * oy)));
        out[k] = cell | (k == dM ? PF_OGM_OCC : 0u);
    }
}

// Rust's f64::clamp for min <= max: NaN stays NaN
__device__ __forceinline__ double pf_ogm_clamp(double l, double lo, double hi) { return l < lo ? lo : (l > hi ? hi : l); }

// one thread per sorted event; the first of each run of equal cells folds the run in order and writes the cell once
__global__ void __launch_bounds__(256) pf_ogm_fold_kernel(const unsigned int* keys, size_t n, double* grid, double occ, double fre,
                                                          double lo, double hi, unsigned int* longest) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const unsigned int cell = keys[t] & ~PF_OGM_OCC;
    if (t > 0 && (keys[t - 1] & ~PF_OGM_OCC) == cell) return;
    double l = grid[cell];
    size_t u = t;
    for (; u < n; ++u) {
        const unsigned int k = keys[u];
        if ((k & ~PF_OGM_OCC) != cell) break;
        l = pf_ogm_clamp(l + ((k & PF_OGM_OCC) ? occ : fre), lo, hi);
    }
    grid[cell] = l;
    atomicMax(longest, (unsigned int)(u - t));
}

// one thread per cell: is_occupied (:136-159) with the contract exp
__global__ void __launch_bounds__(256) pf_ogm_mask_kernel(const double* grid, size_t cells, double threshold, unsigned char* mask) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= cells) return;
    mask[t] = (1.0 - 1.0 / (1.0 + pfc_exp(grid[t]))) > threshold ? 1 : 0;
}

__global__ void __launch_bounds__(256) pf_ogm_fill_kernel(double* grid, size_t cells, double v) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t < cells) grid[t] = v;
}
