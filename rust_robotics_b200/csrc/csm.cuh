// csm.cuh — correlative scan matching (DESIGN §3.13): correlative_scan_match (rust_robotics_slam/src/correlative_scan_matching.rs
// :55-197) with the reference's sequential result bit for bit, and reference points from an occupancy grid's obstacle cells.
//
//   table    extent: one thread per reference point, atomicMin / atomicMax of its centre cell; the dense f64 table over the
//            bounding box grown by R is zeroed, then one thread per (point, window cell) computes the weight and takes the
//            integer atomicMax of its bit pattern.  Every stored weight is in [1e-6, 1], where bit order is value order, and max
//            commutes: the table is the reference's HashMap with 0.0 for absent keys, whatever the order.  No floating-point atomics.
//   trig     one thread per (query, yaw): normalize_angle(yaw + dyaw) and its contract sincos.
//   cells    one thread per (query, yaw, offset, point): the x cell of (point, cand_x) and the y cell of (point, cand_y), stored
//            as table offsets, X = (ix - ox) * TH or PF_CSM_OUT, Y = iy - oy or PF_CSM_OUT, so that X + Y >= 0 exactly when the cell
//            lies in the table.  The rotated point and cand_x depend only on these indices: they are the reference's bits.
//   score    one thread per candidate: per point two index loads, one bounds check, one 8-byte gather and one dependent add; the
//            sum stays one sequential chain per candidate.  Then a per-block best under the total order (score desc, penalty asc,
//            loop index asc).
//   reduce   one block per query with points: the chunk's block bests folded into the query's running best.
// Candidates run in chunks of whole yaws (and groups of queries) so that the cell indices fit the workspace; each candidate's
// sum is independent of the chunking.
#pragma once
#include "common.cuh"
#include "pf_kld.cuh"               // pf_sat_i32
#include "../../include/fs_ekf_math.h"   // fs_normalize_angle
#include <climits>
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#define PF_CSM_NT 256
#define PF_CSM_OUT ((int)0xC0000000)   // -2^30: X + Y < 0 whenever either index is outside (|valid X| < 2^26, 0 <= valid Y < 2^26)

struct PfCsmBest {
    double score, pen;
    unsigned long long idx;
};

// the total order of the winner: larger score, then smaller penalty, then earlier loop index
__device__ __forceinline__ bool pf_csm_better(const PfCsmBest& a, const PfCsmBest& b) {
    if (a.score != b.score) return a.score > b.score;
    if (a.pen != b.pen) return a.pen < b.pen;
    return a.idx < b.idx;
}

// round(v / res) as i32: half away from zero, saturating, NaN -> 0
__device__ __forceinline__ int pf_csm_cell(double v, const pfc_rcp_t& rres) { return pf_sat_i32(round(pfc_div_by(v, rres))); }

// one thread per reference point: the bounding box of the centre cells; ext = (min x, max x, min y, max y), bad = any |cell| > 2^30
__global__ void __launch_bounds__(256) pf_csm_extent_kernel(const double* rx, const double* ry, size_t n, double res, int* ext, int* bad) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const pfc_rcp_t rres = pfc_rcp_make(res);
    const int cx = pf_csm_cell(rx[t], rres), cy = pf_csm_cell(ry[t], rres);
    if (cx > (1 << 30) || cx < -(1 << 30) || cy > (1 << 30) || cy < -(1 << 30)) { atomicOr(bad, 1); return; }
    atomicMin(ext + 0, cx); atomicMax(ext + 1, cx);
    atomicMin(ext + 2, cy); atomicMax(ext + 3, cy);
}

// one thread per (reference point, window cell): the weight of build_lookup_table (:139-156), kept by the maximum of its bits
__global__ void __launch_bounds__(256) pf_csm_fill_kernel(const double* rx, const double* ry, size_t n, double res, double inv, int R,
                                                          long long ox, long long oy, long long TH, unsigned long long* table) {
    const int side = 2 * R + 1;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * (size_t)(side * side)) return;
    const size_t p = t / (size_t)(side * side);
    const int w = (int)(t - p * (size_t)(side * side));
    const double x = rx[p], y = ry[p];
    const pfc_rcp_t rres = pfc_rcp_make(res);
    const int ix = pf_csm_cell(x, rres) - R + w / side, iy = pf_csm_cell(y, rres) - R + w % side;
    const double gx = (double)ix * res, gy = (double)iy * res;
    const double d2 = (gx - x) * (gx - x) + (gy - y) * (gy - y);
    const double wt = pfc_exp((-d2) * inv);
    if (wt < 1.0e-6) return;
    atomicMax(table + ((long long)ix - ox) * TH + ((long long)iy - oy), (unsigned long long)__double_as_longlong(wt));
}

// one thread per (query q of the group, yaw a of the chunk): cs = (cos, sin) of normalize_angle(yaw_q + (a0 + a - na) * astep)
__global__ void __launch_bounds__(256) pf_csm_trig_kernel(const double* pose3, size_t q0, size_t nq, long long a0, int nac, int na,
                                                          double astep, double2* cs) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= nq * (size_t)nac) return;
    const size_t q = t / nac;
    const int a = (int)(t - q * nac);
    const double dyaw = (double)(int)(a0 + a - na) * astep;
    const double yaw = fs_normalize_angle(pose3[3 * (q0 + q) + 2] + dyaw);
    double s, c;
    pfc_sincos(yaw, &s, &c);
    cs[t] = make_double2(c, s);
}

struct PfCsmGeo {
    double res, lstep;
    long long ox, oy, TW, TH;   // the table: cells ox .. ox + TW - 1 by oy .. oy + TH - 1, (ix - ox) * TH + (iy - oy)
    int nl, NL, nac;            // linear offsets -nl ..= nl (NL of them), yaws in the chunk
};

// one thread per (point k of the group, yaw a of the chunk, offset i, axis): the point's x cell for cand_x = x_q + dx_i into
// X[((k_local * nac + a) ... )], laid out as ((P_q * nac + a * n_q + p) * NL + i) with P_q the query's first point in the group
__global__ void __launch_bounds__(256) pf_csm_cells_kernel(PfCsmGeo g, const double* pose3, const double* qx, const double* qy,
                                                           const unsigned long long* offsets, size_t q0, size_t nq, size_t k0, size_t nk,
                                                           const double2* cs, int* X, int* Y) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    const size_t per = (size_t)g.nac * g.NL;
    if (t >= nk * per) return;
    const size_t k = t / per;                       // the point, relative to the group's first point k0
    const size_t r = t - k * per;
    const int a = (int)(r / g.NL), i = (int)(r - (size_t)a * g.NL);
    // the query of point k0 + k: offsets[q0 .. q0 + nq] bracket it
    size_t lo = q0, hi = q0 + nq - 1;
    while (lo < hi) {
        const size_t mid = lo + (hi - lo + 1) / 2;
        if (offsets[mid] <= k0 + k) lo = mid;
        else hi = mid - 1;
    }
    const size_t q = lo, P = offsets[q] - k0, nqp = offsets[q + 1] - offsets[q], p = k - P;
    const double2 c = cs[(q - q0) * g.nac + a];
    const double px = qx[k0 + k], py = qy[k0 + k];
    const double off = (double)(i - g.nl) * g.lstep;
    const pfc_rcp_t rres = pfc_rcp_make(g.res);
    const double wx = ((c.x * px) - (c.y * py)) + (pose3[3 * q] + off);
    const double wy = ((c.y * px) + (c.x * py)) + (pose3[3 * q + 1] + off);
    const long long ix = (long long)pf_csm_cell(wx, rres) - g.ox, iy = (long long)pf_csm_cell(wy, rres) - g.oy;
    const size_t o = ((P * g.nac + (size_t)a * nqp + p) * g.NL) + i;
    X[o] = (ix >= 0 && ix < g.TW) ? (int)(ix * g.TH) : PF_CSM_OUT;
    Y[o] = (iy >= 0 && iy < g.TH) ? (int)iy : PF_CSM_OUT;
}

__device__ __forceinline__ PfCsmBest pf_csm_shfl(const PfCsmBest& b, int d) {
    PfCsmBest o;
    o.score = __shfl_down_sync(0xffffffffu, b.score, d);
    o.pen = __shfl_down_sync(0xffffffffu, b.pen, d);
    o.idx = __shfl_down_sync(0xffffffffu, b.idx, d);
    return o;
}

// the block's best under pf_csm_better, in thread 0
__device__ __forceinline__ PfCsmBest pf_csm_block_best(PfCsmBest b) {
    __shared__ PfCsmBest s_best[PF_CSM_NT / 32];
    for (int d = 16; d > 0; d >>= 1) {
        const PfCsmBest o = pf_csm_shfl(b, d);
        if (pf_csm_better(o, b)) b = o;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_best[warp] = b;
    __syncthreads();
    if (warp == 0) {
        b = lane < (int)(blockDim.x >> 5) ? s_best[lane] : PfCsmBest{-1.0, __longlong_as_double(0x7FF0000000000000ll), ~0ull};
        for (int d = 16; d > 0; d >>= 1) {
            const PfCsmBest o = pf_csm_shfl(b, d);
            if (pf_csm_better(o, b)) b = o;
        }
    }
    return b;
}

// grid (blocks per query, live queries of the group): one thread per candidate (a, ix, iy) of the chunk, iy fastest, grid-striding;
// the score of score_candidate (:161-180) as one sequential sum, its penalty and loop index (ix * NL + iy) * NA + a0 + a.
// live[l0 + blockIdx.y] is the query (one with points); part[blockIdx.y * nb + b] = the block's best.  The candidate index t and its
// remainder within a yaw stay 64-bit: NL * NL exceeds 2^31 from n_linear = 23170 on (NL <= 65537).
__global__ void __launch_bounds__(PF_CSM_NT) pf_csm_score_kernel(PfCsmGeo g, const double* __restrict__ table,
                                                                 const unsigned long long* __restrict__ offsets,
                                                                 const unsigned long long* __restrict__ live, size_t l0, size_t k0,
                                                                 const int* __restrict__ X, const int* __restrict__ Y, long long a0, int na,
                                                                 double astep, PfCsmBest* part) {
    const size_t q = (size_t)live[l0 + blockIdx.y];
    const size_t NL2 = (size_t)g.NL * g.NL, per = NL2 * g.nac;
    PfCsmBest b{-1.0, __longlong_as_double(0x7FF0000000000000ll), ~0ull};
    const size_t P = offsets[q] - k0, n = offsets[q + 1] - offsets[q];
    for (size_t t = (size_t)blockIdx.x * PF_CSM_NT + threadIdx.x; t < per; t += (size_t)gridDim.x * PF_CSM_NT) {
        const size_t at = t / NL2, r = t - at * NL2;
        const int a = (int)at;
        const int ix = (int)(r / (size_t)g.NL), iy = (int)(r - (size_t)ix * g.NL);
        const int* xp = X + (P * g.nac + (size_t)a * n) * g.NL + ix;
        const int* yp = Y + (P * g.nac + (size_t)a * n) * g.NL + iy;
        double score = 0.0;
#pragma unroll 4
        for (size_t p = 0; p < n; ++p) {
            const int c = __ldg(xp + p * g.NL) + __ldg(yp + p * g.NL);
            const double v = c >= 0 ? __ldg(table + c) : 0.0;
            score = score + v;
        }
        const double dx = (double)(ix - g.nl) * g.lstep, dy = (double)(iy - g.nl) * g.lstep;
        const double dyaw = (double)(int)(a0 + a - na) * astep;
        const PfCsmBest cur{score, (dx * dx + dy * dy) + dyaw * dyaw,
                            ((unsigned long long)ix * g.NL + iy) * (unsigned long long)(2 * na + 1) + (unsigned long long)(a0 + a)};
        if (pf_csm_better(cur, b)) b = cur;
    }
    b = pf_csm_block_best(b);
    if (threadIdx.x == 0) part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = b;
}

// one block per live query of the group: the chunk's nb block bests folded into best[q], q = live[l0 + blockIdx.x]
__global__ void __launch_bounds__(PF_CSM_NT) pf_csm_reduce_kernel(const PfCsmBest* part, size_t nb, const unsigned long long* live,
                                                                  size_t l0, PfCsmBest* best) {
    const PfCsmBest* pq = part + (size_t)blockIdx.x * nb;
    const size_t q = (size_t)live[l0 + blockIdx.x];
    PfCsmBest b = threadIdx.x == 0 ? best[q] : PfCsmBest{-1.0, __longlong_as_double(0x7FF0000000000000ll), ~0ull};
    for (size_t j = threadIdx.x; j < nb; j += PF_CSM_NT)
        if (pf_csm_better(pq[j], b)) b = pq[j];
    b = pf_csm_block_best(b);
    if (threadIdx.x == 0) best[q] = b;
}

__global__ void __launch_bounds__(256) pf_csm_best_init_kernel(PfCsmBest* best, size_t n) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t < n) best[t] = PfCsmBest{-1.0, __longlong_as_double(0x7FF0000000000000ll), ~0ull};
}

// one thread per obstacle cell c = ix * H + iy (the compacted indices of the grid's mask): its centre
// (((ix + 0.5) - W / 2.0) * res, ((iy + 0.5) - H / 2.0) * res)
__global__ void __launch_bounds__(256) pf_csm_centres_kernel(const unsigned int* idx, size_t n, unsigned int H, double half_w,
                                                             double half_h, double res, double* rx, double* ry) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n) return;
    const unsigned int c = idx[t], ix = c / H, iy = c - ix * H;
    rx[t] = (((double)ix + 0.5) - half_w) * res;
    ry[t] = (((double)iy + 0.5) - half_h) * res;
}
