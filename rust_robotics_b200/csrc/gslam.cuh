// gslam.cuh — grid-based FastSLAM (DESIGN §3.16): N particles, each with a pose, a weight and its own W x H log-odds grid laid out
// as OccupancyGridMap's (ogm.cuh).  A step (include/pfgpu.h, pfgpu_gs_step) in stream order:
//   move + weigh   one warp per particle: FastSLAM 1.0's odometry move (fs_odom_math.h), then the endpoint model over the used beams
//                  against the particle's grid before this step's scan; w = w * w_raw
//   normalise      xs_total (xsum.cuh) of w, w / S; xs_total of w^2 (PfValWSq), N_eff, the gate
//   comb           (gated) fs1.rs's resample: normalise again, xs_scan of w (the CDF) and of the comb r_0, r_0 + 1/n, ...; ancestors
//   plan           (gated) the first child of each parent inherits its buffer; every further child takes a childless parent's buffer
//   fuse           one CTA per grid that is fused: update_with_scan, beam by beam, a barrier between beams
//   copy           (gated) each further child's buffer gets its parent's fused grid
//   finish         (gated) poses gathered, the slot -> buffer table replaced, w = 1 / N
// Every gated kernel returns at once when the gate is closed.  No floating-point atomics.
#pragma once
#include "common.cuh"
#include "xsum.cuh"
#include "ogm.cuh"
#include "csm.cuh"                  // pf_csm_better, pf_csm_block_best: the proposal's match winner
#include "../../include/fs_odom_math.h"
#include "../../include/gs_prop_math.h"
#include <limits>

#define GS_WARPS 8                  // particles per CTA of the move + weigh kernel
#define GS_FUSE_NT 256
#define GS_MAX_R 8

struct GsDev {
    size_t n = 0, cells = 0;
    double *px = nullptr, *py = nullptr, *pyaw = nullptr, *w = nullptr;   // [n]
    double *tx = nullptr, *ty = nullptr, *tyaw = nullptr;                 // [n] gathered poses of a resample
    double* grids = nullptr;        // [n * cells]: buffer b at b * cells
    unsigned *buf = nullptr, *nbuf = nullptr;   // [n] slot -> buffer, and the next table of a resample
    unsigned* idx = nullptr;        // [n] ancestors of the last resample
    double *cum = nullptr, *comb = nullptr;     // [n] the CDF and the comb positions
    int *nf = nullptr, *enf = nullptr;          // [n] slot t is a further child (not its parent's first), and its exclusive prefix
    int *cl = nullptr, *ecl = nullptr;          // [n] parent j has no child, and its exclusive prefix
    int* has_child = nullptr;       // [n]
    unsigned *free_buf = nullptr, *job_src = nullptr, *job_dst = nullptr;   // [n]
    double* scal = nullptr;         // [0] S  [1] S2  [2] S of the resample's normalisation  [3] r_0  [4] N_eff
    int* gate = nullptr;            // [1]
    unsigned long long* cnt = nullptr;   // [0] resample counter  [1] grids copied  [2] fuse events
};

struct GsModel {
    double res = 1.0, half_w = 0.0, half_h = 0.0;
    int W = 0, H = 0, R = 1;
    double z_hit = 0.0, q_out = 0.0, angle_min = 0.0;
};

// l* over the (2R+1)^2 window around cell (cx, cy) of one grid: *any = 0 when no window cell is inside
__device__ __forceinline__ double gs_window_max(const double* g, const GsModel& m, int cx, int cy, int* any) {
    double best = -INFINITY;
    int hit = 0;
    for (int dx = -m.R; dx <= m.R; ++dx) {
        const long long ix = (long long)cx + dx;
        if (ix < 0 || ix >= m.W) continue;
        for (int dy = -m.R; dy <= m.R; ++dy) {
            const long long iy = (long long)cy + dy;
            if (iy < 0 || iy >= m.H) continue;
            hit = 1;
            const double l = g[ix * m.H + iy];
            if (l > best) best = l;        // NaN never compares greater: skipped
        }
    }
    *any = hit;
    return best;
}

// one warp per particle: the move (lane 0), then the weight of k used beams (r, a) = pairs[2j], pairs[2j + 1] in ascending i; the
// product runs in beam order through the warp's shuffles, the same in every lane
__global__ void __launch_bounds__(GS_WARPS * 32) gs_move_weigh_kernel(GsDev d, PfOdom om, uint64_t seed, uint32_t call, GsModel m,
                                                                      const double* pairs, unsigned k) {
    const size_t i = (size_t)blockIdx.x * GS_WARPS + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= d.n) return;
    double x = 0.0, y = 0.0, yaw = 0.0;
    if (lane == 0) {
        double za, zb, zc, unused;
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)i), &za, &zb);
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_ODOM, call, (uint64_t)i), &zc, &unused);
        x = d.px[i]; y = d.py[i]; yaw = d.pyaw[i];
        fs_odom_move(&om, za, zb, zc, &x, &y, &yaw);
        d.px[i] = x; d.py[i] = y; d.pyaw[i] = yaw;
    }
    x = __shfl_sync(0xffffffffu, x, 0);
    y = __shfl_sync(0xffffffffu, y, 0);
    yaw = __shfl_sync(0xffffffffu, yaw, 0);
    const double* g = d.grids + (size_t)d.buf[i] * d.cells;
    const pfc_rcp_t rres = pfc_rcp_make(m.res);
    double wr = 1.0;
    for (unsigned c0 = 0; c0 < k; c0 += 32) {
        const unsigned j = c0 + lane;
        double q = 1.0;
        if (j < k) {
            const double r = pairs[2 * j], a = pairs[2 * j + 1];
            double sn, cs;
            pfc_sincos((yaw + m.angle_min) + a, &sn, &cs);
            const int cx = pf_lf_sat_i32(floor(pf_ogm_pre(x + r * cs, rres, m.half_w)));
            const int cy = pf_lf_sat_i32(floor(pf_ogm_pre(y + r * sn, rres, m.half_h)));
            int any;
            const double l = gs_window_max(g, m, cx, cy, &any);
            q = any ? m.z_hit * (1.0 - 1.0 / (1.0 + pfc_exp(l))) + m.q_out : m.q_out;
        }
        const unsigned cnt = k - c0 < 32 ? k - c0 : 32;
        for (unsigned t = 0; t < cnt; ++t) wr = wr * __shfl_sync(0xffffffffu, q, t);
    }
    if (lane == 0) d.w[i] = d.w[i] * wr;
}

// w = w / S when S > 0 (normalize_weights fs1.rs:196-203); gated when `gate` is non-null
__global__ void __launch_bounds__(256) gs_normalize_kernel(GsDev d, const double* S, const int* gate) {
    if (gate && !*gate) return;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    const double s = *S;
    if (s > 0.0) d.w[t] = d.w[t] / s;
}

// N_eff (compute_neff fs1.rs:186-193) and the gate; an open gate draws r_0 from the resample counter and advances it
__global__ void gs_gate_kernel(GsDev d, double nth, uint64_t seed) {
    const double s2 = d.scal[1];
    const double neff = s2 > 0.0 ? 1.0 / s2 : 0.0;
    d.scal[4] = neff;
    const int g = neff < nth ? 1 : 0;
    *d.gate = g;
    d.cnt[1] = 0;
    d.cnt[2] = 0;
    if (g) {
        const double u01 = pfc_u01_52(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_FS_RESAMPLE, (uint32_t)d.cnt[0], 0), 0));
        d.scal[3] = u01 * (1.0 / (double)d.n - 0.0) + 0.0;
        d.cnt[0] += 1;
    }
}

// the comb as a sequential sum from 0: r_0, then 1/n per further slot (fs1.rs:219-230), so the inclusive prefix at t is r_t
struct GsCombVal {
    const double* r0; double inv_n;
    __device__ __forceinline__ double operator()(size_t i) const { return i == 0 ? *r0 : inv_n; }
};

// the ancestor of slot t: fs1.rs's loop `while r > cum[j + 1] && j < n - 1 { j += 1 }` from the previous slot's j.  r_t and cum are
// non-decreasing, so that j is the smallest one with r_t <= cum[j + 1], capped at n - 1.  Marks the further children and the parents.
__global__ void __launch_bounds__(256) gs_search_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    const double r = d.comb[t];
    size_t lo = 0, hi = d.n - 1;               // cum[j + 1] = d.cum[j]
    while (lo < hi) {
        const size_t mid = lo + ((hi - lo) >> 1);
        if (r > d.cum[mid]) lo = mid + 1; else hi = mid;
    }
    d.idx[t] = (unsigned)lo;
    d.has_child[lo] = 1;
}
__global__ void __launch_bounds__(256) gs_flags_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    d.nf[t] = (t > 0 && d.idx[t] == d.idx[t - 1]) ? 1 : 0;
    d.cl[t] = d.has_child[t] ? 0 : 1;
}
// the buffers of childless parents in slot order, then every slot's next buffer and the copy jobs (further children in slot order)
__global__ void __launch_bounds__(256) gs_free_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t j = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (j >= d.n) return;
    if (d.cl[j]) d.free_buf[d.ecl[j]] = d.buf[j];
    if (j == d.n - 1) d.cnt[1] = (unsigned long long)(d.enf[j] + d.nf[j]);
}
__global__ void __launch_bounds__(256) gs_plan_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    const unsigned p = d.idx[t], src = d.buf[p];
    if (d.nf[t]) {
        const unsigned dst = d.free_buf[d.enf[t]];
        d.nbuf[t] = dst;
        d.job_src[d.enf[t]] = src;
        d.job_dst[d.enf[t]] = dst;
    } else {
        d.nbuf[t] = src;
    }
    d.tx[t] = d.px[p]; d.ty[t] = d.py[p]; d.tyaw[t] = d.pyaw[p];
}

// One CTA per slot j: update_with_scan (ogm.cuh's rules) of the scan at j's pose into buffer buf[j].  With the gate open only
// parents are fused.  Beams in order; a beam's cells are distinct, so its updates run in parallel, and the barrier after each beam
// orders every cell's updates by beam.  Per tile of GS_FUSE_NT beams the geometry is computed first, one thread per beam.
__global__ void __launch_bounds__(GS_FUSE_NT) gs_fuse_kernel(GsDev d, PfOgmGeom gm, const double* ranges, size_t B, double angle_min,
                                                             double angle_inc, double occ, double fre, double lo, double hi) {
    __shared__ int4 s_geo[GS_FUSE_NT];
    __shared__ unsigned s_cnt[GS_FUSE_NT];
    const size_t j = blockIdx.x;
    if (*d.gate && !d.has_child[j]) return;
    const double x = d.px[j], y = d.py[j], yaw = d.pyaw[j];
    const pfc_rcp_t rres = pfc_rcp_make(gm.res);
    const int ox = pf_lf_sat_i32(floor(pf_ogm_pre(x, rres, gm.half_w))), oy = pf_lf_sat_i32(floor(pf_ogm_pre(y, rres, gm.half_h)));
    if (ox < 0 || ox >= gm.W || oy < 0 || oy >= gm.H) return;
    double* g = d.grids + (size_t)d.buf[j] * d.cells;
    const int H = gm.H;
    unsigned long long ev = 0;
    for (size_t b0 = 0; b0 < B; b0 += GS_FUSE_NT) {
        __syncthreads();
        {
            const size_t i = b0 + threadIdx.x;
            unsigned n = 0;
            int4 q = make_int4(0, 0, 0, 0);
            const double r = i < B ? ranges[i] : 0.0;
            if (i < B && r > 0.0 && isfinite(r)) {
                double sn, cs;
                pfc_sincos((yaw + angle_min) + (double)i * angle_inc, &sn, &cs);
                const double vx = pf_ogm_pre(x + r * cs, rres, gm.half_w), vy = pf_ogm_pre(y + r * sn, rres, gm.half_h);
                int ex = pf_lf_sat_i32(floor(vx)), ey = pf_lf_sat_i32(floor(vy));
                const bool inside = ex >= 0 && ex < gm.W && ey >= 0 && ey < gm.H;
                if (!inside) {
                    ex = min(max(pf_lf_sat_i32(round(vx)), 0), gm.W - 1);
                    ey = min(max(pf_lf_sat_i32(round(vy)), 0), gm.H - 1);
                }
                n = (unsigned)max(abs(ex - ox), abs(ey - oy)) + (inside ? 1u : 0u);
                q = make_int4(ox, oy, ex, ey);
            }
            s_geo[threadIdx.x] = q;
            s_cnt[threadIdx.x] = n;
        }
        __syncthreads();
        const unsigned nb = B - b0 < GS_FUSE_NT ? (unsigned)(B - b0) : GS_FUSE_NT;
        for (unsigned bb = 0; bb < nb; ++bb) {
            const unsigned n = s_cnt[bb];
            if (n == 0) continue;
            const int4 q = s_geo[bb];
            const long long dx = (long long)q.z - q.x, dy = (long long)q.w - q.y;
            const long long adx = dx < 0 ? -dx : dx, ady = dy < 0 ? -dy : dy;
            const bool xmaj = adx >= ady;
            const long long dM = xmaj ? adx : ady, dm = xmaj ? ady : adx;
            const int sx = q.x < q.z ? 1 : -1, sy = q.y < q.w ? 1 : -1;
            const long long den = 2 * dM;
            const double rden = dm ? 1.0 / (double)den : 0.0;
            for (long long kk = threadIdx.x; kk < (long long)n; kk += GS_FUSE_NT) {
                const long long mi = dm ? pf_ogm_bres_minor(kk, dm, dM, den, rden) : 0;
                const long long ddx = xmaj ? kk : mi, ddy = xmaj ? mi : kk;
                const size_t c = (size_t)(q.x + (int)(sx * ddx)) * H + (size_t)(q.y + (int)(sy * ddy));
                g[c] = pf_ogm_clamp(g[c] + (kk == dM ? occ : fre), lo, hi);
            }
            ev += threadIdx.x == 0 ? n : 0;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) atomicAdd(d.cnt + 2, ev);
}

// copy job k < cnt[1]: the fused grid of buffer job_src[k] into buffer job_dst[k] (a childless parent's, read by no one)
__global__ void __launch_bounds__(256) gs_copy_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t stride = (size_t)gridDim.x * 256, jobs = d.cnt[1];
    for (size_t k = blockIdx.y; k < jobs; k += gridDim.y) {
        const double* src = d.grids + (size_t)d.job_src[k] * d.cells;
        double* dst = d.grids + (size_t)d.job_dst[k] * d.cells;
        if (d.cells & 1) {              // odd buffers are only 8-byte aligned
            for (size_t c = (size_t)blockIdx.x * 256 + threadIdx.x; c < d.cells; c += stride) dst[c] = src[c];
            continue;
        }
        const double2* s2 = reinterpret_cast<const double2*>(src);
        double2* d2 = reinterpret_cast<double2*>(dst);
        for (size_t c = (size_t)blockIdx.x * 256 + threadIdx.x; c < d.cells / 2; c += stride) d2[c] = s2[c];
    }
}

__global__ void __launch_bounds__(256) gs_finish_kernel(GsDev d) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    d.px[t] = d.tx[t]; d.py[t] = d.ty[t]; d.pyaw[t] = d.tyaw[t];
    d.buf[t] = d.nbuf[t];
    d.w[t] = 1.0 / (double)d.n;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// The scan-matched proposal (DESIGN §3.17, include/gs_prop_math.h): launched instead of gs_move_weigh_kernel when it is enabled.
#define GS_PROP_NT PF_CSM_NT        // pf_csm_block_best's block size
#define GS_PROP_TRIG 1024           // (r cos, r sin) pairs per tile of (yaw, beam)

struct GsProp {                     // one step's proposal: the match window, the lattice and c
    double ls, as, kl, ka, c;
    int nl, na, k;
    unsigned min_hits;
};
struct GsPropOut {                  // per slot: the match winner x^ (NaN when no match ran), eta (NaN when no lattice ran), took
    double* xh;
    double* eta;
    unsigned char* took;
};

// w_raw and hit counts of the poses (x0 + a ls, y0 + b ls, normalize(yaw0 + e as)), |a|, |b| <= nl, |e| <= na, pose index
// ((a + nl) NL + b + nl) NA + e + na, into s_prod / s_hit: the weigh's used beams and arithmetic in beam order (x + r cos is one add
// on the tile's product), a hit being a beam whose window has a cell inside with l* > 0.  Thread t owns poses t, t + NT, ..; every
// thread of the CTA calls it.
__device__ void gs_prop_score(const double* g, const GsModel& m, const double* pairs, unsigned k, double x0, double y0, double yaw0,
                              int nl, double ls, int na, double as, double2* s_rc, double* s_prod, int* s_hit) {
    const int NL = 2 * nl + 1, NA = 2 * na + 1, n = NL * NL * NA;
    for (int c = threadIdx.x; c < n; c += GS_PROP_NT) { s_prod[c] = 1.0; s_hit[c] = 0; }
    const unsigned bt = GS_PROP_TRIG / (unsigned)NA;
    const pfc_rcp_t rres = pfc_rcp_make(m.res);
    for (unsigned b0 = 0; b0 < k; b0 += bt) {
        const unsigned nb = k - b0 < bt ? k - b0 : bt;
        __syncthreads();
        for (unsigned t = threadIdx.x; t < nb * (unsigned)NA; t += GS_PROP_NT) {
            const unsigned e = t / nb, j = b0 + (t - e * nb);
            const double yaw = fs_normalize_angle(yaw0 + (double)((int)e - na) * as);
            const double r = pairs[2 * j], a = pairs[2 * j + 1];
            double sn, cs;
            pfc_sincos((yaw + m.angle_min) + a, &sn, &cs);
            s_rc[t] = make_double2(r * cs, r * sn);
        }
        __syncthreads();
        for (int c = threadIdx.x; c < n; c += GS_PROP_NT) {
            const int e = c % NA, ab = c / NA;
            const double x = x0 + (double)(ab / NL - nl) * ls, y = y0 + (double)(ab % NL - nl) * ls;
            const double2* rc = s_rc + (size_t)e * nb;
            double p = s_prod[c];
            int h = s_hit[c];
            for (unsigned jj = 0; jj < nb; ++jj) {
                const int cx = pf_lf_sat_i32(floor(pf_ogm_pre(x + rc[jj].x, rres, m.half_w)));
                const int cy = pf_lf_sat_i32(floor(pf_ogm_pre(y + rc[jj].y, rres, m.half_h)));
                int any;
                const double l = gs_window_max(g, m, cx, cy, &any);
                p = p * (any ? m.z_hit * (1.0 - 1.0 / (1.0 + pfc_exp(l))) + m.q_out : m.q_out);
                h += (any && l > 0.0) ? 1 : 0;
            }
            s_prod[c] = p;
            s_hit[c] = h;
        }
    }
    __syncthreads();
}

// One CTA per particle (grid-striding): prior, match, lattice and sample of the rule at include/pfgpu.h pfgpu_gs_proposal, or the
// fallback (gs_move_weigh_kernel's move and weight).  Thread 0 does the per-particle scalar work; no floating-point atomics.
__global__ void __launch_bounds__(GS_PROP_NT) gs_propose_kernel(GsDev d, PfOdom om, uint64_t seed, uint32_t call, GsModel m,
                                                                const double* pairs, unsigned k, GsProp P, GsPropOut out) {
    __shared__ double2 s_rc[GS_PROP_TRIG];
    __shared__ double s_prod[GS_PROP_MAX_CAND];
    __shared__ int s_hit[GS_PROP_MAX_CAND];
    __shared__ double s_mu[3], s_A[9], s_xh[3], s_x[3];
    __shared__ int s_go;
    const int K = (2 * P.k + 1) * (2 * P.k + 1) * (2 * P.k + 1);
    for (size_t i = blockIdx.x; i < d.n; i += gridDim.x) {
        const double* g = d.grids + (size_t)d.buf[i] * d.cells;
        __syncthreads();                                    // the previous particle's shared state is read
        if (threadIdx.x == 0) {
            double cov[9];
            fs_odom_prior(&om, d.px[i], d.py[i], d.pyaw[i], s_mu, cov);
            s_go = !gs_prop_still(&om) && fs2_inv33(cov, s_A);
            const double nan = __longlong_as_double(0x7FF8000000000000ll);
            out.xh[3 * i] = nan; out.xh[3 * i + 1] = nan; out.xh[3 * i + 2] = nan;
            out.eta[i] = nan;
            out.took[i] = 0;
        }
        __syncthreads();
        if (s_go) {                                         // the match
            gs_prop_score(g, m, pairs, k, s_mu[0], s_mu[1], s_mu[2], P.nl, P.ls, P.na, P.as, s_rc, s_prod, s_hit);
            const int NL = 2 * P.nl + 1, NA = 2 * P.na + 1, n = NL * NL * NA;
            PfCsmBest b{-1.0, __longlong_as_double(0x7FF0000000000000ll), ~0ull};
            for (int c = threadIdx.x; c < n; c += GS_PROP_NT) {
                int a, bb, e;
                gs_prop_index(c, P.nl, P.na, &a, &bb, &e);
                const double dx = (double)a * P.ls, dy = (double)bb * P.ls, dyaw = (double)e * P.as;
                const PfCsmBest cur{s_prod[c], (dx * dx + dy * dy) + dyaw * dyaw, (unsigned long long)c};
                if (pf_csm_better(cur, b)) b = cur;
            }
            b = pf_csm_block_best(b);
            if (threadIdx.x == 0) {
                int a, bb, e;
                gs_prop_index((int)b.idx, P.nl, P.na, &a, &bb, &e);
                s_xh[0] = s_mu[0] + (double)a * P.ls;
                s_xh[1] = s_mu[1] + (double)bb * P.ls;
                s_xh[2] = fs_normalize_angle(s_mu[2] + (double)e * P.as);
                for (int j = 0; j < 3; ++j) out.xh[3 * i + j] = s_xh[j];
                s_go = (unsigned)s_hit[b.idx] >= P.min_hits;
            }
            __syncthreads();
        }
        if (s_go) {                                         // the lattice, then the sums and the sample in thread 0
            gs_prop_score(g, m, pairs, k, s_xh[0], s_xh[1], s_xh[2], P.k, P.kl, P.k, P.ka, s_rc, s_prod, s_hit);
            for (int j = threadIdx.x; j < K; j += GS_PROP_NT) s_prod[j] = gs_prop_tau(j, P.k, P.kl, P.ka, s_xh, s_mu, s_A, s_prod[j]);
            __syncthreads();
            if (threadIdx.x == 0) {
                double n0, n1, n2, unused, pose[3], eta;
                pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)i), &n0, &n1);
                pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)i), &n2, &unused);
                s_go = gs_prop_sample(s_prod, P.k, P.kl, P.ka, s_xh, P.c, n0, n1, n2, pose, &eta);
                out.eta[i] = eta;
                if (s_go) {
                    d.px[i] = pose[0]; d.py[i] = pose[1]; d.pyaw[i] = pose[2];
                    d.w[i] = d.w[i] * eta;
                    out.took[i] = 1;
                }
            }
            __syncthreads();
        }
        if (!s_go) {                                        // the fallback: gs_move_weigh_kernel's move and weight
            __syncthreads();
            if (threadIdx.x == 0) {
                double za, zb, zc, unused;
                pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)i), &za, &zb);
                pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_ODOM, call, (uint64_t)i), &zc, &unused);
                double x = d.px[i], y = d.py[i], yaw = d.pyaw[i];
                fs_odom_move(&om, za, zb, zc, &x, &y, &yaw);
                s_x[0] = x; s_x[1] = y; s_x[2] = yaw;
            }
            __syncthreads();
            gs_prop_score(g, m, pairs, k, s_x[0], s_x[1], s_x[2], 0, 0.0, 0, 0.0, s_rc, s_prod, s_hit);
            if (threadIdx.x == 0) {
                d.px[i] = s_x[0]; d.py[i] = s_x[1]; d.pyaw[i] = s_x[2];
                d.w[i] = d.w[i] * s_prod[0];
            }
        }
    }
}

__global__ void __launch_bounds__(256) gs_init_kernel(GsDev d, double x, double y, double yaw) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= d.n) return;
    d.px[t] = x; d.py[t] = y; d.pyaw[t] = yaw;
    d.w[t] = 1.0 / (double)d.n;
    d.buf[t] = (unsigned)t;
}
