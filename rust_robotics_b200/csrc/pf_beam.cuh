// pf_beam.cuh — the beam measurement model (DESIGN §3.11): the clearance table built at set time, the skipping ray caster a beam
// step and the expected-scan query share, and the per-beam factor.  Included by pf_kernels.cuh after pf_lf_sat_i32.
//
// Layout: cell (ix, iy) of a W x H grid at ix * H + iy, like the likelihood field's tables.
#pragma once
#include "common.cuh"

#define PF_BEAM_CAP 255          // clearance is stored in one byte

// The beam model's launch argument: the clearance table, world_to_grid's constants and the factor's constants
struct PfBeam {
    const unsigned char* clr = nullptr;
    double res = 1.0, half_w = 0.0, half_h = 0.0;   // half_w = W as f64 / 2.0 (world_to_grid, occupancy_grid_map.rs:144-153)
    double max_range = 0.0, angle_min = 0.0;
    double hit = 0.0;            // z_hit * coeff, coeff = 1 / sqrt(2 pi (sigma_hit * sigma_hit))
    double denom = 1.0;          // 2 * (sigma_hit * sigma_hit)
    double shrt = 0.0;           // z_short * lambda_short
    double lambda = 0.0;         // lambda_short
    double q_rand = 0.0;         // z_rand / max_range
    double z_max = 0.0;
    int W = 0, H = 0;
    int skip = 1;                // 0: step one cell at a time (PFGPU_BEAM_SKIP=0)
};

// The expected range along one beam from cell (ix0, iy0) of the pose (x, y), heading `angle` (DESIGN §3.11).  The cells are
// bresenham_line(c0, c1)'s (occupancy_grid_map.rs:164-193) in its closed form: step i = 0 .. d_major moves i cells along the major
// axis (x when |dx| >= |dy|) and floor((2 i d_minor + d_major - 1) / (2 d_major)) along the minor one.  The first cell that is
// occupied or outside stops the ray at r = res * sqrt(dx^2 + dy^2) (its integer offset from c0); none up to c1: r = max_range.
// Every step moves at most one cell along each axis, so a cell of clearance c (Chebyshev distance to the nearest occupied or outside
// cell) guarantees steps i + 1 .. i + c - 1 are free and inside: the caster jumps to i + c, and returns the plain loop's bits.
__device__ __forceinline__ double pf_beam_cast(const PfBeam& bm, const pfc_rcp_t& rres, double x, double y, int ix0, int iy0,
                                               double angle) {
    if (ix0 < 0 || ix0 >= bm.W || iy0 < 0 || iy0 >= bm.H) return 0.0;
    double s, c;
    pfc_sincos(angle, &s, &c);
    const int ix1 = pf_lf_sat_i32(floor(pfc_div_by(x + bm.max_range * c, rres) + bm.half_w));
    const int iy1 = pf_lf_sat_i32(floor(pfc_div_by(y + bm.max_range * s, rres) + bm.half_h));
    const long long dx = (long long)ix1 - ix0, dy = (long long)iy1 - iy0;
    const long long adx = dx < 0 ? -dx : dx, ady = dy < 0 ? -dy : dy;
    const bool xmaj = adx >= ady;
    const long long dM = xmaj ? adx : ady, dm = xmaj ? ady : adx;
    const int sx = ix0 < ix1 ? 1 : -1, sy = iy0 < iy1 ? 1 : -1;
    const long long den = 2 * dM;
    const double rden = dm ? 1.0 / (double)den : 0.0;      // an estimate of the minor offset, corrected in integers below
    long long i = 0, mi = 0;
    while (i <= dM) {
        mi = 0;
        if (dm) {
            const long long num = 2 * i * dm + dM - 1;          // < 2^44: exact in f64 and in the products below
            mi = (long long)((double)num * rden);
            if (mi * den > num) mi -= 1;
            else if ((mi + 1) * den <= num) mi += 1;
        }
        const long long ox = xmaj ? i : mi, oy = xmaj ? mi : i;
        const int cx = ix0 + (int)(sx * ox), cy = iy0 + (int)(sy * oy);
        if (cx < 0 || cx >= bm.W || cy < 0 || cy >= bm.H) break;
        const unsigned cl = __ldg(bm.clr + ((size_t)cx * (size_t)bm.H + (size_t)cy));
        if (cl == 0) break;
        i += bm.skip ? (long long)cl : 1;
    }
    if (i > dM) return bm.max_range;
    return bm.res * sqrt((double)(i * i + mi * mi));
}

// one used beam's factor: r is the measured range (max_range for a max reading), rhat the expected one
__device__ __forceinline__ double pf_beam_factor(const PfBeam& bm, const pfc_rcp_t& rdenom, double r, double rhat) {
    const double z = r - rhat;
    double q = bm.hit * pfc_exp(pfc_div_by(-(z * z), rdenom));
    if (z < 0.0) q = q + bm.shrt * pfc_exp(-(bm.lambda * r));
    return q + (r >= bm.max_range ? bm.z_max : bm.q_rand);
}

// world_to_grid of the pose: the start cell of every beam
__device__ __forceinline__ void pf_beam_start(const PfBeam& bm, const pfc_rcp_t& rres, double x, double y, int* ix0, int* iy0) {
    *ix0 = pf_lf_sat_i32(floor(pfc_div_by(x, rres) + bm.half_w));
    *iy0 = pf_lf_sat_i32(floor(pfc_div_by(y, rres) + bm.half_h));
}

// ---- set time: the clearance table (Chebyshev distance in cells to the nearest occupied cell or the ring outside, capped) ----
// pass 1, one thread per cell: g = distance along iy to the nearest obstacle of the line ix (the ring at iy = -1 and iy = H counts)
__global__ void pf_beam_clr_lines_kernel(const unsigned char* mask, unsigned char* g, int W, int H) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)W * (size_t)H) return;
    const int iy = (int)(t % (size_t)H);
    const unsigned char* line = mask + (t - (size_t)iy);
    int best = min(min(iy + 1, H - iy), PF_BEAM_CAP);
    for (int d = 0; d < best; ++d) {
        if ((iy - d >= 0 && line[iy - d]) || (iy + d < H && line[iy + d])) { best = d; break; }
    }
    g[t] = (unsigned char)best;
}
// pass 2, one thread per cell: clr = min over the lines ix + d of max(|d|, g), bounded by the ring at ix = -1 and ix = W
__global__ void pf_beam_clr_cols_kernel(const unsigned char* g, unsigned char* clr, int W, int H) {
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= (size_t)W * (size_t)H) return;
    const int ix = (int)(t / (size_t)H);
    int best = min(min(ix + 1, W - ix), (int)g[t]);
    for (int d = 1; d < best; ++d) {
        int v = PF_BEAM_CAP;
        if (ix - d >= 0) v = min(v, (int)g[t - (size_t)d * H]);
        if (ix + d < W) v = min(v, (int)g[t + (size_t)d * H]);
        best = min(best, max(d, v));
    }
    clr[t] = (unsigned char)best;
}

// ---- the expected-scan query: r_hat for n poses x B beams, one thread per (pose, beam); out[p * B + b] ----
__global__ void __launch_bounds__(256) pf_beam_raycast_kernel(PfBeam bm, const double* pose3, size_t n, size_t B, double angle_inc,
                                                                double* out) {
    const size_t t = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * B) return;
    const size_t p = t / B, b = t - p * B;
    const double x = pose3[3 * p], y = pose3[3 * p + 1], yaw = pose3[3 * p + 2];
    const pfc_rcp_t rres = pfc_rcp_make(bm.res);
    int ix0, iy0;
    pf_beam_start(bm, rres, x, y, &ix0, &iy0);
    out[t] = pf_beam_cast(bm, rres, x, y, ix0, iy0, (yaw + bm.angle_min) + (double)b * angle_inc);
}
