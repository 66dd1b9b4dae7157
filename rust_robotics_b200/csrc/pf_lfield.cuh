// pf_lfield.cuh — set-time kernels of the likelihood-field scan model (DESIGN §3.9): the Euclidean distance field of an obstacle
// mask (compute_udf, rust_robotics_mapping/src/distance_map.rs:15-100) and the per-cell factor table q.
//
// Layout: cell (ix, iy) of a W x H grid at ix * H + iy (the reference's grid[ix][iy]); compute_udf's rows are ix, its columns iy.
#pragma once
#include "common.cuh"

#define PF_LF_INF 1e20           // distance_map.rs:10

// dt_1d (distance_map.rs:15-53) in its operation order over one line of n values: in(q) = src[q * in_stride] (or, with a mask,
// 0 for an obstacle and INF otherwise), out(q) = dst[q * out_stride].  v / z: n + 1 entries of this line's scratch.  The final
// loop reads in(v[k]), the line's input: the reference writes its output over the input and then reads d[v[k]] for v[k] < q,
// which has already been overwritten (its distances come out too small on most masks with two obstacles).
template <bool FROM_MASK>
__device__ __forceinline__ void pf_lf_dt1d(const unsigned char* mask, const double* src, size_t in_stride, double* dst,
                                           size_t out_stride, int n, int* v, double* z) {
    auto in = [&](int q) -> double {
        if constexpr (FROM_MASK) return mask[(size_t)q * in_stride] ? 0.0 : PF_LF_INF;
        else return src[(size_t)q * in_stride];
    };
    int k = 0;
    v[0] = 0;
    z[0] = -PF_LF_INF;
    z[1] = PF_LF_INF;
    for (int q = 1; q < n; ++q) {
        const double fq = in(q) + (double)((uint64_t)q * (uint64_t)q);
        int vk = v[k];
        double s = (fq - (in(vk) + (double)((uint64_t)vk * (uint64_t)vk))) / (2.0 * (double)q - 2.0 * (double)vk);
        while (s <= z[k]) {
            k -= 1;
            vk = v[k];
            s = (fq - (in(vk) + (double)((uint64_t)vk * (uint64_t)vk))) / (2.0 * (double)q - 2.0 * (double)vk);
        }
        k += 1;
        v[k] = q;
        z[k] = s;
        if (k + 1 < n + 1) z[k + 1] = PF_LF_INF;
    }
    k = 0;
    for (int q = 0; q < n; ++q) {
        while (k + 1 < n + 1 && z[k + 1] < (double)q) k += 1;
        const double dx = (double)q - (double)v[k];
        dst[(size_t)q * out_stride] = dx * dx + in(v[k]);
    }
}

// rows first: one thread per ix, the mask's line -> a (squared distances along iy)
__global__ void pf_lf_edt_rows_kernel(const unsigned char* mask, double* a, int W, int H, int* v, double* z) {
    const int ix = blockIdx.x * blockDim.x + threadIdx.x;
    if (ix >= W) return;
    const size_t o = (size_t)ix * H, s = (size_t)ix * (H + 1);
    pf_lf_dt1d<true>(mask + o, nullptr, 1, a + o, 1, H, v + s, z + s);
}
// then columns: one thread per iy, a's line -> d2 (squared distances)
__global__ void pf_lf_edt_cols_kernel(const double* a, double* d2, int W, int H, int* v, double* z) {
    const int iy = blockIdx.x * blockDim.x + threadIdx.x;
    if (iy >= H) return;
    const size_t s = (size_t)iy * (W + 1);
    pf_lf_dt1d<false>(nullptr, a + iy, (size_t)H, d2 + iy, (size_t)H, W, v + s, z + s);
}
// one thread per cell: D = sqrt(d2) in place, t = D * res, q = z_hit * gauss_likelihood(t, sigma_hit) + q_out
// (gauss_likelihood in mcl.rs:408-411's order)
__global__ void pf_lf_table_kernel(double* D, double* q, size_t cells, double res, double sigma, double z_hit, double q_out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= cells) return;
    const double dist = sqrt(D[i]);
    const double t = dist * res;
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (sigma * sigma));
    const double g = coeff * pfc_exp(-(t * t) / (2.0 * (sigma * sigma)));
    D[i] = dist;
    q[i] = z_hit * g + q_out;
}
