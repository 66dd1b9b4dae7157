// fs3_exist.cuh — landmark existence counters for the FastSLAM 2.0 step with unknown data association (DESIGN §3.7), only while
// pfgpu_fs_existence_enable holds them.  Per rank ex [2][m][ld] int32, outside the arena and Fs3Dev, with the landmark fields'
// (buffer, landmark, column) addressing: tau follows the rows and lmst exactly as the fields do.  Bit 30 of a word is the update
// loop's "seen this step" mark; the final pass clears it, so between steps a word is tau itself.
//   fs3_assoc_kernel<true> (fs3_assoc.cuh): tau materialised with the map, maintained by the updates, then the negative
//                        evidence at the sampled pose
//   fs3_ex_fill_kernel   tau = 1 everywhere (enable, upload, seed_map)
//   fs3_ex_pack_kernel   tau of local slots read through the rows, 0 for an empty slot
#pragma once
#include "fs3.cuh"

#define FS3_EX_SEEN 0x40000000         // matched or born in this step (cleared by the final pass)

// every rank's ex array (base[rank] = own; peers: the IPC mapping or, for in-process ranks, the sibling's pointer)
struct Fs3Ex {
    int* base[FS3_MAXG];
    double range;                      // r: a copy within r of the pose (sqrt(dx^2 + dy^2) <= r) counts as "should have been seen"
};

#ifdef __CUDACC__
__global__ void __launch_bounds__(256) fs3_ex_fill_kernel(int* ex, size_t count) {
    for (size_t e = (size_t)blockIdx.x * 256 + threadIdx.x; e < count; e += (size_t)gridDim.x * 256) ex[e] = 1;
}

// out[ip * m + l] = tau of landmark l of local slot i0 + ip (0 when the slot is empty), read through the rows
__global__ void __launch_bounds__(256) fs3_ex_pack_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3Ex X, int* out, size_t i0, size_t cnt) {
    const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x;
    if (e >= cnt * d.m) return;
    const size_t ip = e / d.m, l = e % d.m, plane = (size_t)d.m * d.ld;
    const unsigned i = (unsigned)(i0 + ip);
    const int s = d.lmst[l], buf = s & 1, rcur = d.st->rcur;
    const double c00 = fs3_lm_src(d, l, i, s, rcur)[2 * (size_t)d.ld];
    unsigned rk = (unsigned)d.rank, col = i;
    if (s >> 1) { const unsigned ref = d.rows[rcur][(size_t)((s >> 1) - 1) * d.ld + i]; rk = ref >> 28; col = ref & 0x0FFFFFFFu; }
    out[e] = c00 < 100.0 ? X.base[rk][(size_t)buf * plane + l * d.ld + col] : 0;
}
#endif
