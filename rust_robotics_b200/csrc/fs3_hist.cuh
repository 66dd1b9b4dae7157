// fs3_hist.cuh — FastSLAM particle path history (DESIGN §3.6): a ring of per-step poses and resample parents, the path of one
// particle read back through it, and the genealogy smoother's per-step moments.  Not part of the step's arithmetic: the record
// kernel is one ordinary launch behind the post kernel (only while history is enabled); the queries are ordinary launches between
// steps, like pfgpu_fs_moments.
//
//   fs3_hist_record_kernel   entry e <- the live pose columns and, per local slot, the parent: the global ancestor when the step
//                            resampled (idx), the slot itself when it did not (idx is stale then) or when the entry is a root.  It
//                            reads st->cur and st->gate on the device, so recording needs no host synchronisation.  It never
//                            releases its dependents early: the next step's griddepcontrol.wait covers it (DESIGN §3.4's argument).
//   fs3_hist_path_kernel     one lineage, newest entry first: a chain of dependent loads (the parent read at entry s is the address
//                            of the loads at entry s - 1), one memory round trip per entry.  Latency bound by construction.
//   fs3_hist_moments_kernel  one thread per local slot walks its own lineage newest to oldest; at every entry each block merges
//                            its threads' (w_i, pose) about that entry's centre with fs3_pose_block_merge, one partial per block.
//   fs3_hist_merge_kernel    one thread per entry merges the block partials in block order.
// Ring layout per rank (cap entries, column stride ld, same on every rank): px [cap][ld], py [cap][ld], pyaw [cap][ld] (f64),
// par [cap][ld] (u32, global slot of the parent at the previous entry).  28 bytes per particle and entry.
#pragma once
#include "fs3.cuh"
#include "fs3_est.cuh"

#define FS3_HIST_NT FS3_EST_NT                 // fs3_pose_block_merge's block size
#define FS3_HIST_SCRATCH_CAP ((size_t)64 << 20) // block partials of one moments launch: fewer entries per launch when n is large

// every rank's ring (base[rank] = own; peers: the IPC mapping or, for in-process ranks, the plain pointer)
struct Fs3Hist {
    const char* base[FS3_MAXG];
    unsigned cap, ld, n;                       // entries, column stride, local slots per rank
};

__host__ __device__ __forceinline__ size_t fs3_hist_bytes(size_t cap, size_t ld) { return cap * ld * (3 * sizeof(double) + sizeof(unsigned)); }

#ifdef __CUDACC__
// entry e of global slot g: its pose and parent, from the owner rank's ring
__device__ __forceinline__ void fs3_hist_load(const Fs3Hist& H, unsigned e, unsigned g, double* x, double* y, double* a, unsigned* par) {
    const unsigned r = g / H.n, c = g % H.n;
    const char* B = H.base[r];
    const size_t col = (size_t)e * H.ld + c, plane = (size_t)H.cap * H.ld;
    const double* p = reinterpret_cast<const double*>(B);
    *x = p[col]; *y = p[plane + col]; *a = p[2 * plane + col];
    *par = reinterpret_cast<const unsigned*>(B + 3 * plane * sizeof(double))[col];
}
__device__ __forceinline__ unsigned fs3_hist_prev(unsigned e, unsigned cap) { return e == 0 ? cap - 1 : e - 1; }

// root = 1: every parent is the slot itself (enable, upload, seed_map)
__global__ void __launch_bounds__(FS3_HIST_NT) fs3_hist_record_kernel(const __grid_constant__ Fs3Dev d, char* ring, unsigned cap, unsigned e, int root) {
    const unsigned t = blockIdx.x * FS3_HIST_NT + threadIdx.x;
    if (t >= d.n) return;
    const int cur = d.st->cur;
    const bool resampled = !root && d.st->gate != 0;
    const size_t plane = (size_t)cap * d.ld, col = (size_t)e * d.ld + t;
    double* p = reinterpret_cast<double*>(ring);
    p[col] = d.px[cur][t]; p[plane + col] = d.py[cur][t]; p[2 * plane + col] = d.pyaw[cur][t];
    reinterpret_cast<unsigned*>(ring + 3 * plane * sizeof(double))[col] = resampled ? d.idx[t] : d.off + t;
}

// the newest L entries of global slot g's lineage, newest first: entry e_last, then its predecessors.  slot / pose: [L] / [L][3]
__global__ void fs3_hist_path_kernel(const __grid_constant__ Fs3Hist H, unsigned e_last, unsigned L, unsigned g, unsigned* slot, double* pose) {
    if (threadIdx.x != 0) return;
    unsigned s = g, e = e_last;
#pragma unroll 1
    for (unsigned k = 0; k < L; ++k) {
        double x, y, a; unsigned par;
        fs3_hist_load(H, e, s, &x, &y, &a, &par);
        slot[k] = s; pose[3 * (size_t)k] = x; pose[3 * (size_t)k + 1] = y; pose[3 * (size_t)k + 2] = a;
        s = par; e = fs3_hist_prev(e, H.cap);
    }
}

// entries k0 .. k1 - 1 (newest first; entry index e0 at k0) of every local slot's lineage.  lin: [n] the slot each lineage has
// reached at entry k0 (k0 = 0: the slot itself); left at entry k1 for the next launch.  ctr: [L][3] the centres (the lineage of
// global slot n_glob - 1).  part: [k1 - k0][gridDim.x].
__global__ void __launch_bounds__(FS3_HIST_NT) fs3_hist_moments_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3Hist H, unsigned e0, unsigned k0,
                                                                       unsigned k1, unsigned* lin, const double* ctr, Fs3PoseMom* part) {
    __shared__ Fs3PoseMom sm[FS3_HIST_NT / 32];
    const unsigned i = blockIdx.x * FS3_HIST_NT + threadIdx.x;
    const bool live = i < d.n;
    const double w = live ? d.w[i] : 0.0;                     // the CURRENT weight of slot i, at every entry of its lineage
    unsigned s = live ? (k0 == 0 ? d.off + i : lin[i]) : 0u, e = e0;
#pragma unroll 1
    for (unsigned k = k0; k < k1; ++k) {
        Fs3PoseMom v = {0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}};
        if (live) {
            double x, y, a; unsigned par;
            fs3_hist_load(H, e, s, &x, &y, &a, &par);
            const double dx = x - ctr[3 * (size_t)k], dy = y - ctr[3 * (size_t)k + 1], dt = fs3_wrap_angle(a - ctr[3 * (size_t)k + 2]);
            // fs3_est_pose_kernel's per-thread sums for a single deviation (shift = the deviation itself)
            const double w0 = w * 0.0;
            if (w != 0.0) {
                const double a0 = w0 / w;
                v.w = w; v.m[0] = dx + a0; v.m[1] = dy + a0; v.m[2] = dt + a0;
                const double q0 = w0 * 0.0 - w0 * a0;
#pragma unroll
                for (int j = 0; j < 6; ++j) v.q[j] = q0;
            }
            s = par;
        }
        fs3_pose_block_merge(v, sm);
        if (threadIdx.x == 0) part[(size_t)(k - k0) * gridDim.x + blockIdx.x] = v;
        __syncthreads();                                      // (sm is reused)
        e = fs3_hist_prev(e, H.cap);
    }
    if (live) lin[i] = s;
}

// out[k] (pfgpu_fs_pose_moments: w, c[3], mean[3], m2[6]) for k in k0 .. k1 - 1: block partials merged in block order
__global__ void fs3_hist_merge_kernel(const Fs3PoseMom* part, unsigned nblocks, unsigned k0, unsigned k1, const double* ctr, double* out) {
    const unsigned k = k0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= k1) return;
    Fs3PoseMom acc = {0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}};
    const Fs3PoseMom* p = part + (size_t)(k - k0) * nblocks;
#pragma unroll 1
    for (unsigned b = 0; b < nblocks; ++b) fs3_pose_merge(acc, p[b]);
    double* o = out + 13 * (size_t)k;
    o[0] = acc.w;
    for (int j = 0; j < 3; ++j) o[1 + j] = ctr[3 * (size_t)k + j];
    for (int j = 0; j < 3; ++j) o[4 + j] = acc.m[j];
    for (int j = 0; j < 6; ++j) o[7 + j] = acc.q[j];
}
#endif
