// fs3_exist.cuh — landmark existence counters for the FastSLAM 2.0 step with unknown data association (DESIGN §3.7), only while
// pfgpu_fs_existence_enable holds them.  Per rank ex [2][m][ld] int32, outside the arena and Fs3Dev, with the landmark fields'
// (buffer, landmark, column) addressing: tau follows the rows and lmst exactly as the fields do.  Bit 30 of a word is the update
// loop's "seen this step" mark; the final pass clears it, so between steps a word is tau itself.
//   fs3_assoc_ex_kernel  fs3_assoc_kernel plus tau: materialised with the map, maintained by the updates, then the negative
//                        evidence at the sampled pose.  k = 0: the known-id k = 0 step's motion model, then the same pass.
//   fs3_ex_fill_kernel   tau = 1 everywhere (enable, upload, seed_map)
//   fs3_ex_pack_kernel   tau of local slots read through the rows, 0 for an empty slot
#pragma once
#include "fs3.cuh"
#include "fs3_assoc.cuh"

#define FS3_EX_SEEN 0x40000000         // matched or born in this step (cleared by the final pass)

// every rank's ex array (base[rank] = own; peers: the IPC mapping or, for in-process ranks, the sibling's pointer)
struct Fs3Ex {
    int* base[FS3_MAXG];
    double range;                      // r: a copy within r of the pose (sqrt(dx^2 + dy^2) <= r) counts as "should have been seen"
};

#ifdef __CUDACC__
// own out-of-line copies (see fs3_assoc.cuh: sharing a routine with an existing kernel would change that kernel's allocation)
__device__ __noinline__ int fs3x_d2(const FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11, double* q) {
    return fs_assoc_d2(L, px, py, pyaw, z0, z1, r00, r11, q);
}
__device__ __noinline__ double fs3x_update(FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11) {
    int wrote;
    return fs_update_landmark_v(L, px, py, pyaw, z0, z1, r00, r11, &wrote, 2);    // update_landmark_and_weight fs2.rs:242-280
}
__device__ __noinline__ void fs3x_propose(double* x, double* y, double* a, const FsLm* L, double u0, double u1, double dt, double z0, double z1,
                                          double r00, double r11, double n0, double n1, double n2) {
    const double mc[9] = { 0.1, 0.0, 0.0, 0.0, 0.1, 0.0, 0.0, 0.0, 0.01 };           // MOTION_COV fs2.rs:31
    fs2_propose_pose(x, y, a, L, u0, u1, dt, z0, z1, r00, r11, mc, n0, n1, n2);
}

// counts[0..2] += (matched, born, dropped) as fs3_assoc_kernel; removed[0] += copies removed by this launch.  sq0 / sq1: sqrt(Q)
// for the k = 0 motion step.
__global__ void __launch_bounds__(FS3_ASSOC_NT)
fs3_assoc_ex_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3Ex X, const double* __restrict__ z2, int k, double gate_d2,
                    double u0, double u1, double dt, double sq0, double sq1, double r00, double r11, uint64_t seed, uint32_t call, unsigned step,
                    unsigned long long* counts, unsigned long long* removed) {
    pf_grid_dep_sync();
    __shared__ double s_part[FS3_ASSOC_NT / 32];
    if (d.G > 1 && d.wait_inline) {             // peers' rows / poses / maps / tau are stable once their previous post kernel is over
        if (threadIdx.x == 0) fs3_wait_peers(d, 1, step);
        __syncthreads();
    }
    const Fs3State* st = d.st;
    const int cur = st->cur, rcur = st->rcur, par = (int)(step & 1u);
    const size_t ld = d.ld, plane = (size_t)d.m * ld;
    int* const ex = X.base[d.rank];
    const unsigned i = blockIdx.x * FS3_ASSOC_NT + threadIdx.x;
    double w = 0.0;
    unsigned cm = 0, cb = 0, cd = 0, cr = 0;
    if (i < d.n) {
        double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
        w = d.w[i];
        double n0, n1, n2, unused;
        if (st->noise_call == call + 1u) { n0 = d.nz[0][i]; n1 = d.nz[1][i]; }
        else pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)d.off + i), &n0, &n1);
        // ---- proposal scan at x_pred, materialising every landmark (and its tau) read through a row into column i of the other buffer ----
        const double z0 = k > 0 ? z2[0] : 0.0, z1 = k > 0 ? z2[1] : 0.0;
        double sn, cs;
        pfc_sincos(a, &sn, &cs);
        const double xp0 = x + u0 * dt * cs, xp1 = y + u0 * dt * sn, xp2 = fs_normalize_angle(a + u1 * dt);
        double best = 1.7976931348623157e308;
        int bl = -1;
#pragma unroll 1
        for (unsigned l = 0; l < d.m; ++l) {
            const int s = d.lmst[l], buf = s & 1;
            const size_t lbase = (size_t)l * 6 * ld;
            FsLm L;
            if (s >> 1) {
                const unsigned ref = d.rows[rcur][(size_t)((s >> 1) - 1) * ld + i], col = ref & 0x0FFFFFFFu;
                const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
                L = fs3a_load(base + lbase + col, ld);
                fs3a_store(d.lm[buf ^ 1] + lbase + i, ld, L);
                ex[(size_t)(buf ^ 1) * plane + (size_t)l * ld + i] = X.base[ref >> 28][(size_t)buf * plane + (size_t)l * ld + col];
            } else L = fs3a_load(d.lm[buf] + lbase + i, ld);
            double q;
            if (k > 0 && L.c00 < 100.0 && fs3x_d2(&L, xp0, xp1, xp2, z0, z1, r00, r11, &q) && q < best) { best = q; bl = (int)l; }
        }
        if (k > 0) {
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i), &n2, &unused);
            FsLm P = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };           // no match: compute_proposal's uninitialised branch (fs2.rs:188-191)
            if (bl >= 0 && best < gate_d2) P = fs3a_load(d.lm[fs3a_tbuf(d.lmst[bl])] + (size_t)bl * 6 * ld + i, ld);
            fs3x_propose(&x, &y, &a, &P, u0, u1, dt, z0, z1, r00, r11, n0, n1, n2);
        } else {                                                       // fs2.rs:347-356: the known-id k = 0 step's motion model
            const double un0 = u0 + n0 * sq0, un1 = u1 + n1 * sq1;
            x = x + un0 * dt * cs;
            y = y + un0 * dt * sn;
            a = fs_normalize_angle(a + un1 * dt);
        }
        // ---- the observations in order; a match or a birth marks its slot as seen ----
#pragma unroll 1
        for (int j = 0; j < k; ++j) {
            const double zj0 = z2[2 * j], zj1 = z2[2 * j + 1];
            double best2 = 1.7976931348623157e308;
            int l = -1, e = -1;
#pragma unroll 1
            for (unsigned s = 0; s < d.m; ++s) {                       // fs3a_scan
                const double* p = d.lm[fs3a_tbuf(d.lmst[s])] + (size_t)s * 6 * ld + i;
                if (!(p[2 * ld] < 100.0)) { if (e < 0) e = (int)s; continue; }
                FsLm L = fs3a_load(p, ld);
                double q;
                if (fs3x_d2(&L, x, y, a, zj0, zj1, r00, r11, &q) && q < best2) { best2 = q; l = (int)s; }
            }
            if (!(l >= 0 && best2 < gate_d2)) l = -1;
            const bool born = l < 0;
            if (l >= 0) cm++;
            else if (e >= 0) { l = e; cb++; }
            else { cd++; continue; }                                   // the map is full: the observation is dropped
            const int tb = fs3a_tbuf(d.lmst[l]);
            double* p = d.lm[tb] + (size_t)l * 6 * ld + i;
            FsLm L = fs3a_load(p, ld);
            w = w * fs3x_update(&L, x, y, a, zj0, zj1, r00, r11);
            fs3a_store(p, ld, L);
            int* t = ex + (size_t)tb * plane + (size_t)l * ld + i;
            *t = born ? (1 | FS3_EX_SEEN) : (((*t & ~FS3_EX_SEEN) + 1) | FS3_EX_SEEN);
        }
        // ---- negative evidence at the sampled pose: every initialised copy in range that no observation went to ----
#pragma unroll 1
        for (unsigned l = 0; l < d.m; ++l) {
            const int tb = fs3a_tbuf(d.lmst[l]);
            int* t = ex + (size_t)tb * plane + (size_t)l * ld + i;
            const int v = *t;
            if (v & FS3_EX_SEEN) { *t = v & ~FS3_EX_SEEN; continue; }
            double* p = d.lm[tb] + (size_t)l * 6 * ld + i;
            if (!(p[2 * ld] < 100.0)) continue;
            const double dx = p[0] - x, dy = p[ld] - y;
            if (!(sqrt(dx * dx + dy * dy) <= X.range)) continue;
            *t = v - 1;
            if (v - 1 < 0) {                                           // removed: create_particles' fresh landmark, the slot is empty
                const FsLm F = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
                fs3a_store(p, ld, F);
                cr++;
            }
        }
        d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
    }
    // ---- weights and 64-particle partials to every rank; the counters ----
    const unsigned lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const double ws = warp_sum(w);
    if (lane == 0) s_part[wid] = ws;
    const unsigned long long c4[4] = { __reduce_add_sync(0xffffffffu, cm), __reduce_add_sync(0xffffffffu, cb), __reduce_add_sync(0xffffffffu, cd),
                                       __reduce_add_sync(0xffffffffu, cr) };
    if (lane < 3 && c4[lane]) atomicAdd(counts + lane, c4[lane]);
    if (lane == 3 && c4[3]) atomicAdd(removed, c4[3]);
    __syncthreads();
#pragma unroll 1
    for (int gg = 0; gg < d.G; ++gg) {
        double* wr = (d.G > 1 ? reinterpret_cast<double*>(d.peer[gg] + d.o_wraw[par]) : d.wraw[par]) + d.off;
        if (i < d.n) wr[i] = w;
        const unsigned ge = blockIdx.x * (FS3_ASSOC_NT / 64) + threadIdx.x;
        if (threadIdx.x < FS3_ASSOC_NT / 64 && ge < d.npart) {
            double* pp = d.G > 1 ? reinterpret_cast<double*>(d.peer[gg] + d.o_part[par]) : d.part[par];
            pp[(size_t)d.rank * d.npart + ge] = s_part[2 * threadIdx.x] + s_part[2 * threadIdx.x + 1];
        }
    }
}

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
