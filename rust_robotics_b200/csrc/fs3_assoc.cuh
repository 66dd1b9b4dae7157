// fs3_assoc.cuh — FastSLAM 2.0 step with UNKNOWN data association (DESIGN §3.5): observations arrive as (d, angle) pairs and
// every particle decides against its own map which landmark each one came from (the rule of search_correspond_landmark_id,
// ekf_slam.rs:284-308, per particle: fs_assoc_d2 of include/fs2_math.h).  One launch, fs3_assoc_kernel, replaces
// fs2_propose_kernel and the EKF launch(es) of a known-id step; fs3_assoc_mark_kernel then settles the lazy-clone bookkeeping
// and the unchanged post kernel (fs3.cuh) runs with no observation list of its own.
//
// Lazy clone.  The per-landmark generations of fs3.cuh assume that every particle updates the same landmarks in a step; here
// they do not.  So the kernel's first scan (the proposal's, which visits every slot anyway) MATERIALISES every landmark that is
// read through an ancestry row: slot i's copy, read through the row (maybe on a peer), is stored to column i of the OTHER buffer,
// and fs3_assoc_mark_kernel makes every such landmark "identity" in that buffer afterwards.  From then on the kernel reads and
// updates column i of the landmark's target buffer in place.  That is safe because rows only ever reference the buffer lmst
// names: for a landmark read through a row, peers read buffer `buf` while everybody writes buffer `buf ^ 1`; an identity landmark
// has no row, so nobody but slot i reads its column i.  (lmst is identical on every rank: every rank runs the same steps.)
#pragma once
#include "fs3.cuh"
#include "fs3_exist.cuh"

#define FS3_ASSOC_NT 128          // threads per CTA: two 64-particle groups (the partial sums of wraw_all)

// out-of-line pieces with their own copies (a routine shared with the existing kernels would be register-allocated for all
// callers); one copy per instantiation of fs3_assoc_kernel, so the untracked kernel's allocation does not depend on the tracked one
template <bool EX, bool ODOM = false>
__device__ __noinline__ int fs3a_d2(const FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11, double* q) {
    return fs_assoc_d2(L, px, py, pyaw, z0, z1, r00, r11, q);
}
template <bool EX, bool ODOM = false>
__device__ __noinline__ double fs3a_update(FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11) {
    int wrote;
    return fs_update_landmark_v(L, px, py, pyaw, z0, z1, r00, r11, &wrote, 2);    // update_landmark_and_weight fs2.rs:242-280
}
template <bool EX>
__device__ __noinline__ void fs3a_propose(double* x, double* y, double* a, const FsLm* L, double u0, double u1, double dt, double z0, double z1,
                                          double r00, double r11, double n0, double n1, double n2) {
    const double mc[9] = { 0.1, 0.0, 0.0, 0.0, 0.1, 0.0, 0.0, 0.0, 0.01 };           // MOTION_COV fs2.rs:31
    fs2_propose_pose(x, y, a, L, u0, u1, dt, z0, z1, r00, r11, mc, n0, n1, n2);
}
template <bool EX>
__device__ __noinline__ void fs3a_odom_pose(int kase, const PfOdom* m, double* x, double* y, double* a, const FsLm* L, double z0, double z1,
                                            double r00, double r11, double n0, double n1, double n2) {
    fs2_odom_pose(kase, m, x, y, a, L, z0, z1, r00, r11, n0, n1, n2);
}
__device__ __forceinline__ FsLm fs3a_load(const double* p, size_t ld) {
    FsLm L;
    L.x = p[0]; L.y = p[ld]; L.c00 = p[2 * ld]; L.c01 = p[3 * ld]; L.c10 = p[4 * ld]; L.c11 = p[5 * ld];
    return L;
}
__device__ __forceinline__ void fs3a_store(double* p, size_t ld, const FsLm& L) {
    p[0] = L.x; p[ld] = L.y; p[2 * ld] = L.c00; p[3 * ld] = L.c01; p[4 * ld] = L.c10; p[5 * ld] = L.c11;
}
// buffer that holds slot i's copy of a landmark in state s once this step's first scan has run
__device__ __forceinline__ int fs3a_tbuf(int s) { return (s & 1) ^ ((s >> 1) ? 1 : 0); }

// A(pose, z) over slot i's map (every landmark materialised): the matching slot or -1, and the lowest empty slot or -1
template <bool EX, bool ODOM = false>
__device__ __forceinline__ void fs3a_scan(const Fs3Dev& d, unsigned i, double px, double py, double pyaw, double z0, double z1, double r00,
                                          double r11, double gate_d2, int* match, int* empty) {
    const size_t ld = d.ld;
    double best = 1.7976931348623157e308;                              // f64::MAX: strict `<`, the first minimum wins
    int bl = -1, e = -1;
#pragma unroll 1
    for (unsigned l = 0; l < d.m; ++l) {
        const double* p = d.lm[fs3a_tbuf(d.lmst[l])] + (size_t)l * 6 * ld + i;
        const double c00 = p[2 * ld];
        if (!(c00 < 100.0)) { if (e < 0) e = (int)l; continue; }       // is_initialized fs2.rs:49-51
        FsLm L = fs3a_load(p, ld);
        double q;
        if (fs3a_d2<EX, ODOM>(&L, px, py, pyaw, z0, z1, r00, r11, &q) && q < best) { best = q; bl = (int)l; }
    }
    *match = bl >= 0 && best < gate_d2 ? bl : -1;
    *empty = e;
}

// One thread per local slot, a warp on 32 consecutive slots: every field read of landmark l is one coalesced 256-byte segment of
// the field-major map.  z2 = k (d, angle) pairs in device memory.  counts[0..2] += (matched, born, dropped) of this launch.
// Writes this step's unnormalised weights and 64-particle partial sums into every rank's wraw_all / part_all (the EKF epilogue's
// duty); the post kernel signals "arrived" and waits for the peers as after an EKF launch.
// EX: with landmark existence counters (fs3_exist.cuh, DESIGN §3.7).  tau is materialised with the map, maintained by the
// updates, then the negative evidence at the sampled pose; k = 0 runs the known-id k = 0 step's motion model, then the same pass.
// removed[0] += copies removed by this launch; sq0 / sq1: sqrt(Q) for the k = 0 motion step.  Without EX, k >= 1 (the host runs
// k = 0 as a known-id step) and X / sq0 / sq1 / removed are unused; they come last, so no other parameter's offset depends on them.
template <bool EX>
__global__ void __launch_bounds__(FS3_ASSOC_NT)
fs3_assoc_kernel(const __grid_constant__ Fs3Dev d, const double* __restrict__ z2, int k, double gate_d2, double u0, double u1, double dt,
                 double r00, double r11, uint64_t seed, uint32_t call, unsigned step, unsigned long long* counts,
                 const __grid_constant__ Fs3Ex X, double sq0, double sq1, unsigned long long* removed) {
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
    const bool obs = !EX || k > 0;
    const unsigned i = blockIdx.x * FS3_ASSOC_NT + threadIdx.x;
    double w = 0.0;
    unsigned cm = 0, cb = 0, cd = 0, cr = 0;
    if (i < d.n) {
        double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
        w = d.w[i];                                                    // Particle::weight
        double n0, n1, n2, unused;
        if (st->noise_call == call + 1u) { n0 = d.nz[0][i]; n1 = d.nz[1][i]; }      // drawn by the previous post kernel's idle warps
        else pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)d.off + i), &n0, &n1);
        if constexpr (!EX) pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i), &n2, &unused);
        // ---- proposal scan at the noise-free prediction x_pred (compute_proposal fs2.rs:183), materialising every landmark (and
        //      its tau) read through a row into column i of the other buffer ----
        const double z0 = obs ? z2[0] : 0.0, z1 = obs ? z2[1] : 0.0;
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
                const unsigned ref = d.rows[rcur][(size_t)((s >> 1) - 1) * ld + i];
                const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
                L = fs3a_load(base + lbase + (ref & 0x0FFFFFFFu), ld);
                fs3a_store(d.lm[buf ^ 1] + lbase + i, ld, L);
                if constexpr (EX)
                    ex[(size_t)(buf ^ 1) * plane + (size_t)l * ld + i] = X.base[ref >> 28][(size_t)buf * plane + (size_t)l * ld + (ref & 0x0FFFFFFFu)];
            } else L = fs3a_load(d.lm[buf] + lbase + i, ld);
            double q;
            if (obs && L.c00 < 100.0 && fs3a_d2<EX>(&L, xp0, xp1, xp2, z0, z1, r00, r11, &q) && q < best) { best = q; bl = (int)l; }
        }
        FsLm P = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };               // no match: compute_proposal's uninitialised branch (fs2.rs:188-191)
        if (obs) {
            if constexpr (EX) pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i), &n2, &unused);
            if (bl >= 0 && best < gate_d2) P = fs3a_load(d.lm[fs3a_tbuf(d.lmst[bl])] + (size_t)bl * 6 * ld + i, ld);
            fs3a_propose<EX>(&x, &y, &a, &P, u0, u1, dt, z0, z1, r00, r11, n0, n1, n2);
        } else {                                                       // fs2.rs:347-356: the known-id k = 0 step's motion model
            const double un0 = u0 + n0 * sq0, un1 = u1 + n1 * sq1;
            x = x + un0 * dt * cs;
            y = y + un0 * dt * sn;
            a = fs_normalize_angle(a + un1 * dt);
        }
        // ---- the observations in order: scan at the sampled pose, then update the match, or a birth, or drop; a match or a
        //      birth marks its slot as seen ----
#pragma unroll 1
        for (int j = 0; j < k; ++j) {
            const double zj0 = z2[2 * j], zj1 = z2[2 * j + 1];
            int l, e;
            fs3a_scan<EX>(d, i, x, y, a, zj0, zj1, r00, r11, gate_d2, &l, &e);
            const bool born = l < 0;
            if (l >= 0) cm++;
            else if (e >= 0) { l = e; cb++; }
            else { cd++; continue; }                                   // the map is full: the observation is dropped
            const int tb = fs3a_tbuf(d.lmst[l]);
            double* p = d.lm[tb] + (size_t)l * 6 * ld + i;
            FsLm L = fs3a_load(p, ld);
            w = w * fs3a_update<EX>(&L, x, y, a, zj0, zj1, r00, r11);
            fs3a_store(p, ld, L);
            if constexpr (EX) {
                int* t = ex + (size_t)tb * plane + (size_t)l * ld + i;
                *t = born ? (1 | FS3_EX_SEEN) : (((*t & ~FS3_EX_SEEN) + 1) | FS3_EX_SEEN);
            }
        }
        // ---- negative evidence at the sampled pose: every initialised copy in range that no observation went to ----
        if constexpr (EX) {
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
                if (v - 1 < 0) {                                       // removed: create_particles' fresh landmark, the slot is empty
                    const FsLm F = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
                    fs3a_store(p, ld, F);
                    cr++;
                }
            }
        }
        d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
    }
    // ---- weights and 64-particle partials to every rank; the counters ----
    const unsigned lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const double ws = warp_sum(w);                                     // honest (tree-order) sum: steers x3_classify only
    if (lane == 0) s_part[wid] = ws;
    const unsigned long long c3[3] = { __reduce_add_sync(0xffffffffu, cm), __reduce_add_sync(0xffffffffu, cb), __reduce_add_sync(0xffffffffu, cd) };
    if (lane < 3 && c3[lane]) atomicAdd(counts + lane, c3[lane]);
    if constexpr (EX) {
        const unsigned long long c = __reduce_add_sync(0xffffffffu, cr);
        if (lane == 3 && c) atomicAdd(removed, c);
    }
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

// fs3_assoc_kernel with the odometry motion model (DESIGN §3.15, include/fs_odom_math.h): the increment m replaces (u, dt) and
// sqrt(Q).  The proposal's landmark is the association at the noise-free move mu; the pose comes from fs2_odom_pose (no match: the
// odometry move); without observations (EX, k = 0) it is the odometry move of FastSLAM 1.0.  Everything after the pose is
// fs3_assoc_kernel's.  A kernel of its own, so that the velocity kernel's code stays as it was.
template <bool EX>
__global__ void __launch_bounds__(FS3_ASSOC_NT)
fs3_assoc_odom_kernel(const __grid_constant__ Fs3Dev d, const double* __restrict__ z2, int k, double gate_d2, PfOdom m, double r00, double r11,
                      uint64_t seed, uint32_t call, unsigned step, unsigned long long* counts, const __grid_constant__ Fs3Ex X,
                      unsigned long long* removed) {
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
    const bool obs = !EX || k > 0;
    const unsigned i = blockIdx.x * FS3_ASSOC_NT + threadIdx.x;
    double w = 0.0;
    unsigned cm = 0, cb = 0, cd = 0, cr = 0;
    if (i < d.n) {
        double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
        w = d.w[i];                                                    // Particle::weight
        double n0, n1, n2, unused;
        if (st->noise_call == call + 1u) { n0 = d.nz[0][i]; n1 = d.nz[1][i]; }      // drawn by the previous post kernel's idle warps
        else pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)d.off + i), &n0, &n1);
        // ---- proposal scan at the noise-free move mu, materialising every landmark (and its tau) read through a row into
        //      column i of the other buffer ----
        const double z0 = obs ? z2[0] : 0.0, z1 = obs ? z2[1] : 0.0;
        double xp0 = x, xp1 = y, xp2 = a;
        fs_odom_move(&m, 0.0, 0.0, 0.0, &xp0, &xp1, &xp2);
        double best = 1.7976931348623157e308;
        int bl = -1;
#pragma unroll 1
        for (unsigned l = 0; l < d.m; ++l) {
            const int s = d.lmst[l], buf = s & 1;
            const size_t lbase = (size_t)l * 6 * ld;
            FsLm L;
            if (s >> 1) {
                const unsigned ref = d.rows[rcur][(size_t)((s >> 1) - 1) * ld + i];
                const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
                L = fs3a_load(base + lbase + (ref & 0x0FFFFFFFu), ld);
                fs3a_store(d.lm[buf ^ 1] + lbase + i, ld, L);
                if constexpr (EX)
                    ex[(size_t)(buf ^ 1) * plane + (size_t)l * ld + i] = X.base[ref >> 28][(size_t)buf * plane + (size_t)l * ld + (ref & 0x0FFFFFFFu)];
            } else L = fs3a_load(d.lm[buf] + lbase + i, ld);
            double q;
            if (obs && L.c00 < 100.0 && fs3a_d2<EX, true>(&L, xp0, xp1, xp2, z0, z1, r00, r11, &q) && q < best) { best = q; bl = (int)l; }
        }
        FsLm P = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };               // no match: compute_proposal's uninitialised branch (fs2.rs:188-191)
        if (obs) {
            if (bl >= 0 && best < gate_d2) P = fs3a_load(d.lm[fs3a_tbuf(d.lmst[bl])] + (size_t)bl * 6 * ld + i, ld);
            const int kase = fs2_odom_case(&m, &P);                    // no match: P is fresh, the odometry move
            if (kase != FS_ODOM_STILL)
                pfc_normal_pair(pfc_rng_block(seed, kase == FS_ODOM_MOVE ? PFC_STREAM_FS_ODOM : PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i),
                                &n2, &unused);
            fs3a_odom_pose<EX>(kase, &m, &x, &y, &a, &P, z0, z1, r00, r11, n0, n1, n2);
        } else {                                                       // the known-id k = 0 step's odometry move
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_ODOM, call, (uint64_t)d.off + i), &n2, &unused);
            fs_odom_move(&m, n0, n1, n2, &x, &y, &a);
        }
        // ---- the observations in order: scan at the sampled pose, then update the match, or a birth, or drop; a match or a
        //      birth marks its slot as seen ----
#pragma unroll 1
        for (int j = 0; j < k; ++j) {
            const double zj0 = z2[2 * j], zj1 = z2[2 * j + 1];
            int l, e;
            fs3a_scan<EX, true>(d, i, x, y, a, zj0, zj1, r00, r11, gate_d2, &l, &e);
            const bool born = l < 0;
            if (l >= 0) cm++;
            else if (e >= 0) { l = e; cb++; }
            else { cd++; continue; }                                   // the map is full: the observation is dropped
            const int tb = fs3a_tbuf(d.lmst[l]);
            double* p = d.lm[tb] + (size_t)l * 6 * ld + i;
            FsLm L = fs3a_load(p, ld);
            w = w * fs3a_update<EX, true>(&L, x, y, a, zj0, zj1, r00, r11);
            fs3a_store(p, ld, L);
            if constexpr (EX) {
                int* t = ex + (size_t)tb * plane + (size_t)l * ld + i;
                *t = born ? (1 | FS3_EX_SEEN) : (((*t & ~FS3_EX_SEEN) + 1) | FS3_EX_SEEN);
            }
        }
        // ---- negative evidence at the sampled pose: every initialised copy in range that no observation went to ----
        if constexpr (EX) {
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
                if (v - 1 < 0) {                                       // removed: create_particles' fresh landmark, the slot is empty
                    const FsLm F = { 0.0, 0.0, 1000.0, 0.0, 0.0, 1000.0 };
                    fs3a_store(p, ld, F);
                    cr++;
                }
            }
        }
        d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
    }
    // ---- weights and 64-particle partials to every rank; the counters ----
    const unsigned lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    const double ws = warp_sum(w);                                     // honest (tree-order) sum: steers x3_classify only
    if (lane == 0) s_part[wid] = ws;
    const unsigned long long c3[3] = { __reduce_add_sync(0xffffffffu, cm), __reduce_add_sync(0xffffffffu, cb), __reduce_add_sync(0xffffffffu, cd) };
    if (lane < 3 && c3[lane]) atomicAdd(counts + lane, c3[lane]);
    if constexpr (EX) {
        const unsigned long long c = __reduce_add_sync(0xffffffffu, cr);
        if (lane == 3 && c) atomicAdd(removed, c);
    }
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

// After fs3_assoc_kernel: every landmark it materialised is identity in its target buffer; the launch's counters move to
// counts[3..5] (what pfgpu_fs_assoc_counts reports) and counts[0..2] are cleared for the next step.
__global__ void fs3_assoc_mark_kernel(const __grid_constant__ Fs3Dev d, unsigned long long* counts) {
    pf_grid_dep_sync();
    for (unsigned l = blockIdx.x * blockDim.x + threadIdx.x; l < d.m; l += gridDim.x * blockDim.x) {
        const int s = d.lmst[l];
        if (s >> 1) d.lmst[l] = fs3a_tbuf(s);
    }
    if (blockIdx.x == 0 && threadIdx.x < 3) { counts[3 + threadIdx.x] = counts[threadIdx.x]; counts[threadIdx.x] = 0ull; }
}
