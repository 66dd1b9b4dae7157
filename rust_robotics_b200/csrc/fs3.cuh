// fs3.cuh — FastSLAM 1.0 step (fs1.rs = crates/rust_robotics_slam/src/fastslam1.rs) in TWO kernels per step, the same on
// one GPU and on G GPUs of one NVLink domain:
//
//   fs3_ekf_kernel    predict_particle (fs1.rs:123-137) + update_landmark (fs1.rs:140-183) for every (particle, observation)
//                     pair + the weight products in observation order (fs1.rs:250-256).  A CTA owns 64 particles (two per
//                     lane: 128-bit loads/stores of adjacent columns, two independent dependency chains per thread) and runs
//                     one warp per observation.  Its epilogue pushes the 64 unnormalised weights and their (tree) partial
//                     sum to EVERY rank.
//   fs3_post_kernel   everything after the per-particle work (fs1.rs:258-265, resample fs1.rs:206-234): exact sequential
//                     sums S, S2, the CDF (x3_core.h), normalisation, N_eff gate, the comb in closed form, index search,
//                     pose clone and the lazy clone of the maps — one launch of at most one co-resident CTA per SM, synchronised
//                     through a counter in global memory (one such barrier for a step that does not resample, two for one
//                     that resamples from the certified CDF, four or five for one that runs the exact S2 and CDF sums).  Every rank runs it on ALL n_glob weights (they are 8 B per particle), so the ranks never
//                     wait for each other inside it.
//
// HBM layout per rank (n local particles, column stride ld = n rounded up to 64, m landmarks):
//   px, py, pyaw [2][ld]        pose columns (ping-pong across resamples; st->cur selects the live set)
//   lm [2][m][6][ld]            landmark EKF state, field-major: the six fields of landmark l are six contiguous columns
//   rows [2][m][ld] (u32)       LAZY CLONE BY GENERATION.  The reference's resample deep-copies every particle's map
//                               (particles[j].clone(), fs1.rs:227: 48*m bytes per particle).  Here a resample moves no map
//                               data at all.  Landmarks whose last EKF update happened in the same inter-resample period
//                               share one ancestry row: rows[r][i] = (rank << 28 | column) where slot i's copy of those
//                               landmarks lives.  lmst[l] = buffer bit | (row + 1) << 1, row + 1 == 0: "identity" (slot i's
//                               copy is column i of its own rank).  A resample composes only the LIVE rows (a handful:
//                               one per period in which some not-since-observed landmark was last updated),
//                               rows'[r][t] = rows[r]@(ancestor of t), and gives the identity landmarks one new row that
//                               holds the ancestors themselves.  The next EKF update of a landmark reads through its row
//                               (over NVLink when the ancestor lives on another rank), writes column i of the OTHER buffer
//                               and the landmark is "identity" again.
//   wraw_all [2][n_glob], part_all [2][n_glob/64]   this step's unnormalised weights of ALL particles and their 64-particle
//                               partial sums (double-buffered by step parity; every rank's EKF epilogue writes its slice
//                               into every rank's copy)
// Cross-rank protocol (G > 1): arrive[g] = step+1 is stored into every peer after rank g's EKF pushed its weights; the post
// kernel of step s waits for all arrive == s+1.  done[g] = step+1 after rank g's post kernel; the EKF kernel of step s+1
// waits for all done == s+1 (rows / poses / maps of a peer are only read between those two points, when nobody writes them).
#pragma once
#include <type_traits>
#include "common.cuh"
#include "x3_core.h"
#include "../../include/fs_ekf_math.h"
#include "../../include/fs2_math.h"
#include "../../include/fs_odom_math.h"

#define FS3_MAXG 8
#define FS3_MAX_OBS 31            // observations per EKF launch (one warp each, plus the helper warp)
#define FS3_MAX_TILES 160
#define FS3_ENT_CAP 512           // dirty values itemised per sum (more: that sum takes the serial walk)
#define FS3_ROUNDS 8              // grid-barrier rounds per launch (each one arrival counter, each exact sum one round)
#define FS3_SPIN_LIMIT (1u << 27)
#define FS3_MAX_LM 65536          // landmarks per particle: row ids (< m) fit the u16 row list
#define FS3_ROW_CHUNK 1024        // live rows a post-kernel CTA lists in shared memory at a time (more: several passes)
#define FS3_K1_ROWS 8             // live rows whose gathers the one-value post kernel (KC = 1) keeps in flight per batch
#define FS3_CERT_MAX_LOG2N 16     // certified CDF up to 2^16 particles: about 4 n^3 2^-53 comb values fall within its bound of a
                                  // CDF value, 1/8 at 2^16, 1 at 2^17, 64 at 2^19 (where it would almost always be refused)

// Sum slots (what fs3_value adds): raw weights, squares of the normalised ones (PF / MCL N_eff near its threshold), the normalised
// ones, the normalised ones / S2 (the CDF), the comb (n not a power of two).  flagsg[FS3_CERT_FLAG]: a CTA refused the certificate.
enum Fs3Slot { FS3_S, FS3_Q, FS3_S2, FS3_CDF, FS3_COMB, FS3_SLOTS, FS3_CERT_FLAG = FS3_SLOTS };
// Grid-barrier rounds (< FS3_ROUNDS), one meaning each.  An exact sum's round also indexes where it publishes its results, and
// its parity picks the half of the block scratch (Fs3Sh::wd / wu / wi): two sums of one parity need a block barrier between them.
enum Fs3Round { FS3_R_S, FS3_R_S2, FS3_R_CDF, FS3_R_COMB, FS3_R_CERT, FS3_R_CDF_DONE, FS3_R_BORDER };   // fs3_post_kernel
enum Pf3Round { PF3_R_S, PF3_R_Q, PF3_R_CDF, PF3_R_CDF_DONE, PF3_R_TILES };                           // pf3_post_kernel (pf3.cuh)

__host__ __device__ __forceinline__ unsigned fs3_bm_words(unsigned m) { return (m + 31u) / 32u; }
__host__ __device__ __forceinline__ unsigned fs3_bm_ld(unsigned m) { return fs3_bm_words(m) + FS3_MAX_TILES; }

struct Fs3Obs { double d, angle; int lm_id; int pad; };
struct Fs3ObsParam { Fs3Obs o[32]; };

struct Fs3State {                 // device-resident; written by the last CTA of a launch, read by the next launch
    int cur, rcur;                // live pose buffer / live rows buffer
    unsigned resamples;           // resamples so far = Philox call index of the next comb draw (fs1.rs:220)
    int gate;                     // last step resampled
    unsigned ekf_done, post_done; // CTA completion counters
    unsigned bar_count, bar_gen;  // grid barrier of the post kernel
    int err;                      // sticky: 1 = a barrier or a peer flag timed out
    int serial_walks, cert_fail, dirty_last, border_cnt;
    int cdf_exact;                // resamples that ran the exact S2 and CDF sums (certificate refused, or not applicable)
    unsigned noise_call;          // nz[] holds the predict noise of EKF call `noise_call - 1` (0: none); written by the post kernel
    double S, Q, neff, S2, r0;
};
struct Fs3Rec {                   // mapped pinned host memory: what a caller reads after a step (one 64-byte record)
    unsigned long long seq;       // step + 1, written last
    unsigned long long best_idx;  // get_best_particle fs1.rs:269-274 (global slot; the LAST maximum)
    double best_w, bx, by, byaw, neff;
    int gate, err;
};

struct Fs3Res { double total; unsigned long long Ptot; int D; int fail; };
// Workspace of the exact sums (fs3_xsum, fs3_xsum_emit, fs3_serial_walk) and grid barriers of one post kernel (fs3_sum_alloc)
struct Fs3Sum {
    unsigned long long* tileP; double* tileQ;                  // [FS3_SLOTS][FS3_MAX_TILES] clean-increment sum per tile; [tiles] sum w_raw^2
    unsigned* entCnt;                                          // [FS3_SLOTS] dirty values appended so far (any order)
    unsigned* entKey; unsigned* entTile; unsigned long long* entP; double* entV; int* entL;   // [FS3_SLOTS][FS3_ENT_CAP]
    unsigned* bar;                                             // [FS3_ROUNDS] grid-barrier arrival counters of the running launch
    unsigned* resflag;                                         // [FS3_ROUNDS] "the chain of this round is evaluated" flags
    Fs3Res* res;                                               // [FS3_ROUNDS] its results: total, entry count, failure
    unsigned long long* resTP; unsigned* resKey; unsigned long long* resP; double* resAft;   // [FS3_ROUNDS][tiles] / [FS3_ROUNDS][FS3_ENT_CAP] for the scans
    double* tileEnd;                                           // [FS3_MAX_TILES] last CDF value of every tile (coarse level of the index search)
    int* flagsg;                                               // [FS3_SLOTS + 1] "bad value seen" per sum, then the certificate flag
    unsigned long long* trace;                                 // optional [48] phase timestamps (PFGPU_POST_TRACE)
    Fs3State* st;                                              // the launch's state (FastSLAM: Fs3Dev::st): serial_walks, cert_fail, dirty_last, err, post_done
    // what a serial walk re-reads (fs3_value): raw[par] for FS3_S, wn for FS3_Q, FS3_S2 and FS3_CDF
    const double* raw[2];                                      // [n] raw weights, by step parity
    const double* wn;                                          // [n] normalised weights
    unsigned n;                                                // values per sum
};
// x's arrays and Fs3State in ONE zeroed allocation (x.tileP is its base), and x.n; the caller sets raw, wn.  No peer touches it.
inline cudaError_t fs3_sum_alloc(Fs3Sum& x, unsigned n, bool trace) {
    const size_t nsl = (size_t)FS3_SLOTS * FS3_MAX_TILES, nen = (size_t)FS3_SLOTS * FS3_ENT_CAP, nre = (size_t)FS3_ROUNDS * FS3_ENT_CAP;
    char* base = nullptr; size_t off = 0;
    auto take = [&](auto*& p, size_t cnt) { p = base ? reinterpret_cast<std::remove_reference_t<decltype(p)>>(base + off) : nullptr; off += (cnt * sizeof(*p) + 255) & ~(size_t)255; };
    for (int pass = 0; pass < 2; ++pass) {                     // pass 0 sizes the allocation, pass 1 carves it
        if (pass) { const cudaError_t e = cudaMalloc(&base, off); if (e != cudaSuccess) return e; off = 0; }
        take(x.tileP, nsl); take(x.tileQ, FS3_MAX_TILES); take(x.entCnt, FS3_SLOTS);
        take(x.entKey, nen); take(x.entTile, nen); take(x.entP, nen); take(x.entV, nen); take(x.entL, nen);
        take(x.bar, FS3_ROUNDS); take(x.resflag, FS3_ROUNDS); take(x.res, FS3_ROUNDS); take(x.resTP, (size_t)FS3_ROUNDS * FS3_MAX_TILES);
        take(x.resKey, nre); take(x.resP, nre); take(x.resAft, nre); take(x.tileEnd, FS3_MAX_TILES); take(x.flagsg, FS3_SLOTS + 1);
        take(x.st, 1); x.trace = nullptr;
        if (trace) take(x.trace, 48);
    }
    x.n = n;
    return cudaMemset(base, 0, off);
}
inline void fs3_sum_free(Fs3Sum& x) { cudaFree(x.tileP); x.tileP = nullptr; }
struct Fs3Dev {
    unsigned n, n_glob, off, m, ld;           // local / global particles, first global slot, landmarks, column stride
    int G, rank;
    int wait_inline;                          // 1: kernels spin on the peers' flags themselves; 0: the host launches fs3_wait_kernel
                                              // in front of them (ranks sharing one GPU must not hold SMs while they wait)
    unsigned npart;                           // partial sums per rank (= ld / 64)
    int exact_cdf;                            // 1: every resample runs the exact S2 and CDF sums (PFGPU_FS_EXACT_CDF=1)
    Fs3State* st;
    int* lmst;                                // [m]
    char* peer[FS3_MAXG];                     // arena base of every rank (peer[rank] = own)
    size_t o_flags, o_wraw[2], o_part[2], o_px[2], o_py[2], o_pyaw[2], o_rows[2], o_lm[2];   // offsets inside an arena
    double *px[2], *py[2], *pyaw[2], *lm[2];  // own arena
    unsigned* rows[2];
    double* wraw[2]; double* part[2];         // own copies of wraw_all / part_all
    double* w;                                // [ld] normalised weights of the local slots (Particle::weight)
    double* nz[2];                            // [ld] each: N(0,1) pair of every local slot for the NEXT predict (fs1.rs:129-130), precomputed
                                              // by idle warps of the post kernel (it depends on seed, call and slot only)
    double* wn_all;                           // [n_glob] normalised weights of all slots (post-kernel scratch, fallback walks)
    double* cum_all;                          // [n_glob] CDF of the resample: certified fl(P_j / S), or the exact one
    double* rcomb_all;                        // [n_glob] exact comb (only when n_glob is not a power of two)
    unsigned* idx;                            // [ld] global ancestor of local slot t at the last resample
    Fs3Sum x;                                 // the post kernel's exact sums (n_glob values; x.trace also times the EKF launch)
    unsigned* rowbm;                          // [2][fs3_bm_ld(m)] by step parity: live-row bitmap ([ceil(m/32)] words),
                                              // then one "has an identity landmark" flag per post-kernel CTA
    double* tileBw; unsigned* tileBi;         // [FS3_MAX_TILES] best (weight, global slot) per tile
    Fs3Rec* rec;
};

__device__ __forceinline__ unsigned fs3_ref(int rank, unsigned col) { return ((unsigned)rank << 28) | col; }
__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) { unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_release_gpu(unsigned* p, unsigned v) { asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
// arrival at a grid-wide counter in ONE instruction: release of everything this CTA wrote before the block barrier in front of
// it, acquire for whoever turns out to be the last to arrive (instead of fence + relaxed atomic + fence)
__device__ __forceinline__ unsigned atom_add_acq_rel_gpu(unsigned* p, unsigned v) {
    unsigned o; asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(o) : "l"(p), "r"(v) : "memory"); return o;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) { asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory"); }
__device__ __forceinline__ unsigned* fs3_flag(const Fs3Dev& d, int owner, int which, int src) {
    return reinterpret_cast<unsigned*>(d.peer[owner] + d.o_flags + ((size_t)which * FS3_MAXG + (size_t)src) * 128);
}
// wait until every peer's flag `which` in MY arena has reached `target` (flags only grow)
__device__ __forceinline__ void fs3_wait_peers(const Fs3Dev& d, int which, unsigned target) {
    for (int g = 0; g < d.G; ++g) {
        if (g == d.rank) continue;
        const unsigned* f = fs3_flag(d, d.rank, which, g);
        unsigned spins = 0;
        while ((int)(ld_acquire_sys(f) - target) < 0) {
            if (++spins > FS3_SPIN_LIMIT) { d.st->err = 1; break; }
            __nanosleep(40);
        }
    }
}
__device__ __forceinline__ void fs3_signal_peers(const Fs3Dev& d, int which, unsigned value) {   // call with >= G threads
    const int g = threadIdx.x;
    if (g < d.G && g != d.rank) { __threadfence_system(); st_release_sys(fs3_flag(d, g, which, d.rank), value); }
}

// =====================================================================================================================
// EKF kernel: persistent, software-pipelined
// =====================================================================================================================
// One CTA per SM walks groups of 64 particles (two per lane).  Warps 0..k-1 each own one observation: per group they take the
// group's landmark columns out of a cp.async landing buffer (issued one group ahead, so the HBM latency of the next group
// hides behind the ~600 FP64 instructions of this one), run update_landmark for their two pairs, store the columns and
// publish the two likelihood factors.  Warps k.. (up to three) are helpers: helper h runs predict_particle for trips h, h + nh, ...
// one trip AHEAD (sincos + the motion model on the N(0,1) pairs the previous post kernel's idle warps drew: a dependent chain
// that would otherwise sit in front of every group) and the weight products of the same trips one trip BEHIND.  Hand-offs go
// through shared-memory mbarriers, four per stage (pose full / empty, likelihoods full / empty), see below.
__device__ __noinline__ double fs3_update_slow(FsLm* L, double px, double py, double pyaw, double z0, double z1, double r00, double r11, int variant) {
    int wrote;
    return fs_update_landmark_v(L, px, py, pyaw, z0, z1, r00, r11, &wrote, variant);   // 1.0 whenever the weight is left alone
}
__device__ __forceinline__ void cp_async16(void* smem, const void* g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"((unsigned)__cvta_generic_to_shared(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem, const void* g) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((unsigned)__cvta_generic_to_shared(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }
// Hand-offs between the helper and the EKF warps: mbarriers in shared memory, 4 per stage (stage = trip % number of helper
// warps): which = 0 pose full (1 arrival: the helper), 1 pose empty (k arrivals: one per EKF warp), 2 lik full (k), 3 lik empty (1).
// Unlike a named barrier, waiting on a phase does not make the EKF warps wait for EACH OTHER: a warp whose pose is ready goes
// on, so the warps drift apart and stop hitting the FP64 / XU pipes in the same phase of the computation at the same time.
__device__ __forceinline__ void mb_init(unsigned long long* b, unsigned count) {
    asm volatile("mbarrier.init.shared.b64 [%0], %1;" :: "r"((unsigned)__cvta_generic_to_shared(b)), "r"(count) : "memory");
}
__device__ __forceinline__ void mb_arrive(unsigned long long* b) {
    asm volatile("{ .reg .b64 t; mbarrier.arrive.shared.b64 t, [%0]; }" :: "r"((unsigned)__cvta_generic_to_shared(b)) : "memory");
}
__device__ __forceinline__ void mb_wait(unsigned long long* b, unsigned parity) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(b);
    unsigned ok;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(ok) : "r"(a), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __noinline__ void fs3_normal_pair(uint64_t seed, uint32_t call, uint64_t index, double* z0, double* z1) {
    pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, index), z0, z1);
}
__device__ __noinline__ void fs3_sincos(double x, double* s, double* c) { pfc_sincos(x, s, c); }

// flags: bit 0 = first launch of the step (predict; weights start from Particle::weight)
//        bit 1 = the poses are already this step's (FastSLAM 2.0: fs2_propose_kernel sampled them), no motion model here
//        bit 2 = FastSLAM 2.0's update_landmark_and_weight (fs2.rs:242-280) instead of update_landmark (fs1.rs:140-183)
//        bit 3 = release the next kernel of the stream for scheduling right away (pf_grid_launch_dependents)
// blockDim = 32 * (k_obs + nh), nh >= 1 helper warps.  Dynamic shared memory (doubles):
//   pose [nh][3][64] | lik [nh][k][64] | landing [2][k][6][64]
template <int MAXT>
__global__ void __launch_bounds__(MAXT, 1)
fs3_ekf_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3ObsParam po, double u0, double u1, double dt,
               double sq0, double sq1, double r00, double r11, uint64_t seed, uint32_t call, int k_obs, int flags, unsigned step) {
    pf_grid_dep_sync();
    if (flags & 8) pf_grid_launch_dependents();
    extern __shared__ __align__(16) double s_dyn[];
    const int lane = threadIdx.x & 31, wj = threadIdx.x >> 5;
    const int nh = (int)(blockDim.x >> 5) - k_obs;
    double* s_pose = s_dyn;                                         // [nh][3][64]
    double* s_lik = s_dyn + (size_t)nh * 192;                       // [nh][k][64]
    double* s_land = s_lik + (size_t)nh * k_obs * 64;               // [2][k][6][64]
    __shared__ unsigned long long s_mb[3][4];                       // [stage][which]
    Fs3State* st = d.st;
    if (threadIdx.x < 12) { const int sg = threadIdx.x >> 2, wh = threadIdx.x & 3; mb_init(&s_mb[sg][wh], (wh == 1 || wh == 2) ? (unsigned)(k_obs > 0 ? k_obs : 1) : 1u); }
    __syncthreads();
    if (d.G > 1 && d.wait_inline) {             // peers' rows / poses / maps are stable once their previous post kernel is over
        if (threadIdx.x == 0) fs3_wait_peers(d, 1, step);
        __syncthreads();
    }
    const int cur = st->cur, rcur = st->rcur, par = (int)(step & 1u);
    const size_t ld = d.ld;
    const unsigned ngroups = d.ld / 64;
    if (d.x.trace && blockIdx.x == 0 && threadIdx.x == 0 && (flags & 1)) {     // step timeline (PFGPU_POST_TRACE): [32] idle before this launch
        unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (d.x.trace[36]) d.x.trace[32] += t - d.x.trace[36];
        d.x.trace[38] = t; d.x.trace[37] = 0ull;
    }
    if (wj >= k_obs) {
        // ========== helper warp h: predict for trips h, h + nh, ... (ahead), weight products of the same trips (behind) ==========
        const int h = wj - k_obs;
        double2 Wp = make_double2(0.0, 0.0);                              // weights of this helper's previous trip
        unsigned gprev = 0;
        bool first = true;
        unsigned use = 0;                                                 // how often this helper's stage has been handed over
        for (unsigned g = blockIdx.x + (unsigned)h * gridDim.x; ; g += (unsigned)nh * gridDim.x) {
            const bool have = g < ngroups;
            double2 Wn = make_double2(0.0, 0.0);
            if (have) {
                const unsigned i0 = g * 64u + 2u * (unsigned)lane;
                const double* wsrc = (flags & 1) ? d.w : d.wraw[par] + d.off;
                Wn = *reinterpret_cast<const double2*>(wsrc + i0);                  // needed one trip later
                const double2 X = *reinterpret_cast<const double2*>(d.px[cur] + i0), Y = *reinterpret_cast<const double2*>(d.py[cur] + i0);
                const double2 A = *reinterpret_cast<const double2*>(d.pyaw[cur] + i0);
                double xs[2] = { X.x, X.y }, ys[2] = { Y.x, Y.y }, as[2] = { A.x, A.y };
                if ((flags & 3) == 1) { // predict_particle + motion_model fs1.rs:70-77,123-137, in place
                    const bool pre = st->noise_call == call + 1u;        // the post kernel of the previous step drew this call's noise already
                    double2 Z0 = make_double2(0.0, 0.0), Z1 = make_double2(0.0, 0.0);
                    if (pre) { Z0 = *reinterpret_cast<const double2*>(d.nz[0] + i0); Z1 = *reinterpret_cast<const double2*>(d.nz[1] + i0); }
#pragma unroll 1
                    for (int q = 0; q < 2; ++q) {
                        double z0 = q ? Z0.y : Z0.x, z1 = q ? Z1.y : Z1.x;
                        if (!pre) fs3_normal_pair(seed, call, (uint64_t)d.off + i0 + q, &z0, &z1);
                        const double xq = q ? xs[1] : xs[0], yq = q ? ys[1] : ys[0], aq = q ? as[1] : as[0];
                        const double un0 = u0 + z0 * sq0;                      // fs1.rs:129
                        const double un1 = u1 + z1 * sq1;                      // fs1.rs:130
                        double sn, cs;
                        fs3_sincos(aq, &sn, &cs);
                        const double nx = xq + un0 * dt * cs;                  // motion_model fs1.rs:73-75
                        const double ny = yq + un0 * dt * sn;
                        const double na = fs_normalize_angle(aq + un1 * dt);
                        if (q) { xs[1] = nx; ys[1] = ny; as[1] = na; } else { xs[0] = nx; ys[0] = ny; as[0] = na; }
                    }
                    *reinterpret_cast<double2*>(d.px[cur] + i0) = make_double2(xs[0], xs[1]);
                    *reinterpret_cast<double2*>(d.py[cur] + i0) = make_double2(ys[0], ys[1]);
                    *reinterpret_cast<double2*>(d.pyaw[cur] + i0) = make_double2(as[0], as[1]);
                }
                if (k_obs > 0) {
                    if (!first) mb_wait(&s_mb[h][1], (use - 1u) & 1u);            // the EKF warps have read what this stage held
                    double* sp = s_pose + h * 192;
                    *reinterpret_cast<double2*>(sp + 2 * lane) = make_double2(xs[0], xs[1]);
                    *reinterpret_cast<double2*>(sp + 64 + 2 * lane) = make_double2(ys[0], ys[1]);
                    *reinterpret_cast<double2*>(sp + 128 + 2 * lane) = make_double2(as[0], as[1]);
                    __syncwarp();
                    if (lane == 0) mb_arrive(&s_mb[h][0]);
                }
            }
            // weights of this helper's previous trip (of this trip when there are no observations):
            // w = (((w * l_0) * l_1) ...) in observation order (fs1.rs:181 inside the loops fs1.rs:250-256)
            if (k_obs > 0 ? !first : have) {
                const unsigned ge = k_obs > 0 ? gprev : g;
                const unsigned i0 = ge * 64u + 2u * (unsigned)lane;
                double w0 = k_obs > 0 ? Wp.x : Wn.x, w1 = k_obs > 0 ? Wp.y : Wn.y;
                if (k_obs > 0) {
                    mb_wait(&s_mb[h][2], (use - 1u) & 1u);                       // every EKF warp has published its factors of that trip
                    const double* sl = s_lik + (size_t)h * k_obs * 64;
#pragma unroll 1
                    for (int j = 0; j < k_obs; ++j) {
                        const double2 l = *reinterpret_cast<const double2*>(sl + j * 64 + 2 * lane);
                        w0 = w0 * l.x; w1 = w1 * l.y;
                    }
                    __syncwarp();
                    if (lane == 0) mb_arrive(&s_mb[h][3]);
                }
                const bool v0 = i0 < d.n, v1 = i0 + 1 < d.n;
                if (!v0) w0 = 0.0;
                if (!v1) w1 = 0.0;
                const double psum = warp_sum(w0 + w1);                           // honest (tree-order) sum: steers x3_classify only
#pragma unroll 1
                for (int gg = 0; gg < d.G; ++gg) {
                    double* wr = (d.G > 1 ? reinterpret_cast<double*>(d.peer[gg] + d.o_wraw[par]) : d.wraw[par]) + d.off;
                    if (v1) *reinterpret_cast<double2*>(wr + i0) = make_double2(w0, w1);
                    else if (v0) wr[i0] = w0;
                    if (lane == 0) {
                        double* pp = d.G > 1 ? reinterpret_cast<double*>(d.peer[gg] + d.o_part[par]) : d.part[par];
                        pp[(size_t)d.rank * d.npart + ge] = psum;
                    }
                }
            }
            if (!have) break;
            Wp = Wn; gprev = g; first = false; use++;
        }
        if (d.x.trace && h == 0 && lane == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax(d.x.trace + 37, t); }
        return;
    }
    // =============================== EKF warps: one observation each ===============================
    const Fs3Obs ob = po.o[wj];
    const int sl = d.lmst[ob.lm_id];
    const bool ident = (sl >> 1) == 0;
    const int buf = sl & 1;
    const size_t lbase = (size_t)ob.lm_id * 6 * ld;
    const double* lm_own = d.lm[buf] + lbase;
    double* lm_dst = d.lm[ident ? buf : (buf ^ 1)] + lbase;           // own columns; the other buffer when read through a row
    const unsigned* row = ident ? nullptr : d.rows[rcur] + (size_t)((sl >> 1) - 1) * ld;
    unsigned g = blockIdx.x;
    if (g >= ngroups) return;
    uint2 ref_cur = make_uint2(0u, 0u), ref_next = make_uint2(0u, 0u);
    if (!ident) {
        ref_cur = *reinterpret_cast<const uint2*>(row + g * 64u + 2u * (unsigned)lane);
        if (g + gridDim.x < ngroups) ref_next = *reinterpret_cast<const uint2*>(row + (g + gridDim.x) * 64u + 2u * (unsigned)lane);
    }
    // trip -1 .. last: at the top of trip `it` the landing copies of trip it are in flight; the body issues those of trip it + 1
    int stage = 0;
    for (int it = -1; ; ++it) {
        const unsigned gi = it < 0 ? g : g + gridDim.x;            // group whose copies are issued in this pass
        const bool issue_ok = gi < ngroups;
        FsLm L[2];
        if (it >= 0) {
            // [A] this group's landmark columns out of the landing buffer
            cp_async_wait_all();
            const double* land = s_land + ((size_t)(it & 1) * k_obs + wj) * 384 + 2 * lane;
            const double2 a = *reinterpret_cast<const double2*>(land), b = *reinterpret_cast<const double2*>(land + 64);
            const double2 c = *reinterpret_cast<const double2*>(land + 128), e = *reinterpret_cast<const double2*>(land + 192);
            const double2 f = *reinterpret_cast<const double2*>(land + 256), hh = *reinterpret_cast<const double2*>(land + 320);
            L[0].x = a.x; L[1].x = a.y; L[0].y = b.x; L[1].y = b.y; L[0].c00 = c.x; L[1].c00 = c.y;
            L[0].c01 = e.x; L[1].c01 = e.y; L[0].c10 = f.x; L[1].c10 = f.y; L[0].c11 = hh.x; L[1].c11 = hh.y;
        }
        // [B] issue the landing copies of the next group (each lane copies exactly the 12 doubles it will consume)
        if (issue_ok) {
            double* land = s_land + ((size_t)((it + 1) & 1) * k_obs + wj) * 384 + 2 * lane;
            const unsigned i0n = gi * 64u + 2u * (unsigned)lane;
            if (ident) {
#pragma unroll
                for (int f = 0; f < 6; ++f) cp_async16(land + f * 64, lm_own + f * ld + i0n);
            } else {                                  // lazy clone: the ancestors' copies, through the landmark's row
                const uint2 ref = it < 0 ? ref_cur : ref_next;
                const unsigned rr[2] = { ref.x, ref.y };
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[rr[q] >> 28] + d.o_lm[buf]) + lbase : lm_own;
                    const double* p = base + (rr[q] & 0x0FFFFFFFu);
#pragma unroll
                    for (int f = 0; f < 6; ++f) cp_async8(land + f * 64 + q, p + f * ld);
                }
                if (it >= 0 && gi + gridDim.x < ngroups) ref_next = *reinterpret_cast<const uint2*>(row + (gi + gridDim.x) * 64u + 2u * (unsigned)lane);
            }
            cp_async_commit();
        }
        if (it < 0) continue;
        const unsigned i0 = g * 64u + 2u * (unsigned)lane;
        // [C] the predicted pose of this group
        const unsigned upar = (unsigned)(it / nh) & 1u;             // parity of this use of the stage
        mb_wait(&s_mb[stage][0], upar);
        double px[2], py[2], pyaw[2];
        {
            const double* sp = s_pose + stage * 192;
            const double2 X = *reinterpret_cast<const double2*>(sp + 2 * lane), Y = *reinterpret_cast<const double2*>(sp + 64 + 2 * lane);
            const double2 A = *reinterpret_cast<const double2*>(sp + 128 + 2 * lane);
            px[0] = X.x; px[1] = X.y; py[0] = Y.x; py[1] = Y.y; pyaw[0] = A.x; pyaw[1] = A.y;
        }
        __syncwarp();
        if (lane == 0) mb_arrive(&s_mb[stage][1]);
        // [D] update_landmark for the two pairs
        double lik[2] = { 1.0, 1.0 };
        int ok[2];
        fs_update_landmark_fastw<2>(L, px, py, pyaw, ob.d, ob.angle, r00, r11, lik, ok);
        if (!(ok[0] & ok[1])) {          // rare: a pair outside the fast form's domain -> the contract form, on a COPY (taking the address
#pragma unroll                           // of L itself would park all twelve landmark doubles in local memory on every trip)
            for (int q = 0; q < 2; ++q)
                if (!ok[q] && i0 + q < d.n) {
                    FsLm T = q ? L[1] : L[0];
                    const double lk = fs3_update_slow(&T, q ? px[1] : px[0], q ? py[1] : py[0], q ? pyaw[1] : pyaw[0], ob.d, ob.angle, r00, r11, (flags & 4) ? 2 : 1);
                    if (q) { L[1] = T; lik[1] = lk; } else { L[0] = T; lik[0] = lk; }
                }
        }
        double* o = lm_dst + i0;
        *reinterpret_cast<double2*>(o) = make_double2(L[0].x, L[1].x);
        *reinterpret_cast<double2*>(o + ld) = make_double2(L[0].y, L[1].y);
        *reinterpret_cast<double2*>(o + 2 * ld) = make_double2(L[0].c00, L[1].c00);
        *reinterpret_cast<double2*>(o + 3 * ld) = make_double2(L[0].c01, L[1].c01);
        *reinterpret_cast<double2*>(o + 4 * ld) = make_double2(L[0].c10, L[1].c10);
        *reinterpret_cast<double2*>(o + 5 * ld) = make_double2(L[0].c11, L[1].c11);
        // [E] likelihood factors to the helper
        if (it >= nh) mb_wait(&s_mb[stage][3], upar ^ 1u);          // the helper has consumed this stage's previous factors
        *reinterpret_cast<double2*>(s_lik + ((size_t)stage * k_obs + wj) * 64 + 2 * lane) = make_double2(lik[0], lik[1]);
        __syncwarp();
        if (lane == 0) mb_arrive(&s_mb[stage][2]);
        g += gridDim.x;
        if (g >= ngroups) break;
        stage = stage + 1 == nh ? 0 : stage + 1;
    }
    if (d.x.trace && wj == 0 && lane == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); atomicMax(d.x.trace + 37, t); }
}

// FastSLAM 2.0 (fs2.rs = crates/rust_robotics_slam/src/fastslam2.rs): the pose of every particle is sampled from the proposal that
// fuses the motion prior with the step's FIRST observation (compute_proposal fs2.rs:173-216, sample_pose fs2.rs:219-239,
// set_pose fs2.rs:77-81) — one thread per particle, ahead of the EKF launch (which then runs with flags bit 1).  The landmark is
// read the way the EKF warps read it: own column, or the ancestor's (possibly on a peer) through the landmark's row.
__global__ void __launch_bounds__(128)
fs2_propose_kernel(const __grid_constant__ Fs3Dev d, Fs3Obs ob, double u0, double u1, double dt, double r00, double r11,
                   uint64_t seed, uint32_t call, unsigned step) {
    pf_grid_dep_sync();
    Fs3State* st = d.st;
    if (d.G > 1 && d.wait_inline) {             // peers' rows / maps are stable once their previous post kernel is over
        if (threadIdx.x == 0) fs3_wait_peers(d, 1, step);
        __syncthreads();
    }
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int cur = st->cur, rcur = st->rcur;
    const size_t ld = d.ld;
    const int sl = d.lmst[ob.lm_id];
    const int buf = sl & 1;
    const size_t lbase = (size_t)ob.lm_id * 6 * ld;
    const double* p = d.lm[buf] + lbase + i;
    if (sl >> 1) {
        const unsigned ref = d.rows[rcur][(size_t)((sl >> 1) - 1) * ld + i];
        const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
        p = base + lbase + (ref & 0x0FFFFFFFu);
    }
    FsLm L;
    L.x = p[0]; L.y = p[ld]; L.c00 = p[2 * ld]; L.c01 = p[3 * ld]; L.c10 = p[4 * ld]; L.c11 = p[5 * ld];
    double n0, n1, n2, unused;
    if (st->noise_call == call + 1u) { n0 = d.nz[0][i]; n1 = d.nz[1][i]; }          // drawn by the previous post kernel's idle warps
    else fs3_normal_pair(seed, call, (uint64_t)d.off + i, &n0, &n1);
    pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i), &n2, &unused);
    const double mc[9] = { 0.1, 0.0, 0.0, 0.0, 0.1, 0.0, 0.0, 0.0, 0.01 };          // MOTION_COV fs2.rs:31
    double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
    fs2_propose_pose(&x, &y, &a, &L, u0, u1, dt, ob.d, ob.angle, r00, r11, mc, n0, n1, n2);
    d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
}

// The odometry motion model (DESIGN §3.15, include/fs_odom_math.h).  FastSLAM 1.0, and FastSLAM 2.0 without observations: every
// pose moved by the increment m in place, one thread per slot, ahead of the EKF launch (which then runs with flags bit 1, so its
// helper warps only gather the weights).  (za, zb) are the velocity model's pair, taken from nz[] when the previous post kernel
// drew it; zc is PFC_STREAM_FS_ODOM's.
__global__ void __launch_bounds__(128)
fs3_odom_predict_kernel(const __grid_constant__ Fs3Dev d, PfOdom m, uint64_t seed, uint32_t call, unsigned step) {
    pf_grid_dep_sync();
    if (d.G > 1 && d.wait_inline) {             // peers read this rank's poses until their previous post kernel is over
        if (threadIdx.x == 0) fs3_wait_peers(d, 1, step);
        __syncthreads();
    }
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int cur = d.st->cur;
    double za, zb, zc, unused;
    if (d.st->noise_call == call + 1u) { za = d.nz[0][i]; zb = d.nz[1][i]; }
    else pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)d.off + i), &za, &zb);
    pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_ODOM, call, (uint64_t)d.off + i), &zc, &unused);
    double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
    fs_odom_move(&m, za, zb, zc, &x, &y, &a);
    d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
}

// (fs2_propose_kernel's read, for its odometry twin) slot i's copy of landmark l as it stands before this step's updates: own column, or the ancestor's through the landmark's row
__device__ __forceinline__ FsLm fs3_read_lm(const Fs3Dev& d, int rcur, int l, unsigned i) {
    const size_t ld = d.ld;
    const int sl = d.lmst[l];
    const int buf = sl & 1;
    const size_t lbase = (size_t)l * 6 * ld;
    const double* p = d.lm[buf] + lbase + i;
    if (sl >> 1) {
        const unsigned ref = d.rows[rcur][(size_t)((sl >> 1) - 1) * ld + i];
        const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
        p = base + lbase + (ref & 0x0FFFFFFFu);
    }
    FsLm L;
    L.x = p[0]; L.y = p[ld]; L.c00 = p[2 * ld]; L.c01 = p[3 * ld]; L.c10 = p[4 * ld]; L.c11 = p[5 * ld];
    return L;
}
// FastSLAM 2.0 with odometry and observations: fs2_propose_kernel's twin, the proposal's prior from the increment m
// (fs2_odom_case / fs2_odom_pose: standing still takes the noise-free move, an uninitialised landmark the odometry move)
__global__ void __launch_bounds__(128)
fs2_propose_odom_kernel(const __grid_constant__ Fs3Dev d, Fs3Obs ob, PfOdom m, double r00, double r11, uint64_t seed, uint32_t call,
                        unsigned step) {
    pf_grid_dep_sync();
    Fs3State* st = d.st;
    if (d.G > 1 && d.wait_inline) {             // peers' rows / maps are stable once their previous post kernel is over
        if (threadIdx.x == 0) fs3_wait_peers(d, 1, step);
        __syncthreads();
    }
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.n) return;
    const int cur = st->cur, rcur = st->rcur;
    const FsLm L = fs3_read_lm(d, rcur, ob.lm_id, i);
    const int kase = fs2_odom_case(&m, &L);
    double n0 = 0.0, n1 = 0.0, n2 = 0.0, unused;
    if (kase != FS_ODOM_STILL) {
        if (st->noise_call == call + 1u) { n0 = d.nz[0][i]; n1 = d.nz[1][i]; }
        else pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_FS_PREDICT, call, (uint64_t)d.off + i), &n0, &n1);
        pfc_normal_pair(pfc_rng_block(seed, kase == FS_ODOM_MOVE ? PFC_STREAM_FS_ODOM : PFC_STREAM_FS2_POSE3, call, (uint64_t)d.off + i), &n2, &unused);
    }
    double x = d.px[cur][i], y = d.py[cur][i], a = d.pyaw[cur][i];
    fs2_odom_pose(kase, &m, &x, &y, &a, &L, ob.d, ob.angle, r00, r11, n0, n1, n2);
    d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = a;
}

// lazy-clone bookkeeping after an EKF launch: the landmarks it updated through a row now live in own columns of the other
// buffer.  (Its own tiny launch between the pieces of a split observation list; the post kernel does it for the last piece.)
__device__ __forceinline__ void fs3_mark_updated(const Fs3Dev& d, const Fs3ObsParam& po, int k_obs) {
    for (int j = threadIdx.x; j < k_obs; j += blockDim.x) {
        const int l = po.o[j].lm_id, s = d.lmst[l];
        if (s >> 1) d.lmst[l] = (s & 1) ^ 1;
    }
}
// one-warp launches that stand in for the kernels' own waits / signals when several ranks share a GPU (wait_inline == 0)
__global__ void fs3_wait_kernel(const __grid_constant__ Fs3Dev d, int which, unsigned target) {
    pf_grid_dep_sync();
    if (threadIdx.x == 0) fs3_wait_peers(d, which, target);
}
__global__ void fs3_signal_kernel(const __grid_constant__ Fs3Dev d, int which, unsigned value) {
    pf_grid_dep_sync();
    fs3_signal_peers(d, which, value);
}
__global__ void fs3_mark_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3ObsParam po, int k_obs) {
    pf_grid_dep_sync();
    fs3_mark_updated(d, po, k_obs);
}

// =====================================================================================================================
// post kernel
// =====================================================================================================================
// Written for LATENCY: it moves ~1 MB, so what it costs is instruction fetch (every instruction runs once per warp), waits
// at barriers and dependent memory round trips.  The L2 holds none of its code when a step starts (the EKF launch streams
// more than the L2 through it), so the code every step runs — the S sum, the gate, the certified CDF, normalisation — is laid
// out as one straight run inside the kernel (fs3_xsum_body, fs3_xsum_emit_body, inline divisions), where sequential fetch
// covers it, and what a config-3 step rarely runs stays out of line (fs3_xsum / fs3_xsum_emit for the exact S2, CDF and comb
// sums, fs3_chain_wide, fs3_serial_walk, fs3_classify, fs3_div).  Four block barriers and one grid barrier per sum; the chain
// over the dirty values is evaluated by warp 0 with warp primitives while the other warps sleep at a block barrier; grid
// barriers are per-round arrival counters (no generation juggling).
template <int NT>
struct Fs3Sh {
    double wd[2][NT / 32]; unsigned long long wu[2][NT / 32]; int wi[2][NT / 32];   // warp totals (double-buffered by round)
    double red[2][NT / 32];
    unsigned long long tPoff[FS3_MAX_TILES];                  // clean-increment sum in front of every tile
    unsigned ukey[FS3_ENT_CAP], skey[FS3_ENT_CAP];            // dirty values: global index (unsorted / sorted)
    unsigned long long sP[FS3_ENT_CAP]; double sV[FS3_ENT_CAP]; int sL[FS3_ENT_CAP];
    double bef[FS3_ENT_CAP], aft[FS3_ENT_CAP];                // exact sum in front of / right after each dirty value
    double total, tbase, bcast;
    unsigned long long Ptot;
    int D, fail, last, lead, rany;
    unsigned jr[2];
    unsigned rowscan[2][NT / 32];                             // live-row list: live rows / first free row per warp
    unsigned short rowl[FS3_ROW_CHUNK];                       // live rows [base, base + FS3_ROW_CHUNK) of the ascending list
    double tend[FS3_MAX_TILES];                               // last CDF value of every tile
    x3_comb_table comb;
};

#define FS3_TRACE(k) do { if (x.trace && blockIdx.x == 0 && threadIdx.x == 0) { unsigned long long t__; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t__)); x.trace[k] += t__ - t_prev; t_prev = t__; } } while (0)

// grid barrier `round` of this launch: every CTA arrives once per round; the counters are zeroed by the launch's last CTA
template <int NT>
__device__ __forceinline__ void fs3_grid_sync(const Fs3Sum& x, int round, unsigned nblocks) {
    __syncthreads();
    if (threadIdx.x == 0) {
        (void)atom_add_acq_rel_gpu(x.bar + round, 1u);
        unsigned spins = 0;
#pragma unroll 1
        while (ld_acquire_gpu(x.bar + round) < nblocks) { if (++spins > FS3_SPIN_LIMIT) { x.st->err = 1; break; } __nanosleep(20); }
    }
    __syncthreads();
}

// The loops over the block's NT / 32 warp totals below run rolled (little code) or, with KC = 1 (the post kernel's config-3
// instantiation, whose step path is short), unrolled with every shared-memory load in flight: the same adds in the same order.
// exclusive prefix over the block's threads (thread order) of a double, ONE block barrier (sm: this round's scratch)
template <int NT, int KC = 0>
__device__ __forceinline__ double fs3_scan_d(double x, double* sm) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double inc = x;
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) { const double y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc = y + inc; }
    double ex = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) ex = 0.0;
    if (lane == 31) sm[wid] = inc;
    __syncthreads();
    double woff = 0.0;
    if constexpr (KC == 1) {
#pragma unroll
        for (int w = 0; w < NT / 32 - 1; ++w) if (w < wid) woff += sm[w];
    } else {
#pragma unroll 1
        for (int w = 0; w < wid; ++w) woff += sm[w];
    }
    return woff + ex;
}
// the same for a (u64 increment sum, int count) pair; also returns the block totals
template <int NT, int KC = 0>
__device__ __forceinline__ void fs3_scan_ui(unsigned long long p, int c, unsigned long long* pex, int* cex, unsigned long long* ptot, int* ctot,
                                            unsigned long long* smu, int* smi) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    unsigned long long ip = p; int ic = c;
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, ip, o); const int z = __shfl_up_sync(0xffffffffu, ic, o);
        if (lane >= o) { ip += y; ic += z; }
    }
    if (lane == 31) { smu[wid] = ip; smi[wid] = ic; }
    __syncthreads();
    unsigned long long wp = 0, tp = 0; int wc = 0, tc = 0;
    if constexpr (KC == 1) {
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) { const unsigned long long a = smu[w]; const int b = smi[w]; if (w < wid) { wp += a; wc += b; } tp += a; tc += b; }
    } else {
#pragma unroll 1
        for (int w = 0; w < NT / 32; ++w) { const unsigned long long a = smu[w]; const int b = smi[w]; if (w < wid) { wp += a; wc += b; } tp += a; tc += b; }
    }
    *pex = wp + ip - p; *cex = wc + ic - c; *ptot = tp; *ctot = tc;
}
__device__ __forceinline__ double fs3_warp_sum(double v) {
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// block sums of two doubles at once (tree order, identical in every CTA; valid in all threads); ONE block barrier
template <int NT, int KC = 0>
__device__ __forceinline__ void fs3_block_sum2(double& x, double& y, double* smx, double* smy) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    x = fs3_warp_sum(x); y = fs3_warp_sum(y);
    if (lane == 0) { smx[wid] = x; smy[wid] = y; }
    __syncthreads();
    double a = 0.0, b = 0.0;
    if constexpr (KC == 1) {
#pragma unroll
        for (int w = 0; w < NT / 32; ++w) { a += smx[w]; b += smy[w]; }
    } else {
#pragma unroll 1
        for (int w = 0; w < NT / 32; ++w) { a += smx[w]; b += smy[w]; }
    }
    x = a; y = b;
}

__device__ __noinline__ double fs3_div(double a, double b) { return a / b; }      // one copy of the IEEE division sequence for the rare paths
// value i of the sum `slot`, recomputed from global memory (serial walks only)
__device__ __forceinline__ double fs3_value(const Fs3Sum& x, int slot, size_t i, int par, double S2, double r0, double inv) {
    if (slot == FS3_S) return __ldcg(x.raw[par] + i);
    const double w = slot == FS3_COMB ? 0.0 : __ldcg(x.wn + i);
    if (slot == FS3_Q) return w * w;
    if (slot == FS3_S2) return w;
    if (slot == FS3_CDF) return S2 > 0.0 ? fs3_div(w, S2) : w;
    return i == 0 ? r0 : inv;
}
// exact by construction: one thread walks all values in order (bad values, too many dirty ones, failed certificate).
// The CDF (slot 3) is stored as its running maximum, NaN sticky: on a CDF that goes down (negative weights) or turns NaN the
// lower bound of r in it is the reference's index, the first j with !(c_j < r) (fs1.rs:224-226 carries j over slots with
// non-decreasing r); on a non-decreasing CDF it is the CDF itself.
__device__ __forceinline__ double fs3_runmax(double m, double c) { return (m != m || c <= m) ? m : c; }
template <int NT, bool GT = false>
__device__ __noinline__ void fs3_serial_walk(const Fs3Sum& x, Fs3Sh<NT>& sh, unsigned K, int slot, double* out, int par, double S2, double r0, double inv) {
    if (threadIdx.x == 0) {
        const size_t T = (size_t)NT * K, lo = (size_t)blockIdx.x * T;
        double s = 0.0, mx = -INFINITY, mbase = -INFINITY;
        sh.tbase = 0.0;
#pragma unroll 1
        for (size_t i = 0; i < x.n; ++i) {
            if (i == lo) { sh.tbase = s; mbase = mx; }
            s = s + fs3_value(x, slot, i, par, S2, r0, inv);
            if (slot == FS3_CDF) mx = fs3_runmax(mx, s);
        }
        if (lo >= x.n) sh.tbase = s;
        sh.total = s;
        if (blockIdx.x == 0) x.st->serial_walks += 1;
        if (out) {
            double c = sh.tbase, m = mbase;
#pragma unroll 1
            for (size_t i = lo; i < lo + T && i < x.n; ++i) {
                c = c + fs3_value(x, slot, i, par, S2, r0, inv);
                if (slot == FS3_CDF) { m = fs3_runmax(m, c); out[i] = m; } else out[i] = c;
            }
            if (slot == FS3_CDF) x.tileEnd[blockIdx.x] = m;
        }
    }
    __syncthreads();
}

__device__ __noinline__ int fs3_classify(double v, double a0, double a1, unsigned m32, unsigned long long* inc, int* lvl) {
    return x3_classify(v, a0, a1, m32, inc, lvl);            // one copy of the code for the three passes of fs3_xsum
}
// Work that hides inside an exact sum, on warps that would otherwise sleep at a block barrier while warp 0 waits for the grid
// and evaluates the chain.  First sum of fs3_post_kernel: the lazy-clone bookkeeping of every CTA's landmark slice, the comb table
// and the N(0,1) pairs of the next predict (EKF call step + 1), on the Fs3Dev whose d.x the sum runs in, found by its address (a
// pointer to it in the hook costs fs3_post_kernel<512, true> 32 bytes of spills and pf3_post_kernel four registers).
struct Fs3Hook { unsigned long long comb_n; uint64_t seed; unsigned step; int k_last; const Fs3ObsParam* po; };
static_assert(std::is_standard_layout<Fs3Dev>::value, "fs3_xsum's hook finds the Fs3Dev around d.x with offsetof");
// what fs3_xsum_emit needs of a thread's pass through fs3_xsum: approximate prefix in front of its first value, clean-increment
// sum in front of it inside the tile, and the binade of its run (-1: classified value by value)
struct Fs3Run { double a_first; unsigned long long Pex; int e_run; };
// the certificate of a CDF emitted as fl(P_j / S) (DESIGN §1): comb r0 + t inv, t < n = 2^p; dl, ab: relative and absolute bound
struct Fs3Cert { double S, r0, inv, ninv, dl, ab; unsigned long long n; };

// Landmarks [lo, hi) belong to post-kernel CTA b: it applies their marks, records their rows and retargets them at a resample.
__device__ __forceinline__ void fs3_lm_slice(const Fs3Dev& d, unsigned b, unsigned nt, unsigned* lo, unsigned* hi) {
    const unsigned per = (d.m + nt - 1) / nt;
    *lo = min(d.m, b * per); *hi = min(d.m, *lo + per);
}
// Threads 32 .. NT-1 of CTA b.  (1) The lazy-clone bookkeeping of the EKF launch that just ran, for this CTA's landmarks: those it
// updated through a row now live in own columns of the other buffer.  (2) One bit per row some landmark of the slice still reads
// through, OR-ed into the live-row bitmap of this step's parity, and this CTA's "has an identity landmark" flag.  (3) This CTA's
// share of the OTHER parity's bitmap and its flag are zeroed for the next step (nobody reads them in this launch).
// Thread h owns landmarks lo + h, lo + h + NH, ...; it applies the marks of its own landmarks, so it reads back its own stores.
template <int NT>
__device__ __forceinline__ void fs3_row_scan(const Fs3Dev& d, const Fs3ObsParam& po, int k_last, int par, unsigned b, unsigned nt) {
    constexpr unsigned NH = NT - 32;
    const unsigned h = threadIdx.x - 32u, lane = threadIdx.x & 31u;
    const unsigned W = fs3_bm_words(d.m), ldb = fs3_bm_ld(d.m);
    unsigned* bm = d.rowbm + (size_t)par * ldb;
    unsigned* bmo = d.rowbm + (size_t)(par ^ 1) * ldb;
    unsigned lo, hi;
    fs3_lm_slice(d, b, nt, &lo, &hi);
#pragma unroll 1
    for (int j = 0; j < k_last; ++j) {
        const unsigned l = (unsigned)po.o[j].lm_id;
        if (l >= lo && l < hi && (l - lo) % NH == h) { const int s = d.lmst[l]; if (s >> 1) d.lmst[l] = (s & 1) ^ 1; }
    }
    {
        const unsigned wper = (W + nt - 1) / nt, w0 = min(W, b * wper), w1 = min(W, w0 + wper);
#pragma unroll 1
        for (unsigned w = w0 + h; w < w1; w += NH) bmo[w] = 0u;
        if (h == 0) bmo[W + b] = 0u;
    }
    // consecutive landmarks mostly share a row: a thread ORs its bits per bitmap word and stores a word only when it changes,
    // and a warp whose lanes all ended on the same word stores it once
    unsigned cw = 0xFFFFFFFFu, acc = 0u;
    int ident = 0;
#pragma unroll 4
    for (unsigned l = lo + h; l < hi; l += NH) {
        const int s = d.lmst[l];
        if (s >> 1) {
            const unsigned r = (unsigned)((s >> 1) - 1), w = r >> 5;
            if (w != cw) { if (acc) atomicOr(bm + cw, acc); cw = w; acc = 0u; }
            acc |= 1u << (r & 31u);
        } else ident = 1;
    }
    const unsigned has = __ballot_sync(0xffffffffu, acc != 0u);
    if (has) {
        const unsigned src = (unsigned)__ffs(has) - 1u;
        const unsigned wl = __shfl_sync(0xffffffffu, cw, src);
        if (__all_sync(0xffffffffu, acc == 0u || cw == wl)) {
            const unsigned all = __reduce_or_sync(0xffffffffu, acc);
            if (lane == src) atomicOr(bm + wl, all);
        } else if (acc) atomicOr(bm + cw, acc);
    }
    if (__any_sync(0xffffffffu, ident) && lane == 0) bm[W + b] = 1u;
}
// Every thread of a CTA, on a resample step, behind a grid barrier that follows every CTA's fs3_row_scan of this step: the live
// rows of the bitmap in ascending order.  Thread t owns bitmap words [t per, t per + per) (per <= 8: m <= 65 536, NT >= 256).
// fs3_row_count: *pos = the position of the thread's first live row in that order, *nrows = how many rows are live, *newrow = the
// row the identity landmarks get (the first free id: with an identity landmark at most m - 1 rows are live) or -1 when there is
// none.  Contains one block barrier.
template <int NT, int KC = 0>
__device__ __forceinline__ void fs3_row_count(const Fs3Dev& d, Fs3Sh<NT>& sh, int par, unsigned nt, unsigned* pos, int* nrows, int* newrow) {
    const unsigned tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const unsigned W = fs3_bm_words(d.m);
    const unsigned* bm = d.rowbm + (size_t)par * fs3_bm_ld(d.m);
    const unsigned per = (W + NT - 1) / NT, w0 = min(W, tid * per), w1 = min(W, w0 + per);
    unsigned x[8];                                             // every load in flight before the first use
#pragma unroll
    for (unsigned i = 0; i < 8; ++i) x[i] = w0 + i < w1 ? __ldcg(bm + w0 + i) : 0xFFFFFFFFu;
    int any = 0;
    if (wid == 0) {
#pragma unroll
        for (unsigned i = 0; i < (FS3_MAX_TILES + 31) / 32; ++i) { const unsigned t = lane + 32u * i; if (t < nt) any |= __ldcg(bm + W + t) != 0u ? 1 : 0; }
    }
    int cnt = 0;
    unsigned ff = 0xFFFFFFFFu;                                 // first free row id among my words
#pragma unroll
    for (unsigned i = 0; i < 8; ++i) {
        if (w0 + i < w1) { cnt += __popc(x[i]); if (ff == 0xFFFFFFFFu && ~x[i]) ff = (w0 + i) * 32u + (unsigned)__ffs(~x[i]) - 1u; }
    }
    int incl = cnt;
#pragma unroll 1
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, incl, o); if ((int)lane >= o) incl += y; }
    const unsigned wff = __reduce_min_sync(0xffffffffu, ff);
    if (lane == 31) { sh.rowscan[0][wid] = (unsigned)incl; sh.rowscan[1][wid] = wff; }
    if (wid == 0) { any = __any_sync(0xffffffffu, any); if (lane == 0) sh.rany = any; }
    __syncthreads();
    unsigned p = (unsigned)(incl - cnt), tot = 0, mf = 0xFFFFFFFFu;
    if constexpr (KC == 1) {
#pragma unroll
        for (unsigned v = 0; v < NT / 32; ++v) { const unsigned c = sh.rowscan[0][v]; if (v < wid) p += c; tot += c; mf = min(mf, sh.rowscan[1][v]); }
    } else {
#pragma unroll 1
        for (unsigned v = 0; v < NT / 32; ++v) { const unsigned c = sh.rowscan[0][v]; if (v < wid) p += c; tot += c; mf = min(mf, sh.rowscan[1][v]); }
    }
    *pos = p; *nrows = (int)tot; *newrow = sh.rany ? (int)mf : -1;
}
// the live rows at positions [base, base + FS3_ROW_CHUNK) of the ascending order into sh.rowl (pos from fs3_row_count); the caller
// synchronises before sh.rowl is read
template <int NT>
__device__ __forceinline__ void fs3_row_fill(const Fs3Dev& d, Fs3Sh<NT>& sh, int par, unsigned base, unsigned pos) {
    const unsigned tid = threadIdx.x;
    const unsigned W = fs3_bm_words(d.m);
    const unsigned* bm = d.rowbm + (size_t)par * fs3_bm_ld(d.m);
    const unsigned per = (W + NT - 1) / NT, w0 = min(W, tid * per), w1 = min(W, w0 + per);
    unsigned p = pos;
#pragma unroll 1
    for (unsigned w = w0; w < w1 && p < base + FS3_ROW_CHUNK; ++w)
        for (unsigned x = __ldcg(bm + w); x; x &= x - 1, ++p)
            if (p >= base && p < base + FS3_ROW_CHUNK) sh.rowl[p - base] = (unsigned short)(w * 32u + (unsigned)__ffs(x) - 1u);
}

// The chain of an exact sum over more than 32 dirty values (rare), by warp 0 of the leader CTA behind sh.tPoff: the entries
// ranked by index into shared memory, the serial walk by lane 0 (its total is returned there), the certificates in parallel.
// Any failure sets *fail.  Out of line, so that the usual chain stays one straight run of code.
template <int NT>
__device__ __noinline__ double fs3_chain_wide(const Fs3Sum& x, Fs3Sh<NT>& sh, size_t eb, int D, unsigned long long Ptot, int* fail) {
    const int lane = threadIdx.x & 31;
    double total = 0.0;
#pragma unroll 1
    for (int e = lane; e < D; e += 32) sh.ukey[e] = __ldcg(x.entKey + eb + e);
    __syncwarp();
#pragma unroll 1
    for (int e = lane; e < D; e += 32) {               // rank = position in index order (keys are distinct)
        const unsigned key = sh.ukey[e];
        int rank = 0;
#pragma unroll 1
        for (int j = 0; j < D; ++j) rank += sh.ukey[j] < key ? 1 : 0;
        sh.skey[rank] = key; sh.sP[rank] = sh.tPoff[__ldcg(x.entTile + eb + e)] + __ldcg(x.entP + eb + e);
        sh.sV[rank] = __ldcg(x.entV + eb + e); sh.sL[rank] = __ldcg(x.entL + eb + e);
    }
    __syncwarp();
    if (lane == 0) {                                   // the serial part: one integer add + one FP add per dirty value
        double sq = 0.0; unsigned long long prev = 0;
#pragma unroll 1
        for (int o = 0; o < D; ++o) {
            const unsigned long long p = sh.sP[o];
            sh.bef[o] = sq;
            sq = pfc_u2d(pfc_d2u(sq) + (p - prev)) + sh.sV[o];
            sh.aft[o] = sq; prev = p;
        }
        int ok = 1;
        total = x3_apply(sq, Ptot - prev, -1, &ok);
        if (!ok) *fail = 1;
    }
    __syncwarp();
#pragma unroll 1
    for (int o = lane; o < D; o += 32) {               // certificates of the clean runs, in parallel
        const unsigned long long dp = sh.sP[o] - (o ? sh.sP[o - 1] : 0ull);
        int ok = 1;
        (void)x3_apply(sh.bef[o], dp, sh.sL[o], &ok);
        if (!ok) *fail = 1;
    }
    return total;
}

// One exact sequential sum over the n_glob values held tile-wise in shared memory (thread t owns values t*K .. t*K+K-1 of its
// tile, stored at vals[k*NT + t]).  toff = approximate sum of everything in front of this tile.  Returns the exact total
// (identical in every CTA).  pub = 1: the chain's leader also publishes the tile prefixes and the sorted dirty values, and *run
// keeps this thread's state, so that fs3_xsum_emit can store the exact inclusive prefixes afterwards (sh.fail = 0; with
// sh.fail = 1 the serial walk has already stored them to `out`).  Contains ONE grid barrier (`round`).
// fs3_xsum_body is the sum inlined where it is on every step's path (the post kernel's S sum); fs3_xsum is its one out-of-line
// copy for every other sum.
template <int NT, bool GT = false, int KC = 0>
__device__ __forceinline__ double fs3_xsum_body(const Fs3Sum& x, Fs3Sh<NT>& sh, const double* vals, unsigned K, unsigned nt, double toff, int slot, int round,
                                                unsigned m32, double* out, int par, double S2, double r0, double inv, double extraQ, int pub, Fs3Run* run,
                                                const Fs3Hook* hook) {
    const int tid = threadIdx.x, lane = tid & 31, pp = round & 1;
    const unsigned b = blockIdx.x;
    const size_t T = (size_t)NT * K;
    unsigned long long t_prev = 0;
    const int tb0 = slot == FS3_S ? 8 : (slot == FS3_CDF ? 12 : 24);   // trace slots (PFGPU_POST_TRACE): S -> 8..11, CDF -> 12..15
    if (x.trace && b == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_prev));
    // ---- approximate prefixes, classification, tile aggregate ----
    double ts = 0.0; bool bad = false;
#pragma unroll 1
    for (unsigned k = 0; k < K; ++k) { const double v = vals[k * NT + tid]; ts += v; if (!(v >= 0.0) || !(v <= 1.7976931348623157e308)) bad = true; }
    if (slot == FS3_S) FS3_TRACE(28);
    const double a_first = toff + fs3_scan_d<NT, KC>(ts, sh.wd[pp]);
    if (slot == FS3_S) FS3_TRACE(29);
    unsigned long long P = 0; int nd = 0;
    // Almost every thread's K prefixes stay inside one binade, clear of its edges: then each value is classified at that binade
    // without a running prefix (no loop-carried FP chain, a dozen integer instructions per value).  The same predicate, from the
    // same operands, selects the path in the three passes below.
    const int e_run = x3_interior(a_first, a_first + ts, m32);
    if (e_run >= 0) {
#pragma unroll 2
        for (unsigned k = 0; k < K; ++k) {
            unsigned long long inc;
            if (x3_classify_at(vals[k * NT + tid], e_run, &inc)) nd++; else P += inc;
        }
    } else {
        double a = a_first;
#pragma unroll 1
        for (unsigned k = 0; k < K; ++k) {
            const double v = vals[k * NT + tid], a1 = a + v;
            unsigned long long inc; int lvl;
            if (fs3_classify(v, a, a1, m32, &inc, &lvl)) nd++; else P += inc;
            a = a1;
        }
    }
    if (slot == FS3_S) FS3_TRACE(30);
    unsigned long long Pex, Ptile; int dex, ndtile;
    fs3_scan_ui<NT, KC>(P, nd, &Pex, &dex, &Ptile, &ndtile, sh.wu[pp], sh.wi[pp]);
    if (nd > 0) {                                              // rare: itemise this thread's dirty values (any order; sorted by the chain)
        const unsigned e0 = atomicAdd(x.entCnt + slot, (unsigned)nd);
        double a = a_first; unsigned long long Pr = Pex; unsigned e = e0;
    #pragma unroll 1
    for (unsigned k = 0; k < K; ++k) {
            const double v = vals[k * NT + tid], a1 = a + v;
            unsigned long long inc; int lvl = e_run;
            if (e_run >= 0 ? x3_classify_at(v, e_run, &inc) : fs3_classify(v, a, a1, m32, &inc, &lvl)) {
                if (e < FS3_ENT_CAP) {
                    const size_t o = (size_t)slot * FS3_ENT_CAP + e;
                    x.entKey[o] = (unsigned)((size_t)b * T + (size_t)tid * K + k); x.entTile[o] = b; x.entP[o] = Pr; x.entV[o] = v; x.entL[o] = lvl;
                }
                e++;
            } else Pr += inc;
            a = a1;
        }
    }
    if (bad) x.flagsg[slot] = 1;
    if (tid == 0) { x.tileP[(size_t)slot * FS3_MAX_TILES + b] = Ptile; if (slot == FS3_S) x.tileQ[b] = extraQ; }
    FS3_TRACE(tb0);
    __syncthreads();
    // ---- grid barrier + chain.  The LAST CTA to arrive evaluates the chain (every aggregate is published by then and it reads
    // them uncontended: 128 CTAs fetching the same few sectors at once serialise in L2) and publishes the results; the others
    // wait for its flag.  Warp 0 only; the other warps wait at the block barrier below. ----
    if (hook && tid >= 32) {
        const Fs3Dev& d = *reinterpret_cast<const Fs3Dev*>(reinterpret_cast<const char*>(&x) - offsetof(Fs3Dev, x));
        fs3_row_scan<NT>(d, *hook->po, hook->k_last, (int)(hook->step & 1u), b, nt);
        if (tid < 64) {                            // warp 1
            if (hook->comb_n && lane == 0) x3_comb_build(&sh.comb, r0, inv, (double)hook->comb_n, hook->comb_n);
        } else {                                   // warps 2..: the N(0,1) pairs of the next predict for this CTA's share of the local slots
            const unsigned per = (d.n + nt - 1) / nt, t_lo = b * per, t_hi = min(d.n, t_lo + per);
#pragma unroll 1
            for (unsigned t = t_lo + (unsigned)(tid - 64); t < t_hi; t += (unsigned)(NT - 64)) {
                double z0, z1;
                fs3_normal_pair(hook->seed, hook->step + 1u, (uint64_t)d.off + t, &z0, &z1);
                d.nz[0][t] = z0; d.nz[1][t] = z1;
            }
        }
    }
    if (tid < 32) {
        int leader = 0;
        if (tid == 0) leader = (atom_add_acq_rel_gpu(x.bar + round, 1u) + 1u == nt) ? 1 : 0;
        leader = __shfl_sync(0xffffffffu, leader, 0);
        Fs3Res* res = x.res + round;
        const size_t rb = (size_t)round * FS3_ENT_CAP, rt = (size_t)round * FS3_MAX_TILES;
        if (leader) {
            FS3_TRACE(tb0 + 1);
            // ONE round trip: every load the chain needs is issued before the first use (tile sums, entry count, and — speculatively,
            // their count is not known yet — the first 32 appended entries)
            const size_t eb = (size_t)slot * FS3_ENT_CAP;
            unsigned long long tp[(FS3_MAX_TILES + 31) / 32];
#pragma unroll
            for (unsigned i = 0; i < (FS3_MAX_TILES + 31) / 32; ++i) tp[i] = (i * 32u + lane) < nt ? __ldcg(x.tileP + (size_t)slot * FS3_MAX_TILES + i * 32u + lane) : 0ull;
            const unsigned cnt = __ldcg(x.entCnt + slot);
            int fail = __ldcg(x.flagsg + slot);
            unsigned ekey = __ldcg(x.entKey + eb + lane), etile = __ldcg(x.entTile + eb + lane);
            unsigned long long eP = __ldcg(x.entP + eb + lane);
            double eV = __ldcg(x.entV + eb + lane);
            int eL = __ldcg(x.entL + eb + lane);
            fail |= cnt > FS3_ENT_CAP ? 1 : 0;
#pragma unroll
            for (unsigned i = 0; i < (FS3_MAX_TILES + 31) / 32; ++i) if (i * 32u + lane < nt) sh.tPoff[i * 32u + lane] = tp[i];
            __syncwarp();
            if (slot == FS3_S) FS3_TRACE(16);
            // clean-increment sum in front of every tile: lane owns `per` consecutive tiles
            const unsigned per = (nt + 31u) / 32u, t0 = (unsigned)lane * per;
            unsigned long long lsum = 0;
#pragma unroll 1
            for (unsigned i = 0; i < per; ++i) if (t0 + i < nt) lsum += sh.tPoff[t0 + i];
            unsigned long long inc = lsum;
#pragma unroll 1
            for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
            const unsigned long long Ptot = __shfl_sync(0xffffffffu, inc, 31);
            unsigned long long run = inc - lsum;
#pragma unroll 1
            for (unsigned i = 0; i < per; ++i) if (t0 + i < nt) { const unsigned long long tp = sh.tPoff[t0 + i]; sh.tPoff[t0 + i] = run; run += tp; }
            __syncwarp();
            if (slot == FS3_S) FS3_TRACE(17);
            const int D = fail ? 0 : (int)cnt;
            double total = 0.0;
            if (D <= 32) {
                // ---- the usual case: lane e holds entry e (loaded speculatively above); rank by index with shuffles, move every entry
                // to its rank in shared memory, then the serial walk ----
                const bool have = lane < D;
                if (!have) ekey = 0xFFFFFFFFu;
                const unsigned long long Pg = have ? sh.tPoff[etile < nt ? etile : 0] + eP : 0ull;
                int rank = 0;
#pragma unroll 4
                for (int j = 0; j < 32; ++j) rank += __shfl_sync(0xffffffffu, ekey, j) < ekey ? 1 : 0;
                // move every entry to the lane of its rank (through shared memory: one conflict-free round)
                if (have) { sh.skey[rank] = ekey; sh.sP[rank] = Pg; sh.sV[rank] = eV; sh.sL[rank] = eL; }
                __syncwarp();
                if (slot == FS3_S) FS3_TRACE(18);
                // the serial part, lane 0 over the sorted entries in shared memory: one integer add on the bit pattern + one FP add
                // per dirty value; the loads do not depend on the chain, so the compiler hoists them ahead (unroll 4)
                int ok = 1;
                if (lane == 0) {
                    double sq = 0.0; unsigned long long prev = 0;
#pragma unroll 4
                    for (int o = 0; o < D; ++o) {
                        const unsigned long long p = sh.sP[o]; const double v = sh.sV[o];
                        sh.bef[o] = sq;
                        sq = pfc_u2d(pfc_d2u(sq) + (p - prev)) + v;
                        sh.aft[o] = sq; prev = p;
                    }
                    total = x3_apply(sq, Ptot - prev, -1, &ok);
                }
                __syncwarp();
                if (have) {                                        // certificate of the clean run in front of my entry, in parallel
                    const unsigned long long dp = sh.sP[lane] - (lane ? sh.sP[lane - 1] : 0ull);
                    (void)x3_apply(sh.bef[lane], dp, sh.sL[lane], &ok);
                }
                if (!ok) fail = 1;
            } else {
                total = fs3_chain_wide<NT>(x, sh, eb, D, Ptot, &fail);
            }
            __syncwarp();
            fail = __any_sync(0xffffffffu, fail);
            total = __shfl_sync(0xffffffffu, total, 0);
            if (slot == FS3_S) FS3_TRACE(19);
            // publish: what the other CTAs need to finish on their own
            if (pub && !fail) {
#pragma unroll 1
                for (unsigned t = lane; t < nt; t += 32) x.resTP[rt + t] = sh.tPoff[t];
#pragma unroll 1
                for (int o = lane; o < D; o += 32) { x.resKey[rb + o] = sh.skey[o]; x.resP[rb + o] = sh.sP[o]; x.resAft[rb + o] = sh.aft[o]; }
            }
            if (lane == 0) {
                res->total = total; res->Ptot = Ptot; res->D = D; res->fail = fail;
                sh.total = total; sh.Ptot = Ptot; sh.D = D; sh.fail = fail; sh.lead = 1;
                x.st->dirty_last = (int)cnt;
            }
            __syncwarp();                                          // the other lanes' stores above are ordered before lane 0's release
            if (lane == 0) st_release_gpu(x.resflag + round, 1u);
            if (slot == FS3_S) { FS3_TRACE(20); if (x.trace && b == 0 && tid == 0) x.trace[21] += 1; }
        } else {
            if (lane == 0) {
                unsigned spins = 0;
                while (ld_acquire_gpu(x.resflag + round) == 0u) { if (++spins > FS3_SPIN_LIMIT) { x.st->err = 1; break; } __nanosleep(20); }
            }
            __syncwarp();
            FS3_TRACE(tb0 + 1);
            const double total = __ldcg(&res->total);
            const int D = __ldcg(&res->D), fail = __ldcg(&res->fail);
            if (lane == 0) { sh.total = total; sh.D = D; sh.fail = fail; sh.lead = 0; }
        }
    }
    __syncthreads();
    FS3_TRACE(tb0 + 2);
    if (sh.fail) { fs3_serial_walk<NT, GT>(x, sh, K, slot, out, par, S2, r0, inv); return sh.total; }
    if (run) { run->a_first = a_first; run->Pex = Pex; run->e_run = e_run; }
    return sh.total;
}
template <int NT, bool GT = false>
__device__ __noinline__ double fs3_xsum(const Fs3Sum& x, Fs3Sh<NT>& sh, const double* vals, unsigned K, unsigned nt, double toff, int slot, int round,
                                        unsigned m32, double* out, int par, double S2, double r0, double inv, double extraQ, int pub, Fs3Run* run) {
    return fs3_xsum_body<NT, GT>(x, sh, vals, K, nt, toff, slot, round, m32, out, par, S2, r0, inv, extraQ, pub, run, nullptr);
}

// The exact inclusive prefix c_j of every value of this tile after fs3_xsum(pub = 1) of round `round` (nothing when that sum took
// the serial walk: it has stored them already).  cert == nullptr: c_j goes to out[j].  Otherwise fl(c_j / cert->S) goes to
// out[j], and the return value is 1 when some comb value may lie on the other side of it than of the CDF the reference computes
// (x3_cdf_near_comb), or a clean run failed its certificate.  tend: the tile's last stored value goes to tileEnd[tile].
// vals must still hold the values the sum saw.  Contains one block barrier.  Inlined as fs3_xsum_emit_body where it is on the
// path of a config-3 resample (the certified CDF); fs3_xsum_emit is the out-of-line copy for the exact CDF and comb.
template <int NT, bool GT = false>
__device__ __forceinline__ int fs3_xsum_emit_body(const Fs3Sum& x, Fs3Sh<NT>& sh, const double* vals, unsigned K, unsigned m32, const Fs3Run* run, int round,
                                                  double* out, int tend, const Fs3Cert* cert, int tslot) {
    const int tid = threadIdx.x, lane = tid & 31;
    const unsigned b = blockIdx.x;
    const size_t T = (size_t)NT * K;
    unsigned long long t_prev = 0;
    if (x.trace && b == 0 && tid == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_prev));
    if (sh.fail) return 0;
    if (tid < 32 && !sh.lead) {                               // the sorted dirty entries + my tile's increment prefix, as the leader published them
        const size_t rb = (size_t)round * FS3_ENT_CAP, rt = (size_t)round * FS3_MAX_TILES;
        if (lane == 0) sh.tPoff[b] = __ldcg(x.resTP + rt + b);
#pragma unroll 1
        for (int o = lane; o < sh.D; o += 32) { sh.skey[o] = __ldcg(x.resKey + rb + o); sh.sP[o] = __ldcg(x.resP + rb + o); sh.aft[o] = __ldcg(x.resAft + rb + o); }
    }
    __syncthreads();
    const int D = sh.D, e_run = run->e_run;
    const size_t g0 = (size_t)b * T + (size_t)tid * K;
    int ko = 0;                                                // dirty values in front of this thread's first value
    {
        int lo = 0, hi = D;
#pragma unroll 1
        while (lo < hi) { const int mid = (lo + hi) >> 1; if ((size_t)sh.skey[mid] < g0) lo = mid + 1; else hi = mid; }
        ko = lo;
    }
    double base = ko ? sh.aft[ko - 1] : 0.0;
    unsigned long long Pb = ko ? sh.sP[ko - 1] : 0ull, Pc = sh.tPoff[b] + run->Pex;
    double a = run->a_first, c = base, o = base;
    int ok = 1, near = 0;
    if (e_run >= 0 && !cert) {                                 // the usual exact emission: the whole run inside one binade
#pragma unroll 2
        for (unsigned k = 0; k < K; ++k) {
            unsigned long long inc;
            if (x3_classify_at(vals[k * NT + tid], e_run, &inc)) { base = sh.aft[ko]; Pb = sh.sP[ko]; ko++; c = base; }
            else { Pc += inc; c = x3_apply(base, Pc - Pb, inc ? e_run : -1, &ok); }
            if (g0 + k < x.n) out[g0 + k] = c;
        }
        o = c;
    } else {
#pragma unroll 1
        for (unsigned k = 0; k < K; ++k) {
            const double v = vals[k * NT + tid], a1 = a + v;
            unsigned long long inc; int lvl = e_run;
            if (e_run >= 0 ? x3_classify_at(v, e_run, &inc) : fs3_classify(v, a, a1, m32, &inc, &lvl)) { base = sh.aft[ko]; Pb = sh.sP[ko]; ko++; c = base; }
            else { Pc += inc; c = x3_apply(base, Pc - Pb, inc ? lvl : -1, &ok); }
            o = c;
            if (cert) {
                o = c / cert->S;
                if (g0 + k < x.n) near |= x3_cdf_near_comb(o, cert->r0, cert->inv, cert->ninv, cert->n, cert->dl, cert->ab);
            }
            if (g0 + k < x.n) out[g0 + k] = o;
            a = a1;
        }
    }
    if (tend && tid == NT - 1) x.tileEnd[b] = o;              // coarse level of the index search
    if (!ok) { atomicAdd(&x.st->cert_fail, 1); near = 1; }
    if (tslot >= 0) FS3_TRACE(tslot);
    return near;
}
template <int NT, bool GT = false>
__device__ __noinline__ int fs3_xsum_emit(const Fs3Sum& x, Fs3Sh<NT>& sh, const double* vals, unsigned K, unsigned m32, const Fs3Run* run, int round,
                                          double* out, int tend, const Fs3Cert* cert, int tslot) {
    return fs3_xsum_emit_body<NT, GT>(x, sh, vals, K, m32, run, round, out, tend, cert, tslot);
}

// warp-cooperative 32-way search of one r over c[0 .. n): returns the lower bound (all lanes)
__device__ __forceinline__ unsigned fs3_warp_search(const double* c, unsigned n, double r) {
    const int lane = threadIdx.x & 31;
    unsigned lo = 0, hi = n;                                  // answer in [lo, hi]
#pragma unroll 1
    while (hi - lo > 32) {
        const unsigned step = (hi - lo + 32) / 33;            // probes lo + (lane+1)*step - 1
        const unsigned long long pi = (unsigned long long)lo + (unsigned long long)(lane + 1) * step - 1ull;
        const bool below = pi < hi ? (__ldcg(c + pi) < r) : false;     // monotone: a prefix of lanes is "below"
        const int cnt = __popc(__ballot_sync(0xffffffffu, below));
        const unsigned long long nh = (unsigned long long)lo + (unsigned long long)(cnt + 1) * step - 1ull;
        if (cnt < 32 && nh < hi) hi = (unsigned)nh;           // lane cnt probed c[nh] >= r (with cnt == 32 nobody probed nh)
        if (cnt) lo += (unsigned)cnt * step;
    }
    const unsigned pi = lo + (unsigned)lane;
    const bool below = pi < hi ? (__ldcg(c + pi) < r) : false;
    return lo + (unsigned)__popc(__ballot_sync(0xffffffffu, below));
}
// two-level lower bound of r in the whole CDF (all lanes of a warp): tile from the tiles' last values (shared memory), then inside it
__device__ __forceinline__ unsigned fs3_cdf_search(const double* cdf, const double* tend, unsigned nt, unsigned T, unsigned ng, double r) {
    unsigned lo = 0, hi = nt;
#pragma unroll 1
    while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (tend[mid] < r) lo = mid + 1; else hi = mid; }
    if (lo >= nt) return ng;
    const unsigned base = lo * T, len = min(T, ng - base);
    return base + fs3_warp_search(cdf + base, len, r);
}

// GTILE = false: the tile of K x NT weights lives in dynamic shared memory.  GTILE = true: it lives in this CTA's slice of vtile
// ([tiles][K][NT] doubles of global memory, the same layout: every access stays coalesced), for particle counts whose tile does not
// fit on chip.  A value stored by one thread is read by another only behind a __syncthreads(), which orders global memory inside
// a CTA too.
// The block workspace, one variable for fs3_post_kernel<NT, GTILE, 0> and <NT, GTILE, 1>: the out-of-line routines they share
// (template tag GTILE) then address it directly, as when only one kernel called them, instead of taking it as an argument.
template <int NT, bool GTILE>
__shared__ Fs3Sh<NT> fs3_post_sh;
// KC = 0: K values per thread, K taken at run time.  KC = 1: one value per thread and at most one local slot per thread (config 3:
// 128 tiles x 512 threads x 1), so the loops over a thread's values fold away in the inlined hot-path bodies (the argument K is
// ignored), and the clone phase handles one slot per thread.  The out-of-line rare paths are shared with <NT, GTILE, 0>.
template <int NT, bool GTILE, int KC = 0>
__global__ void __launch_bounds__(NT, 1)
fs3_post_kernel(const __grid_constant__ Fs3Dev d, const __grid_constant__ Fs3ObsParam po, int k_last, double nth, uint64_t seed, unsigned step,
                unsigned K_rt, unsigned m32, int log2n, int early_launch, double* vtile) {
    static_assert(KC == 0 || (KC == 1 && !GTILE), "the one-value kernel keeps its tile in shared memory");
    const unsigned K = KC ? (unsigned)KC : K_rt;
    pf_grid_dep_sync();
    if (early_launch) pf_grid_launch_dependents();
    double* vt;
    { extern __shared__ __align__(16) double vals[]; vt = GTILE ? vtile + (size_t)blockIdx.x * NT * K : vals; }
    double* const vals = vt;                                  // [K][NT]
    Fs3Sh<NT>& sh = fs3_post_sh<NT, GTILE>;
    const Fs3Sum& x = d.x;
    Fs3State* st = d.st;
    const int tid = threadIdx.x;
    const unsigned b = blockIdx.x, nt = gridDim.x;
    const size_t T = (size_t)NT * K, ng = d.n_glob;
    const int par = (int)(step & 1u);
    unsigned long long t_prev = 0;
    if (x.trace && b == 0 && tid == 0) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_prev));
        const unsigned long long e1 = x.trace[37], e0 = x.trace[38];           // step timeline: [33] EKF launch (first CTA in .. last warp out),
        if (e1 && e0) { x.trace[33] += e1 - e0; x.trace[34] += t_prev - e1; }   // [34] idle between the EKF launch and this one
        x.trace[39] = t_prev;
    }
    if (d.G > 1) {      // my EKF launch is complete: its pushes are in every peer's copy.  Say so, then wait for the others'.
        if (b == 0) fs3_signal_peers(d, 0, step + 1u);
        if (d.wait_inline) {
            if (tid == 0) fs3_wait_peers(d, 0, step + 1u);
            __syncthreads();
        }
    }
    // ---- load this tile's weights; approximate sum of everything in front of the tile from the 64-particle partials ----
    const size_t g0 = (size_t)b * T + (size_t)tid * K;
    double q = 0.0;
#pragma unroll 4
    for (unsigned k = 0; k < K; ++k) { const double v = g0 + k < ng ? d.wraw[par][g0 + k] : 0.0; vals[k * NT + tid] = v; q += v * v; }   // (through L1: a thread reads K consecutive doubles)
    double toff = 0.0;
    {
        const unsigned pfirst = (unsigned)(((size_t)b * T) / 64);      // partial p covers global slots [64 p, 64 p + 64)
#pragma unroll 8
        for (unsigned p = tid; p < pfirst; p += NT) toff += __ldcg(d.part[par] + p);
    }
    fs3_block_sum2<NT, KC>(toff, q, sh.red[0], sh.red[1]);
    FS3_TRACE(0);
    // the comb of a resample this step might need: r = Uniform::new(0, 1/n).sample(rng) (fs1.rs:219-220), one draw per resample, and
    // (n a power of two) its closed-form table, built by an otherwise idle warp inside the first exact sum
    const double inv = 1.0 / (double)ng;
    const double r0 = pfc_u01_52(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_FS_RESAMPLE, st->resamples, 0), 0)) * (inv - 0.0) + 0.0;
    // ---------------- S = sum w_raw (normalize_weights fs1.rs:196-203) ----------------
    // With n = 2^p, p <= FS3_CERT_MAX_LOG2N, the leader also publishes what every CTA needs to emit the exact prefixes P_j of w_raw:
    // a resample may then use the certified CDF fl(P_j / S) instead of the S2 and CDF sums (see below)
    const int cert_pub = log2n >= 0 && log2n <= FS3_CERT_MAX_LOG2N && !d.exact_cdf;
    Fs3Hook hook;
    hook.comb_n = log2n >= 0 ? (unsigned long long)ng : 0ull; hook.seed = seed; hook.step = step; hook.k_last = k_last; hook.po = &po;
    Fs3Run run;
    const double S = fs3_xsum_body<NT, GTILE, KC>(x, sh, vals, K, nt, toff, FS3_S, FS3_R_S, m32, nullptr, par, 0.0, r0, inv, q, cert_pub, &run, &hook);
    const int S_walked = sh.fail;
    FS3_TRACE(1);
    // ---------------- gate: neff = 1 / sum w^2 < NTH (compute_neff fs1.rs:186-193, fs1.rs:262-263) ----------------
    // Only the DECISION feeds back into the state.  Q is first taken from the tree-order sums of w_raw^2 published with the
    // aggregates of S: sum (w_raw_i / S)^2 differs from the reference's sequential sum of fl(w_raw_i / S)^2 by at most
    // (n + 64) 2^-51 relatively; only when neff lands that close to NTH is the exact sequential sum walked (below, once wn_all is written).
    double Q = (unsigned)tid < nt ? __ldcg(x.tileQ + tid) : 0.0, dummy = 0.0;
    fs3_block_sum2<NT, KC>(Q, dummy, sh.red[1], sh.wd[1]);
    if (S > 0.0) Q = Q / S / S;
    double neff = Q > 0.0 ? 1.0 / Q : 0.0;
    const double slack = 16.0 * (double)(ng + 64) * 2.220446049250313e-16;
    // The error bound of the shortcut assumes that no w_raw^2 that matters under- or overflows: with S inside [1e-120, 1e120] the
    // squares of all weights within 1e-34 of the largest are normal numbers.  Outside (e.g. an outlier observation that drives
    // EVERY likelihood to 1e-170: the normalised weights are perfectly ordinary, their raw squares are all zero) the exact sum decides.
    const bool scale_ok = !(S > 0.0) || (S >= 1e-120 && S <= 1e120);
    const bool border = !scale_ok || !(fabs(neff - nth) > slack * fmax(fabs(nth), fabs(neff)));     // the same decision in every CTA
    // ---------------- certified CDF (DESIGN §1) ----------------
    // The index rule only COMPARES comb values with CDF values.  On a resample of n = 2^p weights with S > 0 in the window above and
    // no serial walk, every CTA stores c~_j = fl(P_j / S) for its tile to cum_all; |c_j - c~_j| <= dl c~_j + ab for the reference's
    // CDF c_j (normalise, re-normalise by S2, sequential cum_sum).  A CTA that finds a comb value within that distance of one of
    // its c~_j raises the certificate flag, and then every CTA runs the exact S2 and CDF sums behind the next grid barrier.
    const bool cert = cert_pub && !border && neff < nth && S > 0.0 && !S_walked;
    if (cert) {
        Fs3Cert cp;
        const double g = 4.0 * (double)ng * 1.1102230246251565e-16;      // 4 n 2^-53
        cp.S = S; cp.r0 = r0; cp.inv = inv; cp.ninv = (double)ng; cp.n = ng;
        cp.dl = g / (1.0 - g) * (1.0 + 9.5367431640625e-07);             // gamma_4n (1 + 2^-20)
        cp.ab = (4.0 * (double)ng + 4.0) * 4.9406564584124654e-324 + (double)(log2n + 4) * 1.1102230246251565e-16;
        const int near = fs3_xsum_emit_body<NT, GTILE>(x, sh, vals, K, m32, &run, FS3_R_S, d.cum_all, 1, &cp, -1);
        if (__syncthreads_or(near) && tid == 0) x.flagsg[FS3_CERT_FLAG] = 1;
        FS3_TRACE(4);
    }
    // w = w_raw / S; best particle of the tile (LAST maximum, fs1.rs:269-274; from -inf, so weights below -1 take part too)
    double bw = -INFINITY; unsigned bi = 0;
#pragma unroll 1
    for (unsigned k = 0; k < K; ++k) {
        double v = vals[k * NT + tid];
        if (S > 0.0) v = v / S;
        vals[k * NT + tid] = v;
        const size_t i = g0 + k;
        if (i < ng) {
            d.wn_all[i] = v;
            if (i >= d.off && i < (size_t)d.off + d.n) d.w[i - d.off] = v;
            if (v >= bw) { bw = v; bi = (unsigned)i; }
        }
    }
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1) {      // arg-max with "last wins among equals"
        const double ow = __shfl_xor_sync(0xffffffffu, bw, o); const unsigned oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ow > bw || (ow == bw && oi > bi)) { bw = ow; bi = oi; }
    }
    if ((tid & 31) == 0) { sh.red[0][tid >> 5] = bw; sh.wi[0][tid >> 5] = (int)bi; }
    __syncthreads();
    if (tid == 0) {
        if constexpr (KC == 1) {
#pragma unroll
            for (int w = 1; w < NT / 32; ++w) { const double ow = sh.red[0][w]; const unsigned oi = (unsigned)sh.wi[0][w]; if (ow > bw || (ow == bw && oi > bi)) { bw = ow; bi = oi; } }
        } else {
#pragma unroll 1
            for (int w = 1; w < NT / 32; ++w) { const double ow = sh.red[0][w]; const unsigned oi = (unsigned)sh.wi[0][w]; if (ow > bw || (ow == bw && oi > bi)) { bw = ow; bi = oi; } }
        }
        d.tileBw[b] = bw; d.tileBi[b] = bi;
    }
    if (border) {                                              // rare
        fs3_grid_sync<NT>(x, FS3_R_BORDER, nt);                // wn_all is complete
        if (tid == 0) {
            double s = 0.0;
            if constexpr (GTILE) {       // millions of values: sixteen loads in flight per trip, the adds in the same order
                size_t i = 0;
#pragma unroll 1
                for (; i + 16 <= ng; i += 16) {
                    double2 w[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) w[u] = __ldcg(reinterpret_cast<const double2*>(d.wn_all + i) + u);
#pragma unroll
                    for (int u = 0; u < 8; ++u) { s = s + w[u].x * w[u].x; s = s + w[u].y * w[u].y; }
                }
#pragma unroll 1
                for (; i < ng; ++i) { const double w = __ldcg(d.wn_all + i); s = s + w * w; }
            } else {
#pragma unroll 1
                for (size_t i = 0; i < ng; ++i) { const double w = __ldcg(d.wn_all + i); s = s + w * w; }
            }
            sh.bcast = s;
            if (b == 0) st->border_cnt += 1;
        }
        __syncthreads();
        Q = sh.bcast;
        neff = Q > 0.0 ? fs3_div(1.0, Q) : 0.0;
    }
    const int gate = neff < nth ? 1 : 0;
    FS3_TRACE(2);
    double S2 = 0.0;
    if (gate) {
        // this CTA's landmark slice (only this CTA writes it, in the first sum): its first entries are loaded in front of the barrier,
        // so the retarget behind the index walk does not wait for them
        unsigned lm_lo, lm_hi;
        fs3_lm_slice(d, b, nt, &lm_lo, &lm_hi);
        const int s_first = lm_lo + tid < lm_hi ? d.lmst[lm_lo + tid] : 0;
        bool exact = !cert;
        if (cert) {
            fs3_grid_sync<NT>(x, FS3_R_CERT, nt);              // every c~_j and every CTA's verdict are visible
            exact = __ldcg(x.flagsg + FS3_CERT_FLAG) != 0;
            FS3_TRACE(5);
        }
        if (exact) {
            if (b == 0 && tid == 0) st->cdf_exact += 1;
            // ---------------- resample() re-normalises first (fs1.rs:207) ----------------
            const double toff2 = S > 0.0 ? fs3_div(toff, S) : toff;
            S2 = fs3_xsum<NT, GTILE>(x, sh, vals, K, nt, toff2, FS3_S2, FS3_R_S2, m32, nullptr, par, 0.0, 0.0, 0.0, 0.0, 0, nullptr);
            FS3_TRACE(3);
            if (S2 > 0.0) {
#pragma unroll 1
                for (unsigned k = 0; k < K; ++k) vals[k * NT + tid] = fs3_div(vals[k * NT + tid], S2);
            }
            // ---------------- cum_sum fs1.rs:213-216 ----------------
            const double toff3 = S2 > 0.0 ? fs3_div(toff2, S2) : toff2;
            (void)fs3_xsum<NT, GTILE>(x, sh, vals, K, nt, toff3, FS3_CDF, FS3_R_CDF, m32, d.cum_all, par, S2, 0.0, 0.0, 0.0, 1, &run);
            (void)fs3_xsum_emit<NT, GTILE>(x, sh, vals, K, m32, &run, FS3_R_CDF, d.cum_all, 1, nullptr, 15);
            FS3_TRACE(4);
            // ---------------- the comb r, r + 1/n, ... accumulated sequentially (fs1.rs:219-230) ----------------
            if (log2n < 0) {                                   // n not a power of two: every add rounds -> exact scan
#pragma unroll 1
                for (unsigned k = 0; k < K; ++k) { const size_t i = g0 + k; vals[k * NT + tid] = i < ng ? (i == 0 ? r0 : inv) : 0.0; }
                const double toff4 = b == 0 ? 0.0 : r0 + ((double)((size_t)b * T) - 1.0) * inv;
                __syncthreads();
                (void)fs3_xsum<NT, GTILE>(x, sh, vals, K, nt, toff4, FS3_COMB, FS3_R_COMB, m32, d.rcomb_all, par, S2, r0, inv, 0.0, 1, &run);
                (void)fs3_xsum_emit<NT, GTILE>(x, sh, vals, K, m32, &run, FS3_R_COMB, d.rcomb_all, 0, nullptr, -1);
            }
            fs3_grid_sync<NT>(x, FS3_R_CDF_DONE, nt);          // the whole CDF (and comb) is visible
            FS3_TRACE(5);
        }
        // ---------------- index walk, pose clone, lazy map clone for this CTA's share of the local slots ----------------
        // j_t = first j with c_j >= r_t, clamped to n - 1: "while r > cum_sum[j+1] && j < n-1 { j += 1 }" (fs1.rs:224-226) with r and
        // j both non-decreasing over the slots.  The CTA's first and last slot bracket all of its answers; the bracketed piece of
        // the CDF is staged in shared memory (it is about as long as the slot range) and every slot searches there.  The certified
        // CDF is monotone and every comparison with a comb value comes out as with the exact one, so the same search serves both.
        const int cur = st->cur, rcur = st->rcur;
        const unsigned per = (d.n + nt - 1) / nt;              // local slots per CTA
        const unsigned t_lo = b * per, t_hi = min(d.n, t_lo + per);
        const double* cdf = d.cum_all;
#pragma unroll 1
        for (unsigned t = tid; t < nt; t += NT) sh.tend[t] = __ldcg(x.tileEnd + t);
        // the live rows: every CTA's fs3_row_scan (inside the S sum) is ordered before the grid barrier this CTA has just passed
        unsigned rpos; int nrows, newrow;
        fs3_row_count<NT, KC>(d, sh, par, nt, &rpos, &nrows, &newrow);            // (also orders the tileEnd copy)
        if (t_lo < t_hi) {
            if (tid < 64) {
                const size_t te = (size_t)d.off + (tid < 32 ? t_lo : t_hi - 1);
                const double re = log2n >= 0 ? x3_comb_eval(&sh.comb, inv, te) : __ldcg(d.rcomb_all + te);
                const unsigned je = fs3_cdf_search(cdf, sh.tend, nt, (unsigned)T, (unsigned)ng, re);
                if ((tid & 31) == 0) sh.jr[tid >> 5] = je;
            }
        }
        fs3_row_fill<NT>(d, sh, par, 0, rpos);
        __syncthreads();
        if (t_lo < t_hi) {
            FS3_TRACE(22);
            const unsigned jlo = sh.jr[0], jhi = min(sh.jr[1], (unsigned)ng - 1u);        // answers lie in [jlo, jhi] (ng -> clamped)
            const unsigned len = jlo <= jhi ? jhi - jlo + 1u : 0u;
            const bool staged = len <= (unsigned)T;
            if (staged) {
#pragma unroll 4
                for (unsigned i = tid; i < len; i += NT) vals[i] = __ldcg(cdf + jlo + i);
            }
            __syncthreads();
            FS3_TRACE(23);
            unsigned* drows = d.rows[rcur ^ 1];
            if constexpr (KC == 1) {
                // one slot per thread (per <= NT): its search, pose clone and row composition.  The ancestor stays in registers
                // across the row chunks, and the registers the generic kernel spends on four slots hold FS3_K1_ROWS rows of one.
                const unsigned t = t_lo + (unsigned)tid;
                const bool mine = t < t_hi;
                unsigned j = 0;
                if (mine) {
                    const size_t tg = (size_t)d.off + t;
                    const double r = log2n >= 0 ? x3_comb_eval(&sh.comb, inv, tg) : __ldcg(d.rcomb_all + tg);
                    unsigned lo = 0, hi = len;
                    if (staged) {
#pragma unroll 1
                        while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (vals[mid] < r) lo = mid + 1; else hi = mid; }
                    } else {
#pragma unroll 1
                        while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (__ldcg(cdf + jlo + mid) < r) lo = mid + 1; else hi = mid; }
                    }
                    j = jlo + lo;
                    if (j >= ng) j = (unsigned)ng - 1;
                }
                const int jrk = (int)(j / d.n); const unsigned jcol = j % d.n;              // owner rank and column of the ancestor
                {
                    const double* sx = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk] + d.o_px[cur]) : d.px[cur];
                    const double* sy = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk] + d.o_py[cur]) : d.py[cur];
                    const double* sa = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk] + d.o_pyaw[cur]) : d.pyaw[cur];
                    const double gx = sx[jcol], gy = sy[jcol], ga = sa[jcol];
                    if (mine) {
                        d.idx[t] = j;
                        d.px[cur ^ 1][t] = gx; d.py[cur ^ 1][t] = gy; d.pyaw[cur ^ 1][t] = ga;     // particles[j].clone() fs1.rs:227
                        d.w[t] = inv;                                                            // fs1.rs:228
                        if (newrow >= 0) drows[(size_t)newrow * d.ld + t] = fs3_ref(jrk, jcol);
                    }
                }
                const unsigned* srow = (d.G > 1 ? reinterpret_cast<const unsigned*>(d.peer[jrk] + d.o_rows[rcur]) : d.rows[rcur]) + jcol;
#pragma unroll 1
                for (unsigned rbase = 0; ; rbase += FS3_ROW_CHUNK) {
                    const int nr = min(nrows - (int)rbase, FS3_ROW_CHUNK);
                    if (mine) {
#pragma unroll 1
                        for (int x0 = 0; x0 < nr; x0 += FS3_K1_ROWS) {
                            unsigned e[FS3_K1_ROWS];
#pragma unroll
                            for (int i = 0; i < FS3_K1_ROWS; ++i) e[i] = x0 + i < nr ? srow[(size_t)sh.rowl[min(x0 + i, nr - 1)] * d.ld] : 0u;
#pragma unroll
                            for (int i = 0; i < FS3_K1_ROWS; ++i) if (x0 + i < nr) drows[(size_t)sh.rowl[min(x0 + i, nr - 1)] * d.ld + t] = e[i];
                        }
                    }
                    if ((int)(rbase + FS3_ROW_CHUNK) >= nrows) break;
                    __syncthreads();                           // everybody is through this chunk's rows
                    fs3_row_fill<NT>(d, sh, par, rbase + FS3_ROW_CHUNK, rpos);
                    __syncthreads();
                }
            } else {
                // rows in chunks of FS3_ROW_CHUNK (one chunk but for very large maps); the first chunk's pass also searches the slots and
                // clones the poses, later passes take the ancestors from idx (this thread's own stores)
#pragma unroll 1
                for (unsigned rbase = 0; ; rbase += FS3_ROW_CHUNK) {
                    const int nr = min(nrows - (int)rbase, FS3_ROW_CHUNK);
                    // four slots per thread and trip: their searches, pose gathers and row gathers are independent, so the dependent memory
                    // round trips (index -> ancestor's pose -> ancestor's row entries) overlap four-fold
#pragma unroll 1
                    for (unsigned t0 = t_lo + tid; t0 < t_hi; t0 += 4 * NT) {
                        unsigned jj[4]; int jrk[4]; unsigned jcol[4];
                        if (rbase == 0) {
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const unsigned t = t0 + (unsigned)u * NT;
                                jj[u] = 0; jrk[u] = 0; jcol[u] = 0;
                                if (t < t_hi) {
                                    const size_t tg = (size_t)d.off + t;
                                    const double r = log2n >= 0 ? x3_comb_eval(&sh.comb, inv, tg) : __ldcg(d.rcomb_all + tg);
                                    unsigned lo = 0, hi = len;
                                    if (staged) {
#pragma unroll 1
                                        while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (vals[mid] < r) lo = mid + 1; else hi = mid; }
                                    } else {
#pragma unroll 1
                                        while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (__ldcg(cdf + jlo + mid) < r) lo = mid + 1; else hi = mid; }
                                    }
                                    unsigned j = jlo + lo;
                                    if (j >= ng) j = (unsigned)ng - 1;
                                    jj[u] = j; jrk[u] = (int)(j / d.n); jcol[u] = j % d.n;              // owner rank and column of the ancestor
                                }
                            }
                            double gx[4], gy[4], ga[4];
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const double* sx = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk[u]] + d.o_px[cur]) : d.px[cur];
                                const double* sy = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk[u]] + d.o_py[cur]) : d.py[cur];
                                const double* sa = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jrk[u]] + d.o_pyaw[cur]) : d.pyaw[cur];
                                gx[u] = sx[jcol[u]]; gy[u] = sy[jcol[u]]; ga[u] = sa[jcol[u]];
                            }
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const unsigned t = t0 + (unsigned)u * NT;
                                if (t < t_hi) {
                                    d.idx[t] = jj[u];
                                    d.px[cur ^ 1][t] = gx[u]; d.py[cur ^ 1][t] = gy[u]; d.pyaw[cur ^ 1][t] = ga[u];     // particles[j].clone() fs1.rs:227
                                    d.w[t] = inv;                                                            // fs1.rs:228
                                    if (newrow >= 0) drows[(size_t)newrow * d.ld + t] = fs3_ref(jrk[u], jcol[u]);
                                }
                            }
                        } else {
#pragma unroll
                            for (int u = 0; u < 4; ++u) {
                                const unsigned t = t0 + (unsigned)u * NT;
                                const unsigned j = t < t_hi ? d.idx[t] : 0u;
                                jrk[u] = (int)(j / d.n); jcol[u] = j % d.n;
                            }
                        }
                        // the ancestors' row entries: eight rows x four slots of independent gathers in flight per batch (the rows were
                        // written a resample ago; one dependent HBM round trip per batch instead of per row)
                        const unsigned* srow[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u)
                            srow[u] = (d.G > 1 ? reinterpret_cast<const unsigned*>(d.peer[jrk[u]] + d.o_rows[rcur]) : d.rows[rcur]) + jcol[u];
#pragma unroll 1
                        for (int x0 = 0; x0 < nr; x0 += 8) {
                            unsigned e[8][4];
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const size_t ro = (size_t)sh.rowl[min(x0 + i, nr - 1)] * d.ld;
#pragma unroll
                                for (int u = 0; u < 4; ++u) e[i][u] = (x0 + i < nr && t0 + (unsigned)u * NT < t_hi) ? srow[u][ro] : 0u;
                            }
#pragma unroll
                            for (int i = 0; i < 8; ++i) {
                                const size_t ro = (size_t)sh.rowl[min(x0 + i, nr - 1)] * d.ld;
#pragma unroll
                                for (int u = 0; u < 4; ++u) { const unsigned t = t0 + (unsigned)u * NT; if (x0 + i < nr && t < t_hi) drows[ro + t] = e[i][u]; }
                            }
                        }
                    }
                    if ((int)(rbase + FS3_ROW_CHUNK) >= nrows) break;
                    __syncthreads();                               // everybody is through this chunk's rows
                    fs3_row_fill<NT>(d, sh, par, rbase + FS3_ROW_CHUNK, rpos);
                    __syncthreads();
                }
            }
        }
        if (newrow >= 0) {     // the identity landmarks of this CTA's slice now read through the new row (every scan of lmst is over)
#pragma unroll 1
            for (unsigned l = lm_lo + tid; l < lm_hi; l += NT) {
                const int s = l == lm_lo + tid ? s_first : d.lmst[l];
                if ((s >> 1) == 0) d.lmst[l] = (s & 1) | ((newrow + 1) << 1);
            }
        }
        FS3_TRACE(6);
    }
    // ---------------- completion: the last CTA flips the state, writes the record, tells the peers ----------------
    __syncthreads();
    if (tid == 0) sh.last = (atom_add_acq_rel_gpu(&st->post_done, 1u) + 1u == nt) ? 1 : 0;   // release my CTA's writes / acquire everybody's
    __syncthreads();
    if (!sh.last) return;
    if (x.trace && tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); x.trace[40] += t - x.trace[39]; }   // [40] the last CTA is through
    if (tid < FS3_SLOTS) x.entCnt[tid] = 0u;
    if (tid <= FS3_CERT_FLAG) x.flagsg[tid] = 0;
    if (tid < FS3_ROUNDS) { x.bar[tid] = 0u; x.resflag[tid] = 0u; }
    if (tid < 32) {
        // best particle: the last maximum over the tiles (no resample) / the last slot (after a resample every weight is 1/n)
        double bw2 = -INFINITY; unsigned bi2 = 0;
        if constexpr (KC == 1) {                               // every tile's best in flight at once, then the same comparisons in order
            double ow[(FS3_MAX_TILES + 31) / 32]; unsigned oi[(FS3_MAX_TILES + 31) / 32];
#pragma unroll
            for (unsigned i = 0; i < (FS3_MAX_TILES + 31) / 32; ++i) {
                const unsigned u = tid + 32u * i;
                ow[i] = u < nt ? __ldcg(d.tileBw + u) : 0.0; oi[i] = u < nt ? __ldcg(d.tileBi + u) : 0u;
            }
#pragma unroll
            for (unsigned i = 0; i < (FS3_MAX_TILES + 31) / 32; ++i)
                if (tid + 32u * i < nt && (ow[i] > bw2 || (ow[i] == bw2 && oi[i] > bi2))) { bw2 = ow[i]; bi2 = oi[i]; }
        } else {
#pragma unroll 1
            for (unsigned u = tid; u < nt; u += 32) { const double ow = __ldcg(d.tileBw + u); const unsigned oi = __ldcg(d.tileBi + u); if (ow > bw2 || (ow == bw2 && oi > bi2)) { bw2 = ow; bi2 = oi; } }
        }
#pragma unroll 1
        for (int o = 16; o > 0; o >>= 1) {
            const double ow = __shfl_xor_sync(0xffffffffu, bw2, o); const unsigned oi = __shfl_xor_sync(0xffffffffu, bi2, o);
            if (ow > bw2 || (ow == bw2 && oi > bi2)) { bw2 = ow; bi2 = oi; }
        }
        unsigned src = bi2;                                    // slot whose pose (in the buffer live BEFORE the flip) is reported
        if (gate) {
            bi2 = (unsigned)ng - 1; bw2 = inv;
            if (d.G == 1) src = __ldcg(d.idx + (ng - 1));          // the clone phase has just searched that slot (one GPU: it is a local slot)
            else {
                const double rl = log2n >= 0 ? x3_comb_eval(&sh.comb, inv, ng - 1) : __ldcg(d.rcomb_all + ng - 1);
                src = fs3_cdf_search(d.cum_all, sh.tend, nt, (unsigned)T, (unsigned)ng, rl);
                if (src >= ng) src = (unsigned)ng - 1;
            }
        }
        if (tid == 0) {
            const int cur = st->cur;
            const int jr = (int)(src / d.n); const unsigned jc = src % d.n;
            const double* sx = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jr] + d.o_px[cur]) : d.px[cur];
            const double* sy = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jr] + d.o_py[cur]) : d.py[cur];
            const double* sa = d.G > 1 ? reinterpret_cast<const double*>(d.peer[jr] + d.o_pyaw[cur]) : d.pyaw[cur];
            Fs3Rec* rec = d.rec;
            rec->best_idx = bi2; rec->best_w = bw2; rec->bx = sx[jc]; rec->by = sy[jc]; rec->byaw = sa[jc];
            rec->neff = neff; rec->gate = gate; rec->err = st->err;
            st->S = S; st->Q = Q; st->neff = neff; st->S2 = S2; st->r0 = r0; st->gate = gate;
            if (gate) { st->cur ^= 1; st->rcur ^= 1; st->resamples += 1; }
            st->noise_call = NT >= 128 ? step + 2u : 0u;           // nz[] = noise of EKF call step + 1
            st->post_done = 0;
            if (x.trace) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); x.trace[35] += t - x.trace[39]; x.trace[36] = t; }   // [35] this launch
            // (no system fence in front of `seq`: the host reads the record only after it has synchronised with the stream, and a
            //  fence here waits for the PCIe writes above to land — inside every step's critical path)
            *reinterpret_cast<volatile unsigned long long*>(&rec->seq) = (unsigned long long)step + 1ull;
        }
    }
    __syncthreads();
    if (d.G > 1) fs3_signal_peers(d, 1, step + 1u);
}

// =====================================================================================================================
// set-up / transfer kernels
// =====================================================================================================================
// column that holds landmark l of local slot i: own column, or through the landmark's row (maybe on another rank)
__device__ __forceinline__ const double* fs3_lm_src(const Fs3Dev& d, size_t l, unsigned i, int s, int rcur) {
    const int buf = s & 1;
    if ((s >> 1) == 0) return d.lm[buf] + l * 6 * d.ld + i;
    const unsigned ref = d.rows[rcur][(size_t)((s >> 1) - 1) * d.ld + i];
    const double* base = d.G > 1 ? reinterpret_cast<const double*>(d.peer[ref >> 28] + d.o_lm[buf]) : d.lm[buf];
    return base + l * 6 * d.ld + (ref & 0x0FFFFFFFu);
}
// AoS <-> SoA converters for upload/download (pose_w: n x 4 = (weight, x, y, yaw); lm: n x m x 6 particle-major like Vec<Particle>)
__global__ void __launch_bounds__(256) fs3_unpack_pose_kernel(const __grid_constant__ Fs3Dev d, const double* pose_w) {
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= d.n) return;
    const int cur = d.st->cur;
    d.w[i] = pose_w[4 * (size_t)i]; d.px[cur][i] = pose_w[4 * (size_t)i + 1]; d.py[cur][i] = pose_w[4 * (size_t)i + 2]; d.pyaw[cur][i] = pose_w[4 * (size_t)i + 3];
}
__global__ void __launch_bounds__(256) fs3_pack_pose_kernel(const __grid_constant__ Fs3Dev d, double* pose_w) {
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= d.n) return;
    const int cur = d.st->cur;
    pose_w[4 * (size_t)i] = d.w[i]; pose_w[4 * (size_t)i + 1] = d.px[cur][i]; pose_w[4 * (size_t)i + 2] = d.py[cur][i]; pose_w[4 * (size_t)i + 3] = d.pyaw[cur][i];
}
__global__ void __launch_bounds__(256) fs3_unpack_lm_kernel(const __grid_constant__ Fs3Dev d, const double* aos, size_t i0, size_t cnt) {
    const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x, tot = cnt * d.m * 6;
    if (e >= tot) return;
    const size_t ip = e / ((size_t)d.m * 6), rem = e % ((size_t)d.m * 6), l = rem / 6, f = rem % 6;
    d.lm[0][(l * 6 + f) * d.ld + i0 + ip] = aos[e];
}
__global__ void __launch_bounds__(256) fs3_pack_lm_kernel(const __grid_constant__ Fs3Dev d, double* aos, size_t i0, size_t cnt) {
    const size_t e = (size_t)blockIdx.x * 256 + threadIdx.x, tot = cnt * d.m * 6;
    if (e >= tot) return;
    const size_t ip = e / ((size_t)d.m * 6), rem = e % ((size_t)d.m * 6), l = rem / 6, f = rem % 6;
    aos[e] = fs3_lm_src(d, l, (unsigned)(i0 + ip), d.lmst[l], d.st->rcur)[f * d.ld];     // materialise through the rows
}
__global__ void fs3_lmst_reset_kernel(const __grid_constant__ Fs3Dev d) {        // every landmark: own columns of buffer 0
    for (unsigned l = blockIdx.x * blockDim.x + threadIdx.x; l < d.m; l += gridDim.x * blockDim.x) d.lmst[l] = 0;
}
// create_particles fs1.rs:302-306: Particle::new (fs1.rs:54-62) with Landmark::new (fs1.rs:34-40)
__global__ void __launch_bounds__(256) fs3_init_kernel(const __grid_constant__ Fs3Dev d, double init_weight) {
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= d.n) return;
    d.w[i] = init_weight;
    d.px[0][i] = 0.0; d.py[0][i] = 0.0; d.pyaw[0][i] = 0.0;
    for (size_t l = 0; l < d.m; ++l) {
        double* p = d.lm[0] + l * 6 * d.ld + i;
        p[0] = 0.0; p[d.ld] = 0.0; p[2 * (size_t)d.ld] = 1000.0; p[3 * (size_t)d.ld] = 0.0; p[4 * (size_t)d.ld] = 0.0; p[5 * (size_t)d.ld] = 1000.0;
    }
}
// pfgpu_fs_seed_map: initialised map for benchmarks/tests (see include/pfgpu.h)
__global__ void __launch_bounds__(256) fs3_seed_pose_kernel(const __grid_constant__ Fs3Dev d, double x, double y, double yaw) {
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= d.n) return;
    const int cur = d.st->cur;
    d.px[cur][i] = x; d.py[cur][i] = y; d.pyaw[cur][i] = yaw;
    d.w[i] = 1.0 / (double)d.n_glob;
}
__global__ void __launch_bounds__(256) fs3_seed_lm_kernel(const __grid_constant__ Fs3Dev d, const double* lm_xy, double sigma, double cov0, uint64_t seed) {
    const unsigned i = blockIdx.x * 256u + threadIdx.x;
    if (i >= d.n) return;
#pragma unroll 1
    for (size_t l = blockIdx.y; l < d.m; l += gridDim.y) {      // (gridDim.y is at most 65 535)
        double z0, z1;
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_INIT_A, 0, ((uint64_t)d.off + i) * d.m + l), &z0, &z1);
        double* p = d.lm[0] + l * 6 * d.ld + i;
        p[0] = lm_xy[2 * l] + sigma * z0; p[d.ld] = lm_xy[2 * l + 1] + sigma * z1;
        p[2 * (size_t)d.ld] = cov0; p[3 * (size_t)d.ld] = 0.0; p[4 * (size_t)d.ld] = 0.0; p[5 * (size_t)d.ld] = cov0;
    }
}

// get_observations fs1.rs:277-299 (the simulator next to the filter): landmarks within max_range of the true pose, in
// landmark order, range and bearing perturbed by N(0,1) * sqrt(R) drawn from Philox stream PFC_STREAM_OBS (call, landmark id).
// One CTA; order-preserving compaction by ballot.  out_k[0] = number of observations.
__global__ void __launch_bounds__(1024) fs3_get_observations_kernel(double x, double y, double yaw, const double* lm_xy, unsigned n_lm,
                                                                    double max_range, double sr0, double sr1, uint64_t seed, uint32_t call,
                                                                    Fs3Obs* out, unsigned* out_k) {
    __shared__ unsigned s_w[32];
    __shared__ unsigned s_base;
    const unsigned lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (unsigned l0 = 0; l0 < n_lm; l0 += 1024) {
        const unsigned id = l0 + threadIdx.x;
        bool in = false; double d = 0.0, dx = 0.0, dy = 0.0;
        if (id < n_lm) { dx = lm_xy[2 * id] - x; dy = lm_xy[2 * id + 1] - y; d = sqrt(dx * dx + dy * dy); in = d <= max_range; }
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) s_w[wid] = __popc(m);
        __syncthreads();
        unsigned off = s_base;
        for (unsigned w = 0; w < wid; ++w) off += s_w[w];
        if (in) {
            const unsigned o = off + __popc(m & ((1u << lane) - 1u));
            const double angle = fs_normalize_angle(pfc_atan2(dy, dx) - yaw);
            double z0, z1;
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_OBS, call, id), &z0, &z1);
            out[o].d = d + z0 * sr0;                               // fs1.rs:291
            out[o].angle = angle + z1 * sr1;                       // fs1.rs:292
            out[o].lm_id = (int)id; out[o].pad = 0;
        }
        __syncthreads();
        if (threadIdx.x == 0) { unsigned t = 0; for (unsigned w = 0; w < 32; ++w) t += s_w[w]; s_base += t; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *out_k = s_base;
}

