// pf3.cuh — the tail of ParticleFilterLocalizer::try_step / MonteCarloLocalizer::try_step in ONE launch.
//
// pf.rs = crates/rust_robotics_localization/src/particle_filter.rs, mcl.rs = .../monte_carlo_localization.rs.  After the fused
// predict + likelihood kernel (pf_predict_weight_kernel) a step still has to: normalise (pf.rs:426-439), gate on N_eff
// (pf.rs:337-345, 416-423; MCL resamples every step, mcl.rs:298), build the cumulative weights (pf.rs:448-453; MCL forces the
// last entry to 1, mcl.rs:334-336), draw one uniform per output slot and search it (pf.rs:456-470, mcl.rs:344-361, 387-392),
// clone the poses, and refresh the cached estimate + covariance (pf.rs:382-413, 499-503).  Run as separate kernels that is ~21
// launches of a few microseconds each — the step is launch-latency bound below ~10^5 particles.  Here the
// same arithmetic runs in one kernel of <= one co-resident CTA per SM, built on the FastSLAM post kernel's machinery: the exact
// sequential sums are fs3_xsum (fs3.cuh) over tiles held in shared memory, grid barriers are arrival counters (workspace x).
//
// Bit-exactness: the three sums (S = sum w_raw, Q = sum w^2, the cumulative weights) are the reference's sequential f64 sums,
// exactly (x3_core.h); the divisions are IEEE; the uniforms are the Philox stream the unfused path draws (same stream, call
// counter and slot index); estimate / covariance are tolerance-level quantities (1e-6): central moments merged in a fixed tree
// (include/pf_moments.h), as in the unfused path.  Fixed particle count, one GPU (the KLD-adaptive and the sharded forms keep the multi-kernel path).
#pragma once
#include "fs3.cuh"
#include "pf_kernels.cuh"

struct Pf3Arg {
    PfDev pd;
    double threshold;
    int mode;                      // 0 = PF (N_eff gate, fallback index 0), 1 = MCL (every step, last := 1, fallback n - 1)
    uint64_t seed;
    unsigned K, m32;
    double* tsum; double* tsq;     // [tiles] tree-order tile sums of w_raw and w_raw^2 (steer the classification only)
    double* mom;                   // [tiles] PfMom
};

template <int NT>
__global__ void __launch_bounds__(NT, 1)
pf3_post_kernel(const __grid_constant__ Fs3Sum x, const __grid_constant__ Pf3Arg a) {
    static_assert(FS3_MAX_TILES <= NT, "the last CTA merges one tile partial per thread");
    extern __shared__ __align__(16) double vals[];            // [2][K][NT]: the tile's weights, their squares
    __shared__ Fs3Sh<NT> sh;
    const PfDev& pd = a.pd;
    const int tid = threadIdx.x;
    const unsigned b = blockIdx.x, nt = gridDim.x, K = a.K;
    const size_t n = pd.n, T = (size_t)NT * K, g0 = (size_t)b * T + (size_t)tid * K;
    double* vals2 = vals + (size_t)K * NT;
    Fs3State* st = x.st;
    const int cur = *pd.cur;
    // ---- this tile's raw weights; tile sums -> approximate prefixes in front of the tile ----
    double ts = 0.0, tq = 0.0;
#pragma unroll 4
    for (unsigned k = 0; k < K; ++k) { const double v = g0 + k < n ? pd.w_raw[g0 + k] : 0.0; vals[k * NT + tid] = v; ts += v; tq += v * v; }
    fs3_block_sum2<NT>(ts, tq, sh.red[0], sh.red[1]);
    if (tid == 0) { a.tsum[b] = ts; a.tsq[b] = tq; }
    fs3_grid_sync<NT>(x, PF3_R_TILES, nt);
    double toff = 0.0, qoff = 0.0;
#pragma unroll 2
    for (unsigned p = tid; p < b; p += NT) { toff += __ldcg(a.tsum + p); qoff += __ldcg(a.tsq + p); }
    fs3_block_sum2<NT>(toff, qoff, sh.red[0], sh.red[1]);      // (red[] is free again: the grid barrier above is also a block barrier;
                                                               //  wd[] is the first scratch fs3_xsum writes, with no barrier in between)
    // ---------------- S = sum w_raw, sequential (normalize_weights pf.rs:426-439) ----------------
    const double S = fs3_xsum<NT>(x, sh, vals, K, nt, toff, FS3_S, PF3_R_S, a.m32, nullptr, 0, 0.0, 0.0, 0.0, 0.0, 0, nullptr);
    const double unif = 1.0 / (double)pd.n_global;
#pragma unroll 1
    for (unsigned k = 0; k < K; ++k) {
        const size_t i = g0 + k;
        double v = 0.0;
        if (i < n) { v = S > 0.0 ? fs3_div(vals[k * NT + tid], S) : unif; pd.w[i] = v; }      // "else 1.0 / len" pf.rs:435-437
        vals[k * NT + tid] = v; vals2[k * NT + tid] = v * v;
    }
    // ---------------- gate (calc_n_eff pf.rs:416-423, resample pf.rs:337-345; MCL: always, mcl.rs:298) ----------------
    int gate = 1;
    double Q = 0.0, neff = 0.0;
    if (a.mode == 0) {
        // Only the DECISION feeds back into the state.  Q is first taken from the tree-order tile sums of w_raw^2 (already in a.tsq):
        // sum w_raw_i^2 / S^2 differs from the reference's sequential sum of fl(w_raw_i / S)^2 by at most (n + 64) 2^-51 relatively;
        // only when N_eff lands that close to the threshold is the exact sequential sum evaluated (fs3_xsum over the squares).
        double qa = (unsigned)tid < nt ? __ldcg(a.tsq + tid) : 0.0, dummy = 0.0;
        __syncthreads();
        fs3_block_sum2<NT>(qa, dummy, sh.red[0], sh.red[1]);
        Q = S > 0.0 ? fs3_div(fs3_div(qa, S), S) : unif;           // uniform fallback: n * (1/n)^2
        neff = Q > 0.0 ? fs3_div(1.0, Q) : 0.0;
        const double thr = (double)pd.n_global * a.threshold;
        const double slack = 16.0 * (double)(n + 64) * 2.220446049250313e-16;
        // (the bound assumes that no w_raw^2 that matters under- or overflows: S inside [1e-120, 1e120]; K likelihood factors of
        //  1 / sqrt(2 pi sigma^2) each can leave that window in either direction)
        const bool scale_ok = !(S > 0.0) || (S >= 1e-120 && S <= 1e120);
        if (!scale_ok || !(fabs(neff - thr) > slack * fmax(fabs(thr), fabs(neff)))) {     // rare; the same decision in every CTA
            const double toffq = S > 0.0 ? fs3_div(fs3_div(qoff, S), S) : (double)((size_t)b * T) * unif * unif;
            // the steer of the exact sum must be finite: when the w_raw^2 in front of this tile overflowed (S > ~1e154), this
            // CTA flags the sum as bad and it takes the serial walk, exact by construction
            if (tid == 0 && !(fabs(toffq) <= 1.7976931348623157e308)) x.flagsg[FS3_Q] = 1;
            __syncthreads();
            Q = fs3_xsum<NT>(x, sh, vals2, K, nt, toffq, FS3_Q, PF3_R_Q, a.m32, nullptr, 0, 0.0, 0.0, 0.0, 0.0, 0, nullptr);
            neff = Q > 0.0 ? fs3_div(1.0, Q) : 0.0;
        }
        gate = neff < thr ? 1 : 0;
    }
    double ctot = 0.0;
    if (gate) {
        // ---------------- cumulative weights (pf.rs:448-453 / mcl.rs:328-336), exact inclusive prefix of every weight ----------------
        const double toffc = S > 0.0 ? fs3_div(toff, S) : (double)((size_t)b * T) * unif;
        if (tid == 0 && !(fabs(toffc) <= 1.7976931348623157e308)) x.flagsg[FS3_CDF] = 1;     // (the same for the CDF's steer)
        __syncthreads();                                       // (without the Q sum, the S sum used the same scratch half)
        Fs3Run run;
        ctot = fs3_xsum<NT>(x, sh, vals, K, nt, toffc, FS3_CDF, PF3_R_CDF, a.m32, pd.cum, 0, 0.0, 0.0, 0.0, 0.0, 1, &run);
        (void)fs3_xsum_emit<NT>(x, sh, vals, K, a.m32, &run, PF3_R_CDF, pd.cum, 1, nullptr, 15);
        __syncthreads();                                       // every prefix of this tile is stored before the last one is overridden
        if (a.mode == 1 && b == (unsigned)((n - 1) / T) && tid == 0) { pd.cum[n - 1] = 1.0; x.tileEnd[b] = 1.0; }   // *last = 1.0 mcl.rs:334-336
        fs3_grid_sync<NT>(x, PF3_R_CDF_DONE, nt);              // the whole CDF is visible
        if ((unsigned)tid < nt) sh.tend[tid] = __ldcg(x.tileEnd + tid);
        // A CDF with a bad value was stored by the serial walk as its running maximum, NaN sticky: non-decreasing up to the
        // first NaN, NaN from there on (MCL: but for the last entry, 1).  The lower bound below (NaN counts as >= r) then finds
        // the reference's first i with r <= c_i whenever one lies before the first NaN; when it lands on a NaN instead, the
        // reference's linear scan matches nothing up to n - 1 and takes its fallback (PF 0; MCL n - 1, the forced last entry).
        const bool cdf_bad = __ldcg(x.flagsg + FS3_CDF) != 0;
        __syncthreads();
        // ---------------- one uniform per output slot, first index with r <= c_i, clone (pf.rs:456-470, mcl.rs:344-361) ----------------
        const uint32_t call = pd.counters[0];
        const Pose4* src = pf_pose(pd, cur);
        Pose4* dst = pf_pose(pd, cur ^ 1);
#pragma unroll 1
        for (unsigned k = 0; k < K; ++k) {
            const size_t t = g0 + k;
            if (t >= n) break;
            const double r = pfc_u01_53(pfc_blk_u64(pfc_rng_block(a.seed, PFC_STREAM_PF_RESAMPLE, call, pd.offset + t), 0));
            unsigned lo = 0, hi = nt;                          // tile whose last value is the first >= r
#pragma unroll 1
            while (lo < hi) { const unsigned mid = (lo + hi) >> 1; if (sh.tend[mid] < r) lo = mid + 1; else hi = mid; }
            size_t index;
            if (lo >= nt) index = a.mode == 1 ? n - 1 : 0;     // r beyond the last cumulative weight: fallback of pf.rs:459-465 / mcl.rs:387-392
            else {
                size_t jl = (size_t)lo * T, jh = jl + T < n ? jl + T : n;
                const double* __restrict__ c = pd.cum;
#pragma unroll 1
                while (jl < jh) { const size_t mid = jl + ((jh - jl) >> 1); if (__ldcg(c + mid) < r) jl = mid + 1; else jh = mid; }
                index = jl < n ? jl : (a.mode == 1 ? n - 1 : 0);
                if (cdf_bad && jl < n) { const double cj = __ldcg(c + jl); if (cj != cj) index = a.mode == 1 ? n - 1 : 0; }
            }
            pd.idx[t] = (uint32_t)index;
            Pose4 p;
            pose_load(src, index, p);
            pose_store(dst, t, p);
            pd.w[t] = unif;                                    // w = 1/n pf.rs:468
        }
    }
    // ---------------- estimate + covariance (refresh_cache pf.rs:499-503): this tile's central moments ----------------
    __shared__ PfMom smom[NT / 32];
    {
        const Pose4* pose = pf_pose(pd, gate ? cur ^ 1 : cur);
        PfMom v = PF_MOM_EMPTY;
#pragma unroll 1
        for (unsigned k = 0; k < K; ++k) {
            const size_t i = g0 + k;
            if (i >= n) break;
            Pose4 p;
            pose_load(pose, i, p);                             // (a resample step reads the clones this thread just wrote)
            pf_mom_add(&v, gate ? unif : vals[k * NT + tid], p.x, p.y, p.yaw, p.v);
        }
        pf_mom_block_merge<NT>(v, smom);
        if (tid == 0) pf_mom_store(a.mom + (size_t)b * PF_MOM, v);
    }
    // ---------------- completion: the last CTA reduces the moments, flips the state, resets the counters ----------------
    __syncthreads();
    if (tid == 0) sh.last = (atom_add_acq_rel_gpu(&st->post_done, 1u) + 1u == nt) ? 1 : 0;   // release my CTA's writes / acquire everybody's
    __syncthreads();
    if (!sh.last) return;
    if (tid < FS3_SLOTS) { x.flagsg[tid] = 0; x.entCnt[tid] = 0u; }
    if (tid < FS3_ROUNDS) { x.bar[tid] = 0u; x.resflag[tid] = 0u; }
    PfMom v = PF_MOM_EMPTY;                                    // thread t takes tile t (nt <= FS3_MAX_TILES <= NT), then the block tree
    if ((unsigned)tid < nt) pf_mom_load(a.mom + (size_t)tid * PF_MOM, v);
    pf_mom_block_merge<NT>(v, smom);
    if (tid == 0) {
        pf_mom_final(&v, pd.scal + 4, pd.scal + 8);
        pd.scal[0] = S; pd.scal[1] = Q; pd.scal[2] = ctot; pd.scal[3] = neff;
        *pd.gate = gate;
        if (gate) { *pd.cur = cur ^ 1; pd.counters[0] += 1; }      // pf_flip_kernel
        st->post_done = 0;
    }
}
