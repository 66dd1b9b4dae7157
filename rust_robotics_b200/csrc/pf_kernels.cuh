// pf_kernels.cuh — ParticleFilterLocalizer / MonteCarloLocalizer device kernels.
// Reference: pf.rs = crates/rust_robotics_localization/src/particle_filter.rs, mcl.rs = .../monte_carlo_localization.rs.
//
// HBM layout (per shard of n particles):
//   pose[2][n]   32-byte records {x, y, yaw, v} (ping-pong; `cur` on the device selects the live one)
//                — one record = one 32 B DRAM sector, so the multinomial gather (random indices, pf.rs:455-470)
//                costs one sector per particle instead of four with four separate columns.
//   w_raw[n]     likelihood products before normalisation (pf.rs:317-328)
//   w[n]         normalised weights (pf.rs:426-439)
//   cum[n]       exact sequential cumulative weights (pf.rs:448-453)
//   idx[n]       resample ancestry (u32)
#pragma once
#include "common.cuh"
#include "xsum.cuh"
#include "../../include/pf_moments.h"
#include "../../include/pf_odom_math.h"

struct __align__(32) Pose4 { double x, y, yaw, v; };

#define PF_NT 256

struct PfDev {
    size_t n = 0, n_global = 0, offset = 0;
    Pose4* pose[2] = {nullptr, nullptr};
    int* cur = nullptr;            // device: index of the live pose buffer
    double* w_raw = nullptr;
    double* w = nullptr;
    double* cum = nullptr;
    uint32_t* idx = nullptr;
    double* scal = nullptr;        // [0] S=sum w_raw  [1] Q=sum w^2  [2] cum total  [3] neff  [4..7] est  [8..23] cov (row-major)
    int* gate = nullptr;           // device: 1 if this step resamples
    double* partial = nullptr;     // [blocks] PfMom
    double* obs = nullptr;         // device copy of the observation list (k x 3) when it does not fit the launch parameters
    unsigned int* counters = nullptr;   // device: [0] resamples done so far (= Philox call index of the next resample)
};

// Observation lists of up to PF_PARAM_OBS entries travel inside the kernel's launch parameters (no H2D copy).
#define PF_PARAM_OBS 32
struct PfObsParam { double o[3 * PF_PARAM_OBS]; };

// select by ternary: indexing the by-value parameter struct with a runtime index would force a stack copy
__device__ __forceinline__ Pose4* pf_pose(const PfDev& d, int cur) { return cur ? d.pose[1] : d.pose[0]; }
__device__ __forceinline__ void pose_load(const Pose4* p, size_t i, Pose4& o) {
    const double2* q = reinterpret_cast<const double2*>(p + i);
    double2 a = q[0], b = q[1];
    o.x = a.x; o.y = a.y; o.yaw = b.x; o.v = b.y;
}
__device__ __forceinline__ void pose_store(Pose4* p, size_t i, const Pose4& o) {
    double2* q = reinterpret_cast<double2*>(p + i);
    q[0] = make_double2(o.x, o.y); q[1] = make_double2(o.yaw, o.v);
}

// Augmented MCL (DESIGN §3.8): the recovery state lives next to the step's scalars, the injection count next to the draw counter.
#define PF_REC_SLOW 24             // scal[24] w_slow, scal[25] w_fast, scal[26] p (injection probability)
#define PF_REC_FAST 25
#define PF_REC_P 26
#define PF_REC_COUNT 1             // counters[1]: slots injected by the last predict
// injection arguments of a predict: the region (x0, x1, y0, y1) and whether this is the first predict after a resample stage
struct PfInj { double r[4]; int arm; };

// Likelihood-field scan model (DESIGN §3.9).  The table q (f64, cell ix * H + iy) is built at set time (pf_lfield.cuh); a scan
// step reads one cell per used beam.  Lists of up to PF_PARAM_BEAMS (r_i, a_i = i * angle_increment) pairs travel in the launch
// parameters (the first 48 in the observation block, which a scan does not use, the rest in PfBeamParam), longer ones through d.obs.
#define PF_PARAM_BEAMS 64
struct PfBeamParam { double b[2 * PF_PARAM_BEAMS - 3 * PF_PARAM_OBS]; };
struct PfScan {
    const double* q = nullptr;
    double res = 1.0, half_w = 0.0, half_h = 0.0;   // half_w = W as f64 / 2.0 (world_to_grid, occupancy_grid_map.rs:144-153)
    double q_out = 0.0, angle_min = 0.0;
    int W = 0, H = 0;
};
// Rust's `as i32` of a float: saturating, NaN -> 0
__device__ __forceinline__ int pf_lf_sat_i32(double v) {
    if (v != v) return 0;
    if (v >= 2147483647.0) return 2147483647;
    if (v <= -2147483648.0) return -2147483647 - 1;
    return (int)v;
}
// the factor of one beam endpoint: q[ix][iy] inside the grid, q_out outside
__device__ __forceinline__ double pf_lf_factor(const PfScan& sc, const pfc_rcp_t& rres, double ex, double ey) {
    const int ix = pf_lf_sat_i32(floor(pfc_div_by(ex, rres) + sc.half_w));
    const int iy = pf_lf_sat_i32(floor(pfc_div_by(ey, rres) + sc.half_h));
    if (ix < 0 || ix >= sc.W || iy < 0 || iy >= sc.H) return sc.q_out;
    return __ldg(sc.q + ((size_t)ix * (size_t)sc.H + (size_t)iy));
}
#include "pf_beam.cuh"              // the beam model (DESIGN §3.11): PfBeam, the ray caster and the factor

// try_predict_with_control (pf.rs:279-296, mcl.rs:236-253) and/or the likelihood loop of
// try_update_with_observations (pf.rs:316-329, mcl.rs:273-283), fused in one pass over the pose records.
// INJ (augmented MCL): when `inj.arm` and the last resample stage resampled (*d.gate), each slot is first replaced with probability
// p = scal[PF_REC_P] by a pose drawn uniformly over the region (weight unchanged), then predicted like any other.
// SCAN: the weight is the likelihood field of k_obs beams (r_i, a_i) instead of the landmark ranges (DESIGN §3.9).
// SCAN and BEAM: the weight is the beam model of those beams instead (ray-cast in the clearance table bm, DESIGN §3.11).
// ODOM: the predict moves every particle by the odometry increment od (include/pf_odom_math.h, DESIGN §3.14) instead of the
// control (u0, u1); sv, sw and dt are then unused.
template <bool DO_PREDICT, bool DO_WEIGHT, bool PARAM_OBS, bool INJ = false, bool SCAN = false, bool BEAM = false, bool ODOM = false>
__global__ void __launch_bounds__(PF_NT) pf_predict_weight_kernel(PfDev d, const __grid_constant__ PfObsParam po,
                                                                  double u0, double u1, double sv, double sw,
                                                                  double dt, uint64_t seed, uint32_t call,
                                                                  int k_obs, double sigma, PfInj inj, PfScan sc,
                                                                  const __grid_constant__ PfBeamParam pb, PfBeam bm, PfOdom od) {
    extern __shared__ double s_obs_pf[];     // k_obs x (d, lx, ly): the observation vector staged once per CTA; SCAN: k_obs x (r, a)
    if (DO_WEIGHT) {
        if constexpr (SCAN) {
            for (int j = threadIdx.x; j < 2 * k_obs; j += PF_NT)
                s_obs_pf[j] = PARAM_OBS ? (j < 3 * PF_PARAM_OBS ? po.o[j] : pb.b[j - 3 * PF_PARAM_OBS]) : d.obs[j];
        } else {
            for (int j = threadIdx.x; j < 3 * k_obs; j += PF_NT) s_obs_pf[j] = PARAM_OBS ? po.o[j] : d.obs[j];
        }
        __syncthreads();
    }
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    Pose4* pose = pf_pose(d, *d.cur);
    Pose4 p;
    pose_load(pose, i, p);
    if constexpr (INJ) {
        static_assert(DO_PREDICT, "injection happens in a predict");
        const double pinj = d.scal[PF_REC_P];
        if (inj.arm && *d.gate && pinj > 0.0) {                     // the same decision in every thread of the grid
            const pfc_u32x4 a = pfc_rng_block(seed, PFC_STREAM_PF_INJECT_A, call, d.offset + i);
            const bool hit = pfc_u01_53(pfc_blk_u64(a, 0)) < pinj;
            if (hit) {
                const pfc_u32x4 b = pfc_rng_block(seed, PFC_STREAM_PF_INJECT_B, call, d.offset + i);
                pfc_region_pose(inj.r, pfc_u01_53(pfc_blk_u64(a, 1)), pfc_u01_53(pfc_blk_u64(b, 0)), pfc_u01_53(pfc_blk_u64(b, 1)),
                                &p.x, &p.y, &p.yaw);
                p.v = 0.0;
            }
            const unsigned act = __activemask(), votes = __ballot_sync(act, hit);   // one integer atomic per warp
            if (votes && (threadIdx.x & 31) == (unsigned)(__ffs(act) - 1)) atomicAdd(d.counters + PF_REC_COUNT, (unsigned)__popc(votes));
        }
    }
    if constexpr (ODOM) {
        static_assert(DO_PREDICT, "odometry moves particles in a predict");
        double za, zb, zc, unused;
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_PF_PREDICT, call, d.offset + i), &za, &zb);
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_PF_ODOM, call, d.offset + i), &zc, &unused);
        pf_odom_move(&od, za, zb, zc, &p.x, &p.y, &p.yaw);         // v is left as it was
        pose_store(pose, i, p);
    } else if (DO_PREDICT) {
        double z0, z1;
        pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_PF_PREDICT, call, d.offset + i), &z0, &z1);
        double v_noise = sv > 0.0 ? 0.0 + sv * z0 : 0.0;            // Normal::sample = mean + std*z; no draw if sigma == 0
        double yaw_noise = sw > 0.0 ? 0.0 + sw * z1 : 0.0;
        double v_noisy = u0 + v_noise;                              // pf.rs:289
        double yaw_rate_noisy = u1 + yaw_noise;                     // pf.rs:290
        double s, c;
        pfc_sincos(p.yaw, &s, &c);
        p.x = p.x + v_noisy * c * dt;                               // pf.rs:292
        p.y = p.y + v_noisy * s * dt;                               // pf.rs:293
        p.yaw = p.yaw + yaw_rate_noisy * dt;                        // pf.rs:294 (yaw is not wrapped)
        p.v = v_noisy;                                              // pf.rs:295
        pose_store(pose, i, p);
    }
    if constexpr (SCAN && BEAM) {
        static_assert(DO_WEIGHT, "a scan is a weight");
        const pfc_rcp_t rres = pfc_rcp_make(bm.res), rdenom = pfc_rcp_make(bm.denom);
        const double base = p.yaw + bm.angle_min;                   // (yaw + angle_min) + i * angle_increment
        int ix0, iy0;
        pf_beam_start(bm, rres, p.x, p.y, &ix0, &iy0);
        double w = 1.0;
        for (int j = 0; j < k_obs; ++j) {
            const double rhat = pf_beam_cast(bm, rres, p.x, p.y, ix0, iy0, base + s_obs_pf[2 * j + 1]);
            w = w * pf_beam_factor(bm, rdenom, s_obs_pf[2 * j], rhat);
        }
        d.w_raw[i] = w;
    } else if constexpr (SCAN) {
        static_assert(DO_WEIGHT, "a scan is a weight");
        const pfc_rcp_t rres = pfc_rcp_make(sc.res);                // one reciprocal for every IEEE quotient x / res
        const double base = p.yaw + sc.angle_min;                   // (yaw + angle_min) + i * angle_increment
        double w = 1.0;
        for (int j = 0; j < k_obs; ++j) {
            const double r = s_obs_pf[2 * j];
            double s, c;
            pfc_sincos(base + s_obs_pf[2 * j + 1], &s, &c);
            w = w * pf_lf_factor(sc, rres, p.x + r * c, p.y + r * s);
        }
        d.w_raw[i] = w;
    } else if (DO_WEIGHT) {
        const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (sigma * sigma));   // gauss_likelihood pf.rs:476-479
        const double denom = 2.0 * (sigma * sigma);
        const pfc_rcp_t rdenom = pfc_rcp_make(denom);               // one reciprocal for all k_obs IEEE quotients
        double w = 1.0;                                             // pf.rs:317: the previous weight is discarded
        for (int j = 0; j < k_obs; ++j) {
            double dx = p.x - s_obs_pf[3 * j + 1];
            double dy = p.y - s_obs_pf[3 * j + 2];
            double d_pred = sqrt(dx * dx + dy * dy);
            double diff = s_obs_pf[3 * j] - d_pred;
            w = w * (coeff * pfc_exp(pfc_div_by(-(diff * diff), rdenom)));
        }
        d.w_raw[i] = w;
    }
}

// normalize_weights pf.rs:426-439 / mcl.rs:394-406
__global__ void __launch_bounds__(PF_NT) pf_normalize_kernel(PfDev d) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    const double S = d.scal[0];
    d.w[i] = S > 0.0 ? d.w_raw[i] / S : 1.0 / (double)d.n_global;
}

// augmented MCL's averages (Probabilistic Robotics Table 8.3) from S = scal[0] over the n_global weights S sums, then the injection
// probability the next armed predict uses.  Non-finite S: no update.
__global__ void pf_recovery_filter_kernel(PfDev d, double a_slow, double a_fast) {
    const double S = d.scal[0];
    double ws = d.scal[PF_REC_SLOW], wf = d.scal[PF_REC_FAST];
    if (S - S == 0.0) {
        const double w_avg = S / (double)d.n_global;
        ws = ws + a_slow * (w_avg - ws);
        wf = wf + a_fast * (w_avg - wf);
        d.scal[PF_REC_SLOW] = ws; d.scal[PF_REC_FAST] = wf;
    }
    double p = 0.0;
    if (ws > 0.0) {
        const double q = wf / ws;
        if (q - q == 0.0) { p = 1.0 - q; if (!(p > 0.0)) p = 0.0; }
    }
    d.scal[PF_REC_P] = p;
}

// global initialisation: every particle uniform over the region r4 = (x0, x1, y0, y1), v = 0, w = 1/n
__global__ void pf_init_region_kernel(PfDev d, double x0, double x1, double y0, double y1, uint64_t seed) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    const double r4[4] = { x0, x1, y0, y1 };
    const pfc_u32x4 a = pfc_rng_block(seed, PFC_STREAM_REGION_A, 0, d.offset + i);
    const pfc_u32x4 b = pfc_rng_block(seed, PFC_STREAM_REGION_B, 0, d.offset + i);
    Pose4 p;
    pfc_region_pose(r4, pfc_u01_53(pfc_blk_u64(a, 0)), pfc_u01_53(pfc_blk_u64(a, 1)), pfc_u01_53(pfc_blk_u64(b, 0)), &p.x, &p.y, &p.yaw);
    p.v = 0.0;
    pose_store(pf_pose(d, *d.cur), i, p);
    d.w[i] = 1.0 / (double)d.n_global;
    d.w_raw[i] = d.w[i];
}

struct PfValWSq { const double* w; __device__ __forceinline__ double operator()(size_t i) const { double x = w[i]; return x * x; } };

// calc_n_eff + gate: pf.rs:337-345, 416-423.  MCL resamples every step (mcl.rs:298).
__global__ void pf_gate_kernel(PfDev d, double threshold, int mode) {
    double Q = d.scal[1];
    double neff = Q > 0.0 ? 1.0 / Q : 0.0;
    d.scal[3] = neff;
    *d.gate = (mode == 1) ? 1 : (neff < (double)d.n_global * threshold ? 1 : 0);
}

// MCL: "if let Some(last) = cumulative_weights.last_mut() { *last = 1.0 }"  mcl.rs:334-336
__global__ void pf_force_last_kernel(PfDev d) {
    if (!*d.gate) return;
    d.cum[d.n - 1] = 1.0;
}

// index search: first i with r <= c_i (pf.rs:459-465, fallback 0; mcl.rs:387-392, fallback len-1).
// Non-negative finite weights give non-decreasing cumulative weights, so the linear scan equals a lower_bound.  `bad`: the scan
// of the cumulative weights saw a negative, infinite or NaN weight (xs flags[3]); then the CDF may go down or hold NaN, which
// the linear scan skips, and each slot scans as the reference does.
__global__ void __launch_bounds__(PF_NT) pf_search_kernel(PfDev d, uint64_t seed, int mode, const int* bad) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= d.n) return;
    const uint32_t call = d.counters[0];
    double r = pfc_u01_53(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_PF_RESAMPLE, call, d.offset + t), 0));
    const double* __restrict__ c = d.cum;
    size_t lo = 0, hi = d.n;
    if (*bad) {
        while (lo < d.n && !(r <= c[lo])) ++lo;
        hi = lo;
    }
    while (lo < hi) {
        size_t mid = lo + ((hi - lo) >> 1);
        if (c[mid] < r) lo = mid + 1; else hi = mid;
    }
    size_t index = lo < d.n ? lo : (mode == 1 ? d.n - 1 : 0);
    d.idx[t] = (uint32_t)index;
}

// new_particles.push(particles[index].clone()); w = 1/n   (pf.rs:467-469, mcl.rs:351,357-361)
__global__ void __launch_bounds__(PF_NT) pf_gather_kernel(PfDev d) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= d.n) return;
    const int cur = *d.cur;
    Pose4 p;
    pose_load(pf_pose(d, cur), d.idx[t], p);
    pose_store(pf_pose(d, cur ^ 1), t, p);
    d.w[t] = 1.0 / (double)d.n_global;
}
__global__ void pf_flip_kernel(PfDev d) { if (*d.gate) { *d.cur ^= 1; d.counters[0] += 1; } }

// thread 0 receives the block's PfMom values merged in a fixed tree: lanes by shuffle, then the warps in order
template <int NT>
__device__ __forceinline__ void pf_mom_block_merge(PfMom& v, PfMom* sm /* [NT / 32] */) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        PfMom u;
        u.w = __shfl_down_sync(0xffffffffu, v.w, o);
#pragma unroll
        for (int k = 0; k < 4; ++k) u.m[k] = __shfl_down_sync(0xffffffffu, v.m[k], o);
#pragma unroll
        for (int k = 0; k < 10; ++k) u.q[k] = __shfl_down_sync(0xffffffffu, v.q[k], o);
        pf_mom_merge(&v, &u);
    }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < NT / 32; ++w) pf_mom_merge(&v, &sm[w]);
}
__device__ __forceinline__ void pf_mom_store(double* dst, const PfMom& v) {
    dst[0] = v.w;
#pragma unroll
    for (int k = 0; k < 4; ++k) dst[1 + k] = v.m[k];
#pragma unroll
    for (int k = 0; k < 10; ++k) dst[5 + k] = v.q[k];
}
__device__ __forceinline__ void pf_mom_load(const double* src, PfMom& v) {
    v.w = __ldcg(src);
#pragma unroll
    for (int k = 0; k < 4; ++k) v.m[k] = __ldcg(src + 1 + k);
#pragma unroll
    for (int k = 0; k < 10; ++k) v.q[k] = __ldcg(src + 5 + k);
}
#define PF_MOM_EMPTY { 0.0, { 0.0, 0.0, 0.0, 0.0 }, { 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0 } }

// compute_estimate + compute_covariance (pf.rs:382-413) as weighted central moments (include/pf_moments.h): thread t merges
// particles t, t + nblocks * PF_NT, ... one at a time, the block merges its threads in a fixed tree, one PfMom per block.
// Tolerance-level quantity: the merge order is fixed by (n, nblocks), not the reference's sequential order.
__global__ void __launch_bounds__(PF_NT) pf_moments_kernel(PfDev d, int nblocks) {
    __shared__ PfMom sm[PF_NT / 32];
    const Pose4* pose = pf_pose(d, *d.cur);
    PfMom v = PF_MOM_EMPTY;
    const size_t stride = (size_t)nblocks * PF_NT;
    constexpr int B = 4;                               // particles in flight per thread (the merges are one dependent chain)
    for (size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x; i < d.n; i += B * stride) {
        Pose4 p[B];
        double w[B];
#pragma unroll
        for (int b = 0; b < B; ++b)
            if (i + b * stride < d.n) { pose_load(pose, i + b * stride, p[b]); w[b] = d.w[i + b * stride]; }
#pragma unroll
        for (int b = 0; b < B; ++b)
            if (i + b * stride < d.n) pf_mom_add(&v, w[b], p[b].x, p[b].y, p[b].yaw, p[b].v);
    }
    pf_mom_block_merge<PF_NT>(v, sm);
    if (threadIdx.x == 0) pf_mom_store(d.partial + (size_t)blockIdx.x * PF_MOM, v);
}
// one CTA: thread t merges block partials t, t + PF_NT, ... in order, then the block tree; out = this shard's PfMom
__global__ void __launch_bounds__(PF_NT) pf_moments_reduce_kernel(const double* partial, int nblocks, double* out) {
    __shared__ PfMom sm[PF_NT / 32];
    PfMom v = PF_MOM_EMPTY;
    for (int b = threadIdx.x; b < nblocks; b += PF_NT) {
        PfMom u;
        pf_mom_load(partial + (size_t)b * PF_MOM, u);
        pf_mom_merge(&v, &u);
    }
    pf_mom_block_merge<PF_NT>(v, sm);
    if (threadIdx.x == 0) pf_mom_store(out, v);
}
// the shards' PfMom (one per rank, gathered) merged in rank order; est -> scal[4..7], cov -> scal[8..23] (row-major)
__global__ void pf_moments_final_kernel(PfDev d, const double* mom, int shards) {
    if (threadIdx.x != 0) return;
    PfMom v;
    pf_mom_load(mom, v);
    for (int r = 1; r < shards; ++r) {
        PfMom u;
        pf_mom_load(mom + (size_t)r * PF_MOM, u);
        pf_mom_merge(&v, &u);
    }
    pf_mom_final(&v, d.scal + 4, d.scal + 8);
}
