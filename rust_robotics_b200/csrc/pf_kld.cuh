// pf_kld.cuh — MonteCarloLocalizer::resample_adaptive with min_particles < max_particles (mcl.rs:322-365): the number of
// particles of the NEXT generation depends on the draws themselves.
//
// The reference draws one particle at a time and stops at the first length `len` with
//     len >= min_particles  and  len >= required,   required = max over the draws so far of kld_required(k),
// k = number of distinct (x, y, yaw) histogram bins among the particles drawn so far (mcl.rs:343-355), or at max_particles.
// Draw t depends on nothing but the counter-based RNG, so all max_particles candidates are drawn in parallel, and the
// stopping length is recovered exactly:
//   1. pf_kld_draw_kernel     r_t, ancestor index (lower bound in the exact CDF, fallback len-1: mcl.rs:387-392), bin key
//   2. pf_kld_insert_kernel   open-addressing hash set of the keys with the smallest draw number per key
//                             -> draw t opens a new bin  <=>  it is that smallest number (independent of insertion order)
//   3. pf_kld_stop_kernel     k_t = prefix count of new bins, running max of kld_required(k_t), first t that satisfies the
//                             stop rule (one CTA walks chunks of 1024 draws and stops at the first hit)
//   4. pf_kld_gather_kernel   the first n_new candidates become the particle set, weights 1/n_new (mcl.rs:357-361)
// The host reads n_new once per step (the launch grids of the next step depend on it).
#pragma once
#include "pf_kernels.cuh"

struct PfKld {
    size_t cap = 0;             // max_particles
    int* keys = nullptr;        // [3][cap] quantised x, y, yaw of each candidate (mcl.rs:380-385)
    int* owner = nullptr;       // [tcap] hash slots: a draw number that carries the slot's key, -1 = empty
    unsigned* mint = nullptr;   // [tcap] smallest draw number with that key
    int* slot = nullptr;        // [cap] slot of candidate t
    unsigned* n_new = nullptr;  // device: length of the next generation
    unsigned tcap = 0;          // power of two >= 2 cap + 16
};

__device__ __forceinline__ int pf_sat_i32(double v) {          // Rust `as i32`: saturating, NaN -> 0
    if (v != v) return 0;
    if (v >= 2147483647.0) return 2147483647;
    if (v <= -2147483648.0) return (int)(-2147483647 - 1);
    return (int)v;
}

// `bad`: the scan of the cumulative weights saw a negative, infinite or NaN weight (xs flags[3]); then the CDF may go down or
// hold NaN, and each draw scans linearly as the reference does (pf_search_kernel)
__global__ void __launch_bounds__(PF_NT) pf_kld_draw_kernel(PfDev d, uint64_t seed, PfKld k, const int* bad) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= k.cap) return;
    const uint32_t call = d.counters[0];
    const double r = pfc_u01_53(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_PF_RESAMPLE, call, t), 0));
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
    const size_t index = lo < d.n ? lo : d.n - 1;              // sample_index mcl.rs:387-392
    d.idx[t] = (uint32_t)index;
    Pose4 p;
    pose_load(pf_pose(d, *d.cur), index, p);
    const double X_BIN = 0.5, Y_BIN = 0.5, YAW_BIN = 15.0 * PFC_PI / 180.0;     // mcl.rs:26-28
    k.keys[t] = pf_sat_i32(floor(p.x / X_BIN));                // quantize_particle mcl.rs:380-385
    k.keys[k.cap + t] = pf_sat_i32(floor(p.y / Y_BIN));
    k.keys[2 * k.cap + t] = pf_sat_i32(floor(p.yaw / YAW_BIN));
}

// The open-addressing bin hash set shared by the KLD resample and the pose hypotheses (pf_cluster.cuh).  keys = [3][cap]
// (x, y, yaw bin of item t at t, cap + t, 2 cap + t); owner[tcap] = an item that carries the slot's key, -1 = empty; tcap is a power
// of two at least twice the number of distinct keys, so a probe always meets an empty slot.
__device__ __forceinline__ unsigned pf_bin_hash(int a, int b, int c) {
    const unsigned long long h = (unsigned long long)(unsigned)a * 0x9E3779B97F4A7C15ull ^ (unsigned long long)(unsigned)b * 0xC2B2AE3D27D4EB4Full ^
                                 (unsigned long long)(unsigned)c * 0x165667B19E3779F9ull;
    return (unsigned)(h >> 17);
}
// insert item t with key (a, b, c); returns the slot that stands for the key
__device__ __forceinline__ unsigned pf_bin_insert(int* owner, unsigned tcap, const int* keys, size_t cap, size_t t, int a, int b, int c) {
    unsigned i = pf_bin_hash(a, b, c) & (tcap - 1);
    for (;;) {
        int o = atomicCAS(&owner[i], -1, (int)t);
        if (o == -1) break;                                    // the slot is mine: it now stands for my key
        if (keys[o] == a && keys[cap + o] == b && keys[2 * cap + o] == c) break;   // same bin
        i = (i + 1) & (tcap - 1);                              // another bin lives here (the table is never more than half full)
    }
    return i;
}
// the slot of key (a, b, c), -1 when no item carries it (the insertions have completed)
__device__ __forceinline__ int pf_bin_find(const int* owner, unsigned tcap, const int* keys, size_t cap, int a, int b, int c) {
    unsigned i = pf_bin_hash(a, b, c) & (tcap - 1);
    for (;;) {
        const int o = owner[i];
        if (o == -1) return -1;
        if (keys[o] == a && keys[cap + o] == b && keys[2 * cap + o] == c) return (int)i;
        i = (i + 1) & (tcap - 1);
    }
}

__global__ void __launch_bounds__(PF_NT) pf_kld_insert_kernel(PfKld k) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= k.cap) return;
    const int a = k.keys[t], b = k.keys[k.cap + t], c = k.keys[2 * k.cap + t];
    const unsigned i = pf_bin_insert(k.owner, k.tcap, k.keys, k.cap, t, a, b, c);
    atomicMin(&k.mint[i], (unsigned)t);
    k.slot[t] = (int)i;
}

// kld_required_particles mcl.rs:367-378 (IEEE sqrt / division / ceil: the same bits as on the host)
__device__ __forceinline__ unsigned long long pf_kld_required(unsigned long long k_bins, unsigned long long n_min, unsigned long long n_max, double eps, double z) {
    if (k_bins <= 1) return n_min;
    const double km1 = (double)(k_bins - 1);
    const double term = 1.0 - 2.0 / (9.0 * km1) + z * sqrt(2.0 / (9.0 * km1));
    const double nn = (km1 / (2.0 * eps)) * (term * term * term);
    const double cn = ceil(nn);
    unsigned long long v = (cn != cn || cn <= 0.0) ? 0ull : (cn >= 18446744073709551615.0 ? ~0ull : (unsigned long long)cn);   // `as usize`
    if (v < n_min) v = n_min;
    if (v > n_max) v = n_max;
    return v;
}

__global__ void __launch_bounds__(1024) pf_kld_stop_kernel(PfKld k, unsigned long long n_min, unsigned long long n_max, double eps, double z) {
    __shared__ int sm_i[32];
    __shared__ unsigned long long sm_m[32];
    __shared__ unsigned long long s_req;       // running max of kld_required over the draws of the previous chunks
    __shared__ int s_bins;                     // distinct bins in the previous chunks
    __shared__ unsigned s_hit;                 // smallest satisfying draw number in this chunk
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    if (tid == 0) { s_req = n_min; s_bins = 0; s_hit = 0xFFFFFFFFu; }
    __syncthreads();
    unsigned result = (unsigned)k.cap;         // the loop `while len < max` ends at max_particles
    for (size_t base = 0; base < k.cap; base += 1024) {
        const size_t t = base + tid;
        const int flag = (t < k.cap && k.mint[k.slot[t]] == (unsigned)t) ? 1 : 0;     // draw t opens a new bin
        int tot;
        const int ex = block_excl_scan_int<1024>(flag, &tot, sm_i);
        const unsigned long long bins = (unsigned long long)(s_bins + ex + flag);
        unsigned long long req = t < k.cap ? pf_kld_required(bins, n_min, n_max, eps, z) : 0ull;
        // inclusive running max over the block (required = required.max(kld_required(k)), mcl.rs:349-350)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { unsigned long long y = __shfl_up_sync(0xffffffffu, req, o); if (lane >= o && y > req) req = y; }
        __syncthreads();
        if (lane == 31) sm_m[wid] = req;
        __syncthreads();
        unsigned long long pre = s_req;
        for (int w = 0; w < wid; ++w) if (sm_m[w] > pre) pre = sm_m[w];
        if (pre > req) req = pre;
        const unsigned long long len = (unsigned long long)t + 1ull;
        if (t < k.cap && len >= n_min && len >= req) atomicMin(&s_hit, (unsigned)t);  // mcl.rs:352-354
        __syncthreads();
        if (s_hit != 0xFFFFFFFFu) { result = s_hit + 1u; break; }
        if (tid == 1023) { s_req = req; s_bins += tot; }
        __syncthreads();
    }
    if (tid == 0) *k.n_new = result;
}

__global__ void __launch_bounds__(PF_NT) pf_kld_gather_kernel(PfDev d, PfKld k) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    const unsigned n_new = *k.n_new;
    if (t >= n_new) return;
    const int cur = *d.cur;
    Pose4 p;
    pose_load(pf_pose(d, cur), d.idx[t], p);
    pose_store(pf_pose(d, cur ^ 1), t, p);
    d.w[t] = 1.0 / (double)n_new;                              // mcl.rs:357-361
}
