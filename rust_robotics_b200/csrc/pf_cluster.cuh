// pf_cluster.cuh — pose hypotheses of PF / MCL (include/pfgpu.h pfgpu_pf_hypotheses, DESIGN §3.10): the particle cloud clustered in
// a fixed (x, y, yaw) histogram, each cluster's mass, mean and covariance.  A query between steps, on the N particles of the
// (gathered) global set:
//   1. pf_clu_key_kernel      membership and bin key per particle
//      pf_clu_insert_kernel   the bin hash set of pf_kld.cuh; mint[slot] = the smallest member in the bin
//   2. pf_clu_link_kernel     connected components over the occupied slots: lock-free union-find, each slot probes 13 of its 26
//                             neighbours and links the root with the larger mint under the other, so a component's root is the slot
//                             of its smallest member, whatever the order of the links
//      pf_clu_label_kernel    label of every particle (N for a non-member)
//   3. a stable radix sort of (label, slot) and a run-length encoding: cluster j = the j-th label, its members in slot order.  Each
//      cluster is cut into tiles of PF_CLU_TILE sorted members; one warp sums a tile (lane-strided, then a fixed xor tree), one warp
//      sums a cluster's tiles the same way.  Pass 1 sums w, w x, w y, w v, w sin yaw, w cos yaw and the bins; pass 2 the centred
//      second moments.  The order of every sum depends on the sorted set alone: not on the grid, the timing or the rank.
//   4. a stable radix sort of the clusters by ~bits(mass) (masses are positive: descending mass, ties in label order); the first cap
//      clusters and the per-slot ranks go to the host.
#pragma once
#include "pf_kld.cuh"
#include <cub/cub.cuh>

#define PF_CLU_TILE 256            // sorted members per tile: one warp, 8 per lane
#define PF_CLU_V 10                // doubles per tile partial (pass 1 uses 7, pass 2 all 10)

struct PfClu {
    size_t cap = 0;                // particles it holds: world x the largest generation
    unsigned tcap = 0;             // hash slots: a power of two >= 2 cap + 16
    int* keys = nullptr;           // [3][cap] bin key of each particle
    int* slot = nullptr;           // [cap] its hash slot, -1 = not a member
    int* owner = nullptr;          // [tcap] hash set (pf_bin_insert)
    unsigned* mint = nullptr;      // [tcap] smallest member in the bin
    int* parent = nullptr;         // [tcap] union-find parent slot, -1 = root
    unsigned* lab = nullptr;       // [cap] label (N = not a member); later the per-slot ranks
    unsigned* lab_s = nullptr;     // [cap] sorted labels
    unsigned* iota = nullptr;      // [cap] 0, 1, ..
    unsigned* perm = nullptr;      // [cap] slot of each sorted position
    unsigned* cid = nullptr;       // [cap] cluster of each slot (members only)
    unsigned* uniq = nullptr;      // [cap] label of cluster j
    unsigned* cnt = nullptr;       // [cap] members of cluster j
    unsigned* off = nullptr;       // [cap] its first sorted position
    unsigned* toff = nullptr;      // [cap] its first tile
    unsigned* rank = nullptr;      // [cap] its rank
    unsigned* order = nullptr;     // [cap] cluster of rank r
    unsigned* scal = nullptr;      // [2] runs, clusters
    unsigned long long* mkey = nullptr;     // [cap] ~bits(mass) of cluster j
    unsigned long long* mkey_s = nullptr;
    pfgpu_pf_hypothesis* hyp = nullptr;     // [cap] cluster j, in label order
    double* part = nullptr;        // [cap + cap / PF_CLU_TILE + 1][24]: tile partials (PF_CLU_V per tile), then the ranked output
    double* w_all = nullptr;       // sharded: the gathered weights
    void* tmp = nullptr;           // CUB temporary storage
    size_t tmp_bytes = 0;
};

__device__ __forceinline__ bool pf_clu_finite(double v) { return v - v == 0.0; }
__device__ __forceinline__ const Pose4* pf_clu_pose(const PfDev& d, const Pose4* all) { return all ? all : pf_pose(d, *d.cur); }
__device__ __forceinline__ double pf_clu_wrap(double a) { return a - PFC_TWO_PI * floor((a + PFC_PI) / PFC_TWO_PI); }

__global__ void __launch_bounds__(PF_NT) pf_clu_key_kernel(PfDev d, const Pose4* P_all, const double* W_all, size_t N, PfClu c, double r,
                                                           double bw, int K) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= N) return;
    Pose4 p;
    pose_load(pf_clu_pose(d, P_all), t, p);
    const double w = W_all ? W_all[t] : d.w[t];
    const bool member = pf_clu_finite(p.x) && pf_clu_finite(p.y) && pf_clu_finite(p.yaw) && pf_clu_finite(p.v) && w > 0.0 && pf_clu_finite(w);
    c.slot[t] = member ? 0 : -1;
    if (!member) return;
    const double m = PFC_TWO_PI * floor(p.yaw / PFC_TWO_PI);
    const double theta = p.yaw - m;
    const double q = floor(theta / bw);
    c.keys[t] = pf_sat_i32(floor(p.x / r));
    c.keys[c.cap + t] = pf_sat_i32(floor(p.y / r));
    c.keys[2 * c.cap + t] = !(q >= 0.0) ? 0 : (q > (double)(K - 1) ? K - 1 : (int)q);
}

// The members of a warp that share a bin insert once, through their lowest lane (the smallest of their slots): a tracking cloud puts
// most particles in a few bins, and one atomic per particle on those few slots would serialise the launch.
__global__ void __launch_bounds__(PF_NT) pf_clu_insert_kernel(PfClu c, size_t N) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= N || c.slot[t] < 0) return;
    const int a = c.keys[t], b = c.keys[c.cap + t], k = c.keys[2 * c.cap + t];
    const unsigned act = __activemask();
    const unsigned same = __match_any_sync(act, ((unsigned long long)(unsigned)a << 32) | (unsigned)b) & __match_any_sync(act, k);
    const int lead = __ffs(same) - 1;
    unsigned i = 0;
    if ((int)(threadIdx.x & 31) == lead) {
        i = pf_bin_insert(c.owner, c.tcap, c.keys, c.cap, t, a, b, k);
        atomicMin(&c.mint[i], (unsigned)t);
    }
    i = __shfl_sync(same, i, lead);
    c.slot[t] = (int)i;
}

// root of slot x, halving the path on the way (every store replaces a parent by one of its ancestors)
__device__ __forceinline__ int pf_clu_find(int* par, int x) {
    volatile int* vp = par;
    for (;;) {
        const int p = vp[x];
        if (p < 0) return x;
        const int g = vp[p];
        if (g < 0) return p;
        vp[x] = g;
        x = g;
    }
}
__device__ __forceinline__ void pf_clu_unite(int* par, const unsigned* mint, int a, int b) {
    for (;;) {
        a = pf_clu_find(par, a);
        b = pf_clu_find(par, b);
        if (a == b) return;
        if (mint[a] > mint[b]) { const int s = a; a = b; b = s; }
        if (atomicCAS(par + b, -1, a) == -1) return;                 // b was still a root: it now hangs under a
    }
}

__global__ void __launch_bounds__(PF_NT) pf_clu_link_kernel(PfClu c, int K) {
    const unsigned s = blockIdx.x * PF_NT + threadIdx.x;
    if (s >= c.tcap) return;
    const int o = c.owner[s];
    if (o < 0) return;
    const int kx = c.keys[o], ky = c.keys[c.cap + o], kt = c.keys[2 * c.cap + o];
    const int tp = kt + 1 == K ? 0 : kt + 1, tm = kt == 0 ? K - 1 : kt - 1;
    // the 13 offsets (dx, dy, dt) that come after (0, 0, 0) in lexicographic order: every adjacent pair is probed from one side
    for (int q = 0; q < 13; ++q) {
        const int e = q + 14;                                        // 14 .. 26 = the codes 9 dx + 3 dy + dt + 13 > 13
        const int dx = e / 9 - 1, dy = (e / 3) % 3 - 1, dt = e % 3 - 1;
        if ((dx > 0 && kx == 2147483647) || (dy > 0 && ky == 2147483647) || (dy < 0 && ky == -2147483647 - 1)) continue;
        const int nb = pf_bin_find(c.owner, c.tcap, c.keys, c.cap, kx + dx, ky + dy, dt > 0 ? tp : (dt < 0 ? tm : kt));
        if (nb >= 0) pf_clu_unite(c.parent, c.mint, (int)s, nb);
    }
}

__global__ void __launch_bounds__(PF_NT) pf_clu_label_kernel(PfClu c, size_t N) {
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= N) return;
    const int s = c.slot[t];
    c.lab[t] = s < 0 ? (unsigned)N : c.mint[pf_clu_find(c.parent, s)];
    c.iota[t] = (unsigned)t;
}

// clusters = runs, less the run of non-members (label N, the largest)
__global__ void pf_clu_count_kernel(PfClu c, size_t N) {
    const unsigned runs = c.scal[0];
    c.scal[1] = runs - (runs > 0 && c.uniq[runs - 1] == (unsigned)N ? 1u : 0u);
}

struct PfCluTiles { __device__ __forceinline__ unsigned operator()(unsigned n) const { return (n + PF_CLU_TILE - 1) / PF_CLU_TILE; } };
// tiles of every cluster, into rank (free until the ranking); their exclusive sum is toff
__global__ void __launch_bounds__(PF_NT) pf_clu_ntiles_kernel(PfClu c, unsigned nc) {
    const unsigned j = blockIdx.x * PF_NT + threadIdx.x;
    if (j < nc) c.rank[j] = PfCluTiles()(c.cnt[j]);
}

template <int NV>
__device__ __forceinline__ void pf_clu_warp_sum(double (&a)[NV]) {
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a[k] += __shfl_xor_sync(0xffffffffu, a[k], o);
}
// the cluster of tile q: the last j with toff[j] <= q
__device__ __forceinline__ unsigned pf_clu_tile_owner(const unsigned* toff, unsigned nc, unsigned q) {
    unsigned lo = 0, hi = nc;
    while (hi - lo > 1) {
        const unsigned mid = lo + ((hi - lo) >> 1);
        if (toff[mid] <= q) lo = mid; else hi = mid;
    }
    return lo;
}

// one warp per tile.  PASS 1: w, w x, w y, w v, w sin yaw, w cos yaw, bins (a member that is its bin's mint); also cid when asked.
// PASS 2: w d_a d_b over the upper triangle of (x, y, wrapped yaw, v) deviations from the means pass 1 wrote into hyp.
template <int PASS>
__global__ void __launch_bounds__(PF_NT) pf_clu_tile_kernel(PfDev d, const Pose4* P_all, const double* W_all, PfClu c, unsigned nc, int want_cid) {
    constexpr int NV = PASS == 1 ? 7 : 10;
    const unsigned tiles = c.toff[nc - 1] + PfCluTiles()(c.cnt[nc - 1]);
    const unsigned lane = threadIdx.x & 31, warps = gridDim.x * (PF_NT / 32);
    const Pose4* P = pf_clu_pose(d, P_all);
    const double* W = W_all ? W_all : d.w;
    for (unsigned q = blockIdx.x * (PF_NT / 32) + (threadIdx.x >> 5); q < tiles; q += warps) {
        const unsigned j = pf_clu_tile_owner(c.toff, nc, q);
        const unsigned b = c.off[j] + (q - c.toff[j]) * PF_CLU_TILE, e = min(b + PF_CLU_TILE, c.off[j] + c.cnt[j]);
        double m[4] = {0.0, 0.0, 0.0, 0.0};
        if (PASS == 2) { const pfgpu_pf_hypothesis& h = c.hyp[j]; for (int k = 0; k < 4; ++k) m[k] = h.mean[k]; }
        double a[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) a[k] = 0.0;
        for (unsigned i = b + lane; i < e; i += 32) {
            const unsigned t = c.perm[i];
            Pose4 p;
            pose_load(P, t, p);
            const double w = W[t];
            if (PASS == 1) {
                double s, co;
                pfc_sincos(p.yaw, &s, &co);
                a[0] += w; a[1] += w * p.x; a[2] += w * p.y; a[3] += w * p.v; a[4] += w * s; a[5] += w * co;
                a[6] += c.mint[c.slot[t]] == t ? 1.0 : 0.0;
                if (want_cid) c.cid[t] = j;
            } else {
                const double e4[4] = { p.x - m[0], p.y - m[1], pf_clu_wrap(p.yaw - m[2]), p.v - m[3] };
                int k = 0;
#pragma unroll
                for (int u = 0; u < 4; ++u)
#pragma unroll
                    for (int v = u; v < 4; ++v) a[k++] += (w * e4[u]) * e4[v];
            }
        }
        pf_clu_warp_sum<NV>(a);
        if (lane == 0)
#pragma unroll
            for (int k = 0; k < NV; ++k) c.part[(size_t)q * PF_CLU_V + k] = a[k];
    }
}

// one warp per cluster: its tile partials in the same fixed order, then pass 1 the mass, means and counts, pass 2 the covariance
template <int PASS>
__global__ void __launch_bounds__(PF_NT) pf_clu_final_kernel(PfClu c, unsigned nc) {
    constexpr int NV = PASS == 1 ? 7 : 10;
    const unsigned lane = threadIdx.x & 31, warps = gridDim.x * (PF_NT / 32);
    for (unsigned j = blockIdx.x * (PF_NT / 32) + (threadIdx.x >> 5); j < nc; j += warps) {
        const unsigned b = c.toff[j], e = b + PfCluTiles()(c.cnt[j]);
        double a[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) a[k] = 0.0;
        for (unsigned q = b + lane; q < e; q += 32)
#pragma unroll
            for (int k = 0; k < NV; ++k) a[k] += c.part[(size_t)q * PF_CLU_V + k];
        pf_clu_warp_sum<NV>(a);
        if (lane != 0) continue;
        pfgpu_pf_hypothesis& h = c.hyp[j];
        if (PASS == 1) {
            const double M = a[0];
            h.mass = M;
            h.mean[0] = a[1] / M; h.mean[1] = a[2] / M;
            h.mean[2] = (a[4] == 0.0 && a[5] == 0.0) ? 0.0 : pfc_atan2(a[4], a[5]);
            h.mean[3] = a[3] / M;
            h.count = c.cnt[j]; h.bins = (uint64_t)a[6]; h.label = c.uniq[j];
            c.mkey[j] = ~(unsigned long long)pfc_d2u(M);
            c.iota[j] = j;
        } else {
            const double M = h.mass;
            int k = 0;
            for (int u = 0; u < 4; ++u)
                for (int v = u; v < 4; ++v, ++k) { const double x = a[k] / M; h.cov[v * 4 + u] = x; h.cov[u * 4 + v] = x; }
        }
    }
}

// rank of every cluster; the first m in rank order, as the host receives them, into part
__global__ void __launch_bounds__(PF_NT) pf_clu_rank_kernel(PfClu c, unsigned nc, unsigned m) {
    const unsigned r = blockIdx.x * PF_NT + threadIdx.x;
    if (r >= nc) return;
    const unsigned j = c.order[r];
    c.rank[j] = r;
    if (r < m) reinterpret_cast<pfgpu_pf_hypothesis*>(c.part)[r] = c.hyp[j];
}

// each local slot's cluster rank (UINT32_MAX: not a member), into lab
__global__ void __launch_bounds__(PF_NT) pf_clu_slot_rank_kernel(PfClu c, size_t offset, size_t n, unsigned nc) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= n) return;
    const size_t t = offset + i;
    c.lab[i] = (nc == 0 || c.slot[t] < 0) ? 0xFFFFFFFFu : c.rank[c.cid[t]];
}

// ---- host: the workspace, one allocation carved in 256-byte pieces, for `cap` particles (world x the largest generation) ----
static void pf_clu_free(PfClu& c) {
    cudaFree(c.keys);                                                // the allocation starts with keys
    c = PfClu{};
}
static size_t pf_clu_tmp_bytes(size_t cap) {
    size_t b[4] = {0, 0, 0, 0};
    const int n = (int)cap;
    unsigned* u = nullptr;
    unsigned long long* k = nullptr;
    cub::DeviceRadixSort::SortPairs(nullptr, b[0], u, u, u, u, n, 0, 32);
    cub::DeviceRunLengthEncode::Encode(nullptr, b[1], u, u, u, u, n);
    cub::DeviceScan::ExclusiveSum(nullptr, b[2], u, u, n);
    cub::DeviceRadixSort::SortPairs(nullptr, b[3], k, k, u, u, n, 0, 64);
    return std::max(std::max(b[0], b[1]), std::max(b[2], b[3]));
}
// the bytes pf_clu_alloc takes for cap particles (with the gathered weights of a sharded engine when `gathered`)
static size_t pf_clu_layout(PfClu& c, size_t cap, bool gathered, char* base) {
    unsigned tc = 64;
    while ((size_t)tc < 2 * cap + 16) tc <<= 1;
    size_t at = 0;
    auto take = [&](size_t bytes) -> void* { void* p = base ? base + at : nullptr; at += (bytes + 255) & ~(size_t)255; return p; };
    c.cap = cap; c.tcap = tc;
    c.keys = (int*)take(3 * cap * sizeof(int));
    c.slot = (int*)take(cap * sizeof(int));
    c.owner = (int*)take((size_t)tc * sizeof(int));
    c.mint = (unsigned*)take((size_t)tc * sizeof(unsigned));
    c.parent = (int*)take((size_t)tc * sizeof(int));
    unsigned** u32[] = { &c.lab, &c.lab_s, &c.iota, &c.perm, &c.cid, &c.uniq, &c.cnt, &c.off, &c.toff, &c.rank, &c.order };
    for (unsigned** p : u32) *p = (unsigned*)take(cap * sizeof(unsigned));
    c.scal = (unsigned*)take(2 * sizeof(unsigned));
    c.mkey = (unsigned long long*)take(cap * sizeof(unsigned long long));
    c.mkey_s = (unsigned long long*)take(cap * sizeof(unsigned long long));
    c.hyp = (pfgpu_pf_hypothesis*)take(cap * sizeof(pfgpu_pf_hypothesis));
    static_assert(sizeof(pfgpu_pf_hypothesis) == 24 * sizeof(double), "a ranked hypothesis takes 24 doubles of part");
    c.part = (double*)take((cap + cap / PF_CLU_TILE + 1) * 24 * sizeof(double));
    c.w_all = gathered ? (double*)take(cap * sizeof(double)) : nullptr;
    c.tmp_bytes = pf_clu_tmp_bytes(cap);
    c.tmp = take(c.tmp_bytes);
    return at;
}
static int pf_clu_alloc(PfClu& c, size_t cap, bool gathered) {
    const size_t bytes = pf_clu_layout(c, cap, gathered, nullptr);
    char* base = nullptr;
    const cudaError_t e = cudaMalloc(&base, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        c = PfClu{};
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "pose hypotheses: workspace of %zu bytes: %s", bytes, cudaGetErrorString(e));
        return PFGPU_ERR_CUDA;
    }
    pf_clu_layout(c, cap, gathered, base);
    return 0;
}
