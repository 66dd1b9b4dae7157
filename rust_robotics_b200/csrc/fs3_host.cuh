// fs3_host.cuh — host side of the FastSLAM 1.0 engine (kernels: fs3.cuh): the pfgpu_fs_* entry points of include/pfgpu.h.
// Included by pfgpu.cu after the shared helpers (Ctx, Marks, KernelTimer, PF_NCCL, ...).
#pragma once
#include "fs3.cuh"
#include "fs3_est.cuh"
#include "fs3_assoc.cuh"
#include "fs3_hist.cuh"
#include "fs3_exist.cuh"

struct pfgpu_fs {
    Ctx ctx;
    pfgpu_fs_config cfg;
    uint64_t seed = 0;
    Fs3Dev d = {};
    uint32_t n_step = 0;
    uint64_t steps = 0;
    int world = 1, rank = 0;
    KernelTimer timer;
    Marks marks;
    char* arena = nullptr; size_t arena_bytes = 0;
    void* peer_ptr[FS3_MAXG] = {};
    ncclComm_t comm = nullptr;
    Fs3Rec* h_rec = nullptr;          // pinned + mapped
    double* stage = nullptr; size_t stage_bytes = 0;   // device staging buffer for upload / download / seed_map
    bool pdl = true;
    bool early = false;               // PFGPU_EARLY_LAUNCH=1: release the dependent kernel at the START of the previous grid (experiment;
                                      // off by default)
    bool ekf_attr[2] = { false, false };
    int variant = 1;                  // 1 = FastSLAM 1.0 (fs1.rs), 2 = FastSLAM 2.0 (fs2.rs); pfgpu_fs_set_variant
    int ekf_helpers = 0;              // PFGPU_EKF_HELPERS: cap on the helper warps per CTA (0 = as many as fit, at most 3)
    int post_nt = 256; unsigned post_K = 1, post_tiles = 1, m32 = 0; int log2n = -1; size_t post_smem = 0;
    bool post_global = false;         // the post kernel keeps its weight tiles in global memory (fs3_post_kernel<512, true>) ...
    double* vtile = nullptr;          // ... here: [post_tiles][post_K][512]
    bool post_k1 = false;             // fs3_post_kernel<512, false, 1>: one weight and at most one local slot per thread (PFGPU_POST_K1=0: off)
    char* est = nullptr; size_t est_bytes = 0;   // pfgpu_fs_moments scratch, allocated by the first call (fs3_est.cuh)
    double* zbuf = nullptr; size_t zcap = 0;     // pfgpu_fs_step_unknown: the (d, angle) list of the step (grows, never shrinks)
    unsigned long long* acnt = nullptr;         // [8] association counters: this launch's, then the last unknown step's (fs3_assoc.cuh);
                                                // [6]: copies removed by the last tracked unknown step (fs3_exist.cuh)
    pfgpu_fs* sib[FS3_MAXG] = {};               // in-process sharded engine: every rank's handle (pfgpu_fs_create_sharded_local)
    char* hist = nullptr; size_t hist_cap = 0;  // path history ring (fs3_hist.cuh), pfgpu_fs_history_enable
    uint64_t hist_first = 0;                    // oldest entry held (a root); the newest is `steps`
    void* hist_peer[FS3_MAXG] = {};             // peers' rings mapped through cudaIpc (one process per GPU)
    char* hs = nullptr; size_t hs_bytes = 0;    // path / path-moments scratch, grows on demand
    int* ex = nullptr; double ex_range = 0.0;   // landmark existence counters [2][m][ld] and their range (fs3_exist.cuh), pfgpu_fs_existence_enable
    void* ex_peer[FS3_MAXG] = {};               // peers' counters mapped through cudaIpc (one process per GPU)
    double odom_alpha[4] = { PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT };   // DESIGN §3.15
};
static int fs_hist_record(pfgpu_fs* h, int root);
static int fs_ex_fill(pfgpu_fs* h);
static int fs_ex_param(pfgpu_fs* h, Fs3Ex* X);

extern "C" void pfgpu_fs_default_config(pfgpu_fs_config* c) {            // fs1.rs:13-23
    c->dt = 0.1; c->max_range = 20.0; c->nth = 100.0 / 1.5; c->q00 = 0.3; c->q11 = 0.0305; c->r00 = 0.5; c->r11 = 0.0305;
    c->init_weight = 1.0 / 100.0;
}

template <int NT, bool GTILE, int KC = 0>
static int fs3_post_prepare(pfgpu_fs* h) {
    if (cudaFuncSetAttribute(fs3_post_kernel<NT, GTILE, KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)h->post_smem) != cudaSuccess) { cudaGetLastError(); return 1; }
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fs3_post_kernel<NT, GTILE, KC>, NT, h->post_smem) != cudaSuccess) { cudaGetLastError(); return 1; }
    return (size_t)nb * (size_t)h->ctx.num_sms >= h->post_tiles ? 0 : 1;
}

static int fs_stage(pfgpu_fs* h, size_t bytes) {
    if (bytes <= h->stage_bytes) return 0;
    if (h->stage) { cudaFree(h->stage); h->stage = nullptr; h->stage_bytes = 0; }
    PF_CUDA(cudaMalloc(&h->stage, bytes));
    h->stage_bytes = bytes;
    return 0;
}

// every rank's `bytes` from `mine` into all[world] over the handle's communicator (one process per GPU)
static int fs_allgather(pfgpu_fs* h, const void* mine, size_t bytes, void* all, const char* what) {
    char* buf = nullptr;
    PF_CUDA(cudaMalloc(&buf, (size_t)(h->world + 1) * bytes));
    int rc = 0;
    if (cudaMemcpy(buf + (size_t)h->world * bytes, mine, bytes, cudaMemcpyHostToDevice) != cudaSuccess) rc = PFGPU_ERR_CUDA;
    else if (ncclAllGather(buf + (size_t)h->world * bytes, buf, bytes, ncclChar, h->comm, h->ctx.stream) != ncclSuccess) rc = PFGPU_ERR_NCCL;
    else if (cudaStreamSynchronize(h->ctx.stream) != cudaSuccess || cudaMemcpy(all, buf, (size_t)h->world * bytes, cudaMemcpyDeviceToHost) != cudaSuccess)
        rc = PFGPU_ERR_CUDA;
    if (rc) { cudaGetLastError(); snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s: the exchange between ranks failed", what); }
    cudaFree(buf);
    return rc;
}
// closes the cudaIpc mappings of peers' buffers (this rank's own entry is never a mapping)
static void fs_unmap(const pfgpu_fs* h, void* opened[FS3_MAXG]) {
    for (int g = 0; g < FS3_MAXG; ++g) if (g != h->rank && opened[g]) { cudaIpcCloseMemHandle(opened[g]); opened[g] = nullptr; }
}
// One process per GPU: maps this rank's allocation `mine` on every peer rank through cudaIpc, and opened[g] <- rank g's for every
// peer g.  Collective; every rank returns the same outcome, and on failure nothing stays mapped: PFGPU_ERR_CUDA if some rank's
// allocation failed (ok = 0), PFGPU_ERR_INVALID if the ranks' tags differ, PFGPU_ERR_UNSUPPORTED if an allocation cannot be
// exported or mapped, the exchange's own code if that failed.  The second exchange is also a fence: what every rank wrote to its
// allocation before the call is there before any rank returns.
static int fs_share(pfgpu_fs* h, void* mine, int ok, uint64_t tag, void* opened[FS3_MAXG], const char* what) {
    struct Rec { cudaIpcMemHandle_t hd; uint64_t tag; int ok, pad; } me, all[FS3_MAXG];
    memset(&me, 0, sizeof(me));
    if (ok && cudaIpcGetMemHandle(&me.hd, mine) == cudaSuccess) ok = 2;       // 2: shared, 1: no cudaIpc export, 0: no allocation
    else cudaGetLastError();
    me.tag = tag; me.ok = ok;
    int rc = fs_allgather(h, &me, sizeof(me), all, what);
    if (rc) return rc;
    bool same = true;
    for (int g = 0; g < h->world; ++g) { ok = std::min(ok, all[g].ok); same = same && all[g].tag == tag; }
    if (!ok || !same) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), !ok ? "%s: the allocation failed on some rank" : "%s: every rank must pass the same size (%llu here)",
                 what, (unsigned long long)tag);
        return !ok ? PFGPU_ERR_CUDA : PFGPU_ERR_INVALID;
    }
    int mapped = ok == 2, maps[FS3_MAXG];
    for (int g = 0; g < h->world && mapped; ++g)
        if (g != h->rank && cudaIpcOpenMemHandle(&opened[g], all[g].hd, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
            mapped = 0; opened[g] = nullptr; cudaGetLastError();
        }
    rc = fs_allgather(h, &mapped, sizeof(int), maps, what);
    for (int g = 0; g < h->world && !rc; ++g) mapped = mapped && maps[g];
    if (rc || !mapped) {
        fs_unmap(h, opened);
        if (!rc) snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s: mapping a peer's copy through cudaIpc failed (sharded FastSLAM needs peer "
                          "access between all GPUs)", what);
        return rc ? rc : PFGPU_ERR_UNSUPPORTED;
    }
    return 0;
}
// rank g's copy of a per-rank buffer: this rank's own, an in-process sibling's (sib), or the cudaIpc mapping (one process per GPU)
template <class T>
static T* fs_rank_buf(const pfgpu_fs* h, int g, T* pfgpu_fs::*own, void* const* mapped) {
    const pfgpu_fs* o = g == h->rank ? h : h->sib[g];
    return o ? o->*own : static_cast<T*>(mapped[g]);
}

static int fs_create_impl(const pfgpu_fs_config* cfg, size_t n, size_t n_global, size_t offset, size_t m, uint64_t seed, int device,
                          const void* uid, int rank, int world, pfgpu_fs** out) {
    if (!out) return PFGPU_ERR_INVALID;
    *out = nullptr;
    if (!cfg || n == 0 || n_global >= (1ull << 28) * (size_t)world || n >= (1ull << 28) || n_global > 0xFFFFFFF0ull) return PFGPU_ERR_INVALID;
    if (m > FS3_MAX_LM) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "more than %d landmarks per particle are not supported", FS3_MAX_LM); return PFGPU_ERR_UNSUPPORTED; }
    if (world > 1 && n % 64 != 0) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "sharded FastSLAM needs a multiple of 64 particles per GPU"); return PFGPU_ERR_UNSUPPORTED; }
    pfgpu_fs* h = new (std::nothrow) pfgpu_fs();
    if (!h) return PFGPU_ERR_CUDA;
    int rc = ctx_open(h->ctx, device);
    if (rc) { delete h; return rc; }
    h->cfg = *cfg; h->seed = seed; h->world = world; h->rank = rank;
    Fs3Dev& d = h->d;
    const size_t ld = (n + 63) / 64 * 64, mm = m ? m : 1;
    d.n = (unsigned)n; d.n_glob = (unsigned)n_global; d.off = (unsigned)offset; d.m = (unsigned)m; d.ld = (unsigned)ld;
    d.G = world; d.rank = rank; d.npart = (unsigned)(ld / 64); d.wait_inline = 1;
    auto fail = [&](int code) { pfgpu_fs_destroy(h); return code; };
#define FS_TRY(x) do { cudaError_t e__ = (x); if (e__ != cudaSuccess) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s -> %s", #x, cudaGetErrorString(e__)); return fail(PFGPU_ERR_CUDA); } } while (0)
    // post kernel shape: <= 128 tiles (one CTA each, co-resident), NT threads x K values
    {
        // below 65 536 weights: up to 128 tiles of 256 threads (latency matters, not throughput); at 65 536: 128 tiles of 512 threads,
        // one value per thread; beyond that the per-value phases (classify, normalise, emit: ~100 instructions per value and sum)
        // dominate, so every SM gets a tile of 512 threads
        const char* env = getenv("PFGPU_POST_NT");
        const bool big = n_global > (size_t)128 * 256 * 2;
        h->post_nt = env ? (atoi(env) == 512 ? 512 : 256) : (n_global >= (size_t)128 * 512 ? 512 : 256);
        unsigned want = (unsigned)std::min<int>(big ? FS3_MAX_TILES : 128, h->ctx.num_sms);
        { const char* ew = getenv("PFGPU_POST_TILES"); if (ew && atoi(ew) >= 1 && atoi(ew) <= (int)want) want = (unsigned)atoi(ew); }   // tests: several values per thread at small n
        unsigned K = (unsigned)((n_global + (size_t)want * h->post_nt - 1) / ((size_t)want * h->post_nt));
        if (K == 0) K = 1;
        h->post_K = K;
        h->post_tiles = (unsigned)((n_global + (size_t)h->post_nt * K - 1) / ((size_t)h->post_nt * K));
        h->post_smem = (size_t)h->post_nt * K * sizeof(double);
        h->m32 = x3_margin32(n_global);
        h->log2n = -1;
        for (int p = 0; p < 32; ++p) if (((size_t)1 << p) == n_global) h->log2n = p;
        // PFGPU_POST_SMEM_CAP=<bytes> (tests): the most dynamic shared memory the weight tile may take (default: what the device allows)
        const char* ec = getenv("PFGPU_POST_SMEM_CAP");
        const bool capped = ec && ec[0] && (size_t)strtoull(ec, nullptr, 10) < h->post_smem;
        int bad = capped || (h->post_nt == 512 ? fs3_post_prepare<512, false>(h) : fs3_post_prepare<256, false>(h));
        if (bad || h->post_tiles > FS3_MAX_TILES || h->post_tiles > (unsigned)h->post_nt) {
            // the tile does not fit on chip: one tile of 512 threads per SM, its K x 512 weights in global memory (vtile)
            h->post_global = true;
            h->post_nt = 512;
            unsigned tiles = (unsigned)std::min<int>(FS3_MAX_TILES, h->ctx.num_sms);
            { const char* ew = getenv("PFGPU_POST_TILES"); if (ew && atoi(ew) >= 1 && atoi(ew) <= (int)tiles) tiles = (unsigned)atoi(ew); }
            K = (unsigned)((n_global + (size_t)tiles * 512 - 1) / ((size_t)tiles * 512));
            h->post_K = K;
            h->post_tiles = (unsigned)((n_global + (size_t)512 * K - 1) / ((size_t)512 * K));
            h->post_smem = 0;
            if (fs3_post_prepare<512, true>(h)) {
                snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "the post-step kernel cannot keep %u CTAs co-resident on this device", h->post_tiles);
                return fail(PFGPU_ERR_UNSUPPORTED);
            }
        }
        // the shape config 3 runs (2^16 weights on one GPU: 128 tiles x 512 threads x 1) has a kernel compiled for it, with less code
        // on the path of every step; it needs one value per thread and at most one local slot per thread.  Should it not fit where
        // the generic kernel does, the generic kernel (the same results) runs.
        const char* ek = getenv("PFGPU_POST_K1");
        if (!(ek && ek[0] == '0') && !h->post_global && h->post_nt == 512 && h->post_K == 1 && n <= (size_t)h->post_tiles * 512)
            h->post_k1 = fs3_post_prepare<512, false, 1>(h) == 0;
    }
    // ONE allocation for everything a peer may touch, same layout on every rank: one IPC mapping per peer exposes all of it
    {
        size_t off = 0;
        auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
        d.o_flags = take(2 * FS3_MAXG * 128);
        const size_t ngp = (size_t)world * ld + 64;
        for (int b = 0; b < 2; ++b) { d.o_wraw[b] = take(ngp * sizeof(double)); d.o_part[b] = take((size_t)world * d.npart * sizeof(double)); }
        for (int b = 0; b < 2; ++b) { d.o_px[b] = take(ld * sizeof(double)); d.o_py[b] = take(ld * sizeof(double)); d.o_pyaw[b] = take(ld * sizeof(double)); }
        for (int b = 0; b < 2; ++b) d.o_rows[b] = take(mm * ld * sizeof(unsigned));
        const size_t small = off;
        for (int b = 0; b < 2; ++b) d.o_lm[b] = take(mm * 6 * ld * sizeof(double));
        h->arena_bytes = off;
        FS_TRY(cudaMalloc(&h->arena, off));
        FS_TRY(cudaMemset(h->arena, 0, small));
        FS_TRY(cudaMemset(h->arena + d.o_lm[0], 0, mm * 6 * ld * sizeof(double)));
        FS_TRY(cudaMemset(h->arena + d.o_lm[1], 0, mm * 6 * ld * sizeof(double)));
        char* A = h->arena;
        for (int b = 0; b < 2; ++b) {
            d.px[b] = (double*)(A + d.o_px[b]); d.py[b] = (double*)(A + d.o_py[b]); d.pyaw[b] = (double*)(A + d.o_pyaw[b]);
            d.lm[b] = (double*)(A + d.o_lm[b]); d.rows[b] = (unsigned*)(A + d.o_rows[b]);
            d.wraw[b] = (double*)(A + d.o_wraw[b]); d.part[b] = (double*)(A + d.o_part[b]);
        }
        d.peer[rank] = A; h->peer_ptr[rank] = A;
    }
    {
        FS_TRY(fs3_sum_alloc(d.x, (unsigned)n_global, getenv("PFGPU_POST_TRACE") != nullptr));
        FS_TRY(cudaMalloc(&d.lmst, mm * sizeof(int))); FS_TRY(cudaMemset(d.lmst, 0, mm * sizeof(int)));
        FS_TRY(cudaMalloc(&d.w, ld * sizeof(double))); FS_TRY(cudaMemset(d.w, 0, ld * sizeof(double)));
        for (int b = 0; b < 2; ++b) { FS_TRY(cudaMalloc(&d.nz[b], ld * sizeof(double))); FS_TRY(cudaMemset(d.nz[b], 0, ld * sizeof(double))); }
        FS_TRY(cudaMalloc(&d.wn_all, (n_global + 64) * sizeof(double)));
        FS_TRY(cudaMalloc(&d.cum_all, (n_global + 64) * sizeof(double)));
        if (h->log2n < 0) FS_TRY(cudaMalloc(&d.rcomb_all, (n_global + 64) * sizeof(double)));
        FS_TRY(cudaMalloc(&d.idx, ld * sizeof(unsigned))); FS_TRY(cudaMemset(d.idx, 0, ld * sizeof(unsigned)));
        d.st = d.x.st; d.x.raw[0] = d.wraw[0]; d.x.raw[1] = d.wraw[1]; d.x.wn = d.wn_all;
        const size_t nbm = (size_t)2 * fs3_bm_ld((unsigned)m);       // both parities start clear; each post kernel clears the other
        FS_TRY(cudaMalloc(&d.rowbm, nbm * sizeof(unsigned))); FS_TRY(cudaMemset(d.rowbm, 0, nbm * sizeof(unsigned)));
        FS_TRY(cudaMalloc(&d.tileBw, FS3_MAX_TILES * sizeof(double))); FS_TRY(cudaMalloc(&d.tileBi, FS3_MAX_TILES * sizeof(unsigned)));
        FS_TRY(cudaHostAlloc(&h->h_rec, sizeof(Fs3Rec), cudaHostAllocMapped));
        memset(h->h_rec, 0, sizeof(Fs3Rec));
        FS_TRY(cudaHostGetDevicePointer((void**)&d.rec, h->h_rec, 0));
        if (h->post_global) FS_TRY(cudaMalloc(&h->vtile, (size_t)h->post_tiles * h->post_K * 512 * sizeof(double)));
    }
    { const char* e5 = getenv("PFGPU_PDL"); h->pdl = !(e5 && e5[0] == '0'); }
    { const char* e7 = getenv("PFGPU_EARLY_LAUNCH"); if (e7 && atoi(e7) == 1) h->early = true; }
    { const char* e6 = getenv("PFGPU_EKF_HELPERS"); if (e6 && atoi(e6) >= 1 && atoi(e6) <= 3) h->ekf_helpers = atoi(e6); }
    { const char* e8 = getenv("PFGPU_FS_EXACT_CDF"); d.exact_cdf = e8 && atoi(e8) == 1 ? 1 : 0; }   // A/B: every resample runs the exact S2 and CDF sums
    if (world > 1 && uid) {
        ncclUniqueId id;
        memcpy(&id, uid, sizeof(id));
        ncclResult_t nr = ncclCommInitRank(&h->comm, world, id, rank);
        if (nr != ncclSuccess) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "ncclCommInitRank: %s", ncclGetErrorString(nr)); return fail(PFGPU_ERR_NCCL); }
        // map every peer's arena; the second exchange is also the "everybody has zeroed and mapped" fence
        rc = fs_share(h, h->arena, 1, 0, h->peer_ptr, "FastSLAM arena");
        if (rc) return fail(rc);
        for (int g = 0; g < world; ++g) d.peer[g] = (char*)h->peer_ptr[g];
    }
#undef FS_TRY
    fs3_init_kernel<<<cdiv_u(n, 256), 256, 0, h->ctx.stream>>>(d, cfg->init_weight);
    h->ctx.launches += 1;
    if (cudaStreamSynchronize(h->ctx.stream) != cudaSuccess) return fail(PFGPU_ERR_CUDA);
    *out = h;
    return PFGPU_OK;
}
extern "C" int pfgpu_fs_create(const pfgpu_fs_config* cfg, size_t n, size_t m, uint64_t seed, int device, pfgpu_fs** out) {
    return fs_create_impl(cfg, n, n, 0, m, seed, device, nullptr, 0, 1, out);
}
extern "C" int pfgpu_fs_create_sharded(const pfgpu_fs_config* cfg, size_t n_global, size_t m, uint64_t seed, int device,
                                       const void* uid, int rank, int world, pfgpu_fs** out) {
    if (out) *out = nullptr;
    if (!uid || world < 1 || world > FS3_MAXG || rank < 0 || rank >= world || n_global == 0 || n_global % (size_t)world != 0)
        return PFGPU_ERR_INVALID;
    size_t nl = n_global / (size_t)world;
    return fs_create_impl(cfg, nl, n_global, (size_t)rank * nl, m, seed, device, uid, rank, world, out);
}
// All ranks in ONE process (one host thread drives them, no NCCL): peers are plain device pointers (same device) or
// peer-access pointers (different devices).
extern "C" int pfgpu_fs_create_sharded_local(const pfgpu_fs_config* cfg, size_t n_global, size_t m, uint64_t seed, const int* devices,
                                             int world, pfgpu_fs** out) {
    if (!out || !devices || world < 1 || world > FS3_MAXG || n_global == 0 || n_global % (size_t)world != 0) return PFGPU_ERR_INVALID;
    for (int r = 0; r < world; ++r) out[r] = nullptr;
    const size_t nl = n_global / (size_t)world;
    static const char dummy_uid = 0;
    for (int r = 0; r < world; ++r) {
        int rc = fs_create_impl(cfg, nl, n_global, (size_t)r * nl, m, seed, devices[r], world > 1 ? nullptr : &dummy_uid, r, world, &out[r]);
        if (rc) { for (int q = 0; q < r; ++q) { pfgpu_fs_destroy(out[q]); out[q] = nullptr; } return rc; }
    }
    for (int a = 0; a < world; ++a)
        for (int b = 0; b < world; ++b) {
            if (devices[a] != devices[b]) {
                cudaSetDevice(devices[a]);
                cudaError_t e = cudaDeviceEnablePeerAccess(devices[b], 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
                    snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "no peer access from device %d to device %d", devices[a], devices[b]);
                    for (int q = 0; q < world; ++q) { pfgpu_fs_destroy(out[q]); out[q] = nullptr; }
                    return PFGPU_ERR_UNSUPPORTED;
                }
                cudaGetLastError();
            }
            out[a]->d.peer[b] = out[b]->arena;
            out[a]->sib[b] = out[b];
            if (a != b && devices[a] == devices[b]) out[a]->d.wait_inline = 0;     // ranks sharing a GPU must not hold SMs while they wait
        }
    return PFGPU_OK;
}
extern "C" void pfgpu_fs_destroy(pfgpu_fs* h) {
    if (!h) return;
    cudaSetDevice(h->ctx.device);
    if (h->ctx.stream) cudaStreamSynchronize(h->ctx.stream);
    Fs3Dev& d = h->d;
    fs_unmap(h, h->peer_ptr);                      // (local mode: none were opened)
    fs_unmap(h, h->hist_peer);
    fs_unmap(h, h->ex_peer);
    cudaFree(h->arena);
    cudaFree(d.lmst); cudaFree(d.w); cudaFree(d.nz[0]); cudaFree(d.nz[1]); cudaFree(d.wn_all); cudaFree(d.cum_all); cudaFree(d.rcomb_all); cudaFree(d.idx);
    fs3_sum_free(d.x);
    cudaFree(d.rowbm); cudaFree(d.tileBw); cudaFree(d.tileBi); cudaFree(h->vtile); cudaFree(h->stage); cudaFree(h->est);
    cudaFree(h->zbuf); cudaFree(h->acnt);
    cudaFree(h->hist); cudaFree(h->hs); cudaFree(h->ex);
    if (h->h_rec) cudaFreeHost(h->h_rec);
    if (h->comm) ncclCommDestroy(h->comm);
    marks_free(h->marks);
    for (auto& p : h->timer.pending) { cudaEventDestroy(p.first); cudaEventDestroy(p.second); }
    if (h->ctx.stream) cudaStreamDestroy(h->ctx.stream);
    delete h;
}
static int fs_check_err(pfgpu_fs* h) {        // device-side time-outs are sticky and surface at the next synchronising call
    if (h->h_rec && h->h_rec->err) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "FastSLAM step: a barrier or a peer GPU timed out (sticky; destroy the handle)");
        return PFGPU_ERR_CUDA;
    }
    return 0;
}
extern "C" int pfgpu_fs_sync(pfgpu_fs* h) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return fs_check_err(h);
}
extern "C" int pfgpu_fs_count(pfgpu_fs* h, size_t* nl, size_t* ng, size_t* m) {
    if (!h) return PFGPU_ERR_INVALID;
    if (nl) *nl = h->d.n;
    if (ng) *ng = h->d.n_glob;
    if (m) *m = h->d.m;
    return 0;
}
static const size_t FS_XFER_CHUNK_BYTES = (size_t)256 << 20;   // staging chunk for AoS<->SoA conversion
extern "C" int pfgpu_fs_upload(pfgpu_fs* h, const double* pose_w, const double* lm, size_t n) {
    if (!h || !pose_w || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    int rc = fs_stage(h, n * 4 * sizeof(double));
    if (rc) return rc;
    PF_CUDA(cudaMemcpyAsync(h->stage, pose_w, n * 4 * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    PF_LAUNCH(h->ctx, fs3_unpack_pose_kernel, cdiv_u(n, 256), 256, 0, d, h->stage);
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (lm && d.m) {
        const size_t per = (size_t)d.m * 6 * sizeof(double);
        size_t chunk = std::max<size_t>(1, FS_XFER_CHUNK_BYTES / per);
        if (chunk > n) chunk = n;
        rc = fs_stage(h, chunk * per);
        if (rc) return rc;
        for (size_t i0 = 0; i0 < n; i0 += chunk) {
            const size_t cnt = std::min(chunk, n - i0);
            PF_CUDA(cudaMemcpyAsync(h->stage, lm + i0 * d.m * 6, cnt * per, cudaMemcpyHostToDevice, h->ctx.stream));
            PF_LAUNCH(h->ctx, fs3_unpack_lm_kernel, cdiv_u(cnt * d.m * 6, 256), 256, 0, d, h->stage, i0, cnt);
            PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        }
        PF_LAUNCH(h->ctx, fs3_lmst_reset_kernel, 1, 256, 0, d);
    }
    if (h->ex) { rc = fs_ex_fill(h); if (rc) return rc; }       // every existence counter restarts at 1
    return h->hist ? fs_hist_record(h, 1) : 0;       // the uploaded state restarts the path history window
}
extern "C" int pfgpu_fs_download(pfgpu_fs* h, double* pose_w, double* lm, size_t n) {
    if (!h || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    if (pose_w) {
        int rc = fs_stage(h, n * 4 * sizeof(double));
        if (rc) return rc;
        PF_LAUNCH(h->ctx, fs3_pack_pose_kernel, cdiv_u(n, 256), 256, 0, d, h->stage);
        PF_CUDA(cudaMemcpyAsync(pose_w, h->stage, n * 4 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    if (lm && d.m) {
        const size_t per = (size_t)d.m * 6 * sizeof(double);
        size_t chunk = std::max<size_t>(1, FS_XFER_CHUNK_BYTES / per);
        if (chunk > n) chunk = n;
        int rc = fs_stage(h, chunk * per);
        if (rc) return rc;
        for (size_t i0 = 0; i0 < n; i0 += chunk) {
            const size_t cnt = std::min(chunk, n - i0);
            PF_LAUNCH(h->ctx, fs3_pack_lm_kernel, cdiv_u(cnt * d.m * 6, 256), 256, 0, d, h->stage, i0, cnt);
            PF_CUDA(cudaMemcpyAsync(lm + i0 * d.m * 6, h->stage, cnt * per, cudaMemcpyDeviceToHost, h->ctx.stream));
            PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        }
    }
    return fs_check_err(h);
}

extern "C" int pfgpu_fs_seed_map(pfgpu_fs* h, const double pose3[3], const double* lm_xy, size_t m, double sigma, double cov0) {
    if (!h || !pose3 || (m && !lm_xy) || m != h->d.m) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    PF_LAUNCH(h->ctx, fs3_seed_pose_kernel, cdiv_u(d.n, 256), 256, 0, d, pose3[0], pose3[1], pose3[2]);
    if (h->hist) { int rc = fs_hist_record(h, 1); if (rc) return rc; }      // the seeded state restarts the path history window
    if (m) {
        int rc = fs_stage(h, m * 2 * sizeof(double));
        if (rc) return rc;
        PF_CUDA(cudaMemcpyAsync(h->stage, lm_xy, m * 2 * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
        dim3 grid(cdiv_u(d.n, 256), (unsigned)std::min<size_t>(m, 65535));
        PF_LAUNCH(h->ctx, fs3_seed_lm_kernel, grid, 256, 0, d, h->stage, sigma, cov0, h->seed);
        PF_LAUNCH(h->ctx, fs3_lmst_reset_kernel, 1, 256, 0, d);
        if (h->ex) { rc = fs_ex_fill(h); if (rc) return rc; }   // every existence counter restarts at 1
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    return 0;
}

template <int MAXT>
static int fs3_launch_ekf(pfgpu_fs* h, const Fs3ObsParam& po, const double u[2], int kk, int flags) {
    const Fs3Dev& d = h->d;
    // helper warps (predict ahead / weights behind): as many as fit the CTA beside the kk EKF warps, at most 3
    int nh = kk > 0 ? std::min(3, MAXT / 32 - kk) : 1;
    if (h->ekf_helpers > 0 && kk > 0) nh = std::min(nh, h->ekf_helpers);
    const unsigned threads = 32u * (unsigned)(kk + nh);
    auto smem_of = [](int k, int n) { return ((size_t)n * 192 + (size_t)n * k * 64 + (size_t)2 * k * 384) * sizeof(double); };
    const size_t smem = smem_of(kk, nh);
    const unsigned groups = d.ld / 64;
    // persistent: one CTA per SM walks the 64-particle groups; without observations the launch is predict-only and latency
    // bound, so every group gets its own (one-warp) CTA
    const unsigned grid = kk > 0 ? std::min<unsigned>(groups, (unsigned)h->ctx.num_sms) : groups;
    if (!h->ekf_attr[MAXT == 512 ? 0 : 1]) {
        size_t mx = 0;
        for (int k = 0; k < MAXT / 32; ++k) mx = std::max(mx, smem_of(k, std::min(3, MAXT / 32 - k)));
        PF_CUDA(cudaFuncSetAttribute(fs3_ekf_kernel<MAXT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)mx));
        h->ekf_attr[MAXT == 512 ? 0 : 1] = true;
    }
    PF_LAUNCH_PDL(h->ctx, h->pdl, (fs3_ekf_kernel<MAXT>), grid, threads, smem, d, po, u[0], u[1], h->cfg.dt, sqrt(h->cfg.q00), sqrt(h->cfg.q11),
                  h->cfg.r00, h->cfg.r11, h->seed, (uint32_t)h->n_step, kk, flags, (unsigned)h->n_step);
    return 0;
}

// The end of step h->n_step, from the host-side signal / wait pair on.  The post kernel normalises, evaluates the N_eff gate and
// (when it opens) runs the whole resample in one launch; po / k_last: the last EKF launch's observations, whose lazy-clone
// bookkeeping the post kernel applies (k_last = 0: none).
static int fs_step_end(pfgpu_fs* h, const Fs3ObsParam& po, int k_last, bool host_waits, int* did) {
    const Fs3Dev& d = h->d;
    if (host_waits) {      // the post kernel signals "my weights are pushed" itself; the wait for the others' is its own launch here
        PF_LAUNCH(h->ctx, fs3_signal_kernel, 1, 32, 0, d, 0, (unsigned)h->n_step + 1u);
        PF_LAUNCH(h->ctx, fs3_wait_kernel, 1, 32, 0, d, 0, (unsigned)h->n_step + 1u);
    }
    auto post = h->post_global ? fs3_post_kernel<512, true> : h->post_k1 ? fs3_post_kernel<512, false, 1>
              : h->post_nt == 512 ? fs3_post_kernel<512, false> : fs3_post_kernel<256, false>;
    PF_LAUNCH_PDL(h->ctx, h->pdl, post, h->post_tiles, h->post_nt, h->post_smem, d, po, k_last, h->cfg.nth, h->seed, (unsigned)h->n_step, h->post_K,
                  h->m32, h->log2n, h->early && h->pdl && !host_waits ? 1 : 0, h->vtile);
    h->n_step++;
    h->steps++;
    if (h->hist) { int rc = fs_hist_record(h, 0); if (rc) return rc; }      // entry `steps` of the path history (one launch)
    if (did) {     // the gate lives on the device; only a caller who asks pays a sync
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        *did = h->h_rec->gate;
        return fs_check_err(h);
    }
    return 0;
}

// One known-id step.  om == nullptr: the velocity model with control u; otherwise the odometry increment om (DESIGN §3.15), whose
// predict (fs3_odom_predict_kernel) or proposal (fs2_propose_odom_kernel) runs ahead of the EKF launch, which then runs with flags
// bit 1 (poses already this step's).
static int fs_step_impl(pfgpu_fs* h, const double u[2], const PfOdom* om, const pfgpu_fs_obs* z, size_t k, int* did) {
    if (h->ex) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "landmark existence counters are enabled: known-id steps are not supported (the EKF launch "
                 "moves landmarks without their counters); disable them with pfgpu_fs_existence_enable(h, 0) first");
        return PFGPU_ERR_UNSUPPORTED;
    }
    Fs3Dev& d = h->d;
    for (size_t j = 0; j < k; ++j) {
        if (!finite_d(z[j].d) || !finite_d(z[j].angle)) return PFGPU_ERR_INVALID;
        if (z[j].lm_id >= d.m) return PFGPU_ERR_INVALID;             // the reference would panic on the Vec index (fs1.rs:141)
    }
    PF_CUDA(cudaSetDevice(h->ctx.device));
    // One EKF launch runs one warp per observation and the lazy-clone bookkeeping is per launch, so a launch must not see the
    // same lm_id twice and holds at most FS3_MAX_OBS observations: the list is cut before every repeated id / every
    // FS3_MAX_OBS entries and the pieces run as consecutive launches (same per-particle order as fs1.rs:250-256).
    std::vector<size_t> cuts;
    cuts.push_back(0);
    {
        std::vector<uint64_t> seen;
        for (size_t j = 0; j < k; ++j) {
            bool dup = seen.size() >= FS3_MAX_OBS;
            for (uint64_t v : seen) if (v == z[j].lm_id) { dup = true; break; }
            if (dup) { cuts.push_back(j); seen.clear(); }
            seen.push_back(z[j].lm_id);
        }
    }
    cuts.push_back(k);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (h->timer.on) { PF_CUDA(cudaEventCreate(&e0)); PF_CUDA(cudaEventCreate(&e1)); PF_CUDA(cudaEventRecord(e0, h->ctx.stream)); }
    const size_t nseg = cuts.size() - 1;
    Fs3ObsParam po;
    int k_last = 0;
    const bool host_waits = d.G > 1 && !d.wait_inline;
    if (host_waits) PF_LAUNCH(h->ctx, fs3_wait_kernel, 1, 32, 0, d, 1, (unsigned)h->n_step);            // peers' previous post kernels are over
    const bool proposed = h->variant == 2 && k > 0;
    if (proposed) {        // FastSLAM 2.0: sample every pose from the proposal of the first observation (fs2.rs:341-346)
        Fs3Obs ob0; ob0.d = z[0].d; ob0.angle = z[0].angle; ob0.lm_id = (int)z[0].lm_id;
        if (om)
            PF_LAUNCH_PDL(h->ctx, h->pdl, fs2_propose_odom_kernel, cdiv_u(d.n, 128), 128, 0, d, ob0, *om, h->cfg.r00, h->cfg.r11,
                          h->seed, (uint32_t)h->n_step, (unsigned)h->n_step);
        else
            PF_LAUNCH_PDL(h->ctx, h->pdl, fs2_propose_kernel, cdiv_u(d.n, 128), 128, 0, d, ob0, u[0], u[1], h->cfg.dt, h->cfg.r00, h->cfg.r11,
                          h->seed, (uint32_t)h->n_step, (unsigned)h->n_step);
    } else if (om)
        PF_LAUNCH_PDL(h->ctx, h->pdl, fs3_odom_predict_kernel, cdiv_u(d.n, 128), 128, 0, d, *om, h->seed, (uint32_t)h->n_step, (unsigned)h->n_step);
    const bool moved = proposed || om;
    for (size_t seg = 0; seg < nseg; ++seg) {
        const size_t j0 = cuts[seg], kk = cuts[seg + 1] - cuts[seg];
        // (ranks that share a GPU take turns on its SMs through the wait / signal launches: parked early CTAs of one rank could keep
        // another rank's persistent CTAs from ever being scheduled, so nothing is released early there)
        const int flags = (seg == 0 ? 1 : 0) | (moved ? 2 : 0) | (h->variant == 2 ? 4 : 0) | (h->early && h->pdl && !host_waits ? 8 : 0);
        memset(&po, 0, sizeof(po));
        for (size_t j = 0; j < kk; ++j) { po.o[j].d = z[j0 + j].d; po.o[j].angle = z[j0 + j].angle; po.o[j].lm_id = (int)z[j0 + j].lm_id; }
        int rc = kk <= 15 ? fs3_launch_ekf<512>(h, po, u, (int)kk, flags) : fs3_launch_ekf<1024>(h, po, u, (int)kk, flags);
        if (rc) return rc;
        if (seg + 1 < nseg) PF_LAUNCH_PDL(h->ctx, h->pdl, fs3_mark_kernel, 1, 64, 0, d, po, (int)kk);    // the last piece: the post kernel does it
        k_last = (int)kk;
    }
    if (h->timer.on) { PF_CUDA(cudaEventRecord(e1, h->ctx.stream)); h->timer.pending.push_back({e0, e1}); }
    return fs_step_end(h, po, k_last, host_waits, did);
}
extern "C" int pfgpu_fs_step(pfgpu_fs* h, const double u[2], const pfgpu_fs_obs* z, size_t k, int* did) {
    if (!h || !u || (k && !z)) return PFGPU_ERR_INVALID;
    if (!finite_d(u[0]) || !finite_d(u[1])) return PFGPU_ERR_INVALID;
    return fs_step_impl(h, u, nullptr, z, k, did);
}
extern "C" int pfgpu_fs_step_odom(pfgpu_fs* h, const double odom[6], const pfgpu_fs_obs* z, size_t k, int* did) {
    if (!h || !odom || (k && !z)) return PFGPU_ERR_INVALID;
    PfOdom om;
    if (pf_odom_increment(odom, h->odom_alpha, &om) != 0) return PFGPU_ERR_INVALID;
    const double u0[2] = { 0.0, 0.0 };            // unused: the EKF launch runs no motion model after the odometry move
    return fs_step_impl(h, u0, &om, z, k, did);
}
extern "C" int pfgpu_fs_set_odom_noise(pfgpu_fs* h, const double alpha[4]) {
    if (!h || !alpha || !pf_odom_alpha_ok(alpha)) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) h->odom_alpha[j] = alpha[j];
    return 0;
}
extern "C" int pfgpu_fs_odom_noise(pfgpu_fs* h, double alpha[4]) {
    if (!h || !alpha) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) alpha[j] = h->odom_alpha[j];
    return 0;
}
// the association counters [8] (fs3_assoc.cuh), allocated and cleared on the handle's stream by the first call that needs them
static int fs_acnt(pfgpu_fs* h) {
    if (h->acnt) return 0;
    PF_CUDA(cudaMalloc(&h->acnt, 8 * sizeof(unsigned long long)));
    PF_CUDA(cudaMemsetAsync(h->acnt, 0, 8 * sizeof(unsigned long long), h->ctx.stream));
    return 0;
}
// FastSLAM 2.0 with unknown data association (DESIGN §3.5): fs3_assoc_kernel, the lazy-clone bookkeeping, then the post kernel
// (om: the odometry increment in place of u, as in fs_step_impl; the caller has checked h, the variant and the motion)
static int fs_step_unknown_impl(pfgpu_fs* h, const double u[2], const PfOdom* om, const double* z2, size_t k, double gate_d2, int* did) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    int rc = fs_acnt(h);
    if (rc) return rc;
    Fs3Ex X = {};            // zero without existence counters
    if (h->ex) { rc = fs_ex_param(h, &X); if (rc) return rc; }
    if (k == 0 && !h->ex) {  // no observation: the known-id step with k = 0, bit for bit; nothing was associated
        PF_CUDA(cudaMemsetAsync(h->acnt + 3, 0, 3 * sizeof(unsigned long long), h->ctx.stream));
        return fs_step_impl(h, u, om, nullptr, 0, did);
    }
    if (k && 2 * k > h->zcap) {  // (the previous step may still read the old list: wait for it before the buffer goes)
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        cudaFree(h->zbuf); h->zbuf = nullptr; h->zcap = 0;
        const size_t cap = std::max<size_t>(64, 4 * k);
        PF_CUDA(cudaMalloc(&h->zbuf, cap * sizeof(double)));
        h->zcap = cap;
    }
    // stream-ordered behind every kernel of the previous step, so a list is never overwritten while a step reads it
    if (k) PF_CUDA(cudaMemcpyAsync(h->zbuf, z2, 2 * k * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    const bool host_waits = d.G > 1 && !d.wait_inline;
    if (host_waits) PF_LAUNCH(h->ctx, fs3_wait_kernel, 1, 32, 0, d, 1, (unsigned)h->n_step);            // peers' previous post kernels are over
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (h->timer.on) { PF_CUDA(cudaEventCreate(&e0)); PF_CUDA(cudaEventCreate(&e1)); PF_CUDA(cudaEventRecord(e0, h->ctx.stream)); }
    // with existence counters (DESIGN §3.7), acnt[6] collects this step's removals
    if (h->ex) PF_CUDA(cudaMemsetAsync(h->acnt + 6, 0, sizeof(unsigned long long), h->ctx.stream));
    if (om)
        PF_LAUNCH(h->ctx, (h->ex ? fs3_assoc_odom_kernel<true> : fs3_assoc_odom_kernel<false>), cdiv_u(d.ld, FS3_ASSOC_NT), FS3_ASSOC_NT, 0, d,
                  (const double*)h->zbuf, (int)k, gate_d2, *om, h->cfg.r00, h->cfg.r11, h->seed, (uint32_t)h->n_step, (unsigned)h->n_step,
                  h->acnt, X, h->ex ? h->acnt + 6 : nullptr);
    else
        PF_LAUNCH(h->ctx, (h->ex ? fs3_assoc_kernel<true> : fs3_assoc_kernel<false>), cdiv_u(d.ld, FS3_ASSOC_NT), FS3_ASSOC_NT, 0, d,
                  (const double*)h->zbuf, (int)k, gate_d2, u[0], u[1], h->cfg.dt, h->cfg.r00, h->cfg.r11, h->seed, (uint32_t)h->n_step, (unsigned)h->n_step,
                  h->acnt, X, sqrt(h->cfg.q00), sqrt(h->cfg.q11), h->ex ? h->acnt + 6 : nullptr);
    if (h->timer.on) { PF_CUDA(cudaEventRecord(e1, h->ctx.stream)); h->timer.pending.push_back({e0, e1}); }
    PF_LAUNCH_PDL(h->ctx, h->pdl, fs3_assoc_mark_kernel, std::max(1u, std::min(cdiv_u(d.m, 256), 64u)), 256, 0, d, h->acnt);
    Fs3ObsParam po;
    memset(&po, 0, sizeof(po));
    return fs_step_end(h, po, 0, host_waits, did);
}
static int fs_unknown_variant_ok(pfgpu_fs* h) {
    if (h->variant == 2) return 1;
    snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "unknown data association needs FastSLAM 2.0 (pfgpu_fs_set_variant(h, 2)): FastSLAM 1.0 "
             "never initialises a fresh landmark's covariance, so a landmark it adds could never be matched");
    return 0;
}
extern "C" int pfgpu_fs_step_unknown(pfgpu_fs* h, const double u[2], const double* z2, size_t k, double gate_d2, int* did) {
    if (!h || !u || (k && !z2)) return PFGPU_ERR_INVALID;
    if (!fs_unknown_variant_ok(h)) return PFGPU_ERR_UNSUPPORTED;
    if (!finite_d(u[0]) || !finite_d(u[1]) || !(gate_d2 > 0.0)) return PFGPU_ERR_INVALID;      // gate_d2 = +inf is allowed
    for (size_t j = 0; j < 2 * k; ++j) if (!finite_d(z2[j])) return PFGPU_ERR_INVALID;
    return fs_step_unknown_impl(h, u, nullptr, z2, k, gate_d2, did);
}
extern "C" int pfgpu_fs_step_unknown_odom(pfgpu_fs* h, const double odom[6], const double* z2, size_t k, double gate_d2, int* did) {
    if (!h || !odom || (k && !z2)) return PFGPU_ERR_INVALID;
    if (!fs_unknown_variant_ok(h)) return PFGPU_ERR_UNSUPPORTED;
    PfOdom om;
    if (pf_odom_increment(odom, h->odom_alpha, &om) != 0 || !(gate_d2 > 0.0)) return PFGPU_ERR_INVALID;
    for (size_t j = 0; j < 2 * k; ++j) if (!finite_d(z2[j])) return PFGPU_ERR_INVALID;
    const double u0[2] = { 0.0, 0.0 };
    return fs_step_unknown_impl(h, u0, &om, z2, k, gate_d2, did);
}
extern "C" int pfgpu_fs_assoc_counts(pfgpu_fs* h, uint64_t counts[3]) {
    if (!h || !counts) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    unsigned long long c[3] = { 0ull, 0ull, 0ull };
    if (h->acnt) PF_CUDA(cudaMemcpy(c, h->acnt + 3, sizeof(c), cudaMemcpyDeviceToHost));
    for (int j = 0; j < 3; ++j) counts[j] = (uint64_t)c[j];
    return fs_check_err(h);
}

// ---------------------------------------------------------------------------------------------------------------------
// landmark existence counters (DESIGN §3.7): pfgpu_fs_existence_enable / _counts / _removed
// ---------------------------------------------------------------------------------------------------------------------
static size_t fs_ex_words(const pfgpu_fs* h) { return (size_t)2 * (h->d.m ? h->d.m : 1) * h->d.ld; }
static int fs_ex_fill(pfgpu_fs* h) {
    const size_t words = fs_ex_words(h);
    PF_LAUNCH(h->ctx, fs3_ex_fill_kernel, (unsigned)std::min<size_t>(cdiv_u(words, 256), 4096), 256, 0, h->ex, words);
    return 0;
}
// every rank's counters: own, the siblings' (in-process ranks) or the IPC mappings (one process per GPU)
static int fs_ex_param(pfgpu_fs* h, Fs3Ex* X) {
    memset(X, 0, sizeof(*X));
    X->range = h->ex_range;
    for (int g = 0; g < h->world; ++g) {
        int* b = fs_rank_buf(h, g, &pfgpu_fs::ex, h->ex_peer);
        if (!b) {
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "landmark existence counters: rank %d has not enabled them (pfgpu_fs_existence_enable is "
                     "made on every rank)", g);
            return PFGPU_ERR_INVALID;
        }
        X->base[g] = b;
    }
    return 0;
}
static void fs_ex_release(pfgpu_fs* h) {
    fs_unmap(h, h->ex_peer);
    cudaFree(h->ex); h->ex = nullptr; h->ex_range = 0.0;
}

extern "C" int pfgpu_fs_existence_enable(pfgpu_fs* h, double range) {
    if (!h || std::isnan(range) || range < 0.0) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));               // nothing in flight still reads the old counters
    if (range == 0.0) { fs_ex_release(h); return 0; }
    int rc = fs_acnt(h);
    if (rc) return rc;
    PF_CUDA(cudaMemsetAsync(h->acnt + 6, 0, sizeof(unsigned long long), h->ctx.stream));
    if (h->ex) {            // re-enabling: the same storage (and mappings), every counter back to 1
        h->ex_range = range;
        rc = fs_ex_fill(h);
        if (rc) return rc;
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        return 0;
    }
    // every counter is 1 before the exchange below, so before any rank can step
    int ok = cudaMalloc(&h->ex, fs_ex_words(h) * sizeof(int)) == cudaSuccess;
    if (!ok) {
        h->ex = nullptr; cudaGetLastError();
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "landmark existence counters: %zu bytes do not fit in device memory", fs_ex_words(h) * sizeof(int));
    } else ok = fs_ex_fill(h) == 0 && cudaStreamSynchronize(h->ctx.stream) == cudaSuccess;
    // one process per GPU: every rank maps every peer's counters once
    rc = h->comm ? fs_share(h, h->ex, ok, 0, h->ex_peer, "landmark existence counters") : ok ? 0 : PFGPU_ERR_CUDA;
    if (rc) { fs_ex_release(h); return rc; }
    h->ex_range = range;
    return 0;
}
extern "C" int pfgpu_fs_existence_counts(pfgpu_fs* h, size_t first_local, size_t count, int32_t* out) {
    if (!h || !h->ex || (count && !out) || first_local > h->d.n || count > h->d.n - first_local) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    if (!count || !d.m) return 0;
    Fs3Ex X;
    int rc = fs_ex_param(h, &X);
    if (rc) return rc;
    const size_t per = (size_t)d.m * sizeof(int);
    size_t chunk = std::max<size_t>(1, FS_XFER_CHUNK_BYTES / per);
    if (chunk > count) chunk = count;
    rc = fs_stage(h, chunk * per);
    if (rc) return rc;
    for (size_t i0 = 0; i0 < count; i0 += chunk) {
        const size_t cnt = std::min(chunk, count - i0);
        PF_LAUNCH(h->ctx, fs3_ex_pack_kernel, cdiv_u(cnt * d.m, 256), 256, 0, d, X, reinterpret_cast<int*>(h->stage), first_local + i0, cnt);
        PF_CUDA(cudaMemcpyAsync(out + i0 * d.m, h->stage, cnt * per, cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    return fs_check_err(h);
}
extern "C" int pfgpu_fs_existence_removed(pfgpu_fs* h, uint64_t* removed) {
    if (!h || !removed) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    unsigned long long c = 0ull;
    if (h->ex && h->acnt) PF_CUDA(cudaMemcpy(&c, h->acnt + 6, sizeof(c), cudaMemcpyDeviceToHost));
    *removed = (uint64_t)c;
    return fs_check_err(h);
}
extern "C" int pfgpu_fs_set_variant(pfgpu_fs* h, int variant) {
    if (!h || (variant != 1 && variant != 2)) return PFGPU_ERR_INVALID;
    h->variant = variant;
    return 0;
}
extern "C" int pfgpu_fs_best(pfgpu_fs* h, size_t* index, double pose_w4[4]) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    const Fs3Rec* r = h->h_rec;
    if (h->steps == 0) {        // no step yet: every weight equals init_weight, the last particle wins (fs1.rs:269-274)
        if (index) *index = (size_t)h->d.n_glob - 1;
        if (pose_w4) { pose_w4[0] = h->cfg.init_weight; pose_w4[1] = pose_w4[2] = pose_w4[3] = 0.0; }
        return 0;
    }
    if (index) *index = (size_t)r->best_idx;
    if (pose_w4) { pose_w4[0] = r->best_w; pose_w4[1] = r->bx; pose_w4[2] = r->by; pose_w4[3] = r->byaw; }
    return fs_check_err(h);
}
extern "C" int pfgpu_fs_particle_landmarks(pfgpu_fs* h, size_t il, double* lm6) {
    if (!h || !lm6 || il >= h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Fs3Dev& d = h->d;
    if (!d.m) return 0;
    int rc = fs_stage(h, (size_t)d.m * 6 * sizeof(double));
    if (rc) return rc;
    PF_LAUNCH(h->ctx, fs3_pack_lm_kernel, cdiv_u((size_t)d.m * 6, 256), 256, 0, d, h->stage, il, (size_t)1);
    PF_CUDA(cudaMemcpyAsync(lm6, h->stage, (size_t)d.m * 6 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_fs_last_indices(pfgpu_fs* h, uint32_t* idx, size_t cap, size_t* n) {
    if (!h || !idx) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (!h->h_rec->gate) { if (n) *n = 0; return 0; }         // the last step did not resample: no ancestry (as the oracle reports)
    size_t c = cap < h->d.n ? cap : h->d.n;
    PF_CUDA(cudaMemcpyAsync(idx, h->d.idx, c * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (n) *n = c;
    return 0;
}
extern "C" int pfgpu_fs_last_neff(pfgpu_fs* h, double* neff) {
    if (!h || !neff) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    *neff = h->h_rec->neff;
    return 0;
}
// get_observations fs1.rs:277-299 on the device: out (capacity n_landmarks) receives the observed (d, angle, lm_id) tuples
extern "C" int pfgpu_fs_get_observations(pfgpu_fs* h, const double x_true[3], const double* landmarks_xy, size_t n_landmarks, uint32_t call,
                                         pfgpu_fs_obs* out, size_t* k) {
    if (!h || !x_true || (n_landmarks && (!landmarks_xy || !out)) || !k) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    *k = 0;
    if (!n_landmarks) return 0;
    const size_t bytes_xy = n_landmarks * 2 * sizeof(double), bytes_out = n_landmarks * sizeof(Fs3Obs);
    int rc = fs_stage(h, bytes_xy + bytes_out + 256);
    if (rc) return rc;
    char* base = reinterpret_cast<char*>(h->stage);
    double* dxy = reinterpret_cast<double*>(base);
    Fs3Obs* dob = reinterpret_cast<Fs3Obs*>(base + ((bytes_xy + 15) & ~(size_t)15));
    unsigned* dk = reinterpret_cast<unsigned*>(base + ((bytes_xy + 15) & ~(size_t)15) + bytes_out);
    PF_CUDA(cudaMemcpyAsync(dxy, landmarks_xy, bytes_xy, cudaMemcpyHostToDevice, h->ctx.stream));
    PF_LAUNCH(h->ctx, fs3_get_observations_kernel, 1, 1024, 0, x_true[0], x_true[1], x_true[2], dxy, (unsigned)n_landmarks, h->cfg.max_range,
              sqrt(h->cfg.r00), sqrt(h->cfg.r11), h->seed, call, dob, dk);
    std::vector<Fs3Obs> tmp(n_landmarks);
    unsigned kk = 0;
    PF_CUDA(cudaMemcpyAsync(&kk, dk, sizeof(unsigned), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(tmp.data(), dob, bytes_out, cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    for (unsigned j = 0; j < kk; ++j) { out[j].d = tmp[j].d; out[j].angle = tmp[j].angle; out[j].lm_id = (uint64_t)tmp[j].lm_id; }
    *k = kk;
    return 0;
}
extern "C" int pfgpu_fs_last_gate(pfgpu_fs* h, int* did) {
    if (!h || !did) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    *did = h->steps ? h->h_rec->gate : 0;
    return fs_check_err(h);
}
extern "C" int pfgpu_fs_stats(pfgpu_fs* h, pfgpu_stats* s) {
    if (!h || !s) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    memset(s, 0, sizeof(*s));
    timer_drain(h->timer);
    Fs3State st;
    PF_CUDA(cudaMemcpy(&st, h->d.st, sizeof(st), cudaMemcpyDeviceToHost));
    s->kernel_launches = h->ctx.launches; s->steps = h->steps; s->resamples = st.resamples;
    s->main_kernel_ms_sum = h->timer.ms_sum; s->main_kernel_count = h->timer.count;
    s->serial_fallbacks = (uint64_t)st.serial_walks + (uint64_t)st.cert_fail;
    s->xsum_dirty_last = (uint64_t)st.dirty_last;
    return 0;
}
extern "C" int pfgpu_fs_shard_mode(pfgpu_fs* h, int* mode) {
    if (!h || !mode) return PFGPU_ERR_INVALID;
    *mode = h->world <= 1 ? 0 : 2;
    return 0;
}
// debug: accumulated phase times of the post kernel (PFGPU_POST_TRACE=1)
extern "C" int pfgpu_fs_post_trace(pfgpu_fs* h, unsigned long long* out32) {
    if (!h || !out32) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    for (int k = 0; k < 32; ++k) out32[k] = 0;
    if (h->d.x.trace) PF_CUDA(cudaMemcpy(out32, h->d.x.trace, 32 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    out32[31] = h->steps;
    {                     // [11] resamples that ran the exact S2 and CDF sums instead of the certified CDF
        Fs3State st;
        PF_CUDA(cudaMemcpy(&st, h->d.st, sizeof(st), cudaMemcpyDeviceToHost));
        out32[11] = (unsigned long long)st.cdf_exact;
    }
    // step timeline [ns], folded into the free slot pairs: [7] idle before the EKF launch, [24..26] EKF launch, idle between the
    // launches, post launch
    if (h->d.x.trace) {
        unsigned long long t8[9] = {};
        PF_CUDA(cudaMemcpy(t8, h->d.x.trace + 32, 9 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        out32[7] = t8[0]; out32[24] = t8[1]; out32[25] = t8[2]; out32[26] = t8[3]; out32[27] = t8[8];
    }
    return 0;
}
extern "C" int pfgpu_fs_post_shape(pfgpu_fs* h, unsigned* tiles, unsigned* threads, unsigned* values_per_thread, int* global_tile) {
    if (!h) return PFGPU_ERR_INVALID;
    if (tiles) *tiles = h->post_tiles;
    if (threads) *threads = (unsigned)h->post_nt;
    if (values_per_thread) *values_per_thread = h->post_K;
    if (global_tile) *global_tile = h->post_global ? 1 : 0;
    return 0;
}
extern "C" int pfgpu_fs_post_k1(pfgpu_fs* h, int* k1) {
    if (!h || !k1) return PFGPU_ERR_INVALID;
    *k1 = h->post_k1 ? 1 : 0;
    return 0;
}
extern "C" int pfgpu_fs_time_main_kernel(pfgpu_fs* h, int on) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    timer_drain(h->timer);
    h->timer.on = on != 0; h->timer.ms_sum = 0.0; h->timer.count = 0;
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// estimate (DESIGN §3.4): pfgpu_fs_moments on the device, pfgpu_fs_estimate_merge on the host
// ---------------------------------------------------------------------------------------------------------------------
static_assert(sizeof(pfgpu_fs_lm_moments) == sizeof(Fs3LmMom), "pfgpu_fs_lm_moments is Fs3LmMom");
static_assert(sizeof(pfgpu_fs_pose_moments) == sizeof(double) * 3 + sizeof(Fs3PoseMom), "pfgpu_fs_pose_moments: w, c[3], mean[3], m2[6]");
static_assert(sizeof(Fs3PoseMom) == FS3_EST_POSE_SUMS * sizeof(double) && FS3_EST_POSE_MAX_BLOCKS <= FS3_EST_NT, "pose partials");

// chunks of the map pass: enough (chunk, landmark) warps to fill the GPU, at least 32 slots per chunk, and at most
// FS3_EST_SCRATCH_CAP bytes of chunk partials; depends on (n, m) only
static void fs3_est_shape(size_t n, size_t m, unsigned* chunk, unsigned* nchunks) {
    size_t nc = (FS3_EST_TARGET_WARPS + m - 1) / m;
    nc = std::min(nc, (n + 31) / 32);
    nc = std::min(nc, std::max<size_t>(1, FS3_EST_SCRATCH_CAP / (m * sizeof(Fs3LmMom))));
    if (nc < 1) nc = 1;
    const size_t ch = ((n + nc - 1) / nc + 31) / 32 * 32;
    *chunk = (unsigned)ch;
    *nchunks = (unsigned)((n + ch - 1) / ch);
}

extern "C" int pfgpu_fs_moments(pfgpu_fs* h, double cov00_max, pfgpu_fs_pose_moments* pose, pfgpu_fs_lm_moments* lm) {
    if (!h || !pose || std::isnan(cov00_max)) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));          // (a time-out of the last step surfaces here)
    int rc = fs_check_err(h);
    if (rc) return rc;
    const Fs3Dev& d = h->d;
    const bool map = lm && d.m;
    unsigned chunk = 0, nch = 0;
    if (map) fs3_est_shape(d.n, d.m, &chunk, &nch);
    const unsigned pblocks = std::min<unsigned>(cdiv_u(d.n, 4 * FS3_EST_NT), FS3_EST_POSE_MAX_BLOCKS);
    // scratch: ticket | pose block partials | pose moments | map chunk partials | map moments
    const size_t o_part = 256, o_pose = o_part + (size_t)FS3_EST_POSE_MAX_BLOCKS * FS3_EST_POSE_SUMS * sizeof(double), o_lmp = o_pose + 256;
    const size_t o_lmo = o_lmp + (map ? (size_t)d.m * nch * sizeof(Fs3LmMom) : 0), need = o_lmo + (map ? (size_t)d.m * sizeof(Fs3LmMom) : 0);
    if (need > h->est_bytes) {
        if (h->est) { cudaFree(h->est); h->est = nullptr; h->est_bytes = 0; }
        PF_CUDA(cudaMalloc(&h->est, need));
        PF_CUDA(cudaMemset(h->est, 0, 256));
        h->est_bytes = need;
    }
    char* E = h->est;
    PF_LAUNCH(h->ctx, fs3_est_pose_kernel, pblocks, FS3_EST_NT, 0, d, reinterpret_cast<Fs3PoseMom*>(E + o_part), reinterpret_cast<unsigned*>(E),
              reinterpret_cast<double*>(E + o_pose));
    if (map) {
        dim3 grid(nch, cdiv_u(d.m, FS3_EST_NT / 32));
        PF_LAUNCH(h->ctx, fs3_est_map_kernel, grid, FS3_EST_NT, 0, d, cov00_max, chunk, reinterpret_cast<Fs3LmMom*>(E + o_lmp));
        PF_LAUNCH(h->ctx, fs3_est_merge_kernel, cdiv_u(d.m, FS3_EST_NT / 32), FS3_EST_NT, 0, reinterpret_cast<const Fs3LmMom*>(E + o_lmp), nch, d.m,
                  reinterpret_cast<Fs3LmMom*>(E + o_lmo));
        PF_CUDA(cudaMemcpyAsync(lm, E + o_lmo, (size_t)d.m * sizeof(Fs3LmMom), cudaMemcpyDeviceToHost, h->ctx.stream));
    }
    PF_CUDA(cudaMemcpyAsync(pose, E + o_pose, sizeof(*pose), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return fs_check_err(h);
}

extern "C" int pfgpu_fs_estimate_merge(const pfgpu_fs_pose_moments* pose, const pfgpu_fs_lm_moments* const* lm, int world, size_t m,
                                       double pose_mean3[3], double pose_cov9_colmajor[9], double* lm_mass, double* lm_mean2, double* lm_cov4) {
    if (!pose || world < 1) return PFGPU_ERR_INVALID;
    for (int g = 0; g < world; ++g) {
        if (memcmp(pose[g].c, pose[0].c, sizeof(pose[0].c)) != 0) return PFGPU_ERR_INVALID;   // moments about different centres
        if (lm && m && !lm[g]) return PFGPU_ERR_INVALID;
    }
    Fs3PoseMom acc = {0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}};
    for (int g = 0; g < world; ++g) {
        Fs3PoseMom b;
        b.w = pose[g].w;
        for (int k = 0; k < 3; ++k) b.m[k] = pose[g].mean[k];
        for (int k = 0; k < 6; ++k) b.q[k] = pose[g].m2[k];
        fs3_pose_merge(acc, b);
    }
    const double W = acc.w;
    const bool ok = W > 0.0 && std::isfinite(W);
    const double nan = std::numeric_limits<double>::quiet_NaN();
    if (pose_mean3 || pose_cov9_colmajor) {
        double mean[3], cov[9];
        mean[0] = pose[0].c[0] + acc.m[0]; mean[1] = pose[0].c[1] + acc.m[1]; mean[2] = fs3_wrap_angle(pose[0].c[2] + acc.m[2]);
        static const int ix[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) cov[3 * j + i] = acc.q[ix[i][j]] / W;
        if (pose_mean3) for (int k = 0; k < 3; ++k) pose_mean3[k] = ok ? mean[k] : nan;
        if (pose_cov9_colmajor) for (int k = 0; k < 9; ++k) pose_cov9_colmajor[k] = ok ? cov[k] : nan;
    }
    if (!lm) return 0;
    for (size_t l = 0; l < m; ++l) {
        Fs3LmMom acc = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
        for (int g = 0; g < world; ++g) fs3_mom_merge(acc, reinterpret_cast<const Fs3LmMom*>(lm[g])[l]);
        const bool some = ok && acc.w != 0.0;
        if (lm_mass) lm_mass[l] = some ? acc.w / W : 0.0;
        if (lm_mean2) { lm_mean2[2 * l] = some ? acc.mx : nan; lm_mean2[2 * l + 1] = some ? acc.my : nan; }
        if (lm_cov4) {
            lm_cov4[4 * l] = some ? acc.m00 / acc.w : nan; lm_cov4[4 * l + 1] = some ? acc.m01 / acc.w : nan;
            lm_cov4[4 * l + 2] = some ? acc.m10 / acc.w : nan; lm_cov4[4 * l + 3] = some ? acc.m11 / acc.w : nan;
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------------------------------------------------
// path history (DESIGN §3.6): pfgpu_fs_history_enable / _window, pfgpu_fs_path, pfgpu_fs_path_moments
// ---------------------------------------------------------------------------------------------------------------------
static_assert(sizeof(pfgpu_fs_pose_moments) == 13 * sizeof(double), "fs3_hist_merge_kernel writes 13 doubles per entry");

// entry `steps` <- the live poses (root: every parent is the slot itself, and the window restarts there)
static int fs_hist_record(pfgpu_fs* h, int root) {
    const unsigned e = (unsigned)(h->steps % h->hist_cap);
    PF_LAUNCH(h->ctx, fs3_hist_record_kernel, cdiv_u(h->d.n, FS3_HIST_NT), FS3_HIST_NT, 0, h->d, h->hist, (unsigned)h->hist_cap, e, root);
    if (root) h->hist_first = h->steps;
    else if (h->steps - h->hist_first >= h->hist_cap) h->hist_first = h->steps - h->hist_cap + 1;     // the ring is full: drop the oldest
    return 0;
}
static void fs_hist_release(pfgpu_fs* h) {
    fs_unmap(h, h->hist_peer);
    cudaFree(h->hist); h->hist = nullptr; h->hist_cap = 0; h->hist_first = 0;
}
extern "C" int pfgpu_fs_history_enable(pfgpu_fs* h, size_t capacity) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));               // nothing in flight still writes the old ring
    if (capacity == 0) { fs_hist_release(h); return 0; }
    const size_t per = fs3_hist_bytes(1, h->d.ld);
    char* ring = nullptr;
    int ok = capacity <= 0xFFFFFFFFull && capacity <= SIZE_MAX / per;
    if (ok && cudaMalloc(&ring, capacity * per) != cudaSuccess) { ok = 0; ring = nullptr; cudaGetLastError(); }
    void* opened[FS3_MAXG] = {};
    if (h->comm) {          // one process per GPU: every rank maps every peer's ring once, with the same capacity everywhere
        const int rc = fs_share(h, ring, ok, capacity, opened, "path history");
        if (rc) { cudaFree(ring); return rc; }
    } else if (!ok) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "path history: a ring of %zu entries x %u slots does not fit in device memory", capacity, h->d.ld);
        return PFGPU_ERR_CUDA;
    }
    fs_hist_release(h);
    h->hist = ring; h->hist_cap = capacity;
    memcpy(h->hist_peer, opened, sizeof(opened));
    int rc = fs_hist_record(h, 1);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_fs_history_window(pfgpu_fs* h, uint64_t* first_step, uint64_t* last_step) {
    if (!h || !h->hist) return PFGPU_ERR_INVALID;
    if (first_step) *first_step = h->hist_first;
    if (last_step) *last_step = h->steps;
    return 0;
}

static int fs_hist_scratch(pfgpu_fs* h, size_t bytes) {
    if (bytes <= h->hs_bytes) return 0;
    if (h->hs) { cudaFree(h->hs); h->hs = nullptr; h->hs_bytes = 0; }
    PF_CUDA(cudaMalloc(&h->hs, bytes));
    h->hs_bytes = bytes;
    return 0;
}
// common prologue of the queries: synchronise, the rings of every rank, the number of entries L to return
static int fs_hist_begin(pfgpu_fs* h, size_t max_steps, Fs3Hist* H, unsigned* L) {
    if (!h->hist || max_steps == 0) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    int rc = fs_check_err(h);
    if (rc) return rc;
    memset(H, 0, sizeof(*H));
    H->cap = (unsigned)h->hist_cap; H->ld = h->d.ld; H->n = h->d.n;
    for (int g = 0; g < h->world; ++g) {
        const pfgpu_fs* o = h->sib[g];
        const char* b = fs_rank_buf(h, g, &pfgpu_fs::hist, h->hist_peer);
        if (!b || (o && (o->hist_cap != h->hist_cap || o->hist_first != h->hist_first || o->steps != h->steps))) {
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "path history: rank %d holds no ring with this window (pfgpu_fs_history_enable, upload and "
                     "seed_map are made on every rank)", g);
            return PFGPU_ERR_INVALID;
        }
        H->base[g] = b;
    }
    *L = (unsigned)std::min<uint64_t>(h->steps - h->hist_first + 1, (uint64_t)std::min<size_t>(max_steps, 0xFFFFFFFFu));
    return 0;
}

extern "C" int pfgpu_fs_path(pfgpu_fs* h, size_t index_global, size_t max_steps, uint64_t* step, uint32_t* slot, double* pose3, size_t* n) {
    if (!h || !n || index_global >= h->d.n_glob) return PFGPU_ERR_INVALID;
    Fs3Hist H; unsigned L = 0;
    int rc = fs_hist_begin(h, max_steps, &H, &L);
    if (rc) return rc;
    const size_t o_pose = ((size_t)L * sizeof(unsigned) + 255) & ~(size_t)255;
    rc = fs_hist_scratch(h, o_pose + (size_t)L * 3 * sizeof(double));
    if (rc) return rc;
    unsigned* dslot = reinterpret_cast<unsigned*>(h->hs);
    double* dpose = reinterpret_cast<double*>(h->hs + o_pose);
    PF_LAUNCH(h->ctx, fs3_hist_path_kernel, 1, 32, 0, H, (unsigned)(h->steps % h->hist_cap), L, (unsigned)index_global, dslot, dpose);
    std::vector<unsigned> s(L);
    std::vector<double> p(3 * (size_t)L);
    PF_CUDA(cudaMemcpyAsync(s.data(), dslot, (size_t)L * sizeof(unsigned), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(p.data(), dpose, (size_t)L * 3 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    for (size_t j = 0; j < L; ++j) {                              // oldest first
        const size_t k = L - 1 - j;
        if (step) step[j] = h->steps - k;
        if (slot) slot[j] = s[k];
        if (pose3) for (int c = 0; c < 3; ++c) pose3[3 * j + c] = p[3 * k + c];
    }
    *n = L;
    return fs_check_err(h);
}

extern "C" int pfgpu_fs_path_moments(pfgpu_fs* h, size_t max_steps, uint64_t* step, pfgpu_fs_pose_moments* out, size_t* n) {
    if (!h || !out || !n) return PFGPU_ERR_INVALID;
    Fs3Hist H; unsigned L = 0;
    int rc = fs_hist_begin(h, max_steps, &H, &L);
    if (rc) return rc;
    const Fs3Dev& d = h->d;
    const unsigned nb = cdiv_u(d.n, FS3_HIST_NT);
    const unsigned Lc = (unsigned)std::max<size_t>(1, std::min<size_t>(L, FS3_HIST_SCRATCH_CAP / ((size_t)nb * sizeof(Fs3PoseMom))));
    // scratch: centre slots [L] | centres [L][3] | lineage slots [n] | block partials [Lc][nb] | moments [L][13]
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t o_ctr = up((size_t)L * sizeof(unsigned)), o_lin = o_ctr + up((size_t)L * 3 * sizeof(double));
    const size_t o_part = o_lin + up((size_t)d.n * sizeof(unsigned)), o_out = o_part + up((size_t)Lc * nb * sizeof(Fs3PoseMom));
    rc = fs_hist_scratch(h, o_out + (size_t)L * sizeof(pfgpu_fs_pose_moments));
    if (rc) return rc;
    char* S = h->hs;
    const double* ctr = reinterpret_cast<const double*>(S + o_ctr);
    // the centres: the lineage of global slot n - 1, read the same on every rank
    PF_LAUNCH(h->ctx, fs3_hist_path_kernel, 1, 32, 0, H, (unsigned)(h->steps % h->hist_cap), L, d.n_glob - 1u, reinterpret_cast<unsigned*>(S),
              reinterpret_cast<double*>(S + o_ctr));
    for (unsigned k0 = 0; k0 < L; k0 += Lc) {
        const unsigned k1 = std::min(L, k0 + Lc), e0 = (unsigned)((h->steps - k0) % h->hist_cap);
        PF_LAUNCH(h->ctx, fs3_hist_moments_kernel, nb, FS3_HIST_NT, 0, d, H, e0, k0, k1, reinterpret_cast<unsigned*>(S + o_lin), ctr,
                  reinterpret_cast<Fs3PoseMom*>(S + o_part));
        PF_LAUNCH(h->ctx, fs3_hist_merge_kernel, cdiv_u(k1 - k0, 128), 128, 0, reinterpret_cast<const Fs3PoseMom*>(S + o_part), nb, k0, k1, ctr,
                  reinterpret_cast<double*>(S + o_out));
    }
    std::vector<pfgpu_fs_pose_moments> tmp(L);
    PF_CUDA(cudaMemcpyAsync(tmp.data(), S + o_out, (size_t)L * sizeof(pfgpu_fs_pose_moments), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    for (size_t j = 0; j < L; ++j) {                              // oldest first
        const size_t k = L - 1 - j;
        if (step) step[j] = h->steps - k;
        out[j] = tmp[k];
    }
    *n = L;
    return fs_check_err(h);
}
