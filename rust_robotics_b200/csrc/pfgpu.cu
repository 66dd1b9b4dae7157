// pfgpu.cu — the C ABI of include/pfgpu.h: handles, step orchestration, upload/download.
// Single translation unit: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false (see __graft_entry__.build()).
#include "common.cuh"
#include "xsum.cuh"
#include "pf_kernels.cuh"
#include "pf3.cuh"
#include "pf_kld.cuh"
#include "pf_lfield.cuh"
#include "pf_cluster.cuh"
#include "ogm.cuh"
#include "csm.cuh"
#include "xsum_sharded.cuh"
#include <cstdlib>
#include <new>
#include <vector>
#include <cmath>
#include <algorithm>
#include <cfloat>
#include <type_traits>

thread_local char g_pfgpu_err[512] = {0};

// the measurement model of a weight pass: landmark ranges, the likelihood field (DESIGN §3.9) or the beam model (DESIGN §3.11)
#define PF_KIND_LM 0
#define PF_KIND_LF 1
#define PF_KIND_BEAM 2

extern "C" const char* pfgpu_last_error(void) { return g_pfgpu_err; }
extern "C" const char* pfgpu_strerror(int s) {
    switch (s) {
        case PFGPU_OK: return "ok";
        case PFGPU_ERR_INVALID: return "invalid parameter";
        case PFGPU_ERR_UNSUPPORTED: return "valid in the reference but not supported by this build";
        case PFGPU_ERR_NO_DEVICE: return "no usable CUDA device (this library has no CPU fallback)";
        case PFGPU_ERR_CUDA: return "CUDA runtime error (see pfgpu_last_error)";
        case PFGPU_ERR_NCCL: return "NCCL error (see pfgpu_last_error)";
        default: return "unknown status";
    }
}
extern "C" int pfgpu_device_count(int* count) {
    int c = 0;
    cudaError_t e = cudaGetDeviceCount(&c);
    if (e != cudaSuccess) { *count = 0; snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "cudaGetDeviceCount: %s", cudaGetErrorString(e)); return PFGPU_ERR_NO_DEVICE; }
    *count = c;
    return c > 0 ? PFGPU_OK : PFGPU_ERR_NO_DEVICE;
}

static bool finite_d(double v) { return std::isfinite(v); }

static int ctx_open(Ctx& ctx, int device) {
    int count = 0;
    int rc = pfgpu_device_count(&count);
    if (rc) return rc;
    if (device < 0 || device >= count) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "device %d out of range (%d devices)", device, count); return PFGPU_ERR_NO_DEVICE; }
    PF_CUDA(cudaSetDevice(device));
    ctx.device = device;
    PF_CUDA(cudaStreamCreateWithFlags(&ctx.stream, cudaStreamNonBlocking));
    int sms = 0;
    PF_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    ctx.num_sms = sms > 0 ? sms : PFGPU_NUM_SMS;
    return 0;
}

#define PF_MARK_SLOTS 16384
__global__ void pf_l2_read_kernel(const double4* __restrict__ p, size_t n4, double* sink) {
    double acc = 0.0;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
        double4 v = p[i];
        acc += v.x + v.y + v.z + v.w;
    }
    if (acc == 123.456) *sink = acc;      // never true: keeps the loads alive
}
struct Marks {
    std::vector<cudaEvent_t> ev = std::vector<cudaEvent_t>(PF_MARK_SLOTS, nullptr);
    void* l2buf = nullptr;
    void* l2buf_rd = nullptr;
    size_t l2bytes = (size_t)256 << 20;      // several times the 50 MB L2
};
static int marks_mark(Ctx& ctx, Marks& m, int slot) {
    if (slot < 0 || slot >= PF_MARK_SLOTS) return PFGPU_ERR_INVALID;
    if (!m.ev[slot]) PF_CUDA(cudaEventCreate(&m.ev[slot]));
    PF_CUDA(cudaEventRecord(m.ev[slot], ctx.stream));
    return 0;
}
static int marks_elapsed(Marks& m, int a, int b, double* ms) {
    if (a < 0 || a >= PF_MARK_SLOTS || b < 0 || b >= PF_MARK_SLOTS || !m.ev[a] || !m.ev[b] || !ms) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaEventSynchronize(m.ev[b]));
    float f = 0.f;
    PF_CUDA(cudaEventElapsedTime(&f, m.ev[a], m.ev[b]));
    *ms = (double)f;
    return 0;
}
static int marks_flush(Ctx& ctx, Marks& m) {
    if (!m.l2buf) {
        PF_CUDA(cudaMalloc(&m.l2buf, m.l2bytes));
        PF_CUDA(cudaMalloc(&m.l2buf_rd, m.l2bytes));
        PF_CUDA(cudaMemsetAsync(m.l2buf_rd, 0, m.l2bytes, ctx.stream));
    }
    // write a buffer larger than L2 (evicts everything), then stream a second one through it so that the cache is left
    // full of CLEAN lines: the timed kernel then starts cold without inheriting the flush's own write-backs
    PF_CUDA(cudaMemsetAsync(m.l2buf, 0, m.l2bytes, ctx.stream));
    pf_l2_read_kernel<<<ctx.num_sms * 8, 256, 0, ctx.stream>>>((const double4*)m.l2buf_rd, m.l2bytes / 32, (double*)m.l2buf);
    return cudaGetLastError() == cudaSuccess ? 0 : PFGPU_ERR_CUDA;
}
static void marks_free(Marks& m) {
    for (auto e : m.ev) if (e) cudaEventDestroy(e);
    if (m.l2buf) cudaFree(m.l2buf);
    if (m.l2buf_rd) cudaFree(m.l2buf_rd);
}

struct KernelTimer {
    bool on = false;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
    double ms_sum = 0.0; uint64_t count = 0;
};

// ====================================================================================================
// ParticleFilterLocalizer / MonteCarloLocalizer
// ====================================================================================================
// what the map of either scan model has in common; on = a map is loaded
struct PfMap {
    bool on = false;
    size_t W = 0, H = 0;
    uint64_t L = 0;                // the most used beams a scan may have
};
struct pfgpu_pf {
    Ctx ctx;
    pfgpu_pf_config cfg;
    uint64_t seed = 0;
    PfDev d;
    XsWork xs;
    size_t obs_cap = 0;        // the doubles d.obs holds
    double* mom = nullptr;     // [world] PfMom: every shard's estimate moments
    int mom_blocks = 0;
    uint32_t n_predict = 0, n_resample = 0;
    uint64_t steps = 0, resamples_unknown = 0;
    int world = 1, rank = 0;
    KernelTimer timer;
    Marks marks;
    double* h_pin = nullptr;   // pinned scratch (>= 64 doubles)
    FsShard sh;                // multi-GPU state (world == 1: unused)
    int cur_host = 0;          // sharded mode: host mirror of *d.cur (the host knows every gate there)
    bool adaptive = false;     // MCL with min_particles < max_particles: the particle count changes per step (pf_kld.cuh)
    PfKld kld;
    // The fused step (pfgpu_pf_step) of a fixed-size, single-GPU filter is the same ~22 launches every time: predict + weight,
    // the exact-sum pipelines, gate, search, gather, flip, moments — a launch-bound sequence below ~10^5 particles.  It is
    // captured ONCE into a CUDA graph and replayed; only the first kernel's arguments (control, observations, draw counter,
    // range noise) change from step to step and are patched into the instantiated graph before each replay.
    // fused tail of the step (pf3.cuh): everything after the predict + likelihood kernel in one cooperative launch
    struct Fused {
        bool on = false;
        bool last = false;         // it ran the last exact sum (set by pfgpu_pf_step; cleared by pf_total, ahead of every other sum)
        Fs3Sum x = {};             // its exact sums and grid barriers
        Pf3Arg arg = {};
        unsigned tiles = 0;
        size_t smem = 0;
    } fu;
    struct StepGraph {
        cudaGraphExec_t exec = nullptr;
        cudaGraph_t graph = nullptr;
        cudaGraphNode_t main_node = nullptr;
        cudaKernelNodeParams main_params = {};
        size_t k = ~(size_t)0;
        int kind = PF_KIND_LM;     // a scan step's graph (either model) serves every beam count up to PF_PARAM_BEAMS (k is patched like u)
        bool odom = false;         // its predict is the odometry model's (DESIGN §3.14), whose kernel differs from the velocity model's
        uint64_t launches = 0;
        int captures = 0;          // an observation count that keeps changing would re-capture every step: give up after a few
        bool off = false;          // PFGPU_PF_GRAPH=0, capture failed, or too many re-captures: plain launches from then on
    } sg;
    // augmented MCL (DESIGN §3.8): w_slow, w_fast and p live in d.scal[PF_REC_*], the injection count in d.counters[PF_REC_COUNT]
    struct Recovery {
        bool on = false;
        bool armed = false;        // the last stage was a resample stage: the next predict injects if that stage resampled (*d.gate)
        double a_slow = 0.0, a_fast = 0.0;
        double region[4] = {0.0, 0.0, 0.0, 0.0};     // x0, x1, y0, y1
    } rec;
    // likelihood-field scan model (DESIGN §3.9): the map's tables and parameters
    struct LField : PfMap {
        double* D = nullptr;       // distance field [cells], ix * H + iy
        double* q = nullptr;       // per-cell factor
        pfgpu_lfield_config cfg = {};
        double q_out = 0.0;
        bool keep_max() const { return false; }
        void release() { cudaFree(D); cudaFree(q); *this = LField(); }
    } lf;
    // beam model (DESIGN §3.11): the clearance table and parameters.  Separate from the likelihood field's.
    struct BeamMap : PfMap {
        unsigned char* clr = nullptr;   // clearance [cells], ix * H + iy
        pfgpu_beam_config cfg = {};
        int skip = 1;              // PFGPU_BEAM_SKIP=0 at set time: the caster steps one cell at a time
        bool keep_max() const { return cfg.z_max > 0.0; }      // max readings are used beams (as r = max_range)
        void release() { cudaFree(clr); *this = BeamMap(); }
    } bm;
    std::vector<double> pairs;     // the used beams of the current scan call (either model): (r_i, a_i)
    double odom_alpha[4] = { PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT };   // DESIGN §3.14
    PfClu clu;                     // pose hypotheses' workspace (DESIGN §3.10), allocated by the first query
};

extern "C" void pfgpu_pf_default_config(pfgpu_pf_config* c, int mode) {
    memset(c, 0, sizeof(*c));
    c->n_particles = 100; c->resample_threshold = 0.5; c->range_noise = 0.2; c->velocity_noise = 2.0;
    c->yaw_rate_noise = 40.0 * PFC_PI / 180.0; c->dt = 0.1; c->mode = mode;
    c->max_particles = mode == 1 ? 5000 : 100; c->kld_epsilon = 0.05; c->kld_z = 2.326;
}
extern "C" int pfgpu_pf_config_validate(const pfgpu_pf_config* c) {
    if (!c) return PFGPU_ERR_INVALID;
    if (c->n_particles == 0) return PFGPU_ERR_INVALID;                                                   // pf.rs:82, mcl.rs:88
    if (c->mode == 0) {
        if (!finite_d(c->resample_threshold) || c->resample_threshold < 0.0 || c->resample_threshold > 1.0) return PFGPU_ERR_INVALID;  // pf.rs:87-94
    } else if (c->mode == 1) {
        if (c->max_particles < c->n_particles) return PFGPU_ERR_INVALID;                                 // mcl.rs:93-97
        if (!finite_d(c->kld_epsilon) || c->kld_epsilon <= 0.0) return PFGPU_ERR_INVALID;                // mcl.rs:98-102
        if (!finite_d(c->kld_z) || c->kld_z <= 0.0) return PFGPU_ERR_INVALID;                            // mcl.rs:103-107
    } else return PFGPU_ERR_INVALID;
    if (!finite_d(c->range_noise) || c->range_noise <= 0.0) return PFGPU_ERR_INVALID;                    // pf.rs:95-99
    if (!finite_d(c->velocity_noise) || c->velocity_noise < 0.0) return PFGPU_ERR_INVALID;               // pf.rs:100-104
    if (!finite_d(c->yaw_rate_noise) || c->yaw_rate_noise < 0.0) return PFGPU_ERR_INVALID;               // pf.rs:105-109
    if (!finite_d(c->dt) || c->dt <= 0.0) return PFGPU_ERR_INVALID;                                      // pf.rs:110-114
    return PFGPU_OK;
}

__global__ void pf_init_zero_kernel(PfDev d) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    Pose4 z; z.x = 0.0; z.y = 0.0; z.yaw = 0.0; z.v = 0.0;
    pose_store(d.pose[0], i, z);
    d.w[i] = 1.0 / (double)d.n_global;                 // Particle::new pf.rs:35-43
    d.w_raw[i] = d.w[i];
}
// try_with_initial_state pf.rs:181-187 (random::<f64>()*2-1 ...) / mcl.rs:190-196 (random_range(-1.0..1.0) ...)
__global__ void pf_init_state_kernel(PfDev d, double s0, double s1, double s2, double s3, uint64_t seed, int mode) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    pfc_u32x4 a = pfc_rng_block(seed, PFC_STREAM_INIT_A, 0, d.offset + i);
    pfc_u32x4 b = pfc_rng_block(seed, PFC_STREAM_INIT_B, 0, d.offset + i);
    Pose4 p;
    if (mode == 0) {
        p.x = s0 + pfc_u01_53(pfc_blk_u64(a, 0)) * 2.0 - 1.0;
        p.y = s1 + pfc_u01_53(pfc_blk_u64(a, 1)) * 2.0 - 1.0;
        p.yaw = s2 + pfc_u01_53(pfc_blk_u64(b, 0)) * 0.5 - 0.25;
        p.v = s3 + pfc_u01_53(pfc_blk_u64(b, 1)) * 1.0 - 0.5;
    } else {
        p.x = s0 + (pfc_u01_52(pfc_blk_u64(a, 0)) * 2.0 + -1.0);
        p.y = s1 + (pfc_u01_52(pfc_blk_u64(a, 1)) * 2.0 + -1.0);
        p.yaw = s2 + (pfc_u01_52(pfc_blk_u64(b, 0)) * 0.5 + -0.25);
        p.v = s3 + (pfc_u01_52(pfc_blk_u64(b, 1)) * 1.0 + -0.5);
    }
    pose_store(pf_pose(d, *d.cur), i, p);
    d.w[i] = 1.0 / (double)d.n_global;
    d.w_raw[i] = d.w[i];
}
__global__ void pf_unpack_kernel(PfDev d, const double* aos5) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    Pose4 p; p.x = aos5[5 * i]; p.y = aos5[5 * i + 1]; p.yaw = aos5[5 * i + 2]; p.v = aos5[5 * i + 3];
    pose_store(pf_pose(d, *d.cur), i, p);
    d.w[i] = aos5[5 * i + 4];
    d.w_raw[i] = d.w[i];
}
__global__ void pf_pack_kernel(PfDev d, double* aos5) {
    const size_t i = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (i >= d.n) return;
    Pose4 p;
    pose_load(pf_pose(d, *d.cur), i, p);
    aos5[5 * i] = p.x; aos5[5 * i + 1] = p.y; aos5[5 * i + 2] = p.yaw; aos5[5 * i + 3] = p.v; aos5[5 * i + 4] = d.w[i];
}

static int pf_refresh_cache(pfgpu_pf* h) {      // refresh_cache pf.rs:499-503
    double* own = h->mom + (size_t)h->rank * PF_MOM;
    PF_LAUNCH(h->ctx, pf_moments_kernel, h->mom_blocks, PF_NT, 0, h->d, h->mom_blocks);
    PF_LAUNCH(h->ctx, pf_moments_reduce_kernel, 1, PF_NT, 0, h->d.partial, h->mom_blocks, own);
    if (h->world > 1)   // every rank gathers every shard's moments and merges them in rank order: the same bits on every rank
        PF_NCCL(ncclAllGather(own, h->mom, PF_MOM, ncclDouble, h->sh.comm, h->ctx.stream));
    PF_LAUNCH(h->ctx, pf_moments_final_kernel, 1, 32, 0, h->d, h->mom, h->world);
    return 0;
}
// augmented MCL: w_slow = w_fast = p = 0, injection count 0, disarmed
static int pf_recovery_reset(pfgpu_pf* h) {
    h->rec.armed = false;
    PF_CUDA(cudaMemsetAsync(h->d.scal + PF_REC_SLOW, 0, 3 * sizeof(double), h->ctx.stream));
    PF_CUDA(cudaMemsetAsync(h->d.counters + PF_REC_COUNT, 0, sizeof(unsigned int), h->ctx.stream));
    return 0;
}
static bool pf_region_ok(const double* r) {      // finite, x0 < x1, y0 < y1
    if (!r) return false;
    for (int j = 0; j < 4; ++j) if (!finite_d(r[j])) return false;
    return r[0] < r[1] && r[2] < r[3];
}

static int pf_alloc(pfgpu_pf* h, size_t cap) {
    PfDev& d = h->d;
    const size_t n = cap;       // every per-particle array is sized for the largest generation
    PF_CUDA(cudaMalloc(&d.pose[0], n * sizeof(Pose4)));
    PF_CUDA(cudaMalloc(&d.pose[1], n * sizeof(Pose4)));
    PF_CUDA(cudaMalloc(&d.cur, sizeof(int)));
    PF_CUDA(cudaMemset(d.cur, 0, sizeof(int)));
    PF_CUDA(cudaMalloc(&d.w_raw, n * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.w, n * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.cum, n * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.idx, n * sizeof(uint32_t)));
    PF_CUDA(cudaMalloc(&d.scal, 32 * sizeof(double)));
    PF_CUDA(cudaMemset(d.scal, 0, 32 * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.gate, sizeof(int)));
    PF_CUDA(cudaMemset(d.gate, 0, sizeof(int)));
    PF_CUDA(cudaMalloc(&d.counters, 4 * sizeof(unsigned int)));
    PF_CUDA(cudaMemset(d.counters, 0, 4 * sizeof(unsigned int)));
    h->mom_blocks = (int)std::min<size_t>((size_t)h->ctx.num_sms * 4, cdiv_u(n, PF_NT));
    if (h->mom_blocks < 1) h->mom_blocks = 1;
    PF_CUDA(cudaMalloc(&d.partial, (size_t)h->mom_blocks * PF_MOM * sizeof(double)));
    PF_CUDA(cudaMalloc(&h->mom, (size_t)h->world * PF_MOM * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.obs, 3 * 1024 * sizeof(double)));
    h->obs_cap = 3 * 1024;
    PF_CUDA(cudaMallocHost(&h->h_pin, 64 * sizeof(double)));
    if (h->adaptive) {
        PfKld& k = h->kld;
        k.cap = cap;
        unsigned tc = 64;
        while ((size_t)tc < 2 * cap + 16) tc <<= 1;
        k.tcap = tc;
        PF_CUDA(cudaMalloc(&k.keys, 3 * cap * sizeof(int)));
        PF_CUDA(cudaMalloc(&k.owner, (size_t)tc * sizeof(int)));
        PF_CUDA(cudaMalloc(&k.mint, (size_t)tc * sizeof(unsigned)));
        PF_CUDA(cudaMalloc(&k.slot, cap * sizeof(int)));
        PF_CUDA(cudaMalloc(&k.n_new, sizeof(unsigned)));
    }
    return xs_work_alloc(h->xs, n);
}

// workspace + shape of the fused tail (pf3.cuh); leaves h->fu.on false when the configuration keeps the multi-kernel path
static int pf3_setup(pfgpu_pf* h) {
    const char* e = getenv("PFGPU_PF_FUSED");
    if (e && e[0] == '0') return 0;
    const size_t n = h->d.n;
    // up to 2^18 particles (H100 SXM at 400 W, resample every step: 1.44x at 2^16, 1.10x at 2^18 against the separate kernels);
    // beyond that the separate kernels fill the GPU and their launch latency is hidden behind the graph replay
    if (h->world != 1 || h->adaptive || n < 1 || n > ((size_t)1 << 18)) return 0;
    const unsigned NT = 256;
    unsigned tiles = (unsigned)std::min<size_t>((size_t)std::min(h->ctx.num_sms, FS3_MAX_TILES), (n + NT - 1) / NT);
    unsigned K = (unsigned)((n + (size_t)tiles * NT - 1) / ((size_t)tiles * NT));
    tiles = (unsigned)((n + (size_t)NT * K - 1) / ((size_t)NT * K));                       // no empty tile: the last one holds index n - 1
    const size_t smem = (size_t)2 * K * NT * sizeof(double);
    if (cudaFuncSetAttribute(pf3_post_kernel<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) { cudaGetLastError(); return 0; }
    int nb = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, pf3_post_kernel<256>, (int)NT, smem) != cudaSuccess || (size_t)nb * (size_t)h->ctx.num_sms < tiles) { cudaGetLastError(); return 0; }
    Fs3Sum& x = h->fu.x;
    PF_CUDA(fs3_sum_alloc(x, (unsigned)n, false));
    x.raw[0] = x.raw[1] = h->d.w_raw; x.wn = h->d.w;                                       // one raw buffer: PF steps have no parity
    Pf3Arg& a = h->fu.arg;
    a.pd = h->d; a.threshold = h->cfg.resample_threshold; a.mode = h->cfg.mode; a.seed = h->seed; a.K = K; a.m32 = x3_margin32(n);
    PF_CUDA(cudaMalloc(&a.tsum, FS3_MAX_TILES * sizeof(double))); PF_CUDA(cudaMalloc(&a.tsq, FS3_MAX_TILES * sizeof(double)));
    PF_CUDA(cudaMalloc(&a.mom, (size_t)FS3_MAX_TILES * PF_MOM * sizeof(double)));
    h->fu.tiles = tiles; h->fu.smem = smem;
    h->fu.on = true;
    return 0;
}
static void pf3_free(pfgpu_pf* h) {
    fs3_sum_free(h->fu.x);
    cudaFree(h->fu.arg.tsum); cudaFree(h->fu.arg.tsq); cudaFree(h->fu.arg.mom);
}

static int pf_create_impl(const pfgpu_pf_config* cfg, uint64_t seed, int device, const void* uid, int rank, int world, pfgpu_pf** out) {
    if (!out) return PFGPU_ERR_INVALID;
    *out = nullptr;
    int rc = pfgpu_pf_config_validate(cfg);
    if (rc) return rc;
    const bool adaptive = cfg->mode == 1 && cfg->max_particles != cfg->n_particles;     // KLD-adaptive particle count, mcl.rs:322-365
    if (adaptive && world > 1) return PFGPU_ERR_UNSUPPORTED;                            // a changing count is not sharded (yet)
    if (cfg->n_particles > 0xFFFFFFFFull || (adaptive && cfg->max_particles > 0x7FFFFFFFull)) return PFGPU_ERR_UNSUPPORTED;
    if (world > 1 && (cfg->n_particles % (uint64_t)world) != 0) return PFGPU_ERR_INVALID;
    pfgpu_pf* h = new (std::nothrow) pfgpu_pf();
    if (!h) return PFGPU_ERR_CUDA;
    rc = ctx_open(h->ctx, device);
    if (rc) { delete h; return rc; }
    h->cfg = *cfg; h->seed = seed; h->world = world; h->rank = rank;
    { const char* e = getenv("PFGPU_PF_GRAPH"); if (e && e[0] == '0') h->sg.off = true; }
    h->fu.on = false;
    h->d.n_global = cfg->n_particles; h->d.n = cfg->n_particles / (uint64_t)world; h->d.offset = (size_t)rank * h->d.n;
    h->adaptive = adaptive;
    rc = pf_alloc(h, adaptive ? (size_t)cfg->max_particles : h->d.n);
    if (rc) { pfgpu_pf_destroy(h); return rc; }
    if (world > 1) {
        FsShard& sh = h->sh;
        sh.rank = rank; sh.world = world;
        ncclUniqueId id;
        memcpy(&id, uid, sizeof(id));
        ncclResult_t nr = ncclCommInitRank(&sh.comm, world, id, rank);
        if (nr != ncclSuccess) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "ncclCommInitRank: %s", ncclGetErrorString(nr)); pfgpu_pf_destroy(h); return PFGPU_ERR_NCCL; }
        const size_t ng = h->d.n_global;
        bool ok = cudaMalloc(&sh.t_loc, sizeof(double)) == cudaSuccess && cudaMalloc(&sh.t_all, world * sizeof(double)) == cudaSuccess &&
                  cudaMalloc(&sh.approx_off, sizeof(double)) == cudaSuccess && cudaMalloc(&sh.sum_loc, sizeof(ShardSummary)) == cudaSuccess &&
                  cudaMalloc(&sh.sum_all, world * sizeof(ShardSummary)) == cudaSuccess && cudaMalloc(&sh.s_start, sizeof(double)) == cudaSuccess &&
                  cudaMalloc(&sh.err, sizeof(int)) == cudaSuccess && cudaMemset(sh.err, 0, sizeof(int)) == cudaSuccess &&
                  cudaMalloc(&sh.cum_all, ng * sizeof(double)) == cudaSuccess && cudaMalloc(&sh.pose_all, 4 * ng * sizeof(double)) == cudaSuccess;
        if (!ok) { pfgpu_pf_destroy(h); return PFGPU_ERR_CUDA; }
    }
    PF_LAUNCH(h->ctx, pf_init_zero_kernel, cdiv_u(h->d.n, PF_NT), PF_NT, 0, h->d);
    rc = pf_refresh_cache(h);
    if (rc) { pfgpu_pf_destroy(h); return rc; }
    rc = pf3_setup(h);
    if (rc) { pfgpu_pf_destroy(h); return rc; }
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    *out = h;
    return PFGPU_OK;
}
extern "C" int pfgpu_pf_create(const pfgpu_pf_config* cfg, uint64_t seed, int device, pfgpu_pf** out) {
    return pf_create_impl(cfg, seed, device, nullptr, 0, 1, out);
}
extern "C" int pfgpu_pf_create_sharded(const pfgpu_pf_config* cfg, uint64_t seed, int device, const void* uid, int rank, int world, pfgpu_pf** out) {
    if (out) *out = nullptr;
    if (!uid || world < 1 || world > SH_MAX_WORLD || rank < 0 || rank >= world) return PFGPU_ERR_INVALID;
    return pf_create_impl(cfg, seed, device, uid, rank, world, out);
}
extern "C" void pfgpu_pf_destroy(pfgpu_pf* h) {
    if (!h) return;
    cudaSetDevice(h->ctx.device);
    if (h->ctx.stream) cudaStreamSynchronize(h->ctx.stream);
    PfDev& d = h->d;
    cudaFree(d.pose[0]); cudaFree(d.pose[1]); cudaFree(d.cur); cudaFree(d.w_raw); cudaFree(d.w); cudaFree(d.cum);
    cudaFree(d.idx); cudaFree(d.scal); cudaFree(d.gate); cudaFree(d.partial); cudaFree(d.obs); cudaFree(h->mom); cudaFree(d.counters);
    h->lf.release(); h->bm.release();
    if (h->h_pin) cudaFreeHost(h->h_pin);
    if (h->sg.exec) cudaGraphExecDestroy(h->sg.exec);
    if (h->sg.graph) cudaGraphDestroy(h->sg.graph);
    pf3_free(h);
    cudaFree(h->kld.keys); cudaFree(h->kld.owner); cudaFree(h->kld.mint); cudaFree(h->kld.slot); cudaFree(h->kld.n_new);
    pf_clu_free(h->clu);
    {
        FsShard& sh = h->sh;
        cudaFree(sh.t_loc); cudaFree(sh.t_all); cudaFree(sh.approx_off); cudaFree(sh.sum_loc); cudaFree(sh.sum_all); cudaFree(sh.s_start);
        cudaFree(sh.err); cudaFree(sh.cum_all); cudaFree(sh.pose_all);
        if (sh.comm) ncclCommDestroy(sh.comm);
    }
    marks_free(h->marks);
    xs_work_free(h->xs);
    for (auto& p : h->timer.pending) { cudaEventDestroy(p.first); cudaEventDestroy(p.second); }
    if (h->ctx.stream) cudaStreamDestroy(h->ctx.stream);
    delete h;
}
extern "C" int pfgpu_pf_sync(pfgpu_pf* h) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_pf_init_state(pfgpu_pf* h, const double s[4]) {
    if (!h || !s) return PFGPU_ERR_INVALID;
    for (int k = 0; k < 4; ++k) if (!finite_d(s[k])) return PFGPU_ERR_INVALID;     // validate_state pf.rs:505-513
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_LAUNCH(h->ctx, pf_init_state_kernel, cdiv_u(h->d.n, PF_NT), PF_NT, 0, h->d, s[0], s[1], s[2], s[3], h->seed, h->cfg.mode);
    if (h->rec.on) { int rc = pf_recovery_reset(h); if (rc) return rc; }
    return pf_refresh_cache(h);
}
// a device temporary: released on every exit path (PF_CUDA / PF_LAUNCH return early on errors)
struct PfScopedBuf {
    void* p = nullptr;
    ~PfScopedBuf() { if (p) cudaFree(p); }
};
extern "C" int pfgpu_pf_upload(pfgpu_pf* h, const double* aos5, size_t n) {
    if (!h || !aos5 || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PfScopedBuf t;
    PF_CUDA(cudaMalloc(&t.p, n * 5 * sizeof(double)));
    double* tmp = (double*)t.p;
    PF_CUDA(cudaMemcpyAsync(tmp, aos5, n * 5 * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    PF_LAUNCH(h->ctx, pf_unpack_kernel, cdiv_u(n, PF_NT), PF_NT, 0, h->d, tmp);
    if (h->rec.on) { int rc = pf_recovery_reset(h); if (rc) return rc; }
    int rc = pf_refresh_cache(h);
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return rc;
}
extern "C" int pfgpu_pf_download(pfgpu_pf* h, double* aos5, size_t n) {
    if (!h || !aos5 || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PfScopedBuf t;
    PF_CUDA(cudaMalloc(&t.p, n * 5 * sizeof(double)));
    double* tmp = (double*)t.p;
    PF_LAUNCH(h->ctx, pf_pack_kernel, cdiv_u(n, PF_NT), PF_NT, 0, h->d, tmp);
    PF_CUDA(cudaMemcpyAsync(aos5, tmp, n * 5 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_pf_count(pfgpu_pf* h, size_t* nl, size_t* ng) {
    if (!h) return PFGPU_ERR_INVALID;
    if (nl) *nl = h->d.n;
    if (ng) *ng = h->d.n_global;
    return 0;
}

// d.obs with room for n doubles (its contents are dropped when it grows).  A failed allocation leaves no buffer and capacity 0,
// never a freed buffer under a capacity that claims it.
static int pf_obs_reserve(pfgpu_pf* h, size_t n) {
    if (n <= h->obs_cap) return 0;
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));                   // a queued launch may still read the old buffer
    cudaFree(h->d.obs);
    h->d.obs = nullptr; h->obs_cap = 0;
    double* p = nullptr;
    PF_CUDA(cudaMalloc(&p, 2 * n * sizeof(double)));
    h->d.obs = p; h->obs_cap = 2 * n;
    return 0;
}
static int pf_stage_obs(pfgpu_pf* h, const double* obs3, size_t k) {
    for (size_t j = 0; j < k; ++j)                                   // validate_observations pf.rs:538-549
        if (!finite_d(obs3[3 * j]) || !finite_d(obs3[3 * j + 1]) || !finite_d(obs3[3 * j + 2]) || obs3[3 * j] < 0.0)
            return PFGPU_ERR_INVALID;
    if (k <= PF_PARAM_OBS) return 0;                                 // short lists ride in the launch parameters
    int rc = pf_obs_reserve(h, 3 * k);
    if (rc) return rc;
    PF_CUDA(cudaMemcpyAsync(h->d.obs, obs3, k * 3 * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    return 0;
}
// the map slot of a scan model
template <int KIND>
static auto& pf_map(pfgpu_pf* h) {
    if constexpr (KIND == PF_KIND_BEAM) return h->bm;
    else return h->lf;
}
// A scan's used beams under the model KIND (its map must be loaded) -> h->pairs = (r_i, a_i); *k = their count.  Long lists go to
// d.obs.  Candidates i = 0, s, 2s, .. (AMCL's laser_max_beams stride); NaN or r <= 0 is unused (occupancy_grid_map.rs:84);
// r >= max_range is a max reading: unused, or with the model's keep_max used as r = max_range.
template <int KIND>
static int pf_stage_scan(pfgpu_pf* h, const double* ranges, size_t B, double angle_min, double angle_inc, size_t* k) {
    const auto& m = pf_map<KIND>(h);
    if (!m.on || (B && !ranges) || !finite_d(angle_min) || !finite_d(angle_inc)) return PFGPU_ERR_INVALID;
    const double max_range = m.cfg.max_range;
    std::vector<double>& pr = h->pairs;
    pr.clear();
    if (B) {
        const size_t s = std::max<size_t>(1, (B - 1) / (size_t)(m.cfg.max_beams - 1));
        for (size_t i = 0; i < B; i += s) {
            double r = ranges[i];
            if (r != r || r <= 0.0) continue;
            if (r >= max_range) {
                if (!m.keep_max()) continue;
                r = max_range;
            }
            pr.push_back(r);
            pr.push_back((double)i * angle_inc);
        }
    }
    *k = pr.size() / 2;
    if (*k > m.L) return PFGPU_ERR_INVALID;
    if (*k <= PF_PARAM_BEAMS) return 0;
    int rc = pf_obs_reserve(h, pr.size());
    if (rc) return rc;
    PF_CUDA(cudaMemcpyAsync(h->d.obs, pr.data(), pr.size() * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    return 0;
}
static PfScan pf_scan_arg(const pfgpu_pf* h, double angle_min) {
    PfScan s;
    s.q = h->lf.q; s.res = h->lf.cfg.resolution;
    s.half_w = (double)h->lf.W / 2.0; s.half_h = (double)h->lf.H / 2.0;
    s.q_out = h->lf.q_out; s.angle_min = angle_min;
    s.W = (int)h->lf.W; s.H = (int)h->lf.H;
    return s;
}
static PfBeam pf_beam_arg(const pfgpu_pf* h, double angle_min) {
    const pfgpu_beam_config& c = h->bm.cfg;
    PfBeam b;
    b.clr = h->bm.clr; b.res = c.resolution;
    b.half_w = (double)h->bm.W / 2.0; b.half_h = (double)h->bm.H / 2.0;
    b.max_range = c.max_range; b.angle_min = angle_min;
    b.hit = c.z_hit * (1.0 / sqrt(2.0 * PFC_PI * (c.sigma_hit * c.sigma_hit)));
    b.denom = 2.0 * (c.sigma_hit * c.sigma_hit);
    b.shrt = c.z_short * c.lambda_short; b.lambda = c.lambda_short;
    b.q_rand = c.z_rand / c.max_range; b.z_max = c.z_max;
    b.W = (int)h->bm.W; b.H = (int)h->bm.H; b.skip = h->bm.skip;
    return b;
}
// the smem a weight pass stages: k observations (d, lx, ly), or the beams (r, a) of a scan (a fixed size up to PF_PARAM_BEAMS,
// so that one captured scan step serves every beam count)
template <bool SCAN>
static size_t pf_obs_smem(size_t k) {
    if (SCAN) return (k <= PF_PARAM_BEAMS ? PF_PARAM_BEAMS : k) * 2 * sizeof(double);
    return (k ? k : 1) * 3 * sizeof(double);
}

// the injection arguments of the next predict (augmented MCL, DESIGN §3.8)
static PfInj pf_inj(const pfgpu_pf* h) {
    PfInj a = {};
    if (h->rec.on) { for (int j = 0; j < 4; ++j) a.r[j] = h->rec.region[j]; a.arm = h->rec.armed ? 1 : 0; }
    return a;
}
// The motion of a predict: the velocity model's control u (pf.rs:279-296, validated as validate_control pf.rs:515-523), or the
// odometry model's increment (DESIGN §3.14), computed once per call on the host from the two odometry poses and the handle's alphas
struct PfMotion {
    bool odom = false;
    double u[2] = { 0.0, 0.0 };
    PfOdom od = {};
};
static int pf_motion_velocity(const double u[2], PfMotion* m) {
    if (!u || !finite_d(u[0]) || !finite_d(u[1])) return PFGPU_ERR_INVALID;
    m->odom = false; m->u[0] = u[0]; m->u[1] = u[1];
    return 0;
}
static int pf_motion_odom(const pfgpu_pf* h, const double odom[6], PfMotion* m) {
    if (!odom || pf_odom_increment(odom, h->odom_alpha, &m->od) != 0) return PFGPU_ERR_INVALID;
    m->odom = true;
    return 0;
}
// out = (&a...): the kernelParams of a kernel with parameters P..., which the arguments must match type for type
template <class... P, class... A>
static void** pf_kernel_params(void** out, A&... a) {
    static_assert(sizeof...(P) == sizeof...(A) && (std::is_same<P, A>::value && ...), "arguments differ from the kernel's parameters");
    size_t i = 0;
    ((out[i++] = (void*)&a), ...);
    return out;
}
// pf_predict_weight_kernel's arguments in its parameter order.  The plain launch and the graph replay's node patch both pass
// params(kernel), so the two cannot diverge and the compiler checks them against the kernel.
struct PfMainArgs {
    PfDev d; PfObsParam po; double u0, u1, sv, sw, dt; uint64_t seed; uint32_t call; int k; double sigma; PfInj inj; PfScan sc;
    PfBeamParam pb; PfBeam bm; PfOdom od;
    void* p[16];
    template <class... P>
    void** params(void (*)(P...)) { return pf_kernel_params<P...>(p, d, po, u0, u1, sv, sw, dt, seed, call, k, sigma, inj, sc, pb, bm, od); }
};
// obs: k x (d, lx, ly), or for a scan (KIND != PF_KIND_LM) the k used beams (r, a) in h->pairs (angle_min: the scan's); lists
// short enough to ride in the launch parameters are copied there.  m = nullptr: no predict
template <int KIND>
static PfMainArgs pf_main_args(const pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    PfMainArgs a;
    if (KIND == PF_KIND_LM && k <= PF_PARAM_OBS) for (size_t j = 0; j < 3 * k; ++j) a.po.o[j] = obs3[j];
    if (KIND != PF_KIND_LM && k <= PF_PARAM_BEAMS)      // the first pairs in the observation block, the rest in pb
        for (size_t j = 0; j < 2 * k; ++j) (j < 3 * PF_PARAM_OBS ? a.po.o[j] : a.pb.b[j - 3 * PF_PARAM_OBS]) = h->pairs[j];
    a.d = h->d;
    a.u0 = m ? m->u[0] : 0.0; a.u1 = m ? m->u[1] : 0.0;
    a.od = m ? m->od : PfOdom{};
    a.sv = h->cfg.velocity_noise; a.sw = h->cfg.yaw_rate_noise; a.dt = h->cfg.dt; a.sigma = h->cfg.range_noise;
    a.seed = h->seed; a.call = h->n_predict; a.k = (int)k;
    a.inj = pf_inj(h);
    a.sc = KIND == PF_KIND_LF ? pf_scan_arg(h, angle_min) : PfScan{};
    a.bm = KIND == PF_KIND_BEAM ? pf_beam_arg(h, angle_min) : PfBeam{};
    return a;
}
template <bool P, bool W, bool INJ, int KIND, bool ODOM>
static int pf_launch_kernel(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    constexpr bool SCAN = KIND != PF_KIND_LM, BEAM = KIND == PF_KIND_BEAM;
    size_t smem = W ? pf_obs_smem<SCAN>(k) : 0;
    const bool param = !W || k <= (SCAN ? PF_PARAM_BEAMS : PF_PARAM_OBS);
    if (smem > 48 * 1024) {
        PF_CUDA(cudaFuncSetAttribute((pf_predict_weight_kernel<P, W, false, INJ, SCAN, BEAM, ODOM>), cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    }
    const auto kernel = param ? pf_predict_weight_kernel<P, W, true, INJ, SCAN, BEAM, ODOM> : pf_predict_weight_kernel<P, W, false, INJ, SCAN, BEAM, ODOM>;
    PfMainArgs a = pf_main_args<KIND>(h, m, obs3, k, angle_min);
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (h->timer.on) { PF_CUDA(cudaEventCreate(&e0)); PF_CUDA(cudaEventCreate(&e1)); PF_CUDA(cudaEventRecord(e0, h->ctx.stream)); }
    cudaLaunchKernel((const void*)kernel, cdiv_u(h->d.n, PF_NT), PF_NT, a.params(kernel), smem, h->ctx.stream);    // checked as PF_LAUNCH does
    h->ctx.launches++;
    PF_CUDA(cudaGetLastError());
    if (h->timer.on) { PF_CUDA(cudaEventRecord(e1, h->ctx.stream)); h->timer.pending.push_back({e0, e1}); }
    return 0;
}
template <bool P, bool W, int KIND, bool ODOM>
static int pf_launch_motion(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    if constexpr (P) {
        if (h->rec.on) {                                             // every predict counts its injections afresh
            PF_CUDA(cudaMemsetAsync(h->d.counters + PF_REC_COUNT, 0, sizeof(unsigned int), h->ctx.stream));
            return pf_launch_kernel<P, W, true, KIND, ODOM>(h, m, obs3, k, angle_min);
        }
    }
    return pf_launch_kernel<P, W, false, KIND, ODOM>(h, m, obs3, k, angle_min);
}
// m: the predict's motion (P), nullptr without a predict
template <bool P, bool W, int KIND = PF_KIND_LM>
static int pf_launch_main(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min = 0.0) {
    if constexpr (P) {
        if (m->odom) return pf_launch_motion<P, W, KIND, true>(h, m, obs3, k, angle_min);
    }
    return pf_launch_motion<P, W, KIND, false>(h, m, obs3, k, angle_min);
}
// augmented MCL's filter, right after S = sum w_raw has landed in scal[0]
static int pf_recovery_filter(pfgpu_pf* h) {
    if (h->rec.on) PF_LAUNCH(h->ctx, pf_recovery_filter_kernel, 1, 1, 0, h->d, h->rec.a_slow, h->rec.a_fast);
    return 0;
}
// normalize_weights: exact sequential sum of the raw weights, then the division pass
// global index search + pose gather of the sharded mode (pose_all = ncclAllGather of the 32-byte records, rank order)
__global__ void __launch_bounds__(PF_NT) pf_search_sharded_kernel(PfDev d, const double* cum_all, uint64_t seed, int mode) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= d.n) return;
    double r = pfc_u01_53(pfc_blk_u64(pfc_rng_block(seed, PFC_STREAM_PF_RESAMPLE, d.counters[0], d.offset + t), 0));
    size_t lo = 0, hi = d.n_global;
    while (lo < hi) {
        size_t mid = lo + ((hi - lo) >> 1);
        if (cum_all[mid] < r) lo = mid + 1; else hi = mid;
    }
    d.idx[t] = (uint32_t)(lo < d.n_global ? lo : (mode == 1 ? d.n_global - 1 : 0));
}
__global__ void __launch_bounds__(PF_NT) pf_gather_sharded_kernel(PfDev d, const Pose4* pose_all) {
    if (!*d.gate) return;
    const size_t t = (size_t)blockIdx.x * PF_NT + threadIdx.x;
    if (t >= d.n) return;
    Pose4 p;
    pose_load(pose_all, d.idx[t], p);
    pose_store(pf_pose(d, *d.cur ^ 1), t, p);
    d.w[t] = 1.0 / (double)d.n_global;
}
template <class F>
static int pf_total(pfgpu_pf* h, F f, double* out) {
    h->fu.last = false;
    if (h->world > 1) return xs_total_sharded(h->ctx, h->xs, h->sh, f, h->d.n, h->d.n_global, out);
    return xs_total(h->ctx, h->xs, f, h->d.n, h->d.n_global, 0.0, out);
}
static int pf_resample_sharded(pfgpu_pf* h) {
    PfDev& d = h->d; FsShard& sh = h->sh; Ctx& ctx = h->ctx;
    int rc = xs_total_sharded(ctx, h->xs, sh, PfValWSq{d.w}, d.n, d.n_global, d.scal + 1);          // calc_n_eff pf.rs:416-423
    if (rc) return rc;
    PF_LAUNCH(ctx, pf_gate_kernel, 1, 1, 0, d, h->cfg.resample_threshold, h->cfg.mode);
    int gate = 1;
    int* hp = reinterpret_cast<int*>(h->h_pin + 32);
    // the collectives below are host-enqueued: every rank must know the gate (MCL: always open, mcl.rs:298)
    PF_CUDA(cudaMemcpyAsync(hp, d.gate, sizeof(int), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaMemcpyAsync(hp + 1, sh.err, sizeof(int), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaStreamSynchronize(ctx.stream));
    if (hp[1]) { snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "sharded exact sum: a shard was not summarisable (degenerate weights)"); return PFGPU_ERR_UNSUPPORTED; }
    gate = *hp;
    if (!gate) return 0;
    rc = xs_scan_sharded(ctx, h->xs, sh, XsValArray{d.w}, XsSinkStore{d.cum}, d.n, d.n_global, d.scal + 2);   // pf.rs:448-453
    if (rc) return rc;
    if (h->cfg.mode == 1 && sh.rank == sh.world - 1) PF_LAUNCH(ctx, pf_force_last_kernel, 1, 1, 0, d);        // mcl.rs:334-336
    PF_NCCL(ncclAllGather(d.cum, sh.cum_all, d.n, ncclDouble, sh.comm, ctx.stream));
    PF_LAUNCH(ctx, pf_search_sharded_kernel, cdiv_u(d.n, PF_NT), PF_NT, 0, d, sh.cum_all, h->seed, h->cfg.mode);
    PF_NCCL(ncclAllGather(d.pose[h->cur_host], sh.pose_all, 4 * d.n, ncclDouble, sh.comm, ctx.stream));
    PF_LAUNCH(ctx, pf_gather_sharded_kernel, cdiv_u(d.n, PF_NT), PF_NT, 0, d, reinterpret_cast<const Pose4*>(sh.pose_all));
    PF_LAUNCH(ctx, pf_flip_kernel, 1, 1, 0, d);
    h->cur_host ^= 1;
    return 0;
}
static int pf_normalize(pfgpu_pf* h) {
    int rc = pf_total(h, XsValArray{h->d.w_raw}, h->d.scal + 0);
    if (rc) return rc;
    PF_LAUNCH(h->ctx, pf_normalize_kernel, cdiv_u(h->d.n, PF_NT), PF_NT, 0, h->d);
    return pf_recovery_filter(h);
}
// resample_adaptive with a changing particle count (mcl.rs:322-365), see pf_kld.cuh
static int pf_resample_adaptive(pfgpu_pf* h) {
    PfDev& d = h->d; PfKld& k = h->kld; Ctx& ctx = h->ctx;
    PF_LAUNCH(ctx, pf_gate_kernel, 1, 1, 0, d, h->cfg.resample_threshold, h->cfg.mode);           // MCL resamples every step (mcl.rs:298)
    int rc = xs_scan(ctx, h->xs, XsValArray{d.w}, XsSinkStore{d.cum}, d.n, d.n_global, 0.0, d.scal + 2);   // mcl.rs:328-333
    if (rc) return rc;
    PF_LAUNCH(ctx, pf_force_last_kernel, 1, 1, 0, d);                                             // mcl.rs:334-336
    PF_CUDA(cudaMemsetAsync(k.owner, 0xFF, (size_t)k.tcap * sizeof(int), ctx.stream));
    PF_CUDA(cudaMemsetAsync(k.mint, 0xFF, (size_t)k.tcap * sizeof(unsigned), ctx.stream));
    PF_LAUNCH(ctx, pf_kld_draw_kernel, cdiv_u(k.cap, PF_NT), PF_NT, 0, d, h->seed, k, h->xs.flags + 3);
    PF_LAUNCH(ctx, pf_kld_insert_kernel, cdiv_u(k.cap, PF_NT), PF_NT, 0, k);
    PF_LAUNCH(ctx, pf_kld_stop_kernel, 1, 1024, 0, k, (unsigned long long)h->cfg.n_particles, (unsigned long long)h->cfg.max_particles,
              h->cfg.kld_epsilon, h->cfg.kld_z);
    PF_LAUNCH(ctx, pf_kld_gather_kernel, cdiv_u(k.cap, PF_NT), PF_NT, 0, d, k);
    PF_LAUNCH(ctx, pf_flip_kernel, 1, 1, 0, d);
    unsigned* hp = reinterpret_cast<unsigned*>(h->h_pin + 34);
    PF_CUDA(cudaMemcpyAsync(hp, k.n_new, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaStreamSynchronize(ctx.stream));                    // the next launches are sized by the new count
    d.n = d.n_global = (size_t)*hp;
    return 0;
}
static int pf_resample_impl(pfgpu_pf* h) {
    PfDev& d = h->d;
    if (h->world > 1) return pf_resample_sharded(h);
    if (h->adaptive) return pf_resample_adaptive(h);
    int rc = pf_total(h, PfValWSq{d.w}, d.scal + 1);                                           // calc_n_eff pf.rs:416-423
    if (rc) return rc;
    PF_LAUNCH(h->ctx, pf_gate_kernel, 1, 1, 0, d, h->cfg.resample_threshold, h->cfg.mode);
    // cumulative weights (pf.rs:448-453), exact; the kernels below are no-ops when the gate is closed
    h->xs.gate = d.gate;
    rc = xs_scan(h->ctx, h->xs, XsValArray{d.w}, XsSinkStore{d.cum}, d.n, d.n_global, 0.0, d.scal + 2);
    h->xs.gate = nullptr;
    if (rc) return rc;
    if (h->cfg.mode == 1) PF_LAUNCH(h->ctx, pf_force_last_kernel, 1, 1, 0, d);
    PF_LAUNCH(h->ctx, pf_search_kernel, cdiv_u(d.n, PF_NT), PF_NT, 0, d, h->seed, h->cfg.mode, h->xs.flags + 3);
    PF_LAUNCH(h->ctx, pf_gather_kernel, cdiv_u(d.n, PF_NT), PF_NT, 0, d);
    PF_LAUNCH(h->ctx, pf_flip_kernel, 1, 1, 0, d);
    return 0;
}
// The resample draw counter (Philox "call" index) advances only when a resample happened; it lives on the
// device (PfDev::counters[0]) next to the gate, so a step needs no host round trip.
static int pf_read_gate(pfgpu_pf* h, int* gate) {
    int* hp = reinterpret_cast<int*>(h->h_pin + 32);
    PF_CUDA(cudaMemcpyAsync(hp, h->d.gate, sizeof(int), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    *gate = *hp;
    return 0;
}

static int pf_predict_impl(pfgpu_pf* h, const PfMotion& m) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int rc = pf_launch_main<true, false>(h, &m, nullptr, 0);
    if (rc) return rc;
    h->n_predict++;
    h->rec.armed = false;
    return pf_refresh_cache(h);                                                      // pf.rs:299
}
extern "C" int pfgpu_pf_predict(pfgpu_pf* h, const double u[2]) {
    PfMotion m;
    if (!h || pf_motion_velocity(u, &m)) return PFGPU_ERR_INVALID;                  // validate_control pf.rs:515-523
    return pf_predict_impl(h, m);
}
extern "C" int pfgpu_pf_predict_odom(pfgpu_pf* h, const double odom[6]) {
    PfMotion m;
    if (!h || pf_motion_odom(h, odom, &m)) return PFGPU_ERR_INVALID;
    return pf_predict_impl(h, m);
}
extern "C" int pfgpu_pf_set_odom_noise(pfgpu_pf* h, const double alpha[4]) {
    if (!h || !alpha || !pf_odom_alpha_ok(alpha)) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) h->odom_alpha[j] = alpha[j];
    return 0;
}
extern "C" int pfgpu_pf_odom_noise(pfgpu_pf* h, double alpha[4]) {
    if (!h || !alpha) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) alpha[j] = h->odom_alpha[j];
    return 0;
}
// try_update once the measurement is staged: landmarks obs3 (k x 3), or for a scan the k beams in h->pairs
template <int KIND>
static int pf_update_impl(pfgpu_pf* h, const double* obs3, size_t k, double angle_min) {
    int rc = pf_launch_main<false, true, KIND>(h, nullptr, obs3, k, angle_min);
    if (rc) return rc;
    h->rec.armed = false;                                                            // the weights are no longer uniform
    rc = pf_normalize(h);                                                            // pf.rs:331
    if (rc) return rc;
    return pf_refresh_cache(h);                                                      // pf.rs:332
}
extern "C" int pfgpu_pf_update(pfgpu_pf* h, const double* obs3, size_t k) {
    if (!h || (k && !obs3)) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int rc = pf_stage_obs(h, obs3, k);
    if (rc) return rc;
    return pf_update_impl<PF_KIND_LM>(h, obs3, k, 0.0);
}
extern "C" int pfgpu_pf_resample(pfgpu_pf* h, int* did) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int rc = pf_resample_impl(h);
    if (rc) return rc;
    h->rec.armed = true;
    rc = pf_refresh_cache(h);                                                        // pf.rs:343 (same values when the gate was closed)
    if (rc) return rc;
    if (did) { int g = 0; rc = pf_read_gate(h, &g); if (rc) return rc; *did = g; }
    return 0;
}
// a step's tail, from the raw weights in d.w_raw: normalise, gate, resample, refresh_cache (and augmented MCL's filter)
static int pf_step_tail(pfgpu_pf* h) {
    if (h->fu.on) {                                                                  // normalise .. refresh_cache: one launch (pf3.cuh)
        h->fu.arg.pd = h->d;
        h->fu.arg.threshold = h->cfg.resample_threshold;
        PF_LAUNCH(h->ctx, pf3_post_kernel<256>, h->fu.tiles, 256, h->fu.smem, h->fu.x, h->fu.arg);
        return pf_recovery_filter(h);                                                // S is in scal[0] once the launch ends
    }
    int rc = pf_normalize(h);
    if (rc) return rc;
    rc = pf_resample_impl(h);
    if (rc) return rc;
    return pf_refresh_cache(h);
}
// the launches of one fused step, in stream order (what the graph captures).  A scan's used beams are in h->pairs.
template <int KIND>
static int pf_step_launches(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    int rc = pf_launch_main<true, true, KIND>(h, m, obs3, k, angle_min);            // predict + likelihood, one pass
    if (rc) return rc;
    return pf_step_tail(h);
}
static void pf_graph_drop(pfgpu_pf* h) {
    if (h->sg.exec) cudaGraphExecDestroy(h->sg.exec);
    if (h->sg.graph) cudaGraphDestroy(h->sg.graph);
    h->sg.exec = nullptr; h->sg.graph = nullptr; h->sg.main_node = nullptr; h->sg.k = ~(size_t)0; h->sg.kind = PF_KIND_LM;
    h->sg.odom = false;
}
// the measurement kernel of a captured step (the injecting one while recovery is on; the odometry model's for an odometry step)
template <int KIND>
static auto pf_graph_kernel(const pfgpu_pf* h, bool odom) {
    constexpr bool SCAN = KIND != PF_KIND_LM, BEAM = KIND == PF_KIND_BEAM;
    if (odom)
        return h->rec.on ? pf_predict_weight_kernel<true, true, true, true, SCAN, BEAM, true>
                         : pf_predict_weight_kernel<true, true, true, false, SCAN, BEAM, true>;
    return h->rec.on ? pf_predict_weight_kernel<true, true, true, true, SCAN, BEAM> : pf_predict_weight_kernel<true, true, true, false, SCAN, BEAM>;
}
// capture the step at observation count k, or a scan step of either model (no work is executed by the capture itself)
template <int KIND>
static int pf_graph_capture(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    pf_graph_drop(h);
    const uint64_t l0 = h->ctx.launches;
    if (cudaStreamBeginCapture(h->ctx.stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return 1; }
    const int rc = pf_step_launches<KIND>(h, m, obs3, k, angle_min);
    cudaGraph_t g = nullptr;
    const cudaError_t e = cudaStreamEndCapture(h->ctx.stream, &g);
    h->sg.launches = h->ctx.launches - l0;
    h->ctx.launches = l0;
    if (rc || e != cudaSuccess || !g) { cudaGetLastError(); if (g) cudaGraphDestroy(g); return 1; }
    h->sg.graph = g;
    size_t nn = 0;
    if (cudaGraphGetNodes(g, nullptr, &nn) != cudaSuccess || nn == 0) { cudaGetLastError(); pf_graph_drop(h); return 1; }
    std::vector<cudaGraphNode_t> nodes(nn);
    if (cudaGraphGetNodes(g, nodes.data(), &nn) != cudaSuccess) { cudaGetLastError(); pf_graph_drop(h); return 1; }
    const void* want = (const void*)pf_graph_kernel<KIND>(h, m->odom);
    for (cudaGraphNode_t nd : nodes) {
        cudaGraphNodeType ty;
        if (cudaGraphNodeGetType(nd, &ty) != cudaSuccess || ty != cudaGraphNodeTypeKernel) continue;
        cudaKernelNodeParams kp = {};
        if (cudaGraphKernelNodeGetParams(nd, &kp) != cudaSuccess) continue;
        if (kp.func == want) { h->sg.main_node = nd; h->sg.main_params = kp; break; }
    }
    if (!h->sg.main_node || cudaGraphInstantiate(&h->sg.exec, g, 0) != cudaSuccess) { cudaGetLastError(); pf_graph_drop(h); return 1; }
    h->sg.k = k; h->sg.kind = KIND; h->sg.odom = m->odom;
    return 0;
}
// replay with this step's arguments patched into the first kernel
template <int KIND>
static int pf_graph_replay(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min) {
    PfMainArgs a = pf_main_args<KIND>(h, m, obs3, k, angle_min);
    cudaKernelNodeParams kp = h->sg.main_params;
    kp.kernelParams = a.params(pf_graph_kernel<KIND>(h, m->odom)); kp.extra = nullptr;
    PF_CUDA(cudaGraphExecKernelNodeSetParams(h->sg.exec, h->sg.main_node, &kp));
    PF_CUDA(cudaGraphLaunch(h->sg.exec, h->ctx.stream));
    h->ctx.launches += h->sg.launches;
    return 0;
}
// try_step once the measurement is staged: landmarks obs3 (k x 3), or for a scan the k beams in h->pairs
template <int KIND>
static int pf_step_impl(pfgpu_pf* h, const PfMotion* m, const double* obs3, size_t k, double angle_min, double est[4]) {
    int rc = 0;
    // graph replay: fixed particle count, one GPU, observations short enough to ride in the launch parameters, no per-kernel
    // timing events; the first step of a handle runs plainly (lazy set-up such as function attributes happens there).  The graph
    // is keyed by the kind of step (landmark / likelihood field / beam), the motion model (velocity / odometry) and, for landmark
    // steps, the observation count
    constexpr bool SCAN = KIND != PF_KIND_LM;
    const bool graphable = !h->sg.off && h->world == 1 && !h->adaptive && k <= (SCAN ? PF_PARAM_BEAMS : PF_PARAM_OBS) && !h->timer.on &&
                           h->steps > 0;
    bool done = false;
    if (graphable) {
        if (h->sg.exec && h->sg.kind == KIND && h->sg.odom == m->odom && (SCAN || h->sg.k == k)) done = true;
        else if (++h->sg.captures <= 16 && pf_graph_capture<KIND>(h, m, obs3, k, angle_min) == 0) done = true;
        else { h->sg.off = true; pf_graph_drop(h); }
        if (done) { rc = pf_graph_replay<KIND>(h, m, obs3, k, angle_min); if (rc) return rc; }
    }
    if (!done) { rc = pf_step_launches<KIND>(h, m, obs3, k, angle_min); if (rc) return rc; }
    h->fu.last = h->fu.on;
    h->n_predict++;
    h->steps++;
    h->rec.armed = true;                                                             // the step ended with its resample stage
    if (est) {
        PF_CUDA(cudaMemcpyAsync(h->h_pin, h->d.scal + 4, 4 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        for (int a = 0; a < 4; ++a) est[a] = h->h_pin[a];
    }
    return 0;
}
static int pf_lm_step(pfgpu_pf* h, const PfMotion& m, const double* obs3, size_t k, double est[4]) {
    if (k && !obs3) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int rc = pf_stage_obs(h, obs3, k);
    if (rc) return rc;
    return pf_step_impl<PF_KIND_LM>(h, &m, obs3, k, 0.0, est);
}
extern "C" int pfgpu_pf_step(pfgpu_pf* h, const double u[2], const double* obs3, size_t k, double est[4]) {
    PfMotion m;
    if (!h || pf_motion_velocity(u, &m)) return PFGPU_ERR_INVALID;
    return pf_lm_step(h, m, obs3, k, est);
}
extern "C" int pfgpu_pf_step_odom(pfgpu_pf* h, const double odom[6], const double* obs3, size_t k, double est[4]) {
    PfMotion m;
    if (!h || pf_motion_odom(h, odom, &m)) return PFGPU_ERR_INVALID;
    return pf_lm_step(h, m, obs3, k, est);
}
extern "C" int pfgpu_pf_estimate(pfgpu_pf* h, double est[4], double cov_cm[16]) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(h->h_pin, h->d.scal + 4, 20 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (est) for (int a = 0; a < 4; ++a) est[a] = h->h_pin[a];
    if (cov_cm) for (int a = 0; a < 4; ++a) for (int b = 0; b < 4; ++b) cov_cm[b * 4 + a] = h->h_pin[4 + a * 4 + b];
    return 0;
}
extern "C" int pfgpu_pf_neff(pfgpu_pf* h, double* neff) {
    if (!h || !neff) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int rc = pf_total(h, PfValWSq{h->d.w}, h->d.scal + 1);
    if (rc) return rc;
    PF_CUDA(cudaMemcpyAsync(h->h_pin, h->d.scal + 1, sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    double Q = h->h_pin[0];
    *neff = Q > 0.0 ? 1.0 / Q : 0.0;
    return 0;
}
extern "C" int pfgpu_pf_set_range_noise(pfgpu_pf* h, double s) {
    if (!h || !finite_d(s) || s <= 0.0) return PFGPU_ERR_INVALID;                   // pf.rs:228-236
    h->cfg.range_noise = s;
    return 0;
}
extern "C" int pfgpu_pf_last_indices(pfgpu_pf* h, uint32_t* idx, size_t cap, size_t* n) {
    if (!h || !idx) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    int gate = 0;
    { int rc = pf_read_gate(h, &gate); if (rc) return rc; }
    if (!gate) { if (n) *n = 0; return 0; }                   // the last step did not resample: no ancestry (as the oracle reports)
    size_t c = cap < h->d.n ? cap : h->d.n;
    PF_CUDA(cudaMemcpyAsync(idx, h->d.idx, c * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (n) *n = c;
    return 0;
}

// ---- augmented MCL: random-particle injection for global localisation and kidnapped-robot recovery (DESIGN §3.8) ----
extern "C" int pfgpu_pf_recovery_enable(pfgpu_pf* h, double alpha_slow, double alpha_fast, const double region[4]) {
    if (!h) return PFGPU_ERR_INVALID;
    const bool off = alpha_slow == 0.0 && alpha_fast == 0.0;
    if (!off && (!(alpha_slow > 0.0) || !(alpha_slow < alpha_fast) || !(alpha_fast <= 1.0) || !pf_region_ok(region))) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    pf_graph_drop(h);                          // the captured step holds the predict instantiation and the filter's alphas
    h->rec.on = !off;
    h->rec.a_slow = off ? 0.0 : alpha_slow; h->rec.a_fast = off ? 0.0 : alpha_fast;
    for (int j = 0; j < 4; ++j) h->rec.region[j] = off ? 0.0 : region[j];
    return pf_recovery_reset(h);
}
extern "C" int pfgpu_pf_recovery_state(pfgpu_pf* h, double out3[3], uint64_t* injected_last) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    double* hp = h->h_pin + 40;
    PF_CUDA(cudaMemcpyAsync(hp, h->d.scal + PF_REC_SLOW, 3 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(hp + 3, h->d.counters + PF_REC_COUNT, sizeof(unsigned int), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (out3) for (int j = 0; j < 3; ++j) out3[j] = hp[j];
    if (injected_last) { unsigned int c; memcpy(&c, hp + 3, sizeof(c)); *injected_last = c; }
    return 0;
}
extern "C" int pfgpu_pf_init_region(pfgpu_pf* h, const double region[4]) {
    if (!h || !pf_region_ok(region)) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    if (h->adaptive) h->d.n = h->d.n_global = h->cfg.n_particles;           // a fresh start: min_particles, like try_new
    PF_LAUNCH(h->ctx, pf_init_region_kernel, cdiv_u(h->d.n, PF_NT), PF_NT, 0, h->d, region[0], region[1], region[2], region[3], h->seed);
    if (h->rec.on) { int rc = pf_recovery_reset(h); if (rc) return rc; }
    return pf_refresh_cache(h);
}

// ---- scan models: localisation in an occupancy grid from a laser scan, under the likelihood field (DESIGN §3.9) or the beam
// model (DESIGN §3.11, pf_beam.cuh).  Each model has its own map slot; a map is built from a host mask or a grid's (DESIGN §3.12) ----
#define PF_LF_MAX_L 4096           // the beams a scan may use at most (their (r, a) pairs are staged in shared memory)
// L: the largest count <= PF_LF_MAX_L with q_lo^(L+1) >= DBL_MIN and q_hi^(L+1) <= DBL_MAX, powers by repeated multiplication
static uint64_t pf_lf_limit(double q_lo, double q_hi) {
    double pmin = 1.0, pmax = 1.0;
    uint64_t L = 0;
    for (uint64_t m = 1; m <= PF_LF_MAX_L + 1; ++m) {
        pmin = pmin * q_lo;
        pmax = pmax * q_hi;
        if (!(pmin >= DBL_MIN) || !(pmax <= DBL_MAX)) break;
        L = m - 1;
    }
    return L;
}
static bool pf_map_shape_ok(size_t W, size_t H) { return W >= 1 && H >= 1 && W <= 65536 && H <= 65536 && W * H <= ((size_t)1 << 28); }
// the likelihood field's config check; its beam bound L and q_out
static int pf_lf_check(size_t W, size_t H, const pfgpu_lfield_config* c, uint64_t* L, double* q_out) {
    if (!pf_map_shape_ok(W, H)) return PFGPU_ERR_INVALID;
    auto positive = [](double v) { return finite_d(v) && v > 0.0; };
    if (!positive(c->resolution) || !positive(c->sigma_hit) || !positive(c->z_rand) || !positive(c->max_range) || !finite_d(c->z_hit) ||
        c->z_hit < 0.0 || c->max_beams < 2)
        return PFGPU_ERR_INVALID;
    *q_out = c->z_rand / c->max_range;
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (c->sigma_hit * c->sigma_hit));
    *L = pf_lf_limit(*q_out, c->z_hit * coeff + *q_out);
    return *L < 1 ? PFGPU_ERR_INVALID : 0;
}
// the beam model's config check; its beam bound L
static int pf_beam_check(size_t W, size_t H, const pfgpu_beam_config* c, uint64_t* Lout) {
    if (!pf_map_shape_ok(W, H)) return PFGPU_ERR_INVALID;
    auto positive = [](double v) { return finite_d(v) && v > 0.0; };
    auto nonneg = [](double v) { return finite_d(v) && v >= 0.0; };
    if (!positive(c->resolution) || !positive(c->sigma_hit) || !positive(c->z_rand) || !positive(c->max_range) ||
        !positive(c->lambda_short) || !nonneg(c->z_hit) || !nonneg(c->z_short) || !nonneg(c->z_max) || c->max_beams < 2 ||
        !(c->max_range / c->resolution <= 1048576.0))
        return PFGPU_ERR_INVALID;
    const double q_rand = c->z_rand / c->max_range;
    const double coeff = 1.0 / sqrt(2.0 * PFC_PI * (c->sigma_hit * c->sigma_hit));
    const double q_lo = c->z_max > 0.0 ? std::min(q_rand, c->z_max) : q_rand;
    const double q_hi = c->z_hit * coeff + c->z_short * c->lambda_short + std::max(q_rand, c->z_max);
    *Lout = pf_lf_limit(q_lo, q_hi);
    return *Lout < 1 ? PFGPU_ERR_INVALID : 0;
}
static int pf_ogm_mask(const pfgpu_ogm* g, double threshold, unsigned char* mask_dev, Ctx& ctx);
// the obstacle mask of a map being set, into m on the handle's device: the host mask uploaded, or with a grid its mask at threshold
static int pf_map_mask(pfgpu_pf* h, const uint8_t* mask, const pfgpu_ogm* grid, double threshold, size_t cells, PfScopedBuf& m) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMalloc(&m.p, cells));
    if (grid) return pf_ogm_mask(grid, threshold, (unsigned char*)m.p, h->ctx);
    PF_CUDA(cudaMemcpyAsync(m.p, mask, cells, cudaMemcpyHostToDevice, h->ctx.stream));
    return 0;
}
// unload slot m's map, and drop the captured step, which holds its tables' addresses
template <class M>
static int pf_map_clear(pfgpu_pf* h, M& m) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    pf_graph_drop(h);
    m.release();
    return 0;
}
// Replace slot m's map by a W x H one with beam bound L and config c, from an obstacle mask (pf_map_mask's arguments): build(mask)
// allocates the model's tables, enqueues their construction and records what else the model derives at set time
template <class M, class Cfg, class Build>
static int pf_map_load(pfgpu_pf* h, M& m, const uint8_t* mask, const pfgpu_ogm* grid, double threshold, size_t W, size_t H, uint64_t L,
                       const Cfg& c, Build build) {
    PfScopedBuf mask_dev;
    int rc = pf_map_mask(h, mask, grid, threshold, W * H, mask_dev);
    if (!rc) rc = pf_map_clear(h, m);
    if (!rc) rc = build((const unsigned char*)mask_dev.p);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    m.W = W; m.H = H; m.L = L; m.cfg = c;
    m.on = true;
    return 0;
}
static int pf_map_info(const PfMap& m, size_t* W, size_t* H, uint64_t* L) {
    if (W) *W = m.W;
    if (H) *H = m.H;
    if (L) *L = m.L;
    return 0;
}
// the likelihood field: the distance field and the factor table
static int pf_lf_set(pfgpu_pf* h, const uint8_t* mask, const pfgpu_ogm* grid, double threshold, size_t W, size_t H,
                     const pfgpu_lfield_config* c) {
    uint64_t L = 0;
    double q_out = 0.0;
    const int rc = pf_lf_check(W, H, c, &L, &q_out);
    if (rc) return rc;
    const size_t cells = W * H, scratch = std::max(W * (H + 1), H * (W + 1));
    PfScopedBuf v, z;                          // freed after the load's last synchronise
    auto& f = h->lf;
    return pf_map_load(h, f, mask, grid, threshold, W, H, L, *c, [&](const unsigned char* mask_dev) -> int {
        PF_CUDA(cudaMalloc(&f.D, cells * sizeof(double)));
        PF_CUDA(cudaMalloc(&f.q, cells * sizeof(double)));
        PF_CUDA(cudaMalloc(&v.p, scratch * sizeof(int)));
        PF_CUDA(cudaMalloc(&z.p, scratch * sizeof(double)));
        // rows into q (as scratch), columns into D, then D = sqrt and the factor table
        PF_LAUNCH(h->ctx, pf_lf_edt_rows_kernel, cdiv_u(W, 32), 32, 0, mask_dev, f.q, (int)W, (int)H, (int*)v.p, (double*)z.p);
        PF_LAUNCH(h->ctx, pf_lf_edt_cols_kernel, cdiv_u(H, 32), 32, 0, f.q, f.D, (int)W, (int)H, (int*)v.p, (double*)z.p);
        PF_LAUNCH(h->ctx, pf_lf_table_kernel, cdiv_u(cells, 256), 256, 0, f.D, f.q, cells, c->resolution, c->sigma_hit, c->z_hit, q_out);
        f.q_out = q_out;
        return 0;
    });
}
// the beam model: the clearance table
static int pf_beam_set(pfgpu_pf* h, const uint8_t* mask, const pfgpu_ogm* grid, double threshold, size_t W, size_t H,
                       const pfgpu_beam_config* c) {
    uint64_t L = 0;
    const int rc = pf_beam_check(W, H, c, &L);
    if (rc) return rc;
    const size_t cells = W * H;
    PfScopedBuf tmp;                           // freed after the load's last synchronise
    auto& b = h->bm;
    return pf_map_load(h, b, mask, grid, threshold, W, H, L, *c, [&](const unsigned char* mask_dev) -> int {
        PF_CUDA(cudaMalloc(&b.clr, cells));
        PF_CUDA(cudaMalloc(&tmp.p, cells));
        PF_LAUNCH(h->ctx, pf_beam_clr_lines_kernel, cdiv_u(cells, 256), 256, 0, mask_dev, (unsigned char*)tmp.p, (int)W, (int)H);
        PF_LAUNCH(h->ctx, pf_beam_clr_cols_kernel, cdiv_u(cells, 256), 256, 0, (const unsigned char*)tmp.p, b.clr, (int)W, (int)H);
        const char* e = getenv("PFGPU_BEAM_SKIP");
        b.skip = (e && e[0] == '0') ? 0 : 1;
        return 0;
    });
}
// the update and the step from a laser scan under the model KIND
template <int KIND>
static int pf_scan_update(pfgpu_pf* h, const double* ranges, size_t B, double angle_min, double angle_inc) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    size_t k = 0;
    int rc = pf_stage_scan<KIND>(h, ranges, B, angle_min, angle_inc, &k);
    if (rc) return rc;
    return pf_update_impl<KIND>(h, nullptr, k, angle_min);
}
template <int KIND>
static int pf_scan_step(pfgpu_pf* h, const PfMotion& m, const double* ranges, size_t B, double angle_min, double angle_inc, double est[4]) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    size_t k = 0;
    int rc = pf_stage_scan<KIND>(h, ranges, B, angle_min, angle_inc, &k);
    if (rc) return rc;
    return pf_step_impl<KIND>(h, &m, nullptr, k, angle_min, est);
}
// the step from a laser scan under the model KIND with the velocity model's control u, or with the odometry pair odom
template <int KIND>
static int pf_scan_step_u(pfgpu_pf* h, const double u[2], const double* ranges, size_t B, double angle_min, double angle_inc, double est[4]) {
    PfMotion m;
    if (!h || pf_motion_velocity(u, &m)) return PFGPU_ERR_INVALID;
    return pf_scan_step<KIND>(h, m, ranges, B, angle_min, angle_inc, est);
}
template <int KIND>
static int pf_scan_step_odom(pfgpu_pf* h, const double odom[6], const double* ranges, size_t B, double angle_min, double angle_inc,
                             double est[4]) {
    PfMotion m;
    if (!h || pf_motion_odom(h, odom, &m)) return PFGPU_ERR_INVALID;
    return pf_scan_step<KIND>(h, m, ranges, B, angle_min, angle_inc, est);
}

extern "C" int pfgpu_pf_lfield_set(pfgpu_pf* h, const uint8_t* mask, size_t W, size_t H, const pfgpu_lfield_config* c) {
    if (!h || !mask || !c) return PFGPU_ERR_INVALID;
    return pf_lf_set(h, mask, nullptr, 0.0, W, H, c);
}
extern "C" int pfgpu_pf_lfield_clear(pfgpu_pf* h) { return h ? pf_map_clear(h, h->lf) : PFGPU_ERR_INVALID; }
extern "C" int pfgpu_pf_lfield_info(pfgpu_pf* h, size_t* W, size_t* H, uint64_t* L) { return h ? pf_map_info(h->lf, W, H, L) : PFGPU_ERR_INVALID; }
extern "C" int pfgpu_pf_lfield_download(pfgpu_pf* h, double* D, double* q, size_t cells) {
    if (!h || !h->lf.on || cells != h->lf.W * h->lf.H) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    if (D) PF_CUDA(cudaMemcpyAsync(D, h->lf.D, cells * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    if (q) PF_CUDA(cudaMemcpyAsync(q, h->lf.q, cells * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_pf_update_scan(pfgpu_pf* h, const double* ranges, size_t B, double angle_min, double angle_inc) {
    return pf_scan_update<PF_KIND_LF>(h, ranges, B, angle_min, angle_inc);
}
extern "C" int pfgpu_pf_step_scan(pfgpu_pf* h, const double u[2], const double* ranges, size_t B, double angle_min, double angle_inc,
                                  double est[4]) {
    return pf_scan_step_u<PF_KIND_LF>(h, u, ranges, B, angle_min, angle_inc, est);
}
extern "C" int pfgpu_pf_step_scan_odom(pfgpu_pf* h, const double odom[6], const double* ranges, size_t B, double angle_min,
                                       double angle_inc, double est[4]) {
    return pf_scan_step_odom<PF_KIND_LF>(h, odom, ranges, B, angle_min, angle_inc, est);
}

extern "C" int pfgpu_pf_beam_set(pfgpu_pf* h, const uint8_t* mask, size_t W, size_t H, const pfgpu_beam_config* c) {
    if (!h || !mask || !c) return PFGPU_ERR_INVALID;
    return pf_beam_set(h, mask, nullptr, 0.0, W, H, c);
}
extern "C" int pfgpu_pf_beam_clear(pfgpu_pf* h) { return h ? pf_map_clear(h, h->bm) : PFGPU_ERR_INVALID; }
extern "C" int pfgpu_pf_beam_info(pfgpu_pf* h, size_t* W, size_t* H, uint64_t* L) { return h ? pf_map_info(h->bm, W, H, L) : PFGPU_ERR_INVALID; }
extern "C" int pfgpu_pf_beam_download(pfgpu_pf* h, uint8_t* clearance, size_t cells) {
    if (!h || !h->bm.on || !clearance || cells != h->bm.W * h->bm.H) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(clearance, h->bm.clr, cells, cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_pf_update_beam(pfgpu_pf* h, const double* ranges, size_t B, double angle_min, double angle_inc) {
    return pf_scan_update<PF_KIND_BEAM>(h, ranges, B, angle_min, angle_inc);
}
extern "C" int pfgpu_pf_step_beam(pfgpu_pf* h, const double u[2], const double* ranges, size_t B, double angle_min, double angle_inc,
                                  double est[4]) {
    return pf_scan_step_u<PF_KIND_BEAM>(h, u, ranges, B, angle_min, angle_inc, est);
}
extern "C" int pfgpu_pf_step_beam_odom(pfgpu_pf* h, const double odom[6], const double* ranges, size_t B, double angle_min,
                                       double angle_inc, double est[4]) {
    return pf_scan_step_odom<PF_KIND_BEAM>(h, odom, ranges, B, angle_min, angle_inc, est);
}
extern "C" int pfgpu_pf_beam_raycast(pfgpu_pf* h, const double* poses3, size_t n, size_t B, double angle_min, double angle_inc,
                                     double* out) {
    if (!h || !h->bm.on || !finite_d(angle_min) || !finite_d(angle_inc)) return PFGPU_ERR_INVALID;
    if (n == 0 || B == 0) return 0;
    if (!poses3 || !out || n > ((size_t)1 << 40) / B) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PfScopedBuf dp, dout;
    PF_CUDA(cudaMalloc(&dp.p, n * 3 * sizeof(double)));
    PF_CUDA(cudaMalloc(&dout.p, n * B * sizeof(double)));
    PF_CUDA(cudaMemcpyAsync(dp.p, poses3, n * 3 * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    PF_LAUNCH(h->ctx, pf_beam_raycast_kernel, cdiv_u(n * B, 256), 256, 0, pf_beam_arg(h, angle_min), (const double*)dp.p, n, B, angle_inc,
              (double*)dout.p);
    PF_CUDA(cudaMemcpyAsync(out, dout.p, n * B * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}

// ====================================================================================================
// Occupancy grid mapping (DESIGN §3.12, ogm.cuh)
// ====================================================================================================
struct pfgpu_ogm {
    Ctx ctx;
    pfgpu_ogm_config cfg = {};
    size_t W = 0, H = 0;
    double* grid = nullptr;            // [W * H], ix * H + iy
    unsigned long long cap = PF_OGM_EVENT_CAP;
    // the event workspace, allocated by the first update (DESIGN §3.12 gives its size)
    int4* geo = nullptr;               // [PF_OGM_BEAM_CAP] per beam of a window: origin, end cell
    unsigned long long* cnt = nullptr; // [PF_OGM_BEAM_CAP] events per beam
    unsigned long long* incl = nullptr;// [PF_OGM_BEAM_CAP] their inclusive sum
    unsigned int* keys[2] = {nullptr, nullptr};   // [cap] each: the radix sort's double buffer
    void* tmp = nullptr;               // CUB temporary storage
    size_t tmp_bytes = 0;
    unsigned long long* scal = nullptr;// [4] device: chunk end, chunk events, longest run (as u32)
    unsigned long long* h_pin = nullptr;   // [4] pinned host
    pfgpu_ogm_stats st = {};
};

static void pf_ogm_free(pfgpu_ogm* g) {
    cudaFree(g->grid); cudaFree(g->geo); cudaFree(g->cnt); cudaFree(g->incl); cudaFree(g->keys[0]); cudaFree(g->keys[1]);
    cudaFree(g->tmp); cudaFree(g->scal);
    if (g->h_pin) cudaFreeHost(g->h_pin);
    if (g->ctx.stream) cudaStreamDestroy(g->ctx.stream);
}
extern "C" void pfgpu_ogm_destroy(pfgpu_ogm* g) {
    if (!g) return;
    cudaSetDevice(g->ctx.device);
    if (g->ctx.stream) cudaStreamSynchronize(g->ctx.stream);
    pf_ogm_free(g);
    delete g;
}
extern "C" int pfgpu_ogm_create(const pfgpu_ogm_config* c, int device, pfgpu_ogm** out) {
    if (!c || !out) return PFGPU_ERR_INVALID;
    *out = nullptr;
    if (c->width > 65536 || c->height > 65536 || !pf_map_shape_ok((size_t)c->width, (size_t)c->height) || !finite_d(c->resolution) ||
        !(c->resolution > 0.0) || !finite_d(c->prior_log_odds) || !finite_d(c->occupied_log_odds) || !finite_d(c->free_log_odds) ||
        !finite_d(c->max_log_odds) || !finite_d(c->min_log_odds) || !(c->min_log_odds <= c->max_log_odds))
        return PFGPU_ERR_INVALID;
    pfgpu_ogm* g = new (std::nothrow) pfgpu_ogm();
    if (!g) return PFGPU_ERR_CUDA;
    g->cfg = *c;
    g->W = (size_t)c->width; g->H = (size_t)c->height;
    const char* e = getenv("PFGPU_OGM_EVENT_CAP");   // a smaller cap (at least 65536) forces chunking, for tests
    if (e && *e) g->cap = std::max<unsigned long long>(65536ull, std::min<unsigned long long>(strtoull(e, nullptr, 10), PF_OGM_EVENT_CAP));
    const int orc = ctx_open(g->ctx, device);
    if (orc) { pf_ogm_free(g); delete g; return orc; }
    auto fail = [&](cudaError_t err, int line) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s:%d: ogm create -> %s", __FILE__, line, cudaGetErrorString(err));
        pf_ogm_free(g);
        delete g;
        return PFGPU_ERR_CUDA;
    };
    cudaError_t err;
    const size_t cells = g->W * g->H;
    if ((err = cudaMalloc(&g->grid, cells * sizeof(double))) != cudaSuccess) return fail(err, __LINE__);
    pf_ogm_fill_kernel<<<cdiv_u(cells, 256), 256, 0, g->ctx.stream>>>(g->grid, cells, c->prior_log_odds);
    g->ctx.launches++;
    if ((err = cudaGetLastError()) != cudaSuccess || (err = cudaStreamSynchronize(g->ctx.stream)) != cudaSuccess) return fail(err, __LINE__);
    *out = g;
    return 0;
}
// the bits the radix sort compares for cells 0 .. cells - 1: ceil(log2 cells), at least 1
static int pf_ogm_bits(size_t cells) {
    int b = 1;
    while (b < 28 && ((size_t)1 << b) < cells) ++b;
    return b;
}
static int pf_ogm_alloc(pfgpu_ogm* g) {
    PF_CUDA(cudaMalloc(&g->geo, PF_OGM_BEAM_CAP * sizeof(int4)));
    PF_CUDA(cudaMalloc(&g->cnt, PF_OGM_BEAM_CAP * sizeof(unsigned long long)));
    PF_CUDA(cudaMalloc(&g->incl, PF_OGM_BEAM_CAP * sizeof(unsigned long long)));
    PF_CUDA(cudaMalloc(&g->keys[0], g->cap * sizeof(unsigned int)));
    PF_CUDA(cudaMalloc(&g->keys[1], g->cap * sizeof(unsigned int)));
    PF_CUDA(cudaMalloc(&g->scal, 4 * sizeof(unsigned long long)));
    PF_CUDA(cudaMallocHost(&g->h_pin, 4 * sizeof(unsigned long long)));
    size_t b0 = 0, b1 = 0;
    cub::DoubleBuffer<unsigned int> db(g->keys[0], g->keys[1]);
    PF_CUDA(cub::DeviceScan::InclusiveSum(nullptr, b0, g->cnt, g->incl, (int)PF_OGM_BEAM_CAP, g->ctx.stream));
    PF_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, b1, db, (int)g->cap, 0, pf_ogm_bits(g->W * g->H), g->ctx.stream));
    g->tmp_bytes = std::max(b0, b1);
    PF_CUDA(cudaMalloc(&g->tmp, g->tmp_bytes));
    return 0;
}
extern "C" int pfgpu_ogm_update_scans(pfgpu_ogm* g, const double* poses3, size_t S, const double* ranges, size_t B, double angle_min,
                                      double angle_inc) {
    if (!g) return PFGPU_ERR_INVALID;
    g->st.events = g->st.chunks = g->st.longest_run = 0;
    g->st.event_cap = g->cap;
    if (S == 0 || B == 0) return 0;
    if (!poses3 || !ranges || S > ((size_t)1 << 40) / B) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(g->ctx.device));
    if (!g->keys[0]) {
        const int rc = pf_ogm_alloc(g);
        if (rc) {
            cudaFree(g->geo); cudaFree(g->cnt); cudaFree(g->incl); cudaFree(g->keys[0]); cudaFree(g->keys[1]); cudaFree(g->tmp);
            cudaFree(g->scal);
            if (g->h_pin) cudaFreeHost(g->h_pin);
            g->geo = nullptr; g->cnt = g->incl = g->scal = g->h_pin = nullptr; g->keys[0] = g->keys[1] = nullptr; g->tmp = nullptr;
            return rc;
        }
    }
    Ctx& ctx = g->ctx;
    const size_t NB = S * B;
    PfScopedBuf dp, dr;
    PF_CUDA(cudaMalloc(&dp.p, S * 3 * sizeof(double)));
    PF_CUDA(cudaMalloc(&dr.p, NB * sizeof(double)));
    PF_CUDA(cudaMemcpyAsync(dp.p, poses3, S * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    PF_CUDA(cudaMemcpyAsync(dr.p, ranges, NB * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    PF_CUDA(cudaMemsetAsync(g->scal + 2, 0, sizeof(unsigned long long), ctx.stream));
    PfOgmGeom gm;
    gm.res = g->cfg.resolution; gm.half_w = (double)g->W / 2.0; gm.half_h = (double)g->H / 2.0; gm.W = (int)g->W; gm.H = (int)g->H;
    const int bits = pf_ogm_bits(g->W * g->H);
    const pfgpu_ogm_config& c = g->cfg;
    for (size_t w0 = 0; w0 < NB; w0 += PF_OGM_BEAM_CAP) {
        const size_t nb = std::min<size_t>(PF_OGM_BEAM_CAP, NB - w0);
        PF_LAUNCH(ctx, pf_ogm_count_kernel, cdiv_u(nb, 256), 256, 0, gm, (const double*)dp.p, (const double*)dr.p, B, w0, nb, angle_min,
                  angle_inc, g->geo, g->cnt);
        size_t tb = g->tmp_bytes;
        PF_CUDA(cub::DeviceScan::InclusiveSum(g->tmp, tb, g->cnt, g->incl, (int)nb, ctx.stream));
        unsigned long long base = 0;
        for (size_t b = 0; b < nb;) {
            PF_LAUNCH(ctx, pf_ogm_chunk_kernel, 1, 1, 0, (const unsigned long long*)g->incl, b, nb, base, g->cap, g->scal);
            PF_CUDA(cudaMemcpyAsync(g->h_pin, g->scal, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx.stream));
            PF_CUDA(cudaStreamSynchronize(ctx.stream));
            const size_t e = (size_t)g->h_pin[0];
            const unsigned long long E = g->h_pin[1];
            if (E > 0) {
                PF_LAUNCH(ctx, pf_ogm_emit_kernel, cdiv_u((e - b) * 32, 256), 256, 0, (const int4*)g->geo, (const unsigned long long*)g->incl,
                          b, e, base, (int)g->H, g->keys[0]);
                cub::DoubleBuffer<unsigned int> db(g->keys[0], g->keys[1]);
                PF_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, tb, db, (int)E, 0, bits, ctx.stream));
                if (tb > g->tmp_bytes) {
                    snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "ogm: radix sort of %llu keys wants %zu temporary bytes, %zu allocated", E, tb,
                             g->tmp_bytes);
                    return PFGPU_ERR_CUDA;
                }
                PF_CUDA(cub::DeviceRadixSort::SortKeys(g->tmp, tb, db, (int)E, 0, bits, ctx.stream));
                PF_LAUNCH(ctx, pf_ogm_fold_kernel, cdiv_u(E, 256), 256, 0, (const unsigned int*)db.Current(), (size_t)E, g->grid,
                          c.occupied_log_odds, c.free_log_odds, c.min_log_odds, c.max_log_odds, (unsigned int*)(g->scal + 2));
                g->st.events += E;
                g->st.chunks += 1;
            }
            base += E;
            b = e;
        }
    }
    PF_CUDA(cudaMemcpyAsync(g->h_pin + 2, g->scal + 2, sizeof(unsigned long long), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaStreamSynchronize(ctx.stream));
    g->st.longest_run = g->h_pin[2];
    return 0;
}
extern "C" int pfgpu_ogm_set(pfgpu_ogm* g, const double* grid, size_t cells) {
    if (!g || !grid || cells != g->W * g->H) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(g->ctx.device));
    PF_CUDA(cudaMemcpyAsync(g->grid, grid, cells * sizeof(double), cudaMemcpyHostToDevice, g->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(g->ctx.stream));
    return 0;
}
extern "C" int pfgpu_ogm_read(pfgpu_ogm* g, size_t first, size_t count, double* out) {
    if (!g || first > g->W * g->H || count > g->W * g->H - first || (count && !out)) return PFGPU_ERR_INVALID;
    if (count == 0) return 0;
    PF_CUDA(cudaSetDevice(g->ctx.device));
    PF_CUDA(cudaMemcpyAsync(out, g->grid + first, count * sizeof(double), cudaMemcpyDeviceToHost, g->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(g->ctx.stream));
    return 0;
}
// the obstacle mask of g at `threshold` into mask_dev (cells bytes on g's device), enqueued on `ctx`'s stream after g's work
static int pf_ogm_mask(const pfgpu_ogm* g, double threshold, unsigned char* mask_dev, Ctx& ctx) {
    PF_CUDA(cudaStreamSynchronize(g->ctx.stream));
    const size_t cells = g->W * g->H;
    PF_LAUNCH(ctx, pf_ogm_mask_kernel, cdiv_u(cells, 256), 256, 0, (const double*)g->grid, cells, threshold, mask_dev);
    return 0;
}
extern "C" int pfgpu_ogm_obstacles(pfgpu_ogm* g, double threshold, uint8_t* mask_out, size_t cells) {
    if (!g || !mask_out || cells != g->W * g->H || !finite_d(threshold)) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(g->ctx.device));
    PfScopedBuf m;
    PF_CUDA(cudaMalloc(&m.p, cells));
    int rc = pf_ogm_mask(g, threshold, (unsigned char*)m.p, g->ctx);
    if (rc) return rc;
    PF_CUDA(cudaMemcpyAsync(mask_out, m.p, cells, cudaMemcpyDeviceToHost, g->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(g->ctx.stream));
    return 0;
}
extern "C" int pfgpu_ogm_info(pfgpu_ogm* g, size_t* W, size_t* H, pfgpu_ogm_stats* st) {
    if (!g) return PFGPU_ERR_INVALID;
    if (W) *W = g->W;
    if (H) *H = g->H;
    if (st) { *st = g->st; st->event_cap = g->cap; }
    return 0;
}
// a grid handed to a PF handle: on its device, at the model's resolution
static bool pf_grid_ok(const pfgpu_pf* h, const pfgpu_ogm* g, double threshold, double resolution) {
    return g && finite_d(threshold) && g->ctx.device == h->ctx.device && resolution == g->cfg.resolution;
}
extern "C" int pfgpu_pf_lfield_set_grid(pfgpu_pf* h, const pfgpu_ogm* grid, double threshold, const pfgpu_lfield_config* c) {
    if (!h || !c || !pf_grid_ok(h, grid, threshold, c->resolution)) return PFGPU_ERR_INVALID;
    return pf_lf_set(h, nullptr, grid, threshold, grid->W, grid->H, c);
}
extern "C" int pfgpu_pf_beam_set_grid(pfgpu_pf* h, const pfgpu_ogm* grid, double threshold, const pfgpu_beam_config* c) {
    if (!h || !c || !pf_grid_ok(h, grid, threshold, c->resolution)) return PFGPU_ERR_INVALID;
    return pf_beam_set(h, nullptr, grid, threshold, grid->W, grid->H, c);
}

// ====================================================================================================
// Grid-based FastSLAM (DESIGN §3.16): gslam_host.cuh (entry points) + gslam.cuh (kernels)
// ====================================================================================================
#include "gslam_host.cuh"

// ====================================================================================================
// Correlative scan matching (DESIGN §3.13, csm.cuh)
// ====================================================================================================
#define PF_CSM_WS_CAP ((size_t)1 << 28)         // bytes of cell indices per launch (X and Y)
#define PF_CSM_PART_CAP ((size_t)1 << 20)       // block bests per launch
struct pfgpu_csm {
    Ctx ctx;
    double* rx = nullptr;               // [ncap] reference points
    double* ry = nullptr;
    size_t n = 0, ncap = 0;
    unsigned long long* table = nullptr;// [tcap] f64 bits, (ix - ox) * TH + (iy - oy)
    size_t tcap = 0;
    bool table_ok = false;
    double table_res = 0.0;
    long long ox = 0, oy = 0, TW = 0, TH = 0;
    int R = 0;
    int* X = nullptr;                   // [ws_ints] cell indices of one launch
    int* Y = nullptr;
    size_t ws_ints = 0;
    double2* cs = nullptr;              // [cs_cap] (cos, sin) per (query, yaw) of a launch
    size_t cs_cap = 0;
    PfCsmBest* part = nullptr;          // [PF_CSM_PART_CAP] block bests
    PfCsmBest* best = nullptr;          // [best_cap] per query
    size_t best_cap = 0;
    int* ext = nullptr;                 // [5] device: extent and the out-of-range flag
    int* h_ext = nullptr;               // [5] pinned host
    size_t ws_cap = PF_CSM_WS_CAP;
    // pfgpu_csm_set_reference_grid's buffers, kept between calls (a mapping loop sets the reference once per step)
    unsigned char* gmask = nullptr;     // [gmask_cap] obstacle mask
    size_t gmask_cap = 0;
    unsigned int* gidx = nullptr;       // [gidx_cap] compacted obstacle cell indices
    size_t gidx_cap = 0;
    unsigned long long* gnum = nullptr; // [1] their count
    size_t gnum_cap = 0;
    unsigned char* gtmp = nullptr;      // [gtmp_cap] CUB temporary storage
    size_t gtmp_cap = 0;
};

// Rust's `as i32` of a double: saturating, NaN -> 0
static int csm_sat_i32(double v) {
    if (v != v) return 0;
    if (v >= 2147483647.0) return 2147483647;
    if (v <= -2147483648.0) return (int)(-2147483647 - 1);
    return (int)v;
}
// cudaMalloc of `need` elements unless `cap` already holds them (the old contents are dropped)
template <class T> static int csm_grow(T** p, size_t* cap, size_t need) {
    if (need <= *cap) return 0;
    cudaFree(*p);
    *p = nullptr;
    *cap = 0;
    PF_CUDA(cudaMalloc(p, need * sizeof(T)));
    *cap = need;
    return 0;
}
static void pf_csm_free(pfgpu_csm* h) {
    cudaFree(h->rx); cudaFree(h->ry); cudaFree(h->table); cudaFree(h->X); cudaFree(h->Y); cudaFree(h->cs); cudaFree(h->part);
    cudaFree(h->best); cudaFree(h->ext); cudaFree(h->gmask); cudaFree(h->gidx); cudaFree(h->gnum); cudaFree(h->gtmp);
    if (h->h_ext) cudaFreeHost(h->h_ext);
    if (h->ctx.stream) cudaStreamDestroy(h->ctx.stream);
}
extern "C" void pfgpu_csm_destroy(pfgpu_csm* h) {
    if (!h) return;
    cudaSetDevice(h->ctx.device);
    if (h->ctx.stream) cudaStreamSynchronize(h->ctx.stream);
    pf_csm_free(h);
    delete h;
}
extern "C" int pfgpu_csm_create(int device, pfgpu_csm** out) {
    if (!out) return PFGPU_ERR_INVALID;
    *out = nullptr;
    pfgpu_csm* h = new (std::nothrow) pfgpu_csm();
    if (!h) return PFGPU_ERR_CUDA;
    const char* e = getenv("PFGPU_CSM_WS_CAP");    // a smaller workspace (at least 2^16 bytes) forces chunking, for tests
    if (e && *e) h->ws_cap = std::max<size_t>((size_t)1 << 16, std::min<size_t>(strtoull(e, nullptr, 10), PF_CSM_WS_CAP));
    int rc = ctx_open(h->ctx, device);
    if (!rc) {
        auto alloc = [&]() -> int {
            PF_CUDA(cudaMalloc(&h->ext, 5 * sizeof(int)));
            PF_CUDA(cudaMallocHost(&h->h_ext, 5 * sizeof(int)));
            PF_CUDA(cudaMalloc(&h->part, PF_CSM_PART_CAP * sizeof(PfCsmBest)));
            return 0;
        };
        rc = alloc();
    }
    if (rc) { pf_csm_free(h); delete h; return rc; }
    *out = h;
    return 0;
}
extern "C" int pfgpu_csm_set_reference(pfgpu_csm* h, const double* x, const double* y, size_t n) {
    if (!h || (n && (!x || !y)) || n > ((size_t)1 << 31)) return PFGPU_ERR_INVALID;
    for (size_t i = 0; i < n; ++i)
        if (!finite_d(x[i]) || !finite_d(y[i])) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    h->table_ok = false;
    h->n = 0;
    if (n) {
        size_t c = h->ncap;
        int rc = csm_grow(&h->rx, &c, n);
        if (!rc) { c = h->ncap; rc = csm_grow(&h->ry, &c, n); }
        if (rc) { cudaFree(h->rx); cudaFree(h->ry); h->rx = h->ry = nullptr; h->ncap = 0; return rc; }
        h->ncap = std::max(h->ncap, n);
        PF_CUDA(cudaMemcpyAsync(h->rx, x, n * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
        PF_CUDA(cudaMemcpyAsync(h->ry, y, n * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    h->n = n;
    return 0;
}
extern "C" int pfgpu_csm_set_reference_grid(pfgpu_csm* h, const pfgpu_ogm* g, double threshold) {
    if (!h || !g || !finite_d(threshold) || g->ctx.device != h->ctx.device) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    const size_t cells = g->W * g->H;
    thrust::counting_iterator<unsigned int> it(0u);
    size_t tb = 0;
    PF_CUDA(cub::DeviceSelect::Flagged(nullptr, tb, it, (const unsigned char*)nullptr, (unsigned int*)nullptr,
                                       (unsigned long long*)nullptr, (long long)cells, h->ctx.stream));
    int rc = csm_grow(&h->gmask, &h->gmask_cap, cells);
    if (!rc) rc = csm_grow(&h->gidx, &h->gidx_cap, cells);
    if (!rc) rc = csm_grow(&h->gnum, &h->gnum_cap, 1);
    if (!rc) rc = csm_grow(&h->gtmp, &h->gtmp_cap, std::max<size_t>(tb, 1));
    if (rc) return rc;
    rc = pf_ogm_mask(g, threshold, h->gmask, h->ctx);
    if (rc) return rc;
    PF_CUDA(cub::DeviceSelect::Flagged(h->gtmp, tb, it, (const unsigned char*)h->gmask, h->gidx, h->gnum, (long long)cells, h->ctx.stream));
    unsigned long long n = 0;
    PF_CUDA(cudaMemcpyAsync(&n, h->gnum, sizeof(n), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    h->table_ok = false;
    h->n = 0;
    if (n) {
        size_t c = h->ncap;
        rc = csm_grow(&h->rx, &c, n);
        if (!rc) { c = h->ncap; rc = csm_grow(&h->ry, &c, n); }
        if (rc) { cudaFree(h->rx); cudaFree(h->ry); h->rx = h->ry = nullptr; h->ncap = 0; return rc; }
        h->ncap = std::max<size_t>(h->ncap, n);
        PF_LAUNCH(h->ctx, pf_csm_centres_kernel, cdiv_u(n, 256), 256, 0, (const unsigned int*)h->gidx, (size_t)n, (unsigned int)g->H,
                  (double)g->W / 2.0, (double)g->H / 2.0, g->cfg.resolution, h->rx, h->ry);
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    h->n = n;
    return 0;
}
extern "C" int pfgpu_csm_reference_size(pfgpu_csm* h, size_t* n) {
    if (!h || !n) return PFGPU_ERR_INVALID;
    *n = h->n;
    return 0;
}
// the lookup table for `res` (build_lookup_table :129-159), kept until the reference or the resolution changes
static int pf_csm_table(pfgpu_csm* h, double res) {
    if (h->table_ok && h->table_res == res) return 0;
    if (!(res >= 0x1p-500 && res <= 0x1p500)) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "csm: grid_resolution %g outside [2^-500, 2^500]", res);
        return PFGPU_ERR_UNSUPPORTED;
    }
    h->table_ok = false;
    const double sigma = res;
    const int R = csm_sat_i32(ceil(3.0 * sigma / res));
    const double inv = 0.5 / (sigma * sigma);
    if (h->n == 0) {
        h->ox = h->oy = h->TW = h->TH = 0; h->R = R;
        h->table_ok = true; h->table_res = res;
        return 0;
    }
    PF_CUDA(cudaSetDevice(h->ctx.device));
    const int init[5] = {INT_MAX, INT_MIN, INT_MAX, INT_MIN, 0};
    memcpy(h->h_ext, init, sizeof(init));
    PF_CUDA(cudaMemcpyAsync(h->ext, h->h_ext, sizeof(init), cudaMemcpyHostToDevice, h->ctx.stream));
    PF_LAUNCH(h->ctx, pf_csm_extent_kernel, cdiv_u(h->n, 256), 256, 0, (const double*)h->rx, (const double*)h->ry, h->n, res, h->ext,
              h->ext + 4);
    PF_CUDA(cudaMemcpyAsync(h->h_ext, h->ext, sizeof(init), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (h->h_ext[4]) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "csm: a reference cell beyond 2^30 at resolution %g", res);
        return PFGPU_ERR_INVALID;
    }
    const long long ox = (long long)h->h_ext[0] - R, oy = (long long)h->h_ext[2] - R;
    const long long TW = (long long)h->h_ext[1] + R + 1 - ox, TH = (long long)h->h_ext[3] + R + 1 - oy;
    if (TW > (long long)PFGPU_CSM_TABLE_CAP || TH > (long long)PFGPU_CSM_TABLE_CAP || (uint64_t)(TW * TH) > PFGPU_CSM_TABLE_CAP) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "csm: a %lld x %lld table exceeds %llu cells", TW, TH,
                 (unsigned long long)PFGPU_CSM_TABLE_CAP);
        return PFGPU_ERR_UNSUPPORTED;
    }
    const size_t cells = (size_t)(TW * TH);
    int rc = csm_grow(&h->table, &h->tcap, cells);
    if (rc) return rc;
    PF_CUDA(cudaMemsetAsync(h->table, 0, cells * sizeof(double), h->ctx.stream));
    const size_t side = 2 * (size_t)R + 1;
    PF_LAUNCH(h->ctx, pf_csm_fill_kernel, cdiv_u(h->n * side * side, 256), 256, 0, (const double*)h->rx, (const double*)h->ry, h->n, res,
              inv, R, ox, oy, TH, h->table);
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    h->ox = ox; h->oy = oy; h->TW = TW; h->TH = TH; h->R = R;
    h->table_ok = true; h->table_res = res;
    return 0;
}
extern "C" int pfgpu_csm_table_info(pfgpu_csm* h, double res, int64_t* ox, int64_t* oy, uint64_t* W, uint64_t* H, int32_t* R) {
    if (!h || !finite_d(res) || !(res > 0.0)) return PFGPU_ERR_INVALID;
    const int rc = pf_csm_table(h, res);
    if (rc) return rc;
    if (ox) *ox = h->ox;
    if (oy) *oy = h->oy;
    if (W) *W = (uint64_t)h->TW;
    if (H) *H = (uint64_t)h->TH;
    if (R) *R = h->R;
    return 0;
}
extern "C" int pfgpu_csm_table_read(pfgpu_csm* h, size_t first, size_t count, double* out) {
    if (!h || !h->table_ok) return PFGPU_ERR_INVALID;
    const size_t cells = (size_t)(h->TW * h->TH);
    if (first > cells || count > cells - first || (count && !out)) return PFGPU_ERR_INVALID;
    if (count == 0) return 0;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(out, h->table + first, count * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_csm_match(pfgpu_csm* h, const pfgpu_csm_config* c, const double* poses3, size_t Q, const double* qx, const double* qy,
                               const uint64_t* offsets, pfgpu_csm_result* results) {
    if (!h || !c) return PFGPU_ERR_INVALID;
    if (Q == 0) return 0;
    if (!poses3 || !offsets || !results || Q > ((size_t)1 << 32) || offsets[0] != 0) return PFGPU_ERR_INVALID;
    if (!finite_d(c->linear_search_range) || !finite_d(c->angular_search_range) || !finite_d(c->linear_step) ||
        !finite_d(c->angular_step) || !finite_d(c->grid_resolution))
        return PFGPU_ERR_INVALID;
    for (size_t q = 0; q < Q; ++q)
        if (offsets[q + 1] < offsets[q] || !finite_d(poses3[3 * q]) || !finite_d(poses3[3 * q + 1]) || !finite_d(poses3[3 * q + 2]))
            return PFGPU_ERR_INVALID;
    const size_t K = (size_t)offsets[Q];
    if (K && (!qx || !qy)) return PFGPU_ERR_INVALID;
    for (size_t k = 0; k < K; ++k)
        if (!finite_d(qx[k]) || !finite_d(qy[k])) return PFGPU_ERR_INVALID;
    const double ls = c->linear_step, as = c->angular_step, res = c->grid_resolution;
    // the reference's invalid input (:63-78)
    const bool invalid = h->n == 0 || ls <= 0.0 || as <= 0.0 || res <= 0.0;
    auto np = [&](size_t q) { return (size_t)(offsets[q + 1] - offsets[q]); };
    size_t live = 0;
    for (size_t q = 0; q < Q; ++q) {
        if (invalid || np(q) == 0) results[q] = pfgpu_csm_result{poses3[3 * q], poses3[3 * q + 1], poses3[3 * q + 2], 0.0, 0u, 0u};
        else ++live;
    }
    if (live == 0) return 0;
    const int nl = csm_sat_i32(round(c->linear_search_range / ls)), na = csm_sat_i32(round(c->angular_search_range / as));
    if (nl < 0 || na < 0) {                     // no candidate (:84-90)
        for (size_t q = 0; q < Q; ++q)
            if (np(q)) results[q] = pfgpu_csm_result{poses3[3 * q], poses3[3 * q + 1], fs_normalize_angle(poses3[3 * q + 2]), -1.0, 0u, 0u};
        return 0;
    }
    const size_t NL = 2 * (size_t)nl + 1, NA = 2 * (size_t)na + 1;
    if (nl > (1 << 15) || na > (1 << 22) || NL * NL * NA > ((size_t)1 << 34)) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "csm: %zu x %zu x %zu candidates per query exceed the caps", NL, NL, NA);
        return PFGPU_ERR_UNSUPPORTED;
    }
    for (size_t q = 0; q < Q; ++q)
        if (8 * NL * np(q) > h->ws_cap) {
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "csm: query %zu's cell indices for one yaw exceed %zu bytes", q, h->ws_cap);
            return PFGPU_ERR_UNSUPPORTED;
        }
    int rc = pf_csm_table(h, res);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Ctx& ctx = h->ctx;
    const size_t ws_ints = h->ws_cap / 8;       // per array
    size_t cap = h->ws_ints;
    rc = csm_grow(&h->X, &cap, ws_ints);
    if (!rc) { cap = h->ws_ints; rc = csm_grow(&h->Y, &cap, ws_ints); }
    if (rc) { cudaFree(h->X); cudaFree(h->Y); h->X = h->Y = nullptr; h->ws_ints = 0; return rc; }
    h->ws_ints = ws_ints;
    if ((rc = csm_grow(&h->best, &h->best_cap, Q))) return rc;
    // the queries with points: only they get score and reduce blocks (an empty one keeps the invalid result set above)
    std::vector<unsigned long long> lq;
    for (size_t q = 0; q < Q; ++q)
        if (np(q)) lq.push_back(q);
    PfScopedBuf dp, dx, dy, doff, dlive;
    PF_CUDA(cudaMalloc(&dp.p, Q * 3 * sizeof(double)));
    PF_CUDA(cudaMalloc(&doff.p, (Q + 1) * sizeof(unsigned long long)));
    PF_CUDA(cudaMalloc(&dlive.p, lq.size() * sizeof(unsigned long long)));
    PF_CUDA(cudaMemcpyAsync(dlive.p, lq.data(), lq.size() * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx.stream));
    PF_CUDA(cudaMalloc(&dx.p, std::max<size_t>(K, 1) * sizeof(double)));
    PF_CUDA(cudaMalloc(&dy.p, std::max<size_t>(K, 1) * sizeof(double)));
    PF_CUDA(cudaMemcpyAsync(dp.p, poses3, Q * 3 * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    PF_CUDA(cudaMemcpyAsync(doff.p, offsets, (Q + 1) * sizeof(unsigned long long), cudaMemcpyHostToDevice, ctx.stream));
    if (K) {
        PF_CUDA(cudaMemcpyAsync(dx.p, qx, K * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
        PF_CUDA(cudaMemcpyAsync(dy.p, qy, K * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    }
    PF_LAUNCH(ctx, pf_csm_best_init_kernel, cdiv_u(Q, 256), 256, 0, h->best, Q);
    PfCsmGeo g;
    g.res = res; g.lstep = ls; g.ox = h->ox; g.oy = h->oy; g.TW = h->TW; g.TH = h->TH; g.nl = nl; g.NL = (int)NL;
    const unsigned long long* off = (const unsigned long long*)doff.p;
    const unsigned long long* dl = (const unsigned long long*)dlive.p;
    size_t l0 = 0;                              // the group's first entry of lq
    for (size_t q0 = 0; q0 < Q;) {
        // a group of queries whose cell indices for one yaw fit the workspace
        size_t q1 = q0, P = 0;
        while (q1 < Q && q1 - q0 < 65535 && (8 * NL * (P + np(q1)) <= h->ws_cap)) P += np(q1++);
        const size_t nq = q1 - q0, k0 = (size_t)offsets[q0];
        size_t l1 = l0;
        while (l1 < lq.size() && lq[l1] < q1) ++l1;
        const size_t nlive = l1 - l0;
        if (nlive == 0) { q0 = q1; continue; }
        const size_t nac_ws = P ? std::max<size_t>(1, h->ws_cap / (8 * NL * P)) : NA;
        const size_t nac = std::min(NA, nac_ws);
        PfCsmBest* part = h->part;
        for (size_t a0 = 0; a0 < NA; a0 += nac) {
            const int n_a = (int)std::min(nac, NA - a0);
            g.nac = n_a;
            if ((rc = csm_grow(&h->cs, &h->cs_cap, nq * (size_t)n_a))) return rc;
            PF_LAUNCH(ctx, pf_csm_trig_kernel, cdiv_u(nq * (size_t)n_a, 256), 256, 0, (const double*)dp.p, q0, nq, (long long)a0, n_a, na,
                      as, h->cs);
            if (P)
                PF_LAUNCH(ctx, pf_csm_cells_kernel, cdiv_u(P * (size_t)n_a * NL, 256), 256, 0, g, (const double*)dp.p, (const double*)dx.p,
                          (const double*)dy.p, off, q0, nq, k0, P, (const double2*)h->cs, h->X, h->Y);
            const size_t per = NL * NL * (size_t)n_a;
            const size_t nb = std::max<size_t>(1, std::min<size_t>(cdiv_u(per, PF_CSM_NT), PF_CSM_PART_CAP / nlive));
            PF_LAUNCH(ctx, pf_csm_score_kernel, dim3((unsigned)nb, (unsigned)nlive), PF_CSM_NT, 0, g, (const double*)h->table, off, dl, l0,
                      k0, (const int*)h->X, (const int*)h->Y, (long long)a0, na, as, part);
            PF_LAUNCH(ctx, pf_csm_reduce_kernel, (unsigned)nlive, PF_CSM_NT, 0, (const PfCsmBest*)part, nb, dl, l0, h->best);
        }
        l0 = l1;
        q0 = q1;
    }
    std::vector<PfCsmBest> best(Q);
    PF_CUDA(cudaMemcpyAsync(best.data(), h->best, Q * sizeof(PfCsmBest), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaStreamSynchronize(ctx.stream));
    for (size_t q = 0; q < Q; ++q) {
        if (invalid || np(q) == 0) continue;
        const unsigned long long i = best[q].idx;
        const long long ia = (long long)(i % NA), iy = (long long)((i / NA) % NL), ix = (long long)(i / (NA * NL));
        const double dxo = (double)(int)(ix - nl) * ls, dyo = (double)(int)(iy - nl) * ls, dyaw = (double)(int)(ia - na) * as;
        results[q] = pfgpu_csm_result{poses3[3 * q] + dxo, poses3[3 * q + 1] + dyo, fs_normalize_angle(poses3[3 * q + 2] + dyaw),
                                      best[q].score, best[q].score > 0.0 ? 1u : 0u, 0u};
    }
    return 0;
}

// ---- pose hypotheses: the cloud clustered in a fixed (x, y, yaw) histogram (DESIGN §3.10, pf_cluster.cuh) ----
extern "C" int pfgpu_pf_hypotheses(pfgpu_pf* h, double xy_res, uint32_t yaw_bins, pfgpu_pf_hypothesis* out, size_t cap, size_t* n_total,
                                   uint32_t* rank_of_slot) {
    if (!h || !finite_d(xy_res) || !(xy_res > 0.0) || yaw_bins == 0 || yaw_bins > 65536 || (cap > 0 && !out)) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PfDev& d = h->d; PfClu& c = h->clu; Ctx& ctx = h->ctx;
    const size_t most = h->adaptive ? (size_t)h->cfg.max_particles : (size_t)d.n_global;     // the largest global set
    if (most > 0x7FFFFFFFull) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "pose hypotheses: more than 2^31 - 1 particles");
        return PFGPU_ERR_UNSUPPORTED;
    }
    if (!c.keys) { int rc = pf_clu_alloc(c, most, h->world > 1); if (rc) return rc; }
    const size_t N = d.n_global;
    const Pose4* P_all = nullptr;
    const double* W_all = nullptr;
    if (h->world > 1) {                                  // every rank clusters the global set in rank order
        PF_NCCL(ncclAllGather(d.pose[h->cur_host], h->sh.pose_all, 4 * d.n, ncclDouble, h->sh.comm, ctx.stream));
        PF_NCCL(ncclAllGather(d.w, c.w_all, d.n, ncclDouble, h->sh.comm, ctx.stream));
        P_all = reinterpret_cast<const Pose4*>(h->sh.pose_all); W_all = c.w_all;
    }
    PF_CUDA(cudaMemsetAsync(c.owner, 0xFF, (size_t)c.tcap * sizeof(int), ctx.stream));
    PF_CUDA(cudaMemsetAsync(c.mint, 0xFF, (size_t)c.tcap * sizeof(unsigned), ctx.stream));
    PF_CUDA(cudaMemsetAsync(c.parent, 0xFF, (size_t)c.tcap * sizeof(int), ctx.stream));
    const double bw = PFC_TWO_PI / (double)yaw_bins;
    PF_LAUNCH(ctx, pf_clu_key_kernel, cdiv_u(N, PF_NT), PF_NT, 0, d, P_all, W_all, N, c, xy_res, bw, (int)yaw_bins);
    PF_LAUNCH(ctx, pf_clu_insert_kernel, cdiv_u(N, PF_NT), PF_NT, 0, c, N);
    PF_LAUNCH(ctx, pf_clu_link_kernel, cdiv_u(c.tcap, PF_NT), PF_NT, 0, c, (int)yaw_bins);
    PF_LAUNCH(ctx, pf_clu_label_kernel, cdiv_u(N, PF_NT), PF_NT, 0, c, N);
    int bits = 1;
    while (((size_t)1 << bits) <= N) ++bits;             // labels are <= N (N: not a member)
    size_t tb = c.tmp_bytes;
    PF_CUDA(cub::DeviceRadixSort::SortPairs(c.tmp, tb, c.lab, c.lab_s, c.iota, c.perm, (int)N, 0, bits, ctx.stream));
    tb = c.tmp_bytes;
    PF_CUDA(cub::DeviceRunLengthEncode::Encode(c.tmp, tb, c.lab_s, c.uniq, c.cnt, c.scal, (int)N, ctx.stream));
    PF_LAUNCH(ctx, pf_clu_count_kernel, 1, 1, 0, c, N);
    unsigned* hp = reinterpret_cast<unsigned*>(h->h_pin + 50);
    PF_CUDA(cudaMemcpyAsync(hp, c.scal + 1, sizeof(unsigned), cudaMemcpyDeviceToHost, ctx.stream));
    PF_CUDA(cudaStreamSynchronize(ctx.stream));          // the launches below are sized by the number of clusters
    const unsigned nc = *hp;
    const unsigned m = (unsigned)std::min<size_t>(cap, nc);
    if (nc > 0) {
        tb = c.tmp_bytes;
        PF_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, tb, c.cnt, c.off, (int)nc, ctx.stream));
        PF_LAUNCH(ctx, pf_clu_ntiles_kernel, cdiv_u(nc, PF_NT), PF_NT, 0, c, nc);
        tb = c.tmp_bytes;
        PF_CUDA(cub::DeviceScan::ExclusiveSum(c.tmp, tb, c.rank, c.toff, (int)nc, ctx.stream));
        const size_t warps_per_cta = PF_NT / 32, tiles_max = N / PF_CLU_TILE + nc;
        const unsigned g_tile = (unsigned)std::min<size_t>(cdiv_u(tiles_max, warps_per_cta), (size_t)ctx.num_sms * 16);
        const unsigned g_clu = (unsigned)std::min<size_t>(cdiv_u(nc, warps_per_cta), (size_t)ctx.num_sms * 16);
        PF_LAUNCH(ctx, pf_clu_tile_kernel<1>, g_tile, PF_NT, 0, d, P_all, W_all, c, nc, rank_of_slot ? 1 : 0);
        PF_LAUNCH(ctx, pf_clu_final_kernel<1>, g_clu, PF_NT, 0, c, nc);
        PF_LAUNCH(ctx, pf_clu_tile_kernel<2>, g_tile, PF_NT, 0, d, P_all, W_all, c, nc, 0);
        PF_LAUNCH(ctx, pf_clu_final_kernel<2>, g_clu, PF_NT, 0, c, nc);
        tb = c.tmp_bytes;
        PF_CUDA(cub::DeviceRadixSort::SortPairs(c.tmp, tb, c.mkey, c.mkey_s, c.iota, c.order, (int)nc, 0, 64, ctx.stream));
        PF_LAUNCH(ctx, pf_clu_rank_kernel, cdiv_u(nc, PF_NT), PF_NT, 0, c, nc, m);
        if (m) PF_CUDA(cudaMemcpyAsync(out, c.part, (size_t)m * sizeof(pfgpu_pf_hypothesis), cudaMemcpyDeviceToHost, ctx.stream));
    }
    if (rank_of_slot) {
        PF_LAUNCH(ctx, pf_clu_slot_rank_kernel, cdiv_u(d.n, PF_NT), PF_NT, 0, c, d.offset, d.n, nc);
        PF_CUDA(cudaMemcpyAsync(rank_of_slot, c.lab, d.n * sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx.stream));
    }
    PF_CUDA(cudaStreamSynchronize(ctx.stream));
    if (n_total) *n_total = nc;
    return 0;
}

static void timer_drain(KernelTimer& t) {
    for (auto& p : t.pending) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, p.first, p.second) == cudaSuccess) { t.ms_sum += ms; t.count++; }
        cudaEventDestroy(p.first); cudaEventDestroy(p.second);
    }
    t.pending.clear();
}
extern "C" int pfgpu_pf_stats(pfgpu_pf* h, pfgpu_stats* s) {
    if (!h || !s) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    memset(s, 0, sizeof(*s));
    timer_drain(h->timer);
    unsigned int cnt = 0;
    PF_CUDA(cudaMemcpy(&cnt, h->d.counters, sizeof(unsigned int), cudaMemcpyDeviceToHost));
    s->kernel_launches = h->ctx.launches; s->steps = h->steps; s->resamples = cnt;
    s->main_kernel_ms_sum = h->timer.ms_sum; s->main_kernel_count = h->timer.count;
    int f[4] = {0, 0, 0, 0};                                   // the separate kernels' exact sums (xsum.cuh)
    PF_CUDA(cudaMemcpy(f, h->xs.flags + 4, 4 * sizeof(int), cudaMemcpyDeviceToHost));
    s->serial_fallbacks = (uint64_t)f[0];
    s->xsum_dirty_last = (uint64_t)(f[1] < 0 ? 0 : f[1]);
    if (!h->fu.on) return 0;
    Fs3State st; PF_CUDA(cudaMemcpy(&st, h->fu.x.st, sizeof(st), cudaMemcpyDeviceToHost));     // the fused tail's (pf3.cuh)
    s->serial_fallbacks += (uint64_t)st.serial_walks + (uint64_t)st.cert_fail;
    if (h->fu.last) s->xsum_dirty_last = (uint64_t)st.dirty_last;
    return 0;
}
extern "C" int pfgpu_pf_time_main_kernel(pfgpu_pf* h, int on) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    timer_drain(h->timer);
    h->timer.on = on != 0; h->timer.ms_sum = 0.0; h->timer.count = 0;
    return 0;
}

// ====================================================================================================
// FastSLAM 1.0: fs3_host.cuh (entry points) + fs3.cuh (kernels)
// ====================================================================================================
#include "fs3_host.cuh"

extern "C" int pfgpu_pf_mark(pfgpu_pf* h, int slot) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_mark(h->ctx, h->marks, slot); }
extern "C" int pfgpu_pf_elapsed_ms(pfgpu_pf* h, int a, int b, double* ms) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_elapsed(h->marks, a, b, ms); }
extern "C" int pfgpu_fs_mark(pfgpu_fs* h, int slot) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_mark(h->ctx, h->marks, slot); }
extern "C" int pfgpu_fs_elapsed_ms(pfgpu_fs* h, int a, int b, double* ms) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_elapsed(h->marks, a, b, ms); }
extern "C" int pfgpu_pf_flush_l2(pfgpu_pf* h) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_flush(h->ctx, h->marks); }
extern "C" int pfgpu_fs_flush_l2(pfgpu_fs* h) { if (!h) return PFGPU_ERR_INVALID; PF_CUDA(cudaSetDevice(h->ctx.device)); return marks_flush(h->ctx, h->marks); }

extern "C" int pfgpu_nccl_unique_id(void* out128) {
    if (!out128) return PFGPU_ERR_INVALID;
    ncclUniqueId id;
    PF_NCCL(ncclGetUniqueId(&id));
    static_assert(sizeof(id) == 128, "ncclUniqueId is 128 bytes");
    memcpy(out128, &id, sizeof(id));
    return 0;
}

// ====================================================================================================
// test hook: the device's reciprocal-based division (PFC_DIV) against the IEEE `/` on n random + adversarial pairs
__global__ void pf_test_div_kernel(unsigned long long n, uint64_t seed, unsigned long long* mismatches) {
    unsigned long long bad = 0;
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        pfc_u32x4 r = pfc_rng_block(seed, 7, 0, i), r2 = pfc_rng_block(seed, 7, 1, i);
        uint64_t x = pfc_blk_u64(r, 0), z = pfc_blk_u64(r, 1), m = pfc_blk_u64(r2, 0);
        int ea = (int)(m % 801) - 400, eb = (int)((m >> 10) % 801) - 400;
        int kind = (int)((m >> 20) & 7);
        if (kind == 0) z |= 0x000FFFFFFFFFF000ull; else if (kind == 1) z &= 0xFFF0000000000FFFull;
        else if (kind == 2) x |= 0x000FFFFFFFFFFF00ull; else if (kind == 3) { x &= 0xFFF00000000000FFull; z &= 0xFFF00000000000FFull; }
        double a = pfc_u2d((x & 0x800FFFFFFFFFFFFFull) | ((uint64_t)(ea + 1023) << 52));
        double b = pfc_u2d((z & 0x800FFFFFFFFFFFFFull) | ((uint64_t)(eb + 1023) << 52));
        if (kind == 7) a = (m & (1ull << 40)) ? 0.0 : -0.0;
        double q = PFC_DIV(a, b), t = a / b;
        if (pfc_d2u(q) != pfc_d2u(t)) bad++;
    }
    if (bad) atomicAdd(mismatches, bad);
}
extern "C" int pfgpu_test_div(unsigned long long n, uint64_t seed, unsigned long long* mismatches, int device) {
    PF_CUDA(cudaSetDevice(device));
    unsigned long long* d = nullptr;
    PF_CUDA(cudaMalloc(&d, sizeof(*d)));
    PF_CUDA(cudaMemset(d, 0, sizeof(*d)));
    pf_test_div_kernel<<<PFGPU_NUM_SMS * 8, 256>>>(n, seed, d);
    PF_CUDA(cudaDeviceSynchronize());
    PF_CUDA(cudaMemcpy(mismatches, d, sizeof(*d), cudaMemcpyDeviceToHost));
    cudaFree(d);
    return 0;
}

// ====================================================================================================
// test hook: the exact scan on an arbitrary host array (used by tests/test_gpu_xsum.py)
// ====================================================================================================
extern "C" int pfgpu_test_xsum(const double* host_v, size_t n, double* host_scan, double* host_total, int* flags4, int device) {
    Ctx ctx;
    int rc = ctx_open(ctx, device);
    if (rc) return rc;
    XsWork xs;
    rc = xs_work_alloc(xs, n);
    if (rc) return rc;
    double *dv = nullptr, *dc = nullptr, *dt = nullptr;
    PF_CUDA(cudaMalloc(&dv, n * sizeof(double))); PF_CUDA(cudaMalloc(&dc, n * sizeof(double))); PF_CUDA(cudaMalloc(&dt, sizeof(double)));
    PF_CUDA(cudaMemcpy(dv, host_v, n * sizeof(double), cudaMemcpyHostToDevice));
    rc = xs_scan(ctx, xs, XsValArray{dv}, XsSinkStore{dc}, n, n, 0.0, dt);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(ctx.stream));
    if (host_scan) PF_CUDA(cudaMemcpy(host_scan, dc, n * sizeof(double), cudaMemcpyDeviceToHost));
    if (host_total) PF_CUDA(cudaMemcpy(host_total, dt, sizeof(double), cudaMemcpyDeviceToHost));
    if (flags4) PF_CUDA(cudaMemcpy(flags4, xs.flags, 4 * sizeof(int), cudaMemcpyDeviceToHost));
    cudaFree(dv); cudaFree(dc); cudaFree(dt);
    xs_work_free(xs);
    cudaStreamDestroy(ctx.stream);
    return 0;
}

// ====================================================================================================
// test hook: a step's tail on arbitrary raw weights (used by tests/test_gpu_pf_tail_edges.py).  w_raw[n] replaces the raw
// weights, then exactly what a step issues after its predict + likelihood kernel runs (the fused tail, or the separate kernels
// of a PFGPU_PF_FUSED=0 handle).  scal4 (optional): S = sum w_raw, Q = sum w^2, the last cumulative weight, N_eff, as the tail
// left them; gate (optional): 1 when it resampled.
// ====================================================================================================
extern "C" int pfgpu_test_pf_tail(pfgpu_pf* h, const double* w_raw, size_t n, double* scal4, int* gate) {
    if (!h || !w_raw || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(h->d.w_raw, w_raw, n * sizeof(double), cudaMemcpyHostToDevice, h->ctx.stream));
    int rc = pf_step_tail(h);
    if (rc) return rc;
    h->fu.last = h->fu.on;
    h->rec.armed = true;
    if (scal4) PF_CUDA(cudaMemcpyAsync(scal4, h->d.scal, 4 * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    if (gate) PF_CUDA(cudaMemcpyAsync(gate, h->d.gate, sizeof(int), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
