// gslam_host.cuh — the C ABI of grid-based FastSLAM (include/pfgpu.h pfgpu_gs_*, DESIGN §3.16); kernels in gslam.cuh.  Included by
// pfgpu.cu after the occupancy grid mapping section, whose handle (pfgpu_ogm) and checks it uses.
#include "gslam.cuh"

struct pfgpu_gs {
    Ctx ctx;
    pfgpu_gs_config cfg = {};
    uint64_t seed = 0, L = 0, steps = 0;
    double q_out = 0.0;
    double alpha[4] = { PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT, PF_ODOM_ALPHA_DEFAULT };
    GsDev d;
    XsWork xs;
    void* tmp = nullptr;               // CUB scan storage
    size_t tmp_bytes = 0;
    double* ranges = nullptr;          // [rcap] the step's scan
    double* pairs = nullptr;           // [2 * L] its used beams (r, i * angle_inc)
    size_t rcap = 0;
    std::vector<double> hp;            // host staging of the used beams
    pfgpu_gs_proposal prop = {};       // the scan-matched proposal (DESIGN §3.17); off until pfgpu_gs_set_proposal enables it
    GsPropOut pout = {};               // [3n], [n], [n]: allocated when the proposal is first enabled
    bool last_prop = false;            // the last step ran the proposal
};

static void gs_free(pfgpu_gs* h) {
    GsDev& d = h->d;
    void* p[] = { d.px, d.py, d.pyaw, d.w, d.tx, d.ty, d.tyaw, d.grids, d.buf, d.nbuf, d.idx, d.cum, d.comb, d.nf, d.enf, d.cl, d.ecl,
                  d.has_child, d.free_buf, d.job_src, d.job_dst, d.scal, d.gate, d.cnt, h->tmp, h->ranges, h->pairs,
                  h->pout.xh, h->pout.eta, h->pout.took };
    for (void* q : p) cudaFree(q);
    if (h->xs.flags) xs_work_free(h->xs);
    if (h->ctx.stream) cudaStreamDestroy(h->ctx.stream);
}
extern "C" void pfgpu_gs_destroy(pfgpu_gs* h) {
    if (!h) return;
    cudaSetDevice(h->ctx.device);
    if (h->ctx.stream) cudaStreamSynchronize(h->ctx.stream);
    gs_free(h);
    delete h;
}
extern "C" void pfgpu_gs_default_config(pfgpu_gs_config* c) {
    if (!c) return;
    *c = pfgpu_gs_config();
    c->ogm.resolution = 0.5; c->ogm.width = 100; c->ogm.height = 100;
    c->ogm.prior_log_odds = 0.0; c->ogm.occupied_log_odds = 0.85; c->ogm.free_log_odds = -0.4;
    c->ogm.max_log_odds = 5.0; c->ogm.min_log_odds = -5.0;
    c->n_particles = 100; c->nth = 50.0;
    c->z_hit = 0.95; c->z_rand = 0.05; c->max_range = 30.0; c->max_beams = 60; c->search_radius = 1;
}
extern "C" void pfgpu_gs_default_proposal(pfgpu_gs_proposal* p) {
    if (!p) return;
    *p = pfgpu_gs_proposal();
    p->enabled = 0; p->half_width = 1; p->min_hits = 10;
    p->linear_range = 0.1; p->linear_step = 0.025; p->angular_range = 0.05; p->angular_step = 0.0125;
    p->lattice_linear_step = 0.01; p->lattice_angular_step = 0.005;
}
// the match's half-widths n = round(range / step) (CSM's rule) of a validated config
static void gs_prop_window(const pfgpu_gs_proposal& p, int* nl, int* na) {
    *nl = (int)round(p.linear_range / p.linear_step);
    *na = (int)round(p.angular_range / p.angular_step);
}
// pfgpu_ogm_create's checks of the grid fields
static bool gs_ogm_cfg_ok(const pfgpu_ogm_config* c) {
    return c->width <= 65536 && c->height <= 65536 && pf_map_shape_ok((size_t)c->width, (size_t)c->height) && finite_d(c->resolution) &&
           c->resolution > 0.0 && finite_d(c->prior_log_odds) && finite_d(c->occupied_log_odds) && finite_d(c->free_log_odds) &&
           finite_d(c->max_log_odds) && finite_d(c->min_log_odds) && c->min_log_odds <= c->max_log_odds;
}
static int gs_alloc(pfgpu_gs* h) {
    GsDev& d = h->d;
    const size_t n = d.n;
    double** dv[] = { &d.px, &d.py, &d.pyaw, &d.w, &d.tx, &d.ty, &d.tyaw, &d.cum, &d.comb };
    for (double** p : dv) PF_CUDA(cudaMalloc(p, n * sizeof(double)));
    unsigned** uv[] = { &d.buf, &d.nbuf, &d.idx, &d.free_buf, &d.job_src, &d.job_dst };
    for (unsigned** p : uv) PF_CUDA(cudaMalloc(p, n * sizeof(unsigned)));
    int** iv[] = { &d.nf, &d.enf, &d.cl, &d.ecl, &d.has_child };
    for (int** p : iv) PF_CUDA(cudaMalloc(p, n * sizeof(int)));
    PF_CUDA(cudaMalloc(&d.scal, 8 * sizeof(double)));
    PF_CUDA(cudaMalloc(&d.gate, sizeof(int)));
    PF_CUDA(cudaMalloc(&d.cnt, 4 * sizeof(unsigned long long)));
    PF_CUDA(cudaMemset(d.scal, 0, 8 * sizeof(double)));
    PF_CUDA(cudaMemset(d.gate, 0, sizeof(int)));
    PF_CUDA(cudaMemset(d.cnt, 0, 4 * sizeof(unsigned long long)));
    PF_CUDA(cudaMalloc(&h->pairs, 2 * h->L * sizeof(double)));
    int rc = xs_work_alloc(h->xs, n);
    if (rc) return rc;
    size_t tb = 0;
    PF_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, d.nf, d.enf, (int)n, h->ctx.stream));
    h->tmp_bytes = std::max<size_t>(tb, 16);
    PF_CUDA(cudaMalloc(&h->tmp, h->tmp_bytes));
    PF_CUDA(cudaMalloc(&d.grids, n * d.cells * sizeof(double)));
    return 0;
}
extern "C" int pfgpu_gs_create(const pfgpu_gs_config* c, uint64_t seed, const double start[3], int device, pfgpu_gs** out) {
    if (!c || !start || !out) return PFGPU_ERR_INVALID;
    *out = nullptr;
    auto positive = [](double v) { return finite_d(v) && v > 0.0; };
    if (!gs_ogm_cfg_ok(&c->ogm) || c->n_particles < 1 || c->n_particles >= ((uint64_t)1 << 32) || c->nth != c->nth || !finite_d(c->z_hit) ||
        c->z_hit < 0.0 || !positive(c->z_rand) || !positive(c->max_range) || c->max_beams < 2 || c->search_radius > GS_MAX_R ||
        !finite_d(start[0]) || !finite_d(start[1]) || !finite_d(start[2]))
        return PFGPU_ERR_INVALID;
    const double q_out = c->z_rand / c->max_range;
    const uint64_t L = pf_lf_limit(q_out, c->z_hit + q_out);
    if (L < 1) return PFGPU_ERR_INVALID;
    const size_t n = (size_t)c->n_particles, cells = (size_t)(c->ogm.width * c->ogm.height);
    pfgpu_gs* h = new (std::nothrow) pfgpu_gs();
    if (!h) return PFGPU_ERR_CUDA;
    h->cfg = *c; h->seed = seed; h->L = L; h->q_out = q_out;
    pfgpu_gs_default_proposal(&h->prop);
    h->d.n = n; h->d.cells = cells;
    int rc = ctx_open(h->ctx, device);
    if (rc) { gs_free(h); delete h; return rc; }
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess || cells > ((size_t)1 << 60) / 8 / n || n * cells * sizeof(double) > free_b) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "grid FastSLAM: %zu grids of %zu cells do not fit in %zu free bytes", n, cells, free_b);
        gs_free(h); delete h;
        return PFGPU_ERR_UNSUPPORTED;
    }
    rc = gs_alloc(h);
    if (rc) { gs_free(h); delete h; return rc; }
    GsDev& d = h->d;
    PF_LAUNCH(h->ctx, gs_init_kernel, cdiv_u(n, 256), 256, 0, d, start[0], start[1], start[2]);
    PF_LAUNCH(h->ctx, pf_ogm_fill_kernel, cdiv_u(n * cells, 256), 256, 0, d.grids, n * cells, c->ogm.prior_log_odds);
    cudaError_t err = cudaStreamSynchronize(h->ctx.stream);
    if (err == cudaSuccess) err = cudaGetLastError();
    if (err != cudaSuccess) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "grid FastSLAM create: %s", cudaGetErrorString(err));
        gs_free(h); delete h;
        return PFGPU_ERR_CUDA;
    }
    *out = h;
    return 0;
}
extern "C" int pfgpu_gs_set_odom_noise(pfgpu_gs* h, const double alpha[4]) {
    if (!h || !alpha || !pf_odom_alpha_ok(alpha)) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) h->alpha[j] = alpha[j];
    return 0;
}
extern "C" int pfgpu_gs_odom_noise(pfgpu_gs* h, double alpha[4]) {
    if (!h || !alpha) return PFGPU_ERR_INVALID;
    for (int j = 0; j < 4; ++j) alpha[j] = h->alpha[j];
    return 0;
}
// S = the exact sum of the weights, then w / S (gated when `gate` is non-null)
static int gs_normalize(pfgpu_gs* h, double* S, const int* gate) {
    GsDev& d = h->d;
    h->xs.gate = gate;
    int rc = xs_total(h->ctx, h->xs, XsValArray{d.w}, d.n, d.n, 0.0, S);
    h->xs.gate = nullptr;
    if (rc) return rc;
    PF_LAUNCH(h->ctx, gs_normalize_kernel, cdiv_u(d.n, 256), 256, 0, d, (const double*)S, gate);
    return 0;
}
extern "C" int pfgpu_gs_step(pfgpu_gs* h, const double odom[6], const double* ranges, size_t B, double angle_min, double angle_inc) {
    if (!h || !odom || (B && !ranges) || !finite_d(angle_min) || !finite_d(angle_inc)) return PFGPU_ERR_INVALID;
    PfOdom om;
    if (pf_odom_increment(odom, h->alpha, &om) != 0) return PFGPU_ERR_INVALID;
    const pfgpu_gs_config& c = h->cfg;
    std::vector<double>& hp = h->hp;
    hp.clear();
    if (B) {
        const size_t s = std::max<size_t>(1, (B - 1) / (size_t)(c.max_beams - 1));
        for (size_t i = 0; i < B; i += s) {
            const double r = ranges[i];
            if (r <= 0.0 || !finite_d(r) || r >= c.max_range) continue;
            hp.push_back(r);
            hp.push_back((double)i * angle_inc);
        }
    }
    const size_t k = hp.size() / 2;
    if (k > h->L) return PFGPU_ERR_INVALID;
    // the proposal's constants, and the high side of its bound: c K q_hi^k <= DBL_MAX (a still step proposes nothing)
    const pfgpu_gs_proposal& pc = h->prop;
    GsProp P = {};
    if (pc.enabled) {
        gs_prop_window(pc, &P.nl, &P.na);
        P.ls = pc.linear_step; P.as = pc.angular_step; P.kl = pc.lattice_linear_step; P.ka = pc.lattice_angular_step;
        P.k = (int)pc.half_width; P.min_hits = pc.min_hits;
        P.c = gs_prop_norm(&om, P.kl, P.ka);
        if (!gs_prop_still(&om)) {
            const double S = (double)(2 * P.k + 1);
            double hi = P.c * ((S * S) * S);
            const double q_hi = c.z_hit + h->q_out;
            for (size_t j = 0; j < k; ++j) hi = hi * q_hi;
            if (!(hi <= DBL_MAX)) {
                snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "grid FastSLAM proposal: eta's bound c K q_hi^k exceeds DBL_MAX at %zu used beams", k);
                return PFGPU_ERR_INVALID;
            }
        }
    }
    PF_CUDA(cudaSetDevice(h->ctx.device));
    Ctx& ctx = h->ctx;
    GsDev& d = h->d;
    if (B > h->rcap) {
        PF_CUDA(cudaStreamSynchronize(ctx.stream));
        cudaFree(h->ranges);
        h->ranges = nullptr; h->rcap = 0;
        PF_CUDA(cudaMalloc(&h->ranges, B * sizeof(double)));
        h->rcap = B;
    }
    if (B) PF_CUDA(cudaMemcpyAsync(h->ranges, ranges, B * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    if (k) PF_CUDA(cudaMemcpyAsync(h->pairs, hp.data(), hp.size() * sizeof(double), cudaMemcpyHostToDevice, ctx.stream));
    GsModel m;
    m.res = c.ogm.resolution; m.half_w = (double)c.ogm.width / 2.0; m.half_h = (double)c.ogm.height / 2.0;
    m.W = (int)c.ogm.width; m.H = (int)c.ogm.height; m.R = (int)c.search_radius;
    m.z_hit = c.z_hit; m.q_out = h->q_out; m.angle_min = angle_min;
    const size_t n = d.n;
    // move + weigh, normalise, N_eff and the gate
    if (pc.enabled)
        PF_LAUNCH(ctx, gs_propose_kernel, (unsigned)std::min<size_t>(n, (size_t)1 << 20), GS_PROP_NT, 0, d, om, h->seed, (uint32_t)h->steps,
                  m, (const double*)h->pairs, (unsigned)k, P, h->pout);
    else
        PF_LAUNCH(ctx, gs_move_weigh_kernel, cdiv_u(n, GS_WARPS), GS_WARPS * 32, 0, d, om, h->seed, (uint32_t)h->steps, m,
                  (const double*)h->pairs, (unsigned)k);
    h->last_prop = pc.enabled != 0;
    int rc = gs_normalize(h, d.scal + 0, nullptr);
    if (rc) return rc;
    rc = xs_total(ctx, h->xs, PfValWSq{d.w}, n, n, 0.0, d.scal + 1);
    if (rc) return rc;
    PF_LAUNCH(ctx, gs_gate_kernel, 1, 1, 0, d, c.nth, h->seed);
    // the resample's normalisation, CDF, comb and plan (no-ops when the gate is closed)
    rc = gs_normalize(h, d.scal + 2, d.gate);
    if (rc) return rc;
    h->xs.gate = d.gate;
    rc = xs_scan(ctx, h->xs, XsValArray{d.w}, XsSinkStore{d.cum}, n, n, 0.0, d.scal + 5);
    if (!rc) rc = xs_scan(ctx, h->xs, GsCombVal{d.scal + 3, 1.0 / (double)n}, XsSinkStore{d.comb}, n, n, 0.0, d.scal + 6);
    h->xs.gate = nullptr;
    if (rc) return rc;
    PF_CUDA(cudaMemsetAsync(d.has_child, 0, n * sizeof(int), ctx.stream));
    PF_LAUNCH(ctx, gs_search_kernel, cdiv_u(n, 256), 256, 0, d);
    PF_LAUNCH(ctx, gs_flags_kernel, cdiv_u(n, 256), 256, 0, d);
    size_t tb = h->tmp_bytes;
    PF_CUDA(cub::DeviceScan::ExclusiveSum(h->tmp, tb, d.nf, d.enf, (int)n, ctx.stream));
    tb = h->tmp_bytes;
    PF_CUDA(cub::DeviceScan::ExclusiveSum(h->tmp, tb, d.cl, d.ecl, (int)n, ctx.stream));
    PF_LAUNCH(ctx, gs_free_kernel, cdiv_u(n, 256), 256, 0, d);
    PF_LAUNCH(ctx, gs_plan_kernel, cdiv_u(n, 256), 256, 0, d);
    // fuse each grid that survives once, then copy it to its further children
    PfOgmGeom gm;
    gm.res = m.res; gm.half_w = m.half_w; gm.half_h = m.half_h; gm.W = m.W; gm.H = m.H;
    if (B) PF_LAUNCH(ctx, gs_fuse_kernel, (unsigned)n, GS_FUSE_NT, 0, d, gm, (const double*)h->ranges, B, angle_min, angle_inc,
                     c.ogm.occupied_log_odds, c.ogm.free_log_odds, c.ogm.min_log_odds, c.ogm.max_log_odds);
    const unsigned cx = std::max(1u, std::min<unsigned>(cdiv_u(d.cells, 256 * 4), 64u));
    PF_LAUNCH(ctx, gs_copy_kernel, dim3(cx, (unsigned)std::min<size_t>(n, 65535)), 256, 0, d);
    PF_LAUNCH(ctx, gs_finish_kernel, cdiv_u(n, 256), 256, 0, d);
    h->steps++;
    return 0;
}
extern "C" int pfgpu_gs_sync(pfgpu_gs* h) {
    if (!h) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_gs_download(pfgpu_gs* h, double* poses3, double* weights, size_t n) {
    if (!h || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    if (poses3) {
        std::vector<double> x(n), y(n), a(n);
        PF_CUDA(cudaMemcpyAsync(x.data(), h->d.px, n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaMemcpyAsync(y.data(), h->d.py, n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaMemcpyAsync(a.data(), h->d.pyaw, n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        for (size_t i = 0; i < n; ++i) { poses3[3 * i] = x[i]; poses3[3 * i + 1] = y[i]; poses3[3 * i + 2] = a[i]; }
    }
    if (weights) PF_CUDA(cudaMemcpyAsync(weights, h->d.w, n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_gs_best(pfgpu_gs* h, size_t* slot, double pose3[3]) {
    if (!h) return PFGPU_ERR_INVALID;
    const size_t n = h->d.n;
    std::vector<double> p(3 * n), w(n);
    int rc = pfgpu_gs_download(h, p.data(), w.data(), n);
    if (rc) return rc;
    size_t b = 0;
    for (size_t i = 1; i < n; ++i) if (w[i] > w[b]) b = i;
    if (slot) *slot = b;
    if (pose3) for (int j = 0; j < 3; ++j) pose3[j] = p[3 * b + j];
    return 0;
}
// the buffer slot's grid lives in, after the handle's work so far
static int gs_buffer(pfgpu_gs* h, size_t slot, unsigned* b) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(b, h->d.buf + slot, sizeof(unsigned), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_gs_grid_read(pfgpu_gs* h, size_t slot, size_t first, size_t count, double* out) {
    if (!h || slot >= h->d.n || first > h->d.cells || count > h->d.cells - first || (count && !out)) return PFGPU_ERR_INVALID;
    unsigned b = 0;
    int rc = gs_buffer(h, slot, &b);
    if (rc || count == 0) return rc;
    PF_CUDA(cudaMemcpyAsync(out, h->d.grids + (size_t)b * h->d.cells + first, count * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
extern "C" int pfgpu_gs_grid_to_ogm(pfgpu_gs* h, size_t slot, pfgpu_ogm* g) {
    if (!h || !g || slot >= h->d.n || g->ctx.device != h->ctx.device || memcmp(&g->cfg, &h->cfg.ogm, sizeof(pfgpu_ogm_config)) != 0)
        return PFGPU_ERR_INVALID;
    unsigned b = 0;
    int rc = gs_buffer(h, slot, &b);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(g->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(g->grid, h->d.grids + (size_t)b * h->d.cells, h->d.cells * sizeof(double), cudaMemcpyDeviceToDevice, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
// (gate, grids copied, fuse events, N_eff) of the last step
static int gs_last(pfgpu_gs* h, int* gate, unsigned long long cnt[4], double* neff) {
    PF_CUDA(cudaSetDevice(h->ctx.device));
    PF_CUDA(cudaMemcpyAsync(gate, h->d.gate, sizeof(int), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(cnt, h->d.cnt, 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaMemcpyAsync(neff, h->d.scal + 4, sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    if (h->steps == 0) *gate = 0;
    return 0;
}
extern "C" int pfgpu_gs_last_indices(pfgpu_gs* h, uint32_t* idx, size_t cap, size_t* n) {
    if (!h || !n || (cap && !idx)) return PFGPU_ERR_INVALID;
    int gate = 0;
    unsigned long long cnt[4];
    double neff;
    int rc = gs_last(h, &gate, cnt, &neff);
    if (rc) return rc;
    *n = gate ? h->d.n : 0;
    const size_t m = std::min(*n, cap);
    if (m) {
        PF_CUDA(cudaMemcpyAsync(idx, h->d.idx, m * sizeof(uint32_t), cudaMemcpyDeviceToHost, h->ctx.stream));
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    }
    return 0;
}
extern "C" int pfgpu_gs_info(pfgpu_gs* h, size_t* W, size_t* H, size_t* n, uint64_t* L, pfgpu_gs_stats* st) {
    if (!h) return PFGPU_ERR_INVALID;
    if (W) *W = (size_t)h->cfg.ogm.width;
    if (H) *H = (size_t)h->cfg.ogm.height;
    if (n) *n = h->d.n;
    if (L) *L = h->L;
    if (st) {
        int gate = 0;
        unsigned long long cnt[4];
        double neff = 0.0;
        int rc = gs_last(h, &gate, cnt, &neff);
        if (rc) return rc;
        st->steps = h->steps;
        st->neff = h->steps ? neff : 0.0;
        st->resampled = (uint64_t)gate;
        st->copies = gate ? cnt[1] : 0;
        st->events = h->steps ? cnt[2] : 0;
    }
    return 0;
}
extern "C" int pfgpu_gs_set_proposal(pfgpu_gs* h, const pfgpu_gs_proposal* p) {
    if (!h || !p || p->enabled > 1) return PFGPU_ERR_INVALID;
    auto step_ok = [](double v) { return finite_d(v) && v > 0.0; };
    auto range_ok = [](double v) { return finite_d(v) && v >= 0.0; };
    if (!range_ok(p->linear_range) || !step_ok(p->linear_step) || !range_ok(p->angular_range) || !step_ok(p->angular_step) ||
        !step_ok(p->lattice_linear_step) || !step_ok(p->lattice_angular_step))
        return PFGPU_ERR_INVALID;
    const double rl = round(p->linear_range / p->linear_step), ra = round(p->angular_range / p->angular_step);
    const double cand = (2.0 * rl + 1.0) * (2.0 * rl + 1.0) * (2.0 * ra + 1.0);
    if (p->half_width > GS_PROP_MAX_K || !(cand <= GS_PROP_MAX_CAND) || !(2.0 * ra + 1.0 <= GS_PROP_MAX_YAWS)) {
        snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "grid FastSLAM proposal: lattice half-width %u (at most %d) or %.0f match candidates "
                 "(at most %d)", p->half_width, GS_PROP_MAX_K, cand, GS_PROP_MAX_CAND);
        return PFGPU_ERR_UNSUPPORTED;
    }
    if (p->enabled && !h->pout.xh) {
        const size_t n = h->d.n;
        PF_CUDA(cudaSetDevice(h->ctx.device));
        GsPropOut o = {};
        if (cudaMalloc(&o.xh, 3 * n * sizeof(double)) != cudaSuccess || cudaMalloc(&o.eta, n * sizeof(double)) != cudaSuccess ||
            cudaMalloc(&o.took, n) != cudaSuccess) {
            cudaFree(o.xh); cudaFree(o.eta); cudaFree(o.took);
            cudaGetLastError();
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "grid FastSLAM proposal: out of device memory for %zu slots", n);
            return PFGPU_ERR_CUDA;
        }
        h->pout = o;
    }
    h->prop = *p;
    return 0;
}
extern "C" int pfgpu_gs_get_proposal(pfgpu_gs* h, pfgpu_gs_proposal* p) {
    if (!h || !p) return PFGPU_ERR_INVALID;
    *p = h->prop;
    return 0;
}
extern "C" int pfgpu_gs_last_proposal(pfgpu_gs* h, double* matched3, double* eta, uint8_t* took, size_t n) {
    if (!h || n != h->d.n) return PFGPU_ERR_INVALID;
    PF_CUDA(cudaSetDevice(h->ctx.device));
    if (!h->last_prop) {
        const double nan = std::numeric_limits<double>::quiet_NaN();
        PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
        if (matched3) std::fill(matched3, matched3 + 3 * n, nan);
        if (eta) std::fill(eta, eta + n, nan);
        if (took) std::fill(took, took + n, (uint8_t)0);
        return 0;
    }
    if (matched3) PF_CUDA(cudaMemcpyAsync(matched3, h->pout.xh, 3 * n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    if (eta) PF_CUDA(cudaMemcpyAsync(eta, h->pout.eta, n * sizeof(double), cudaMemcpyDeviceToHost, h->ctx.stream));
    if (took) PF_CUDA(cudaMemcpyAsync(took, h->pout.took, n, cudaMemcpyDeviceToHost, h->ctx.stream));
    PF_CUDA(cudaStreamSynchronize(h->ctx.stream));
    return 0;
}
