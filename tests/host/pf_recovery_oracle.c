/*
 * pf_recovery_oracle.c — CPU oracle of augmented MCL (DESIGN §3.8, the rule of include/pfgpu.h pfgpu_pf_recovery_*).  TEST
 * INFRASTRUCTURE ONLY.  Includes oracle/pf_oracle.c unchanged and adds the filter, the injection and init_region in the engine's
 * operation order.  Draws from Philox, or injected (non-NULL arrays) so that tests/golden/make_recovery_golden.py pins the
 * arithmetic without Philox.  Built twice by tests/_recovery_oracle.py (contract math; glibc libm with -DPF_ORACLE_LIBM).
 */
#include "../../oracle/pf_oracle.c"

typedef struct {
    orc_pf* f;
    int on, armed;
    double a_slow, a_fast, region[4];
    double w_slow, w_fast, p;
    uint64_t injected;
} orc_rec;

static int region_ok(const double* r) {
    if (!r) return 0;
    for (int j = 0; j < 4; ++j) if (!finite_(r[j])) return 0;
    return r[0] < r[1] && r[2] < r[3];
}
static void rec_reset(orc_rec* r) { r->w_slow = r->w_fast = r->p = 0.0; r->injected = 0; r->armed = 0; }

orc_rec* orc_rec_new(const orc_pf_config* cfg, uint64_t seed) {
    orc_pf* f = orc_pf_new(cfg, seed);
    if (!f) return NULL;
    orc_rec* r = (orc_rec*)calloc(1, sizeof(orc_rec));
    r->f = f;
    return r;
}
void orc_rec_free(orc_rec* r) { if (r) { orc_pf_free(r->f); free(r); } }
orc_pf* orc_rec_pf(orc_rec* r) { return r->f; }

int orc_rec_enable(orc_rec* r, double a_slow, double a_fast, const double region[4]) {
    const int off = a_slow == 0.0 && a_fast == 0.0;
    if (!off && (!(a_slow > 0.0) || !(a_slow < a_fast) || !(a_fast <= 1.0) || !region_ok(region))) return -1;
    r->on = !off;
    r->a_slow = off ? 0.0 : a_slow; r->a_fast = off ? 0.0 : a_fast;
    for (int j = 0; j < 4; ++j) r->region[j] = off ? 0.0 : region[j];
    rec_reset(r);
    return 0;
}
void orc_rec_state(const orc_rec* r, double out3[3], uint64_t* injected) {
    out3[0] = r->w_slow; out3[1] = r->w_fast; out3[2] = r->p;
    *injected = r->injected;
}

static void rec_filter(orc_rec* r, double S, size_t n) {
    if (!r->on) return;
    if (finite_(S)) {
        const double w_avg = S / (double)n;
        r->w_slow = r->w_slow + r->a_slow * (w_avg - r->w_slow);
        r->w_fast = r->w_fast + r->a_fast * (w_avg - r->w_fast);
    }
    double p = 0.0;
    if (r->w_slow > 0.0) {
        const double q = r->w_fast / r->w_slow;
        if (finite_(q)) { p = 1.0 - q; if (!(p > 0.0)) p = 0.0; }
    }
    r->p = p;
}

/* u3: n x (x, y, yaw fractions), or NULL for Philox */
int orc_rec_init_region_with_uniforms(orc_rec* r, const double region[4], const double* u3) {
    if (!region_ok(region)) return -1;
    orc_pf* f = r->f;
    f->n = f->cfg.n_particles;
    for (size_t i = 0; i < f->n; ++i) {
        double fx, fy, fyaw;
        if (u3) { fx = u3[3 * i]; fy = u3[3 * i + 1]; fyaw = u3[3 * i + 2]; }
        else {
            pfc_u32x4 a = pfc_rng_block(f->seed, PFC_STREAM_REGION_A, 0, i), b = pfc_rng_block(f->seed, PFC_STREAM_REGION_B, 0, i);
            fx = pfc_u01_53(pfc_blk_u64(a, 0)); fy = pfc_u01_53(pfc_blk_u64(a, 1)); fyaw = pfc_u01_53(pfc_blk_u64(b, 0));
        }
        orc_particle* q = &f->p[i];
        pfc_region_pose(region, fx, fy, fyaw, &q->x, &q->y, &q->yaw);
        q->v = 0.0;
        q->w = 1.0 / (double)f->n;
    }
    rec_reset(r);
    refresh_cache(f);
    return 0;
}
int orc_rec_init_state(orc_rec* r, const double s[4]) {
    const int rc = orc_pf_init_state(r->f, s);
    if (!rc) rec_reset(r);
    return rc;
}
void orc_rec_upload(orc_rec* r, const double* aos5, size_t n) { orc_pf_set_particles(r->f, aos5, n); rec_reset(r); }

/* zv, zw: n motion draws or NULL; inj4: n x (a0, a1, b0, b1) or NULL (Philox) */
int orc_rec_predict_with_draws(orc_rec* r, const double u[2], const double* zv, const double* zw, const double* inj4) {
    orc_pf* f = r->f;
    if (!finite_(u[0]) || !finite_(u[1])) return -1;
    if (r->on) {
        r->injected = 0;
        if (r->armed && r->p > 0.0) {
            for (size_t i = 0; i < f->n; ++i) {
                const pfc_u32x4 a = pfc_rng_block(f->seed, PFC_STREAM_PF_INJECT_A, f->n_predict, i);
                const double a0 = inj4 ? inj4[4 * i] : pfc_u01_53(pfc_blk_u64(a, 0));
                if (!(a0 < r->p)) continue;
                const pfc_u32x4 b = pfc_rng_block(f->seed, PFC_STREAM_PF_INJECT_B, f->n_predict, i);
                const double a1 = inj4 ? inj4[4 * i + 1] : pfc_u01_53(pfc_blk_u64(a, 1));
                const double b0 = inj4 ? inj4[4 * i + 2] : pfc_u01_53(pfc_blk_u64(b, 0)), b1 = inj4 ? inj4[4 * i + 3] : pfc_u01_53(pfc_blk_u64(b, 1));
                orc_particle* q = &f->p[i];
                pfc_region_pose(r->region, a1, b0, b1, &q->x, &q->y, &q->yaw);
                q->v = 0.0;
                r->injected++;
            }
        }
    }
    r->armed = 0;
    return predict_impl(f, u, zv, zw);
}

/* orc_pf_update, keeping S = sum w_raw (the sequential sum normalize_weights takes) for the filter */
int orc_rec_update(orc_rec* r, const double* obs, size_t k) {
    orc_pf* f = r->f;
    for (size_t j = 0; j < k; ++j)
        if (!finite_(obs[3 * j]) || !finite_(obs[3 * j + 1]) || !finite_(obs[3 * j + 2]) || obs[3 * j] < 0.0)
            return -1;
    const double sigma = f->cfg.range_noise;
    long n = (long)f->n;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1)
    for (long i = 0; i < n; ++i) {
        orc_particle* q = &f->p[i];
        double w = 1.0;
        for (size_t j = 0; j < k; ++j) {                       /* orc_pf_update's order: diff = d - sqrt(dx dx + dy dy) */
            const double dx = q->x - obs[3 * j + 1], dy = q->y - obs[3 * j + 2];
            w *= gauss_likelihood(obs[3 * j] - sqrt(dx * dx + dy * dy), sigma);
        }
        q->w = w;
    }
    double S = 0.0;
    for (size_t i = 0; i < f->n; ++i) S += f->p[i].w;
    rec_filter(r, S, f->n);
    normalize_weights(f);
    refresh_cache(f);
    r->armed = 0;
    return 0;
}

/* the resample stage; r = NULL: Philox.  PF keeps its N_eff gate (unlike orc_pf_resample_with_uniforms) */
int orc_rec_resample_with_uniforms(orc_rec* r, const double* rs, size_t nr) {
    orc_pf* f = r->f;
    int did;
    if (!rs) did = orc_pf_resample(f);
    else if (f->cfg.mode == 1) { mcl_resample_adaptive(f, rs, nr); did = 1; }
    else {
        did = orc_pf_neff(f) < (double)f->cfg.n_particles * f->cfg.resample_threshold;
        if (did) { pf_resample_particles(f, rs); refresh_cache(f); }
    }
    r->armed = did;
    return did;
}

