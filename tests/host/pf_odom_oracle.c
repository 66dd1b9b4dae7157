/*
 * pf_odom_oracle.c — CPU oracle of the odometry motion model (DESIGN §3.14, the rule of include/pfgpu.h pfgpu_pf_*_odom).  TEST
 * INFRASTRUCTURE ONLY.  Includes tests/host/pf_beam_oracle.c (and so the likelihood-field, recovery and PF oracles) unchanged, and
 * adds the odometry predict through include/pf_odom_math.h, the header the library uses.  Draws from Philox, or injected (non-NULL
 * arrays) so that tests/golden/make_odom_golden.py pins the arithmetic without Philox.  Built twice by tests/_odom_oracle.py
 * (contract math; glibc libm with -DPF_ORACLE_LIBM, where atan2 and sin / cos are glibc's, as in Python's math module).
 */
#include "pf_beam_oracle.c"

#ifdef PF_ORACLE_LIBM
#define PF_ODOM_ATAN2(y, x) atan2((y), (x))
#define PF_ODOM_SINCOS(a, s, c) (*(s) = sin(a), *(c) = cos(a))
#endif
#include "../../include/pf_odom_math.h"

/* the host-side values of one call: out6 = (rot1, trans, rot2, s_rot1, s_trans, s_rot2); -1 when refused */
int orc_od_increment(const double odom6[6], const double alpha4[4], double out6[6]) {
    PfOdom m;
    if (!pf_odom_alpha_ok(alpha4) || pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
    out6[0] = m.rot1; out6[1] = m.trans; out6[2] = m.rot2; out6[3] = m.s_rot1; out6[4] = m.s_trans; out6[5] = m.s_rot2;
    return 0;
}
int orc_od_alpha_ok(const double alpha4[4]) { return pf_odom_alpha_ok(alpha4); }

/* pfgpu_pf_predict_odom on the recovery oracle r: the injection of orc_rec_predict_with_draws (inj4 as there), then every particle
 * moved by the increment.  z3: n x (za, zb, zc) or NULL (Philox: PF_PREDICT's pair, PF_ODOM's first normal) */
int orc_od_predict(orc_rec* r, const double odom6[6], const double alpha4[4], const double* z3, const double* inj4) {
    orc_pf* f = r->f;
    PfOdom m;
    if (!pf_odom_alpha_ok(alpha4) || pf_odom_increment(odom6, alpha4, &m) != 0) return -1;
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
    const uint64_t seed = f->seed;
    const uint32_t call = f->n_predict;
    long n = (long)f->n;
#pragma omp parallel for num_threads(f->threads) schedule(static) if (f->threads > 1)
    for (long i = 0; i < n; ++i) {
        orc_particle* q = &f->p[i];
        double za, zb, zc, unused;
        if (z3) { za = z3[3 * i]; zb = z3[3 * i + 1]; zc = z3[3 * i + 2]; }
        else {
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_PF_PREDICT, call, (uint64_t)i), &za, &zb);
            pfc_normal_pair(pfc_rng_block(seed, PFC_STREAM_PF_ODOM, call, (uint64_t)i), &zc, &unused);
        }
        pf_odom_move(&m, za, zb, zc, &q->x, &q->y, &q->yaw);
    }
    f->n_predict++;
    refresh_cache(f);
    return 0;
}
