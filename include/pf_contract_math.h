/*
 * pf_contract_math.h — the NUMERICAL CONTRACT shared by the CUDA kernels and the CPU oracle.
 *
 * Why this file exists
 * --------------------
 * The reference (rust_robotics, crates/rust_robotics_localization/src/particle_filter.rs,
 * monte_carlo_localization.rs, crates/rust_robotics_slam/src/fastslam1.rs) computes in IEEE f64 and
 * calls, besides + - * / sqrt, exactly five libm functions: sin, cos (pf.rs:292-293, fs1.rs:73-74,146-147),
 * exp (pf.rs:478, fs1.rs:180), atan2 (fs1.rs:97) and — through rand_distr — whatever the ziggurat
 * normal sampler needs.  It seeds nothing (rand::rng(), pf.rs:258,443; fs1.rs:129-130,220).
 *
 * To make "GPU result == oracle result" a BIT-EXACT statement for every particle, weight and resample
 * index, both sides must evaluate the same correctly-specified arithmetic.  + - * / sqrt and fma are
 * correctly rounded by IEEE-754 on x86-64 and on sm_90a, so every function below is written ONLY in
 * terms of those operations (explicit fma(), never compiler contraction) plus integer bit manipulation.
 * Build rules that make this hold:
 *     device:  nvcc --fmad=false            (no implicit a*b+c fusion)
 *     host:    gcc  -ffp-contract=off       (ditto; Rust never contracts either, SURVEY.md App. A)
 *
 * Deviations from the reference that this contract introduces (both documented in DESIGN.md):
 *   1. RNG: counter-based Philox4x32-10 + Box–Muller instead of thread-local ChaCha12 + ziggurat
 *      (the reference is unseeded, so no bit stream exists to reproduce).
 *   2. libm: pfc_exp/pfc_sincos/pfc_atan2 agree with glibc (what Rust's f64 methods call on Linux) to
 *      <= 2 ulp (tests/test_contract_math.py measures it); the oracle can also be built against glibc
 *      (-DPF_ORACLE_LIBM) to bound what that deviation does to a trajectory.
 *
 * The polynomial kernels follow the classic, publicly documented fdlibm (Sun, 1993) argument-reduction
 * schemes and coefficient sets, re-expressed with fma.
 */
#ifndef PF_CONTRACT_MATH_H
#define PF_CONTRACT_MATH_H

#include <stdint.h>
#include <math.h>
#include <string.h>

#if defined(__CUDACC__)
#define PFC_HD __host__ __device__ __forceinline__
#else
#define PFC_HD static inline __attribute__((always_inline))
#endif

/* ------------------------------------------------------------------------------------------------ */
/* bit casts                                                                                        */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD uint64_t pfc_d2u(double x) {
#if defined(__CUDA_ARCH__)
    return (uint64_t)__double_as_longlong(x);
#else
    uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
PFC_HD double pfc_u2d(uint64_t u) {
#if defined(__CUDA_ARCH__)
    return __longlong_as_double((long long)u);
#else
    double x; memcpy(&x, &u, 8); return x;
#endif
}
/* ------------------------------------------------------------------------------------------------ */
/* Division.  The CONTRACT is IEEE-754 correctly rounded a/b.  On the host that is the `/` operator.  On the device the
 * same value is obtained ~4x cheaper from a correctly rounded reciprocal y = RN(1/b) (__drcp_rn) and two fma
 * correction steps (Markstein): q0 = a*y; r0 = a - b*q0 (exact in fma); q1 = q0 + r0*y; r1 = a - b*q1; q = q1 + r1*y.
 * With y correctly rounded and no over/underflow this is RN(a/b) for every a, b (tests/host/divtest.c: 0 mismatches in
 * 4e9 random and adversarial cases; the one-correction form already has none).  Operands outside [1e-150, 1e150]
 * (and zeros, for the sign of zero) take the plain division, so the result is ALWAYS the IEEE quotient. */
#if defined(__CUDA_ARCH__)
typedef struct { double b, y; int ok; } pfc_rcp_t;
PFC_HD int pfc_div_inrange(double x) { double ax = fabs(x); return ax > 1e-150 && ax < 1e150; }
PFC_HD pfc_rcp_t pfc_rcp_make(double b) { pfc_rcp_t r; r.b = b; r.ok = pfc_div_inrange(b); r.y = __drcp_rn(b); return r; }
PFC_HD double pfc_div_by(double a, const pfc_rcp_t r) {
    if (r.ok && pfc_div_inrange(a)) {
        double q0 = a * r.y;
        double r0 = fma(-r.b, q0, a);
        double q1 = fma(r0, r.y, q0);
        double r1 = fma(-r.b, q1, a);
        return fma(r1, r.y, q1);
    }
    return a / r.b;
}
#define PFC_DIV(a, b) pfc_div_by((a), pfc_rcp_make(b))
#else
typedef struct { double b; } pfc_rcp_t;
PFC_HD pfc_rcp_t pfc_rcp_make(double b) { pfc_rcp_t r; r.b = b; return r; }
PFC_HD double pfc_div_by(double a, const pfc_rcp_t r) { return a / r.b; }
#define PFC_DIV(a, b) ((a) / (b))
#endif

/* 2^k for k in [-1022, 1023] */
PFC_HD double pfc_pow2i(int k) { return pfc_u2d((uint64_t)(k + 1023) << 52); }

#define PFC_PI      3.14159265358979323846
#define PFC_TWO_PI  6.28318530717958647692

/* ------------------------------------------------------------------------------------------------ */
/* Philox4x32-10 (Salmon et al., SC'11).  ctr = 128-bit counter, key = 64-bit key.                  */
/* ------------------------------------------------------------------------------------------------ */
typedef struct { uint32_t v[4]; } pfc_u32x4;

PFC_HD pfc_u32x4 pfc_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                   uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0;
        uint64_t p1 = (uint64_t)M1 * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += W0; k1 += W1;
    }
    pfc_u32x4 o; o.v[0] = c0; o.v[1] = c1; o.v[2] = c2; o.v[3] = c3; return o;
}

/* Stream ids: which reference draw a Philox block stands for. */
enum {
    PFC_STREAM_PF_PREDICT  = 0,  /* pf.rs:280-287 / mcl.rs:237-244: (v_noise, yaw_noise) of particle i   */
    PFC_STREAM_PF_RESAMPLE = 1,  /* pf.rs:456 / mcl.rs:344: uniform r of output slot t                  */
    PFC_STREAM_FS_PREDICT  = 2,  /* fs1.rs:129-130: two N(0,1) of particle i                            */
    PFC_STREAM_FS_RESAMPLE = 3,  /* fs1.rs:219-220: the single U[0,1/n) draw                            */
    PFC_STREAM_INIT_A      = 4,  /* pf.rs:182-183 / mcl.rs:191-192: x,y jitter of particle i            */
    PFC_STREAM_INIT_B      = 5,  /* pf.rs:184-185 / mcl.rs:193-194: yaw,v jitter of particle i          */
    PFC_STREAM_OBS         = 6,  /* synthetic observation noise (examples / bench drivers)              */
    PFC_STREAM_FS2_POSE3   = 7,  /* fs2.rs:234: the third N(0,1) of sample_pose (the first two use FS_PREDICT) */
    /* augmented MCL (not in the reference; DESIGN §3.8), 53-bit uniforms, call = the predict's call index, index = global slot */
    PFC_STREAM_PF_INJECT_A = 8,  /* (decision u < p, x fraction) of the slot                            */
    PFC_STREAM_PF_INJECT_B = 9,  /* (y fraction, yaw fraction) of the slot                              */
    PFC_STREAM_REGION_A    = 10, /* init_region, call 0: (x fraction, y fraction) of particle i         */
    PFC_STREAM_REGION_B    = 11, /* init_region, call 0: (yaw fraction, unused) of particle i           */
    /* odometry motion model (not in the reference; DESIGN §3.14, include/pf_odom_math.h), call and index as PF_PREDICT's */
    PFC_STREAM_PF_ODOM     = 12, /* (zc = the third normal, unused) of particle i                       */
    /* FastSLAM's odometry motion model (DESIGN §3.15, include/fs_odom_math.h), call and index as FS_PREDICT's */
    PFC_STREAM_FS_ODOM     = 13  /* (zc = the third normal of the odometry move, unused) of particle i  */
};
/* A pose drawn uniformly over the box [x0, x1] x [y0, y1] from three 53-bit fractions (augmented MCL's injection and init_region):
 * x = x0 + fx * (x1 - x0), y = y0 + fy * (y1 - y0), yaw = fyaw * 2 pi - pi. */
PFC_HD void pfc_region_pose(const double r4[4], double fx, double fy, double fyaw, double* x, double* y, double* yaw) {
    *x = r4[0] + fx * (r4[1] - r4[0]);
    *y = r4[2] + fy * (r4[3] - r4[2]);
    *yaw = fyaw * PFC_TWO_PI - PFC_PI;
}

/* One block per (seed, stream, call#, index): counter = (index_lo, index_hi, call#, stream). */
PFC_HD pfc_u32x4 pfc_rng_block(uint64_t seed, uint32_t stream, uint32_t call, uint64_t index) {
    return pfc_philox4x32_10((uint32_t)index, (uint32_t)(index >> 32), call, stream,
                             (uint32_t)seed, (uint32_t)(seed >> 32));
}
PFC_HD uint64_t pfc_blk_u64(const pfc_u32x4 b, int which) {
    return ((uint64_t)b.v[2 * which + 1] << 32) | (uint64_t)b.v[2 * which];
}
/* U[0,1) with 53 bits: rand 0.9 `random::<f64>()` = (u64 >> 11) * 2^-53 (pf.rs:456, mcl.rs:344). */
PFC_HD double pfc_u01_53(uint64_t x) { return (double)(x >> 11) * 1.1102230246251565e-16; }
/* U(0,1) open at 0, for the logarithm in Box–Muller. */
PFC_HD double pfc_u01_open(uint64_t x) { return ((double)(x >> 11) + 0.5) * 1.1102230246251565e-16; }
/* U[0,1) with 52 bits: rand 0.9 `Uniform<f64>` = (bits(1.0 | x>>12) - 1.0) (fs1.rs:219-220). */
PFC_HD double pfc_u01_52(uint64_t x) { return pfc_u2d((x >> 12) | 0x3FF0000000000000ull) - 1.0; }

/* ------------------------------------------------------------------------------------------------ */
/* Polynomial / reduction constants.  On the device they live in constant memory, so an FP64 instruction takes them as
 * a constant-bank operand; as literals each one costs two 32-bit moves in front of the FMA that uses it (that was a
 * quarter of the instructions of the EKF kernel).  Host and device read the same list: same bits either way.        */
/* ------------------------------------------------------------------------------------------------ */
#define PFC_CONST_LIST(X) \
    X(LOG2E, 1.44269504088896338700e+00) \
    X(LN2_HI, 6.93147180369123816490e-01) \
    X(LN2_LO, 1.90821492927058770002e-10) \
    X(E13, 1.6059043836821613e-10) \
    X(E12, 2.08767569878681e-09) \
    X(E11, 2.505210838544172e-08) \
    X(E10, 2.755731922398589e-07) \
    X(E9, 2.7557319223985893e-06) \
    X(E8, 2.48015873015873e-05) \
    X(E7, 1.984126984126984e-04) \
    X(E6, 1.388888888888889e-03) \
    X(E5, 8.333333333333333e-03) \
    X(E4, 4.1666666666666664e-02) \
    X(E3, 1.6666666666666666e-01) \
    X(LG1, 6.666666666666735130e-01) \
    X(LG2, 3.999999999940941908e-01) \
    X(LG3, 2.857142874366239149e-01) \
    X(LG4, 2.222219843214978396e-01) \
    X(LG5, 1.818357216161805012e-01) \
    X(LG6, 1.531383769920937332e-01) \
    X(LG7, 1.479819860511658591e-01) \
    X(S1, -1.66666666666666324348e-01) \
    X(S2, 8.33333333332248946124e-03) \
    X(S3, -1.98412698298579493134e-04) \
    X(S4, 2.75573137070700676789e-06) \
    X(S5, -2.50507602534068634195e-08) \
    X(S6, 1.58969099521155010221e-10) \
    X(C1, 4.16666666666666019037e-02) \
    X(C2, -1.38888888888741095749e-03) \
    X(C3, 2.48015872894767294178e-05) \
    X(C4, -2.75573143513906633035e-07) \
    X(C5, 2.08757232129817482790e-09) \
    X(C6, -1.13596475577881948265e-11) \
    X(TWO_OVER_PI, 6.36619772367581382433e-01) \
    X(PIO2_1, 1.57079632679489655800e+00) \
    X(PIO2_2, 6.12323399573676603587e-17) \
    X(PIO2_3, -1.4973849048591698e-33) \
    X(AT0, 3.33333333333329318027e-01) \
    X(AT1, -1.99999999998764832476e-01) \
    X(AT2, 1.42857142725034663711e-01) \
    X(AT3, -1.11111104054623557880e-01) \
    X(AT4, 9.09088713343650656196e-02) \
    X(AT5, -7.69187620504482999495e-02) \
    X(AT6, 6.66107313738753120669e-02) \
    X(AT7, -5.83357013379057348645e-02) \
    X(AT8, 4.97687799461593236017e-02) \
    X(AT9, -3.65315727442169155270e-02) \
    X(AT10, 1.62858201153657823623e-02)
#define PFC_X_ENUM(n, v) PFC_K_##n,
enum { PFC_CONST_LIST(PFC_X_ENUM) PFC_K_COUNT };
#define PFC_X_VAL(n, v) v,
static const double pfc_k_host[PFC_K_COUNT] = { PFC_CONST_LIST(PFC_X_VAL) };
#ifdef __CUDACC__
static __constant__ double pfc_k_dev[PFC_K_COUNT] = { PFC_CONST_LIST(PFC_X_VAL) };
#endif
#ifdef __CUDA_ARCH__
#define PFC_K(n) pfc_k_dev[PFC_K_##n]
#else
#define PFC_K(n) pfc_k_host[PFC_K_##n]
#endif

/* ------------------------------------------------------------------------------------------------ */
/* exp                                                                                              */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD double pfc_exp(double x) {
    if (x != x) return x;
    if (x > 709.782712893384) return pfc_u2d(0x7FF0000000000000ull);
    if (x < -745.2) return 0.0;
    const double LOG2E  = PFC_K(LOG2E);
    const double LN2_HI = PFC_K(LN2_HI);
    const double LN2_LO = PFC_K(LN2_LO);
    double kf = floor(fma(x, LOG2E, 0.5));
    double r  = fma(-kf, LN2_HI, x);
    r = fma(-kf, LN2_LO, r);
    /* q(r) = sum_{j=2..13} r^(j-2)/j!  (Taylor; |r| <= 0.3466 -> truncation < 2^-57) */
    double q = PFC_K(E13);            /* 1/13! */
    q = fma(q, r, PFC_K(E12));          /* 1/12! */
    q = fma(q, r, PFC_K(E11));         /* 1/11! */
    q = fma(q, r, PFC_K(E10));         /* 1/10! */
    q = fma(q, r, PFC_K(E9));        /* 1/9!  */
    q = fma(q, r, PFC_K(E8));          /* 1/8!  */
    q = fma(q, r, PFC_K(E7));         /* 1/7!  */
    q = fma(q, r, PFC_K(E6));         /* 1/6!  */
    q = fma(q, r, PFC_K(E5));         /* 1/5!  */
    q = fma(q, r, PFC_K(E4));        /* 1/4!  */
    q = fma(q, r, PFC_K(E3));        /* 1/3!  */
    q = fma(q, r, 0.5);                           /* 1/2!  */
    double t = fma(r * r, q, r);
    double y = 1.0 + t;
    /* y * 2^k in two steps, k = k1 + k2 with both halves in pow2i's range: the first product is exact (normal), the
     * second rounds once — also when the result is subnormal or overflows — so no case split is needed */
    const int k = (int)kf, k1 = k >> 1, k2 = k - k1;
    return (y * pfc_pow2i(k1)) * pfc_pow2i(k2);
}

/* ------------------------------------------------------------------------------------------------ */
/* log (x > 0 finite; used only by Box–Muller)                                                      */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD double pfc_log(double x) {
    if (x != x || x < 0.0) return pfc_u2d(0x7FF8000000000000ull);
    if (x == 0.0) return -pfc_u2d(0x7FF0000000000000ull);
    uint64_t ux = pfc_d2u(x);
    int k = 0;
    if ((ux >> 52) == 0) { x *= 18014398509481984.0; ux = pfc_d2u(x); k = -54; }   /* subnormal */
    if ((ux >> 52) == 0x7FF) return x;
    k += (int)(ux >> 52) - 1023;
    uint64_t mant = ux & 0x000FFFFFFFFFFFFFull;
    double m = pfc_u2d(mant | 0x3FF0000000000000ull);          /* [1,2) */
    if (m > 1.4142135623730951) { m *= 0.5; k += 1; }           /* -> [sqrt2/2, sqrt2) */
    const double LN2_HI = PFC_K(LN2_HI), LN2_LO = PFC_K(LN2_LO);
    const double Lg1 = PFC_K(LG1), Lg2 = PFC_K(LG2),
                 Lg3 = PFC_K(LG3), Lg4 = PFC_K(LG4),
                 Lg5 = PFC_K(LG5), Lg6 = PFC_K(LG6),
                 Lg7 = PFC_K(LG7);
    double f = m - 1.0;
    double s = PFC_DIV(f, 2.0 + f);
    double z = s * s, w = z * z;
    double t1 = w * fma(w, fma(w, Lg6, Lg4), Lg2);
    double t2 = z * fma(w, fma(w, fma(w, Lg7, Lg5), Lg3), Lg1);
    double R = t2 + t1;
    double hfsq = 0.5 * f * f;
    double dk = (double)k;
    return dk * LN2_HI - ((hfsq - fma(s, hfsq + R, dk * LN2_LO)) - f);
}

/* ------------------------------------------------------------------------------------------------ */
/* sin / cos                                                                                        */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD double pfc_sin_kernel(double r) {
    const double S1 = PFC_K(S1), S2 = PFC_K(S2),
                 S3 = PFC_K(S3), S4 = PFC_K(S4),
                 S5 = PFC_K(S5), S6 = PFC_K(S6);
    double z = r * r;
    double p = fma(z, fma(z, fma(z, fma(z, fma(z, S6, S5), S4), S3), S2), S1);
    return fma(r * z, p, r);
}
PFC_HD double pfc_cos_kernel(double r) {
    const double C1 = PFC_K(C1), C2 = PFC_K(C2),
                 C3 = PFC_K(C3), C4 = PFC_K(C4),
                 C5 = PFC_K(C5), C6 = PFC_K(C6);
    double z = r * r;
    double p = fma(z, fma(z, fma(z, fma(z, fma(z, C6, C5), C4), C3), C2), C1);
    double hz = 0.5 * z;
    double w = 1.0 - hz;
    return w + (((1.0 - w) - hz) + (z * z) * p);
}
/* Accuracy contract: |x| <= 2^20*pi/2 (~1.6e6 rad).  Larger arguments are reduced by the same formula
 * with gracefully degrading accuracy; host and device still agree bit for bit. */
PFC_HD void pfc_sincos(double x, double* s, double* c) {
    if (!(fabs(x) <= 1.7976931348623157e308)) { *s = *c = pfc_u2d(0x7FF8000000000000ull); return; }
    const double TWO_OVER_PI = PFC_K(TWO_OVER_PI);
    const double P1 = PFC_K(PIO2_1);      /* fl(pi/2)            */
    const double P2 = PFC_K(PIO2_2);      /* fl(pi/2 - P1)       */
    const double P3 = PFC_K(PIO2_3);         /* fl(pi/2 - P1 - P2)  */
    double fn = floor(fma(x, TWO_OVER_PI, 0.5));
    double r = fma(-fn, P1, x);
    r = fma(-fn, P2, r);
    r = fma(-fn, P3, r);
    /* quadrant = fn mod 4, valid for |fn| < 2^52 */
    double q4 = fn - 4.0 * floor(fn * 0.25);
    int n = (int)q4;
    double sk = pfc_sin_kernel(r), ck = pfc_cos_kernel(r);
    double ss = (n & 1) ? ck : sk;
    double cc = (n & 1) ? sk : ck;
    if (n == 2 || n == 3) ss = -ss;
    if (n == 1 || n == 2) cc = -cc;
    *s = ss; *c = cc;
}
PFC_HD double pfc_sin(double x) { double s, c; pfc_sincos(x, &s, &c); return s; }
PFC_HD double pfc_cos(double x) { double s, c; pfc_sincos(x, &s, &c); return c; }

/* ------------------------------------------------------------------------------------------------ */
/* atan / atan2                                                                                     */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD double pfc_atan(double x) {
    if (x != x) return x;
    const double aT0 = PFC_K(AT0), aT1 = PFC_K(AT1),
                 aT2 = PFC_K(AT2), aT3 = PFC_K(AT3),
                 aT4 = PFC_K(AT4), aT5 = PFC_K(AT5),
                 aT6 = PFC_K(AT6), aT7 = PFC_K(AT7),
                 aT8 = PFC_K(AT8), aT9 = PFC_K(AT9),
                 aT10 = PFC_K(AT10);
    double ax = fabs(x);
    if (ax >= 7.378697629483821e19) {                 /* 2^66 */
        double r = 1.57079632679489655800e+00 + 6.12323399573676603587e-17;
        return x < 0.0 ? -r : r;
    }
    if (ax < 7.450580596923828e-09) return x;         /* 2^-27 */
    /* argument reduction atan(x) = hi + lo + atan(num/den), interval picked by selects: ONE division site and no
     * divergent region.  The first interval uses num/den = ax/1 (exact) and hi = lo = 0, for which the general
     * recombination below reduces, bit for bit, to t - t*(s1+s2). */
    const int i1 = ax >= 0.4375, i2 = ax >= 0.6875, i3 = ax >= 1.1875, i4 = ax >= 2.4375;
    double num = ax, den = 1.0, hi = 0.0, lo = 0.0;
    if (i1) { num = 2.0 * ax - 1.0; den = 2.0 + ax;       hi = 4.63647609000806093515e-01; lo = 2.26987774529616870924e-17; }
    if (i2) { num = ax - 1.0;       den = ax + 1.0;       hi = 7.85398163397448278999e-01; lo = 3.06161699786838301793e-17; }
    if (i3) { num = ax - 1.5;       den = 1.0 + 1.5 * ax; hi = 9.82793723247329054082e-01; lo = 1.39033110312309984516e-17; }
    if (i4) { num = -1.0;           den = ax;             hi = 1.57079632679489655800e+00; lo = 6.12323399573676603587e-17; }
    const double t = PFC_DIV(num, den);
    double z = t * t, w = z * z;
    double s1 = z * fma(w, fma(w, fma(w, fma(w, fma(w, aT10, aT8), aT6), aT4), aT2), aT0);
    double s2 = w * fma(w, fma(w, fma(w, fma(w, aT9, aT7), aT5), aT3), aT1);
    double r = hi - ((t * (s1 + s2) - lo) - t);
    return x < 0.0 ? -r : r;
}

PFC_HD double pfc_atan2(double y, double x) {
    if (x != x || y != y) return x + y;
    const double PI = 3.14159265358979311600e+00, PI_LO = 1.2246467991473531772e-16;
    const double PIO2 = 1.57079632679489655800e+00, PIO4 = 7.85398163397448278999e-01;
    const double INF = pfc_u2d(0x7FF0000000000000ull);
    int ysign = (int)(pfc_d2u(y) >> 63), xsign = (int)(pfc_d2u(x) >> 63);
    int m = ysign | (xsign << 1);
    double ay = fabs(y), ax = fabs(x);
    if (ay == 0.0) {
        switch (m) { case 0: case 1: return y; case 2: return PI; default: return -PI; }
    }
    if (ax == 0.0) return ysign ? -PIO2 : PIO2;
    if (ax == INF) {
        if (ay == INF) {
            switch (m) { case 0: return PIO4; case 1: return -PIO4;
                         case 2: return 3.0 * PIO4; default: return -3.0 * PIO4; }
        }
        switch (m) { case 0: return 0.0; case 1: return -0.0; case 2: return PI; default: return -PI; }
    }
    if (ay == INF) return ysign ? -PIO2 : PIO2;
    int ey = (int)((pfc_d2u(ay) >> 52) & 0x7FF), ex = (int)((pfc_d2u(ax) >> 52) & 0x7FF);
    int k = ey - ex;
    double z;
    if (k > 60) { z = PIO2 + 0.5 * PI_LO; m &= 1; }
    else if (xsign && k < -60) z = 0.0;
    else z = pfc_atan(PFC_DIV(ay, ax));
    switch (m) {
        case 0: return z;
        case 1: return -z;
        case 2: return PI - (z - PI_LO);
        default: return (z - PI_LO) - PI;
    }
}

/* ------------------------------------------------------------------------------------------------ */
/* N(0,1) pair by Box–Muller from one Philox block.  z0 uses cos, z1 uses sin.                      */
/* Stands in for rand_distr::Normal (pf.rs:260,269; fs1.rs:124); draw order "first, second" maps to  */
/* (z0, z1).                                                                                        */
/* ------------------------------------------------------------------------------------------------ */
PFC_HD void pfc_normal_pair(const pfc_u32x4 b, double* z0, double* z1) {
    double u1 = pfc_u01_open(pfc_blk_u64(b, 0));
    double u2 = pfc_u01_53(pfc_blk_u64(b, 1));
    double rad = sqrt(-2.0 * pfc_log(u1));
    double s, c;
    pfc_sincos(PFC_TWO_PI * u2, &s, &c);
    *z0 = rad * c; *z1 = rad * s;
}

#endif /* PF_CONTRACT_MATH_H */
