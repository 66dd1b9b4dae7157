/*
 * x3_core.h — element-level logic of the exact sequential-order sum / scan used by the fused FastSLAM post-step kernel
 * (fs3_post.cuh).  Same theory as xsum_core.h (read that header first): while the running sum stays inside one binade its
 * ulp is constant and adding a tie-free value is an integer increment of the mantissa, independent of the sum.  What is new:
 *
 *   - a value is classified with integer operations on the bit patterns of the approximate prefix before / after it
 *     (no floating-point margin arithmetic): "clean" needs both prefixes in the same binade and at least M units (of 2^-32
 *     of the binade) away from its edges, M >= 2*rel*2^32 + 2 with the rigorous rel = 8(n+64)2^-53 — any summation order
 *     of the same non-negative terms differs from the sequential one by less than that (xsum_core.h);
 *   - clean increments are summed by an ordinary (non-segmented) 64-bit prefix sum P over all values; a dirty value records
 *     P in front of it, so the clean run between two dirty values is a difference of two prefixes and the chain that applies
 *     the dirty values in order is   s = bits(s) + (P_k - P_{k-1});  s = s + v_k   — two dependent operations per entry;
 *   - the systematic comb r_t = fl(r_{t-1} + 1/n) (fs1.rs:219-230) has a closed form per slot when n is a power of two.
 *
 * Shared with tests/host/x3_emul.cpp, which runs the same pass structure on the CPU against a plain loop.
 */
#ifndef X3_CORE_H
#define X3_CORE_H

#include "../../include/pf_contract_math.h"

/* margin in units of 2^-32 of a binade for sums of up to n terms (see above; the +2 absorbs the truncation to 32 bits) */
PFC_HD unsigned x3_margin32(unsigned long long n) {
    unsigned long long m = ((n + 64ull) * 8ull + ((1ull << 20) - 1ull)) >> 20;      /* ceil(2*rel*2^52 / 2^20), rel = 8(n+64)2^-53 */
    return (unsigned)(m + 2ull);
}

/* One value v >= 0 (finite) with approximate prefix a0 before and a1 = fl(a0 + v) after it.
 * Returns 0: clean, *inc = mantissa increment at the binade of a0 (biased exponent *lvl);  1: dirty (genuine FP add). */
PFC_HD int x3_classify(double v, double a0, double a1, unsigned m32, unsigned long long* inc, int* lvl) {
    const uint64_t bv = pfc_d2u(v), b0 = pfc_d2u(a0), b1 = pfc_d2u(a1);
    const int e0 = (int)(b0 >> 52), e1 = (int)(b1 >> 52), ev = (int)(bv >> 52);
    *inc = 0ull; *lvl = e0;
    if (v == 0.0) return 0;                                   /* no effect on any sum */
    /* the true prefix is >= a0(1-rel) >= 2^(e0-1): its ulp is >= 2^(e0-1-52); v < 2^(ev+1) <= half of that: no effect,
     * whatever binade the sum is really in (keeps long tails of negligible weights clean even at a binade edge) */
    if (e0 - ev >= 55) return 0;
    const unsigned f0 = (unsigned)(b0 >> 20), f1 = (unsigned)(b1 >> 20);      /* top 32 fraction bits */
    const unsigned span = 0xFFFFFFFFu - 2u * m32;
    if (e0 == 0 || e1 != e0 || (f0 - m32) > span || (f1 - m32) > span) return 1;
    const int evn = ev ? ev : 1;                              /* subnormal v: same scale as exponent 1 */
    const int sh = e0 - evn;                                  /* 0..54: v <= a1 < 2^(e0+1) */
    const uint64_t mant = (bv & 0x000FFFFFFFFFFFFFull) | (ev ? 0x0010000000000000ull : 0ull);
    if (sh == 0) { *inc = mant; return 0; }
    const uint64_t half = 1ull << (sh - 1);
    const uint64_t t = mant + half;
    if ((t & ((half << 1) - 1ull)) == 0ull) return 1;         /* exact tie: rounding depends on the parity of the sum */
    *inc = t >> sh;
    return 0;
}

/* A run of consecutive values whose approximate prefixes before the first (a_first) and after the last (a_last) lie in the SAME
 * binade, both at least the margin away from its edges: every true prefix in between does too (the prefixes are monotone), so
 * every value of the run is classified at that binade without looking at its own prefix.  Returns the biased exponent, or -1. */
PFC_HD int x3_interior(double a_first, double a_last, unsigned m32) {
    const uint64_t b0 = pfc_d2u(a_first), b1 = pfc_d2u(a_last);
    const int e0 = (int)(b0 >> 52), e1 = (int)(b1 >> 52);
    const unsigned f0 = (unsigned)(b0 >> 20), f1 = (unsigned)(b1 >> 20);
    const unsigned span = 0xFFFFFFFFu - 2u * m32;
    if (e0 == 0 || e0 >= 2047 || e1 != e0 || (f0 - m32) > span || (f1 - m32) > span) return -1;
    return e0;
}
/* x3_classify for a value inside such a run (same decisions, same increments): 0 clean, 1 dirty (an exact tie) */
PFC_HD int x3_classify_at(double v, int e0, unsigned long long* inc) {
    const uint64_t bv = pfc_d2u(v);
    const int ev = (int)(bv >> 52);
    *inc = 0ull;
    if (v == 0.0 || e0 - ev >= 55) return 0;
    const int evn = ev ? ev : 1;
    const int sh = e0 - evn;
    const uint64_t mant = (bv & 0x000FFFFFFFFFFFFFull) | (ev ? 0x0010000000000000ull : 0ull);
    if (sh == 0) { *inc = mant; return 0; }
    const uint64_t half = 1ull << (sh - 1);
    const uint64_t t = mant + half;
    if ((t & ((half << 1) - 1ull)) == 0ull) return 1;
    *inc = t >> sh;
    return 0;
}

/* apply a clean run (mantissa increment dp at biased exponent lvl, lvl < 0: unknown) to the exact sum s.
 * *ok = 0 when the certificate fails (the run was classified for another binade, or leaves it). */
PFC_HD double x3_apply(double s, unsigned long long dp, int lvl, int* ok) {
    if (dp == 0ull) return s;
    const uint64_t b = pfc_d2u(s), nb = b + dp;
    if (dp >= (1ull << 53) || (nb >> 52) != (b >> 52) || (lvl >= 0 && (int)(b >> 52) != lvl)) *ok = 0;
    return pfc_u2d(nb);
}

/* r_t of the systematic comb for n = 2^p: r_0 = r0 in [0, 1/n), r_t = fl(r_{t-1} + inv), inv = 2^-p.
 * Inside a binade every addition is exact (r is a multiple of the binade's ulp, and so is inv); the step that enters the
 * next binade rounds once (to even).  So the sequential value is reached in <= p + 2 jumps. */
PFC_HD double x3_comb_pow2(double r0, double inv, double ninv /* = 2^p */, unsigned long long t) {
    double v = r0;
    unsigned long long done = 0;
    while (done < t) {
        const uint64_t b = pfc_d2u(v);
        const int e = (int)(b >> 52);
        const double top = e >= 2046 ? v : pfc_u2d((uint64_t)(e + 1) << 52);          /* upper edge of v's binade */
        /* steps until r reaches `top`: ceil((top - v) / inv), all exact */
        double j = ceil((top - v) * ninv);
        if (!(j >= 1.0)) j = 1.0;
        const unsigned long long left = t - done;
        if ((double)left < j) { v = v + (double)left * inv; break; }
        v = v + (j - 1.0) * inv;          /* exact */
        v = v + inv;                      /* the one rounding step */
        done += (unsigned long long)j;
    }
    return v;
}

/* The same comb as a table: segment k covers slots [T_k, T_{k+1}) on which r_t = V_k + (t - T_k) * inv EXACTLY (no rounding
 * inside a binade); V_{k+1} is the one rounded addition that enters the next binade.  At most p + 3 segments for n = 2^p. */
#define X3_COMB_SEGS 72
typedef struct { int n; unsigned long long T[X3_COMB_SEGS + 1]; double V[X3_COMB_SEGS]; } x3_comb_table;
PFC_HD void x3_comb_build(x3_comb_table* tb, double r0, double inv, double ninv, unsigned long long n) {
    unsigned long long t = 0; double v = r0; int k = 0;
    while (t < n && k < X3_COMB_SEGS) {
        tb->T[k] = t; tb->V[k] = v; k++;
        const int e = (int)(pfc_d2u(v) >> 52);
        const double top = e >= 2046 ? v : pfc_u2d((uint64_t)(e + 1) << 52);
        double j = ceil((top - v) * ninv);
        if (!(j >= 1.0)) j = 1.0;
        if (j >= 1.8e19 || t + (unsigned long long)j >= n) { t = n; break; }
        v = v + (j - 1.0) * inv;
        v = v + inv;
        t += (unsigned long long)j;
    }
    tb->n = k; tb->T[k] = n;
}
PFC_HD double x3_comb_eval(const x3_comb_table* tb, double inv, unsigned long long t) {
    int k = 0;
    while (k + 1 < tb->n && tb->T[k + 1] <= t) ++k;
    return tb->V[k] + (double)(t - tb->T[k]) * inv;
}

/* Certified CDF (DESIGN §1).  c is fl(P_j / S); the CDF value the reference computes lies within dl * c + ab of it.  Returns 1
 * when a comb value r_t (n = 2^p values, r_0 = r0, step inv = 2^-p, ninv = 2^p) may lie within that distance of c, i.e. when
 * "c_j >= r_t" might come out differently for c than for the reference's value.  r0 + t inv stands in for the sequential r_t:
 * the accumulation rounds at most p + 3 times (once per binade it enters), by at most 2^-54 each, and the stand-in once more;
 * ab carries that (p + 4) 2^-53.  A comb value within distance 1 / (2n) of c has t within one of (c - r0) n: four candidates. */
PFC_HD int x3_cdf_near_comb(double c, double r0, double inv, double ninv, unsigned long long n, double dl, double ab) {
    const double lim = dl * c + ab;
    const double t0 = floor((c - r0) * ninv) - 1.0;
    int near = 0;
    for (int i = 0; i < 4; ++i) {
        const double t = t0 + (double)i;
        if (t >= 0.0 && t < (double)n && fabs((r0 + t * inv) - c) <= lim) near = 1;
    }
    return near;
}

#endif
