/* divtest_one.c — the fast form's one-correction quotient (fsm_div, include/fs_ekf_math.h) against IEEE a / b:
 *   q0 = RN(a y), r = RN(a - b q0), q = RN(q0 + r y), y = RN(1/b),
 * for a and b inside the window |x| in [2^-498, 2^498).  DESIGN §3.1 proves q = RN(a/b) there except possibly when both
 * significands lie within 10 ulp of 2; set E below checks that region exhaustively (a far wider one, in fact), the other
 * sets aim at the places where a short correction could go wrong.  Prints the counts; exit status 1 on any mismatch.
 * Driven by tests/test_div_one_correction_host.py. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

static double fd1(double a, double b, double y) { double q0 = a * y; double r = fma(-b, q0, a); return fma(r, y, q0); }
static double u2d(uint64_t u) { double d; memcpy(&d, &u, 8); return d; }
static uint64_t d2u(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
static uint64_t s[4] = { 0x9E3779B97F4A7C15ull, 0xBF58476D1CE4E5B9ull, 0x94D049BB133111EBull, 12345 };
static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
static uint64_t next(void) {                      /* xoshiro256** */
    uint64_t res = rotl(s[1] * 5, 7) * 9, t = s[1] << 17;
    s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3]; s[2] ^= t; s[3] = rotl(s[3], 45);
    return res;
}
/* sign | exponent e (unbiased) | 52-bit significand field m */
static double mk(int neg, int e, uint64_t m) { return u2d(((uint64_t)neg << 63) | ((uint64_t)(e + 1023) << 52) | (m & 0xFFFFFFFFFFFFFull)); }
static int in_window(double x) { double ax = fabs(x); return ax >= 0x1p-498 && ax < 0x1p498; }

static long long cases, bad;
static void check(double a, double b) {
    if (!in_window(a) || !in_window(b)) return;
    ++cases;
    const double y = 1.0 / b, q = a / b, f = fd1(a, b, y);
    if (d2u(f) != d2u(q)) {
        if (bad < 10) printf("mismatch a=%a b=%a: %a vs %a\n", a, b, f, q);
        ++bad;
    }
}
/* exponent pairs: the unit binade and the window's four corners (quotients from 2^-996 to 2^996) */
static const int EP[5][2] = { { 0, 0 }, { -498, 497 }, { 497, -498 }, { -498, -498 }, { 497, 497 } };

int main(int argc, char** argv) {
    long long nrand = argc > 1 ? atoll(argv[1]) : 20000000LL;
    long long c0;
    /* E: both significands among the 4096 largest (>= 2 - 2^-40), every pair, both signs of a, five exponent pairs */
    c0 = cases;
    for (uint64_t i = 0; i < 4096; ++i)
        for (uint64_t j = 0; j < 4096; ++j)
            for (int k = 0; k < 5; ++k) {
                check(mk(0, EP[k][0], 0xFFFFFFFFFFFFFull - i), mk(0, EP[k][1], 0xFFFFFFFFFFFFFull - j));
                if (k == 0) check(mk(1, 0, 0xFFFFFFFFFFFFFull - i), mk(0, 0, 0xFFFFFFFFFFFFFull - j));
            }
    printf("E  top significands     %lld cases\n", cases - c0);
    /* N: significands near all-ones or near 1 (few low bits free), every combination, random exponents in the window */
    c0 = cases;
    for (long long n = 0; n < nrand / 4; ++n) {
        uint64_t x = next(), z = next(), m = next();
        const int kind = (int)(m & 3), ea = (int)((m >> 8) % 995) - 498, eb = (int)((m >> 20) % 995) - 498;
        uint64_t ma = x, mb = z;
        if (kind == 0) { ma |= 0xFFFFFFFFFF000ull; mb |= 0xFFFFFFFFFF000ull; }
        if (kind == 1) { ma |= 0xFFFFFFFFFF000ull; mb &= 0xFFFull; }
        if (kind == 2) { ma &= 0xFFFull; mb |= 0xFFFFFFFFFF000ull; }
        if (kind == 3) { ma &= 0xFFFFull; mb &= 0xFFFFull; }
        check(mk((int)(m >> 40) & 1, ea, ma), mk((int)(m >> 41) & 1, eb, mb));
    }
    printf("N  near all-ones / one  %lld cases\n", cases - c0);
    /* B: quotients at binade edges, a = b * 2^k moved by -64..64 ulp (a/b just below and above a power of two) */
    c0 = cases;
    for (long long n = 0; n < nrand / 512; ++n) {
        uint64_t z = next(), m = next();
        if (m & 1) z |= 0xFFFFFFFF00000ull;
        const int eb = (int)((m >> 8) % 995) - 498, sh = (int)((m >> 20) % 9) - 4;
        const double b = mk(0, eb, z);
        const double a0 = ldexp(b, sh);
        uint64_t ua = d2u(a0);
        for (int t = -64; t <= 64; ++t) check(u2d(ua + (uint64_t)(int64_t)t), b);
    }
    printf("B  binade edges         %lld cases\n", cases - c0);
    /* M: quotients next to rounding midpoints, a ~= b (q + ulp(q)/2) moved by -2..2 ulp */
    c0 = cases;
    for (long long n = 0; n < nrand / 8; ++n) {
        uint64_t z = next(), x = next(), m = next();
        const double b = mk(0, (int)(m % 61) - 30, z), q = mk(0, (int)((m >> 8) % 61) - 30, x);
        const double h = ldexp(1.0, ilogb(q) - 53);
        const double a0 = fma(b, q, b * h);
        uint64_t ua = d2u(a0);
        for (int t = -2; t <= 2; ++t) check(u2d(ua + (uint64_t)(int64_t)t), b);
    }
    printf("M  near midpoints       %lld cases\n", cases - c0);
    /* W: operands at the window's ends, random significands */
    c0 = cases;
    for (long long n = 0; n < nrand / 4; ++n) {
        uint64_t x = next(), z = next(), m = next();
        const int ea = (m & 1) ? 497 : -498, eb = (m & 2) ? 497 : -498;
        check(mk((int)(m >> 2) & 1, ea, x), mk((int)(m >> 3) & 1, eb, z));
        check(mk(0, ea, x), mk(0, (int)((m >> 8) % 995) - 498, z));
    }
    printf("W  window ends          %lld cases\n", cases - c0);
    /* R: uniform random significands and exponents over the window */
    c0 = cases;
    for (long long n = 0; n < nrand; ++n) {
        uint64_t x = next(), z = next(), m = next();
        check(mk((int)(m >> 40) & 1, (int)(m % 995) - 498, x), mk((int)(m >> 41) & 1, (int)((m >> 12) % 995) - 498, z));
    }
    printf("R  random               %lld cases\n", cases - c0);
    printf("cases=%lld mismatches=%lld\n", cases, bad);
    return bad ? 1 : 0;
}
