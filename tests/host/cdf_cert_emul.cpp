// Host model of the certified CDF of the fused FastSLAM post kernel (rust_robotics_b200/csrc/fs3.cuh, DESIGN §1): the kernel
// stores c~_j = fl(P_j / S), P_j the exact sequential prefix of the raw weights, and checks every c~_j against the comb with
// x3_cdf_near_comb (x3_core.h).  Compared by tests/test_cdf_cert_host.py with the reference's own steps: normalise, re-normalise
// by S2, cum_sum, r += 1/n, "while r > cum_sum[j+1] && j < n-1 { j += 1 }" (fs1.rs:196-230).
#include <cstdint>
#include <cmath>
#include <vector>
#include "../../rust_robotics_b200/csrc/x3_core.h"

// the kernel's bounds for n = 2^p (fs3_post_kernel)
static void cert_bounds(unsigned long long n, int p, double* dl, double* ab) {
    const double g = 4.0 * (double)n * 1.1102230246251565e-16;
    *dl = g / (1.0 - g) * (1.0 + 9.5367431640625e-07);
    *ab = (4.0 * (double)n + 4.0) * 4.9406564584124654e-324 + (double)(p + 4) * 1.1102230246251565e-16;
}

static void comb_indices(const double* cdf, size_t n, double r0, double inv, unsigned* idx) {
    double r = r0;
    size_t j = 0;
    for (size_t t = 0; t < n; ++t) {
        while (r > cdf[j] && j < n - 1) j += 1;
        idx[t] = (unsigned)j;
        r = r + inv;
    }
}

// returns 1 when the certificate refuses (some comb value may sit on the other side of a c~_j); idx_cert: the indices searched
// in c~, idx_ref: the reference's.  cert_out / ref_out (may be null): c~ and the reference's CDF.
extern "C" int cdf_cert_emul(const double* w_raw, int p, double r0, unsigned* idx_cert, unsigned* idx_ref, double* cert_out, double* ref_out) {
    const size_t n = (size_t)1 << p;
    const double inv = std::ldexp(1.0, -p), ninv = std::ldexp(1.0, p);
    double S = 0.0;
    for (size_t i = 0; i < n; ++i) S = S + w_raw[i];
    // reference: normalize_weights, resample's re-normalisation, cum_sum
    std::vector<double> w(n), c(n), ct(n);
    for (size_t i = 0; i < n; ++i) w[i] = w_raw[i] / S;
    double S2 = 0.0;
    for (size_t i = 0; i < n; ++i) S2 = S2 + w[i];
    double acc = 0.0;
    for (size_t i = 0; i < n; ++i) { acc = acc + w[i] / S2; c[i] = acc; }
    // certified: exact sequential prefixes of the raw weights, one division each
    double dl, ab;
    cert_bounds(n, p, &dl, &ab);
    int near = 0;
    double P = 0.0;
    for (size_t i = 0; i < n; ++i) {
        P = P + w_raw[i];
        ct[i] = P / S;
        near |= x3_cdf_near_comb(ct[i], r0, inv, ninv, n, dl, ab);
    }
    comb_indices(ct.data(), n, r0, inv, idx_cert);
    comb_indices(c.data(), n, r0, inv, idx_ref);
    if (cert_out) for (size_t i = 0; i < n; ++i) cert_out[i] = ct[i];
    if (ref_out) for (size_t i = 0; i < n; ++i) ref_out[i] = c[i];
    return near;
}
