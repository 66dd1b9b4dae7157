/* GPU probe for fsm_rcp / fsm_sqrt of include/fs_ekf_math.h: the branch-free reciprocal and square root of the EKF fast form
 * must return the same bits as __drcp_rn / __dsqrt_rn (RN(1/b), RN(sqrt(x))) on the window [2^-498, 2^498) that the fast
 * form certifies for every one of their operands.  Built by rust_robotics_b200/build.py (build_probe) with the library's
 * flags into a shared object of its own; tests/test_gpu_fast_rcp_sqrt.py calls fsm_probe_run through ctypes.
 *
 * Operand classes (each operand is a pure function of its class and index):
 *   0  random significands in every binade of the window (996 binades), random sign for the reciprocal
 *   1  both ends of the window: the first and the last 2^15 operands inside it
 *   2  powers of two and all-ones significands of every binade, 16 ulps either side (clipped to the window)
 *   3  the range of the atan denominator: random significands in the binades of [1, 2^64) (den in [1, 4.66) for the
 *      first four intervals, den = |dy|/|dx| in [2.4375, 2^62) for the last)
 *   4  den2 = 2 pi sqrt(det) for random det in the window (the square root is checked on det, the reciprocal on den2)
 */
#include <cstdint>
#include <cuda_runtime.h>

#include "../../include/fs_ekf_math.h"

#define FSM_PROBE_CLASSES 5
#define FSM_PROBE_FIELDS 4            /* per class: operands, reciprocal mismatches, square-root mismatches, first bad operand */

static const int64_t kLoExp = -498, kBinades = 996;       /* the window: biased exponents 525 .. 1520 */

__device__ __forceinline__ uint64_t fsm_probe_mix(uint64_t z) {      /* splitmix64 finaliser */
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}
__device__ __forceinline__ uint64_t fsm_probe_pow2_bits(int64_t e) { return (uint64_t)(e + 1023) << 52; }
__device__ __forceinline__ double fsm_probe_random_in_window(uint64_t i, uint64_t salt) {
    const int64_t e = kLoExp + (int64_t)(i % (uint64_t)kBinades);
    return __longlong_as_double((long long)(fsm_probe_pow2_bits(e) | (fsm_probe_mix(i ^ salt) & 0xFFFFFFFFFFFFFull)));
}

/* operand i of class cls: *x for the square root, *b for the reciprocal; returns 0 when the index names no operand */
__device__ int fsm_probe_operand(int cls, uint64_t i, double* x, double* b) {
    const uint64_t lo = fsm_probe_pow2_bits(kLoExp), hi = fsm_probe_pow2_bits(kLoExp + kBinades);   /* window [lo, hi) */
    uint64_t bits;
    switch (cls) {
    case 0: {
        *x = fsm_probe_random_in_window(i, 0x5EEDull);
        const int neg = (int)(fsm_probe_mix(i ^ 0xA5A5ull) >> 63);
        *b = neg ? -*x : *x;
        return 1;
    }
    case 1:
        bits = (i & 1) ? hi - 1 - (i >> 1) : lo + (i >> 1);
        break;
    case 2: {
        const int64_t e = kLoExp + (int64_t)(i / 64);
        const int64_t j = (int64_t)(i % 64);
        bits = j < 32 ? fsm_probe_pow2_bits(e) + (uint64_t)(j - 16) : fsm_probe_pow2_bits(e + 1) - 1 + (uint64_t)(j - 48);
        if (bits < lo || bits >= hi) return 0;
        break;
    }
    case 3:
        bits = fsm_probe_pow2_bits((int64_t)(i % 64)) | (fsm_probe_mix(i ^ 0xDE4ull) & 0xFFFFFFFFFFFFFull);
        break;
    default: {
        const double det = fsm_probe_random_in_window(i, 0xDE7ull);
        *x = det;
        *b = 2.0 * PFC_PI * __dsqrt_rn(det);
        return 1;
    }
    }
    *x = *b = __longlong_as_double((long long)bits);
    return 1;
}

__global__ void fsm_probe_kernel(int cls, uint64_t n, unsigned long long* out) {
    unsigned long long cnt = 0, brcp = 0, bsqrt = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        double x, b;
        if (!fsm_probe_operand(cls, i, &x, &b)) continue;
        ++cnt;
        const bool r_bad = __double_as_longlong(fsm_rcp(b)) != __double_as_longlong(__drcp_rn(b));
        const bool s_bad = __double_as_longlong(fsm_sqrt(x)) != __double_as_longlong(__dsqrt_rn(x));
        brcp += r_bad;
        bsqrt += s_bad;
        if (r_bad || s_bad) atomicCAS(out + 3, 0ull, (unsigned long long)__double_as_longlong(r_bad ? b : x));
    }
    atomicAdd(out + 0, cnt);
    atomicAdd(out + 1, brcp);
    atomicAdd(out + 2, bsqrt);
}

/* operands of each class for log2_random = log2(size of class 0) */
static uint64_t fsm_probe_count(int cls, unsigned log2_random) {
    switch (cls) {
    case 0: return 1ull << log2_random;
    case 1: return 2ull << 15;
    case 2: return (uint64_t)kBinades * 64;
    case 3: return 1ull << 22;
    default: return 1ull << 24;
    }
}

/* out[FSM_PROBE_CLASSES][FSM_PROBE_FIELDS]; returns the CUDA error code (0 = success) */
extern "C" int fsm_probe_run(int device, unsigned log2_random, unsigned long long* out) {
    cudaError_t e = cudaSetDevice(device);
    if (e != cudaSuccess) return (int)e;
    const size_t bytes = sizeof(unsigned long long) * FSM_PROBE_CLASSES * FSM_PROBE_FIELDS;
    unsigned long long* d_out = nullptr;
    if ((e = cudaMalloc(&d_out, bytes)) != cudaSuccess) return (int)e;
    if ((e = cudaMemset(d_out, 0, bytes)) == cudaSuccess) {
        for (int c = 0; c < FSM_PROBE_CLASSES; ++c)
            fsm_probe_kernel<<<132 * 16, 256>>>(c, fsm_probe_count(c, log2_random), d_out + c * FSM_PROBE_FIELDS);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpy(out, d_out, bytes, cudaMemcpyDeviceToHost);
    }
    cudaFree(d_out);
    return (int)e;
}
