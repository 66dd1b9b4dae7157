// common.cuh — launch bookkeeping, error handling and block-level primitives shared by all kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "../../include/pfgpu.h"
#include "../../include/pf_contract_math.h"

#ifndef PFGPU_NUM_SMS
#define PFGPU_NUM_SMS 132          // H100 SXM; ctx_open reads the device's own count
#endif

extern thread_local char g_pfgpu_err[512];

#define PF_CUDA(call)                                                                                   \
    do {                                                                                                \
        cudaError_t e__ = (call);                                                                       \
        if (e__ != cudaSuccess) {                                                                       \
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s:%d: %s -> %s", __FILE__, __LINE__, #call,    \
                     cudaGetErrorString(e__));                                                          \
            return PFGPU_ERR_CUDA;                                                                      \
        }                                                                                               \
    } while (0)

// One per handle: device, stream, counters.
struct Ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    uint64_t launches = 0;
    int num_sms = PFGPU_NUM_SMS;
};

#define PF_LAUNCH(ctx, kernel, grid, block, smem, ...)                                                  \
    do {                                                                                                \
        kernel<<<(grid), (block), (smem), (ctx).stream>>>(__VA_ARGS__);                                 \
        (ctx).launches++;                                                                               \
        cudaError_t e__ = cudaGetLastError();                                                           \
        if (e__ != cudaSuccess) {                                                                       \
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s:%d: launch %s -> %s", __FILE__, __LINE__,    \
                     #kernel, cudaGetErrorString(e__));                                                 \
            return PFGPU_ERR_CUDA;                                                                      \
        }                                                                                               \
    } while (0)

// Programmatic dependent launch (sm_90+): the launch may be set up while the previous kernel of the stream still runs; the
// kernel itself waits (pf_grid_dep_sync, its FIRST statement) until that kernel has completed and its writes are visible.
// Takes the scheduling latency between the dependent kernels of a step off the timeline; everything else is unchanged.
#define PF_LAUNCH_PDL(ctx, pdl, kernel, grid, block, smem, ...)                                          \
    do {                                                                                                \
        cudaLaunchConfig_t c__ = {};                                                                    \
        c__.gridDim = dim3(grid); c__.blockDim = dim3(block); c__.dynamicSmemBytes = (smem); c__.stream = (ctx).stream; \
        cudaLaunchAttribute a__[1];                                                                     \
        a__[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;                                 \
        a__[0].val.programmaticStreamSerializationAllowed = 1;                                          \
        c__.attrs = a__; c__.numAttrs = (pdl) ? 1 : 0;                                                  \
        cudaError_t e__ = cudaLaunchKernelEx(&c__, kernel, __VA_ARGS__);                                \
        (ctx).launches++;                                                                               \
        if (e__ != cudaSuccess) {                                                                       \
            snprintf(g_pfgpu_err, sizeof(g_pfgpu_err), "%s:%d: launch %s -> %s", __FILE__, __LINE__,    \
                     #kernel, cudaGetErrorString(e__));                                                 \
            return PFGPU_ERR_CUDA;                                                                      \
        }                                                                                               \
    } while (0)
#ifdef __CUDACC__
__device__ __forceinline__ void pf_grid_dep_sync() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// Let the NEXT kernel of the stream (if it was launched with the attribute above) be scheduled now: its CTAs take the SMs this
// grid's CTAs leave as they retire and park in their own griddepcontrol.wait until this grid has completed and flushed.  Issued
// by every CTA at its start, i.e. once the whole (one-CTA-per-SM) grid is resident, so the early CTAs cannot crowd out ours.
__device__ __forceinline__ void pf_grid_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

static inline unsigned int cdiv_u(size_t a, size_t b) { return (unsigned int)((a + b - 1) / b); }

// ---------------------------------------------------------------------------------------------------
// block-level sum (tree order; used only for tolerance-level quantities and approximate prefixes)
// ---------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// sum over the block; result valid in thread 0 (and broadcast through smem[0] after the final sync)
template <int NT>
__device__ __forceinline__ double block_sum(double v, double* smem /* >= NT/32 */) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) smem[wid] = v;
    __syncthreads();
    double t = 0.0;
    if (wid == 0) {
        t = lane < NT / 32 ? smem[lane] : 0.0;
        t = warp_sum(t);
    }
    return t;
}

// exclusive prefix sum of one double per thread, in thread order; *total = block total
template <int NT>
__device__ __forceinline__ double block_excl_scan(double x, double* total, double* smem /* >= NT/32 */) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    double inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        double y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc = y + inc;
    }
    double excl = __shfl_up_sync(0xffffffffu, inc, 1);
    if (lane == 0) excl = 0.0;
    __syncthreads();
    if (lane == 31) smem[wid] = inc;
    __syncthreads();
    double woff = 0.0, tot = 0.0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) {
        double t = smem[w];
        if (w < wid) woff += t;
        tot += t;
    }
    *total = tot;
    return woff + excl;
}

template <int NT>
__device__ __forceinline__ int block_excl_scan_int(int x, int* total, int* smem /* >= NT/32 */) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    int excl = inc - x;
    __syncthreads();
    if (lane == 31) smem[wid] = inc;
    __syncthreads();
    int woff = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; ++w) {
        int t = smem[w];
        if (w < wid) woff += t;
        tot += t;
    }
    *total = tot;
    return woff + excl;
}
