// fs3_est.cuh — the FastSLAM estimate (pfgpu_fs_moments): weighted moments of the pose cloud and, per landmark, of the copies
// that pass `cov00 < cov00_max` (DESIGN §3.4).  Not part of the step: ordinary launches on the engine's stream, between one
// step's post kernel and the next step's EKF launch, reading the live buffers the way pfgpu_fs_download does.
//
//   fs3_est_pose_kernel   one pass over (w, px, py, pyaw) of the local slots: deviations from a centre every rank reads from the
//                         current state, per-thread moments about the thread's own shift, pairwise (Chan) merges in a block tree,
//                         then the last CTA to finish merges the block partials in a fixed tree
//   fs3_est_map_kernel    grid = particle chunks x groups of 8 landmarks, one warp per (chunk, landmark): every (landmark, slot)
//                         copy is read once through fs3_lm_src (own columns, or the ancestry row, maybe on a peer rank); each lane
//                         accumulates about its own shift, the warp merges its lanes (Chan) and writes one partial per chunk
//   fs3_est_merge_kernel  one warp per landmark: merges the chunk partials in chunk order
// Every reduction order depends on (n, m, world) only, so two calls on the same state return the same bits.
#pragma once
#include "fs3.cuh"
#include <cmath>
#include <limits>

#define FS3_EST_NT 256
#define FS3_EST_POSE_MAX_BLOCKS 256
#define FS3_EST_POSE_SUMS 10               // Fs3PoseMom: w, mean (3), m2 (6)
#define FS3_EST_TARGET_WARPS 16384         // (chunk, landmark) warps the map pass aims for
#define FS3_EST_SCRATCH_CAP ((size_t)64 << 20)   // chunk partials: fewer chunks when m is large

// weighted moments of a set of landmark copies: total weight, weighted mean of (x, y), and
// m2 = sum w (P + (mu - mean)(mu - mean)^T) in lm6 order (c00, c01, c10, c11); the layout of pfgpu_fs_lm_moments
struct Fs3LmMom { double w, mx, my, m00, m01, m10, m11; };

// pairwise (Chan) update a <- a (+) b; an empty side (w == 0) leaves the other unchanged.  Host and device use this one
// formula (both compiled without contraction), so the host's rank merge adds like the device's chunk merge.
__host__ __device__ __forceinline__ void fs3_mom_merge(Fs3LmMom& a, const Fs3LmMom& b) {
    if (b.w == 0.0) return;
    if (a.w == 0.0) { a = b; return; }
    const double w = a.w + b.w, f = b.w / w, g = a.w * f, dx = b.mx - a.mx, dy = b.my - a.my;
    a.mx = a.mx + dx * f; a.my = a.my + dy * f;
    const double cxy = dx * dy * g;
    a.m00 = a.m00 + b.m00 + dx * dx * g; a.m01 = a.m01 + b.m01 + cxy; a.m10 = a.m10 + b.m10 + cxy; a.m11 = a.m11 + b.m11 + dy * dy * g;
    a.w = w;
}

// weighted moments of pose deviations d = (x - cx, y - cy, wrap(yaw - cyaw)) from the centre: total weight, weighted mean of d,
// m2 = sum w (d - mean)(d - mean)^T as (xx, xy, xyaw, yy, yyaw, yawyaw); the layout of pfgpu_fs_pose_moments after w and c
struct Fs3PoseMom { double w, m[3], q[6]; };
__host__ __device__ __forceinline__ void fs3_pose_merge(Fs3PoseMom& a, const Fs3PoseMom& b) {
    if (b.w == 0.0) return;
    if (a.w == 0.0) { a = b; return; }
    const double w = a.w + b.w, f = b.w / w, g = a.w * f;
    const double d0 = b.m[0] - a.m[0], d1 = b.m[1] - a.m[1], d2 = b.m[2] - a.m[2];
    a.m[0] = a.m[0] + d0 * f; a.m[1] = a.m[1] + d1 * f; a.m[2] = a.m[2] + d2 * f;
    a.q[0] = a.q[0] + b.q[0] + d0 * d0 * g; a.q[1] = a.q[1] + b.q[1] + d0 * d1 * g; a.q[2] = a.q[2] + b.q[2] + d0 * d2 * g;
    a.q[3] = a.q[3] + b.q[3] + d1 * d1 * g; a.q[4] = a.q[4] + b.q[4] + d1 * d2 * g; a.q[5] = a.q[5] + b.q[5] + d2 * d2 * g;
    a.w = w;
}

// yaw difference wrapped to [-pi, pi] (IEEE remainder by 2 pi; the common case |d| <= pi costs one compare)
__host__ __device__ __forceinline__ double fs3_wrap_angle(double d) {
    const double PI = 3.141592653589793;
    return fabs(d) <= PI ? d : remainder(d, 2.0 * PI);
}

#ifdef __CUDACC__
__device__ __forceinline__ Fs3LmMom fs3_mom_shfl_down(const Fs3LmMom& v, int o) {
    Fs3LmMom r;
    r.w = __shfl_down_sync(0xffffffffu, v.w, o); r.mx = __shfl_down_sync(0xffffffffu, v.mx, o); r.my = __shfl_down_sync(0xffffffffu, v.my, o);
    r.m00 = __shfl_down_sync(0xffffffffu, v.m00, o); r.m01 = __shfl_down_sync(0xffffffffu, v.m01, o);
    r.m10 = __shfl_down_sync(0xffffffffu, v.m10, o); r.m11 = __shfl_down_sync(0xffffffffu, v.m11, o);
    return r;
}
// lane 0 receives lanes 0..31 merged in a fixed tree
__device__ __forceinline__ void fs3_mom_warp_merge(Fs3LmMom& v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const Fs3LmMom u = fs3_mom_shfl_down(v, o); fs3_mom_merge(v, u); }
}

// thread 0 receives the block's Fs3PoseMom values merged in a fixed tree (lanes by shuffle, then the warps in order)
__device__ __forceinline__ void fs3_pose_block_merge(Fs3PoseMom& v, Fs3PoseMom* sm /* [FS3_EST_NT / 32] */) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Fs3PoseMom u;
        u.w = __shfl_down_sync(0xffffffffu, v.w, o);
#pragma unroll
        for (int k = 0; k < 3; ++k) u.m[k] = __shfl_down_sync(0xffffffffu, v.m[k], o);
#pragma unroll
        for (int k = 0; k < 6; ++k) u.q[k] = __shfl_down_sync(0xffffffffu, v.q[k], o);
        fs3_pose_merge(v, u);
    }
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < FS3_EST_NT / 32; ++w) fs3_pose_merge(v, sm[w]);
}

// centre c = the current pose of the last slot of the last rank (read through the peer mapping when sharded), so every rank
// uses the same bits and c is always a member of the cloud.  part: [gridDim.x] Fs3PoseMom; out: pfgpu_fs_pose_moments
// (w, c[3], mean[3], m2[6]); *ticket is 0 between launches.
__global__ void __launch_bounds__(FS3_EST_NT) fs3_est_pose_kernel(const __grid_constant__ Fs3Dev d, Fs3PoseMom* part, unsigned* ticket, double* out) {
    __shared__ Fs3PoseMom sm[FS3_EST_NT / 32];
    __shared__ bool last;
    const int cur = d.st->cur;
    const char* cbase = d.G > 1 ? d.peer[d.G - 1] : d.peer[d.rank];
    const size_t jc = (size_t)d.n - 1;
    const double cx = reinterpret_cast<const double*>(cbase + d.o_px[cur])[jc];
    const double cy = reinterpret_cast<const double*>(cbase + d.o_py[cur])[jc];
    const double cyaw = reinterpret_cast<const double*>(cbase + d.o_pyaw[cur])[jc];
    // per thread: sums about the thread's first deviation k (no cancellation however far the cloud lies from c)
    bool have = false;
    double k0 = 0.0, k1 = 0.0, k2 = 0.0, sw = 0.0, s0 = 0.0, s1 = 0.0, s2 = 0.0, q[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    const double* px = d.px[cur]; const double* py = d.py[cur]; const double* pa = d.pyaw[cur];
    for (size_t i = (size_t)blockIdx.x * FS3_EST_NT + threadIdx.x; i < d.n; i += (size_t)gridDim.x * FS3_EST_NT) {
        const double w = d.w[i], dx = px[i] - cx, dy = py[i] - cy, dt = fs3_wrap_angle(pa[i] - cyaw);
        if (!have) { k0 = dx; k1 = dy; k2 = dt; have = true; }
        const double e0 = dx - k0, e1 = dy - k1, e2 = dt - k2, w0 = w * e0, w1 = w * e1, w2 = w * e2;
        sw += w; s0 += w0; s1 += w1; s2 += w2;
        q[0] += w0 * e0; q[1] += w0 * e1; q[2] += w0 * e2; q[3] += w1 * e1; q[4] += w1 * e2; q[5] += w2 * e2;
    }
    Fs3PoseMom v = {0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}};
    if (sw != 0.0) {
        const double a0 = s0 / sw, a1 = s1 / sw, a2 = s2 / sw;
        v.w = sw; v.m[0] = k0 + a0; v.m[1] = k1 + a1; v.m[2] = k2 + a2;
        v.q[0] = q[0] - s0 * a0; v.q[1] = q[1] - s0 * a1; v.q[2] = q[2] - s0 * a2;
        v.q[3] = q[3] - s1 * a1; v.q[4] = q[4] - s1 * a2; v.q[5] = q[5] - s2 * a2;
    }
    fs3_pose_block_merge(v, sm);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = v;
        __threadfence();
        last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    // the last CTA: thread t takes block partial t (gridDim.x <= FS3_EST_NT), then the same fixed tree
    Fs3PoseMom b = {0.0, {0.0, 0.0, 0.0}, {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}};
    if (threadIdx.x < gridDim.x) {
        const double* src = reinterpret_cast<const double*>(part + threadIdx.x);
        b.w = __ldcg(src);
#pragma unroll
        for (int k = 0; k < 3; ++k) b.m[k] = __ldcg(src + 1 + k);
#pragma unroll
        for (int k = 0; k < 6; ++k) b.q[k] = __ldcg(src + 4 + k);
    }
    __syncthreads();                                  // (sm is reused)
    fs3_pose_block_merge(b, sm);
    if (threadIdx.x == 0) {
        out[0] = b.w; out[1] = cx; out[2] = cy; out[3] = cyaw;
        for (int k = 0; k < 3; ++k) out[4 + k] = b.m[k];
        for (int k = 0; k < 6; ++k) out[7 + k] = b.q[k];
        *ticket = 0u;
    }
}

// part: [m][gridDim.x] Fs3LmMom; blockIdx.x = chunk of `chunk` local slots, warp w of block y = landmark 8 y + w
__global__ void __launch_bounds__(FS3_EST_NT, 2) fs3_est_map_kernel(const __grid_constant__ Fs3Dev d, double cov00_max, unsigned chunk, Fs3LmMom* part) {
    const unsigned lane = threadIdx.x & 31, l = blockIdx.y * (FS3_EST_NT / 32) + (threadIdx.x >> 5);
    if (l >= d.m) return;
    const unsigned i0 = blockIdx.x * chunk, i1 = min(d.n, i0 + chunk);
    const int s = d.lmst[l], rcur = d.st->rcur;
    const size_t ld = d.ld;
    bool have = false;
    double kx = 0.0, ky = 0.0;
    double sw = 0.0, sx = 0.0, sy = 0.0, sxx = 0.0, sxy = 0.0, syy = 0.0, p00 = 0.0, p01 = 0.0, p10 = 0.0, p11 = 0.0;
    constexpr int B = 4;                          // copies in flight per lane
#pragma unroll 1
    for (unsigned ib = i0 + lane; ib < i1; ib += 32 * B) {
        double w[B], v[B][6];
#pragma unroll
        for (int b = 0; b < B; ++b) {
            const unsigned i = ib + 32u * b;
            if (i < i1) {
                const double* p = fs3_lm_src(d, l, i, s, rcur);
                w[b] = d.w[i];
#pragma unroll
                for (int f = 0; f < 6; ++f) v[b][f] = p[f * ld];
            } else {
                w[b] = 0.0; v[b][2] = cov00_max;  // (fails the test)
            }
        }
#pragma unroll
        for (int b = 0; b < B; ++b) {
            if (!(v[b][2] < cov00_max)) continue;
            if (!have) { kx = v[b][0]; ky = v[b][1]; have = true; }
            const double dx = v[b][0] - kx, dy = v[b][1] - ky, wx = w[b] * dx, wy = w[b] * dy;
            sw += w[b]; sx += wx; sy += wy; sxx += wx * dx; sxy += wx * dy; syy += wy * dy;
            p00 += w[b] * v[b][2]; p01 += w[b] * v[b][3]; p10 += w[b] * v[b][4]; p11 += w[b] * v[b][5];
        }
    }
    Fs3LmMom m = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    if (sw != 0.0) {
        const double ax = sx / sw, ay = sy / sw;
        m.w = sw; m.mx = kx + ax; m.my = ky + ay;
        m.m00 = p00 + (sxx - sx * ax); m.m01 = p01 + (sxy - sx * ay); m.m10 = p10 + (sxy - sx * ay); m.m11 = p11 + (syy - sy * ay);
    }
    fs3_mom_warp_merge(m);
    if (lane == 0) part[(size_t)l * gridDim.x + blockIdx.x] = m;
}

// out[l] = part[l][0] (+) part[l][1] (+) ... : lane j takes chunks j, j + 32, ... in order, then the warp tree
__global__ void __launch_bounds__(FS3_EST_NT) fs3_est_merge_kernel(const Fs3LmMom* part, unsigned nchunks, unsigned m, Fs3LmMom* out) {
    const unsigned lane = threadIdx.x & 31, l = blockIdx.x * (FS3_EST_NT / 32) + (threadIdx.x >> 5);
    if (l >= m) return;
    Fs3LmMom a = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (unsigned c = lane; c < nchunks; c += 32) fs3_mom_merge(a, part[(size_t)l * nchunks + c]);
    fs3_mom_warp_merge(a);
    if (lane == 0) out[l] = a;
}
#endif
