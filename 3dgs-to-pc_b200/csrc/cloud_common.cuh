// cloud_common.cuh — device code the point-cloud stages share (s8_cull.cu, s9_clean.cu, s10_mesh.cu): the bounding box
// of the finite points and the two steps of the fixed-order float64 sums that make their re-runs bit-identical.  Every
// kernel stays in an anonymous namespace, like the rest of the library's.
#pragma once
#include "common.cuh"

namespace {

constexpr int BBOX_THREADS = 256;
constexpr int BBOX_PER_CTA = BBOX_THREADS * 8;

__device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

inline int bbox_blocks(int64_t n) { return (int)((n + BBOX_PER_CTA - 1) / BBOX_PER_CTA); }

// per-CTA min / max of the finite coordinates: part[6 * b ..] = (min x, min y, min z, max x, max y, max z), over
// bbox_blocks(n) CTAs of BBOX_THREADS threads.  A template only so that s8_cull.cu, which includes this header but does
// not launch the kernel, does not compile it.
template <int NT = BBOX_THREADS>
__global__ void __launch_bounds__(NT) bbox_kernel(const float* __restrict__ xyz, int64_t n, float* __restrict__ part) {
    __shared__ float s[6][NT / 32];
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    const int64_t base = (int64_t)blockIdx.x * BBOX_PER_CTA;
    for (int r = 0; r < BBOX_PER_CTA / NT; ++r) {
        const int64_t i = base + r * NT + threadIdx.x;
        if (i >= n) break;
        const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
        if (!finite3(x, y, z)) continue;
        mn[0] = fminf(mn[0], x); mn[1] = fminf(mn[1], y); mn[2] = fminf(mn[2], z);
        mx[0] = fmaxf(mx[0], x); mx[1] = fmaxf(mx[1], y); mx[2] = fmaxf(mx[2], z);
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
    }
    if ((threadIdx.x & 31) == 0)
        for (int a = 0; a < 3; ++a) { s[a][threadIdx.x >> 5] = mn[a]; s[3 + a][threadIdx.x >> 5] = mx[a]; }
    __syncthreads();
    if (threadIdx.x < 6) {
        float v = s[threadIdx.x][0];
        for (int w = 1; w < NT / 32; ++w)
            v = threadIdx.x < 3 ? fminf(v, s[threadIdx.x][w]) : fmaxf(v, s[threadIdx.x][w]);
        part[6 * blockIdx.x + threadIdx.x] = v;
    }
}

// one thread: fold the nb per-CTA boxes of bbox_kernel; mn[0] > mx[0] when no point is finite
__device__ __forceinline__ void fold_bbox(const float* __restrict__ part, int nb, float (&mn)[3], float (&mx)[3]) {
    for (int a = 0; a < 3; ++a) { mn[a] = INFINITY; mx[a] = -INFINITY; }
    for (int b = 0; b < nb; ++b)
        for (int a = 0; a < 3; ++a) { mn[a] = fminf(mn[a], part[6 * b + a]); mx[a] = fmaxf(mx[a], part[6 * b + 3 + a]); }
}

// Step 1 of a fixed-order float64 sum, over one CTA of NT threads: an xor tree in each warp, then thread 0 adds the warp
// totals in warp order, starting from +0.0.  s_w: NT / 32 doubles of shared memory.  The sum is valid in thread 0.
template <int NT>
__device__ __forceinline__ double block_sum_f64(double v, double* s_w) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < NT / 32; ++w) t = __dadd_rn(t, s_w[w]);
    return t;
}

// Step 2, one CTA of 1024 threads over the nb per-CTA partials: thread t adds partial[t], partial[t + 1024], ... starting
// from +0.0, then a 512 -> 1 shared-memory tree.  s: 1024 doubles of shared memory.  The sum is valid in thread 0.
__device__ __forceinline__ double sum_partials_f64(const double* __restrict__ partial, int nb, double* s) {
    double t = 0.0;
    for (int i = threadIdx.x; i < nb; i += 1024) t = __dadd_rn(t, partial[i]);
    s[threadIdx.x] = t;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if (threadIdx.x < o) s[threadIdx.x] = __dadd_rn(s[threadIdx.x], s[threadIdx.x + o]);
        __syncthreads();
    }
    return s[0];
}

}  // namespace
