// common.cuh — shared device helpers for libg2pc (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/g2pc.h"

// ---- error plumbing (no exceptions across the C ABI) ------------------------------------------------
void g2pc_set_error(const char* fmt, ...);

#define G2PC_CHECK_ARG(cond, msg)                                  \
    do {                                                           \
        if (!(cond)) {                                             \
            g2pc_set_error("%s: %s", __func__, msg);               \
            return G2PC_ERR_INVALID;                               \
        }                                                          \
    } while (0)

// caller-provided workspace: at least `need` bytes, base aligned to `align` (a power of two)
#define G2PC_CHECK_WORKSPACE(ptr, bytes, need, align)                                        \
    do {                                                                                     \
        if ((int64_t)(bytes) < (int64_t)(need)) {                                            \
            g2pc_set_error("%s: workspace too small", __func__);                             \
            return G2PC_ERR_WORKSPACE;                                                       \
        }                                                                                    \
        if (((uintptr_t)(ptr) & ((uintptr_t)(align) - 1)) != 0) {                            \
            g2pc_set_error("%s: workspace must be %d-byte aligned", __func__, (int)(align)); \
            return G2PC_ERR_WORKSPACE;                                                       \
        }                                                                                    \
    } while (0)

// Typed slices of a workspace, each padded to a multiple of 256 bytes, so each starts 256-byte aligned relative to the
// base.  A null base only adds up the size, so one layout function serves both the size query and the entry point.
struct WsCarve {
    char* base;
    size_t used = 0;
    static size_t pad(size_t bytes) { return (bytes + 255) & ~(size_t)255; }
    template <class T>
    T* take(size_t count) {
        T* p = base ? (T*)(base + used) : nullptr;
        used += pad(count * sizeof(T));
        return p;
    }
};

#define G2PC_CHECK_LAUNCH()                                                        \
    do {                                                                           \
        cudaError_t e__ = cudaGetLastError();                                      \
        if (e__ != cudaSuccess) {                                                  \
            g2pc_set_error("%s: CUDA error: %s", __func__, cudaGetErrorString(e__)); \
            return G2PC_ERR_CUDA;                                                  \
        }                                                                          \
    } while (0)

#define G2PC_CUDA(call)                                                            \
    do {                                                                           \
        cudaError_t e__ = (call);                                                  \
        if (e__ != cudaSuccess) {                                                  \
            g2pc_set_error("%s: CUDA error: %s", __func__, cudaGetErrorString(e__)); \
            return G2PC_ERR_CUDA;                                                  \
        }                                                                          \
    } while (0)

// ---- Philox4x32-10 counter-based RNG -----------------------------------------------------------------
// Stream definition (sharding-invariant, regenerable in pass 2):
//   key = (seed_lo, seed_hi), counter = (global Gaussian id, sample index, attempt, call id)
// The same function is restated in oracle/philox.py.
struct Philox4 {
    uint32_t x, y, z, w;
};

__host__ __device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                          uint32_t k0, uint32_t k1) {
    const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)M0 * c0;
        uint64_t p1 = (uint64_t)M1 * c2;
        uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0;
        uint32_t hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
        uint32_t n0 = hi1 ^ c1 ^ k0;
        uint32_t n2 = hi0 ^ c3 ^ k1;
        c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
        k0 += W0; k1 += W1;
    }
    Philox4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
    return o;
}

// u32 -> uniform in (0,1): ((x >> 9) + 0.5) * 2^-23.  x >> 9 < 2^23, so the +0.5 is exact in fp32 and the result lies
// in [2^-24, 1 - 2^-24]: never 0, never 1.
__device__ __forceinline__ float u32_to_unit(uint32_t x) {
    return ((float)(x >> 9) + 0.5f) * 1.1920928955078125e-07f;
}

__device__ __forceinline__ float fast_sqrt(float x) {
    float r;
    asm("sqrt.approx.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// three standard normals for (gid, sample, attempt, call): two Box-Muller pairs, the 4th value unused
__device__ __forceinline__ float3 draw_eps(uint32_t gid, uint32_t sample, uint32_t attempt, uint32_t call,
                                           uint32_t k0, uint32_t k1) {
    Philox4 r = philox4x32_10(gid, sample, attempt, call, k0, k1);
    const float TWO_PI = 6.283185307179586f;
    float u1 = u32_to_unit(r.x), u2 = u32_to_unit(r.y), u3 = u32_to_unit(r.z), u4 = u32_to_unit(r.w);
    // the approximate log of u just below 1 may come out slightly positive: clamp before the square root
    float ra = fast_sqrt(fmaxf(0.0f, -2.0f * __logf(u1)));
    float rb = fast_sqrt(fmaxf(0.0f, -2.0f * __logf(u3)));
    float sa, ca, cb;
    __sincosf(TWO_PI * u2, &sa, &ca);
    cb = __cosf(TWO_PI * u4);
    return make_float3(ra * ca, ra * sa, rb * cb);
}

// Eigenvalues of a symmetric 3x3 (row-major f32, off-diagonal pairs averaged like a general solver sees them),
// trigonometric closed form in f64, returned ASCENDING.  Used by g2pc_eigvals_sym3 (s1_cov.cu) and the magnitudes
// kernel (s8_cull.cu).  A diagonal matrix (p1 == 0: identity / axis-aligned quaternions) takes the diagonal as is, and
// l1 = 3q - l0 - l2 may round past a nearly equal neighbour, so the three values are sorted before they are returned.
__device__ __forceinline__ void g2pc_eig3_sym(const float* S, double& lo, double& mid, double& hi) {
    const double a00 = S[0], a11 = S[4], a22 = S[8];
    const double a01 = 0.5 * ((double)S[1] + (double)S[3]);
    const double a02 = 0.5 * ((double)S[2] + (double)S[6]);
    const double a12 = 0.5 * ((double)S[5] + (double)S[7]);
    const double p1 = a01 * a01 + a02 * a02 + a12 * a12;
    const double q = (a00 + a11 + a22) / 3.0;
    double l0, l1, l2;
    if (p1 == 0.0) {
        l0 = a00; l1 = a11; l2 = a22;
    } else {
        const double d0 = a00 - q, d1 = a11 - q, d2 = a22 - q;
        const double p2 = d0 * d0 + d1 * d1 + d2 * d2 + 2.0 * p1;
        const double p = sqrt(p2 / 6.0);
        const double ip = 1.0 / p;
        const double b00 = d0 * ip, b11 = d1 * ip, b22 = d2 * ip;
        const double b01 = a01 * ip, b02 = a02 * ip, b12 = a12 * ip;
        double r = 0.5 * (b00 * (b11 * b22 - b12 * b12) - b01 * (b01 * b22 - b12 * b02) +
                          b02 * (b01 * b12 - b11 * b02));
        r = r < -1.0 ? -1.0 : (r > 1.0 ? 1.0 : r);
        const double phi = acos(r) / 3.0;
        l0 = q + 2.0 * p * cos(phi);
        l2 = q + 2.0 * p * cos(phi + 2.0943951023931953);
        l1 = 3.0 * q - l0 - l2;
    }
    // three-element sorting network
    double t;
    if (l0 > l1) { t = l0; l0 = l1; l1 = t; }
    if (l1 > l2) { t = l1; l1 = l2; l2 = t; }
    if (l0 > l1) { t = l0; l0 = l1; l1 = t; }
    lo = l0; mid = l1; hi = l2;
}

// Block-wide exclusive scan for 1024 threads: returns the thread's prefix and sets `total` to the block's sum.  s_warp is
// 33 ints of shared memory; every thread must call.
__device__ __forceinline__ int block_scan_1024(int v, int* s_warp, int& total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        int w = s_warp[lane];
        int winc = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, winc, o);
            if (lane >= o) winc += t;
        }
        s_warp[lane] = winc - w;            // exclusive prefix of warp totals
        if (lane == 31) s_warp[32] = winc;  // grand total
    }
    __syncthreads();
    const int res = s_warp[warp] + inc - v;
    total = s_warp[32];
    __syncthreads();
    return res;
}

// x = mu + L*eps with L lower-triangular (l00,l10,l11,l20,l21,l22); the SAME expression is used by the
// count pass (explicit Mahalanobis) and the emit pass, so both see bit-identical positions.
__device__ __forceinline__ float3 mvn_point(const float3 mu, float l00, float l10, float l11, float l20,
                                            float l21, float l22, const float3 e) {
    float dx = l00 * e.x;
    float dy = fmaf(l11, e.y, l10 * e.x);
    float dz = fmaf(l22, e.z, fmaf(l21, e.y, l20 * e.x));
    return make_float3(mu.x + dx, mu.y + dy, mu.z + dz);
}
