// s1_cov.cu — S1: covariance build, normals, magnitudes (one thread per Gaussian, smem-transposed stores).
//
// Reference semantics restated (not copied):
//   gauss_handler.py:26-63   build_rotation / build_scaling_rotation / build_covariance_from_scaling_rotation
//   gauss_handler.py:89-106  Gaussians.calculate_normals
//   gauss_handler.py:108-112,259 torch.linalg.eigvals(covariances).real  (symmetric 3x3 -> closed form)
#include "common.cuh"

namespace {

template <typename T>
__device__ __forceinline__ T t_exp(T x);
template <>
__device__ __forceinline__ float t_exp<float>(float x) { return expf(x); }
template <>
__device__ __forceinline__ double t_exp<double>(double x) { return exp(x); }

// R(q) with q = (r, x, y, z), NOT normalised (gauss_handler.py:26-47); elements formed in T, rounded to f32.
template <typename T>
__device__ __forceinline__ void rotation_f32(const T* __restrict__ q, float R[9]) {
    const T r = q[0], x = q[1], y = q[2], z = q[3];
    R[0] = (float)(T(1) - T(2) * (y * y + z * z));
    R[1] = (float)(T(2) * (x * y - r * z));
    R[2] = (float)(T(2) * (x * z + r * y));
    R[3] = (float)(T(2) * (x * y + r * z));
    R[4] = (float)(T(1) - T(2) * (x * x + z * z));
    R[5] = (float)(T(2) * (y * z - r * x));
    R[6] = (float)(T(2) * (x * z - r * y));
    R[7] = (float)(T(2) * (y * z + r * x));
    R[8] = (float)(T(1) - T(2) * (x * x + y * y));
}

template <typename T>
__global__ void __launch_bounds__(256) cov_build_kernel(const T* __restrict__ scales, const T* __restrict__ rots,
                                                        float mod, int64_t n, float* __restrict__ cov) {
    __shared__ float tile[256 * 9];
    const int64_t base = (int64_t)blockIdx.x * 256;
    const int64_t i = base + threadIdx.x;
    if (i < n) {
        T q[4];
        if constexpr (sizeof(T) == 4) {
            float4 v = *reinterpret_cast<const float4*>(rots + 4 * i);
            q[0] = v.x; q[1] = v.y; q[2] = v.z; q[3] = v.w;
        } else {
            double2 a = *reinterpret_cast<const double2*>(rots + 4 * i);
            double2 b = *reinterpret_cast<const double2*>(rots + 4 * i + 2);
            q[0] = a.x; q[1] = a.y; q[2] = b.x; q[3] = b.y;
        }
        float R[9];
        rotation_f32<T>(q, R);
        // exp(mod * s) in T, rounded to f32 on assignment (gauss_handler.py:53-55, :61)
        const float e0 = (float)t_exp<T>((T)mod * scales[3 * i + 0]);
        const float e1 = (float)t_exp<T>((T)mod * scales[3 * i + 1]);
        const float e2 = (float)t_exp<T>((T)mod * scales[3 * i + 2]);
        // L = R * diag(e)  (f32 bmm with a diagonal right factor is exact per element)
        float L[9];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            L[3 * r + 0] = R[3 * r + 0] * e0;
            L[3 * r + 1] = R[3 * r + 1] * e1;
            L[3 * r + 2] = R[3 * r + 2] * e2;
        }
        // Sigma = L * L^T (f32)
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c)
                tile[threadIdx.x * 9 + 3 * r + c] =
                    fmaf(L[3 * r + 2], L[3 * c + 2], fmaf(L[3 * r + 1], L[3 * c + 1], L[3 * r + 0] * L[3 * c + 0]));
    }
    __syncthreads();
    const int64_t rem = n - base;
    const int cnt = (int)(rem < 256 ? rem : 256) * 9;
    float* out = cov + base * 9;
    if (cnt == 256 * 9) {  // full tile: 16-byte stores (base*9*4 B is a multiple of 16)
        const float4* s4 = reinterpret_cast<const float4*>(tile);
        float4* o4 = reinterpret_cast<float4*>(out);
        for (int k = threadIdx.x; k < 256 * 9 / 4; k += 256) o4[k] = s4[k];
    } else {
        for (int k = threadIdx.x; k < cnt; k += 256) out[k] = tile[k];
    }
}

template <typename T>
__global__ void __launch_bounds__(256) normals_kernel(const T* __restrict__ scales, const T* __restrict__ rots,
                                                      int64_t n, float* __restrict__ normals) {
    __shared__ float tile[256 * 3];
    const int64_t base = (int64_t)blockIdx.x * 256;
    const int64_t i = base + threadIdx.x;
    if (i < n) {
        T q[4] = {rots[4 * i], rots[4 * i + 1], rots[4 * i + 2], rots[4 * i + 3]};
        float R[9];
        rotation_f32<T>(q, R);
        const T s0 = scales[3 * i], s1 = scales[3 * i + 1], s2 = scales[3 * i + 2];
        int a = 0;  // first minimum wins (torch.min index on ties: first occurrence)
        T m = s0;
        if (s1 < m) { m = s1; a = 1; }
        if (s2 < m) { m = s2; a = 2; }
        tile[threadIdx.x * 3 + 0] = R[0 + a];
        tile[threadIdx.x * 3 + 1] = R[3 + a];
        tile[threadIdx.x * 3 + 2] = R[6 + a];
    }
    __syncthreads();
    const int64_t rem = n - base;
    const int cnt = (int)(rem < 256 ? rem : 256) * 3;
    float* out = normals + base * 3;
    for (int k = threadIdx.x; k < cnt; k += 256) out[k] = tile[k];
}

// eigenvalues of a symmetric 3x3 (trigonometric closed form) in f64.
__global__ void __launch_bounds__(256) eigvals_sym3_kernel(const float* __restrict__ cov, int64_t n,
                                                           float* __restrict__ eig) {
    __shared__ float tile[256 * 9];
    const int64_t base = (int64_t)blockIdx.x * 256;
    const int64_t rem = n - base;
    const int cnt = (int)(rem < 256 ? rem : 256);
    for (int k = threadIdx.x; k < cnt * 9; k += 256) tile[k] = cov[base * 9 + k];
    __syncthreads();
    if (threadIdx.x >= cnt) return;
    double lo, mid, hi;
    g2pc_eig3_sym(tile + threadIdx.x * 9, lo, mid, hi);
    // ascending order, rounded to f32 (the reference's eigvals are f32: gauss_handler.py:112,259)
    float* o = eig + (base + threadIdx.x) * 3;
    o[0] = (float)lo; o[1] = (float)mid; o[2] = (float)hi;
}

}  // namespace

extern "C" int g2pc_cov_build(const void* scales, const void* rots, int in_dtype, float scale_modifier,
                              int64_t n, float* cov, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(in_dtype == G2PC_F32 || in_dtype == G2PC_F64, "in_dtype must be G2PC_F32 or G2PC_F64");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(scales && rots && cov, "null pointer");
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (in_dtype == G2PC_F32)
        cov_build_kernel<float><<<grid, 256, 0, st>>>((const float*)scales, (const float*)rots, scale_modifier, n, cov);
    else
        cov_build_kernel<double><<<grid, 256, 0, st>>>((const double*)scales, (const double*)rots, scale_modifier, n, cov);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_normals(const void* scales, const void* rots, int in_dtype, int64_t n, float* normals,
                            void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(in_dtype == G2PC_F32 || in_dtype == G2PC_F64, "in_dtype must be G2PC_F32 or G2PC_F64");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(scales && rots && normals, "null pointer");
    const unsigned grid = (unsigned)((n + 255) / 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (in_dtype == G2PC_F32)
        normals_kernel<float><<<grid, 256, 0, st>>>((const float*)scales, (const float*)rots, n, normals);
    else
        normals_kernel<double><<<grid, 256, 0, st>>>((const double*)scales, (const double*)rots, n, normals);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_eigvals_sym3(const float* cov, int64_t n, float* eigvals, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(cov && eigvals, "null pointer");
    const unsigned grid = (unsigned)((n + 255) / 256);
    eigvals_sym3_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(cov, n, eigvals);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
