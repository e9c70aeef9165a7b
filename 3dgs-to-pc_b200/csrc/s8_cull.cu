// s8_cull.cu — N4: fused cull + compaction of the per-Gaussian arrays; N1: magnitudes -> points per Gaussian on the device.
//
// Reference semantics restated (not copied):
//   gauss_to_pc.py:483-496        cull masks after the colour stage: surface distance, visibility, min opacity, bounding box
//   gauss_handler.py:168-224      add_gaussians_to_cull / filter_gaussians (9 boolean-index passes, one host sync each),
//                                 apply_min_opacity, apply_bounding_box
//   gauss_handler.py:252-279      get_gaussian_magnitudes: sqrt(ellipsoid area, p = 1.6075) * contribution, float64
//   gauss_to_pc.py:73-90          distribute_points: round(size * P / sum), first min(deficit, #zeros) zero entries -> 1
// Here: ONE kernel evaluates every cull criterion and counts per block, one tiny scan, one kernel writes the ascending
// index list; g2pc_gather_rows compacts any number of row-major arrays through that list (the host reads the count once
// to size the outputs).  The magnitude chain is one kernel + a fixed-order reduction (deterministic sum), the point
// budget three small kernels — no `.item()` on the way (the reference syncs at :87 and inside every boolean index).
#include "cloud_common.cuh"

namespace {

constexpr int CB = 256;          // threads per CTA
constexpr int CPT = 4;           // elements per thread
constexpr int CTILE = CB * CPT;  // elements per CTA

struct CullParams {
    const float* max_contrib; float vis_thr;        // keep max_contrib > vis_thr                 (null: skip)
    const float* opacity; float min_opacity;        // keep opacity > min_opacity                 (null: skip)
    const float* xyz; float bmin[3], bmax[3]; int use_bmin, use_bmax;  // keep bmin < xyz < bmax, open box
    const float* surf; const float* surf_thr;       // keep surf < *surf_thr (device scalar)      (null: skip)
    const uint8_t* extra;                           // keep extra != 0                            (null: skip)
    int64_t lo, hi, n;                              // keep lo <= i < hi (index shard)
};

__device__ __forceinline__ bool cull_keep(const CullParams& p, int64_t i) {
    if (i < p.lo || i >= p.hi) return false;
    if (p.max_contrib && !(p.max_contrib[i] > p.vis_thr)) return false;
    if (p.opacity && !(p.opacity[i] > p.min_opacity)) return false;
    if (p.use_bmin | p.use_bmax) {
        const float x = p.xyz[3 * i], y = p.xyz[3 * i + 1], z = p.xyz[3 * i + 2];
        if (p.use_bmin && !(x > p.bmin[0] && y > p.bmin[1] && z > p.bmin[2])) return false;
        if (p.use_bmax && !(x < p.bmax[0] && y < p.bmax[1] && z < p.bmax[2])) return false;
    }
    if (p.surf && !(p.surf[i] < *p.surf_thr)) return false;
    if (p.extra && !p.extra[i]) return false;
    return true;
}

__device__ __forceinline__ int block_sum_256(int v, int* s_w) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = v;
    __syncthreads();
    int t = 0;
#pragma unroll
    for (int w = 0; w < CB / 32; ++w) t += s_w[w];
    __syncthreads();
    return t;
}

__global__ void __launch_bounds__(CB) cull_count_kernel(const CullParams p, int32_t* __restrict__ block_cnt) {
    __shared__ int s_w[CB / 32];
    const int64_t base = (int64_t)blockIdx.x * CTILE;
    int c = 0;
#pragma unroll
    for (int k = 0; k < CPT; ++k) {
        const int64_t i = base + k * CB + threadIdx.x;
        c += (i < p.n && cull_keep(p, i)) ? 1 : 0;
    }
    const int t = block_sum_256(c, s_w);
    if (threadIdx.x == 0) block_cnt[blockIdx.x] = t;
}

// exclusive scan of the block counts in place (one CTA), total -> count[0]
__global__ void __launch_bounds__(1024) cull_scan_kernel(int32_t* __restrict__ block_cnt, int32_t nblocks,
                                                         int64_t* __restrict__ count) {
    __shared__ int s_w[33];
    long long run = 0;
    for (int b0 = 0; b0 < nblocks; b0 += 1024) {
        const int b = b0 + threadIdx.x;
        int total;
        const int pre = block_scan_1024(b < nblocks ? block_cnt[b] : 0, s_w, total);
        if (b < nblocks) block_cnt[b] = (int32_t)(run + pre);
        run += total;
    }
    if (threadIdx.x == 0) count[0] = run;
}

__global__ void __launch_bounds__(CB) cull_write_kernel(const CullParams p, const int32_t* __restrict__ block_off,
                                                        int32_t* __restrict__ index) {
    __shared__ int s_w[CB / 32];
    const int64_t base = (int64_t)blockIdx.x * CTILE;
    int run = block_off[blockIdx.x];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int k = 0; k < CPT; ++k) {  // ascending order: element (k, thread) precedes (k + 1, *)
        const int64_t i = base + k * CB + threadIdx.x;
        const bool keep = i < p.n && cull_keep(p, i);
        const unsigned m = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) s_w[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
#pragma unroll
        for (int w = 0; w < CB / 32; ++w) { const int c = s_w[w]; before += w < warp ? c : 0; total += c; }
        if (keep) index[run + before + __popc(m & ((1u << lane) - 1u))] = (int32_t)i;
        run += total;
        __syncthreads();
    }
}

// dst[r, :] = src[index[r], :] for rows of `words` 32-bit words
__global__ void __launch_bounds__(256) gather_rows_kernel(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst,
                                                          const int32_t* __restrict__ index, int64_t m, int32_t words) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= m * words) return;
    const int64_t r = t / words;
    const int w = (int)(t - r * words);
    dst[t] = src[(int64_t)index[r] * words + w];
}

// ---- N1 ----------------------------------------------------------------------------------------------------------
// eigenvalues of a symmetric 3x3 (g2pc_eig3_sym, ascending), rounded to f32 like the reference's eigvals
__device__ __forceinline__ void eig3(const float* S, float& e0, float& e1, float& e2) {
    double lo, mid, hi;
    g2pc_eig3_sym(S, lo, mid, hi);
    e0 = (float)lo; e1 = (float)mid; e2 = (float)hi;
}

// magnitude = sqrt(4 pi ((a^p b^p + a^p c^p + b^p c^p) / 3)^(1/p)) * contribution, a,b,c = sqrt(eigenvalues), float32 chain
// then float64 (gauss_handler.py:261-279); per-CTA partial sums in float64 for the deterministic total
__global__ void __launch_bounds__(256) magnitudes_kernel(const float* __restrict__ cov, const float* __restrict__ contrib,
                                                         int64_t n, double* __restrict__ mag, double* __restrict__ partial) {
    __shared__ float tile[256 * 9];
    __shared__ double s_w[8];
    const int64_t base = (int64_t)blockIdx.x * 256;
    const int64_t rem = n - base;
    const int cnt = (int)(rem < 256 ? rem : 256);
    for (int k = threadIdx.x; k < cnt * 9; k += 256) tile[k] = cov[base * 9 + k];
    __syncthreads();
    double m = 0.0;
    if (threadIdx.x < cnt) {
        float e0, e1, e2;
        eig3(tile + threadIdx.x * 9, e0, e1, e2);
        const float p = 1.6075f;
        const float a = sqrtf(e0), b = sqrtf(e1), c = sqrtf(e2);
        const float radicand = (powf(a * b, p) + powf(a * c, p) + powf(b * c, p)) / 3.0f;
        const float area = sqrtf(4.0f * 3.14159265358979323846f * powf(radicand, 1.0f / p));
        m = (double)(area * contrib[base + threadIdx.x]);
        mag[base + threadIdx.x] = m;
    }
    const double t = block_sum_f64<256>(m, s_w);
    if (threadIdx.x == 0) partial[blockIdx.x] = t;
}

// fixed-order sum of the partials (one CTA): sum[0]
__global__ void __launch_bounds__(1024) sum_partials_kernel(const double* __restrict__ partial, int32_t nb,
                                                            double* __restrict__ sum) {
    __shared__ double s[1024];
    const double t = sum_partials_f64(partial, nb, s);
    if (threadIdx.x == 0) sum[0] = t;
}

// ppg = rint(mag * (P / sum)) (torch.round = round half to even); per-CTA (sum of ppg, zero count)
__global__ void __launch_bounds__(256) ppg_round_kernel(const double* __restrict__ mag, const double* __restrict__ sum,
                                                        double num_points, int64_t n, int32_t* __restrict__ ppg,
                                                        long long* __restrict__ blk) {
    __shared__ long long s_a[8];
    __shared__ int s_z[8];
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const double ratio = num_points / sum[0];
    long long v = 0;
    int z = 0;
    if (i < n) {
        const double r = rint(mag[i] * ratio);
        v = (long long)r;
        ppg[i] = (int32_t)v;
        z = (r == 0.0) ? 1 : 0;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { v += __shfl_xor_sync(0xffffffffu, v, o); z += __shfl_xor_sync(0xffffffffu, z, o); }
    if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = v; s_z[threadIdx.x >> 5] = z; }
    __syncthreads();
    if (threadIdx.x == 0) {
        long long a = 0; int zz = 0;
        for (int w = 0; w < 8; ++w) { a += s_a[w]; zz += s_z[w]; }
        blk[2 * blockIdx.x] = a;
        blk[2 * blockIdx.x + 1] = zz;
    }
}

// one CTA: exclusive scan of the zero counts (in place), take = min(deficit, #zeros) with the reference's slice semantics
// for a negative deficit (zeros[:negative] keeps all but the last |deficit|): take_out[0]
__global__ void __launch_bounds__(1024) ppg_plan_kernel(long long* __restrict__ blk, int32_t nb, double num_points,
                                                        long long* __restrict__ take_out) {
    __shared__ long long s_sum[1024];
    __shared__ long long s_zero[1024];
    long long a = 0, z = 0;
    for (int i = threadIdx.x; i < nb; i += 1024) { a += blk[2 * i]; z += blk[2 * i + 1]; }
    s_sum[threadIdx.x] = a; s_zero[threadIdx.x] = z;
    __syncthreads();
    for (int o = 512; o > 0; o >>= 1) {
        if (threadIdx.x < o) { s_sum[threadIdx.x] += s_sum[threadIdx.x + o]; s_zero[threadIdx.x] += s_zero[threadIdx.x + o]; }
        __syncthreads();
    }
    const long long total = s_sum[0], zeros = s_zero[0];
    __syncthreads();
    if (threadIdx.x == 0) {
        long long run = 0;
        for (int i = 0; i < nb; ++i) { const long long c = blk[2 * i + 1]; blk[2 * i + 1] = run; run += c; }
        const double deficit = num_points - (double)total;
        long long take = (long long)(deficit < (double)zeros ? deficit : (double)zeros);  // int(min(deficit, zeros))
        if (take < 0) take = zeros + take;
        take_out[0] = take < 0 ? 0 : take;
    }
}

__global__ void __launch_bounds__(256) ppg_fix_kernel(int32_t* __restrict__ ppg, const long long* __restrict__ blk,
                                                      const long long* __restrict__ take, int64_t n) {
    __shared__ int s_w[8];
    const int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const bool zero = i < n && ppg[i] == 0;
    const unsigned m = __ballot_sync(0xffffffffu, zero);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) s_w[warp] = __popc(m);
    __syncthreads();
    long long before = blk[2 * blockIdx.x + 1];
    for (int w = 0; w < warp; ++w) before += s_w[w];
    if (zero && before + __popc(m & ((1u << lane) - 1u)) < take[0]) ppg[i] = 1;
}

// workspace of g2pc_points_per_gaussian; a null base only sizes it
struct PpgWs {
    double* partial;  // per-CTA magnitude sums
    long long* blk;   // per-CTA (sum of ppg, zero count), then the zero counts' exclusive scan
    double* sum;
    long long* take;
    size_t bytes;
};

PpgWs ppg_ws(void* base, int64_t n) {
    const size_t nb = (size_t)((n + 255) / 256);
    WsCarve w{(char*)base};
    PpgWs l;
    l.partial = w.take<double>(nb);
    l.blk = w.take<long long>(2 * nb);
    l.sum = w.take<double>(1);
    l.take = w.take<long long>(1);
    l.bytes = w.used;
    return l;
}

}  // namespace

extern "C" int64_t g2pc_cull_workspace_bytes(int64_t n) {
    return (int64_t)(((n + CTILE - 1) / CTILE + 1) * sizeof(int32_t));
}

extern "C" int g2pc_cull_select(const float* max_contrib, float vis_threshold, const float* opacity, float min_opacity,
                                const float* xyz, const float* bbox_min3_host, const float* bbox_max3_host,
                                const float* surface_dist, const float* surface_threshold_dev, const uint8_t* extra_mask,
                                int64_t lo, int64_t hi, int64_t n, int32_t* index, int64_t* count, void* workspace,
                                int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(index || n == 0, "null index");
    G2PC_CHECK_ARG(count && workspace, "null pointer");
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, g2pc_cull_workspace_bytes(n), 4);
    G2PC_CHECK_ARG(n < 0x7FFFFFFFll, "n must fit int32 indices");
    G2PC_CHECK_ARG(!(bbox_min3_host || bbox_max3_host) || xyz, "bounding box needs xyz");
    G2PC_CHECK_ARG((surface_dist == nullptr) == (surface_threshold_dev == nullptr), "surface distance needs its threshold");
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) { G2PC_CUDA(cudaMemsetAsync(count, 0, sizeof(int64_t), st)); return G2PC_OK; }
    CullParams p;
    p.max_contrib = max_contrib; p.vis_thr = vis_threshold; p.opacity = opacity; p.min_opacity = min_opacity;
    p.xyz = xyz; p.use_bmin = bbox_min3_host ? 1 : 0; p.use_bmax = bbox_max3_host ? 1 : 0;
    for (int k = 0; k < 3; ++k) { p.bmin[k] = bbox_min3_host ? bbox_min3_host[k] : 0.f; p.bmax[k] = bbox_max3_host ? bbox_max3_host[k] : 0.f; }
    p.surf = surface_dist; p.surf_thr = surface_threshold_dev; p.extra = extra_mask;
    p.lo = lo; p.hi = hi; p.n = n;
    const int nb = (int)((n + CTILE - 1) / CTILE);
    int32_t* blk = (int32_t*)workspace;
    cull_count_kernel<<<nb, CB, 0, st>>>(p, blk);
    G2PC_CHECK_LAUNCH();
    cull_scan_kernel<<<1, 1024, 0, st>>>(blk, nb, count);
    G2PC_CHECK_LAUNCH();
    cull_write_kernel<<<nb, CB, 0, st>>>(p, blk, index);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_gather_rows(const int32_t* index, int64_t m, int32_t num_arrays, const void* const* srcs,
                                void* const* dsts, const int32_t* row_bytes, void* stream) {
    G2PC_CHECK_ARG(m >= 0 && num_arrays >= 0, "negative size");
    if (m == 0 || num_arrays == 0) return G2PC_OK;
    G2PC_CHECK_ARG(index && srcs && dsts && row_bytes, "null pointer");
    for (int a = 0; a < num_arrays; ++a) {
        G2PC_CHECK_ARG(srcs[a] && dsts[a] && row_bytes[a] > 0 && (row_bytes[a] & 3) == 0, "rows must be whole 32-bit words");
        const int words = row_bytes[a] / 4;
        const int64_t tot = m * words;
        gather_rows_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
            (const uint32_t*)srcs[a], (uint32_t*)dsts[a], index, m, words);
        G2PC_CHECK_LAUNCH();
    }
    return G2PC_OK;
}

extern "C" int64_t g2pc_ppg_workspace_bytes(int64_t n) { return (int64_t)ppg_ws(nullptr, n).bytes; }

/* magnitudes (n float64) and points per Gaussian (n int32) from covariances (n,3,3) f32 and contributions (n) f32. */
extern "C" int g2pc_points_per_gaussian(const float* cov, const float* contrib, int64_t n, double num_points,
                                        double* magnitudes, int32_t* ppg, void* workspace, int64_t workspace_bytes,
                                        void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(cov && contrib && magnitudes && ppg && workspace, "null pointer");
    const PpgWs l = ppg_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 8);
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = (int)((n + 255) / 256);
    magnitudes_kernel<<<nb, 256, 0, st>>>(cov, contrib, n, magnitudes, l.partial);
    G2PC_CHECK_LAUNCH();
    sum_partials_kernel<<<1, 1024, 0, st>>>(l.partial, nb, l.sum);
    G2PC_CHECK_LAUNCH();
    ppg_round_kernel<<<nb, 256, 0, st>>>(magnitudes, l.sum, num_points, n, ppg, l.blk);
    G2PC_CHECK_LAUNCH();
    ppg_plan_kernel<<<1, 1024, 0, st>>>(l.blk, nb, num_points, l.take);
    G2PC_CHECK_LAUNCH();
    ppg_fix_kernel<<<nb, 256, 0, st>>>(ppg, l.blk, l.take, n);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
