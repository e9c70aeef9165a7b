// s14_tsdf.cu — mesh a Gaussian scene by truncated signed-distance (TSDF) fusion of its rendered depth (N10): the frame
// of the voxel grid, the per-camera integration of the fusion blend's median depth, and the gather / compaction that
// keep the part of the marching-tetrahedra surface whose corners some camera observed.
//
// Grid: R = 2^depth voxels per axis at origin + (i + 1/2) h, the frame rule and node index (k R + j) R + i of the Poisson
// mesher (s10_mesh.cu), so that g2pc_mesh_extract_count / _emit run unchanged on the tsdf grid.  Per voxel: tsdf (f32,
// initially +1), weight (f32 camera count, initially 0) and colour (3 planes of f32, initially 0): 20 bytes.
// Integration is one thread per voxel per camera, the cameras in order on one stream: no atomics, bit-identical re-runs.
// DESIGN.md §2 (N10) writes the rules down; tests/f64ref_tsdf.py restates them.  Float64 expressions use the __d*_rn
// intrinsics and float32 updates the __f*_rn ones: no FMA contraction anywhere a test compares bits.
#include <cub/cub.cuh>
#include "mesh_common.cuh"
#include "colour_common.cuh"

namespace {

// one thread: the frame words of s10_mesh.cu's frame_kernel from the bounding box of the finite means
__global__ void tsdf_frame_kernel(const float* __restrict__ part, int nb, int R, double* __restrict__ fr) {
    float mn[3], mx[3];
    fold_bbox(part, nb, mn, mx);
    double ext = 0.0;
    const bool any = mn[0] <= mx[0];
    if (any)
        for (int a = 0; a < 3; ++a) ext = fmax(ext, __dsub_rn((double)mx[a], (double)mn[a]));
    const double L = __dmul_rn(1.1, ext);
    for (int a = 0; a < 3; ++a)
        fr[FR_ORIGIN + a] = any ? __dsub_rn(__dmul_rn(__dadd_rn((double)mn[a], (double)mx[a]), 0.5), __dmul_rn(L, 0.5))
                                : 0.0;
    fr[FR_H] = __ddiv_rn(L, (double)R);
    fr[FR_L] = L;
    fr[FR_MEANB] = 0.0;
    fr[FR_EXTENT] = ext;
    fr[FR_R] = (double)R;
}

struct IntegrateParams {
    const double* fr;
    const float* zmed;     // (H,W)
    const float* T;        // (H,W)
    const float* image;    // (3,H,W) = C + T bg
    const int32_t* mask;   // (H*W) or null
    const uint32_t* fail;
    int32_t frame, R, W, H;
    double view[16], proj[16];  // the camera's float32 matrices, exactly
    double trunc;               // mu = float(trunc * h)
    float bg[3];
    float* tsdf;
    float* weight;
    float* colour;              // (3, R^3)
};

// row-vector convention: v' = [x y z 1] M, M row-major (g2pc_raster_t)
__device__ __forceinline__ double affine(const double* M, int c, double x, double y, double z) {
    return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[c], x), __dmul_rn(M[4 + c], y)), __dmul_rn(M[8 + c], z)), M[12 + c]);
}

__global__ void __launch_bounds__(MB) tsdf_integrate_kernel(const IntegrateParams p) {
    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    const int64_t cells = (int64_t)p.R * p.R * p.R;
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= cells) return;
    const int i = (int)(v % p.R), j = (int)((v / p.R) % p.R), k = (int)(v / ((int64_t)p.R * p.R));
    const double x = node_coord(p.fr, 0, i), y = node_coord(p.fr, 1, j), z = node_coord(p.fr, 2, k);
    const double zv = affine(p.view, 2, x, y, z);
    if (!(zv > 0.2)) return;
    const double hx = affine(p.proj, 0, x, y, z), hy = affine(p.proj, 1, x, y, z), hw = affine(p.proj, 3, x, y, z);
    const double pw = __ddiv_rn(1.0, __dadd_rn(hw, 1e-7));
    const double px = __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(hx, pw), 1.0), (double)p.W), 1.0), 0.5);
    const double py = __dmul_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dmul_rn(hy, pw), 1.0), (double)p.H), 1.0), 0.5);
    const double fx = floor(__dadd_rn(px, 0.5)), fy = floor(__dadd_rn(py, 0.5));
    if (!(fx >= 0.0 && fx < (double)p.W && fy >= 0.0 && fy < (double)p.H)) return;  // NaN fails too
    const int64_t pix = (int64_t)fy * p.W + (int64_t)fx;
    if (p.mask && p.mask[pix] == 0) return;
    const float zm = p.zmed[pix];
    if (zm == 0.0f) return;
    const float mu = __double2float_rn(__dmul_rn(p.trunc, p.fr[FR_H]));
    const float sdf = __fsub_rn(zm, __double2float_rn(zv));
    if (sdf < -mu) return;
    const float tv = fminf(1.0f, __fdiv_rn(sdf, mu));
    const float Tp = p.T[pix];
    const float w = p.weight[v], w1 = __fadd_rn(w, 1.0f);
    p.tsdf[v] = __fdiv_rn(__fadd_rn(__fmul_rn(p.tsdf[v], w), tv), w1);
    const int64_t hwp = (int64_t)p.W * p.H;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float raw = __fdiv_rn(__fsub_rn(p.image[c * hwp + pix], __fmul_rn(Tp, p.bg[c])), __fsub_rn(1.0f, Tp));
        const float cc = fminf(fmaxf(raw, 0.0f), 1.0f);
        float* col = p.colour + c * cells + v;
        *col = __fdiv_rn(__fadd_rn(__fmul_rn(*col, w), cc), w1);
    }
    p.weight[v] = w1;
}

// per vertex of the extraction (key = node * 8 + d, edge node -> node + (d & 1, d >> 1 & 1, d >> 2)): kept iff both
// ends have weight > 0; density (1 - t) w_a + t w_b, colour floor(255 ((1 - t) c_a + t c_b) + 1/2) clamped to 0..255
__global__ void __launch_bounds__(MB) tsdf_gather_kernel(const float* __restrict__ weight, const float* __restrict__ colour,
                                                         int R, const long long* __restrict__ vkey,
                                                         const double* __restrict__ vt, int64_t m,
                                                         uint8_t* __restrict__ keep, int32_t* __restrict__ flag,
                                                         double* __restrict__ dens, uint8_t* __restrict__ vcol) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int64_t cells = (int64_t)R * R * R;
    const long long key = vkey[v];
    const int64_t a = key >> 3;
    const int d = (int)(key & 7);
    const int64_t b = a + (d & 1) + (int64_t)((d >> 1) & 1) * R + (int64_t)(d >> 2) * R * R;
    const float wa = weight[a], wb = weight[b];
    const int kp = (wa > 0.0f && wb > 0.0f) ? 1 : 0;
    keep[v] = (uint8_t)kp;
    flag[v] = kp;
    const double t = vt[v], s = __dsub_rn(1.0, t);
    dens[v] = __dadd_rn(__dmul_rn(s, (double)wa), __dmul_rn(t, (double)wb));
    if (vcol)
        for (int c = 0; c < 3; ++c) {
            const double x = __dadd_rn(__dmul_rn(s, (double)colour[c * cells + a]), __dmul_rn(t, (double)colour[c * cells + b]));
            const double q = floor(__dadd_rn(__dmul_rn(255.0, x), 0.5));
            vcol[3 * v + c] = (uint8_t)fmin(fmax(q, 0.0), 255.0);
        }
}

__global__ void __launch_bounds__(MB) tsdf_tri_flag_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                           const uint8_t* __restrict__ keep, int32_t* __restrict__ flag) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    flag[f] = keep[faces[3 * f]] & keep[faces[3 * f + 1]] & keep[faces[3 * f + 2]];
}

__global__ void __launch_bounds__(MB) tsdf_compact_kernel(const uint8_t* __restrict__ keep, const int32_t* __restrict__ vmap,
                                                          int64_t m, const double* __restrict__ dens,
                                                          const double* __restrict__ vpos, const uint8_t* __restrict__ vcol,
                                                          const int32_t* __restrict__ faces, const int32_t* __restrict__ tflag,
                                                          const int32_t* __restrict__ tmap, int64_t t,
                                                          double* __restrict__ dens_o, double* __restrict__ vpos_o,
                                                          uint8_t* __restrict__ vcol_o, int32_t* __restrict__ faces_o) {
    const int64_t e = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (e < m && keep[e]) {
        const int64_t o = vmap[e];
        dens_o[o] = dens[e];
        for (int a = 0; a < 3; ++a) vpos_o[3 * o + a] = vpos[3 * e + a];
        if (vcol)
            for (int a = 0; a < 3; ++a) vcol_o[3 * o + a] = vcol[3 * e + a];
    }
    if (e < t && tflag[e]) {
        const int64_t o = tmap[e];
        for (int s = 0; s < 3; ++s) faces_o[3 * o + s] = vmap[faces[3 * e + s]];
    }
}

__global__ void tsdf_counts_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ map, int64_t m,
                                   const int32_t* __restrict__ tflag, const int32_t* __restrict__ tmap, int64_t t,
                                   long long* __restrict__ counts) {
    counts[0] = m ? (long long)map[m - 1] + flag[m - 1] : 0;
    counts[1] = t ? (long long)tmap[t - 1] + tflag[t - 1] : 0;
}

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

bool depth_ok(int depth) { return depth >= 2 && depth <= G2PC_MESH_DEPTH_MAX; }

struct CompactWs {
    int32_t *vflag, *vmap, *tflag, *tmap;
    void* tmp;
    size_t tmp_bytes, bytes;
};
CompactWs compact_ws(void* base, int64_t m, int64_t t) {
    size_t scan_v = 0, scan_t = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_v, (const int32_t*)nullptr, (int32_t*)nullptr, (int)m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_t, (const int32_t*)nullptr, (int32_t*)nullptr, (int)t);
    WsCarve w{(char*)base};
    CompactWs l;
    l.vflag = w.take<int32_t>(m);
    l.vmap = w.take<int32_t>(m);
    l.tflag = w.take<int32_t>(t);
    l.tmap = w.take<int32_t>(t);
    l.tmp_bytes = WsCarve::pad(scan_v > scan_t ? scan_v : scan_t);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int64_t g2pc_tsdf_frame_workspace_bytes(int64_t n) {
    return (int64_t)(n > 0 ? bbox_blocks(n) : 1) * 6 * (int64_t)sizeof(float);
}

extern "C" int g2pc_tsdf_frame(const float* xyz, int64_t n, int32_t depth, double* frame, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(frame && workspace && (n == 0 || xyz), "null pointer");
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, g2pc_tsdf_frame_workspace_bytes(n), 4);
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = bbox_blocks(n);
    if (n > 0) {
        bbox_kernel<<<nb, BBOX_THREADS, 0, st>>>(xyz, n, (float*)workspace);
        G2PC_CHECK_LAUNCH();
    }
    tsdf_frame_kernel<<<1, 1, 0, st>>>((const float*)workspace, nb, 1 << depth, frame);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_tsdf_integrate(const double* frame, int32_t depth, double trunc_voxels, const float* zmed,
                                   const float* transmittance, const float* image, const int32_t* mask, int32_t width,
                                   int32_t height, const g2pc_raster_t* rs_host, const float* background3_host,
                                   const uint32_t* fail, int32_t frame_index, float* tsdf, float* weight, float* colour,
                                   void* stream) {
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(trunc_voxels > 0.0, "the truncation must be > 0 voxels");
    G2PC_CHECK_ARG(frame && zmed && transmittance && image && rs_host && background3_host && fail && tsdf && weight &&
                       colour, "null pointer");
    G2PC_CHECK_ARG(width > 0 && height > 0 && rs_host->width == width && rs_host->height == height, "bad image size");
    G2PC_CHECK_ARG(frame_index >= 0, "frame < 0");
    IntegrateParams p;
    p.fr = frame; p.zmed = zmed; p.T = transmittance; p.image = image; p.mask = mask; p.fail = fail;
    p.frame = frame_index; p.R = 1 << depth; p.W = width; p.H = height;
    for (int i = 0; i < 16; ++i) { p.view[i] = (double)rs_host->viewmatrix[i]; p.proj[i] = (double)rs_host->projmatrix[i]; }
    p.trunc = trunc_voxels;
    for (int c = 0; c < 3; ++c) p.bg[c] = background3_host[c];
    p.tsdf = tsdf; p.weight = weight; p.colour = colour;
    const int64_t cells = (int64_t)1 << (3 * depth);
    tsdf_integrate_kernel<<<grid_of(cells), MB, 0, (cudaStream_t)stream>>>(p);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_tsdf_compact_workspace_bytes(int64_t m, int64_t t) {
    return (int64_t)compact_ws(nullptr, m, t).bytes;
}

extern "C" int g2pc_tsdf_gather_compact(const float* weight, const float* colour, int32_t depth, const int64_t* vkey,
                                        const double* vt, const double* vpos, int64_t m, const int32_t* faces, int64_t t,
                                        uint8_t* keep, double* density, uint8_t* vcolours, int64_t* counts,
                                        double* density_out, double* vpos_out, uint8_t* vcolours_out, int32_t* faces_out,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(m > 0 && m < 0x7FFFFFFFll && t >= 0 && t < 0x7FFFFFFFll, "need 1..2^31-2 vertices");
    G2PC_CHECK_ARG(weight && vkey && vt && vpos && keep && density && counts && density_out && vpos_out && workspace,
                   "null pointer");
    G2PC_CHECK_ARG(!colour == !vcolours && !vcolours == !vcolours_out, "colours need the grid and both outputs");
    G2PC_CHECK_ARG(t == 0 || (faces && faces_out), "null pointer");
    const CompactWs l = compact_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    tsdf_gather_kernel<<<grid_of(m), MB, 0, st>>>(weight, colour, 1 << depth, (const long long*)vkey, vt, m, keep,
                                                  l.vflag, density, vcolours);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.vflag, l.vmap, (int)m, st));
    if (t > 0) {
        tsdf_tri_flag_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, keep, l.tflag);
        G2PC_CHECK_LAUNCH();
        b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.tflag, l.tmap, (int)t, st));
    }
    tsdf_compact_kernel<<<grid_of(m > t ? m : t), MB, 0, st>>>(keep, l.vmap, m, density, vpos, vcolours, faces, l.tflag,
                                                               l.tmap, t, density_out, vpos_out, vcolours_out, faces_out);
    G2PC_CHECK_LAUNCH();
    tsdf_counts_kernel<<<1, 1, 0, st>>>(l.vflag, l.vmap, m, l.tflag, l.tmap, t, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
