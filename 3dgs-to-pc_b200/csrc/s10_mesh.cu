// s10_mesh.cu — Poisson surface reconstruction of an oriented point cloud (N6): splat, multigrid solve, iso-value,
// marching tetrahedra, per-vertex density / colour gathers, density trim, Laplacian smoothing and vertex normals.
//
// Reference semantics restated (not copied): mesh_handler.py:23-40 generate_mesh = Open3D statistical outlier removal,
// create_from_point_cloud_poisson(depth), removal of the vertices below the 10 % density quantile, Laplacian smoothing.
// The rules below are this project's own (Open3D's octree solver is not restated); DESIGN.md §2 writes them down and
// tests/f64ref_mesh.py restates them in float64.
//
// Grid: R = 2^depth nodes per axis at the cell centres origin + (i + 1/2) h of a cube of edge L = 1.1 x the largest
// extent, centred on the bounding box; node index (k R + j) R + i.  Every point has a dual cell i0 (the 2x2x2 nodes
// around it) and trilinear weights w = (wx * wy) * wz.  B (int64) is the central-difference divergence of the splatted
// normals in units of 2^-32: exact integer atomics, so re-runs are bit-identical.  The solve works on float32 grids with
// the right-hand side b = (B - mean B) * h * 2^-33 formed on the fly from B (no float copy of b is stored).
// All float64 expressions that a test compares bit for bit are written with __d*_rn intrinsics: no FMA contraction.
#include <cub/cub.cuh>
#include "mesh_common.cuh"

namespace {

constexpr int COARSE_SWEEPS = 100;              // red-black sweeps of the 4^3 coarsest level

// ---- splat ------------------------------------------------------------------------------------------------------
// one thread: L = 1.1 * largest extent, origin = centre - L / 2, h = L / R (h = 0 when no finite point / zero extent)
__global__ void frame_kernel(const float* __restrict__ part, int nb, int R, double* __restrict__ fr) {
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

// per point: skip zero / non-finite normals (status[0]) and non-finite points (status[1]); otherwise every (node c,
// axis a) of the dual cell adds q = llrint(w * n_a * 2^32) to B[c - e_a] and subtracts it from B[c + e_a]
template <typename NT>
__global__ void __launch_bounds__(MB) splat_kernel(const float* __restrict__ xyz, const NT* __restrict__ nrm, int64_t n,
                                                   int R, const double* __restrict__ fr,
                                                   unsigned long long* __restrict__ B, uint32_t* __restrict__ cell,
                                                   int32_t* __restrict__ status) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= n) return;
    cell[i] = CELL_NONE;
    if (!finite3(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2])) { atomicAdd(&status[1], 1); return; }
    if (!(fr[FR_H] > 0.0)) return;
    double nh[3];
    if (!unit_normal(nrm, i, nh)) { atomicAdd(&status[0], 1); return; }
    const PointCell c = point_cell(xyz, i, fr, R);
    cell[i] = cell_id(c, R);
    const int64_t stride[3] = {1, R, (int64_t)R * R};
    for (int o = 0; o < 8; ++o) {
        const double w = corner_weight(c, o);
        const int cc[3] = {c.i0[0] + (o & 1), c.i0[1] + ((o >> 1) & 1), c.i0[2] + (o >> 2)};
        const int64_t node = ((int64_t)cc[2] * R + cc[1]) * R + cc[0];
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const long long q = splat_q(w, nh[a]);
            if (q == 0) continue;
            if (cc[a] > 0) atomicAdd(&B[node - stride[a]], (unsigned long long)q);
            if (cc[a] < R - 1) atomicAdd(&B[node + stride[a]], (unsigned long long)(-q));
        }
    }
}

// exact int64 sum of B (wrap-around arithmetic: the total is exact whenever it fits int64)
__global__ void __launch_bounds__(MB) sum_b_kernel(const long long* __restrict__ B, int64_t cells,
                                                   unsigned long long* __restrict__ total) {
    unsigned long long v = 0;
    for (int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x; i < cells; i += (int64_t)gridDim.x * MB)
        v += (unsigned long long)B[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) atomicAdd(total, v);
}

__global__ void mean_b_kernel(const unsigned long long* __restrict__ total, int64_t cells, double* __restrict__ fr) {
    fr[FR_MEANB] = __ddiv_rn((double)(long long)*total, (double)cells);
}

// ---- multigrid ---------------------------------------------------------------------------------------------------
// right-hand side of a level: the finest reads B, the coarser ones their float grid
struct Rhs {
    const long long* B;
    const float* f;
    const double* fr;
    __device__ __forceinline__ float operator()(int64_t i) const {
        if (f) return f[i];
        return (float)__dmul_rn(__dsub_rn((double)B[i], fr[FR_MEANB]), __dmul_rn(fr[FR_H], 0x1p-33));
    }
};

// sum of the in-grid neighbours of (i, j, k) and their count (a mirrored ghost equals the cell itself)
template <typename T>
__device__ __forceinline__ T neighbour_sum(const float* __restrict__ chi, int n, int i, int j, int k, int64_t c, int& cnt) {
    const int64_t nn = (int64_t)n * n;
    T s = 0;
    cnt = 0;
    if (i > 0) { s += (T)chi[c - 1]; ++cnt; }
    if (i < n - 1) { s += (T)chi[c + 1]; ++cnt; }
    if (j > 0) { s += (T)chi[c - n]; ++cnt; }
    if (j < n - 1) { s += (T)chi[c + n]; ++cnt; }
    if (k > 0) { s += (T)chi[c - nn]; ++cnt; }
    if (k < n - 1) { s += (T)chi[c + nn]; ++cnt; }
    return s;
}

// b - (sum of neighbours - 6 chi) with mirrored ghosts = b - (sum of in-grid neighbours - count * chi), in float64
__device__ __forceinline__ double residual(const float* __restrict__ chi, const Rhs& rhs, int n, int i, int j, int k) {
    const int64_t c = ((int64_t)k * n + j) * n + i;
    int cnt;
    const double s = neighbour_sum<double>(chi, n, i, j, k, c, cnt);
    return (double)rhs(c) - (s - (double)cnt * (double)chi[c]);
}

// one colour of a red-black Gauss-Seidel sweep: cells with (i + j + k) % 2 == colour
__global__ void __launch_bounds__(MB) rb_smooth_kernel(float* __restrict__ chi, Rhs rhs, int n, int colour) {
    const int64_t t = (int64_t)blockIdx.x * MB + threadIdx.x;
    const int half = n >> 1;
    if (t >= (int64_t)n * n * half) return;
    const int64_t row = t / half;
    const int j = (int)(row % n), k = (int)(row / n);
    const int i = 2 * (int)(t % half) + ((j + k + colour) & 1);
    const int64_t c = ((int64_t)k * n + j) * n + i;
    int cnt;
    const float s = neighbour_sum<float>(chi, n, i, j, k, c, cnt);
    chi[c] = (s - rhs(c)) / (float)cnt;
}

// coarse right-hand side = 4 x the mean of the 8 fine residuals (the stencil is not scaled by 1/h^2)
__global__ void __launch_bounds__(MB) restrict_kernel(const float* __restrict__ chi, Rhs rhs, int n,
                                                      float* __restrict__ rc) {
    const int nc = n >> 1;
    const int64_t t = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (t >= (int64_t)nc * nc * nc) return;
    const int I = (int)(t % nc), J = (int)((t / nc) % nc), K = (int)(t / ((int64_t)nc * nc));
    double s = 0.0;
    for (int o = 0; o < 8; ++o) s += residual(chi, rhs, n, 2 * I + (o & 1), 2 * J + ((o >> 1) & 1), 2 * K + (o >> 2));
    rc[t] = (float)(0.5 * s);
}

// fine += trilinear (cell-centred: 3/4, 1/4 per axis, clamped at the faces) interpolation of the coarse correction
__global__ void __launch_bounds__(MB) prolong_kernel(float* __restrict__ chi, int n, const float* __restrict__ ec) {
    const int64_t t = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (t >= (int64_t)n * n * n) return;
    const int nc = n >> 1;
    const int p[3] = {(int)(t % n), (int)((t / n) % n), (int)(t / ((int64_t)n * n))};
    int lo[3], hi[3];
    for (int a = 0; a < 3; ++a) {
        lo[a] = p[a] >> 1;
        const int q = lo[a] + ((p[a] & 1) ? 1 : -1);
        hi[a] = q < 0 ? 0 : (q > nc - 1 ? nc - 1 : q);
    }
    float e = 0.f;
    for (int o = 0; o < 8; ++o) {
        const int x = (o & 1) ? hi[0] : lo[0], y = (o & 2) ? hi[1] : lo[1], z = (o & 4) ? hi[2] : lo[2];
        const float w = ((o & 1) ? 0.25f : 0.75f) * ((o & 2) ? 0.25f : 0.75f) * ((o & 4) ? 0.25f : 0.75f);
        e += w * ec[((int64_t)z * nc + y) * nc + x];
    }
    chi[t] += e;
}

// the 4^3 coarsest level in one CTA: right-hand side made mean-free, then red-black sweeps from the current chi
__global__ void __launch_bounds__(64) coarse_kernel(float* __restrict__ chi, Rhs rhs) {
    __shared__ float x[64], b[64];
    __shared__ float mean;
    const int t = threadIdx.x;
    x[t] = chi[t];
    b[t] = rhs(t);
    __syncthreads();
    if (t == 0) {
        double s = 0.0;
        for (int q = 0; q < 64; ++q) s += b[q];
        mean = (float)(s / 64.0);
    }
    __syncthreads();
    b[t] -= mean;
    const int i = t & 3, j = (t >> 2) & 3, k = t >> 4;
    __syncthreads();
    for (int it = 0; it < COARSE_SWEEPS; ++it) {
        for (int colour = 0; colour < 2; ++colour) {
            if (((i + j + k) & 1) == colour) {
                int cnt;
                const float s = neighbour_sum<float>(x, 4, i, j, k, t, cnt);
                x[t] = (s - b[t]) / (float)cnt;
            }
            __syncthreads();
        }
    }
    chi[t] = x[t];
}

// MODE 0: partial sums of r^2 at the finest level; 1: of b^2; 2: of chi
template <int MODE>
__global__ void __launch_bounds__(MB) grid_partial_kernel(const float* __restrict__ chi, Rhs rhs, int n,
                                                          double* __restrict__ partial) {
    __shared__ double s_w[MB / 32];
    const int64_t cells = (int64_t)n * n * n;
    double v = 0.0;
    for (int64_t t = (int64_t)blockIdx.x * MB + threadIdx.x; t < cells; t += (int64_t)RED_BLOCKS * MB) {
        if (MODE == 0) {
            const double r = residual(chi, rhs, n, (int)(t % n), (int)((t / n) % n), (int)(t / ((int64_t)n * n)));
            v = __dadd_rn(v, __dmul_rn(r, r));
        } else if (MODE == 1) {
            const double b = (double)rhs(t);
            v = __dadd_rn(v, __dmul_rn(b, b));
        } else {
            v = __dadd_rn(v, (double)chi[t]);
        }
    }
    const double tot = block_sum_f64<MB>(v, s_w);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(MB) shift_kernel(float* __restrict__ chi, int64_t cells, const double* __restrict__ mean) {
    const int64_t t = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (t < cells) chi[t] = (float)__dsub_rn((double)chi[t], *mean);
}

// iso: partial sums of (trilinear chi at the point) and of the count over the splatted points
__global__ void __launch_bounds__(MB) iso_partial_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ cell,
                                                         int64_t n, const double* __restrict__ fr, int R,
                                                         const float* __restrict__ chi, double* __restrict__ partial) {
    __shared__ double s_w[MB / 32];
    double v = 0.0, cnt = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x; i < n; i += (int64_t)RED_BLOCKS * MB) {
        if (cell[i] == CELL_NONE) continue;
        const PointCell c = point_cell(xyz, i, fr, R);
        double x = 0.0;
        for (int o = 0; o < 8; ++o) {
            const int64_t node = ((int64_t)(c.i0[2] + (o >> 2)) * R + c.i0[1] + ((o >> 1) & 1)) * R + c.i0[0] + (o & 1);
            x = __dadd_rn(x, __dmul_rn(corner_weight(c, o), (double)chi[node]));
        }
        v = __dadd_rn(v, x);
        cnt += 1.0;
    }
    const double tv = block_sum_f64<MB>(v, s_w);
    __syncthreads();
    const double tc = block_sum_f64<MB>(cnt, s_w);
    if (threadIdx.x == 0) { partial[blockIdx.x] = tv; partial[RED_BLOCKS + blockIdx.x] = tc; }
}

__global__ void iso_div_kernel(double* __restrict__ iso2) {
    iso2[1] = iso2[2] > 0.0 ? __ddiv_rn(iso2[1], iso2[2]) : 0.0;
}


// ---- marching tetrahedra --------------------------------------------------------------------------------------------
__device__ __forceinline__ Cube load_cube(const float* __restrict__ chi, int R, int i, int j, int k, double iso) {
    Cube c{0u, 0u};
#pragma unroll
    for (int o = 0; o < 8; ++o) {
        const int x = i + (o & 1), y = j + ((o >> 1) & 1), z = k + (o >> 2);
        if (x < R && y < R && z < R) {
            c.valid |= 1u << o;
            if ((double)chi[((int64_t)z * R + y) * R + x] < iso) c.inside |= 1u << o;
        }
    }
    return c;
}


__device__ __forceinline__ void node_ijk(int64_t node, int R, int& i, int& j, int& k) {
    i = (int)(node % R);
    j = (int)((node / R) % R);
    k = (int)(node / ((int64_t)R * R));
}

// per CTA (NODES_PER_CTA consecutive nodes): crossed edges and triangles of the cubes whose lowest corner they are
__global__ void __launch_bounds__(MB) mt_count_kernel(const float* __restrict__ chi, int R, const double* __restrict__ iso2,
                                                      long long* __restrict__ vblk, long long* __restrict__ tblk) {
    __shared__ double s_w[MB / 32];
    const double iso = iso2[1];
    const int64_t cells = (int64_t)R * R * R;
    int nv = 0, nt = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t node = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        if (node >= cells) break;
        int i, j, k;
        node_ijk(node, R, i, j, k);
        const Cube c = load_cube(chi, R, i, j, k, iso);
        nv += __popc(cross_mask(c));
        if (c.valid == 0xFFu) nt += cube_triangle_count(c.inside);
    }
    const double sv = block_sum_f64<MB>((double)nv, s_w);
    __syncthreads();
    const double st = block_sum_f64<MB>((double)nt, s_w);
    if (threadIdx.x == 0) { vblk[blockIdx.x] = (long long)sv; tblk[blockIdx.x] = (long long)st; }
}

__global__ void totals_kernel(const long long* __restrict__ voff, const long long* __restrict__ toff, int64_t nb,
                              long long* __restrict__ counts) {
    counts[0] = voff[nb];
    counts[1] = toff[nb];
}

// vertices in ascending edge key (node * 8 + d); node_base[node] = index of the node's first vertex, node_mask[node] =
// its crossed-edge mask (both read by the triangle pass)
__global__ void __launch_bounds__(MB) mt_vertex_kernel(const float* __restrict__ chi, int R, const double* __restrict__ fr,
                                                       const double* __restrict__ iso2, const long long* __restrict__ voff,
                                                       int32_t* __restrict__ node_base, uint8_t* __restrict__ node_mask,
                                                       long long* __restrict__ vkey, double* __restrict__ vt,
                                                       double* __restrict__ vpos) {
    typedef cub::BlockScan<int, MB> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const double iso = iso2[1];
    const int64_t cells = (int64_t)R * R * R;
    uint32_t m[NPT];
    int nv = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t node = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        m[q] = 0;
        if (node >= cells) continue;
        int i, j, k;
        node_ijk(node, R, i, j, k);
        m[q] = cross_mask(load_cube(chi, R, i, j, k, iso));
        nv += __popc(m[q]);
    }
    int pre;
    Scan(tmp).ExclusiveSum(nv, pre);
    long long cur = voff[blockIdx.x] + pre;
    for (int q = 0; q < NPT; ++q) {
        const int64_t node = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        if (node >= cells) break;
        node_base[node] = (int32_t)cur;
        node_mask[node] = (uint8_t)m[q];
        if (!m[q]) continue;
        int i, j, k;
        node_ijk(node, R, i, j, k);
        const double ca = (double)chi[node];
        const double pa[3] = {node_coord(fr, 0, i), node_coord(fr, 1, j), node_coord(fr, 2, k)};
        for (int d = 1; d < 8; ++d) {
            if (!((m[q] >> d) & 1u)) continue;
            const int ib = i + (d & 1), jb = j + ((d >> 1) & 1), kb = k + (d >> 2);
            const double cb = (double)chi[((int64_t)kb * R + jb) * R + ib];
            const double t = __ddiv_rn(__dsub_rn(iso, ca), __dsub_rn(cb, ca));
            const double pb[3] = {node_coord(fr, 0, ib), node_coord(fr, 1, jb), node_coord(fr, 2, kb)};
            vkey[cur] = node * 8 + d;
            vt[cur] = t;
            for (int a = 0; a < 3; ++a) vpos[3 * cur + a] = __dadd_rn(pa[a], __dmul_rn(t, __dsub_rn(pb[a], pa[a])));
            ++cur;
        }
    }
}

// triangles in ascending (cube, tetrahedron, triangle)
__global__ void __launch_bounds__(MB) mt_triangle_kernel(const float* __restrict__ chi, int R,
                                                         const double* __restrict__ iso2, const long long* __restrict__ toff,
                                                         const int32_t* __restrict__ node_base,
                                                         const uint8_t* __restrict__ node_mask,
                                                         int32_t* __restrict__ faces) {
    typedef cub::BlockScan<int, MB> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const double iso = iso2[1];
    const int64_t cells = (int64_t)R * R * R;
    uint32_t ins[NPT];
    int nt = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t node = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        ins[q] = 0xFFu;  // no triangles
        if (node >= cells) continue;
        int i, j, k;
        node_ijk(node, R, i, j, k);
        const Cube c = load_cube(chi, R, i, j, k, iso);
        if (c.valid != 0xFFu) continue;
        ins[q] = c.inside;
        nt += cube_triangle_count(c.inside);
    }
    int pre;
    Scan(tmp).ExclusiveSum(nt, pre);
    long long cur = toff[blockIdx.x] + pre;
    for (int q = 0; q < NPT; ++q) {
        if (ins[q] == 0xFFu || ins[q] == 0u) continue;
        const int64_t node = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        for (int p = 0; p < 6; ++p) {
            int tri[2][3][2];
            const int n = tet_triangles(p, ins[q], tri);
            for (int t = 0; t < n; ++t, ++cur) {
                for (int s = 0; s < 3; ++s) {
                    const int lo = tri[t][s][0], d = tri[t][s][1] ^ lo;
                    const int64_t pn = node + (lo & 1) + (int64_t)((lo >> 1) & 1) * R + (int64_t)(lo >> 2) * R * R;
                    faces[3 * cur + s] = node_base[pn] + __popc(node_mask[pn] & ((1u << d) - 1u));
                }
            }
        }
    }
}

// ---- density and colour gathers ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MB) iota_kernel(uint32_t* __restrict__ v, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i < n) v[i] = (uint32_t)i;
}

// first sorted position of every non-empty dual cell (the others stay -1)
__global__ void __launch_bounds__(MB) cell_start_kernel(const uint32_t* __restrict__ sk, int64_t n,
                                                        int32_t* __restrict__ start) {
    const int64_t j = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (j >= n) return;
    const uint32_t key = sk[j];
    if (key != CELL_NONE && (j == 0 || sk[j - 1] != key)) start[key] = (int32_t)j;
}

// W = sum of w, C = sum of w * colour over the points of the 8 dual cells around the node: cells in ascending index,
// points in ascending input index, sequential float64
__device__ __forceinline__ void node_sums(int x, int y, int z, int R, const uint32_t* __restrict__ sk,
                                          const uint32_t* __restrict__ sidx, int64_t n, const int32_t* __restrict__ start,
                                          const float* __restrict__ xyz, const int32_t* __restrict__ col,
                                          const double* __restrict__ fr, double& W, double (&C)[3]) {
    W = 0.0;
    C[0] = C[1] = C[2] = 0.0;
    for (int o = 7; o >= 0; --o) {
        const int cx = x - (o & 1), cy = y - ((o >> 1) & 1), cz = z - (o >> 2);
        if (cx < 0 || cy < 0 || cz < 0 || cx > R - 2 || cy > R - 2 || cz > R - 2) continue;
        const uint32_t id = ((uint32_t)cz * (uint32_t)(R - 1) + (uint32_t)cy) * (uint32_t)(R - 1) + (uint32_t)cx;
        int64_t j = start[id];
        if (j < 0) continue;
        for (; j < n && sk[j] == id; ++j) {
            const uint32_t pi = sidx[j];
            const double w = corner_weight(point_cell(xyz, pi, fr, R), o);
            W = __dadd_rn(W, w);
            if (col)
                for (int a = 0; a < 3; ++a) C[a] = __dadd_rn(C[a], __dmul_rn(w, (double)col[3 * (int64_t)pi + a]));
        }
    }
}

__global__ void __launch_bounds__(MB) gather_kernel(const long long* __restrict__ vkey, const double* __restrict__ vt,
                                                    int64_t m, int R, const uint32_t* __restrict__ sk,
                                                    const uint32_t* __restrict__ sidx, int64_t n,
                                                    const int32_t* __restrict__ start, const float* __restrict__ xyz,
                                                    const int32_t* __restrict__ col, const double* __restrict__ fr,
                                                    double* __restrict__ dens, uint8_t* __restrict__ vcol) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const long long key = vkey[v];
    const int64_t node = key >> 3;
    const int d = (int)(key & 7);
    int i, j, k;
    node_ijk(node, R, i, j, k);
    double Wa, Wb, Ca[3], Cb[3];
    node_sums(i, j, k, R, sk, sidx, n, start, xyz, col, fr, Wa, Ca);
    node_sums(i + (d & 1), j + ((d >> 1) & 1), k + (d >> 2), R, sk, sidx, n, start, xyz, col, fr, Wb, Cb);
    const double t = vt[v], s = __dsub_rn(1.0, t);
    const double D = __dadd_rn(__dmul_rn(s, Wa), __dmul_rn(t, Wb));
    dens[v] = D;
    if (!vcol) return;
    for (int a = 0; a < 3; ++a) {
        double c = 0.0;
        if (D > 0.0) {
            c = floor(__dadd_rn(__ddiv_rn(__dadd_rn(__dmul_rn(s, Ca[a]), __dmul_rn(t, Cb[a])), D), 0.5));
            c = fmin(fmax(c, 0.0), 255.0);
        }
        vcol[3 * v + a] = (uint8_t)c;
    }
}

// ---- density trim -------------------------------------------------------------------------------------------------
// numpy's default (linear) quantile q = 0.1 of the sorted densities: virtual index (m - 1) * q, then
// a + (b - a) * g, or b - (b - a) * (1 - g) when g >= 0.5
__global__ void quantile_kernel(const double* __restrict__ sorted, int64_t m, double* __restrict__ thr) {
    const double vi = __dmul_rn((double)(m - 1), 0.1);
    int64_t lo, hi;
    double g;
    if (vi >= (double)(m - 1)) {
        lo = hi = m - 1;
        g = 0.0;
    } else {
        const double fl = floor(vi);
        lo = (int64_t)fl;
        hi = lo + 1;
        g = __dsub_rn(vi, fl);
    }
    const double a = sorted[lo], b = sorted[hi], diff = __dsub_rn(b, a);
    *thr = g >= 0.5 ? __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(diff, g));
}

__global__ void __launch_bounds__(MB) keep_kernel(const double* __restrict__ dens, int64_t m,
                                                  const double* __restrict__ thr, uint8_t* __restrict__ keep,
                                                  int32_t* __restrict__ flag) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int k = dens[v] < *thr ? 0 : 1;
    keep[v] = (uint8_t)k;
    flag[v] = k;
}

// ---- smoothing, normals (their one-ring / incidence lists: mesh_common.cuh) ----------------------------------------
// one Jacobi step, lambda = 1/2: v + (sum w_j v_j / sum w_j - v) / 2, w_j = 1 / (|v - v_j| + 1e-12), distinct
// neighbours in ascending index
__global__ void __launch_bounds__(MB) smooth_kernel(const double* __restrict__ p, int64_t m,
                                                    const unsigned long long* __restrict__ keys,
                                                    const int32_t* __restrict__ row, double* __restrict__ q) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const double x[3] = {p[3 * v], p[3 * v + 1], p[3 * v + 2]};
    double sw = 0.0, s[3] = {0.0, 0.0, 0.0};
    const int64_t r0 = row[v], r1 = row[v + 1];
    for (int64_t j = r0; j < r1; ++j) {
        if (j > r0 && keys[j] == keys[j - 1]) continue;
        const int64_t u = (int64_t)(keys[j] & 0xFFFFFFFFull);
        const double y[3] = {p[3 * u], p[3 * u + 1], p[3 * u + 2]};
        const double dx = __dsub_rn(x[0], y[0]), dy = __dsub_rn(x[1], y[1]), dz = __dsub_rn(x[2], y[2]);
        const double dist = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
        const double w = __ddiv_rn(1.0, __dadd_rn(dist, 1e-12));
        sw = __dadd_rn(sw, w);
        for (int a = 0; a < 3; ++a) s[a] = __dadd_rn(s[a], __dmul_rn(w, y[a]));
    }
    for (int a = 0; a < 3; ++a)
        q[3 * v + a] = r1 > r0 ? __dadd_rn(x[a], __dmul_rn(0.5, __dsub_rn(__ddiv_rn(s[a], sw), x[a]))) : x[a];
}

// normal = normalised sum of cross(p1 - p0, p2 - p0) over the incident triangles in ascending order (zero stays zero)
__global__ void __launch_bounds__(MB) normals_kernel(const double* __restrict__ p, int64_t m,
                                                     const int32_t* __restrict__ faces,
                                                     const unsigned long long* __restrict__ keys,
                                                     const int32_t* __restrict__ row, float* __restrict__ vout,
                                                     float* __restrict__ nout) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    double n[3] = {0.0, 0.0, 0.0};
    for (int64_t j = row[v]; j < row[v + 1]; ++j) {
        const int64_t f = (int64_t)(keys[j] & 0xFFFFFFFFull);
        const int64_t a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
        double u[3], w[3];
        for (int x = 0; x < 3; ++x) { u[x] = __dsub_rn(p[3 * b + x], p[3 * a + x]); w[x] = __dsub_rn(p[3 * c + x], p[3 * a + x]); }
        n[0] = __dadd_rn(n[0], __dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1])));
        n[1] = __dadd_rn(n[1], __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2])));
        n[2] = __dadd_rn(n[2], __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0])));
    }
    const double s = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(n[0], n[0]), __dmul_rn(n[1], n[1])), __dmul_rn(n[2], n[2])));
    for (int x = 0; x < 3; ++x) {
        nout[3 * v + x] = s > 0.0 ? (float)__ddiv_rn(n[x], s) : 0.f;
        vout[3 * v + x] = (float)p[3 * v + x];
    }
}

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

int64_t cells_of(int depth) { return (int64_t)1 << (3 * depth); }

bool depth_ok(int depth) { return depth >= 2 && depth <= G2PC_MESH_DEPTH_MAX; }

// ---- workspace layouts: one function per entry point carves the slices; a null base only sizes them ---------------
struct SplatWs {
    float* part;
    unsigned long long* total;
    size_t bytes;
};
SplatWs splat_ws(void* base, int64_t n) {
    const int nb = bbox_blocks(n);
    WsCarve w{(char*)base};
    SplatWs l;
    l.part = w.take<float>((size_t)(nb > 0 ? nb : 1) * 6);
    l.total = w.take<unsigned long long>(1);
    l.bytes = w.used;
    return l;
}

// the coarse levels 1 .. depth - 2 of the multigrid
struct SolveWs {
    float *chi[G2PC_MESH_DEPTH_MAX], *rhs[G2PC_MESH_DEPTH_MAX];
    double* partial;
    size_t bytes;
};
SolveWs solve_ws(void* base, int depth) {
    WsCarve w{(char*)base};
    SolveWs l;
    for (int lv = 1; lv <= depth - 2; ++lv) {
        l.chi[lv] = w.take<float>(cells_of(depth - lv));
        l.rhs[lv] = w.take<float>(cells_of(depth - lv));
    }
    l.partial = w.take<double>(2 * RED_BLOCKS);
    l.bytes = w.used;
    return l;
}

struct ExtractWs {
    long long *vblk, *tblk, *voff, *toff;
    void* tmp;
    size_t tmp_bytes, bytes;
    int64_t nb;
};
ExtractWs extract_ws(void* base, int depth) {
    ExtractWs l;
    l.nb = (cells_of(depth) + NODES_PER_CTA - 1) / NODES_PER_CTA;
    size_t scan_b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const long long*)nullptr, (long long*)nullptr, (int)(l.nb + 1));
    WsCarve w{(char*)base};
    l.vblk = w.take<long long>(l.nb + 1);
    l.tblk = w.take<long long>(l.nb + 1);
    l.voff = w.take<long long>(l.nb + 1);
    l.toff = w.take<long long>(l.nb + 1);
    l.tmp_bytes = WsCarve::pad(scan_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct GatherWs {
    uint32_t *keys_a, *keys_b, *idx_a, *idx_b;
    void* tmp;
    size_t tmp_bytes, bytes;
};
GatherWs gather_ws(void* base, int64_t n) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, 31);
    WsCarve w{(char*)base};
    GatherWs l;
    l.keys_a = w.take<uint32_t>(n);
    l.keys_b = w.take<uint32_t>(n);
    l.idx_a = w.take<uint32_t>(n);
    l.idx_b = w.take<uint32_t>(n);
    l.tmp_bytes = WsCarve::pad(sort_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct TrimWs {
    double* sorted;
    int32_t *vflag, *vmap, *tflag, *tmap;
    void* tmp;
    size_t tmp_bytes, bytes;
};
TrimWs trim_ws(void* base, int64_t m, int64_t t) {
    size_t sort_b = 0, scan_v = 0, scan_t = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const double*)nullptr, (double*)nullptr, (int)m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_v, (const int32_t*)nullptr, (int32_t*)nullptr, (int)m);
    cub::DeviceScan::ExclusiveSum(nullptr, scan_t, (const int32_t*)nullptr, (int32_t*)nullptr, (int)t);
    size_t tb = sort_b > scan_v ? sort_b : scan_v;
    tb = tb > scan_t ? tb : scan_t;
    WsCarve w{(char*)base};
    TrimWs l;
    l.sorted = w.take<double>(m);
    w.take<double>(1);  // unused slot, kept so that the workspace size stays what callers were told
    l.vflag = w.take<int32_t>(m);
    l.vmap = w.take<int32_t>(m);
    l.tflag = w.take<int32_t>(t);
    l.tmap = w.take<int32_t>(t);
    l.tmp_bytes = WsCarve::pad(tb);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

// one-ring (smooth: e = 6t directed edges, with the second position buffer) or incidence (normals: e = 3t) lists
struct ListWs {
    unsigned long long *keys_a, *keys_b;
    int32_t* row;
    double* pos;
    void* tmp;
    size_t tmp_bytes, bytes;
};
ListWs list_ws(void* base, int64_t m, int64_t e, bool pos) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                   (int)e);
    WsCarve w{(char*)base};
    ListWs l;
    l.keys_a = w.take<unsigned long long>(e);
    l.keys_b = w.take<unsigned long long>(e);
    l.row = w.take<int32_t>(m + 1);
    l.pos = w.take<double>(pos ? 3 * m : 0);
    l.tmp_bytes = WsCarve::pad(sort_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

// sort the keys of an e-entry list (from keys_a into keys_b) and bound its rows
int build_lists(const ListWs& l, int64_t m, int64_t e, cudaStream_t st) {
    int end_bit = 33;  // the high word holds a vertex index < m <= 2^31
    while (end_bit < 64 && ((unsigned long long)m >> (end_bit - 32)) != 0) ++end_bit;
    size_t b = l.tmp_bytes;
    if (e > 0) G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, l.keys_a, l.keys_b, (int)e, 0, end_bit, st));
    row_kernel<<<grid_of(m + 1), MB, 0, st>>>(l.keys_b, e, m, l.row);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int64_t g2pc_mesh_splat_workspace_bytes(int64_t n) { return (int64_t)splat_ws(nullptr, n).bytes; }

extern "C" int g2pc_mesh_splat(const float* xyz, const void* normals, int normal_dtype, int64_t n, int32_t depth,
                               double* frame, int64_t* B, uint32_t* cell, int32_t* status, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(normal_dtype == G2PC_F32 || normal_dtype == G2PC_F64, "normals must be float32 or float64");
    G2PC_CHECK_ARG(frame && B && status && workspace, "null pointer");
    G2PC_CHECK_ARG(n == 0 || (xyz && normals && cell), "null pointer");
    const SplatWs l = splat_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    const int R = 1 << depth;
    const int64_t cells = cells_of(depth);
    const int nb = bbox_blocks(n);
    G2PC_CUDA(cudaMemsetAsync(status, 0, 2 * sizeof(int32_t), st));
    G2PC_CUDA(cudaMemsetAsync(B, 0, (size_t)cells * 8, st));
    G2PC_CUDA(cudaMemsetAsync(l.total, 0, 8, st));
    if (n > 0) {
        bbox_kernel<<<nb, BBOX_THREADS, 0, st>>>(xyz, n, l.part);
        G2PC_CHECK_LAUNCH();
    }
    frame_kernel<<<1, 1, 0, st>>>(l.part, nb, R, frame);
    G2PC_CHECK_LAUNCH();
    if (n > 0) {
        unsigned long long* Bu = (unsigned long long*)B;
        if (normal_dtype == G2PC_F32)
            splat_kernel<float><<<grid_of(n), MB, 0, st>>>(xyz, (const float*)normals, n, R, frame, Bu, cell, status);
        else
            splat_kernel<double><<<grid_of(n), MB, 0, st>>>(xyz, (const double*)normals, n, R, frame, Bu, cell, status);
        G2PC_CHECK_LAUNCH();
    }
    sum_b_kernel<<<RED_BLOCKS, MB, 0, st>>>((const long long*)B, cells, l.total);
    G2PC_CHECK_LAUNCH();
    mean_b_kernel<<<1, 1, 0, st>>>(l.total, cells, frame);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_solve_workspace_bytes(int32_t depth) {
    return depth_ok(depth) ? (int64_t)solve_ws(nullptr, depth).bytes : 0;
}

extern "C" int g2pc_mesh_vcycle(const int64_t* B, const double* frame, int32_t depth, float* chi, int32_t first,
                                double* norms, void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(B && frame && chi && norms && workspace, "null pointer");
    const SolveWs l = solve_ws(workspace, depth);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    const int R = 1 << depth, levels = depth - 2;  // level lv has R >> lv cells per axis; the last one has 4
    double* partial = l.partial;
    float* lchi[G2PC_MESH_DEPTH_MAX];
    Rhs lrhs[G2PC_MESH_DEPTH_MAX];
    lchi[0] = chi;
    lrhs[0] = Rhs{(const long long*)B, nullptr, frame};
    for (int lv = 1; lv <= levels; ++lv) {
        lchi[lv] = l.chi[lv];
        lrhs[lv] = Rhs{nullptr, l.rhs[lv], frame};
    }
    const Rhs rhs0 = lrhs[0];
    if (first) {
        G2PC_CUDA(cudaMemsetAsync(chi, 0, (size_t)cells_of(depth) * 4, st));
        grid_partial_kernel<1><<<RED_BLOCKS, MB, 0, st>>>(chi, rhs0, R, partial);
        G2PC_CHECK_LAUNCH();
        finish_kernel<<<1, 1024, 0, st>>>(partial, 1.0, norms + 1);
        G2PC_CHECK_LAUNCH();
    }
    auto smooth = [&](int lv, int sweeps) -> int {
        const int n = R >> lv;
        for (int s = 0; s < sweeps; ++s)
            for (int colour = 0; colour < 2; ++colour) {
                rb_smooth_kernel<<<grid_of((int64_t)n * n * (n / 2)), MB, 0, st>>>(lchi[lv], lrhs[lv], n, colour);
                G2PC_CHECK_LAUNCH();
            }
        return G2PC_OK;
    };
    for (int lv = 0; lv < levels; ++lv) {
        const int n = R >> lv, nc = n >> 1;
        if (smooth(lv, 2)) return G2PC_ERR_CUDA;
        restrict_kernel<<<grid_of((int64_t)nc * nc * nc), MB, 0, st>>>(lchi[lv], lrhs[lv], n, (float*)lrhs[lv + 1].f);
        G2PC_CHECK_LAUNCH();
        G2PC_CUDA(cudaMemsetAsync(lchi[lv + 1], 0, (size_t)nc * nc * nc * 4, st));
    }
    coarse_kernel<<<1, 64, 0, st>>>(lchi[levels], lrhs[levels]);
    G2PC_CHECK_LAUNCH();
    for (int lv = levels - 1; lv >= 0; --lv) {
        const int n = R >> lv;
        prolong_kernel<<<grid_of((int64_t)n * n * n), MB, 0, st>>>(lchi[lv], n, lchi[lv + 1]);
        G2PC_CHECK_LAUNCH();
        if (smooth(lv, 2)) return G2PC_ERR_CUDA;
    }
    grid_partial_kernel<0><<<RED_BLOCKS, MB, 0, st>>>(chi, rhs0, R, partial);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(partial, 1.0, norms);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_iso_workspace_bytes(void) { return (int64_t)(2 * RED_BLOCKS * sizeof(double)); }

extern "C" int g2pc_mesh_iso(const float* xyz, const uint32_t* cell, int64_t n, const double* frame, int32_t depth,
                             float* chi, double* iso, void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(frame && chi && iso && workspace, "null pointer");
    G2PC_CHECK_ARG(n == 0 || (xyz && cell), "null pointer");
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, g2pc_mesh_iso_workspace_bytes(), 8);
    cudaStream_t st = (cudaStream_t)stream;
    double* partial = (double*)workspace;
    const int R = 1 << depth;
    const int64_t cells = cells_of(depth);
    const Rhs none{nullptr, nullptr, frame};
    grid_partial_kernel<2><<<RED_BLOCKS, MB, 0, st>>>(chi, none, R, partial);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(partial, 1.0 / (double)cells, iso);
    G2PC_CHECK_LAUNCH();
    shift_kernel<<<grid_of(cells), MB, 0, st>>>(chi, cells, iso);
    G2PC_CHECK_LAUNCH();
    iso_partial_kernel<<<RED_BLOCKS, MB, 0, st>>>(xyz, cell, n, frame, R, chi, partial);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(partial, 1.0, iso + 1);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(partial + RED_BLOCKS, 1.0, iso + 2);
    G2PC_CHECK_LAUNCH();
    iso_div_kernel<<<1, 1, 0, st>>>(iso);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_extract_workspace_bytes(int32_t depth) {
    return depth_ok(depth) ? (int64_t)extract_ws(nullptr, depth).bytes : 0;
}

extern "C" int g2pc_mesh_extract_count(const float* chi, int32_t depth, const double* iso, int64_t* counts,
                                       void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(chi && iso && counts && workspace, "null pointer");
    const ExtractWs l = extract_ws(workspace, depth);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(l.vblk + l.nb, 0, 8, st));
    G2PC_CUDA(cudaMemsetAsync(l.tblk + l.nb, 0, 8, st));
    mt_count_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, 1 << depth, iso, l.vblk, l.tblk);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.vblk, l.voff, (int)(l.nb + 1), st));
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.tblk, l.toff, (int)(l.nb + 1), st));
    totals_kernel<<<1, 1, 0, st>>>(l.voff, l.toff, l.nb, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_extract_emit(const float* chi, int32_t depth, const double* frame, const double* iso,
                                      void* node_scratch, int64_t node_scratch_bytes, const void* workspace,
                                      int64_t workspace_bytes, int64_t* vkey, double* vt, double* vpos, int32_t* faces,
                                      void* stream) {
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(chi && frame && iso && node_scratch && workspace, "null pointer");
    const ExtractWs l = extract_ws(const_cast<void*>(workspace), depth);  // read only here
    const int64_t cells = cells_of(depth);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    G2PC_CHECK_ARG(node_scratch_bytes >= 5 * cells, "node scratch too small (5 bytes per node)");
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* base = (int32_t*)node_scratch;
    uint8_t* mask = (uint8_t*)node_scratch + 4 * cells;
    const int R = 1 << depth;
    mt_vertex_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, R, frame, iso, l.voff, base, mask, (long long*)vkey, vt, vpos);
    G2PC_CHECK_LAUNCH();
    mt_triangle_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, R, iso, l.toff, base, mask, faces);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_gather_workspace_bytes(int64_t n) { return (int64_t)gather_ws(nullptr, n).bytes; }

extern "C" int g2pc_mesh_gather(const float* xyz, const int32_t* colours, const uint32_t* cell, int64_t n,
                                const double* frame, int32_t depth, const int64_t* vkey, const double* vt, int64_t m,
                                void* cell_scratch, int64_t cell_scratch_bytes, double* density, uint8_t* vcolours,
                                void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll && m >= 0, "bad sizes");
    G2PC_CHECK_ARG(depth_ok(depth), "depth must be in 2..G2PC_MESH_DEPTH_MAX");
    G2PC_CHECK_ARG(frame && cell_scratch && workspace, "null pointer");
    const int R = 1 << depth;
    const int64_t dual = (int64_t)(R - 1) * (R - 1) * (R - 1);
    G2PC_CHECK_ARG(cell_scratch_bytes >= 4 * dual, "cell scratch too small (4 bytes per dual cell)");
    const GatherWs l = gather_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(vkey && vt && density && (n == 0 || (xyz && cell)), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    uint32_t *ka = l.keys_a, *kb = l.keys_b, *ia = l.idx_a, *ib = l.idx_b;
    int32_t* start = (int32_t*)cell_scratch;
    G2PC_CUDA(cudaMemsetAsync(start, 0xFF, (size_t)dual * 4, st));
    if (n > 0) {
        G2PC_CUDA(cudaMemcpyAsync(ka, cell, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        iota_kernel<<<grid_of(n), MB, 0, st>>>(ia, n);
        G2PC_CHECK_LAUNCH();
        size_t b = l.tmp_bytes;  // stable: a cell's points stay in input order
        G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, ka, kb, ia, ib, (int)n, 0, 31, st));
        cell_start_kernel<<<grid_of(n), MB, 0, st>>>(kb, n, start);
        G2PC_CHECK_LAUNCH();
    }
    gather_kernel<<<grid_of(m), MB, 0, st>>>((const long long*)vkey, vt, m, R, kb, ib, n, start, xyz, colours, frame,
                                             density, vcolours);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_trim_workspace_bytes(int64_t m, int64_t t) { return (int64_t)trim_ws(nullptr, m, t).bytes; }

extern "C" int g2pc_mesh_trim(const double* density, const double* vpos, const uint8_t* vcolours, int64_t m,
                              const int32_t* faces, int64_t t, uint8_t* keep, double* threshold, int64_t* counts,
                              double* density_out, double* vpos_out, uint8_t* vcolours_out, int32_t* faces_out,
                              void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(m > 0 && m < 0x7FFFFFFFll && t >= 0 && t < 0x7FFFFFFFll, "need 1..2^31-2 vertices");
    G2PC_CHECK_ARG(density && vpos && keep && threshold && counts && density_out && vpos_out && workspace,
                   "null pointer");
    G2PC_CHECK_ARG(!vcolours == !vcolours_out, "vertex colours need an output");
    G2PC_CHECK_ARG(t == 0 || (faces && faces_out), "null pointer");
    const TrimWs l = trim_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    double* sorted = l.sorted;
    int32_t *vflag = l.vflag, *vmap = l.vmap, *tflag = l.tflag, *tmap = l.tmap;
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, density, sorted, (int)m, 0, 64, st));
    quantile_kernel<<<1, 1, 0, st>>>(sorted, m, threshold);
    G2PC_CHECK_LAUNCH();
    keep_kernel<<<grid_of(m), MB, 0, st>>>(density, m, threshold, keep, vflag);
    G2PC_CHECK_LAUNCH();
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, vflag, vmap, (int)m, st));
    if (t > 0) {
        tri_flag_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, keep, tflag);
        G2PC_CHECK_LAUNCH();
        b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, tflag, tmap, (int)t, st));
        compact_faces_kernel<<<grid_of(t), MB, 0, st>>>(faces, tflag, tmap, t, vmap, faces_out);
        G2PC_CHECK_LAUNCH();
    }
    compact_vertices_kernel<<<grid_of(m), MB, 0, st>>>(keep, vmap, m, density, vpos, vcolours, density_out, vpos_out,
                                                       vcolours_out);
    G2PC_CHECK_LAUNCH();
    trim_counts_kernel<<<1, 1, 0, st>>>(vflag, vmap, m, tflag, tmap, t, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_smooth_workspace_bytes(int64_t m, int64_t t) {
    return (int64_t)list_ws(nullptr, m, 6 * t, true).bytes;
}

extern "C" int g2pc_mesh_smooth(double* vpos, int64_t m, const int32_t* faces, int64_t t, int32_t iterations,
                                void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(m >= 0 && m < 0x7FFFFFFFll && t >= 0 && 6 * t < 0x7FFFFFFFll, "bad sizes");
    G2PC_CHECK_ARG(iterations >= 0, "iterations < 0");
    if (m == 0 || iterations == 0) return G2PC_OK;
    G2PC_CHECK_ARG(vpos && workspace && (t == 0 || faces), "null pointer");
    const ListWs l = list_ws(workspace, m, 6 * t, true);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (t > 0) {
        ring_keys_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.keys_a);
        G2PC_CHECK_LAUNCH();
    }
    if (build_lists(l, m, 6 * t, st)) return G2PC_ERR_CUDA;
    double* src = vpos;
    double* dst = l.pos;
    for (int it = 0; it < iterations; ++it) {
        smooth_kernel<<<grid_of(m), MB, 0, st>>>(src, m, l.keys_b, l.row, dst);
        G2PC_CHECK_LAUNCH();
        double* x = src; src = dst; dst = x;
    }
    if (src != vpos) G2PC_CUDA(cudaMemcpyAsync(vpos, src, (size_t)m * 24, cudaMemcpyDeviceToDevice, st));
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_normals_workspace_bytes(int64_t m, int64_t t) {
    return (int64_t)list_ws(nullptr, m, 3 * t, false).bytes;
}

extern "C" int g2pc_mesh_normals(const double* vpos, int64_t m, const int32_t* faces, int64_t t, float* vertices,
                                 float* normals, void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(m >= 0 && m < 0x7FFFFFFFll && t >= 0 && 3 * t < 0x7FFFFFFFll, "bad sizes");
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(vpos && vertices && normals && workspace && (t == 0 || faces), "null pointer");
    const ListWs l = list_ws(workspace, m, 3 * t, false);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (t > 0) {
        incidence_keys_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.keys_a);
        G2PC_CHECK_LAUNCH();
    }
    if (build_lists(l, m, 3 * t, st)) return G2PC_ERR_CUDA;
    normals_kernel<<<grid_of(m), MB, 0, st>>>(vpos, m, faces, l.keys_b, l.row, vertices, normals);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
