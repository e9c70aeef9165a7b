// mesh_common.cuh — device code the dense Poisson mesher (s10_mesh.cu), its narrow-band levels (s12_mesh_band.cu),
// the decimation (s13_decimate.cu), the component filter (s15_components.cu) and the hole filling (s16_holes.cu) share:
// the frame words, a point's dual cell and trilinear weights, the fixed-order float64 finish step, the
// marching-tetrahedra tables, the stable mesh compaction, the union-find and the one-ring / incidence list builders.
// Every kernel stays in an anonymous namespace.
#pragma once
#include "cloud_common.cuh"

namespace {

constexpr int MB = 256;                         // threads per CTA of the per-point / per-cell kernels
constexpr int RED_BLOCKS = 1024;                // fixed partition of every float64 reduction: bit-identical re-runs
constexpr int NPT = 4;                          // lattice nodes per thread in the extraction kernels
constexpr int NODES_PER_CTA = MB * NPT;
constexpr uint32_t CELL_NONE = 0x7FFFFFFFu;     // dual cell of a point that was not splatted (sorts last)
constexpr double TWO32 = 4294967296.0;

// frame words (float64, device): written by g2pc_mesh_splat
enum { FR_ORIGIN = 0, FR_H = 3, FR_L = 4, FR_MEANB = 5, FR_EXTENT = 6, FR_R = 7 };


struct PointCell {
    int i0[3];
    double f[3];
};

// u = (p - origin) / h - 1/2, i0 = clamp(floor(u), 0, R - 2), f = clamp(u - i0, 0, 1)
__device__ __forceinline__ PointCell point_cell(const float* __restrict__ xyz, int64_t i, const double* __restrict__ fr,
                                                int R) {
    PointCell c;
    const double h = fr[FR_H];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const double u = __dsub_rn(__ddiv_rn(__dsub_rn((double)xyz[3 * i + a], fr[FR_ORIGIN + a]), h), 0.5);
        const double fl = fmin(fmax(floor(u), 0.0), (double)(R - 2));
        c.i0[a] = (int)fl;
        c.f[a] = fmin(fmax(__dsub_rn(u, fl), 0.0), 1.0);
    }
    return c;
}

// weight of dual-cell corner o (bit 0 = x): (wx * wy) * wz with w = f on the upper side, 1 - f on the lower
__device__ __forceinline__ double corner_weight(const PointCell& c, int o) {
    double w[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) w[a] = (o >> a) & 1 ? c.f[a] : __dsub_rn(1.0, c.f[a]);
    return __dmul_rn(__dmul_rn(w[0], w[1]), w[2]);
}

// unit normal of a point in float64; false for a zero or non-finite normal (not splatted)
template <typename NT>
__device__ __forceinline__ bool unit_normal(const NT* __restrict__ nrm, int64_t i, double (&nh)[3]) {
    const double nx = (double)nrm[3 * i], ny = (double)nrm[3 * i + 1], nz = (double)nrm[3 * i + 2];
    const double s = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
    if (!(s > 0.0) || !isfinite(s)) return false;
    nh[0] = __ddiv_rn(nx, s);
    nh[1] = __ddiv_rn(ny, s);
    nh[2] = __ddiv_rn(nz, s);
    return true;
}

// the integer splat term of one (corner weight, normal component): llrint(w * n_a * 2^32)
__device__ __forceinline__ long long splat_q(double w, double na) { return llrint(__dmul_rn(__dmul_rn(w, na), TWO32)); }

__device__ __forceinline__ uint32_t cell_id(const PointCell& c, int R) {
    return ((uint32_t)c.i0[2] * (uint32_t)(R - 1) + (uint32_t)c.i0[1]) * (uint32_t)(R - 1) + (uint32_t)c.i0[0];
}

__device__ __forceinline__ double node_coord(const double* __restrict__ fr, int a, int i) {
    return __dadd_rn(fr[FR_ORIGIN + a], __dmul_rn((double)i + 0.5, fr[FR_H]));
}

// ---- fixed-order float64 reductions -----------------------------------------------------------------------------
// one CTA of 1024 threads: *out = sum of RED_BLOCKS partials (x scale), in a fixed order.  Each thread adds its one
// partial to +0.0, which changes nothing: a partial comes from block_sum_f64, which starts at +0.0, so it is never -0.0.
__global__ void __launch_bounds__(1024) finish_kernel(const double* __restrict__ partial, double scale,
                                                      double* __restrict__ out) {
    __shared__ double s[1024];
    const double t = sum_partials_f64(partial, RED_BLOCKS, s);
    if (threadIdx.x == 0) *out = __dmul_rn(t, scale);
}

// ---- marching tetrahedra --------------------------------------------------------------------------------------------
// inside / in-grid bits of the 8 corners P + {0,1}^3 (bit o: x = o & 1, y = o >> 1 & 1, z = o >> 2)
struct Cube {
    uint32_t inside, valid;
};

// bit d (1..7) set iff the lattice edge (P, P + d) exists and crosses the surface
__device__ __forceinline__ uint32_t cross_mask(Cube c) {
    uint32_t m = 0;
    const uint32_t in0 = c.inside & 1u;
#pragma unroll
    for (int d = 1; d < 8; ++d)
        if (((c.valid >> d) & 1u) && ((c.inside >> d) & 1u) != in0) m |= 1u << d;
    return m;
}

// corner (bitmask) q of Kuhn tetrahedron p: 0, e_a, e_a + e_b, 1 for the p-th axis permutation (a, b, c) in
// lexicographic order
__device__ __forceinline__ int tet_corner(int p, int q) {
    const int a = p >> 1;
    const int r0 = a == 0 ? 1 : 0, r1 = a == 2 ? 1 : 2;
    const int b = (p & 1) ? r1 : r0;
    return q == 0 ? 0 : (q == 1 ? 1 << a : (q == 2 ? (1 << a) | (1 << b) : 7));
}

__device__ __forceinline__ int tet_triangle_count(int p, uint32_t inside) {
    int ni = 0;
    for (int q = 0; q < 4; ++q) ni += (inside >> tet_corner(p, q)) & 1;
    return ni == 2 ? 2 : (ni == 1 || ni == 3 ? 1 : 0);
}

__device__ __forceinline__ int cube_triangle_count(uint32_t inside) {
    int t = 0;
    for (int p = 0; p < 6; ++p) t += tet_triangle_count(p, inside);
    return t;
}

// The triangles of tetrahedron p: edges as (lower corner, upper corner) bitmask pairs.  One inside corner I or one
// outside corner O: one triangle over the three edges of that corner; two and two (inside I0 < I1, outside O0 < O1,
// tetrahedron-local order): the quad I0O0, I0O1, I1O1, I1O0 split along I0O0-I1O1.  Each triangle is wound
// counter-clockwise seen from the outside (chi >= iso): the normal of the triangle of the edge midpoints must point from
// an inside to an outside corner, else its last two edges swap.  Integer arithmetic (doubled midpoints): exact.
__device__ __forceinline__ int tet_triangles(int p, uint32_t inside, int (&tri)[2][3][2]) {
    int v[4], I[4], O[4], ni = 0, no = 0;
    for (int q = 0; q < 4; ++q) {
        v[q] = tet_corner(p, q);
        if ((inside >> v[q]) & 1) I[ni++] = q; else O[no++] = q;
    }
    int e[2][3][2], nt;  // tetrahedron-local vertex pairs
    if (ni == 1 || ni == 3) {
        const int apex = ni == 1 ? I[0] : O[0];
        const int* other = ni == 1 ? O : I;
        for (int s = 0; s < 3; ++s) { e[0][s][0] = apex; e[0][s][1] = other[s]; }
        nt = 1;
    } else if (ni == 2) {
        const int q[2][3][2] = {{{I[0], O[0]}, {I[0], O[1]}, {I[1], O[1]}}, {{I[0], O[0]}, {I[1], O[1]}, {I[1], O[0]}}};
        for (int t = 0; t < 2; ++t)
            for (int s = 0; s < 3; ++s) { e[t][s][0] = q[t][s][0]; e[t][s][1] = q[t][s][1]; }
        nt = 2;
    } else {
        return 0;
    }
    const int din[3] = {v[O[0]] & 1, (v[O[0]] >> 1) & 1, v[O[0]] >> 2};
    const int dio[3] = {din[0] - (v[I[0]] & 1), din[1] - ((v[I[0]] >> 1) & 1), din[2] - (v[I[0]] >> 2)};
    for (int t = 0; t < nt; ++t) {
        int M[3][3];
        for (int s = 0; s < 3; ++s) {
            const int a = v[e[t][s][0]], b = v[e[t][s][1]];
            for (int x = 0; x < 3; ++x) M[s][x] = ((a >> x) & 1) + ((b >> x) & 1);
        }
        const int u[3] = {M[1][0] - M[0][0], M[1][1] - M[0][1], M[1][2] - M[0][2]};
        const int w[3] = {M[2][0] - M[0][0], M[2][1] - M[0][1], M[2][2] - M[0][2]};
        const int N[3] = {u[1] * w[2] - u[2] * w[1], u[2] * w[0] - u[0] * w[2], u[0] * w[1] - u[1] * w[0]};
        const bool flip = N[0] * dio[0] + N[1] * dio[1] + N[2] * dio[2] < 0;
        for (int s = 0; s < 3; ++s) {
            const int src = flip && s > 0 ? 3 - s : s;
            const int a = v[e[t][src][0]], b = v[e[t][src][1]];
            // corners of a tetrahedron are nested bitmasks: the smaller one is the lower end of the lattice edge
            tri[t][s][0] = a < b ? a : b;
            tri[t][s][1] = a < b ? b : a;
        }
    }
    return nt;
}

// ---- stable compaction of a mesh by vertex keep flags (density trim in s10_mesh.cu, s15_components.cu) ---------------
// a triangle is kept iff its three vertices are; vmap / fmap are the exclusive scans of the vertex / triangle flags
__global__ void __launch_bounds__(MB) tri_flag_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                      const uint8_t* __restrict__ keep, int32_t* __restrict__ flag) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    flag[f] = keep[faces[3 * f]] & keep[faces[3 * f + 1]] & keep[faces[3 * f + 2]];
}

__global__ void __launch_bounds__(MB) compact_vertices_kernel(const uint8_t* __restrict__ keep,
                                                              const int32_t* __restrict__ vmap, int64_t m,
                                                              const double* __restrict__ dens,
                                                              const double* __restrict__ vpos,
                                                              const uint8_t* __restrict__ vcol, double* __restrict__ dens_o,
                                                              double* __restrict__ vpos_o, uint8_t* __restrict__ vcol_o) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || !keep[v]) return;
    const int64_t o = vmap[v];
    dens_o[o] = dens[v];
    for (int a = 0; a < 3; ++a) vpos_o[3 * o + a] = vpos[3 * v + a];
    if (vcol)
        for (int a = 0; a < 3; ++a) vcol_o[3 * o + a] = vcol[3 * v + a];
}

__global__ void __launch_bounds__(MB) compact_faces_kernel(const int32_t* __restrict__ faces, const int32_t* __restrict__ flag,
                                                           const int32_t* __restrict__ fmap, int64_t t,
                                                           const int32_t* __restrict__ vmap, int32_t* __restrict__ faces_o) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t || !flag[f]) return;
    const int64_t o = fmap[f];
    for (int s = 0; s < 3; ++s) faces_o[3 * o + s] = vmap[faces[3 * f + s]];
}

__global__ void trim_counts_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ map, int64_t m,
                                   const int32_t* __restrict__ tflag, const int32_t* __restrict__ tmap, int64_t t,
                                   long long* __restrict__ counts) {
    counts[0] = m ? (long long)map[m - 1] + flag[m - 1] : 0;
    counts[1] = t ? (long long)tmap[t - 1] + tflag[t - 1] : 0;
}

// ---- concurrent union-find whose roots are their sets' smallest vertices (s15_components.cu, s16_holes.cu) ----------
// Every read of a parent pointer goes to memory (volatile): a value cached in a register across iterations could be
// stale.  Writes are atomics.
__device__ __forceinline__ int parent_of(const int32_t* parent, int x) { return ((const volatile int32_t*)parent)[x]; }

// The root of x's set as seen now.  Path halving: x's pointer moves to its grandparent, an ancestor below its parent.
__device__ int find_root(int32_t* parent, int x) {
    while (true) {
        const int p = parent_of(parent, x);
        if (p == x) return x;
        const int g = parent_of(parent, p);
        if (g == p) return p;
        atomicMin(&parent[x], g);
        x = g;
    }
}

// Joins the sets of a and b: the larger root is hooked under the smaller one when it is still a root, else the union
// retries from the root it was hooked under meanwhile.
__device__ void unite(int32_t* parent, int a, int b) {
    while (true) {
        a = find_root(parent, a);
        b = find_root(parent, b);
        if (a == b) return;
        const int hi = a > b ? a : b, lo = a > b ? b : a;
        const int old = atomicCAS(&parent[hi], hi, lo);
        if (old == hi) return;
        a = old;
        b = lo;
    }
}

__global__ void __launch_bounds__(MB) parent_init_kernel(int32_t* __restrict__ parent, int64_t m) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v < m) parent[v] = (int32_t)v;
}

// after every union: parent[v] = the root of v (its label)
__global__ void __launch_bounds__(MB) compress_kernel(int32_t* parent, int64_t m) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int r = find_root(parent, (int)v);
    atomicMin(&parent[v], r);
}

// ---- one-ring / incidence lists of a triangle mesh (smoothing and normals in s10_mesh.cu, s13_decimate.cu) --------
// directed one-ring edges (u << 32 | v), both directions of every triangle edge
__global__ void __launch_bounds__(MB) ring_keys_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                       unsigned long long* __restrict__ keys) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    for (int s = 0; s < 3; ++s) {
        const unsigned long long a = (uint32_t)faces[3 * f + s], b = (uint32_t)faces[3 * f + (s + 1) % 3];
        keys[6 * f + 2 * s] = a << 32 | b;
        keys[6 * f + 2 * s + 1] = b << 32 | a;
    }
}

// incident triangles (v << 32 | triangle)
__global__ void __launch_bounds__(MB) incidence_keys_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                            unsigned long long* __restrict__ keys) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    for (int s = 0; s < 3; ++s) keys[3 * f + s] = (unsigned long long)(uint32_t)faces[3 * f + s] << 32 | (uint64_t)f;
}

// row[v] = first sorted key with high word >= v, for v = 0..m
__global__ void __launch_bounds__(MB) row_kernel(const unsigned long long* __restrict__ keys, int64_t e, int64_t m,
                                                 int32_t* __restrict__ row) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v > m) return;
    const unsigned long long K = (unsigned long long)v << 32;
    int64_t lo = 0, hi = e;
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (keys[mid] < K) lo = mid + 1; else hi = mid;
    }
    row[v] = (int32_t)lo;
}

}  // namespace
