// s12_mesh_band.cu — narrow-band levels of the Poisson mesher (DESIGN.md §2, N6b): the finest one or two levels above
// the dense solve, stored only in 8^3-node bricks around the points.  Brick map and list, band splat, ghosts and initial
// guess prolonged from the level below, a Jacobi-preconditioned conjugate-gradient solve, iso-value, marching
// tetrahedra over the fully active cubes, and the density / colour gather.  tests/f64ref_mesh_band.py restates every
// rule in float64.
//
// Level D: R = 2^D nodes per axis, h = L / R with the dense level's origin and L.  Brick b = (i >> 3, j >> 3, k >> 3),
// NB = R / 8 bricks per axis, linear brick index (bz NB + by) NB + bx.  map[b] = slot of an active brick or -1; slots
// number the active bricks in ascending brick index; node storage slot * 512 + ((lz * 8 + ly) * 8 + lx) (int64).
// The band operator is the dense one, (sum of the in-grid neighbours - their count x chi); a neighbour outside the band
// (a ghost) has the fixed value s P(chi of the level below), s = 1/8, P the node-centred trilinear prolongation.
#include <cub/cub.cuh>
#include "mesh_common.cuh"

namespace {

constexpr int BRICK = G2PC_MESH_BRICK;
constexpr int BRICK_NODES = BRICK * BRICK * BRICK;
constexpr int MARGIN = G2PC_MESH_BAND_MARGIN;
constexpr double GHOST_SCALE = 0.125;  // chi scales as h^3 (DESIGN.md §2, N6b rule 4)
constexpr uint64_t CELL64_NONE = ~0ull;

// scalars of the conjugate-gradient solve (float64, device)
enum { CG_CC = 0, CG_PQ = 1, CG_RR = 2, CG_RZ = 3, CG_WORDS = 5 };  // CG_RZ + parity: r.z of the two last iterations

bool band_depth_ok(int depth) { return depth >= 3 && depth <= G2PC_MESH_BAND_DEPTH_MAX; }

int64_t nb3(int depth) { return (int64_t)1 << (3 * (depth - 3)); }

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

// storage index of in-grid node (i, j, k), or -1 when its brick is not active.  map == nullptr: a dense level
__device__ __forceinline__ int64_t band_node(const int32_t* __restrict__ map, int R, int i, int j, int k) {
    if (!map) return ((int64_t)k * R + j) * R + i;
    const int NB = R / BRICK;
    const int32_t s = map[((int64_t)(k >> 3) * NB + (j >> 3)) * NB + (i >> 3)];
    if (s < 0) return -1;
    return (int64_t)s * BRICK_NODES + (((k & 7) * BRICK + (j & 7)) * BRICK + (i & 7));
}

// global (i, j, k) of storage index u
__device__ __forceinline__ void band_ijk(const int32_t* __restrict__ list, int R, int64_t u, int& i, int& j, int& k) {
    const int NB = R / BRICK;
    const int64_t b = list[u / BRICK_NODES];
    const int l = (int)(u % BRICK_NODES);
    i = (int)(b % NB) * BRICK + (l & 7);
    j = (int)((b / NB) % NB) * BRICK + ((l >> 3) & 7);
    k = (int)(b / ((int64_t)NB * NB)) * BRICK + (l >> 6);
}

// s P(chi_c)(fine node i, j, k): per axis the coarse nodes lo = i >> 1 (weight 3/4) and lo +- 1 towards i (1/4),
// clamped to the grid; corners o = 0..7 (bit a set: the 1/4 node on axis a), w = (wx * wy) * wz, summed in order o,
// then times s.  Every coarse node read must be active (the nesting rule guarantees it).
__device__ __forceinline__ double prolong(const float* __restrict__ chi_c, const int32_t* __restrict__ map_c, int Rc,
                                          int i, int j, int k) {
    const int p[3] = {i, j, k};
    int lo[3], hi[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        lo[a] = p[a] >> 1;
        const int q = lo[a] + ((p[a] & 1) ? 1 : -1);
        hi[a] = q < 0 ? 0 : (q > Rc - 1 ? Rc - 1 : q);
    }
    double v = 0.0;
    for (int o = 0; o < 8; ++o) {
        const int x = (o & 1) ? hi[0] : lo[0], y = (o & 2) ? hi[1] : lo[1], z = (o & 4) ? hi[2] : lo[2];
        const double w = __dmul_rn(__dmul_rn((o & 1) ? 0.25 : 0.75, (o & 2) ? 0.25 : 0.75), (o & 4) ? 0.25 : 0.75);
        v = __dadd_rn(v, __dmul_rn(w, (double)chi_c[band_node(map_c, Rc, x, y, z)]));
    }
    return __dmul_rn(GHOST_SCALE, v);
}

// ---- bricks -----------------------------------------------------------------------------------------------------
// band frame: the dense frame with h = L / R and R of level D
__global__ void band_frame_kernel(const double* __restrict__ fr, int R, double* __restrict__ bf) {
    for (int w = 0; w < G2PC_MESH_FRAME_WORDS; ++w) bf[w] = fr[w];
    bf[FR_H] = __ddiv_rn(fr[FR_L], (double)R);
    bf[FR_R] = (double)R;
}

// seed bricks: the brick of every node the splat writes for a splatted point (the 8 dual-cell corners, each +- e_a
// inside the grid)
__global__ void __launch_bounds__(MB) seed_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ cell,
                                                  int64_t n, const double* __restrict__ bf, int R,
                                                  uint8_t* __restrict__ seed) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= n || cell[i] == CELL_NONE) return;
    const PointCell c = point_cell(xyz, i, bf, R);
    const int NB = R / BRICK;
    for (int o = 0; o < 8; ++o) {
        const int cc[3] = {c.i0[0] + (o & 1), c.i0[1] + ((o >> 1) & 1), c.i0[2] + (o >> 2)};
        for (int a = 0; a < 3; ++a)
            for (int s = -1; s <= 1; s += 2) {
                int q[3] = {cc[0], cc[1], cc[2]};
                q[a] += s;
                if (q[a] < 0 || q[a] > R - 1) continue;
                seed[((int64_t)(q[2] >> 3) * NB + (q[1] >> 3)) * NB + (q[0] >> 3)] = 1;
            }
    }
}

// keep[b] = 1 iff brick b is within MARGIN bricks of a seed brick and nested in the level below: every coarse node
// 4 b - 1 .. 4 b + 4 (clamped) on every axis, which holds the prolongation stencils of the brick and its one-node halo,
// is active there.  A seed brick that fails the nesting test is counted in *lost.
__global__ void __launch_bounds__(MB) keep_kernel(const uint8_t* __restrict__ seed, int NB,
                                                  const int32_t* __restrict__ map_c, int32_t* __restrict__ keep,
                                                  unsigned long long* __restrict__ lost) {
    const int64_t b = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (b >= (int64_t)NB * NB * NB) return;
    const int p[3] = {(int)(b % NB), (int)((b / NB) % NB), (int)(b / ((int64_t)NB * NB))};
    bool near = false;
    for (int dz = -MARGIN; dz <= MARGIN && !near; ++dz)
        for (int dy = -MARGIN; dy <= MARGIN && !near; ++dy)
            for (int dx = -MARGIN; dx <= MARGIN; ++dx) {
                const int x = p[0] + dx, y = p[1] + dy, z = p[2] + dz;
                if (x < 0 || y < 0 || z < 0 || x >= NB || y >= NB || z >= NB) continue;
                if (seed[((int64_t)z * NB + y) * NB + x]) { near = true; break; }
            }
    bool nested = true;
    if (near && map_c) {
        const int NBc = NB / 2, Rc = NBc * BRICK;  // the coarse level has half the nodes per axis
        int lo[3], hi[3];
        for (int a = 0; a < 3; ++a) {
            lo[a] = max(4 * p[a] - 1, 0) / BRICK;
            hi[a] = min(4 * p[a] + 4, Rc - 1) / BRICK;
        }
        for (int z = lo[2]; z <= hi[2]; ++z)
            for (int y = lo[1]; y <= hi[1]; ++y)
                for (int x = lo[0]; x <= hi[0]; ++x)
                    if (map_c[((int64_t)z * NBc + y) * NBc + x] < 0) nested = false;
    }
    keep[b] = near && nested ? 1 : 0;
    if (seed[b] && !nested) atomicAdd(lost, 1ull);
}

// map[b] = slot or -1; counts[0] = active bricks
__global__ void __launch_bounds__(MB) map_kernel(const int32_t* __restrict__ keep, const int32_t* __restrict__ scan,
                                                 int64_t nb, int32_t* __restrict__ map, long long* __restrict__ counts,
                                                 const unsigned long long* __restrict__ lost) {
    const int64_t b = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (b >= nb) return;
    map[b] = keep[b] ? scan[b] : -1;
    if (b == nb - 1) {
        counts[0] = (long long)scan[b] + keep[b];
        counts[1] = (long long)*lost;
    }
}

__global__ void __launch_bounds__(MB) list_kernel(const int32_t* __restrict__ map, int64_t nb, int32_t* __restrict__ list) {
    const int64_t b = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (b < nb && map[b] >= 0) list[map[b]] = (int32_t)b;
}

// ---- band splat ---------------------------------------------------------------------------------------------------
// the dense splat's integer terms at level D, added at the band storage of their nodes (all active: they are seeds)
template <typename NT>
__global__ void __launch_bounds__(MB) band_splat_kernel(const float* __restrict__ xyz, const NT* __restrict__ nrm,
                                                        const uint32_t* __restrict__ cell, int64_t n, int R,
                                                        const double* __restrict__ bf, const int32_t* __restrict__ map,
                                                        unsigned long long* __restrict__ B, int32_t* __restrict__ status) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= n || cell[i] == CELL_NONE) return;
    double nh[3];
    if (!unit_normal(nrm, i, nh)) return;
    const PointCell c = point_cell(xyz, i, bf, R);
    for (int o = 0; o < 8; ++o) {
        const double w = corner_weight(c, o);
        const int cc[3] = {c.i0[0] + (o & 1), c.i0[1] + ((o >> 1) & 1), c.i0[2] + (o >> 2)};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const long long q = splat_q(w, nh[a]);
            if (q == 0) continue;
            for (int s = -1; s <= 1; s += 2) {
                int x[3] = {cc[0], cc[1], cc[2]};
                x[a] += s;
                if (x[a] < 0 || x[a] > R - 1) continue;
                const int64_t u = band_node(map, R, x[0], x[1], x[2]);
                if (u < 0) { atomicAdd(status, 1); continue; }
                atomicAdd(&B[u], (unsigned long long)(s < 0 ? q : -q));
            }
        }
    }
}

// ---- ghosts, initial guess, right-hand side ---------------------------------------------------------------------
// per active node: g = sum of s P(chi_c) over its in-grid inactive neighbours (-x, +x, -y, +y, -z, +z in order),
// chi = s P(chi_c) at the node, c = (float)(g - b) with b = B h 2^-33 (the conjugate-gradient right-hand side of the
// positive definite form: count x chi - sum of the active neighbours = g - b)
__global__ void __launch_bounds__(MB) ghost_kernel(const float* __restrict__ chi_c, const int32_t* __restrict__ map_c,
                                                   int R, const int32_t* __restrict__ map,
                                                   const int32_t* __restrict__ list, int64_t nodes,
                                                   const long long* __restrict__ B, const double* __restrict__ bf,
                                                   double* __restrict__ ghost, float* __restrict__ chi,
                                                   float* __restrict__ c) {
    const int64_t u = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (u >= nodes) return;
    int i, j, k;
    band_ijk(list, R, u, i, j, k);
    const int Rc = R / 2;
    double g = 0.0;
    for (int e = 0; e < 6; ++e) {
        int x[3] = {i, j, k};
        x[e >> 1] += (e & 1) ? 1 : -1;
        if (x[e >> 1] < 0 || x[e >> 1] > R - 1) continue;
        if (band_node(map, R, x[0], x[1], x[2]) >= 0) continue;
        g = __dadd_rn(g, prolong(chi_c, map_c, Rc, x[0], x[1], x[2]));
    }
    if (ghost) ghost[u] = g;
    chi[u] = (float)prolong(chi_c, map_c, Rc, i, j, k);
    const double b = __dmul_rn((double)B[u], __dmul_rn(bf[FR_H], 0x1p-33));
    c[u] = (float)__dsub_rn(g, b);
}

// ---- conjugate gradients on M chi = c, M = count x chi - sum of the active in-grid neighbours ------------------------
// (M x)[u] in float64 and the in-grid neighbour count
__device__ __forceinline__ double apply_m(const float* __restrict__ x, const int32_t* __restrict__ map,
                                          const int32_t* __restrict__ list, int R, int64_t u, int& cnt) {
    int i, j, k;
    band_ijk(list, R, u, i, j, k);
    double s = 0.0;
    cnt = 0;
    for (int e = 0; e < 6; ++e) {
        int p[3] = {i, j, k};
        p[e >> 1] += (e & 1) ? 1 : -1;
        if (p[e >> 1] < 0 || p[e >> 1] > R - 1) continue;
        ++cnt;
        const int64_t v = band_node(map, R, p[0], p[1], p[2]);
        if (v >= 0) s = __dadd_rn(s, (double)x[v]);
    }
    return __dsub_rn(__dmul_rn((double)cnt, (double)x[u]), s);
}

__device__ __forceinline__ int grid_count(const int32_t* __restrict__ list, int R, int64_t u) {
    int i, j, k;
    band_ijk(list, R, u, i, j, k);
    return 6 - (i == 0) - (i == R - 1) - (j == 0) - (j == R - 1) - (k == 0) - (k == R - 1);
}

// three fixed-order partial sums per CTA (RED_BLOCKS CTAs, grid-stride)
__device__ __forceinline__ void write_partials(double v0, double v1, double v2, double* s_w, double* __restrict__ part) {
    const double t0 = block_sum_f64<MB>(v0, s_w);
    __syncthreads();
    const double t1 = block_sum_f64<MB>(v1, s_w);
    __syncthreads();
    const double t2 = block_sum_f64<MB>(v2, s_w);
    if (threadIdx.x == 0) {
        part[blockIdx.x] = t0;
        part[RED_BLOCKS + blockIdx.x] = t1;
        part[2 * RED_BLOCKS + blockIdx.x] = t2;
    }
}

// r = c - M chi, z = r / count, p = z; partial sums of r.r, r.z, c.c
__global__ void __launch_bounds__(MB) cg_init_kernel(const float* __restrict__ chi, const float* __restrict__ c,
                                                     const int32_t* __restrict__ map, const int32_t* __restrict__ list,
                                                     int R, int64_t nodes, float* __restrict__ r, float* __restrict__ p,
                                                     double* __restrict__ part) {
    __shared__ double s_w[MB / 32];
    double rr = 0.0, rz = 0.0, cc = 0.0;
    for (int64_t u = (int64_t)blockIdx.x * MB + threadIdx.x; u < nodes; u += (int64_t)RED_BLOCKS * MB) {
        int cnt;
        const double mx = apply_m(chi, map, list, R, u, cnt);
        const float rv = (float)__dsub_rn((double)c[u], mx);
        const float zv = rv / (float)cnt;
        r[u] = rv;
        p[u] = zv;
        rr = __dadd_rn(rr, __dmul_rn((double)rv, (double)rv));
        rz = __dadd_rn(rz, __dmul_rn((double)rv, (double)zv));
        cc = __dadd_rn(cc, __dmul_rn((double)c[u], (double)c[u]));
    }
    write_partials(rr, rz, cc, s_w, part);
}

// q = M p; partial sums of p.q
__global__ void __launch_bounds__(MB) cg_apply_kernel(const float* __restrict__ p, const int32_t* __restrict__ map,
                                                      const int32_t* __restrict__ list, int R, int64_t nodes,
                                                      float* __restrict__ q, double* __restrict__ part) {
    __shared__ double s_w[MB / 32];
    double pq = 0.0;
    for (int64_t u = (int64_t)blockIdx.x * MB + threadIdx.x; u < nodes; u += (int64_t)RED_BLOCKS * MB) {
        int cnt;
        const float qv = (float)apply_m(p, map, list, R, u, cnt);
        q[u] = qv;
        pq = __dadd_rn(pq, __dmul_rn((double)p[u], (double)qv));
    }
    const double t = block_sum_f64<MB>(pq, s_w);
    if (threadIdx.x == 0) part[blockIdx.x] = t;
}

// alpha = r.z / p.q; chi += alpha p, r -= alpha q; partial sums of r.r and r.z (z = r / count)
__global__ void __launch_bounds__(MB) cg_update_kernel(float* __restrict__ chi, float* __restrict__ r,
                                                       const float* __restrict__ p, const float* __restrict__ q,
                                                       const int32_t* __restrict__ list, int R, int64_t nodes,
                                                       const double* __restrict__ sc, int par,
                                                       double* __restrict__ part) {
    __shared__ double s_w[MB / 32];
    const double pq = sc[CG_PQ];
    const float alpha = pq > 0.0 ? (float)__ddiv_rn(sc[CG_RZ + par], pq) : 0.f;
    double rr = 0.0, rz = 0.0;
    for (int64_t u = (int64_t)blockIdx.x * MB + threadIdx.x; u < nodes; u += (int64_t)RED_BLOCKS * MB) {
        chi[u] += alpha * p[u];
        const float rv = r[u] - alpha * q[u];
        r[u] = rv;
        const float zv = rv / (float)grid_count(list, R, u);
        rr = __dadd_rn(rr, __dmul_rn((double)rv, (double)rv));
        rz = __dadd_rn(rz, __dmul_rn((double)rv, (double)zv));
    }
    write_partials(rr, rz, 0.0, s_w, part);
}

// beta = r.z (new) / r.z (old); p = z + beta p
__global__ void __launch_bounds__(MB) cg_direction_kernel(float* __restrict__ p, const float* __restrict__ r,
                                                          const int32_t* __restrict__ list, int R, int64_t nodes,
                                                          const double* __restrict__ sc, int par) {
    const int64_t u = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (u >= nodes) return;
    const double old = sc[CG_RZ + par];
    const float beta = old > 0.0 ? (float)__ddiv_rn(sc[CG_RZ + (par ^ 1)], old) : 0.f;
    p[u] = r[u] / (float)grid_count(list, R, u) + beta * p[u];
}

// ---- iso ------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MB) band_iso_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ cell,
                                                      int64_t n, const double* __restrict__ bf, int R,
                                                      const int32_t* __restrict__ map, const float* __restrict__ chi,
                                                      double* __restrict__ part) {
    __shared__ double s_w[MB / 32];
    double v = 0.0, cnt = 0.0;
    for (int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x; i < n; i += (int64_t)RED_BLOCKS * MB) {
        if (cell[i] == CELL_NONE) continue;
        const PointCell c = point_cell(xyz, i, bf, R);
        double x = 0.0;
        for (int o = 0; o < 8; ++o) {
            const int64_t u = band_node(map, R, c.i0[0] + (o & 1), c.i0[1] + ((o >> 1) & 1), c.i0[2] + (o >> 2));
            x = __dadd_rn(x, __dmul_rn(corner_weight(c, o), (double)chi[u]));
        }
        v = __dadd_rn(v, x);
        cnt += 1.0;
    }
    const double tv = block_sum_f64<MB>(v, s_w);
    __syncthreads();
    const double tc = block_sum_f64<MB>(cnt, s_w);
    if (threadIdx.x == 0) { part[blockIdx.x] = tv; part[RED_BLOCKS + blockIdx.x] = tc; }
}

__global__ void band_iso_div_kernel(double* __restrict__ iso) {
    iso[0] = 0.0;
    iso[1] = iso[2] > 0.0 ? __ddiv_rn(iso[1], iso[2]) : 0.0;
}

// ---- marching tetrahedra over the covered cubes ---------------------------------------------------------------------
// Node Q's view of the band: vmask bit d (1..7) iff the edge (Q, Q + d) crosses the surface and lies in a covered cube
// (one whose 8 corners are active: the cubes Q - lo with lo & d == 0 hold the edge); cube = inside bits of the cube
// with lowest corner Q, valid iff that cube is covered.
struct BandNode {
    uint32_t vmask, inside;
    bool covered;
};

__device__ __forceinline__ BandNode band_view(const float* __restrict__ chi, const int32_t* __restrict__ map, int R,
                                              int i, int j, int k, double iso) {
    uint32_t act = 0;  // bit (dz + 1) * 9 + (dy + 1) * 3 + dx + 1 of the 27 nodes around Q
    uint32_t inside = 0;
    for (int t = 0; t < 27; ++t) {
        const int x = i + t % 3 - 1, y = j + (t / 3) % 3 - 1, z = k + t / 9 - 1;
        if (x < 0 || y < 0 || z < 0 || x > R - 1 || y > R - 1 || z > R - 1) continue;
        const int64_t v = band_node(map, R, x, y, z);
        if (v < 0) continue;
        act |= 1u << t;
        if (t % 3 >= 1 && (t / 3) % 3 >= 1 && t / 9 >= 1 && (double)chi[v] < iso)
            inside |= 1u << ((t % 3 - 1) | ((t / 3) % 3 - 1) << 1 | (t / 9 - 1) << 2);
    }
    uint32_t cov = 0;  // bit lo: cube Q - lo covered
    for (int lo = 0; lo < 8; ++lo) {
        bool all = true;
        for (int o = 0; o < 8; ++o) {
            const int dx = (o & 1) - (lo & 1), dy = ((o >> 1) & 1) - ((lo >> 1) & 1), dz = (o >> 2) - (lo >> 2);
            if (!((act >> ((dz + 1) * 9 + (dy + 1) * 3 + dx + 1)) & 1u)) { all = false; break; }
        }
        if (all) cov |= 1u << lo;
    }
    BandNode b{0u, inside, (cov & 1u) != 0};
    const uint32_t in0 = inside & 1u;
    for (int d = 1; d < 8; ++d) {
        uint32_t held = 0;
        for (int lo = 0; lo < 8; ++lo)
            if (!(lo & d)) held |= (cov >> lo) & 1u;
        if (held && ((inside >> d) & 1u) != in0) b.vmask |= 1u << d;
    }
    return b;
}

__global__ void __launch_bounds__(MB) band_count_kernel(const float* __restrict__ chi, int R,
                                                        const int32_t* __restrict__ map,
                                                        const int32_t* __restrict__ list, int64_t nodes,
                                                        const double* __restrict__ iso2, long long* __restrict__ vblk,
                                                        long long* __restrict__ tblk) {
    __shared__ double s_w[MB / 32];
    const double iso = iso2[1];
    int nv = 0, nt = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t u = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        if (u >= nodes) break;
        int i, j, k;
        band_ijk(list, R, u, i, j, k);
        const BandNode b = band_view(chi, map, R, i, j, k, iso);
        nv += __popc(b.vmask);
        if (b.covered) nt += cube_triangle_count(b.inside);
    }
    const double sv = block_sum_f64<MB>((double)nv, s_w);
    __syncthreads();
    const double st = block_sum_f64<MB>((double)nt, s_w);
    if (threadIdx.x == 0) { vblk[blockIdx.x] = (long long)sv; tblk[blockIdx.x] = (long long)st; }
}

__global__ void band_totals_kernel(const long long* __restrict__ voff, const long long* __restrict__ toff, int64_t nb,
                                   long long* __restrict__ counts) {
    counts[0] = voff[nb];
    counts[1] = toff[nb];
}

// vertices in ascending (storage index, d); key = global node * 8 + d
__global__ void __launch_bounds__(MB) band_vertex_kernel(const float* __restrict__ chi, int R,
                                                         const int32_t* __restrict__ map,
                                                         const int32_t* __restrict__ list, int64_t nodes,
                                                         const double* __restrict__ bf, const double* __restrict__ iso2,
                                                         const long long* __restrict__ voff,
                                                         int32_t* __restrict__ node_base, uint8_t* __restrict__ node_mask,
                                                         long long* __restrict__ vkey, double* __restrict__ vt,
                                                         double* __restrict__ vpos) {
    typedef cub::BlockScan<int, MB> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const double iso = iso2[1];
    uint32_t m[NPT];
    int nv = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t u = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        m[q] = 0;
        if (u >= nodes) continue;
        int i, j, k;
        band_ijk(list, R, u, i, j, k);
        m[q] = band_view(chi, map, R, i, j, k, iso).vmask;
        nv += __popc(m[q]);
    }
    int pre;
    Scan(tmp).ExclusiveSum(nv, pre);
    long long cur = voff[blockIdx.x] + pre;
    for (int q = 0; q < NPT; ++q) {
        const int64_t u = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        if (u >= nodes) break;
        node_base[u] = (int32_t)cur;
        node_mask[u] = (uint8_t)m[q];
        if (!m[q]) continue;
        int i, j, k;
        band_ijk(list, R, u, i, j, k);
        const int64_t node = ((int64_t)k * R + j) * R + i;
        const double ca = (double)chi[u];
        const double pa[3] = {node_coord(bf, 0, i), node_coord(bf, 1, j), node_coord(bf, 2, k)};
        for (int d = 1; d < 8; ++d) {
            if (!((m[q] >> d) & 1u)) continue;
            const int ib = i + (d & 1), jb = j + ((d >> 1) & 1), kb = k + (d >> 2);
            const double cb = (double)chi[band_node(map, R, ib, jb, kb)];
            const double t = __ddiv_rn(__dsub_rn(iso, ca), __dsub_rn(cb, ca));
            const double pb[3] = {node_coord(bf, 0, ib), node_coord(bf, 1, jb), node_coord(bf, 2, kb)};
            vkey[cur] = node * 8 + d;
            vt[cur] = t;
            for (int a = 0; a < 3; ++a) vpos[3 * cur + a] = __dadd_rn(pa[a], __dmul_rn(t, __dsub_rn(pb[a], pa[a])));
            ++cur;
        }
    }
}

// triangles in ascending (storage index of the cube's lowest corner, tetrahedron, triangle)
__global__ void __launch_bounds__(MB) band_triangle_kernel(const float* __restrict__ chi, int R,
                                                           const int32_t* __restrict__ map,
                                                           const int32_t* __restrict__ list, int64_t nodes,
                                                           const double* __restrict__ iso2,
                                                           const long long* __restrict__ toff,
                                                           const int32_t* __restrict__ node_base,
                                                           const uint8_t* __restrict__ node_mask,
                                                           int32_t* __restrict__ faces) {
    typedef cub::BlockScan<int, MB> Scan;
    __shared__ typename Scan::TempStorage tmp;
    const double iso = iso2[1];
    uint32_t ins[NPT];
    int nt = 0;
    for (int q = 0; q < NPT; ++q) {
        const int64_t u = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        ins[q] = 0xFFu;  // no triangles
        if (u >= nodes) continue;
        int i, j, k;
        band_ijk(list, R, u, i, j, k);
        const BandNode b = band_view(chi, map, R, i, j, k, iso);
        if (!b.covered) continue;
        ins[q] = b.inside;
        nt += cube_triangle_count(b.inside);
    }
    int pre;
    Scan(tmp).ExclusiveSum(nt, pre);
    long long cur = toff[blockIdx.x] + pre;
    for (int q = 0; q < NPT; ++q) {
        if (ins[q] == 0xFFu || ins[q] == 0u) continue;
        const int64_t u = (int64_t)blockIdx.x * NODES_PER_CTA + threadIdx.x * NPT + q;
        int i, j, k;
        band_ijk(list, R, u, i, j, k);
        for (int p = 0; p < 6; ++p) {
            int tri[2][3][2];
            const int n = tet_triangles(p, ins[q], tri);
            for (int t = 0; t < n; ++t, ++cur) {
                for (int s = 0; s < 3; ++s) {
                    const int lo = tri[t][s][0], d = tri[t][s][1] ^ lo;
                    const int64_t pn = band_node(map, R, i + (lo & 1), j + ((lo >> 1) & 1), k + (lo >> 2));
                    faces[3 * cur + s] = node_base[pn] + __popc(node_mask[pn] & ((1u << d) - 1u));
                }
            }
        }
    }
}

// ---- density and colour gathers ------------------------------------------------------------------------------------
// int64 dual cell ((cz (R - 1) + cy) (R - 1) + cx) at level D of every splatted point (CELL64_NONE otherwise)
__global__ void __launch_bounds__(MB) band_cell_kernel(const float* __restrict__ xyz, const uint32_t* __restrict__ cell,
                                                       int64_t n, const double* __restrict__ bf, int R,
                                                       unsigned long long* __restrict__ key, uint32_t* __restrict__ idx) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= n) return;
    idx[i] = (uint32_t)i;
    if (cell[i] == CELL_NONE) { key[i] = CELL64_NONE; return; }
    const PointCell c = point_cell(xyz, i, bf, R);
    key[i] = ((uint64_t)c.i0[2] * (uint64_t)(R - 1) + (uint64_t)c.i0[1]) * (uint64_t)(R - 1) + (uint64_t)c.i0[0];
}

// the dense node sums (cells in ascending index, points in ascending input index), with the cell's first sorted
// position found by binary search
__device__ __forceinline__ void band_node_sums(int x, int y, int z, int R, const unsigned long long* __restrict__ sk,
                                               const uint32_t* __restrict__ sidx, int64_t n,
                                               const float* __restrict__ xyz, const int32_t* __restrict__ col,
                                               const double* __restrict__ bf, double& W, double (&C)[3]) {
    W = 0.0;
    C[0] = C[1] = C[2] = 0.0;
    for (int o = 7; o >= 0; --o) {
        const int cx = x - (o & 1), cy = y - ((o >> 1) & 1), cz = z - (o >> 2);
        if (cx < 0 || cy < 0 || cz < 0 || cx > R - 2 || cy > R - 2 || cz > R - 2) continue;
        const uint64_t id = ((uint64_t)cz * (uint64_t)(R - 1) + (uint64_t)cy) * (uint64_t)(R - 1) + (uint64_t)cx;
        int64_t lo = 0, hi = n;
        while (lo < hi) {
            const int64_t mid = (lo + hi) >> 1;
            if (sk[mid] < id) lo = mid + 1; else hi = mid;
        }
        for (int64_t j = lo; j < n && sk[j] == id; ++j) {
            const uint32_t pi = sidx[j];
            const double w = corner_weight(point_cell(xyz, pi, bf, R), o);
            W = __dadd_rn(W, w);
            if (col)
                for (int a = 0; a < 3; ++a) C[a] = __dadd_rn(C[a], __dmul_rn(w, (double)col[3 * (int64_t)pi + a]));
        }
    }
}

__global__ void __launch_bounds__(MB) band_gather_kernel(const long long* __restrict__ vkey, const double* __restrict__ vt,
                                                         int64_t m, int R, const unsigned long long* __restrict__ sk,
                                                         const uint32_t* __restrict__ sidx, int64_t n,
                                                         const float* __restrict__ xyz, const int32_t* __restrict__ col,
                                                         const double* __restrict__ bf, double* __restrict__ dens,
                                                         uint8_t* __restrict__ vcol) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const long long key = vkey[v];
    const int64_t node = key >> 3;
    const int d = (int)(key & 7);
    const int i = (int)(node % R), j = (int)((node / R) % R), k = (int)(node / ((int64_t)R * R));
    double Wa, Wb, Ca[3], Cb[3];
    band_node_sums(i, j, k, R, sk, sidx, n, xyz, col, bf, Wa, Ca);
    band_node_sums(i + (d & 1), j + ((d >> 1) & 1), k + (d >> 2), R, sk, sidx, n, xyz, col, bf, Wb, Cb);
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

// ---- workspace layouts ----------------------------------------------------------------------------------------------
struct BricksWs {
    uint8_t* seed;
    int32_t *keep, *scan;
    unsigned long long* lost;
    void* tmp;
    size_t tmp_bytes, bytes;
};
BricksWs bricks_ws(void* base, int depth) {
    const int64_t nb = nb3(depth);
    size_t scan_b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)nb);
    WsCarve w{(char*)base};
    BricksWs l;
    l.seed = w.take<uint8_t>(nb);
    l.keep = w.take<int32_t>(nb);
    l.scan = w.take<int32_t>(nb);
    l.lost = w.take<unsigned long long>(1);
    l.tmp_bytes = WsCarve::pad(scan_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct CgWs {
    float *r, *p, *q;
    double* part;
    size_t bytes;
};
CgWs cg_ws(void* base, int64_t nodes) {
    WsCarve w{(char*)base};
    CgWs l;
    l.r = w.take<float>(nodes);
    l.p = w.take<float>(nodes);
    l.q = w.take<float>(nodes);
    l.part = w.take<double>(3 * RED_BLOCKS);
    l.bytes = w.used;
    return l;
}

struct BandExtractWs {
    long long *vblk, *tblk, *voff, *toff;
    void* tmp;
    size_t tmp_bytes, bytes;
    int64_t nb;
};
BandExtractWs band_extract_ws(void* base, int64_t nodes) {
    BandExtractWs l;
    l.nb = (nodes + NODES_PER_CTA - 1) / NODES_PER_CTA;
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

struct BandGatherWs {
    unsigned long long *keys_a, *keys_b;
    uint32_t *idx_a, *idx_b;
    void* tmp;
    size_t tmp_bytes, bytes;
};
BandGatherWs band_gather_ws(void* base, int64_t n) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n, 0, 64);
    WsCarve w{(char*)base};
    BandGatherWs l;
    l.keys_a = w.take<unsigned long long>(n);
    l.keys_b = w.take<unsigned long long>(n);
    l.idx_a = w.take<uint32_t>(n);
    l.idx_b = w.take<uint32_t>(n);
    l.tmp_bytes = WsCarve::pad(sort_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

bool nodes_ok(int depth, int64_t nbricks) { return nbricks >= 1 && nbricks <= nb3(depth); }

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int64_t g2pc_mesh_band_bricks_workspace_bytes(int32_t depth) {
    return band_depth_ok(depth) ? (int64_t)bricks_ws(nullptr, depth).bytes : 0;
}

extern "C" int g2pc_mesh_band_bricks(const float* xyz, const uint32_t* cell, int64_t n, const double* frame,
                                     int32_t depth, const int32_t* parent_map, double* band_frame, int32_t* map,
                                     int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(band_depth_ok(depth), "band depth must be in 3..G2PC_MESH_BAND_DEPTH_MAX");
    G2PC_CHECK_ARG(frame && band_frame && map && counts && workspace && (n == 0 || (xyz && cell)), "null pointer");
    const BricksWs l = bricks_ws(workspace, depth);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    const int R = 1 << depth, NB = R / BRICK;
    const int64_t nb = nb3(depth);
    G2PC_CUDA(cudaMemsetAsync(l.seed, 0, (size_t)nb, st));
    G2PC_CUDA(cudaMemsetAsync(l.lost, 0, 8, st));
    band_frame_kernel<<<1, 1, 0, st>>>(frame, R, band_frame);
    G2PC_CHECK_LAUNCH();
    if (n > 0) {
        seed_kernel<<<grid_of(n), MB, 0, st>>>(xyz, cell, n, band_frame, R, l.seed);
        G2PC_CHECK_LAUNCH();
    }
    keep_kernel<<<grid_of(nb), MB, 0, st>>>(l.seed, NB, parent_map, l.keep, l.lost);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.keep, l.scan, (int)nb, st));
    map_kernel<<<grid_of(nb), MB, 0, st>>>(l.keep, l.scan, nb, map, (long long*)counts, l.lost);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_band_list(const int32_t* map, int32_t depth, int32_t* list, void* stream) {
    G2PC_CHECK_ARG(band_depth_ok(depth), "band depth must be in 3..G2PC_MESH_BAND_DEPTH_MAX");
    G2PC_CHECK_ARG(map && list, "null pointer");
    list_kernel<<<grid_of(nb3(depth)), MB, 0, (cudaStream_t)stream>>>(map, nb3(depth), list);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_band_splat(const float* xyz, const void* normals, int normal_dtype, const uint32_t* cell,
                                    int64_t n, const double* band_frame, int32_t depth, const int32_t* map,
                                    int64_t nbricks, int64_t* B, int32_t* status, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(band_depth_ok(depth) && nodes_ok(depth, nbricks), "bad band depth or brick count");
    G2PC_CHECK_ARG(normal_dtype == G2PC_F32 || normal_dtype == G2PC_F64, "normals must be float32 or float64");
    G2PC_CHECK_ARG(band_frame && map && B && status && (n == 0 || (xyz && normals && cell)), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int R = 1 << depth;
    G2PC_CUDA(cudaMemsetAsync(B, 0, (size_t)nbricks * BRICK_NODES * 8, st));
    G2PC_CUDA(cudaMemsetAsync(status, 0, 4, st));
    if (n > 0) {
        unsigned long long* Bu = (unsigned long long*)B;
        if (normal_dtype == G2PC_F32)
            band_splat_kernel<float><<<grid_of(n), MB, 0, st>>>(xyz, (const float*)normals, cell, n, R, band_frame, map,
                                                               Bu, status);
        else
            band_splat_kernel<double><<<grid_of(n), MB, 0, st>>>(xyz, (const double*)normals, cell, n, R, band_frame,
                                                                map, Bu, status);
        G2PC_CHECK_LAUNCH();
    }
    return G2PC_OK;
}

extern "C" int g2pc_mesh_band_ghosts(const float* parent_chi, const int32_t* parent_map, int32_t depth,
                                     const int32_t* map, const int32_t* list, int64_t nbricks, const int64_t* B,
                                     const double* band_frame, double* ghost, float* chi, float* rhs, void* stream) {
    G2PC_CHECK_ARG(band_depth_ok(depth) && nodes_ok(depth, nbricks), "bad band depth or brick count");
    G2PC_CHECK_ARG(parent_chi && map && list && B && band_frame && chi && rhs, "null pointer");
    const int64_t nodes = nbricks * BRICK_NODES;
    ghost_kernel<<<grid_of(nodes), MB, 0, (cudaStream_t)stream>>>(parent_chi, parent_map, 1 << depth, map, list, nodes,
                                                                  (const long long*)B, band_frame, ghost, chi, rhs);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_band_cg_workspace_bytes(int64_t nbricks) {
    return nbricks >= 0 ? (int64_t)cg_ws(nullptr, nbricks * BRICK_NODES).bytes : 0;
}

// checks and carves the arguments the two conjugate-gradient entry points share
#define BAND_CG_ARGS()                                                                                   \
    G2PC_CHECK_ARG(band_depth_ok(depth) && nodes_ok(depth, nbricks), "bad band depth or brick count");  \
    G2PC_CHECK_ARG(rhs && map && list && chi && scalars && workspace, "null pointer");                 \
    const int64_t nodes = nbricks * BRICK_NODES;                                                         \
    const CgWs l = cg_ws(workspace, nodes);                                                              \
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);                                      \
    cudaStream_t st = (cudaStream_t)stream;                                                              \
    const int R = 1 << depth

extern "C" int g2pc_mesh_band_cg_start(const float* rhs, int32_t depth, const int32_t* map, const int32_t* list,
                                       int64_t nbricks, float* chi, double* scalars, void* workspace,
                                       int64_t workspace_bytes, void* stream) {
    BAND_CG_ARGS();
    cg_init_kernel<<<RED_BLOCKS, MB, 0, st>>>(chi, rhs, map, list, R, nodes, l.r, l.p, l.part);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part, 1.0, scalars + CG_RR);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part + RED_BLOCKS, 1.0, scalars + CG_RZ);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part + 2 * RED_BLOCKS, 1.0, scalars + CG_CC);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_band_cg_step(const float* rhs, int32_t depth, const int32_t* map, const int32_t* list,
                                      int64_t nbricks, float* chi, int32_t iteration, double* scalars,
                                      void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(iteration >= 1, "iteration < 1");
    BAND_CG_ARGS();
    const int par = (iteration - 1) & 1;  // r.z of the last iteration is in CG_RZ + par, the new one goes to the other
    cg_apply_kernel<<<RED_BLOCKS, MB, 0, st>>>(l.p, map, list, R, nodes, l.q, l.part);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part, 1.0, scalars + CG_PQ);
    G2PC_CHECK_LAUNCH();
    cg_update_kernel<<<RED_BLOCKS, MB, 0, st>>>(chi, l.r, l.p, l.q, list, R, nodes, scalars, par, l.part);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part, 1.0, scalars + CG_RR);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(l.part + RED_BLOCKS, 1.0, scalars + CG_RZ + (par ^ 1));
    G2PC_CHECK_LAUNCH();
    cg_direction_kernel<<<grid_of(nodes), MB, 0, st>>>(l.p, l.r, list, R, nodes, scalars, par);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_band_iso_workspace_bytes(void) { return (int64_t)(2 * RED_BLOCKS * sizeof(double)); }

extern "C" int g2pc_mesh_band_iso(const float* xyz, const uint32_t* cell, int64_t n, const double* band_frame,
                                  int32_t depth, const int32_t* map, const float* chi, double* iso, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll, "n must be in 0..2^31-2");
    G2PC_CHECK_ARG(band_depth_ok(depth), "band depth must be in 3..G2PC_MESH_BAND_DEPTH_MAX");
    G2PC_CHECK_ARG(band_frame && map && chi && iso && workspace && (n == 0 || (xyz && cell)), "null pointer");
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, g2pc_mesh_band_iso_workspace_bytes(), 8);
    cudaStream_t st = (cudaStream_t)stream;
    double* part = (double*)workspace;
    band_iso_kernel<<<RED_BLOCKS, MB, 0, st>>>(xyz, cell, n, band_frame, 1 << depth, map, chi, part);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(part, 1.0, iso + 1);
    G2PC_CHECK_LAUNCH();
    finish_kernel<<<1, 1024, 0, st>>>(part + RED_BLOCKS, 1.0, iso + 2);
    G2PC_CHECK_LAUNCH();
    band_iso_div_kernel<<<1, 1, 0, st>>>(iso);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_band_extract_workspace_bytes(int64_t nbricks) {
    return nbricks >= 0 ? (int64_t)band_extract_ws(nullptr, nbricks * BRICK_NODES).bytes : 0;
}

extern "C" int g2pc_mesh_band_extract_count(const float* chi, int32_t depth, const int32_t* map, const int32_t* list,
                                            int64_t nbricks, const double* iso, int64_t* counts, void* workspace,
                                            int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(band_depth_ok(depth) && nodes_ok(depth, nbricks), "bad band depth or brick count");
    G2PC_CHECK_ARG(chi && map && list && iso && counts && workspace, "null pointer");
    const int64_t nodes = nbricks * BRICK_NODES;
    const BandExtractWs l = band_extract_ws(workspace, nodes);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(l.vblk + l.nb, 0, 8, st));
    G2PC_CUDA(cudaMemsetAsync(l.tblk + l.nb, 0, 8, st));
    band_count_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, 1 << depth, map, list, nodes, iso, l.vblk, l.tblk);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.vblk, l.voff, (int)(l.nb + 1), st));
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.tblk, l.toff, (int)(l.nb + 1), st));
    band_totals_kernel<<<1, 1, 0, st>>>(l.voff, l.toff, l.nb, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_band_extract_emit(const float* chi, int32_t depth, const int32_t* map, const int32_t* list,
                                           int64_t nbricks, const double* band_frame, const double* iso,
                                           void* node_scratch, int64_t node_scratch_bytes, const void* workspace,
                                           int64_t workspace_bytes, int64_t* vkey, double* vt, double* vpos,
                                           int32_t* faces, void* stream) {
    G2PC_CHECK_ARG(band_depth_ok(depth) && nodes_ok(depth, nbricks), "bad band depth or brick count");
    G2PC_CHECK_ARG(chi && map && list && band_frame && iso && node_scratch && workspace, "null pointer");
    const int64_t nodes = nbricks * BRICK_NODES;
    const BandExtractWs l = band_extract_ws(const_cast<void*>(workspace), nodes);  // read only here
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    G2PC_CHECK_ARG(node_scratch_bytes >= 5 * nodes, "node scratch too small (5 bytes per band node)");
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* base = (int32_t*)node_scratch;
    uint8_t* mask = (uint8_t*)node_scratch + 4 * nodes;
    const int R = 1 << depth;
    band_vertex_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, R, map, list, nodes, band_frame, iso, l.voff, base, mask,
                                                      (long long*)vkey, vt, vpos);
    G2PC_CHECK_LAUNCH();
    band_triangle_kernel<<<(unsigned)l.nb, MB, 0, st>>>(chi, R, map, list, nodes, iso, l.toff, base, mask, faces);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_band_gather_workspace_bytes(int64_t n) { return (int64_t)band_gather_ws(nullptr, n).bytes; }

extern "C" int g2pc_mesh_band_gather(const float* xyz, const int32_t* colours, const uint32_t* cell, int64_t n,
                                     const double* band_frame, int32_t depth, const int64_t* vkey, const double* vt,
                                     int64_t m, double* density, uint8_t* vcolours, void* workspace,
                                     int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && n < 0x7FFFFFFFll && m >= 0, "bad sizes");
    G2PC_CHECK_ARG(band_depth_ok(depth), "band depth must be in 3..G2PC_MESH_BAND_DEPTH_MAX");
    G2PC_CHECK_ARG(band_frame && workspace, "null pointer");
    const BandGatherWs l = band_gather_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(vkey && vt && density && (n == 0 || (xyz && cell)), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int R = 1 << depth;
    if (n > 0) {
        band_cell_kernel<<<grid_of(n), MB, 0, st>>>(xyz, cell, n, band_frame, R, l.keys_a, l.idx_a);
        G2PC_CHECK_LAUNCH();
        size_t b = l.tmp_bytes;  // stable: a cell's points stay in input order
        G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, l.keys_a, l.keys_b, l.idx_a, l.idx_b, (int)n, 0, 64, st));
    }
    band_gather_kernel<<<grid_of(m), MB, 0, st>>>((const long long*)vkey, vt, m, R, l.keys_b, l.idx_b, n, xyz, colours,
                                                  band_frame, density, vcolours);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
