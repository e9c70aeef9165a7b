// s13_decimate.cu — decimation of a triangle mesh to a target triangle count by parallel quadric edge collapse (N9).
// The rules are this project's own (DESIGN.md §2, N9) and tests/f64ref_decimate.py restates them in float64.
//
// prepare (once): per-vertex plane quadrics Q_v (10 float64: A00 A01 A02 A11 A12 A22 b0 b1 b2 c) summed over the
// incident faces in ascending face id, and the free flags (closed manifold fan).  Per round: select (incidence lists,
// unique edges, candidates, 2-ring minimum selection; the host reads the counts), then apply (the k selected edges with
// the smallest keys collapse, faces are remapped and compacted stably).  finish: stable vertex compaction.
// Every float64 expression a test compares bit for bit is written with __d*_rn intrinsics: no FMA contraction.
#include <cub/cub.cuh>
#include "mesh_common.cuh"

namespace {

constexpr unsigned long long KEY_NONE = ~0ull;  // not a candidate
constexpr int FAN_MAX = 128;                    // a vertex with more incident faces is locked (bounds the fan walk)
constexpr int QW = 10;                          // quadric words per vertex

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

// radix-sort end bit of keys whose high word is a vertex index < m
int end_bit_of(int64_t m) {
    int end_bit = 33;
    while (end_bit < 64 && ((unsigned long long)m >> (end_bit - 32)) != 0) ++end_bit;
    return end_bit;
}

struct V3 {
    double x[3];
};

__device__ __forceinline__ V3 load3(const double* __restrict__ p, int64_t v) { return V3{{p[3 * v], p[3 * v + 1], p[3 * v + 2]}}; }

// cross(p1 - p0, p2 - p0), as normals_kernel forms it
__device__ __forceinline__ V3 face_normal(const V3& p0, const V3& p1, const V3& p2) {
    double u[3], w[3];
    for (int a = 0; a < 3; ++a) { u[a] = __dsub_rn(p1.x[a], p0.x[a]); w[a] = __dsub_rn(p2.x[a], p0.x[a]); }
    return V3{{__dsub_rn(__dmul_rn(u[1], w[2]), __dmul_rn(u[2], w[1])),
               __dsub_rn(__dmul_rn(u[2], w[0]), __dmul_rn(u[0], w[2])),
               __dsub_rn(__dmul_rn(u[0], w[1]), __dmul_rn(u[1], w[0]))}};
}

__device__ __forceinline__ double dot3(const V3& a, const V3& b) {
    return __dadd_rn(__dadd_rn(__dmul_rn(a.x[0], b.x[0]), __dmul_rn(a.x[1], b.x[1])), __dmul_rn(a.x[2], b.x[2]));
}

// max(0, v^T A v + 2 b^T v + c): Av_i = (A_i0 v0 + A_i1 v1) + A_i2 v2, then (v . Av + 2 (b . v)) + c
__device__ __forceinline__ double quadric_cost(const double (&q)[QW], const V3& v) {
    const double A[3][3] = {{q[0], q[1], q[2]}, {q[1], q[3], q[4]}, {q[2], q[4], q[5]}};
    V3 Av;
    for (int i = 0; i < 3; ++i)
        Av.x[i] = __dadd_rn(__dadd_rn(__dmul_rn(A[i][0], v.x[0]), __dmul_rn(A[i][1], v.x[1])), __dmul_rn(A[i][2], v.x[2]));
    const V3 b{{q[6], q[7], q[8]}};
    const double r = __dadd_rn(__dadd_rn(dot3(v, Av), __dmul_rn(2.0, dot3(b, v))), q[9]);
    return r > 0.0 ? r : 0.0;
}

// The position of the merged vertex and its cost for Q = Q_a + Q_b: the minimiser of v^T Q v by the adjugate when
// |det A| > 1e-12 max|A_ij|^3 and it lies within |b - a| of the midpoint; else the cheapest of a, b, the midpoint (ties
// in that order).
__device__ __forceinline__ double place(const double* __restrict__ Q, int64_t a, int64_t b, const V3& pa, const V3& pb,
                                        V3& v) {
    double q[QW];
    for (int i = 0; i < QW; ++i) q[i] = __dadd_rn(Q[QW * a + i], Q[QW * b + i]);
    const double A00 = q[0], A01 = q[1], A02 = q[2], A11 = q[3], A12 = q[4], A22 = q[5];
    const double C00 = __dsub_rn(__dmul_rn(A11, A22), __dmul_rn(A12, A12));
    const double C01 = __dsub_rn(__dmul_rn(A02, A12), __dmul_rn(A01, A22));
    const double C02 = __dsub_rn(__dmul_rn(A01, A12), __dmul_rn(A02, A11));
    const double C11 = __dsub_rn(__dmul_rn(A00, A22), __dmul_rn(A02, A02));
    const double C12 = __dsub_rn(__dmul_rn(A01, A02), __dmul_rn(A00, A12));
    const double C22 = __dsub_rn(__dmul_rn(A00, A11), __dmul_rn(A01, A01));
    const double det = __dadd_rn(__dadd_rn(__dmul_rn(A00, C00), __dmul_rn(A01, C01)), __dmul_rn(A02, C02));
    double nA = fabs(A00);
    nA = fmax(nA, fabs(A01));
    nA = fmax(nA, fabs(A02));
    nA = fmax(nA, fabs(A11));
    nA = fmax(nA, fabs(A12));
    nA = fmax(nA, fabs(A22));
    V3 mid, d, e;
    for (int x = 0; x < 3; ++x) mid.x[x] = __dmul_rn(__dadd_rn(pa.x[x], pb.x[x]), 0.5);
    if (fabs(det) > __dmul_rn(1e-12, __dmul_rn(__dmul_rn(nA, nA), nA))) {
        const double C[3][3] = {{C00, C01, C02}, {C01, C11, C12}, {C02, C12, C22}};
        V3 s;
        for (int i = 0; i < 3; ++i) {
            const double t = __dadd_rn(__dadd_rn(__dmul_rn(C[i][0], q[6]), __dmul_rn(C[i][1], q[7])), __dmul_rn(C[i][2], q[8]));
            s.x[i] = __ddiv_rn(-t, det);
        }
        for (int x = 0; x < 3; ++x) { d.x[x] = __dsub_rn(s.x[x], mid.x[x]); e.x[x] = __dsub_rn(pb.x[x], pa.x[x]); }
        if (dot3(d, d) <= dot3(e, e)) {
            v = s;
            return quadric_cost(q, s);
        }
    }
    v = pa;
    double c = quadric_cost(q, pa);
    const double cb = quadric_cost(q, pb), cm = quadric_cost(q, mid);
    if (cb < c) { v = pb; c = cb; }
    if (cm < c) { v = mid; c = cm; }
    return c;
}

// ---- prepare --------------------------------------------------------------------------------------------------------
// Q_v = sum over the incident faces in ascending id of K_f = [n n^T, -n (n . p0); (n . p0)^2] / (2 |n|), n = cross(p1 -
// p0, p2 - p0); a face with |n| = 0 adds nothing.  K_f's entries: (n_i n_j) / s, (-(n_i d)) / s, (d d) / s with
// d = (n0 p0x + n1 p0y) + n2 p0z and s = 2 |n|, |n| = sqrt((n0 n0 + n1 n1) + n2 n2).
__global__ void __launch_bounds__(MB) quadric_kernel(const double* __restrict__ p, int64_t m,
                                                     const int32_t* __restrict__ faces,
                                                     const unsigned long long* __restrict__ keys,
                                                     const int32_t* __restrict__ row, double* __restrict__ Q) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    double q[QW];
    for (int i = 0; i < QW; ++i) q[i] = 0.0;
    for (int64_t j = row[v]; j < row[v + 1]; ++j) {
        const int64_t f = (int64_t)(keys[j] & 0xFFFFFFFFull);
        const V3 p0 = load3(p, faces[3 * f]);
        const V3 n = face_normal(p0, load3(p, faces[3 * f + 1]), load3(p, faces[3 * f + 2]));
        const double len = sqrt(dot3(n, n));
        if (!(len > 0.0)) continue;
        const double s = __dmul_rn(2.0, len), d = dot3(n, p0);
        const double k[QW] = {__dmul_rn(n.x[0], n.x[0]), __dmul_rn(n.x[0], n.x[1]), __dmul_rn(n.x[0], n.x[2]),
                              __dmul_rn(n.x[1], n.x[1]), __dmul_rn(n.x[1], n.x[2]), __dmul_rn(n.x[2], n.x[2]),
                              -__dmul_rn(n.x[0], d),     -__dmul_rn(n.x[1], d),     -__dmul_rn(n.x[2], d),
                              __dmul_rn(d, d)};
        for (int i = 0; i < QW; ++i) q[i] = __dadd_rn(q[i], __ddiv_rn(k[i], s));
    }
    for (int i = 0; i < QW; ++i) Q[QW * v + i] = q[i];
}

// the two vertices of face f after v in the face's cyclic order; false when v is not in f exactly once
__device__ __forceinline__ bool others(const int32_t* __restrict__ faces, int64_t f, int64_t v, int32_t& x, int32_t& y) {
    const int32_t a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
    if ((a == v) + (b == v) + (c == v) != 1) return false;
    if (a == v) { x = b; y = c; } else if (b == v) { x = c; y = a; } else { x = a; y = b; }
    return true;
}

// free[v] = 1 iff v has 1..FAN_MAX incident faces, every edge at v is used by exactly two of them, and they form one
// closed fan: the walk from the first face across shared edges returns to it after visiting every face.
__global__ void __launch_bounds__(MB) free_kernel(int64_t m, const int32_t* __restrict__ faces,
                                                  const unsigned long long* __restrict__ keys,
                                                  const int32_t* __restrict__ row, uint8_t* __restrict__ fl) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int64_t r0 = row[v], nf = row[v + 1] - r0;
    fl[v] = 0;
    if (nf < 1 || nf > FAN_MAX) return;
    auto face = [&](int64_t j) { return (int64_t)(keys[r0 + j] & 0xFFFFFFFFull); };
    for (int64_t j = 0; j < nf; ++j) {
        int32_t x, y;
        if (!others(faces, face(j), v, x, y)) return;
        for (int s = 0; s < 2; ++s) {
            const int32_t w = s ? y : x;
            int cnt = 0;
            for (int64_t i = 0; i < nf; ++i) {
                const int64_t g = face(i);
                cnt += faces[3 * g] == w || faces[3 * g + 1] == w || faces[3 * g + 2] == w;
            }
            if (cnt != 2) return;
        }
    }
    int32_t x, y;
    others(faces, face(0), v, x, y);
    int64_t cur = 0, steps = 0;
    int32_t through = y;
    do {
        int64_t nxt = -1;
        for (int64_t i = 0; i < nf && nxt < 0; ++i) {
            if (i == cur) continue;
            const int64_t g = face(i);
            if (faces[3 * g] == through || faces[3 * g + 1] == through || faces[3 * g + 2] == through) nxt = i;
        }
        int32_t gx, gy;
        others(faces, face(nxt), v, gx, gy);
        through = gx == through ? gy : gx;
        cur = nxt;
        ++steps;
    } while (cur != 0 && steps <= nf);
    fl[v] = cur == 0 && steps == nf;
}

// ---- select ---------------------------------------------------------------------------------------------------------
// undirected edge keys (min << 32 | max) of every triangle edge, with the triangle as the value
__global__ void __launch_bounds__(MB) edge_keys_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                       unsigned long long* __restrict__ keys, int32_t* __restrict__ vals) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    for (int s = 0; s < 3; ++s) {
        const unsigned long long a = (uint32_t)faces[3 * f + s], b = (uint32_t)faces[3 * f + (s + 1) % 3];
        keys[3 * f + s] = a < b ? a << 32 | b : b << 32 | a;
        vals[3 * f + s] = (int32_t)f;
    }
}

__global__ void __launch_bounds__(MB) head_kernel(const unsigned long long* __restrict__ ek, int64_t e,
                                                  int32_t* __restrict__ head) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i < e) head[i] = i == 0 || ek[i] != ek[i - 1];
}

__device__ __forceinline__ bool has_vertex(const int32_t* __restrict__ faces, int64_t f, int64_t w) {
    return faces[3 * f] == w || faces[3 * f + 1] == w || faces[3 * f + 2] == w;
}

// is x a neighbour of v (in one of v's faces)?
__device__ bool adjacent(const int32_t* __restrict__ faces, const unsigned long long* __restrict__ ik,
                         const int32_t* __restrict__ row, int64_t v, int64_t x) {
    for (int64_t j = row[v]; j < row[v + 1]; ++j)
        if (has_vertex(faces, (int64_t)(ik[j] & 0xFFFFFFFFull), x)) return true;
    return false;
}

// does v have a face {v, c, d}?
__device__ bool has_face(const int32_t* __restrict__ faces, const unsigned long long* __restrict__ ik,
                         const int32_t* __restrict__ row, int64_t v, int64_t c, int64_t d) {
    for (int64_t j = row[v]; j < row[v + 1]; ++j) {
        const int64_t g = (int64_t)(ik[j] & 0xFFFFFFFFull);
        if (has_vertex(faces, g, c) && has_vertex(faces, g, d)) return true;
    }
    return false;
}

// does moving vertex u to y keep every face of u other than f1, f2 unflipped (dot(n_old, n_new) > 0)?
__device__ bool no_flip(const double* __restrict__ p, const int32_t* __restrict__ faces,
                        const unsigned long long* __restrict__ ik, const int32_t* __restrict__ row, int64_t u,
                        int64_t f1, int64_t f2, const V3& y) {
    for (int64_t j = row[u]; j < row[u + 1]; ++j) {
        const int64_t g = (int64_t)(ik[j] & 0xFFFFFFFFull);
        if (g == f1 || g == f2) continue;
        V3 o[3], n[3];
        for (int s = 0; s < 3; ++s) {
            const int64_t w = faces[3 * g + s];
            o[s] = load3(p, w);
            n[s] = w == u ? y : o[s];
        }
        if (!(dot3(face_normal(o[0], o[1], o[2]), face_normal(n[0], n[1], n[2])) > 0.0)) return false;
    }
    return true;
}

// One thread per sorted edge-key entry; the first entry of each run is edge id escan[i].  ends[id] = the edge's key;
// key[id] = float32(cost) bits << 32 | id for a candidate, KEY_NONE otherwise; M1[v] = min key at v.
__global__ void __launch_bounds__(MB) candidate_kernel(const double* __restrict__ p, const int32_t* __restrict__ faces,
                                                       const unsigned long long* __restrict__ ik,
                                                       const int32_t* __restrict__ row, const double* __restrict__ Q,
                                                       const uint8_t* __restrict__ fl,
                                                       const unsigned long long* __restrict__ ek,
                                                       const int32_t* __restrict__ ev, const int32_t* __restrict__ escan,
                                                       int64_t e, unsigned long long* __restrict__ ends,
                                                       unsigned long long* __restrict__ key,
                                                       unsigned long long* __restrict__ M1,
                                                       unsigned long long* __restrict__ ncand) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= e) return;
    const unsigned long long k = ek[i];
    if (i > 0 && ek[i - 1] == k) return;
    const int64_t id = escan[i];
    ends[id] = k;
    key[id] = KEY_NONE;
    const int64_t a = (int64_t)(k >> 32), b = (int64_t)(k & 0xFFFFFFFFull);
    if (!fl[a] || !fl[b]) return;
    if (i + 1 >= e || ek[i + 1] != k || (i + 2 < e && ek[i + 2] == k)) return;
    const int64_t f1 = ev[i], f2 = ev[i + 1];
    int64_t c = -1, d = -1;
    for (int s = 0; s < 3; ++s) {
        const int64_t w1 = faces[3 * f1 + s], w2 = faces[3 * f2 + s];
        if (w1 != a && w1 != b) c = w1;
        if (w2 != a && w2 != b) d = w2;
    }
    if (c == d) return;
    // link condition: the common neighbours of a and b are exactly c and d, and {a,c,d}, {b,c,d} are not both faces
    for (int64_t j = row[a]; j < row[a + 1]; ++j) {
        const int64_t g = (int64_t)(ik[j] & 0xFFFFFFFFull);
        for (int s = 0; s < 3; ++s) {
            const int64_t x = faces[3 * g + s];
            if (x == a || x == b || x == c || x == d) continue;
            if (adjacent(faces, ik, row, b, x)) return;
        }
    }
    if (has_face(faces, ik, row, a, c, d) && has_face(faces, ik, row, b, c, d)) return;
    const V3 pa = load3(p, a), pb = load3(p, b);
    V3 v;
    const double cost = place(Q, a, b, pa, pb, v);
    if (!no_flip(p, faces, ik, row, a, f1, f2, v) || !no_flip(p, faces, ik, row, b, f1, f2, v)) return;
    const unsigned long long kk = (unsigned long long)__float_as_uint(__double2float_rn(cost)) << 32 |
                                  (unsigned long long)id;
    key[id] = kk;
    atomicMin(&M1[a], kk);
    atomicMin(&M1[b], kk);
    atomicAdd(ncand, 1ull);
}

// M2[v] = min of M1 over v and its neighbours (M2 starts as a copy of M1)
__global__ void __launch_bounds__(MB) spread_kernel(const unsigned long long* __restrict__ ek, int64_t e,
                                                    const unsigned long long* __restrict__ M1,
                                                    unsigned long long* __restrict__ M2) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= e) return;
    const unsigned long long k = ek[i];
    if (i > 0 && ek[i - 1] == k) return;
    const int64_t a = (int64_t)(k >> 32), b = (int64_t)(k & 0xFFFFFFFFull);
    const unsigned long long ma = M1[a], mb = M1[b];
    if (mb < M2[a]) atomicMin(&M2[a], mb);
    if (ma < M2[b]) atomicMin(&M2[b], ma);
}

// an edge is selected iff key = M2[a] = M2[b]
__global__ void __launch_bounds__(MB) pick_kernel(const unsigned long long* __restrict__ ek, int64_t e,
                                                  const int32_t* __restrict__ escan,
                                                  const unsigned long long* __restrict__ key,
                                                  const unsigned long long* __restrict__ M2, int32_t* __restrict__ flag) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= e) return;
    const unsigned long long k = ek[i];
    if (i > 0 && ek[i - 1] == k) return;
    const int64_t id = escan[i];
    const unsigned long long kk = key[id];
    flag[id] = kk != KEY_NONE && kk == M2[k >> 32] && kk == M2[k & 0xFFFFFFFFull];
}

__global__ void edge_count_kernel(const int32_t* __restrict__ escan, const int32_t* __restrict__ head, int64_t e,
                                  long long* __restrict__ counts) {
    counts[0] = e ? (long long)escan[e - 1] + head[e - 1] : 0;
}

// ---- apply ----------------------------------------------------------------------------------------------------------
// The j-th smallest selected key collapses b into a: a moves to the placed position, Q_a += Q_b, the colour sums,
// merge counts and density sums add, b dies and vmap[b] = a.
__global__ void __launch_bounds__(MB) collapse_kernel(const unsigned long long* __restrict__ sel, int64_t k,
                                                      const unsigned long long* __restrict__ ends,
                                                      double* __restrict__ p, double* __restrict__ Q,
                                                      long long* __restrict__ csum, int32_t* __restrict__ merged,
                                                      double* __restrict__ dsum, uint8_t* __restrict__ alive,
                                                      int32_t* __restrict__ vmap,
                                                      unsigned long long* __restrict__ applied,
                                                      int32_t* __restrict__ applied_ab) {
    const int64_t j = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (j >= k) return;
    const unsigned long long kk = sel[j], ed = ends[kk & 0xFFFFFFFFull];
    const int64_t a = (int64_t)(ed >> 32), b = (int64_t)(ed & 0xFFFFFFFFull);
    V3 v;
    place(Q, a, b, load3(p, a), load3(p, b), v);
    for (int x = 0; x < 3; ++x) p[3 * a + x] = v.x[x];
    for (int i = 0; i < QW; ++i) Q[QW * a + i] = __dadd_rn(Q[QW * a + i], Q[QW * b + i]);
    if (csum)
        for (int x = 0; x < 3; ++x) csum[3 * a + x] += csum[3 * b + x];
    merged[a] += merged[b];
    if (dsum) dsum[a] = __dadd_rn(dsum[a], dsum[b]);
    alive[b] = 0;
    vmap[b] = (int32_t)a;
    if (applied) applied[j] = kk;
    if (applied_ab) { applied_ab[2 * j] = (int32_t)a; applied_ab[2 * j + 1] = (int32_t)b; }
}

__global__ void __launch_bounds__(MB) iota_kernel(int32_t* __restrict__ x, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i < n) x[i] = (int32_t)i;
}

// a face survives iff its three remapped vertices are distinct (only the two faces of a collapsed edge lose one)
__global__ void __launch_bounds__(MB) face_flag_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                       const int32_t* __restrict__ vmap, int32_t* __restrict__ flag) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    const int32_t a = vmap[faces[3 * f]], b = vmap[faces[3 * f + 1]], c = vmap[faces[3 * f + 2]];
    flag[f] = a != b && b != c && a != c;
}

__global__ void __launch_bounds__(MB) face_compact_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                          const int32_t* __restrict__ flag,
                                                          const int32_t* __restrict__ pos,
                                                          const int32_t* __restrict__ vmap,
                                                          int32_t* __restrict__ out) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t || !flag[f]) return;
    const int64_t o = pos[f];
    for (int s = 0; s < 3; ++s) out[3 * o + s] = vmap[faces[3 * f + s]];
}

__global__ void total_kernel(const int32_t* __restrict__ flag, const int32_t* __restrict__ pos, int64_t n,
                             long long* __restrict__ out) {
    *out = n ? (long long)pos[n - 1] + flag[n - 1] : 0;
}

// ---- finish ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(MB) alive_flag_kernel(const uint8_t* __restrict__ alive, int64_t m,
                                                        int32_t* __restrict__ flag) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v < m) flag[v] = alive[v] != 0;
}

// every vertex of a face is alive: its rank among the alive vertices is its new index
__global__ void __launch_bounds__(MB) renumber_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                      const int32_t* __restrict__ pos, int32_t* __restrict__ out) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i < 3 * t) out[i] = pos[faces[i]];
}

// colour = floor(sum / count + 1/2) = (2 sum + count) / (2 count) in integers; density = sum / count
__global__ void __launch_bounds__(MB) vertex_compact_kernel(const int32_t* __restrict__ flag,
                                                            const int32_t* __restrict__ pos, int64_t m,
                                                            const double* __restrict__ p,
                                                            const long long* __restrict__ csum,
                                                            const int32_t* __restrict__ merged,
                                                            const double* __restrict__ dsum,
                                                            double* __restrict__ p_out, uint8_t* __restrict__ c_out,
                                                            double* __restrict__ d_out) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || !flag[v]) return;
    const int64_t o = pos[v];
    const long long n = merged[v];
    for (int x = 0; x < 3; ++x) p_out[3 * o + x] = p[3 * v + x];
    if (c_out)
        for (int x = 0; x < 3; ++x) c_out[3 * o + x] = (uint8_t)((2 * csum[3 * v + x] + n) / (2 * n));
    if (d_out) d_out[o] = __ddiv_rn(dsum[v], (double)n);
}

// ---- workspace layouts ----------------------------------------------------------------------------------------------
struct PrepareWs {
    unsigned long long *keys_a, *keys_b;
    int32_t* row;
    void* tmp;
    size_t tmp_bytes, bytes;
};
PrepareWs prepare_ws(void* base, int64_t m, int64_t t) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                   (int)(3 * t));
    WsCarve w{(char*)base};
    PrepareWs l;
    l.keys_a = w.take<unsigned long long>(3 * t);
    l.keys_b = w.take<unsigned long long>(3 * t);
    l.row = w.take<int32_t>(m + 1);
    l.tmp_bytes = WsCarve::pad(sort_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

// select and apply of one round share this layout (apply reads ends and sel)
struct RoundWs {
    unsigned long long *ik[2], *ek[2], *ends, *M1, *M2, *sel_a, *sel_b;
    int32_t *ev[2], *escan, *flag, *row, *vmap, *fflag, *fpos;
    void* tmp;
    size_t tmp_bytes, bytes;
};
RoundWs round_ws(void* base, int64_t m, int64_t t) {
    const int e = (int)(3 * t);
    size_t b[7] = {0, 0, 0, 0, 0, 0, 0};
    cub::DoubleBuffer<unsigned long long> dk(nullptr, nullptr);
    cub::DoubleBuffer<int32_t> dv(nullptr, nullptr);
    cub::DeviceRadixSort::SortKeys(nullptr, b[0], dk, e);
    cub::DeviceRadixSort::SortPairs(nullptr, b[1], dk, dv, e);
    cub::DeviceScan::ExclusiveSum(nullptr, b[2], (const int32_t*)nullptr, (int32_t*)nullptr, e);
    cub::DeviceSelect::Flagged(nullptr, b[3], (const unsigned long long*)nullptr, (const int32_t*)nullptr,
                               (unsigned long long*)nullptr, (long long*)nullptr, e);
    cub::DeviceRadixSort::SortKeys(nullptr, b[4], (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                   (int)m);
    cub::DeviceScan::ExclusiveSum(nullptr, b[5], (const int32_t*)nullptr, (int32_t*)nullptr, (int)t);
    size_t tb = 0;
    for (size_t x : b) tb = tb > x ? tb : x;
    WsCarve w{(char*)base};
    RoundWs l;
    for (int s = 0; s < 2; ++s) {
        l.ik[s] = w.take<unsigned long long>(e);
        l.ek[s] = w.take<unsigned long long>(e);
        l.ev[s] = w.take<int32_t>(e);
    }
    l.ends = w.take<unsigned long long>(e);
    l.escan = w.take<int32_t>(e);
    l.flag = w.take<int32_t>(e);
    l.row = w.take<int32_t>(m + 1);
    l.M1 = w.take<unsigned long long>(m);
    l.M2 = w.take<unsigned long long>(m);
    l.sel_a = w.take<unsigned long long>(m);
    l.sel_b = w.take<unsigned long long>(m);
    l.vmap = w.take<int32_t>(m);
    l.fflag = w.take<int32_t>(t);
    l.fpos = w.take<int32_t>(t);
    l.tmp_bytes = WsCarve::pad(tb);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct FinishWs {
    int32_t *flag, *pos;
    void* tmp;
    size_t tmp_bytes, bytes;
};
FinishWs finish_ws(void* base, int64_t m) {
    size_t scan_b = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (const int32_t*)nullptr, (int32_t*)nullptr, (int)m);
    WsCarve w{(char*)base};
    FinishWs l;
    l.flag = w.take<int32_t>(m);
    l.pos = w.take<int32_t>(m);
    l.tmp_bytes = WsCarve::pad(scan_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

bool sizes_ok(int64_t m, int64_t t) { return m >= 0 && m < 0x7FFFFFFFll && t >= 0 && 3 * t < 0x7FFFFFFFll; }

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int64_t g2pc_mesh_decimate_prepare_workspace_bytes(int64_t m, int64_t t) {
    return sizes_ok(m, t) ? (int64_t)prepare_ws(nullptr, m, t).bytes : 0;
}

extern "C" int g2pc_mesh_decimate_prepare(const double* vpos, int64_t m, const int32_t* faces, int64_t t,
                                          double* quadrics, uint8_t* free_flags, void* workspace,
                                          int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 0..2^31-2 vertices and 3 t < 2^31 - 1");
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(vpos && quadrics && free_flags && workspace && (t == 0 || faces), "null pointer");
    const PrepareWs l = prepare_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (t > 0) {
        incidence_keys_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.keys_a);
        G2PC_CHECK_LAUNCH();
        size_t b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, l.keys_a, l.keys_b, (int)(3 * t), 0, end_bit_of(m), st));
    }
    row_kernel<<<grid_of(m + 1), MB, 0, st>>>(l.keys_b, 3 * t, m, l.row);
    G2PC_CHECK_LAUNCH();
    quadric_kernel<<<grid_of(m), MB, 0, st>>>(vpos, m, faces, l.keys_b, l.row, quadrics);
    G2PC_CHECK_LAUNCH();
    free_kernel<<<grid_of(m), MB, 0, st>>>(m, faces, l.keys_b, l.row, free_flags);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_decimate_round_workspace_bytes(int64_t m, int64_t t) {
    return sizes_ok(m, t) ? (int64_t)round_ws(nullptr, m, t).bytes : 0;
}

extern "C" int g2pc_mesh_decimate_select(const double* vpos, int64_t m, const int32_t* faces, int64_t t,
                                         const double* quadrics, const uint8_t* free_flags, int64_t* counts,
                                         void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t) && m > 0 && t > 0, "need 1..2^31-2 vertices and 1 <= 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(vpos && faces && quadrics && free_flags && counts && workspace, "null pointer");
    const RoundWs l = round_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t e = 3 * t;
    const int eb = end_bit_of(m);
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 3 * sizeof(int64_t), st));
    // incidence lists: sorted (v << 32 | face) keys and their rows
    incidence_keys_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.ik[0]);
    G2PC_CHECK_LAUNCH();
    cub::DoubleBuffer<unsigned long long> ik(l.ik[0], l.ik[1]);
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, ik, (int)e, 0, eb, st));
    row_kernel<<<grid_of(m + 1), MB, 0, st>>>(ik.Current(), e, m, l.row);
    G2PC_CHECK_LAUNCH();
    // unique edges in ascending (a << 32 | b), each run holding its faces in ascending id (the sort is stable)
    edge_keys_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.ek[0], l.ev[0]);
    G2PC_CHECK_LAUNCH();
    cub::DoubleBuffer<unsigned long long> ek(l.ek[0], l.ek[1]);
    cub::DoubleBuffer<int32_t> ev(l.ev[0], l.ev[1]);
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, ek, ev, (int)e, 0, eb, st));
    int32_t* head = ev.Alternate();
    unsigned long long* key = ek.Alternate();
    head_kernel<<<grid_of(e), MB, 0, st>>>(ek.Current(), e, head);
    G2PC_CHECK_LAUNCH();
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, head, l.escan, (int)e, st));
    edge_count_kernel<<<1, 1, 0, st>>>(l.escan, head, e, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    G2PC_CUDA(cudaMemsetAsync(l.M1, 0xFF, (size_t)m * 8, st));
    candidate_kernel<<<grid_of(e), MB, 0, st>>>(vpos, faces, ik.Current(), l.row, quadrics, free_flags, ek.Current(),
                                                ev.Current(), l.escan, e, l.ends, key, l.M1,
                                                (unsigned long long*)counts + 1);
    G2PC_CHECK_LAUNCH();
    G2PC_CUDA(cudaMemcpyAsync(l.M2, l.M1, (size_t)m * 8, cudaMemcpyDeviceToDevice, st));
    spread_kernel<<<grid_of(e), MB, 0, st>>>(ek.Current(), e, l.M1, l.M2);
    G2PC_CHECK_LAUNCH();
    G2PC_CUDA(cudaMemsetAsync(l.flag, 0, (size_t)e * 4, st));
    pick_kernel<<<grid_of(e), MB, 0, st>>>(ek.Current(), e, l.escan, key, l.M2, l.flag);
    G2PC_CHECK_LAUNCH();
    // selected keys in ascending edge id; the flags past the last edge are 0
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceSelect::Flagged(l.tmp, b, key, l.flag, l.sel_a, (long long*)counts + 2, (int)e, st));
    return G2PC_OK;
}

extern "C" int g2pc_mesh_decimate_apply(double* vpos, int64_t m, const int32_t* faces, int64_t t, double* quadrics,
                                        int64_t* colour_sums, int32_t* merged, double* density_sums, uint8_t* alive,
                                        int64_t selected, int64_t k, int32_t* faces_out, int64_t* kept,
                                        uint64_t* applied, int32_t* applied_ab, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t) && m > 0 && t > 0, "need 1..2^31-2 vertices and 1 <= 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(selected >= 0 && 2 * selected <= m && k >= 0 && k <= selected && 2 * k <= t,
                   "need 0 <= k <= selected <= m / 2 and 2 k <= t");
    G2PC_CHECK_ARG(vpos && faces && quadrics && merged && alive && faces_out && kept && workspace, "null pointer");
    const RoundWs l = round_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (selected > 0) {
        size_t b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, l.sel_a, l.sel_b, (int)selected, 0, 64, st));
    }
    iota_kernel<<<grid_of(m), MB, 0, st>>>(l.vmap, m);
    G2PC_CHECK_LAUNCH();
    if (k > 0) {
        collapse_kernel<<<grid_of(k), MB, 0, st>>>(l.sel_b, k, l.ends, vpos, quadrics, (long long*)colour_sums, merged,
                                                   density_sums, alive, l.vmap, (unsigned long long*)applied,
                                                   applied_ab);
        G2PC_CHECK_LAUNCH();
    }
    face_flag_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.vmap, l.fflag);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.fflag, l.fpos, (int)t, st));
    face_compact_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, l.fflag, l.fpos, l.vmap, faces_out);
    G2PC_CHECK_LAUNCH();
    total_kernel<<<1, 1, 0, st>>>(l.fflag, l.fpos, t, (long long*)kept);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_decimate_finish_workspace_bytes(int64_t m) {
    return m >= 0 && m < 0x7FFFFFFFll ? (int64_t)finish_ws(nullptr, m).bytes : 0;
}

extern "C" int g2pc_mesh_decimate_finish(const double* vpos, int64_t m, const int32_t* faces, int64_t t,
                                         const uint8_t* alive, const int64_t* colour_sums, const int32_t* merged,
                                         const double* density_sums, double* vpos_out, uint8_t* colours_out,
                                         double* densities_out, int32_t* faces_out, int64_t* counts, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t) && m > 0, "need 1..2^31-2 vertices and 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(vpos && alive && merged && vpos_out && counts && workspace && (t == 0 || (faces && faces_out)),
                   "null pointer");
    G2PC_CHECK_ARG(!colour_sums == !colours_out && !density_sums == !densities_out, "an attribute needs an output");
    const FinishWs l = finish_ws(workspace, m);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    alive_flag_kernel<<<grid_of(m), MB, 0, st>>>(alive, m, l.flag);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.flag, l.pos, (int)m, st));
    vertex_compact_kernel<<<grid_of(m), MB, 0, st>>>(l.flag, l.pos, m, vpos, (const long long*)colour_sums, merged,
                                                     density_sums, vpos_out, colours_out, densities_out);
    G2PC_CHECK_LAUNCH();
    if (t > 0) {
        renumber_kernel<<<grid_of(3 * t), MB, 0, st>>>(faces, t, l.pos, faces_out);
        G2PC_CHECK_LAUNCH();
    }
    total_kernel<<<1, 1, 0, st>>>(l.flag, l.pos, m, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
