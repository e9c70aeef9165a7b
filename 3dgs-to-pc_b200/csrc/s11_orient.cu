// s11_orient.cu — consistent orientation of point-cloud normals (N7, g2pc/orient.py, mesh_pc.py --orient_normals):
// Hoppe et al. 1992, as Open3D's orient_normals_consistent_tangent_plane does it, with this project's own rules
// (DESIGN.md §2).
//
//   prepare  the usable points (finite coordinate, finite non-zero normal), compacted in row order, with unit normals
//            n / sqrt((nx*nx + ny*ny) + nz*nz) in float64, as the N6 splat computes them
//   (k-NN)   g2pc_knn_ids (s9_clean.cu) on the compacted points: k nearest other points by ascending (d2, id)
//   edges    the undirected edges {i, j} of the k-NN graph, sorted by (min, max) and deduplicated: edge e gets the key
//            (float32 bits of max(0, 1 - |dot|)) << 32 | e, unique, and the flip bit dot < 0
//   rounds   Borůvka on the keys.  Every component takes its smallest outgoing key and hooks to the other side (in a
//            mutual pair the smaller representative stays the root); the hook carries the parity rel(u) ^ f ^ rel(v);
//            every hooking representative chases its pointer to the new root, accumulating the parity; every vertex
//            then takes its representative's root and parity.  rel(v) is thus the XOR of the flip bits along the
//            spanning-tree path from v to its representative, without rooting the tree or walking it level by level.
//            Edges inside one component are dropped by a stable compaction, so every round reads fewer.
//   finish   the seed of every component (largest z, then smallest index: one packed 64-bit atomicMax), flip(v) =
//            rel(v) ^ rel(seed) ^ (seed's unit normal z < 0), and the output: the input normals with the sign of the
//            flipped rows negated.
//
// The minimum-key atomics of a round go to one slot per component; once one component holds most of the cloud, most
// edges target its slot.  The lanes of a warp that target the same slot are therefore reduced first (__match_any_sync,
// then two __reduce_*_sync over the key's halves) and one lane per slot issues the atomic.  Minimum and maximum do not
// depend on the order of the atomics, so every result is the same on every run.
#include <cub/cub.cuh>
#include "cloud_common.cuh"

namespace {

constexpr int OB = 256;  // threads per CTA of every kernel here
constexpr uint64_t NO_KEY = ~0ull;
constexpr uint32_t PARENT_MASK = 0x7FFFFFFFu;  // packed hook: parent | parity << 31
constexpr uint32_t PARITY_BIT = 0x80000000u;

inline unsigned grid_of(int64_t n) { return (unsigned)((n + OB - 1) / OB); }

// every lane of the warp calls; the lanes with the same slot >= 0 fold their values and one of them issues the atomic
template <bool MAX>
__device__ __forceinline__ void warp_atomic_u64(unsigned long long* base, int slot, uint64_t v) {
    const unsigned peers = __match_any_sync(0xffffffffu, slot);
    const unsigned hi = (unsigned)(v >> 32), lo = (unsigned)v;
    const unsigned bhi = MAX ? __reduce_max_sync(peers, hi) : __reduce_min_sync(peers, hi);
    const unsigned cand = hi == bhi ? lo : (MAX ? 0u : 0xffffffffu);
    const unsigned blo = MAX ? __reduce_max_sync(peers, cand) : __reduce_min_sync(peers, cand);
    if (slot >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) {
        const unsigned long long b = (unsigned long long)bhi << 32 | blo;
        if (MAX) atomicMax(base + slot, b); else atomicMin(base + slot, b);
    }
}

// every lane of the warp calls; adds the number of lanes with `flag` to *counter
__device__ __forceinline__ void warp_count(unsigned long long* counter, bool flag) {
    const unsigned b = __ballot_sync(0xffffffffu, flag);
    if ((threadIdx.x & 31) == 0 && b) atomicAdd(counter, (unsigned long long)__popc(b));
}

// unit normal of row i in float64 (the N6 splat's expression); false when the normal is zero or not finite
template <typename NT>
__device__ __forceinline__ bool unit_normal(const NT* __restrict__ nrm, int64_t i, double (&nh)[3]) {
    const double nx = (double)nrm[3 * i], ny = (double)nrm[3 * i + 1], nz = (double)nrm[3 * i + 2];
    const double s = sqrt(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz)));
    if (!(s > 0.0) || !isfinite(s)) return false;
    nh[0] = __ddiv_rn(nx, s); nh[1] = __ddiv_rn(ny, s); nh[2] = __ddiv_rn(nz, s);
    return true;
}

// ---- prepare ----------------------------------------------------------------------------------------------------
template <typename NT>
__global__ void __launch_bounds__(OB) usable_kernel(const float* __restrict__ xyz, const NT* __restrict__ nrm, int64_t n,
                                                    uint8_t* __restrict__ flag) {
    const int64_t i = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (i >= n) return;
    double nh[3];
    flag[i] = finite3(xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2]) && unit_normal(nrm, i, nh);
}

template <typename NT>
__global__ void __launch_bounds__(OB) compact_kernel(const float* __restrict__ xyz, const NT* __restrict__ nrm,
                                                     int64_t n, const int32_t* __restrict__ rows,
                                                     const int64_t* __restrict__ count, float* __restrict__ uxyz,
                                                     double* __restrict__ unh) {
    const int64_t t = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (t >= *count) return;
    const int64_t i = rows[t];
    double nh[3];
    unit_normal(nrm, i, nh);
    for (int a = 0; a < 3; ++a) { uxyz[3 * t + a] = xyz[3 * i + a]; unh[3 * t + a] = nh[a]; }
}

// ---- edges ------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OB) candidate_kernel(const int32_t* __restrict__ ids, int64_t m, int k, int kp,
                                                       uint64_t* __restrict__ cand) {
    const int64_t t = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (t >= m * kp) return;
    const int64_t i = t / kp, r = t - i * kp;
    const uint32_t a = (uint32_t)i, b = (uint32_t)ids[i * k + r];
    cand[t] = a < b ? (uint64_t)a << 32 | b : (uint64_t)b << 32 | a;
}

// key and flip bit of edge e < E; the slots E..c-1 get NO_KEY, which every round drops
__global__ void __launch_bounds__(OB) edge_key_kernel(const uint64_t* __restrict__ edges, const int64_t* __restrict__ count,
                                                      int64_t c, const double* __restrict__ unh,
                                                      uint64_t* __restrict__ keys, uint8_t* __restrict__ flips) {
    const int64_t e = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (e >= c) return;
    if (e >= *count) { keys[e] = NO_KEY; return; }
    const uint64_t uv = edges[e];
    const double* a = unh + 3 * (uv >> 32);
    const double* b = unh + 3 * (uv & 0xFFFFFFFFu);
    const double dot = __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
    const double w = fmax(0.0, __dsub_rn(1.0, fabs(dot)));
    keys[e] = (uint64_t)__float_as_uint(__double2float_rn(w)) << 32 | (uint64_t)e;
    flips[e] = dot < 0.0;
}

// ---- Borůvka rounds ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OB) init_kernel(int64_t m, int32_t* __restrict__ comp, uint8_t* __restrict__ rel) {
    const int64_t v = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (v >= m) return;
    comp[v] = (int32_t)v;
    rel[v] = 0;
}

__global__ void __launch_bounds__(OB) fill_u64_kernel(uint64_t* __restrict__ p, int64_t n, uint64_t v) {
    const int64_t i = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (i < n) p[i] = v;
}

// every active edge: live = its ends lie in different components; a live edge offers its key to both components
__global__ void __launch_bounds__(OB) min_edge_kernel(const uint64_t* __restrict__ cur, int64_t active,
                                                      const uint64_t* __restrict__ edges, const int32_t* __restrict__ comp,
                                                      uint8_t* __restrict__ live, unsigned long long* __restrict__ best) {
    const int64_t i = (int64_t)blockIdx.x * OB + threadIdx.x;
    uint64_t key = NO_KEY;
    int cu = -1, cv = -1;
    if (i < active) {
        key = cur[i];
        bool ok = false;
        if (key != NO_KEY) {
            const uint64_t uv = edges[(uint32_t)key];
            cu = comp[uv >> 32];
            cv = comp[uv & 0xFFFFFFFFu];
            ok = cu != cv;
        }
        live[i] = ok;
        if (!ok) { key = NO_KEY; cu = cv = -1; }
    }
    warp_atomic_u64<false>(best, cu, key);
    warp_atomic_u64<false>(best, cv, key);
}

// every representative c with an outgoing edge hooks to the component across its smallest key, unless that component
// chose the same edge and has the larger representative; packed[c] = parent | parity << 31 (a root: c itself)
__global__ void __launch_bounds__(OB) hook_kernel(int64_t m, const uint64_t* __restrict__ edges,
                                                  const uint8_t* __restrict__ flips, const int32_t* __restrict__ comp,
                                                  const uint8_t* __restrict__ rel, const uint64_t* __restrict__ best,
                                                  uint32_t* __restrict__ packed, uint8_t* __restrict__ mst,
                                                  unsigned long long* __restrict__ hooked) {
    const int64_t c = (int64_t)blockIdx.x * OB + threadIdx.x;
    bool hook = false;
    if (c < m && comp[c] == (int32_t)c) {
        uint32_t x = (uint32_t)c;
        const uint64_t b = best[c];
        if (b != NO_KEY) {
            const uint32_t e = (uint32_t)b;
            const uint64_t uv = edges[e];
            const uint32_t u = (uint32_t)(uv >> 32), w = (uint32_t)(uv & 0xFFFFFFFFu);
            const int32_t cu = comp[u], cw = comp[w];
            const int32_t other = cu == (int32_t)c ? cw : cu;
            if (!(best[other] == b && (int32_t)c < other)) {
                x = (uint32_t)other | (uint32_t)(rel[u] ^ flips[e] ^ rel[w]) << 31;
                mst[e] = 1;
                hook = true;
            }
        }
        packed[c] = x;
    }
    warp_count(hooked, hook);
}

// every representative follows its hooks to the root, XOR-ing the parities.  Each step stores the shortcut, so chains
// that other threads walk get shorter while they run; a 32-bit word always holds a consistent (ancestor, parity) pair.
__global__ void __launch_bounds__(OB) chase_kernel(int64_t m, const int32_t* __restrict__ comp, uint32_t* packed_) {
    const int64_t c = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (c >= m || comp[c] != (int32_t)c) return;
    volatile uint32_t* packed = packed_;
    uint32_t x = packed[c];
    for (;;) {
        const uint32_t p = x & PARENT_MASK;
        const uint32_t y = packed[p];
        if ((y & PARENT_MASK) == p) break;  // p is a root (c itself when c did not hook)
        x = (y & PARENT_MASK) | ((x ^ y) & PARITY_BIT);
        packed[c] = x;
    }
}

__global__ void __launch_bounds__(OB) relabel_kernel(int64_t m, const uint32_t* __restrict__ packed,
                                                     int32_t* __restrict__ comp, uint8_t* __restrict__ rel) {
    const int64_t v = (int64_t)blockIdx.x * OB + threadIdx.x;
    if (v >= m) return;
    const uint32_t x = packed[comp[v]];
    comp[v] = (int32_t)(x & PARENT_MASK);
    rel[v] ^= (uint8_t)(x >> 31);
}

// ---- finish -----------------------------------------------------------------------------------------------------
// z as an unsigned key ordered like the float (-0 counts as +0), then the complement of the index: the largest packed
// value is the largest z with the smallest index
__device__ __forceinline__ uint64_t seed_key(float z, uint32_t v) {
    const uint32_t u = __float_as_uint(z == 0.f ? 0.f : z);
    const uint32_t o = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (uint64_t)o << 32 | (0xFFFFFFFFu - v);
}

__global__ void __launch_bounds__(OB) seed_kernel(const float* __restrict__ uxyz, int64_t m,
                                                  const int32_t* __restrict__ comp, unsigned long long* __restrict__ seed,
                                                  unsigned long long* __restrict__ stats) {
    const int64_t v = (int64_t)blockIdx.x * OB + threadIdx.x;
    int root = -1;
    uint64_t key = 0;
    if (v < m) {
        root = comp[v];
        key = seed_key(uxyz[3 * v + 2], (uint32_t)v);
    }
    warp_atomic_u64<true>(seed, root, key);
    warp_count(&stats[0], v < m && root == (int32_t)v);
}

template <typename NT>
__global__ void __launch_bounds__(OB) flip_kernel(const double* __restrict__ unh, const int32_t* __restrict__ rows,
                                                  int64_t m, const int32_t* __restrict__ comp,
                                                  const uint8_t* __restrict__ rel, const uint64_t* __restrict__ seed,
                                                  const NT* __restrict__ nrm, NT* __restrict__ out,
                                                  int32_t* __restrict__ seed_out, uint8_t* __restrict__ rel_out,
                                                  unsigned long long* __restrict__ stats) {
    const int64_t v = (int64_t)blockIdx.x * OB + threadIdx.x;
    bool flip = false;
    if (v < m) {
        const uint32_t s = 0xFFFFFFFFu - (uint32_t)seed[comp[v]];
        const uint8_t r = rel[v] ^ rel[s];
        flip = (r ^ (unh[3 * (int64_t)s + 2] < 0.0)) != 0;
        if (flip) {
            const int64_t i = rows[v];
            for (int a = 0; a < 3; ++a) out[3 * i + a] = -nrm[3 * i + a];
        }
        if (seed_out) seed_out[v] = (int32_t)s;
        if (rel_out) rel_out[v] = r;
    }
    warp_count(&stats[1], flip);
}

// ---- workspaces -------------------------------------------------------------------------------------------------
struct PrepWs {
    uint8_t* flag;
    void* tmp;
    size_t tmp_bytes, bytes;
};

PrepWs prep_ws(void* base, int64_t n) {
    size_t sel = 0;
    cub::DeviceSelect::Flagged(nullptr, sel, cub::CountingInputIterator<int32_t>(0), (const uint8_t*)nullptr,
                               (int32_t*)nullptr, (int64_t*)nullptr, n);
    WsCarve w{(char*)base};
    PrepWs l;
    l.flag = w.take<uint8_t>(n);
    l.tmp_bytes = WsCarve::pad(sel);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct EdgeWs {
    uint64_t *cand, *sorted;
    void* tmp;
    size_t tmp_bytes, bytes;
};

EdgeWs edge_ws(void* base, int64_t c) {
    size_t sort_b = 0, uniq_b = 0;
    cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const uint64_t*)nullptr, (uint64_t*)nullptr, c, 0, 64);
    cub::DeviceSelect::Unique(nullptr, uniq_b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t*)nullptr, c);
    WsCarve w{(char*)base};
    EdgeWs l;
    l.cand = w.take<uint64_t>(c);
    l.sorted = w.take<uint64_t>(c);
    l.tmp_bytes = WsCarve::pad(sort_b > uniq_b ? sort_b : uniq_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct RoundWs {
    uint64_t* act[2];  // the active keys: round r reads act[r & 1] (round 0 reads the caller's keys), writes the other
    uint8_t* live;
    uint64_t* best;
    uint32_t* packed;
    void* tmp;
    size_t tmp_bytes, bytes;
};

RoundWs round_ws(void* base, int64_t m, int64_t c) {
    size_t sel = 0;
    cub::DeviceSelect::Flagged(nullptr, sel, (const uint64_t*)nullptr, (const uint8_t*)nullptr, (uint64_t*)nullptr,
                               (int64_t*)nullptr, c);
    WsCarve w{(char*)base};
    RoundWs l;
    l.act[0] = w.take<uint64_t>(c);
    l.act[1] = w.take<uint64_t>(c);
    l.live = w.take<uint8_t>(c);
    l.best = w.take<uint64_t>(m);
    l.packed = w.take<uint32_t>(m);
    l.tmp_bytes = WsCarve::pad(sel);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

struct FinishWs {
    uint64_t* seed;
    size_t bytes;
};

FinishWs finish_ws(void* base, int64_t m) {
    WsCarve w{(char*)base};
    FinishWs l;
    l.seed = w.take<uint64_t>(m);
    l.bytes = w.used;
    return l;
}

}  // namespace

extern "C" int64_t g2pc_orient_prepare_workspace_bytes(int64_t n) {
    return n <= 0 ? 0 : (int64_t)prep_ws(nullptr, n).bytes;
}

extern "C" int g2pc_orient_prepare(const float* xyz, const void* normals, int normal_dtype, int64_t n, int32_t* rows,
                                   float* uxyz, double* unh, int64_t* count, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(n < 0x7FFFFFFFll, "n must fit int32 indices");
    G2PC_CHECK_ARG(normal_dtype == G2PC_F32 || normal_dtype == G2PC_F64, "normals must be float32 or float64");
    G2PC_CHECK_ARG(count, "null count");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(count, 0, sizeof(int64_t), st));
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(xyz && normals && rows && uxyz && unh && workspace, "null pointer");
    const PrepWs l = prep_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    if (normal_dtype == G2PC_F32)
        usable_kernel<<<grid_of(n), OB, 0, st>>>(xyz, (const float*)normals, n, l.flag);
    else
        usable_kernel<<<grid_of(n), OB, 0, st>>>(xyz, (const double*)normals, n, l.flag);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceSelect::Flagged(l.tmp, b, cub::CountingInputIterator<int32_t>(0), l.flag, rows, count, n, st));
    if (normal_dtype == G2PC_F32)
        compact_kernel<<<grid_of(n), OB, 0, st>>>(xyz, (const float*)normals, n, rows, count, uxyz, unh);
    else
        compact_kernel<<<grid_of(n), OB, 0, st>>>(xyz, (const double*)normals, n, rows, count, uxyz, unh);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

namespace {
int64_t edge_capacity(int64_t m, int32_t k) { return m <= 1 ? 0 : m * (int64_t)(k < m - 1 ? k : m - 1); }
}  // namespace

extern "C" int64_t g2pc_orient_edges_workspace_bytes(int64_t m, int32_t k) {
    const int64_t c = edge_capacity(m, k);
    return c <= 0 ? 0 : (int64_t)edge_ws(nullptr, c).bytes;
}

extern "C" int g2pc_orient_edges(const int32_t* ids, int64_t m, int32_t k, const double* unh, uint64_t* edges,
                                 uint64_t* keys, uint8_t* flips, int64_t* count, void* workspace,
                                 int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(m >= 0 && m < 0x7FFFFFFFll, "m must be in 0..2^31-2");
    G2PC_CHECK_ARG(k >= 1 && k <= G2PC_ORIENT_K_MAX, "k must be in 1..G2PC_ORIENT_K_MAX");
    G2PC_CHECK_ARG(count, "null count");
    const int64_t c = edge_capacity(m, k);
    G2PC_CHECK_ARG(c < 0xFFFFFFFFll, "m * min(k, m - 1) must be below 2^32 (edge numbers are 32-bit)");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(count, 0, sizeof(int64_t), st));
    if (c == 0) return G2PC_OK;
    G2PC_CHECK_ARG(ids && unh && edges && keys && flips && workspace, "null pointer");
    const EdgeWs l = edge_ws(workspace, c);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    const int kp = (int)(c / m);
    candidate_kernel<<<grid_of(c), OB, 0, st>>>(ids, m, k, kp, l.cand);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, l.cand, l.sorted, c, 0, 64, st));
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceSelect::Unique(l.tmp, b, l.sorted, edges, count, c, st));
    edge_key_kernel<<<grid_of(c), OB, 0, st>>>(edges, count, c, unh, keys, flips);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_orient_round_workspace_bytes(int64_t m, int64_t c) {
    return m <= 0 ? 0 : (int64_t)round_ws(nullptr, m, c).bytes;
}

extern "C" int g2pc_orient_round(const uint64_t* edges, const uint64_t* keys, const uint8_t* flips, int64_t m, int64_t c,
                                 int32_t round_index, int64_t active, int32_t* comp, uint8_t* rel, uint8_t* mst,
                                 int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(m >= 1 && m < 0x7FFFFFFFll, "m must be in 1..2^31-2");
    G2PC_CHECK_ARG(c >= 0 && c < 0xFFFFFFFFll && round_index >= 0, "bad edge capacity or round");
    G2PC_CHECK_ARG(active >= 0 && active <= c && (round_index > 0 || active == c), "active must be c in round 0, <= c after");
    G2PC_CHECK_ARG(comp && rel && counts && workspace && (c == 0 || (edges && keys && flips && mst)), "null pointer");
    const RoundWs l = round_ws(workspace, m, c);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (round_index == 0) {
        init_kernel<<<grid_of(m), OB, 0, st>>>(m, comp, rel);
        G2PC_CHECK_LAUNCH();
        if (c) G2PC_CUDA(cudaMemsetAsync(mst, 0, (size_t)c, st));
    }
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), st));
    if (active == 0) return G2PC_OK;
    const uint64_t* cur = round_index == 0 ? keys : l.act[round_index & 1];
    uint64_t* next = l.act[(round_index + 1) & 1];
    fill_u64_kernel<<<grid_of(m), OB, 0, st>>>(l.best, m, NO_KEY);
    G2PC_CHECK_LAUNCH();
    min_edge_kernel<<<grid_of(active), OB, 0, st>>>(cur, active, edges, comp, l.live, (unsigned long long*)l.best);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceSelect::Flagged(l.tmp, b, cur, l.live, next, counts + 1, active, st));
    hook_kernel<<<grid_of(m), OB, 0, st>>>(m, edges, flips, comp, rel, l.best, l.packed, mst,
                                           (unsigned long long*)counts);
    G2PC_CHECK_LAUNCH();
    chase_kernel<<<grid_of(m), OB, 0, st>>>(m, comp, l.packed);
    G2PC_CHECK_LAUNCH();
    relabel_kernel<<<grid_of(m), OB, 0, st>>>(m, l.packed, comp, rel);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_orient_finish_workspace_bytes(int64_t m) {
    return m <= 0 ? 0 : (int64_t)finish_ws(nullptr, m).bytes;
}

extern "C" int g2pc_orient_finish(const float* uxyz, const double* unh, const int32_t* rows, int64_t m,
                                  const void* normals, int normal_dtype, int64_t n, const int32_t* comp,
                                  const uint8_t* rel, void* out, int32_t* seed, uint8_t* seed_rel, int64_t* stats,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0 && m >= 0 && m <= n && n < 0x7FFFFFFFll, "need 0 <= m <= n < 2^31 - 1");
    G2PC_CHECK_ARG(normal_dtype == G2PC_F32 || normal_dtype == G2PC_F64, "normals must be float32 or float64");
    G2PC_CHECK_ARG(stats, "null stats");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(stats, 0, 2 * sizeof(int64_t), st));
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(normals && out, "null pointer");
    const size_t es = normal_dtype == G2PC_F32 ? sizeof(float) : sizeof(double);
    G2PC_CUDA(cudaMemcpyAsync(out, normals, (size_t)n * 3 * es, cudaMemcpyDeviceToDevice, st));
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(uxyz && unh && rows && comp && rel && workspace, "null pointer");
    const FinishWs l = finish_ws(workspace, m);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    unsigned long long* s = (unsigned long long*)stats;
    fill_u64_kernel<<<grid_of(m), OB, 0, st>>>(l.seed, m, 0);
    G2PC_CHECK_LAUNCH();
    seed_kernel<<<grid_of(m), OB, 0, st>>>(uxyz, m, comp, (unsigned long long*)l.seed, s);
    G2PC_CHECK_LAUNCH();
    if (normal_dtype == G2PC_F32)
        flip_kernel<<<grid_of(m), OB, 0, st>>>(unh, rows, m, comp, rel, l.seed, (const float*)normals, (float*)out, seed,
                                               seed_rel, s);
    else
        flip_kernel<<<grid_of(m), OB, 0, st>>>(unh, rows, m, comp, rel, l.seed, (const double*)normals, (double*)out,
                                               seed, seed_rel, s);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

// ---- normals turned toward the camera that saw each Gaussian best ----------------------------------------------
// One grid-stride pass.  Row r reads f = cam_of[ids[r]]; a row whose id or camera index is out of range is invalid, a row
// with f == INT32_MAX unseen; both are copied.  Otherwise dot = (nx*dx + ny*dy) + nz*dz with d = c_f - mu, in float64
// from the stored values without FMA: dot < 0 negates the row, dot == 0 or NaN leaves it (undecided).  Each thread counts
// its rows; at the end every warp folds its counts and one lane issues the four atomics.
namespace {

constexpr int FC_CTAS_MAX = 1024;

template <typename NT>
__global__ void __launch_bounds__(OB) face_cameras_kernel(const float* __restrict__ means, const NT* __restrict__ nrm,
                                                          const int32_t* __restrict__ ids, int64_t m,
                                                          const int32_t* __restrict__ cam_of, int64_t n,
                                                          const float* __restrict__ cams, int64_t ncam,
                                                          NT* __restrict__ out, unsigned long long* __restrict__ counts) {
    unsigned c[4] = {0u, 0u, 0u, 0u};  // flipped, unseen, undecided, invalid
    const int64_t stride = (int64_t)gridDim.x * OB;
    for (int64_t r = (int64_t)blockIdx.x * OB + threadIdx.x; r < m; r += stride) {
        const NT x = nrm[3 * r], y = nrm[3 * r + 1], z = nrm[3 * r + 2];
        bool flip = false;
        const int32_t g = ids[r];
        if (g < 0 || g >= n) {
            ++c[3];
        } else {
            const int32_t f = cam_of[g];
            if (f == INT32_MAX) {
                ++c[1];
            } else if (f < 0 || f >= ncam) {
                ++c[3];
            } else {
                const double dx = __dsub_rn((double)cams[3 * (int64_t)f], (double)means[3 * r]);
                const double dy = __dsub_rn((double)cams[3 * (int64_t)f + 1], (double)means[3 * r + 1]);
                const double dz = __dsub_rn((double)cams[3 * (int64_t)f + 2], (double)means[3 * r + 2]);
                const double dot = __dadd_rn(__dadd_rn(__dmul_rn((double)x, dx), __dmul_rn((double)y, dy)),
                                             __dmul_rn((double)z, dz));
                flip = dot < 0.0;
                if (flip) ++c[0];
                else if (!(dot > 0.0)) ++c[2];
            }
        }
        out[3 * r] = flip ? -x : x;
        out[3 * r + 1] = flip ? -y : y;
        out[3 * r + 2] = flip ? -z : z;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const unsigned s = __reduce_add_sync(0xffffffffu, c[k]);
        if ((threadIdx.x & 31) == 0 && s) atomicAdd(counts + k, (unsigned long long)s);
    }
}

}  // namespace

extern "C" int g2pc_face_cameras(const float* means, const void* normals, int normal_dtype, const int32_t* ids,
                                 int64_t m, const int32_t* cam_of, int64_t n, const float* cams, int64_t ncam,
                                 void* out, int64_t* counts, void* stream) {
    G2PC_CHECK_ARG(m >= 0 && n >= 0 && ncam >= 0, "m, n and ncam must be >= 0");
    G2PC_CHECK_ARG(normal_dtype == G2PC_F32 || normal_dtype == G2PC_F64, "normals must be float32 or float64");
    if (m == 0) return G2PC_OK;
    G2PC_CHECK_ARG(means && normals && ids && out && counts && (n == 0 || cam_of) && (ncam == 0 || cams),
                   "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 4 * sizeof(int64_t), st));
    const unsigned grid = grid_of(m) < (unsigned)FC_CTAS_MAX ? grid_of(m) : (unsigned)FC_CTAS_MAX;
    unsigned long long* cnt = (unsigned long long*)counts;
    if (normal_dtype == G2PC_F32)
        face_cameras_kernel<<<grid, OB, 0, st>>>(means, (const float*)normals, ids, m, cam_of, n, cams, ncam,
                                                 (float*)out, cnt);
    else
        face_cameras_kernel<<<grid, OB, 0, st>>>(means, (const double*)normals, ids, m, cam_of, n, cams, ncam,
                                                 (double*)out, cnt);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
