// s9_clean.cu — statistical outlier removal of the finished point cloud (--clean_pointcloud): exact k-nearest-neighbour
// mean distances and the keep mask.
//
// Reference semantics restated (not copied):
//   gauss_to_pc.py:743-759   the clean runs once on the whole cloud after generation
//   mesh_handler.py:89-94    clean_point_cloud -> Open3D PointCloud::RemoveStatisticalOutliers(nb_neighbors=20, std_ratio)
// avg[i] = (sum of sqrt(d2) over the k smallest d2 of point i, self included, ascending) / min(k, n), d2 in float64 as
// (dx*dx + dy*dy) + dz*dz of the upcast float32 coordinates; keep[i] = avg[i] > 0 && avg[i] < mean + std_ratio * std.
//
// Index: an implicit linear octree.  Every point gets a 126-bit Morton key: 42 bits per axis over a cube of power-of-two
// edge E that holds the bounding box, split into two 63-bit words (hi = the top 21 bits of each axis, lo = the low 21).
// Two stable cub radix sorts (lo first, then hi) order the points by the full key, so every octree cell at every level
// 0..42 is one contiguous range of the sorted array.  Exact duplicates share their key and sit next to each other.
//
// Query (one thread per sorted point, so a warp holds 32 spatial neighbours): the WIN = 2*K_MAX sorted neighbours around
// the query are scanned first, which gives a tight k-th distance at once and answers a query with >= k exact copies
// (k-th distance 0) without any further work.  Then a stackless walk of the octree in Morton order: a cell whose box is
// not nearer than the current k-th distance is skipped without touching memory; otherwise its range is found by
// galloping search from the previous position, and it is scanned if it holds <= LEAF_T points (or is a 42-bit cell),
// else entered.  The k smallest d2 live in registers; indices are not needed (only the multiset of distances matters).
// g2pc_knn_ids (the normal orientation, N7) runs the same index and walk with a register list of (d2, row id) pairs
// instead, ordered lexicographically over the other points, and writes the ids.
// Box distances are lowered by a margin of E * 2^-48, which covers the rounding of the quantisation and of the distance
// arithmetic, so a cell is skipped only when no point in it can enter the list: the result is exact.
#include <cub/cub.cuh>
#include "cloud_common.cuh"

namespace {

typedef unsigned __int128 u128;

constexpr int K_MAX = G2PC_SOR_K_MAX;
constexpr int WIN = 2 * K_MAX;     // a run of >= k exact copies through the query always lies K_MAX deep in the window
constexpr int LEAF_T = 32;         // a cell with at most this many points is scanned, a larger one is entered
constexpr int QBITS = 42;          // quantisation bits per axis (deepest octree level)
constexpr int QB = 128;            // query threads per CTA
constexpr int BB = 256;            // key / gather threads per CTA
constexpr uint64_t MASK21 = (1ull << 21) - 1;
constexpr uint64_t KEY_NONFINITE = (1ull << 63) - 1;  // non-finite points sort last and are nobody's neighbour

struct Frame {
    double lo[3];   // bounding-box minimum (finite points)
    double scale;   // 2^42 / E
    double edge;    // E: power of two >= the largest bounding-box extent
    double margin;  // E * 2^-48
};

// 21-bit integer -> every third bit of 63
__device__ __forceinline__ uint64_t spread3(uint64_t v) {
    v &= MASK21;
    v = (v | v << 32) & 0x001f00000000ffffull;
    v = (v | v << 16) & 0x001f0000ff0000ffull;
    v = (v | v << 8) & 0x100f00f00f00f00full;
    v = (v | v << 4) & 0x10c30c30c30c30c3ull;
    v = (v | v << 2) & 0x1249249249249249ull;
    return v;
}

__device__ __forceinline__ uint64_t morton63(uint64_t x, uint64_t y, uint64_t z) {
    return spread3(x) << 2 | spread3(y) << 1 | spread3(z);
}

// 126-bit key of the 42-bit cell coordinates (x, y, z)
__device__ __forceinline__ u128 key126(uint64_t x, uint64_t y, uint64_t z) {
    return (u128)morton63(x >> 21, y >> 21, z >> 21) << 63 | morton63(x & MASK21, y & MASK21, z & MASK21);
}

// one thread: fold the per-CTA boxes into the quantisation frame
__global__ void frame_kernel(const float* __restrict__ part, int nb, Frame* __restrict__ fr) {
    float mn[3], mx[3];
    fold_bbox(part, nb, mn, mx);
    Frame f;
    double ext = 0.0;
    if (mn[0] <= mx[0]) {
        for (int a = 0; a < 3; ++a) { f.lo[a] = mn[a]; ext = fmax(ext, (double)mx[a] - (double)mn[a]); }
    } else {  // no finite point
        f.lo[0] = f.lo[1] = f.lo[2] = 0.0;
    }
    int e = 0;
    if (ext > 0.0) frexp(ext, &e);  // ext < 2^e
    f.edge = ldexp(1.0, e);
    f.scale = ldexp(1.0, QBITS - e);
    f.margin = ldexp(1.0, e - 48);
    *fr = f;
}

// hi / lo key words per input row, idx = row; non-finite rows get KEY_NONFINITE and are counted in status[0]
__global__ void __launch_bounds__(BB) key_kernel(const float* __restrict__ xyz, int64_t n, const Frame* __restrict__ fr,
                                                 uint64_t* __restrict__ hi, uint64_t* __restrict__ lo,
                                                 uint32_t* __restrict__ idx, int32_t* __restrict__ status) {
    const int64_t i = (int64_t)blockIdx.x * BB + threadIdx.x;
    if (i >= n) return;
    const float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    idx[i] = (uint32_t)i;
    if (!finite3(x, y, z)) {
        hi[i] = KEY_NONFINITE; lo[i] = KEY_NONFINITE;
        atomicAdd(status, 1);
        return;
    }
    const double top = 4398046511103.0;  // 2^42 - 1
    uint64_t q[3];
    const float c[3] = {x, y, z};
    for (int a = 0; a < 3; ++a) {
        const double u = ((double)c[a] - fr->lo[a]) * fr->scale;
        q[a] = (uint64_t)fmin(fmax(u, 0.0), top);
    }
    hi[i] = morton63(q[0] >> 21, q[1] >> 21, q[2] >> 21);
    lo[i] = morton63(q[0] & MASK21, q[1] & MASK21, q[2] & MASK21);
}

__global__ void __launch_bounds__(BB) gather_u64_kernel(const uint64_t* __restrict__ src, const uint32_t* __restrict__ idx,
                                                        int64_t n, uint64_t* __restrict__ dst) {
    const int64_t j = (int64_t)blockIdx.x * BB + threadIdx.x;
    if (j < n) dst[j] = src[idx[j]];
}

// sorted index -> (lo, hi) key pair and the point as float4, its row id in the bits of w
__global__ void __launch_bounds__(BB) gather_sorted_kernel(const uint64_t* __restrict__ hi_sorted,
                                                           const uint64_t* __restrict__ lo, const uint32_t* __restrict__ idx,
                                                           const float* __restrict__ xyz, int64_t n,
                                                           ulonglong2* __restrict__ keys, float4* __restrict__ pts) {
    const int64_t j = (int64_t)blockIdx.x * BB + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = idx[j];
    keys[j] = make_ulonglong2(lo[i], hi_sorted[j]);
    pts[j] = make_float4(xyz[3 * (int64_t)i], xyz[3 * (int64_t)i + 1], xyz[3 * (int64_t)i + 2], __uint_as_float(i));
}

__device__ __forceinline__ u128 key_at(const ulonglong2* __restrict__ keys, int j) {
    const ulonglong2 v = keys[j];
    return (u128)v.y << 63 | v.x;
}

// first j in [a, n) with key(j) >= K (n if none): galloping from a, then bisection
__device__ __forceinline__ int lower_bound_from(const ulonglong2* __restrict__ keys, int a, int n, u128 K) {
    if (a >= n || key_at(keys, a) >= K) return a;
    int lo = a, hi, step = 1;  // key(lo) < K
    for (;;) {
        if (step >= n - lo) { hi = n; break; }
        hi = lo + step;
        if (key_at(keys, hi) >= K) break;
        lo = hi;
        step <<= 1;
    }
    while (hi - lo > 1) {
        const int mid = lo + ((hi - lo) >> 1);
        if (key_at(keys, mid) < K) lo = mid; else hi = mid;
    }
    return hi;
}

// float64 d2 of two float32 points, in the order of the restatements: (dx*dx + dy*dy) + dz*dz
__device__ __forceinline__ double dist2(const float4 q, const float4 p) {
    const double dx = __dsub_rn((double)q.x, (double)p.x), dy = __dsub_rn((double)q.y, (double)p.y),
                 dz = __dsub_rn((double)q.z, (double)p.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// The register list of a query: the k smallest d2 (N5, the query itself included).  d[] holds them ascending in its
// LAST k slots (the others are -inf), so the k-th distance is always d[K_MAX - 1] and every index below is a
// compile-time constant (the list stays in registers).
struct DistList {
    double d[K_MAX];
    __device__ __forceinline__ void init(int kp) {
#pragma unroll
        for (int j = 0; j < K_MAX; ++j) d[j] = j >= K_MAX - kp ? INFINITY : -INFINITY;
    }
    __device__ __forceinline__ double kth() const { return d[K_MAX - 1]; }
    __device__ __forceinline__ void consider(const float4 q, const float4 p) {
        const double d2 = dist2(q, p);
        if (d2 < d[K_MAX - 1]) {  // insert, dropping the largest: new[j] = max(old[j-1], min(old[j], d2))
#pragma unroll
            for (int j = K_MAX - 1; j > 0; --j) d[j] = fmax(d[j - 1], fmin(d[j], d2));
            d[0] = fmin(d[0], d2);
        }
    }
};

// The k smallest (d2, id) pairs in lexicographic order over the other points (g2pc_knn_ids): ties of d2 go to the
// smaller row id, so the list is unique.  The row id of every sorted point travels in the bits of its float4's w.
struct IdList {
    double d[K_MAX];
    uint32_t id[K_MAX];
    uint32_t self;
    __device__ __forceinline__ void init(int kp) {
#pragma unroll
        for (int j = 0; j < K_MAX; ++j) { d[j] = j >= K_MAX - kp ? INFINITY : -INFINITY; id[j] = 0xFFFFFFFFu; }
    }
    __device__ __forceinline__ double kth() const { return d[K_MAX - 1]; }
    static __device__ __forceinline__ bool less(double ad, uint32_t ai, double bd, uint32_t bi) {
        return ad < bd || (ad == bd && ai < bi);
    }
    __device__ __forceinline__ bool contains(uint32_t j) const {
        bool c = false;
#pragma unroll
        for (int s = 0; s < K_MAX; ++s) c |= id[s] == j && d[s] != -INFINITY;
        return c;
    }
    __device__ __forceinline__ void consider(const float4 q, const float4 p) {
        const uint32_t j = __float_as_uint(p.w);
        if (j == self) return;
        const double d2 = dist2(q, p);
        if (!less(d2, j, d[K_MAX - 1], id[K_MAX - 1])) return;
#pragma unroll
        for (int s = K_MAX - 1; s > 0; --s) {
            const bool lo = less(d2, j, d[s], id[s]);  // min(old[s], x)
            const double md = lo ? d2 : d[s];
            const uint32_t mi = lo ? j : id[s];
            const bool up = less(d[s - 1], id[s - 1], md, mi);  // max(old[s-1], that)
            d[s] = up ? md : d[s - 1];
            id[s] = up ? mi : id[s - 1];
        }
        if (less(d2, j, d[0], id[0])) { d[0] = d2; id[0] = j; }
    }
};

template <class List>
__device__ __forceinline__ void scan_range(List& best, const float4 q, const float4* __restrict__ pts, int j0, int j1) {
    for (int j = j0; j < j1; ++j) best.consider(q, pts[j]);
}

// distance of the shifted query s from the cell [c*w, (c+1)*w] along one axis, lowered by the margin
__device__ __forceinline__ double axis_gap(double s, uint64_t c, double w, double margin) {
    const double lo = (double)c * w, hi = (double)(c + 1) * w;
    const double g = fmax(fmax(lo - s, s - hi), 0.0);
    return fmax(g - margin, 0.0);
}

// The search of sorted point t: its window, then the stackless octree walk.  One copy for both lists.
template <class List>
__device__ __forceinline__ void knn_query(List& best, const ulonglong2* __restrict__ keys, const float4* __restrict__ pts,
                                          const Frame& fr, int n, int t, const float4 q) {
    const int W = n < WIN ? n : WIN;
    int w0 = t - WIN / 2;
    w0 = w0 < 0 ? 0 : (w0 > n - W ? n - W : w0);
    const int w1 = w0 + W;
    scan_range(best, q, pts, w0, w1);

    // the same shifted frame as the quantisation
    const double sx = (double)q.x - fr.lo[0], sy = (double)q.y - fr.lo[1], sz = (double)q.z - fr.lo[2];
    int L = 1, a = 0;
    uint64_t cx = 0, cy = 0, cz = 0;
    double w = fr.edge * 0.5;  // cell edge at level L
    for (;;) {
        const double gx = axis_gap(sx, cx, w, fr.margin), gy = axis_gap(sy, cy, w, fr.margin),
                     gz = axis_gap(sz, cz, w, fr.margin);
        if (gx * gx + gy * gy + gz * gz < best.kth()) {
            const int sh = QBITS - L;
            const u128 start = key126(cx << sh, cy << sh, cz << sh);
            const int a0 = lower_bound_from(keys, a, n, start);
            const int b0 = lower_bound_from(keys, a0, n, start + ((u128)1 << (3 * sh)));
            if (b0 - a0 > LEAF_T && L < QBITS) {  // enter: first child
                ++L; cx <<= 1; cy <<= 1; cz <<= 1; w *= 0.5; a = a0;
                continue;
            }
            scan_range(best, q, pts, a0, b0 < w0 ? b0 : w0);
            scan_range(best, q, pts, a0 > w1 ? a0 : w1, b0);
            a = b0;
        }
        // next cell in Morton order: climb out of finished last children, then step to the next sibling
        while (L > 0 && (cx & cy & cz & 1)) { cx >>= 1; cy >>= 1; cz >>= 1; --L; w *= 2.0; }
        if (L == 0) break;
        const uint32_t d = (uint32_t)((cx & 1) << 2 | (cy & 1) << 1 | (cz & 1)) + 1;
        cx = (cx & ~1ull) | (d >> 2); cy = (cy & ~1ull) | ((d >> 1) & 1); cz = (cz & ~1ull) | (d & 1);
    }
}

__global__ void __launch_bounds__(QB) knn_kernel(const ulonglong2* __restrict__ keys, const float4* __restrict__ pts,
                                                 const uint32_t* __restrict__ order, const Frame* __restrict__ frp, int n,
                                                 int k, double* __restrict__ avg) {
    const int t = blockIdx.x * QB + threadIdx.x;
    if (t >= n) return;
    const float4 q = pts[t];
    if (!finite3(q.x, q.y, q.z)) { avg[order[t]] = __longlong_as_double(0x7ff8000000000000ll); return; }
    const Frame fr = *frp;
    const int kp = k < n ? k : n;
    DistList best;
    best.init(kp);
    knn_query(best, keys, pts, fr, n, t, q);
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < K_MAX; ++j)
        if (j >= K_MAX - kp) s = __dadd_rn(s, sqrt(best.d[j]));
    avg[order[t]] = s / (double)kp;
}

// ids[row * k + r], d2[row * k + r] for r < k' = min(k, n - 1): the neighbours of `row` by ascending (d2, id); the
// slots r >= k' hold id -1 and d2 +inf.  A non-finite row gets id -1 and d2 NaN in every slot.
__global__ void __launch_bounds__(QB) knn_ids_kernel(const ulonglong2* __restrict__ keys, const float4* __restrict__ pts,
                                                     const Frame* __restrict__ frp, int n, int k,
                                                     int32_t* __restrict__ ids, double* __restrict__ d2) {
    const int t = blockIdx.x * QB + threadIdx.x;
    if (t >= n) return;
    const float4 q = pts[t];
    const uint32_t row = __float_as_uint(q.w);
    const int kp = k < n - 1 ? k : n - 1;
    if (!finite3(q.x, q.y, q.z)) {
        for (int r = 0; r < k; ++r) {
            ids[(int64_t)row * k + r] = -1;
            if (d2) d2[(int64_t)row * k + r] = __longlong_as_double(0x7ff8000000000000ll);
        }
        return;
    }
    const Frame fr = *frp;
    IdList best;
    best.self = row;
    best.init(kp);
    knn_query(best, keys, pts, fr, n, t, q);
    // k' exact copies of the query fill the list at distance 0, and the walk then prunes every cell; copies with
    // smaller ids may still be missing.  Copies share the query's key, and equal keys keep their row order through the
    // stable sorts, so the key run's first copies (up to k' of them besides the query) are the smallest ids.
    if (kp > 0 && best.kth() == 0.0) {
        const u128 K = key_at(keys, t);
        int found = 0;
        for (int j = lower_bound_from(keys, 0, n, K); j < n && found < kp && key_at(keys, j) == K; ++j) {
            const float4 p = pts[j];
            const uint32_t jid = __float_as_uint(p.w);
            if (jid == row) continue;
            if (dist2(q, p) == 0.0) ++found;
            if (!best.contains(jid)) best.consider(q, p);
        }
    }
    int32_t* out = ids + (int64_t)row * k;
    double* od = d2 ? d2 + (int64_t)row * k : nullptr;
#pragma unroll
    for (int j = 0; j < K_MAX; ++j) {
        const int r = j - (K_MAX - kp);
        if (r >= 0) { out[r] = (int32_t)best.id[j]; if (od) od[r] = best.d[j]; }
    }
    for (int r = kp; r < k; ++r) { out[r] = -1; if (od) od[r] = INFINITY; }
}

// ---- statistics and keep mask ------------------------------------------------------------------------------------
constexpr int SB = 256;
constexpr int SOR_PER_CTA = SB * 8;

// pass 0: per-CTA sum of avg over avg > 0;  pass 1: of (avg - mean)^2 over avg > 0.  Fixed order: bit-identical re-runs.
template <int PASS>
__global__ void __launch_bounds__(SB) sor_partial_kernel(const double* __restrict__ avg, int64_t n,
                                                         const double* __restrict__ stats, double* __restrict__ partial) {
    __shared__ double s_w[SB / 32];
    const double mean = PASS == 1 ? stats[0] : 0.0;
    const int64_t base = (int64_t)blockIdx.x * SOR_PER_CTA;
    double v = 0.0;
    for (int r = 0; r < SOR_PER_CTA / SB; ++r) {
        const int64_t i = base + r * SB + threadIdx.x;
        if (i >= n) break;
        const double x = avg[i];
        if (x > 0.0) v = __dadd_rn(v, PASS == 0 ? x : __dmul_rn(x - mean, x - mean));
    }
    const double tot = block_sum_f64<SB>(v, s_w);
    if (threadIdx.x == 0) partial[blockIdx.x] = tot;
}

// one CTA: fixed-order sum of the partials; pass 0 -> stats[0] = mean, pass 1 -> stats[1] = std, stats[2] = threshold.
// Every point has a neighbour (itself), so the count of valid distances is n.
template <int PASS>
__global__ void __launch_bounds__(1024) sor_finish_kernel(const double* __restrict__ partial, int nb, int64_t n,
                                                          double std_ratio, double* __restrict__ stats) {
    __shared__ double s[1024];
    const double t = sum_partials_f64(partial, nb, s);
    if (threadIdx.x == 0) {
        if (PASS == 0) {
            stats[0] = t / (double)n;
        } else {
            const double sd = sqrt(t / (double)(n - 1));  // n == 1: 0 / 0 = NaN, nothing is kept
            stats[1] = sd;
            stats[2] = __dadd_rn(stats[0], __dmul_rn(std_ratio, sd));
        }
    }
}

__global__ void __launch_bounds__(SB) sor_keep_kernel(const double* __restrict__ avg, int64_t n,
                                                      const double* __restrict__ stats, uint8_t* __restrict__ keep) {
    const int64_t i = (int64_t)blockIdx.x * SB + threadIdx.x;
    if (i >= n) return;
    const double x = avg[i];
    keep[i] = (x > 0.0 && x < stats[2]) ? 1 : 0;
}

// workspace of g2pc_knn_mean_dist; a null base only sizes it
struct KnnWs {
    Frame* fr;
    float* part;
    uint64_t *hi, *lo;
    uint64_t *lo_by_lo, *hi_by_lo;  // sort 1 output keys and hi gathered in that order; later the (lo, hi) key pairs
    uint32_t *idx_a, *idx_b;
    float4* pts;
    void* tmp;
    size_t tmp_bytes, bytes;
};

KnnWs knn_ws(void* base, int64_t n) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                    (const uint32_t*)nullptr, (uint32_t*)nullptr, n, 0, 63);
    WsCarve w{(char*)base};
    KnnWs l;
    l.fr = w.take<Frame>(1);
    l.part = w.take<float>((size_t)bbox_blocks(n) * 6);
    l.hi = w.take<uint64_t>(n);
    l.lo = w.take<uint64_t>(n);
    l.lo_by_lo = w.take<uint64_t>(n);  // adjacent to hi_by_lo: together at least 16n bytes for the key pairs
    l.hi_by_lo = w.take<uint64_t>(n);
    l.idx_a = w.take<uint32_t>(n);
    l.idx_b = w.take<uint32_t>(n);
    l.pts = w.take<float4>(n);
    l.tmp_bytes = WsCarve::pad(sort_b);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

// The index of both k-NN entry points: frame, keys, the two stable sorts, the sorted key pairs and points.  Returns the
// key pairs; the sorted points are in l.pts and their rows in l.idx_a.
int build_index(const float* xyz, int64_t n, int32_t* status, const KnnWs& l, cudaStream_t st, ulonglong2** keys_out) {
    uint64_t* hi_sorted = l.hi;                          // sort 2 output keys (hi is dead by then)
    ulonglong2* keys = (ulonglong2*)l.lo_by_lo;          // both sort 1 buffers are dead by then
    const int nbox = bbox_blocks(n);
    const unsigned g = (unsigned)((n + BB - 1) / BB);
    bbox_kernel<<<nbox, BBOX_THREADS, 0, st>>>(xyz, n, l.part);
    G2PC_CHECK_LAUNCH();
    frame_kernel<<<1, 1, 0, st>>>(l.part, nbox, l.fr);
    G2PC_CHECK_LAUNCH();
    key_kernel<<<g, BB, 0, st>>>(xyz, n, l.fr, l.hi, l.lo, l.idx_a, status);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, l.lo, l.lo_by_lo, l.idx_a, l.idx_b, n, 0, 63, st));
    gather_u64_kernel<<<g, BB, 0, st>>>(l.hi, l.idx_b, n, l.hi_by_lo);
    G2PC_CHECK_LAUNCH();
    b = l.tmp_bytes;  // stable: points with equal hi keep their lo order
    G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, l.hi_by_lo, hi_sorted, l.idx_b, l.idx_a, n, 0, 63, st));
    gather_sorted_kernel<<<g, BB, 0, st>>>(hi_sorted, l.lo, l.idx_a, xyz, n, keys, l.pts);
    G2PC_CHECK_LAUNCH();
    *keys_out = keys;
    return G2PC_OK;
}

}  // namespace

extern "C" int64_t g2pc_knn_workspace_bytes(int64_t n) { return n <= 0 ? 0 : (int64_t)knn_ws(nullptr, n).bytes; }

extern "C" int g2pc_knn_mean_dist(const float* xyz, int64_t n, int32_t k, double* avg, int32_t* status, void* workspace,
                                  int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(n < 0x7FFFFFFFll, "n must fit int32 indices");
    G2PC_CHECK_ARG(k >= 1 && k <= K_MAX, "k must be in 1..G2PC_SOR_K_MAX");
    G2PC_CHECK_ARG(status, "null status");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(xyz && avg && workspace, "null pointer");
    const KnnWs l = knn_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    ulonglong2* keys = nullptr;
    const int rc = build_index(xyz, n, status, l, st, &keys);
    if (rc != G2PC_OK) return rc;
    knn_kernel<<<(unsigned)((n + QB - 1) / QB), QB, 0, st>>>(keys, l.pts, l.idx_a, l.fr, (int)n, k, avg);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_knn_ids(const float* xyz, int64_t n, int32_t k, int32_t* ids, double* d2, int32_t* status,
                            void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(n < 0x7FFFFFFFll, "n must fit int32 indices");
    G2PC_CHECK_ARG(k >= 1 && k <= G2PC_ORIENT_K_MAX, "k must be in 1..G2PC_ORIENT_K_MAX");
    G2PC_CHECK_ARG(status, "null status");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(xyz && ids && workspace, "null pointer");
    const KnnWs l = knn_ws(workspace, n);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    ulonglong2* keys = nullptr;
    const int rc = build_index(xyz, n, status, l, st, &keys);
    if (rc != G2PC_OK) return rc;
    knn_ids_kernel<<<(unsigned)((n + QB - 1) / QB), QB, 0, st>>>(keys, l.pts, l.fr, (int)n, k, ids, d2);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_sor_workspace_bytes(int64_t n) {
    return (int64_t)(((n + SOR_PER_CTA - 1) / SOR_PER_CTA + 1) * sizeof(double));
}

extern "C" int g2pc_sor_mask(const double* avg, int64_t n, double std_ratio, uint8_t* keep, double* stats,
                             void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    G2PC_CHECK_ARG(std_ratio > 0.0, "std_ratio must be > 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(avg && keep && stats && workspace, "null pointer");
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, g2pc_sor_workspace_bytes(n), 8);
    cudaStream_t st = (cudaStream_t)stream;
    const int nb = (int)((n + SOR_PER_CTA - 1) / SOR_PER_CTA);
    double* partial = (double*)workspace;
    sor_partial_kernel<0><<<nb, SB, 0, st>>>(avg, n, stats, partial);
    G2PC_CHECK_LAUNCH();
    sor_finish_kernel<0><<<1, 1024, 0, st>>>(partial, nb, n, std_ratio, stats);
    G2PC_CHECK_LAUNCH();
    sor_partial_kernel<1><<<nb, SB, 0, st>>>(avg, n, stats, partial);
    G2PC_CHECK_LAUNCH();
    sor_finish_kernel<1><<<1, 1024, 0, st>>>(partial, nb, n, std_ratio, stats);
    G2PC_CHECK_LAUNCH();
    sor_keep_kernel<<<(unsigned)((n + SB - 1) / SB), SB, 0, st>>>(avg, n, stats, keep);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
