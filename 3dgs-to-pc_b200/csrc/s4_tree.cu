// s4_tree.cu — S4: resolve the python renderer's tile quadtree on the device, then build every leaf's depth-ordered list.
//
// Reference semantics restated (not copied): gauss_render.py:290-344
//   BFS over tiles; a tile is skipped if w <= 1 or h <= 1 (:301), background-filled if no Gaussian overlaps it
//   (:313-315), split into TL, BL, TR, BR children if it holds more than max_gaussians_per_tile Gaussians or is wider /
//   taller than max_tile_size (:319-335), else rendered with its Gaussians ordered nearest-first (:340-344).
// Role of rasterizer_impl.cu:69-137,285-326 (duplicateWithKeys + 64-bit radix sort + identifyTileRanges) in the CUDA
// back-end of the reference; none of its structure is kept.
//
// Pipeline per camera (all sizes stay on the device; the host never waits for a count):
//   1. g2pc_depth_sort      one radix sort of N (depth key, value) pairs, value = (packed node range << 32 | Gaussian id)
//                           written by the preprocess kernel (cub::DeviceRadixSort, library call).
//   2. g2pc_build_tree      one CTA walks the levels top-down on the per-node overlap counts of the preprocess kernel,
//                           numbers the leaves in the reference's BFS order (level-major, then child-rank path order),
//                           lays out instance / pixel offsets, sorts the leaves heaviest-first for the blend and writes
//                           the frame header.  A frame that does not fit the caller's buffers (or needs a deeper table)
//                           sets the sticky POISON word: every later kernel of this and the following frames becomes a
//                           no-op until the host has read the header, fixed the sizes and replayed.
//   3. g2pc_multisplit      stable multisplit of the depth-ordered stream into the leaves' lists, without any sort of
//                           the ~7 N instances (the round-1 path emitted (leaf, id) pairs and ran a 2-pass 20 M-pair
//                           radix sort per camera).  A base-level leaf is one cell (ix, iy) of a grid of at most 256 x 256
//                           (the quadtree's base level, or the CUDA back-end's super-tiles), and an entry covers a
//                           rectangle of cells, so its base-level lists are two stable splits of <= 256 buckets each:
//        rows     the sorted stream -> one list of 64-bit entries per row iy, in stream order       (row_list)
//        columns  each row's list -> one list per cell, written straight into the leaf's list in inst_gid
//                 Each split is count -> scan -> scatter over warp tiles of 512 consecutive entries.  Within a batch of
//                 32 entries (one per lane) a 32 x 32 bit transpose gives lane b the ballot of the lanes whose entry
//                 falls in bucket b; an entry's place is the bucket's running offset + its rank among those lanes, and
//                 lane b keeps the running offset of bucket b in a register.  No shared-memory bit matrix and no CTA
//                 barrier inside the walk; the count matrices are tiles x buckets, kilobytes.
//        deeper   leaves below the base level (count-driven splits) come from the older chunked multisplit (count /
//                 scan / scatter with a shared-memory bit matrix per sub-step), which runs only when the table has such
//                 levels and emits only those leaves.  Splats that cover many tiles are walked by the whole warp
//                 (colour_common.cuh warp_for_each_node).
#include <cub/cub.cuh>
#include "colour_common.cuh"

namespace {

constexpr int TB = 1024;
constexpr int SORT_CAP = 4096;  // leaves sorted heaviest-first in shared memory (more leaves: launch order = BFS order)

struct TreeParams {
    QtMeta meta;
    QtTables tab;
    int32_t n1;
    uint32_t* node_cnt;      // read, then cleared for the next frame
    uint8_t* node_state;
    int32_t* node_leaf;      // per node: leaf id, -1 (no leaf: empty / absent / dropped) or -2 (split)
    g2pc_leaf_t* leaves;
    int32_t* leaf_order;     // leaves sorted by descending work (longest-processing-time-first launch order)
    int32_t max_leaves;
    int64_t inst_capacity, pix_capacity, matrix_capacity;
    int32_t ms_chunks;
    int32_t frame;
    int32_t* header;         // G2PC_HDR_WORDS
    uint32_t* fail;          // shared failure word (colour_common.cuh)
    int32_t* work_counters;  // G2PC_WORK_COUNTERS ints, cleared here for the blend of this frame
    int32_t nodes_2d;
};

// key (BFS rank within a level: child rank = 2*xbit + ybit per level, most significant first) -> (ix, iy)
__device__ __forceinline__ void deinterleave(int key, int level, int& ix, int& iy) {
    ix = 0; iy = 0;
    for (int b = 0; b < level; ++b) {
        iy |= ((key >> (2 * b)) & 1) << b;
        ix |= ((key >> (2 * b + 1)) & 1) << b;
    }
}

__global__ void __launch_bounds__(TB) tree_kernel(const TreeParams p) {
    __shared__ int s_warp[33];
    __shared__ int s_flags[2];
    __shared__ unsigned long long s_sort[SORT_CAP];
    if (g2pc_report_skipped_frame(p.fail, p.frame, p.header)) return;  // this or an earlier frame failed
    const int L = p.meta.num_levels;
    if (threadIdx.x == 0) { s_flags[0] = 0; s_flags[1] = 0; }
    __syncthreads();
    int leaf_base = 0;
    long long inst_total = 0;
    for (int l = 0; l < L; ++l) {
        const int nn = 1 << (2 * l);
        const int o1 = (1 << l) - 1, o2 = off2d(l);
        for (int k0 = 0; k0 < nn; k0 += TB) {
            const int key = k0 + threadIdx.x;
            int is_leaf = 0, node = -1, ix = 0, iy = 0;
            uint32_t cnt = 0;
            if (key < nn) {
                deinterleave(key, l, ix, iy);
                node = o2 + (iy << l) + ix;
                bool exists = (l == 0);
                if (l > 0) {
                    const int pnode = off2d(l - 1) + ((iy >> 1) << (l - 1)) + (ix >> 1);
                    exists = p.node_state[pnode] == NODE_SPLIT;
                }
                uint8_t st = NODE_NONE;
                int32_t nl = -1;
                if (exists) {
                    const int fx = p.tab.xf[o1 + ix], fy = p.tab.yf[o1 + iy];
                    if (!((fx | fy) & QT_FLAG_DROPPED)) {
                        cnt = p.node_cnt[node];
                        // cnt: exact on the leaf-candidate levels, a non-empty flag above them (a node larger than
                        // max_tile_size splits whatever it holds — unless it is empty: then it is background and has
                        // no children, gauss_render.py:313-335)
                        const bool big = ((fx | fy) & QT_FLAG_BIG) != 0;
                        if (cnt == 0) st = NODE_EMPTY;
                        else if (big || cnt > (uint32_t)p.meta.max_gaussians_per_tile) {
                            st = NODE_SPLIT;
                            nl = -2;
                            if (l == L - 1) { st = NODE_NONE; nl = -1; s_flags[0] = 1; }  // deeper than the tabulated levels
                        } else {
                            st = NODE_LEAF;
                            is_leaf = 1;
                        }
                    }
                }
                p.node_state[node] = st;
                p.node_leaf[node] = nl;
            }
            int tot;
            const int pre = block_scan_1024(is_leaf, s_warp, tot);
            if (is_leaf) {
                const int li = leaf_base + pre;
                if (li < p.max_leaves) {
                    g2pc_leaf_t lf;
                    lf.r0 = p.tab.ys[o1 + iy];
                    lf.c0 = p.tab.xs[o1 + ix];
                    lf.w = p.tab.xe[o1 + ix] - lf.c0 + 1;
                    lf.h = p.tab.ye[o1 + iy] - lf.r0 + 1;
                    lf.inst_begin = 0;
                    lf.inst_count = (int32_t)cnt;
                    lf.pix_offset = 0;
                    lf.node = node;
                    p.leaves[li] = lf;
                    p.node_leaf[node] = li;
                } else {
                    s_flags[1] = 1;
                }
            }
            leaf_base += tot;
        }
        __syncthreads();  // node_state of level l visible to level l+1
    }
    const int nl = leaf_base < p.max_leaves ? leaf_base : p.max_leaves;
    // exclusive scans of the instance counts and pixel counts over the leaves, in order
    int pix_base = 0;
    for (int k0 = 0; k0 < nl; k0 += TB) {
        const int i = k0 + threadIdx.x;
        int c = 0, a = 0;
        // every list starts on a 16-byte boundary (the blend stages id chunks with TMA bulk copies): pad to 4 ids
        if (i < nl) { c = (p.leaves[i].inst_count + 3) & ~3; a = p.leaves[i].w * p.leaves[i].h; }
        int tc, ta;
        const int pc = block_scan_1024(c, s_warp, tc);
        const int pa = block_scan_1024(a, s_warp, ta);
        if (i < nl) {
            // 32-bit list offsets: a frame with more than 2^31 instances is reported through the capacity check below
            p.leaves[i].inst_begin = (int32_t)(inst_total + pc);
            p.leaves[i].pix_offset = pix_base + pa;
        }
        inst_total += tc;
        pix_base += ta;
    }
    __syncthreads();
    // launch order for the blend: heaviest leaves first (instances x pixels, ties by index)
    g2pc_launch_order<TB, SORT_CAP>(s_sort, nl, [&](int i) {
        unsigned long long w = (unsigned long long)p.leaves[i].inst_count *
                               (unsigned long long)(p.leaves[i].w * p.leaves[i].h);
        w = w < (1ull << 44) - 1ull ? w : (1ull << 44) - 1ull;
        return (((1ull << 44) - 1ull - w) << 16) | (unsigned long long)i;  // ascending key = descending work
    }, 0xFFFFull, p.leaf_order);
    // the counts are consumed: clear them for the next frame's preprocess
    for (int k = threadIdx.x; k < p.nodes_2d; k += TB) p.node_cnt[k] = 0u;
    if (threadIdx.x < G2PC_WORK_COUNTERS) p.work_counters[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        const int cap_over = (inst_total > p.inst_capacity || (long long)pix_base > p.pix_capacity ||
                              (long long)p.ms_chunks * (long long)nl > p.matrix_capacity || inst_total > 0x7FFFFFFFll)
                             // (ms_chunks = rows the multisplit needs: one per chunk, g2pc_multisplit_rows)
                                 ? 1 : 0;
        g2pc_write_frame_header(p.header, p.fail, p.frame, leaf_base, inst_total, pix_base, s_flags[0], s_flags[1],
                                cap_over);
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Multisplit below the base level.  An entry of the sorted stream is (range << 32 | gid); Gaussians that touch a split
// base node (or sit in the one-node overhang of one) re-derive their rect from the projection record and query the deeper
// candidate levels.
struct MsParams {
    const unsigned long long* val_sorted;
    int64_t n;
    const float4* proj;
    int32_t width, height;
    float inv_width, inv_height;  // 1 / width, 1 / height (IEEE division on the host: no division subroutine on the device)
    QtMeta meta;
    QtTables tab;
    int32_t n1;
    uint32_t level_mask;
    int32_t base_level;
    const int32_t* node_leaf;
    const int32_t* header;
    const uint32_t* fail;
    int32_t frame;
    const g2pc_leaf_t* leaves;
    uint32_t* matrix;      // [chunk][num_leaves]: counts, then absolute list offsets (in place)
    uint32_t* inst_gid;
    int32_t leaf_cap;      // leaves the shared-memory tables are sized for (<= max_leaves of the tree)
    int32_t base_clean;    // the base level has no dropped / degenerate node: membership = the packed range, no table look-ups
    uint32_t clean_mask;   // the same, per level
    const uint32_t* base_split;  // written by the row split: 1 iff a base-level node of this frame was split (else no list
                                 // below the base level, and these kernels return at once)
    int32_t steps;         // sub-steps of C entries per chunk (ms_steps)
};

// f(leaf, owner_lane, owner_gid) for every leaf BELOW the base level that the lane's entry overlaps (the base-level lists
// come from the row / column split further down); warp-cooperative (all 32 lanes must call).
template <typename F>
__device__ __forceinline__ void for_each_leaf(const MsParams& p, const QtTables& T, const int32_t* __restrict__ s_leaf,
                                              uint32_t range, uint32_t gid, F f) {
    const int lb = p.base_level;
    const int o1 = (1 << lb) - 1;
    unsigned deeper = 0;
    if (p.base_clean) {
        warp_for_each_node(range, gid, [&](int ix, int iy, int owner, uint32_t) {
            if (s_leaf[(iy << lb) + ix] == -2) deeper |= 1u << owner;
        });
    } else {
        warp_for_each_node(range, gid, [&](int ix, int iy, int owner, uint32_t) {
            if (!axis_member(T.ys + o1, T.ye + o1, T.yf + o1, iy) || !axis_member(T.xs + o1, T.xe + o1, T.xf + o1, ix)) return;
            if (s_leaf[(iy << lb) + ix] == -2) deeper |= 1u << owner;
        });
    }
    int xlo, xhi, ylo, yhi;
    g2pc_unpack_range(range, xlo, xhi, ylo, yhi);
    // ---- count-driven splits below the base level ----
    // Rare at 1280 px; at 1920 px with 6 M Gaussians most of the sphere's base nodes split two levels down (C5: 150 M
    // instances per camera, almost all from here), so the deeper levels get the same warp-cooperative walk as the base
    // level (per-lane loops with per-node table checks ran at 5 of 32 threads: 69 + 13 ms per camera, ncu r02g).
    // combine the flags raised on behalf of each owner
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) deeper |= __shfl_xor_sync(0xffffffffu, deeper, o);
    const int lane = threadIdx.x & 31;
    bool mine = (deeper >> lane) & 1u;
    if (!mine && xlo <= xhi) {
        // a child tile may overhang its parent by a pixel to the right / below (children are ceil(size / 2) wide): a
        // Gaussian can sit in a deeper leaf of the base node just left of / above its own base range
        const int ex = max(xlo - 1, 0), ey = max(ylo - 1, 0);
        for (int iy = ey; iy <= yhi; ++iy)
            for (int ix = ex; ix <= xhi; ++ix)
                if ((iy < ylo || ix < xlo) && s_leaf[(iy << lb) + ix] == -2) mine = true;
    }
    if (!__any_sync(0xffffffffu, mine)) return;
    float x0 = 0.f, x1 = 0.f, y0 = 0.f, y1 = 0.f;
    if (mine) {
        const float4 q0 = __ldg(p.proj + 3 * (int64_t)gid);
        const float4 q2 = __ldg(p.proj + 3 * (int64_t)gid + 2);
        gaussian_rect(q0.x, q0.y, q2.z, p.width, p.height, x0, x1, y0, y1);
    }
    const float isx0 = p.inv_width, isy0 = p.inv_height;
    for (int l = lb + 1; l < p.meta.num_levels; ++l) {  // (uniform)
        if (!((p.level_mask >> l) & 1u)) continue;
        const int ol = (1 << l) - 1;
        int axlo = 1, axhi = 0, aylo = 1, ayhi = 0;
        if (mine) {
            axis_range(T.xs + ol, T.xe + ol, l, x0, x1, isx0 * (float)(1 << l), axlo, axhi);
            if (axlo <= axhi) axis_range(T.ys + ol, T.ye + ol, l, y0, y1, isy0 * (float)(1 << l), aylo, ayhi);
        }
        const bool some = axlo <= axhi && aylo <= ayhi;
        const int32_t* nl = p.node_leaf + off2d(l);
        if (((p.clean_mask >> l) & 1u) && l <= G2PC_RANGE_MAX_LEVEL) {
            // no dropped / degenerate node at this level: membership = the range; cooperative walk
            const uint32_t rl = some ? g2pc_pack_range(axlo, axhi, aylo, ayhi) : (uint32_t)G2PC_RANGE_EMPTY;
            warp_for_each_node(rl, gid, [&](int ix, int iy, int owner, uint32_t og) {
                const int32_t v = __ldg(nl + (iy << l) + ix);
                if (v >= 0) f(v, owner, og);
            });
            continue;
        }
        if (!some) continue;
        for (int iy = aylo; iy <= ayhi; ++iy) {
            if (!axis_member(T.ys + ol, T.ye + ol, T.yf + ol, iy)) continue;
            for (int ix = axlo; ix <= axhi; ++ix) {
                if (!axis_member(T.xs + ol, T.xe + ol, T.xf + ol, ix)) continue;
                const int32_t v = __ldg(nl + (iy << l) + ix);
                if (v >= 0) f(v, lane, gid);
            }
        }
    }
}

// The sorted stream is cut into chunks of E = steps x C consecutive entries, one CTA per chunk; a CTA walks its chunk in
// `steps` sub-steps of C entries (one per thread), in stream order.  The per-chunk set-up (tables, node->leaf map, one
// matrix row) is paid once per E entries.
__device__ __forceinline__ unsigned long long ms_entry(const MsParams& p, int64_t k) {
    return k < p.n ? p.val_sorted[k] : (unsigned long long)G2PC_RANGE_EMPTY << 32;
}

// shared memory of the count / scatter kernels: [6 * n1 table ints][4^base node->leaf ints][payload]
__device__ __forceinline__ int32_t* ms_load_common(const MsParams& p, int32_t* smem, QtTables& T) {
    T = load_tables(p.tab, p.n1, smem);  // ends with __syncthreads()
    int32_t* s_leaf = smem + 6 * p.n1;
    const int nb = 1 << (2 * p.base_level);
    const int32_t* src = p.node_leaf + off2d(p.base_level);
    for (int i = threadIdx.x; i < nb; i += blockDim.x) s_leaf[i] = src[i];
    return s_leaf;
}

// count:   matrix[c][leaf] = instances of `leaf` in chunk c (one shared-memory histogram over the chunk's sub-steps)
// scan:    per leaf, exclusive prefix over the chunks + the leaf's list offset (one kernel, 32 leaves per CTA)
// scatter: position = running offset of the leaf + rank inside the sub-step (bit matrix)
// (minimum CTAs per SM in the launch bounds: with the thread count alone ptxas held both kernels to 40-48 registers and
// spilled; 1024 / C and 768 / C leave them 61 and 80 registers, no spill, and the scatter still fits 3 CTAs per SM at C = 256)
template <int C>
__global__ void __launch_bounds__(C, 1024 / C) ms_count_kernel(const MsParams p) {
    extern __shared__ int32_t smem_ms[];
    if (g2pc_frame_skipped(p.fail, p.frame) || *p.base_split == 0u) return;
    const int nl = p.header[G2PC_HDR_NUM_LEAVES];
    QtTables T;
    int32_t* s_leaf = ms_load_common(p, smem_ms, T);
    uint32_t* s_hist = reinterpret_cast<uint32_t*>(s_leaf + (1 << (2 * p.base_level)));
    for (int i = threadIdx.x; i < nl; i += C) s_hist[i] = 0u;
    __syncthreads();
    // no barrier between the sub-steps: the warps only add to the histogram
    const int64_t k0 = (int64_t)blockIdx.x * p.steps * C;
    for (int s = 0; s < p.steps; ++s) {
        const int64_t b = k0 + (int64_t)s * C;
        if (b >= p.n) break;  // (uniform)
        const unsigned long long v = ms_entry(p, b + threadIdx.x);
        for_each_leaf(p, T, s_leaf, (uint32_t)(v >> 32), (uint32_t)v,
                      [&](int leaf, int, uint32_t) { atomicAdd(s_hist + leaf, 1u); });
    }
    __syncthreads();
    uint32_t* row = p.matrix + (int64_t)blockIdx.x * nl;
    for (int i = threadIdx.x; i < nl; i += C) row[i] = s_hist[i];
}

// Column-wise exclusive scan of matrix (rows x num_leaves), rewritten in place as absolute list offsets.  CTA = 32
// leaves x 32 row bands: each thread sums its band of one column, the bands' sums are scanned in shared memory, then each
// thread rewrites its band as running offsets.  The whole matrix is a few MB and was just written: L2 traffic only.
constexpr int SCAN_BATCH = 8;  // matrix loads in flight per thread
__global__ void __launch_bounds__(1024) ms_scan_kernel(const MsParams p, int32_t rows) {
    __shared__ uint32_t s_sum[32][33];
    if (g2pc_frame_skipped(p.fail, p.frame) || *p.base_split == 0u) return;
    const int nl = p.header[G2PC_HDR_NUM_LEAVES];
    if (blockIdx.x * 32 >= nl) return;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int leaf = blockIdx.x * 32 + tx;
    const int band = (rows + 31) / 32;
    const int r0 = min(rows, ty * band), r1 = min(rows, r0 + band);
    uint32_t* col = p.matrix + leaf;
    uint32_t sum = 0;
    if (leaf < nl) {
#pragma unroll 8
        for (int r = r0; r < r1; ++r) sum += col[(int64_t)r * nl];
    }
    s_sum[ty][tx] = sum;
    __syncthreads();
    if (leaf >= nl) return;
    uint32_t run = (uint32_t)p.leaves[leaf].inst_begin;
    for (int s = 0; s < ty; ++s) run += s_sum[s][tx];
    for (int r = r0; r < r1; r += SCAN_BATCH) {
        // load a batch before storing any of it (the stores would otherwise serialise the loads behind them)
        uint32_t c[SCAN_BATCH];
#pragma unroll
        for (int q = 0; q < SCAN_BATCH; ++q) c[q] = r + q < r1 ? col[(int64_t)(r + q) * nl] : 0u;
#pragma unroll
        for (int q = 0; q < SCAN_BATCH; ++q) {
            if (r + q < r1) col[(int64_t)(r + q) * nl] = run;
            run += c[q];
        }
    }
}

template <int C>
__global__ void __launch_bounds__(C, 768 / C) ms_scatter_kernel(const MsParams p) {
    extern __shared__ int32_t smem_ms[];
    if (g2pc_frame_skipped(p.fail, p.frame) || *p.base_split == 0u) return;
    const int nl = p.header[G2PC_HDR_NUM_LEAVES];
    constexpr int WORDS = C / 32;
    QtTables T;
    int32_t* s_leaf = ms_load_common(p, smem_ms, T);
    uint32_t* s_row = reinterpret_cast<uint32_t*>(s_leaf + (1 << (2 * p.base_level)));  // [nl]
    uint32_t* s_bits = s_row + p.leaf_cap;                                                                   // [WORDS][nl]
    {
        // the chunk's list offsets (one coalesced row of the matrix) and a zeroed bit matrix; 16-byte stores where the
        // carve-up allows (leaf_cap is a multiple of 4 and the dynamic smem base is 16-byte aligned)
        const uint32_t* grow = p.matrix + (int64_t)blockIdx.x * nl;
        for (int i = threadIdx.x; i < nl; i += C) s_row[i] = grow[i];
        if (((reinterpret_cast<uintptr_t>(s_bits) & 15) == 0) && ((nl & 3) == 0)) {
            uint4* b4 = reinterpret_cast<uint4*>(s_bits);
            for (int i = threadIdx.x; i < WORDS * nl / 4; i += C) b4[i] = make_uint4(0u, 0u, 0u, 0u);
        } else {
            for (int i = threadIdx.x; i < WORDS * nl; i += C) s_bits[i] = 0u;
        }
    }
    __syncthreads();
    const int w = threadIdx.x >> 5;  // the warp = the 32-entry group of the sub-step
    uint32_t* mybits = s_bits + w * nl;
    const int64_t k0 = (int64_t)blockIdx.x * p.steps * C;
    unsigned long long v = ms_entry(p, k0 + threadIdx.x);
    for (int s = 0; s < p.steps; ++s) {
        const int64_t b = k0 + (int64_t)s * C;
        if (b >= p.n) break;  // (uniform)
        const bool more = s + 1 < p.steps && b + C < p.n;
        const uint32_t range = (uint32_t)(v >> 32), gid = (uint32_t)v;
        // 1. mark (leaf, k) in the bit matrix: order-free
        for_each_leaf(p, T, s_leaf, range, gid, [&](int leaf, int owner, uint32_t) { atomicOr(mybits + leaf, 1u << owner); });
        __syncthreads();
        const unsigned long long vn = more ? ms_entry(p, b + C + threadIdx.x) : 0ull;  // next sub-step, in flight early
        // 2. every instance finds its place: the running offset of the leaf, the instances of the same leaf in earlier
        //    32-entry groups of the sub-step, then the earlier lanes of its own group (bit order = depth order)
        for_each_leaf(p, T, s_leaf, range, gid, [&](int leaf, int owner, uint32_t og) {
            uint32_t pos = s_row[leaf] + (uint32_t)__popc(mybits[leaf] & ((1u << owner) - 1u));
            for (int w2 = 0; w2 < w; ++w2) pos += (uint32_t)__popc(s_bits[w2 * nl + leaf]);
            p.inst_gid[pos] = og;
        });
        if (!more) break;
        __syncthreads();
        // 3. move every leaf's offset past this sub-step's instances and clear the bit matrix for the next sub-step
        for (int i = threadIdx.x; i < nl; i += C) {
            uint32_t cnt = 0;
#pragma unroll
            for (int w2 = 0; w2 < WORDS; ++w2) {
                cnt += (uint32_t)__popc(s_bits[w2 * nl + i]);
                s_bits[w2 * nl + i] = 0u;
            }
            s_row[i] += cnt;
        }
        __syncthreads();
        v = vn;
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Base-level lists: two stable splits, rows then columns.  Level 1 splits the sorted stream into one list per row (the
// 64-bit entries, in stream order); level 2 splits each row's list into its cells and writes the Gaussian ids straight
// into the leaves' lists.  Each level is count -> scan -> scatter over warp tiles of SP_TILE consecutive entries; the
// SP_WARPS tiles of a CTA form a band (level 2: a band never crosses a row).  The count kernel writes each tile's
// exclusive offsets within its band (m) and the band's totals (b); the scan turns the band totals into absolute offsets
// (level 1: also the rows' list offsets and the level-2 band layout); the scatter starts every bucket at b + m.
constexpr int SP_BATCHES = 8;                // 32-entry batches per warp tile
constexpr int SP_TILE = 32 * SP_BATCHES;     // entries per warp tile
constexpr int SP_WARPS = 16;                 // warp tiles per CTA = per band
constexpr int SP_BAND = SP_TILE * SP_WARPS;  // entries per band
constexpr int SP_MAX_CELLS = 256;            // cells per axis (G2PC_RANGE_MAX_LEVEL)
constexpr int SP_MAX_GROUPS = SP_MAX_CELLS / 32;
constexpr int SP_STAGE_BYTES = 6 * 1024;     // per warp: a tile's output staged in shared memory, written out bucket by bucket

struct SplitParams {
    const unsigned long long* val_sorted;
    int64_t n;
    int32_t rows, cols;          // grid of base cells
    int32_t rows_p, cols_p;      // rounded up to whole groups of 32 (row width of the count matrices)
    const int32_t* cell_leaf;    // rows x cols leaf ids (< 0: no base-level leaf), or NULL: leaf = iy * cols + ix
    QtTables tab;                // base-level axis tables (level offset applied) when the base level is not clean
    int32_t clean;               // 1: every cell in an entry's range is a member, no table look-ups
    const g2pc_leaf_t* leaves;
    int32_t* header;
    uint32_t* fail;
    int32_t frame;
    unsigned long long* row_list;
    int64_t row_capacity;
    uint32_t* m1;                // [bands1][SP_WARPS + 1][rows_p] (row SP_WARPS: the band's totals)
    uint32_t* b1;                // [bands1][rows_p]
    uint32_t* m2;                // [bands2][SP_WARPS + 1][cols_p]
    uint32_t* b2;                // [bands2][cols_p]
    uint32_t* row_begin;         // [rows + 1]: offset of each row's list in row_list
    uint32_t* band_begin;        // [rows + 1]: first level-2 band of each row
    uint32_t* base_split;        // quadtree only (else NULL): set to 1 iff a cell is a split node (cell_leaf == -2)
    int32_t bands1;
    uint32_t* inst_gid;
};

// bits of [lo, hi] inside the group of 32 buckets that starts at `base`
__device__ __forceinline__ uint32_t span_bits(int lo, int hi, int base) {
    lo = max(lo - base, 0);
    hi = min(hi - base, 31);
    return lo > hi ? 0u : ((0xFFFFFFFFu >> (31 - hi)) & (0xFFFFFFFFu << lo));
}

// 32 x 32 bit transpose across the warp: lane i brings row i, lane j gets column j (bit i = bit j of lane i).  Five
// rounds of block swaps: at distance s the lanes with bit s clear trade their high s-bit halves for their partner's low.
__device__ __forceinline__ uint32_t warp_transpose32(uint32_t x) {
    const int lane = threadIdx.x & 31;
    const uint32_t masks[5] = {0x0000FFFFu, 0x00FF00FFu, 0x0F0F0F0Fu, 0x33333333u, 0x55555555u};
#pragma unroll
    for (int i = 0, s = 16; i < 5; ++i, s >>= 1) {
        const uint32_t t = __shfl_xor_sync(0xffffffffu, x, s);
        x = (lane & s) ? ((x & ~masks[i]) | ((t & ~masks[i]) >> s)) : ((x & masks[i]) | ((t & masks[i]) << s));
    }
    return x;
}

// One warp walks entries [beg, end) of src in batches of 32, in order.  Buckets are rows (LEVEL 1) or columns (LEVEL 2);
// member[g]: the buckets of group g an entry may go to (warp-uniform).  COUNT: acc[g] (lane b: bucket 32 g + b) += the
// batch's entries in the bucket.  Otherwise acc[g] is the bucket's running offset: lane b writes the bucket's entries of
// the batch, in lane order, at acc[g]++ (level 1: the entry into row_list; level 2: its Gaussian id into inst_gid).
template <int LEVEL, int G, bool COUNT, typename Out>
__device__ __forceinline__ void split_walk(const SplitParams& p, const unsigned long long* __restrict__ src, int64_t beg,
                                           int64_t end, const uint32_t (&member)[G], uint32_t (&acc)[G], Out out) {
    const int lane = threadIdx.x & 31;
    for (int64_t b = beg; b < end; b += 32) {  // (uniform)
        const int64_t k = b + lane;
        const unsigned long long v = k < end ? src[k] : (unsigned long long)G2PC_RANGE_EMPTY << 32;
        int xlo, xhi, ylo, yhi;
        g2pc_unpack_range((uint32_t)(v >> 32), xlo, xhi, ylo, yhi);
        const bool some = xlo <= xhi && ylo <= yhi;
        const int lo = LEVEL == 1 ? ylo : xlo, hi = LEVEL == 1 ? yhi : xhi;
#pragma unroll
        for (int g = 0; g < G; ++g) {
            const uint32_t m = some ? span_bits(lo, hi, 32 * g) & member[g] : 0u;
            if (G > 1 && !__any_sync(0xffffffffu, m != 0u)) continue;
            const uint32_t bal = warp_transpose32(m);  // lanes whose entry falls in bucket 32 g + lane
            if (COUNT) {
                acc[g] += (uint32_t)__popc(bal);
                continue;
            }
            uint32_t rem = bal, pos = acc[g];
            while (__any_sync(0xffffffffu, rem != 0u)) {
                const int s = rem ? __ffs(rem) - 1 : 0;
                if (LEVEL == 1) {
                    const uint32_t lo32 = __shfl_sync(0xffffffffu, (uint32_t)v, s);
                    const uint32_t hi32 = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), s);
                    if (rem) out(pos++, ((unsigned long long)hi32 << 32) | lo32);
                } else {
                    const uint32_t gid = __shfl_sync(0xffffffffu, (uint32_t)v, s);
                    if (rem) out(pos++, (unsigned long long)gid);
                }
                rem &= rem - 1u;
            }
            acc[g] = pos;
        }
    }
}

// buckets of group g an entry may go to: level 1 the member rows, level 2 the cells of row `row` that are base-level
// leaves (on a non-clean base level also member columns)
template <int LEVEL, int G>
__device__ __forceinline__ void split_members(const SplitParams& p, int row, uint32_t (&member)[G]) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const int c = 32 * g + lane;
        bool in;
        if (LEVEL == 1) {
            in = c < p.rows && (p.clean || axis_member(p.tab.ys, p.tab.ye, p.tab.yf, c));
        } else {
            in = c < p.cols && (p.cell_leaf == nullptr || p.cell_leaf[row * p.cols + c] >= 0) &&
                 (p.clean || axis_member(p.tab.xs, p.tab.xe, p.tab.xf, c));
        }
        member[g] = __ballot_sync(0xffffffffu, in);
    }
}

// level-2 band -> its row (the last row whose first band is <= band) and the band's entries [beg, end) in row_list
__device__ __forceinline__ int split_band_row(const SplitParams& p, int band, int64_t& beg, int64_t& end) {
    int lo = 0, hi = p.rows - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if ((int)p.band_begin[mid] <= band) lo = mid; else hi = mid - 1;
    }
    beg = (int64_t)p.row_begin[lo] + (int64_t)(band - (int)p.band_begin[lo]) * SP_BAND;
    end = min(beg + SP_BAND, (int64_t)p.row_begin[lo + 1]);
    return lo;
}

// count: per warp tile, entries per bucket; per band, the tiles' exclusive offsets (m) and the band's totals (b)
template <int LEVEL, int G>
__global__ void __launch_bounds__(32 * SP_WARPS) split_count_kernel(const SplitParams p) {
    __shared__ uint32_t s_cnt[SP_WARPS][32 * G];
    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, band = blockIdx.x;
    int64_t beg, end;
    int row = 0;
    if (LEVEL == 1) {
        beg = (int64_t)band * SP_BAND;
        end = min(beg + SP_BAND, p.n);
    } else {
        if (band >= (int)p.band_begin[p.rows]) return;  // (uniform: the launch covers the largest band count)
        row = split_band_row(p, band, beg, end);
    }
    uint32_t member[G], cnt[G];
    split_members<LEVEL, G>(p, row, member);
#pragma unroll
    for (int g = 0; g < G; ++g) cnt[g] = 0u;
    const int64_t tb = beg + (int64_t)w * SP_TILE;
    split_walk<LEVEL, G, true>(p, LEVEL == 1 ? p.val_sorted : p.row_list, tb, min(tb + SP_TILE, end), member, cnt,
                               [](uint32_t, unsigned long long) {});
#pragma unroll
    for (int g = 0; g < G; ++g) s_cnt[w][32 * g + lane] = cnt[g];
    __syncthreads();
    const int width = 32 * G;
    uint32_t* m = (LEVEL == 1 ? p.m1 : p.m2) + (int64_t)band * (SP_WARPS + 1) * width;
    for (int c = threadIdx.x; c < width; c += 32 * SP_WARPS) {
        uint32_t run = 0;
#pragma unroll
        for (int w2 = 0; w2 < SP_WARPS; ++w2) {
            m[w2 * width + c] = run;
            run += s_cnt[w2][c];
        }
        m[SP_WARPS * width + c] = run;
        (LEVEL == 1 ? p.b1 : p.b2)[(int64_t)band * width + c] = run;
    }
}

// scatter: every bucket starts at its band's offset + the tile's offset within the band.  A tile whose output fits
// SP_STAGE_BYTES is first ranked into shared memory, bucket after bucket, then copied out one contiguous run per bucket
// (coalesced stores; ranked straight into global memory every store of the warp hit 32 different runs).
template <int LEVEL, int G>
__global__ void __launch_bounds__(32 * SP_WARPS) split_scatter_kernel(const SplitParams p) {
    using T = typename std::conditional<LEVEL == 1, unsigned long long, uint32_t>::type;
    extern __shared__ __align__(16) unsigned char smem_sp[];
    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, band = blockIdx.x;
    int64_t beg, end;
    int row = 0;
    if (LEVEL == 1) {
        beg = (int64_t)band * SP_BAND;
        end = min(beg + SP_BAND, p.n);
    } else {
        if (band >= (int)p.band_begin[p.rows]) return;
        row = split_band_row(p, band, beg, end);
    }
    const int64_t tb = beg + (int64_t)w * SP_TILE;
    if (tb >= end) return;  // (uniform per warp; no barrier below)
    const int width = 32 * G;
    const uint32_t* m = (LEVEL == 1 ? p.m1 : p.m2) + ((int64_t)band * (SP_WARPS + 1) + w) * width;
    const uint32_t* bo = (LEVEL == 1 ? p.b1 : p.b2) + (int64_t)band * width;
    T* dst = LEVEL == 1 ? (T*)p.row_list : (T*)p.inst_gid;
    uint32_t member[G], off[G], cnt[G], sbeg[G], pos[G];
    split_members<LEVEL, G>(p, row, member);
    uint32_t total = 0;
#pragma unroll
    for (int g = 0; g < G; ++g) {
        const uint32_t m0 = m[32 * g + lane];
        off[g] = bo[32 * g + lane] + m0;
        cnt[g] = m[width + 32 * g + lane] - m0;
        // exclusive scan of the counts over the buckets: where the bucket's run starts in the staging area
        uint32_t inc = cnt[g];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        sbeg[g] = total + inc - cnt[g];
        total += __shfl_sync(0xffffffffu, inc, 31);
    }
    const int64_t te = min(tb + SP_TILE, end);
    constexpr int CAP = SP_STAGE_BYTES / (int)sizeof(T);
    if (total > (uint32_t)CAP) {  // (uniform) a tile of wide splats: rank straight into global memory
        split_walk<LEVEL, G, false>(p, LEVEL == 1 ? p.val_sorted : p.row_list, tb, te, member, off,
                                    [&](uint32_t q, unsigned long long x) { dst[q] = (T)x; });
        return;
    }
    T* stage = reinterpret_cast<T*>(smem_sp + w * SP_STAGE_BYTES);
#pragma unroll
    for (int g = 0; g < G; ++g) pos[g] = sbeg[g];
    split_walk<LEVEL, G, false>(p, LEVEL == 1 ? p.val_sorted : p.row_list, tb, te, member, pos,
                                [&](uint32_t q, unsigned long long x) { stage[q] = (T)x; });
    __syncwarp();
#pragma unroll
    for (int g = 0; g < G; ++g) {
        unsigned todo = __ballot_sync(0xffffffffu, cnt[g] != 0u);
        while (todo) {
            const int b = __ffs(todo) - 1;
            todo &= todo - 1u;
            const uint32_t len = __shfl_sync(0xffffffffu, cnt[g], b), s0 = __shfl_sync(0xffffffffu, sbeg[g], b);
            const uint32_t d0 = __shfl_sync(0xffffffffu, off[g], b);
            for (uint32_t k = lane; k < len; k += 32) dst[d0 + k] = stage[s0 + k];
        }
    }
}

// Level-1 scan (one CTA): per row, the total over the bands; the rows' list offsets and level-2 band layout; every band
// total of b1 rewritten as the absolute offset of the band's first entry in its row.  Row lists that do not fit
// row_capacity fail the frame (CAP_OVERFLOW, the row-list size in ROW_INST: the caller grows the buffer and replays).
__global__ void __launch_bounds__(1024) split_rows_scan_kernel(const SplitParams p) {
    __shared__ uint32_t s_part[SP_MAX_GROUPS][32][33];
    __shared__ uint32_t s_begin[SP_MAX_CELLS];
    __shared__ int s_over;
    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    if (p.base_split) {
        int split = 0;
        for (int i = threadIdx.x; i < p.rows * p.cols; i += 1024) split |= p.cell_leaf[i] == -2;
        split = __syncthreads_or(split);
        if (threadIdx.x == 0) *p.base_split = split ? 1u : 0u;
    }
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int groups = p.rows_p / 32;
    const int per = (p.bands1 + 31) / 32;
    const int c0 = min(p.bands1, ty * per), c1 = min(p.bands1, c0 + per);
    for (int g = 0; g < groups; ++g) {
        const uint32_t* col = p.b1 + 32 * g + tx;
        uint32_t sum = 0;
#pragma unroll 8
        for (int c = c0; c < c1; ++c) sum += col[(int64_t)c * p.rows_p];
        s_part[g][ty][tx] = sum;
    }
    __syncthreads();
    if (ty == 0) {
        // warp 0: row totals, then an exclusive scan over the rows (each lane takes 8 consecutive rows)
        unsigned long long tot[SP_MAX_GROUPS], bands[SP_MAX_GROUPS], st = 0, sb = 0;
#pragma unroll
        for (int i = 0; i < SP_MAX_GROUPS; ++i) {
            const int r = tx * SP_MAX_GROUPS + i;
            uint32_t t = 0;
            if (r < p.rows)
                for (int s = 0; s < 32; ++s) t += s_part[r >> 5][s][r & 31];
            tot[i] = t;
            bands[i] = (t + SP_BAND - 1) / SP_BAND;
            st += tot[i];
            sb += bands[i];
        }
        unsigned long long it = st, ib = sb;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long a = __shfl_up_sync(0xffffffffu, it, o), b = __shfl_up_sync(0xffffffffu, ib, o);
            if (tx >= o) { it += a; ib += b; }
        }
        unsigned long long rt = it - st, rb = ib - sb;
        const unsigned long long total = __shfl_sync(0xffffffffu, it, 31);
        const bool over = total > (unsigned long long)p.row_capacity;
        if (!over) {
#pragma unroll
            for (int i = 0; i < SP_MAX_GROUPS; ++i) {
                const int r = tx * SP_MAX_GROUPS + i;
                if (r < p.rows) {
                    p.row_begin[r] = (uint32_t)rt;
                    p.band_begin[r] = (uint32_t)rb;
                    s_begin[r] = (uint32_t)rt;
                }
                rt += tot[i];
                rb += bands[i];
            }
            if (tx == 31) {
                p.row_begin[p.rows] = (uint32_t)rt;
                p.band_begin[p.rows] = (uint32_t)rb;
            }
        }
        if (tx == 0) {
            s_over = over ? 1 : 0;
            p.header[G2PC_HDR_ROW_INST] = (int32_t)min(total, 0x7FFFFFFFull);
            if (over) {
                p.header[G2PC_HDR_CAP_OVERFLOW] = 1;
                atomicMin(p.fail, (uint32_t)(p.frame + 1));
                p.header[G2PC_HDR_POISON] = (int32_t)*(volatile uint32_t*)p.fail;
            }
        }
    }
    __syncthreads();
    if (s_over) return;
    for (int g = 0; g < groups; ++g) {
        const int r = 32 * g + tx;
        if (r >= p.rows) continue;
        uint32_t run = s_begin[r];
        for (int s = 0; s < ty; ++s) run += s_part[g][s][tx];
        uint32_t* col = p.b1 + r;
        for (int c = c0; c < c1; ++c) {
            const uint32_t t = col[(int64_t)c * p.rows_p];
            col[(int64_t)c * p.rows_p] = run;
            run += t;
        }
    }
}

// Level-2 scan: one thread per cell (row, column): its bands' totals rewritten as the absolute offset of each band's
// first id in the leaf's list (starting at the leaf's inst_begin).
__global__ void __launch_bounds__(256) split_cols_scan_kernel(const SplitParams p) {
    if (g2pc_frame_skipped(p.fail, p.frame)) return;
    const int i = blockIdx.x * 256 + threadIdx.x;
    const int row = i / p.cols_p, c = i - row * p.cols_p;
    if (row >= p.rows) return;
    uint32_t run = 0;
    if (c < p.cols) {
        const int leaf = p.cell_leaf ? p.cell_leaf[row * p.cols + c] : row * p.cols + c;
        if (leaf >= 0) run = (uint32_t)p.leaves[leaf].inst_begin;
    }
    const int b0 = (int)p.band_begin[row], b1 = (int)p.band_begin[row + 1];
    uint32_t* col = p.b2 + c;
    for (int b = b0; b < b1; ++b) {
        const uint32_t t = col[(int64_t)b * p.cols_p];
        col[(int64_t)b * p.cols_p] = run;
        run += t;
    }
}

size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

int64_t split_bands1(int64_t n) { return (n + SP_BAND - 1) / SP_BAND; }
int64_t split_bands2(int64_t row_capacity, int rows) { return (row_capacity + SP_BAND - 1) / SP_BAND + rows; }

// workspace of the two splits: [base_split][row_list][m1][b1][m2][b2][row_begin][band_begin], each 256-byte aligned
int64_t split_workspace_bytes(int64_t n, int64_t row_capacity, int rows, int cols) {
    const int64_t rp = (rows + 31) / 32 * 32, cp = (cols + 31) / 32 * 32;
    const int64_t b1 = split_bands1(n), b2 = split_bands2(row_capacity, rows);
    return (int64_t)(align256(4) + align256((size_t)row_capacity * 8) + align256((size_t)(b1 * (SP_WARPS + 1) * rp * 4)) +
                     align256((size_t)(b1 * rp * 4)) + align256((size_t)(b2 * (SP_WARPS + 1) * cp * 4)) +
                     align256((size_t)(b2 * cp * 4)) + 2 * align256((size_t)(rows + 1) * 4));
}

template <int LEVEL, int G>
void split_launch_level(const SplitParams& p, int64_t bands, cudaStream_t st) {
    split_count_kernel<LEVEL, G><<<(unsigned)bands, 32 * SP_WARPS, 0, st>>>(p);
    if (LEVEL == 1) split_rows_scan_kernel<<<1, 1024, 0, st>>>(p);
    else split_cols_scan_kernel<<<(unsigned)((p.rows * p.cols_p + 255) / 256), 256, 0, st>>>(p);
    constexpr size_t smem = (size_t)SP_WARPS * SP_STAGE_BYTES;
    cudaFuncSetAttribute(split_scatter_kernel<LEVEL, G>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    split_scatter_kernel<LEVEL, G><<<(unsigned)bands, 32 * SP_WARPS, smem, st>>>(p);
}

template <int LEVEL>
void split_level(const SplitParams& p, int64_t bands, cudaStream_t st) {
    switch ((LEVEL == 1 ? p.rows_p : p.cols_p) / 32) {
        case 1: split_launch_level<LEVEL, 1>(p, bands, st); break;
        case 2: split_launch_level<LEVEL, 2>(p, bands, st); break;
        case 3: split_launch_level<LEVEL, 3>(p, bands, st); break;
        case 4: split_launch_level<LEVEL, 4>(p, bands, st); break;
        case 5: split_launch_level<LEVEL, 5>(p, bands, st); break;
        case 6: split_launch_level<LEVEL, 6>(p, bands, st); break;
        case 7: split_launch_level<LEVEL, 7>(p, bands, st); break;
        default: split_launch_level<LEVEL, 8>(p, bands, st); break;
    }
}

// The base-level lists of an n-entry stream over a rows x cols grid (both <= 256).  Returns G2PC_OK or an error code.
int run_split(SplitParams p, void* workspace, int64_t workspace_bytes, cudaStream_t st) {
    if (workspace_bytes < split_workspace_bytes(p.n, p.row_capacity, p.rows, p.cols)) {
        g2pc_set_error("g2pc_multisplit: workspace smaller than g2pc_multisplit_workspace_bytes");
        return G2PC_ERR_WORKSPACE;
    }
    p.rows_p = (p.rows + 31) / 32 * 32;
    p.cols_p = (p.cols + 31) / 32 * 32;
    const int64_t b1 = split_bands1(p.n), b2 = split_bands2(p.row_capacity, p.rows);
    char* ws = (char*)workspace;
    auto take = [&](size_t bytes) { char* q = ws; ws += align256(bytes); return q; };
    uint32_t* flag = (uint32_t*)take(4);
    p.base_split = p.cell_leaf ? flag : nullptr;
    p.row_list = (unsigned long long*)take((size_t)p.row_capacity * 8);
    p.m1 = (uint32_t*)take((size_t)(b1 * (SP_WARPS + 1) * p.rows_p * 4));
    p.b1 = (uint32_t*)take((size_t)(b1 * p.rows_p * 4));
    p.m2 = (uint32_t*)take((size_t)(b2 * (SP_WARPS + 1) * p.cols_p * 4));
    p.b2 = (uint32_t*)take((size_t)(b2 * p.cols_p * 4));
    p.row_begin = (uint32_t*)take((size_t)(p.rows + 1) * 4);
    p.band_begin = (uint32_t*)take((size_t)(p.rows + 1) * 4);
    p.bands1 = (int32_t)b1;
    split_level<1>(p, b1, st);
    split_level<2>(p, b2, st);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}


// Sub-steps per chunk for n entries: as many as keep about MS_TARGET_CTAS chunks, ~10 waves of the 3 scatter CTAs an SM
// of an H100 SXM (132 SMs) holds at C = 256.  Measured at 3 M Gaussians / 1280x720 (count + scatter per camera, H100
// 80GB HBM3 at 400 W): 1 sub-step 565 us, 2 sub-steps (~4 k chunks) 522 us, 7 sub-steps (~1.5 k chunks) 601 us — longer
// chunks save set-up but leave the waves unbalanced.  C3 (C = 256): 2 sub-steps, E = 512, 5860 chunks.
constexpr int64_t MS_TARGET_CTAS = 4096;
constexpr int64_t MS_MAX_STEPS = 32;
int32_t ms_steps(int64_t n, int C) {
    const int64_t s = n / ((int64_t)C * MS_TARGET_CTAS);
    return (int32_t)(s < 1 ? 1 : (s > MS_MAX_STEPS ? MS_MAX_STEPS : s));
}

int32_t ms_chunks(int64_t n, int C) {
    const int64_t e = (int64_t)C * ms_steps(n, C);
    return (int32_t)((n + e - 1) / e);
}

template <int C>
int launch_multisplit(const MsParams& p, int32_t chunks, cudaStream_t st) {
    const size_t common = ((size_t)6 * p.n1 + ((size_t)1 << (2 * p.base_level))) * sizeof(int32_t);
    const size_t smem_count = common + (size_t)p.leaf_cap * sizeof(uint32_t);
    const size_t smem_scatter = common + (size_t)(C / 32 + 1) * p.leaf_cap * sizeof(uint32_t);
    if (smem_scatter > 200 * 1024 || smem_count > 200 * 1024) {
        g2pc_set_error("g2pc_multisplit: shared memory budget exceeded");
        return G2PC_ERR_INVALID;
    }
    if (smem_count > 48 * 1024)
        G2PC_CUDA(cudaFuncSetAttribute(ms_count_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_count));
    if (smem_scatter > 48 * 1024)
        G2PC_CUDA(cudaFuncSetAttribute(ms_scatter_kernel<C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_scatter));
    ms_count_kernel<C><<<(unsigned)chunks, C, smem_count, st>>>(p);
    G2PC_CHECK_LAUNCH();
    ms_scan_kernel<<<(unsigned)((p.leaf_cap + 31) / 32), 1024, 0, st>>>(p, chunks);
    G2PC_CHECK_LAUNCH();
    ms_scatter_kernel<C><<<(unsigned)chunks, C, smem_scatter, st>>>(p);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

// the rest of g2pc_multisplit / g2pc_multisplit_grid once p is filled: sub-steps and chunks for n entries at C per sub-step
int run_multisplit(MsParams p, int C, cudaStream_t st) {
    p.steps = ms_steps(p.n, C);
    const int32_t chunks = ms_chunks(p.n, C);
    if (C == 256) return launch_multisplit<256>(p, chunks, st);
    if (C == 128) return launch_multisplit<128>(p, chunks, st);
    return launch_multisplit<64>(p, chunks, st);
}

}  // namespace

extern "C" int g2pc_build_tree(const int32_t* tables, int32_t num_levels, int32_t max_gaussians_per_tile,
                               uint32_t* node_cnt, uint8_t* node_state, int32_t* node_leaf, g2pc_leaf_t* leaves,
                               int32_t* leaf_order, int32_t max_leaves, int64_t inst_capacity, int64_t pix_capacity,
                               int64_t matrix_capacity, int32_t ms_chunks, int32_t frame, int32_t* header,
                               uint32_t* fail, int32_t* work_counters, void* stream) {
    G2PC_CHECK_ARG(tables && node_cnt && node_state && node_leaf && leaves && leaf_order && header && fail &&
                       work_counters, "null pointer");
    G2PC_CHECK_ARG(num_levels >= 1 && num_levels <= G2PC_MAX_LEVELS && max_leaves >= 1, "bad sizes");
    G2PC_CHECK_ARG(frame >= 0 && ms_chunks >= 0, "bad frame / chunk count");
    TreeParams p;
    p.meta.num_levels = num_levels; p.meta.max_gaussians_per_tile = max_gaussians_per_tile;
    p.meta.width = 0; p.meta.height = 0;
    p.n1 = (1 << num_levels) - 1;
    p.tab = make_tables(tables, p.n1);
    p.node_cnt = node_cnt; p.node_state = node_state; p.node_leaf = node_leaf; p.leaves = leaves;
    p.leaf_order = leaf_order; p.max_leaves = max_leaves;
    p.inst_capacity = inst_capacity; p.pix_capacity = pix_capacity; p.matrix_capacity = matrix_capacity;
    p.ms_chunks = ms_chunks; p.frame = frame; p.header = header; p.fail = fail; p.work_counters = work_counters;
    p.nodes_2d = off2d(num_levels);
    tree_kernel<<<1, TB, 0, (cudaStream_t)stream>>>(p);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

// workspace layout of g2pc_depth_sort: [keys_out n u32][cub temp]
extern "C" int64_t g2pc_depth_sort_workspace_bytes(int64_t n) {
    size_t sort_b = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, sort_b, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                    (const unsigned long long*)nullptr, (unsigned long long*)nullptr, n);
    return (int64_t)(align256((size_t)n * 4) + align256(sort_b));
}

/* Sort the (depth key, value) pairs by key (stable: ties keep index order) -> val_sorted[k] = value of the k-th nearest
 * Gaussian. */
extern "C" int g2pc_depth_sort(const uint32_t* depth_key, const uint64_t* val, int64_t n, uint64_t* val_sorted,
                               void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(depth_key && val && val_sorted && workspace, "null pointer");
    G2PC_CHECK_ARG(workspace_bytes >= g2pc_depth_sort_workspace_bytes(n), "workspace too small");
    char* ws = (char*)workspace;
    uint32_t* keys_out = (uint32_t*)ws;
    void* tmp = ws + align256((size_t)n * 4);
    size_t b = (size_t)workspace_bytes - align256((size_t)n * 4);
    G2PC_CUDA(cub::DeviceRadixSort::SortPairs(tmp, b, depth_key, keys_out, (const unsigned long long*)val,
                                              (unsigned long long*)val_sorted, n, 0, 32, (cudaStream_t)stream));
    return G2PC_OK;
}

extern "C" int32_t g2pc_multisplit_chunk(int32_t leaf_cap) {
    // entries per sub-step: the scatter kernel keeps leaf_cap x (sub-step bits + one offset) in shared memory.  Prefer a
    // footprint that lets 3 CTAs share an SM (the kernel is a chain of short latency-bound phases: with one resident CTA
    // per SM the 3600-tile grid of the CUDA back-end ran 3.5x slower per instance than the 1024 leaves of the python one)
    const int64_t n = leaf_cap;
    if (n * 36 <= 74 * 1024) return 256;
    if (n * 20 <= 74 * 1024) return 128;
    if (n * 12 <= 110 * 1024) return 64;
    if (n * 20 <= 200 * 1024) return 128;
    if (n * 12 <= 200 * 1024) return 64;
    return 0;
}

extern "C" int32_t g2pc_multisplit_rows(int64_t n, int32_t leaf_cap) {
    // matrix rows the multisplit needs for n entries: one per chunk of ms_steps x C entries
    const int C = g2pc_multisplit_chunk(leaf_cap);
    if (C <= 0) return 0;
    return ms_chunks(n, C);
}

extern "C" int64_t g2pc_multisplit_workspace_bytes(int64_t n, int64_t row_capacity, int32_t grid_w, int32_t grid_h) {
    if (n < 0 || row_capacity < 0 || grid_w < 1 || grid_h < 1 || grid_w > SP_MAX_CELLS || grid_h > SP_MAX_CELLS) return -1;
    return split_workspace_bytes(n, row_capacity, grid_h, grid_w);
}

extern "C" int g2pc_multisplit(const uint64_t* val_sorted, int64_t n, const void* proj, int32_t width, int32_t height,
                               const int32_t* tables, int32_t num_levels, uint32_t level_mask, uint32_t clean_mask,
                               const int32_t* node_leaf, const g2pc_leaf_t* leaves, int32_t* header,
                               const uint32_t* fail, int32_t frame, int32_t leaf_cap, uint32_t* matrix,
                               int64_t row_capacity, void* workspace, int64_t workspace_bytes, uint32_t* inst_gid,
                               void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(val_sorted && proj && tables && node_leaf && leaves && header && fail && workspace && inst_gid,
                   "null pointer");
    G2PC_CHECK_ARG(num_levels >= 1 && num_levels <= G2PC_MAX_LEVELS && level_mask != 0u, "bad levels");
    G2PC_CHECK_ARG(row_capacity >= 0 && row_capacity <= 0x7FFFFFFFll, "bad row capacity");
    const int base = __builtin_ctz(level_mask);
    G2PC_CHECK_ARG(base <= G2PC_RANGE_MAX_LEVEL, "first leaf-candidate level too deep");
    const int n1 = (1 << num_levels) - 1, o1 = (1 << base) - 1;
    const QtTables tab = make_tables(tables, n1);
    cudaStream_t st = (cudaStream_t)stream;
    SplitParams s{};
    s.val_sorted = (const unsigned long long*)val_sorted; s.n = n;
    s.rows = s.cols = 1 << base;
    s.cell_leaf = node_leaf + off2d(base);
    s.tab.xs = tab.xs + o1; s.tab.xe = tab.xe + o1; s.tab.xf = tab.xf + o1;
    s.tab.ys = tab.ys + o1; s.tab.ye = tab.ye + o1; s.tab.yf = tab.yf + o1;
    s.clean = (int32_t)((clean_mask >> base) & 1u);
    s.leaves = leaves; s.header = header; s.fail = const_cast<uint32_t*>(fail); s.frame = frame;
    s.row_capacity = row_capacity; s.inst_gid = inst_gid;
    const int rc = run_split(s, workspace, workspace_bytes, st);
    if (rc != G2PC_OK || num_levels <= base + 1) return rc;
    // leaves below the base level (count-driven splits): the chunked multisplit
    const int C = g2pc_multisplit_chunk(leaf_cap);
    G2PC_CHECK_ARG(C > 0, "too many leaves for the multisplit");
    G2PC_CHECK_ARG(matrix, "null matrix with levels below the base level");
    MsParams p;
    p.val_sorted = (const unsigned long long*)val_sorted; p.n = n; p.proj = (const float4*)proj;
    p.width = width; p.height = height;
    p.inv_width = 1.0f / (float)width; p.inv_height = 1.0f / (float)height;
    p.meta.num_levels = num_levels; p.meta.max_gaussians_per_tile = 0; p.meta.width = width; p.meta.height = height;
    p.n1 = n1;
    p.tab = tab;
    p.level_mask = level_mask; p.base_level = base;
    p.node_leaf = node_leaf; p.header = header; p.fail = fail; p.frame = frame; p.leaves = leaves; p.matrix = matrix;
    p.inst_gid = inst_gid;
    p.leaf_cap = leaf_cap;
    p.base_clean = s.clean;
    p.clean_mask = clean_mask;
    p.base_split = (const uint32_t*)workspace;  // (first word of the workspace, run_split)
    return run_multisplit(p, C, st);
}

/* The same lists over a flat grid of tiles (s7_tiles.cu): leaf = tile index, the packed range is the tile rect. */
extern "C" int g2pc_multisplit_grid(const uint64_t* val_sorted, int64_t n, int32_t grid_w, int32_t grid_h,
                                    const g2pc_leaf_t* leaves, int32_t* header, const uint32_t* fail, int32_t frame,
                                    int64_t row_capacity, void* workspace, int64_t workspace_bytes, uint32_t* inst_gid,
                                    void* stream) {
    G2PC_CHECK_ARG(n >= 0, "n < 0");
    if (n == 0) return G2PC_OK;
    G2PC_CHECK_ARG(val_sorted && leaves && header && fail && workspace && inst_gid, "null pointer");
    G2PC_CHECK_ARG(grid_w >= 1 && grid_h >= 1 && grid_w <= SP_MAX_CELLS && grid_h <= SP_MAX_CELLS, "bad tile grid");
    G2PC_CHECK_ARG(row_capacity >= 0 && row_capacity <= 0x7FFFFFFFll, "bad row capacity");
    SplitParams s{};  // no quadtree tables or node -> leaf map: every cell is a leaf, every range is exact
    s.val_sorted = (const unsigned long long*)val_sorted; s.n = n;
    s.rows = grid_h; s.cols = grid_w;
    s.clean = 1;
    s.leaves = leaves; s.header = header; s.fail = const_cast<uint32_t*>(fail); s.frame = frame;
    s.row_capacity = row_capacity; s.inst_gid = inst_gid;
    return run_split(s, workspace, workspace_bytes, (cudaStream_t)stream);
}
