// s15_components.cu — connected components of a triangle mesh and the filter that removes the small ones (N11).
// The rules are this project's own (DESIGN.md §2, N11) and tests/f64ref_components.py restates them.
//
// label: a concurrent union-find over the vertices, two unions per face ((a, b) and (a, c)).  A union hooks the larger
// root under the smaller with atomicCAS and retries from the new root when the CAS fails; path halving stores only
// ancestors, with atomicMin.  Every parent pointer therefore only decreases and stays below its vertex, so each root is
// the smallest vertex of its set: the labels do not depend on the order the atomics take.  One pass then stores every
// vertex's root (its label) and integer atomics count the triangles per label.  select: the keep flag per vertex (size
// >= max(1, min_triangles), rank < keep_largest by (size descending, label ascending) from a CUB sort of the roots) and
// the exclusive scans of the vertex and triangle flags.  compact: the density trim's stable compaction (mesh_common.cuh).
#include <cub/cub.cuh>
#include "mesh_common.cuh"

namespace {

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

__global__ void __launch_bounds__(MB) union_kernel(const int32_t* __restrict__ faces, int64_t t, int32_t* parent) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f >= t) return;
    const int a = faces[3 * f], b = faces[3 * f + 1], c = faces[3 * f + 2];
    unite(parent, a, b);
    unite(parent, a, c);
}

__global__ void __launch_bounds__(MB) size_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                  const int32_t* __restrict__ labels, int32_t* __restrict__ sizes) {
    const int64_t f = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (f < t) atomicAdd(&sizes[labels[faces[3 * f]]], 1);
}

// counts[0] = components with at least one triangle, counts[1] = the largest size
__global__ void __launch_bounds__(MB) component_count_kernel(const int32_t* __restrict__ labels,
                                                             const int32_t* __restrict__ sizes, int64_t m,
                                                             unsigned long long* __restrict__ counts) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || labels[v] != v || sizes[v] == 0) return;
    atomicAdd(&counts[0], 1ull);
    atomicMax(&counts[1], (unsigned long long)sizes[v]);
}

// (~size) << 32 | label of every root with a triangle, in any order (the sort fixes it)
__global__ void __launch_bounds__(MB) root_keys_kernel(const int32_t* __restrict__ labels,
                                                       const int32_t* __restrict__ sizes, int64_t m,
                                                       unsigned long long* __restrict__ slot,
                                                       unsigned long long* __restrict__ keys) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || labels[v] != v || sizes[v] == 0) return;
    keys[atomicAdd(slot, 1ull)] = (unsigned long long)(~(uint32_t)sizes[v]) << 32 | (uint64_t)v;
}

// the k first sorted roots have rank < keep_largest
__global__ void __launch_bounds__(MB) rank_mark_kernel(const unsigned long long* __restrict__ sorted, int64_t k,
                                                       uint8_t* __restrict__ ranked) {
    const int64_t r = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (r < k) ranked[(uint32_t)sorted[r]] = 1;
}

// keep[v] = its component has >= min_size triangles and (ranked null or) a rank below keep_largest; counts[2] = kept
// components
__global__ void __launch_bounds__(MB) component_keep_kernel(const int32_t* __restrict__ labels,
                                                            const int32_t* __restrict__ sizes, int64_t m,
                                                            int64_t min_size, const uint8_t* __restrict__ ranked,
                                                            uint8_t* __restrict__ keep, int32_t* __restrict__ flag,
                                                            unsigned long long* __restrict__ kept) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int L = labels[v];
    const int k = sizes[L] >= min_size && (!ranked || ranked[L]) ? 1 : 0;
    keep[v] = (uint8_t)k;
    flag[v] = k;
    if (k && L == v) atomicAdd(kept, 1ull);
}

// select and compact share this layout (compact reads vmap, tflag, tmap)
struct SelectWs {
    int32_t *vflag, *vmap, *tflag, *tmap;
    unsigned long long *keys_a, *keys_b, *slot;
    uint8_t* ranked;
    void* tmp;
    size_t tmp_bytes, bytes;
};
SelectWs select_ws(void* base, int64_t m, int64_t t) {
    size_t b[3] = {0, 0, 0};
    cub::DeviceScan::ExclusiveSum(nullptr, b[0], (const int32_t*)nullptr, (int32_t*)nullptr, (int)m);
    cub::DeviceScan::ExclusiveSum(nullptr, b[1], (const int32_t*)nullptr, (int32_t*)nullptr, (int)t);
    cub::DeviceRadixSort::SortKeys(nullptr, b[2], (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                   (int)m);
    size_t tb = 0;
    for (size_t x : b) tb = tb > x ? tb : x;
    WsCarve w{(char*)base};
    SelectWs l;
    l.vflag = w.take<int32_t>(m);
    l.vmap = w.take<int32_t>(m);
    l.tflag = w.take<int32_t>(t);
    l.tmap = w.take<int32_t>(t);
    l.keys_a = w.take<unsigned long long>(m);
    l.keys_b = w.take<unsigned long long>(m);
    l.slot = w.take<unsigned long long>(1);
    l.ranked = w.take<uint8_t>(m);
    l.tmp_bytes = WsCarve::pad(tb);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

bool sizes_ok(int64_t m, int64_t t) { return m > 0 && m < 0x7FFFFFFFll && t >= 0 && 3 * t < 0x7FFFFFFFll; }

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int g2pc_mesh_components_label(const int32_t* faces, int64_t m, int64_t t, int32_t* labels, int32_t* sizes,
                                          int64_t* counts, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(labels && sizes && counts && (t == 0 || faces), "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 2 * sizeof(int64_t), st));
    G2PC_CUDA(cudaMemsetAsync(sizes, 0, (size_t)m * 4, st));
    parent_init_kernel<<<grid_of(m), MB, 0, st>>>(labels, m);
    G2PC_CHECK_LAUNCH();
    if (t > 0) {
        union_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, labels);
        G2PC_CHECK_LAUNCH();
    }
    compress_kernel<<<grid_of(m), MB, 0, st>>>(labels, m);
    G2PC_CHECK_LAUNCH();
    if (t > 0) {
        size_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, labels, sizes);
        G2PC_CHECK_LAUNCH();
    }
    component_count_kernel<<<grid_of(m), MB, 0, st>>>(labels, sizes, m, (unsigned long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int64_t g2pc_mesh_components_select_workspace_bytes(int64_t m, int64_t t) {
    return sizes_ok(m, t) ? (int64_t)select_ws(nullptr, m, t).bytes : 0;
}

extern "C" int g2pc_mesh_components_select(const int32_t* faces, int64_t m, int64_t t, const int32_t* labels,
                                           const int32_t* sizes, int64_t components, int64_t min_triangles,
                                           int64_t keep_largest, uint8_t* keep, int64_t* counts, void* workspace,
                                           int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(components >= 0 && components <= m && min_triangles >= 0 && keep_largest >= 0,
                   "need 0 <= components <= m, min_triangles >= 0 and keep_largest >= 0");
    G2PC_CHECK_ARG(labels && sizes && keep && counts && workspace && (t == 0 || faces), "null pointer");
    const SelectWs l = select_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 3 * sizeof(int64_t), st));
    const uint8_t* ranked = nullptr;
    if (keep_largest > 0 && keep_largest < components) {
        G2PC_CUDA(cudaMemsetAsync(l.slot, 0, 8, st));
        root_keys_kernel<<<grid_of(m), MB, 0, st>>>(labels, sizes, m, l.slot, l.keys_a);
        G2PC_CHECK_LAUNCH();
        size_t b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceRadixSort::SortKeys(l.tmp, b, l.keys_a, l.keys_b, (int)components, 0, 64, st));
        G2PC_CUDA(cudaMemsetAsync(l.ranked, 0, (size_t)m, st));
        rank_mark_kernel<<<grid_of(keep_largest), MB, 0, st>>>(l.keys_b, keep_largest, l.ranked);
        G2PC_CHECK_LAUNCH();
        ranked = l.ranked;
    }
    const int64_t min_size = min_triangles > 1 ? min_triangles : 1;
    component_keep_kernel<<<grid_of(m), MB, 0, st>>>(labels, sizes, m, min_size, ranked, keep, l.vflag,
                                                     (unsigned long long*)counts + 2);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.vflag, l.vmap, (int)m, st));
    if (t > 0) {
        tri_flag_kernel<<<grid_of(t), MB, 0, st>>>(faces, t, keep, l.tflag);
        G2PC_CHECK_LAUNCH();
        b = l.tmp_bytes;
        G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.tflag, l.tmap, (int)t, st));
    }
    trim_counts_kernel<<<1, 1, 0, st>>>(l.vflag, l.vmap, m, l.tflag, l.tmap, t, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_components_compact(const double* vpos, const uint8_t* vcolours, const double* density,
                                            int64_t m, const int32_t* faces, int64_t t, const uint8_t* keep,
                                            double* vpos_out, uint8_t* vcolours_out, double* density_out,
                                            int32_t* faces_out, const void* workspace, int64_t workspace_bytes,
                                            void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(vpos && density && keep && vpos_out && density_out && workspace, "null pointer");
    G2PC_CHECK_ARG(!vcolours == !vcolours_out, "vertex colours need an output");
    G2PC_CHECK_ARG(t == 0 || (faces && faces_out), "null pointer");
    const SelectWs l = select_ws(const_cast<void*>(workspace), m, t);  // read only here
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    if (t > 0) {
        compact_faces_kernel<<<grid_of(t), MB, 0, st>>>(faces, l.tflag, l.tmap, t, l.vmap, faces_out);
        G2PC_CHECK_LAUNCH();
    }
    compact_vertices_kernel<<<grid_of(m), MB, 0, st>>>(keep, l.vmap, m, density, vpos, vcolours, density_out, vpos_out,
                                                       vcolours_out);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
