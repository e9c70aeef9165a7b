// s16_holes.cu — closing the small holes of a triangle mesh by filling its short boundary loops (N12).
// The rules are this project's own (DESIGN.md §2, N12) and tests/f64ref_holes.py restates them.
//
// find: the 3t undirected edge keys (min << 32 | max) of the half-edges, with the half-edge (3 face + corner) as
// payload, sorted by CUB; a run of one key is a boundary half-edge.  Integer atomics count each vertex's outgoing and
// incoming boundary half-edges; succ[u] is the target of u's boundary half-edge where u has exactly one.  The union-find
// of N11 (mesh_common.cuh) over the boundary half-edges labels the boundary sets by their smallest vertex, and integer
// atomics give each label its vertex count L and a pinched flag (a vertex without exactly one outgoing and one incoming
// boundary half-edge).  plan: the filled flag per label (a hole with L <= H that is not a lone triangle) and the exclusive
// scans that give each filled hole its centre index and its first face.  fill: the input copied into the outputs, then
// one thread per filled hole walks its loop from the label and writes its faces and centre.  Every float64 sum runs in
// loop order in one thread, so no output depends on the order the atomics take.
#include <cub/cub.cuh>
#include "mesh_common.cuh"

namespace {

unsigned grid_of(int64_t n) { return (unsigned)((n + MB - 1) / MB); }

// half-edge c = 3 f + s runs from corner s of face f to corner s + 1
__device__ __forceinline__ void half_edge(const int32_t* __restrict__ faces, int c, int& u, int& v) {
    const int s = c % 3;
    u = faces[c];
    v = faces[c - s + (s == 2 ? 0 : s + 1)];
}

__global__ void __launch_bounds__(MB) edge_keys_kernel(const int32_t* __restrict__ faces, int64_t t,
                                                       unsigned long long* __restrict__ keys,
                                                       int32_t* __restrict__ vals) {
    const int64_t c = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (c >= 3 * t) return;
    int u, v;
    half_edge(faces, (int)c, u, v);
    const unsigned long long lo = (uint32_t)(u < v ? u : v), hi = (uint32_t)(u < v ? v : u);
    keys[c] = lo << 32 | hi;
    vals[c] = (int32_t)c;
}

// the sorted key at i is the only one of its value: its half-edge is on the boundary
__device__ __forceinline__ bool run_of_one(const unsigned long long* __restrict__ keys, int64_t e, int64_t i) {
    const unsigned long long k = keys[i];
    return (i == 0 || keys[i - 1] != k) && (i + 1 == e || keys[i + 1] != k);
}

// boundary out / in degree per vertex; counts[0] = boundary half-edges (one atomic per warp)
__global__ void __launch_bounds__(MB) degree_kernel(const unsigned long long* __restrict__ keys,
                                                    const int32_t* __restrict__ vals, int64_t e,
                                                    const int32_t* __restrict__ faces, int32_t* __restrict__ outdeg,
                                                    int32_t* __restrict__ indeg, unsigned long long* __restrict__ counts) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    const bool b = i < e && run_of_one(keys, e, i);
    if (b) {
        int u, v;
        half_edge(faces, vals[i], u, v);
        atomicAdd(&outdeg[u], 1);
        atomicAdd(&indeg[v], 1);
    }
    const unsigned n = __popc(__ballot_sync(0xffffffffu, b));
    if ((threadIdx.x & 31) == 0 && n) atomicAdd(&counts[0], (unsigned long long)n);
}

// succ and the face of each vertex's only outgoing boundary half-edge; the union of the half-edge's two ends
__global__ void __launch_bounds__(MB) link_kernel(const unsigned long long* __restrict__ keys,
                                                  const int32_t* __restrict__ vals, int64_t e,
                                                  const int32_t* __restrict__ faces, const int32_t* __restrict__ outdeg,
                                                  int32_t* __restrict__ succ, int32_t* __restrict__ bface,
                                                  int32_t* parent) {
    const int64_t i = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (i >= e || !run_of_one(keys, e, i)) return;
    const int c = vals[i];
    int u, v;
    half_edge(faces, c, u, v);
    if (outdeg[u] == 1) {
        succ[u] = v;
        bface[u] = c / 3;
    }
    unite(parent, u, v);
}

// labels[v] = -1 off the boundary; per label: the vertex count and the pinched flag
__global__ void __launch_bounds__(MB) set_kernel(const int32_t* __restrict__ outdeg, const int32_t* __restrict__ indeg,
                                                 int64_t m, int32_t* __restrict__ labels, int32_t* __restrict__ lengths,
                                                 int32_t* __restrict__ pinched) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    const int o = outdeg[v], n = indeg[v];
    if (o == 0 && n == 0) {
        labels[v] = -1;  // a singleton set: no other vertex reads its parent
        return;
    }
    const int r = labels[v];
    atomicAdd(&lengths[r], 1);
    if (o != 1 || n != 1) atomicOr(&pinched[r], 1);
}

// counts[1] = holes, counts[2] = pinched sets
__global__ void __launch_bounds__(MB) set_count_kernel(const int32_t* __restrict__ labels,
                                                       const int32_t* __restrict__ pinched, int64_t m,
                                                       unsigned long long* __restrict__ counts) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || labels[v] != v) return;
    atomicAdd(&counts[pinched[v] ? 2 : 1], 1ull);
}

// filled[v], the centre (nv) and face (nf) counts of each filled hole; counts[2..4] = filled, too long, lone triangles
__global__ void __launch_bounds__(MB) plan_kernel(const int32_t* __restrict__ labels, const int32_t* __restrict__ succ,
                                                  const int32_t* __restrict__ lengths,
                                                  const int32_t* __restrict__ pinched, const int32_t* __restrict__ bface,
                                                  int64_t m, int64_t H, uint8_t* __restrict__ filled,
                                                  int32_t* __restrict__ nv, int32_t* __restrict__ nf,
                                                  long long* __restrict__ counts) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m) return;
    int fl = 0, a = 0, b = 0;
    if (labels[v] == v && !pinched[v]) {
        const int L = lengths[v];
        if (L > H) {
            atomicAdd((unsigned long long*)&counts[3], 1ull);
        } else if (L == 3 && bface[succ[v]] == bface[v] && bface[succ[succ[v]]] == bface[v]) {
            atomicAdd((unsigned long long*)&counts[4], 1ull);
        } else {
            fl = 1;
            a = L >= 4;
            b = L == 3 ? 1 : L;
            atomicAdd((unsigned long long*)&counts[2], 1ull);
        }
    }
    filled[v] = (uint8_t)fl;
    nv[v] = a;
    nf[v] = b;
}

// One thread per filled hole: L = 3 adds (v0, v2, v1); L >= 4 adds (v(k+1), v(k), c) for k = 0..L-1 and the centre c:
// position = (sum in loop order) / L, colour = (2 sum + L) div 2L, density = (sum in loop order) / L.
__global__ void __launch_bounds__(MB) fill_kernel(const double* __restrict__ vpos, const uint8_t* __restrict__ vcol,
                                                  const double* __restrict__ dens, int64_t m, int64_t t,
                                                  const int32_t* __restrict__ succ, const int32_t* __restrict__ lengths,
                                                  const uint8_t* __restrict__ filled, const int32_t* __restrict__ vrank,
                                                  const int32_t* __restrict__ frank, double* __restrict__ vpos_o,
                                                  uint8_t* __restrict__ vcol_o, double* __restrict__ dens_o,
                                                  int32_t* __restrict__ faces_o) {
    const int64_t v = (int64_t)blockIdx.x * MB + threadIdx.x;
    if (v >= m || !filled[v]) return;
    const int L = lengths[v];
    const int64_t fo = t + frank[v];
    if (L == 3) {
        const int v1 = succ[v], v2 = v1 >= 0 ? succ[v1] : -1;
        if (v2 < 0) return;  // only a face that uses a vertex twice could break a loop
        faces_o[3 * fo] = (int32_t)v;
        faces_o[3 * fo + 1] = v2;
        faces_o[3 * fo + 2] = v1;
        return;
    }
    const int64_t c = m + vrank[v];
    double p[3] = {0.0, 0.0, 0.0}, d = 0.0;
    int col[3] = {0, 0, 0};
    int u = (int)v;
    for (int k = 0; k < L; ++k) {
        const int w = succ[u];
        if (w < 0) return;
        faces_o[3 * (fo + k)] = w;
        faces_o[3 * (fo + k) + 1] = u;
        faces_o[3 * (fo + k) + 2] = (int32_t)c;
        for (int a = 0; a < 3; ++a) p[a] = k ? __dadd_rn(p[a], vpos[3 * u + a]) : vpos[3 * u + a];
        if (dens) d = k ? __dadd_rn(d, dens[u]) : dens[u];
        if (vcol)
            for (int a = 0; a < 3; ++a) col[a] += vcol[3 * u + a];
        u = w;
    }
    for (int a = 0; a < 3; ++a) vpos_o[3 * c + a] = __ddiv_rn(p[a], (double)L);
    if (dens) dens_o[c] = __ddiv_rn(d, (double)L);
    if (vcol)
        for (int a = 0; a < 3; ++a) vcol_o[3 * c + a] = (uint8_t)((2 * col[a] + L) / (2 * L));
}

// find, plan and fill share this layout (plan reads find's degrees and faces, fill reads plan's ranks)
struct HolesWs {
    unsigned long long *keys_a, *keys_b;
    int32_t *vals_a, *vals_b, *outdeg, *indeg, *bface, *pinched, *nv, *nf, *vrank, *frank;
    void* tmp;
    size_t tmp_bytes, bytes;
};
HolesWs holes_ws(void* base, int64_t m, int64_t t) {
    size_t b[2] = {0, 0};
    cub::DeviceRadixSort::SortPairs(nullptr, b[0], (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (const int32_t*)nullptr, (int32_t*)nullptr, (int)(3 * t));
    cub::DeviceScan::ExclusiveSum(nullptr, b[1], (const int32_t*)nullptr, (int32_t*)nullptr, (int)m);
    WsCarve w{(char*)base};
    HolesWs l;
    l.keys_a = w.take<unsigned long long>(3 * t);
    l.keys_b = w.take<unsigned long long>(3 * t);
    l.vals_a = w.take<int32_t>(3 * t);
    l.vals_b = w.take<int32_t>(3 * t);
    l.outdeg = w.take<int32_t>(m);
    l.indeg = w.take<int32_t>(m);
    l.bface = w.take<int32_t>(m);
    l.pinched = w.take<int32_t>(m);
    l.nv = w.take<int32_t>(m);
    l.nf = w.take<int32_t>(m);
    l.vrank = w.take<int32_t>(m);
    l.frank = w.take<int32_t>(m);
    l.tmp_bytes = WsCarve::pad(b[0] > b[1] ? b[0] : b[1]);
    l.tmp = w.take<char>(l.tmp_bytes);
    l.bytes = w.used;
    return l;
}

bool sizes_ok(int64_t m, int64_t t) { return m > 0 && m < 0x7FFFFFFFll && t > 0 && 3 * t < 0x7FFFFFFFll; }

int bits_of(int64_t x) {
    int b = 0;
    while (x >> b) ++b;
    return b;
}

}  // namespace

// ---- C ABI -----------------------------------------------------------------------------------------------------------
extern "C" int64_t g2pc_mesh_holes_workspace_bytes(int64_t m, int64_t t) {
    return sizes_ok(m, t) ? (int64_t)holes_ws(nullptr, m, t).bytes : 0;
}

extern "C" int g2pc_mesh_holes_find(const int32_t* faces, int64_t m, int64_t t, int32_t* labels, int32_t* succ,
                                    int32_t* lengths, int64_t* counts, void* workspace, int64_t workspace_bytes,
                                    void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 1 <= t, 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(faces && labels && succ && lengths && counts && workspace, "null pointer");
    const HolesWs l = holes_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    const int64_t e = 3 * t;
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 3 * sizeof(int64_t), st));
    G2PC_CUDA(cudaMemsetAsync(succ, 0xFF, (size_t)m * 4, st));
    G2PC_CUDA(cudaMemsetAsync(lengths, 0, (size_t)m * 4, st));
    G2PC_CUDA(cudaMemsetAsync(l.outdeg, 0, (size_t)m * 4, st));
    G2PC_CUDA(cudaMemsetAsync(l.indeg, 0, (size_t)m * 4, st));
    G2PC_CUDA(cudaMemsetAsync(l.bface, 0xFF, (size_t)m * 4, st));
    G2PC_CUDA(cudaMemsetAsync(l.pinched, 0, (size_t)m * 4, st));
    edge_keys_kernel<<<grid_of(e), MB, 0, st>>>(faces, t, l.keys_a, l.vals_a);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    // the high word is < m and the low word < 2^31: bits from 32 + bits(m - 1) up are zero
    G2PC_CUDA(cub::DeviceRadixSort::SortPairs(l.tmp, b, l.keys_a, l.keys_b, l.vals_a, l.vals_b, (int)e, 0,
                                              32 + bits_of(m - 1), st));
    degree_kernel<<<grid_of(e), MB, 0, st>>>(l.keys_b, l.vals_b, e, faces, l.outdeg, l.indeg,
                                             (unsigned long long*)counts);
    G2PC_CHECK_LAUNCH();
    parent_init_kernel<<<grid_of(m), MB, 0, st>>>(labels, m);
    G2PC_CHECK_LAUNCH();
    link_kernel<<<grid_of(e), MB, 0, st>>>(l.keys_b, l.vals_b, e, faces, l.outdeg, succ, l.bface, labels);
    G2PC_CHECK_LAUNCH();
    compress_kernel<<<grid_of(m), MB, 0, st>>>(labels, m);
    G2PC_CHECK_LAUNCH();
    set_kernel<<<grid_of(m), MB, 0, st>>>(l.outdeg, l.indeg, m, labels, lengths, l.pinched);
    G2PC_CHECK_LAUNCH();
    set_count_kernel<<<grid_of(m), MB, 0, st>>>(labels, l.pinched, m, (unsigned long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_holes_plan(int64_t m, int64_t t, const int32_t* labels, const int32_t* succ,
                                    const int32_t* lengths, int64_t max_hole_edges, uint8_t* filled, int64_t* counts,
                                    void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 1 <= t, 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(max_hole_edges >= 3 && max_hole_edges <= 1024, "need 3 <= max_hole_edges <= 1024");
    G2PC_CHECK_ARG(labels && succ && lengths && filled && counts && workspace, "null pointer");
    const HolesWs l = holes_ws(workspace, m, t);
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemsetAsync(counts, 0, 5 * sizeof(int64_t), st));
    plan_kernel<<<grid_of(m), MB, 0, st>>>(labels, succ, lengths, l.pinched, l.bface, m, max_hole_edges, filled, l.nv,
                                           l.nf, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    size_t b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.nv, l.vrank, (int)m, st));
    b = l.tmp_bytes;
    G2PC_CUDA(cub::DeviceScan::ExclusiveSum(l.tmp, b, l.nf, l.frank, (int)m, st));
    trim_counts_kernel<<<1, 1, 0, st>>>(l.nv, l.vrank, m, l.nf, l.frank, m, (long long*)counts);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}

extern "C" int g2pc_mesh_holes_fill(const double* vpos, const uint8_t* vcolours, const double* density, int64_t m,
                                    const int32_t* faces, int64_t t, const int32_t* succ, const int32_t* lengths,
                                    const uint8_t* filled, int64_t added_vertices, int64_t added_faces,
                                    double* vpos_out, uint8_t* vcolours_out, double* density_out, int32_t* faces_out,
                                    const void* workspace, int64_t workspace_bytes, void* stream) {
    G2PC_CHECK_ARG(sizes_ok(m, t), "need 1..2^31-2 vertices and 1 <= t, 3 t < 2^31 - 1");
    G2PC_CHECK_ARG(added_vertices >= 0 && added_faces >= 0 && m + added_vertices < 0x7FFFFFFFll &&
                       3 * (t + added_faces) < 0x7FFFFFFFll,
                   "need m + added vertices < 2^31 - 1 and 3 (t + added faces) < 2^31 - 1");
    G2PC_CHECK_ARG(vpos && faces && succ && lengths && filled && vpos_out && faces_out && workspace, "null pointer");
    G2PC_CHECK_ARG(!vcolours == !vcolours_out && !density == !density_out, "colours and densities need an output");
    const HolesWs l = holes_ws(const_cast<void*>(workspace), m, t);  // read only here
    G2PC_CHECK_WORKSPACE(workspace, workspace_bytes, l.bytes, 256);
    cudaStream_t st = (cudaStream_t)stream;
    G2PC_CUDA(cudaMemcpyAsync(vpos_out, vpos, (size_t)m * 24, cudaMemcpyDeviceToDevice, st));
    if (vcolours) G2PC_CUDA(cudaMemcpyAsync(vcolours_out, vcolours, (size_t)m * 3, cudaMemcpyDeviceToDevice, st));
    if (density) G2PC_CUDA(cudaMemcpyAsync(density_out, density, (size_t)m * 8, cudaMemcpyDeviceToDevice, st));
    G2PC_CUDA(cudaMemcpyAsync(faces_out, faces, (size_t)t * 12, cudaMemcpyDeviceToDevice, st));
    fill_kernel<<<grid_of(m), MB, 0, st>>>(vpos, vcolours, density, m, t, succ, lengths, filled, l.vrank, l.frank,
                                           vpos_out, vcolours_out, density_out, faces_out);
    G2PC_CHECK_LAUNCH();
    return G2PC_OK;
}
