/*
 * g2pc.h — C ABI of libg2pc.so: H100-native (sm_90a) kernels for the 3DGS-to-PC hot path
 * (per-Gaussian point sampling + Mahalanobis cull, per-camera colour / visibility rasterisation).
 *
 * This is the drop-in boundary.  The reference has two native/op boundaries on this path:
 *   - pybind11 module `gaussian_pointcloud_rasterization._C`
 *       (gaussian-pointcloud-rasterization/ext.cpp:15-17, rasterize_points.cu:36-145, rasterize_points.h:18-46)
 *   - pure-torch call chains for the sampler
 *       (gauss_to_pc.py:140-275, gauss_handler.py:26-63)
 * Both are replaced by the plain-C entry points below.  Conventions (all entry points):
 *   - every pointer is a DEVICE pointer unless the name ends in `_host`; the caller owns all memory,
 *     including scratch (sizes come from the *_bytes query functions or are stated in the comment);
 *   - every call is asynchronous on `stream` (a cudaStream_t passed as void*); no allocation, no host
 *     synchronisation and no global mutable state inside the library, except the blend switches
 *     set by g2pc_blend_set_compact and g2pc_blend_set_cull;
 *   - return value: 0 = G2PC_OK, otherwise an error code; g2pc_last_error() gives a thread-local message;
 *   - no C++ exception crosses the ABI.
 */
#ifndef G2PC_H
#define G2PC_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define G2PC_OK 0
#define G2PC_ERR_INVALID 1   /* bad argument */
#define G2PC_ERR_CUDA 2      /* a CUDA runtime call / launch failed */
#define G2PC_ERR_WORKSPACE 3 /* caller-provided workspace too small or misaligned */

#define G2PC_F32 0
#define G2PC_F64 1

/* ---- misc ------------------------------------------------------------------------------------ */
int g2pc_version(void);
const char* g2pc_last_error(void);

/* ---- S1: covariance build ------------------------------------------------------------------- */
/* Replaces build_rotation / build_scaling_rotation / build_covariance_from_scaling_rotation
 * (gauss_handler.py:26-63): R(q) without re-normalisation, L = R*diag(exp(mod*s)), Sigma = L*L^T.
 * scales (n,3) log-space and rots (n,4) in `in_dtype` (the ply loader feeds f64, gauss_dataloader.py:66-80;
 * the elements of R and exp(s) are formed in the input precision and then rounded to f32, as the
 * reference's slice-assignments into float tensors do).  cov: (n,3,3) f32 row-major. */
int g2pc_cov_build(const void* scales, const void* rots, int in_dtype, float scale_modifier,
                   int64_t n, float* cov, void* stream);

/* Replaces Gaussians.calculate_normals (gauss_handler.py:89-106): column argmin(scale) of R(q).
 * normals: (n,3) f32. */
int g2pc_normals(const void* scales, const void* rots, int in_dtype, int64_t n, float* normals,
                 void* stream);

/* Replaces torch.linalg.eigvals(covariances).real on the N x 3 x 3 covariance batch
 * (gauss_handler.py:112 non_posdef_covariances, :259 get_gaussian_magnitudes): eigenvalues of the symmetric part,
 * closed form in f64, rounded to f32, ascending.  eigvals: (n,3) f32.  The callers keep the reference's
 * elementwise f32 chains (ellipsoid area, <= epsilon tests) in torch. */
int g2pc_eigvals_sym3(const float* cov, int64_t n, float* eigvals, void* stream);

/* ---- S2: sampling + Mahalanobis cull --------------------------------------------------------- */
/* Replaces sample_from_multivariate_normal + mahalanobis + create_new_gaussian_points +
 * the bin loop of generate_pointcloud (gauss_to_pc.py:92-103,140-371) and
 * torch.distributions.MultivariateNormal (Cholesky + loc + L*eps).
 *
 * Work is described by host-built tables (the reference builds the same bins on the host,
 * gauss_to_pc.py:308-343):
 *   tile  = <=256/lpg consecutive Gaussians (in bin order) of one bin, all drawing k samples per attempt
 *   unit  = one contiguous span of the output, in the reference's output order:
 *           the centre points of a bin, or the samples one tile emits in one attempt.            */
typedef struct {
    int32_t j0;    /* first Gaussian (bin-order index) */
    int32_t count; /* Gaussians in the tile (<= 256/lpg) */
    int32_t k;     /* samples drawn per Gaussian per attempt = bin's points-per-Gaussian - 1 */
    int32_t lpg;   /* threads cooperating on one Gaussian: power of two, 1..256 */
} g2pc_tile_t;

typedef struct {
    int32_t attempt; /* >=0: sample unit of that attempt; -1: centre-point unit */
    int32_t j0;      /* first Gaussian (bin-order index) */
    int32_t count;   /* Gaussians covered */
    int32_t k;       /* samples per Gaussian per attempt (0 for centre units) */
} g2pc_unit_t;

#define G2PC_CULL_EPS_NORM 0 /* accept iff |eps| <= std (exact-arithmetic identity of the reference test) */
#define G2PC_CULL_EXPLICIT 1 /* accept iff sqrt(d^T Sigma^-1 d) <= std, d = mu - x, fp32 (gauss_to_pc.py:92-103) */

/* status words written by g2pc_sample_count (int32 each) */
#define G2PC_ST_OVERFLOW 0  /* !=0: some Gaussian emitted in an attempt >= attempts_stored (re-run with more) */
#define G2PC_ST_CHOLFAIL 1  /* number of Gaussians whose covariance had no Cholesky factor even after +2e-6*I */
#define G2PC_ST_CHOLREG 2   /* number of Gaussians that needed +1e-6*I or +2e-6*I (gauss_to_pc.py:147-155) */
#define G2PC_ST_WORDS 4

/* Pass 1.  For every tile: gather the tile's Gaussians through `perm`, factor Sigma (closed-form
 * Cholesky), write one 64-byte record per Gaussian in bin order, then simulate the attempt loop of
 * create_new_gaussian_points: draw k samples per unfinished Gaussian with Philox4x32-10
 * (key = seed, counter = (gid, sample, attempt, call_id)) + Box-Muller, count the accepted ones,
 * m = min(k - added, count), and write the tile-local exclusive prefix of m
 * (xl[attempt*n + j]) and the tile total (tile_totals[tile*attempts_stored + attempt]).
 *   xyz (N,3) f32 · cov (N,3,3) f32 · colours (N,3) colour_dtype · normals (N,3) f32 or NULL
 *   perm (n,) int32: bin-order index -> row of the input arrays;  the RNG is keyed by the global Gaussian id
 *   gids[row] (uint32 per input row; survives culls and sharding) or, if gids is NULL, row + gid_offset
 *   records: n*64 bytes, 16-byte aligned · xl: attempts_stored*n uint32 · tile_totals: num_tiles*attempts_stored
 *   uint32, MUST be zero-filled by the caller · status: G2PC_ST_WORDS int32, zero-filled by the caller. */
int g2pc_sample_count(const float* xyz, const float* cov, const void* colours, int colour_dtype,
                      const float* normals, const int32_t* perm, const uint32_t* gids, int64_t gid_offset, int64_t n,
                      const g2pc_tile_t* tiles, int32_t num_tiles, int32_t num_attempts,
                      int32_t attempts_stored, float mahalanobis_std, int32_t cull_mode, uint64_t seed,
                      uint32_t call_id, void* records, uint32_t* xl, uint32_t* tile_totals,
                      int32_t* status, void* stream);

/* Pass 2.  Load-balanced expansion over OUTPUT points: point p belongs to unit u (unit_base[u] <= p <
 * unit_base[u+1], unit_base = exclusive prefix sum of the unit lengths, num_units+1 int64 entries, built by the
 * caller from tile_totals); inside a sample unit the Gaussian and sample index come from a search of xl;
 * eps is regenerated from the counter and x = mu + L*eps written ("first m samples of the block",
 * gauss_to_pc.py:247-258).  Outputs: out_xyz (capacity,3) f32; out_rgb / out_nrm (capacity,3) in out_dtype
 * (out_nrm may be NULL).  The launch covers `capacity` points in chunks of C = g2pc_sample_emit_chunk_points();
 * threads beyond unit_base[num_units] exit.  chunk_unit (optional, ceil(capacity/C)+1 int32): index of the unit holding
 * output point c*C (last u with unit_base[u] <= c*C, clamped to num_units - 1) — saves the per-CTA search. */
int g2pc_sample_emit_chunk_points(void); /* output points per CTA of g2pc_sample_emit (chunk size of chunk_unit) */
int g2pc_sample_emit(const void* records, const uint32_t* xl, int64_t n, const g2pc_unit_t* units,
                     const int64_t* unit_base, const int32_t* chunk_unit, int32_t num_units, uint64_t seed,
                     uint32_t call_id,
                     float* out_xyz, void* out_rgb, void* out_nrm, int out_dtype, int64_t capacity,
                     void* stream);

/* The standard-normal draws the sampler uses: eps[s, i, :] for sample s < k of Gaussian gids[i] in `attempt`
 * — the (k, n', 3) tensor torch's MultivariateNormal.rsample would have drawn (gauss_to_pc.py:149).
 * Used to inject the kernel's random stream into the reference/oracle for parity tests. */
int g2pc_dump_eps(const int64_t* gids, int64_t n_gids, int32_t k, int32_t attempt, uint64_t seed,
                  uint32_t call_id, float* eps, void* stream);

/* ---- N4 / N1: culls and point budget (s8_cull.cu) ----------------------------------------------------------------- */
/* Fused cull + compaction.  Replaces the mask chain of gauss_to_pc.py:483-496 and Gaussians.filter_gaussians
 * (gauss_handler.py:171-193: one boolean-index pass and one host sync per array).  keep(i) = lo <= i < hi
 * && max_contrib[i] > vis_threshold && opacity[i] > min_opacity && bbox_min < xyz[i] < bbox_max (open box)
 * && surface_dist[i] < *surface_threshold_dev && extra_mask[i]; every criterion whose array is NULL is skipped
 * (bbox_*_host: 3 host floats or NULL).  index: ascending row numbers of the kept Gaussians (capacity n int32);
 * count: one int64 in device memory.  workspace: g2pc_cull_workspace_bytes(n), 4-byte aligned. */
int64_t g2pc_cull_workspace_bytes(int64_t n);
int g2pc_cull_select(const float* max_contrib, float vis_threshold, const float* opacity, float min_opacity,
                     const float* xyz, const float* bbox_min3_host, const float* bbox_max3_host,
                     const float* surface_dist, const float* surface_threshold_dev, const uint8_t* extra_mask,
                     int64_t lo, int64_t hi, int64_t n, int32_t* index, int64_t* count, void* workspace,
                     int64_t workspace_bytes, void* stream);
/* dsts[a][r, :] = srcs[a][index[r], :] for r < m, rows of row_bytes[a] bytes (multiples of 4); srcs / dsts / row_bytes
 * are HOST arrays of num_arrays entries (device pointers inside). */
int g2pc_gather_rows(const int32_t* index, int64_t m, int32_t num_arrays, const void* const* srcs, void* const* dsts,
                     const int32_t* row_bytes, void* stream);

/* Magnitudes and point budget without a host round trip: magnitudes[i] (float64) = sqrt(ellipsoid area of Sigma_i,
 * p = 1.6075) * contrib[i] (gauss_handler.py:252-279, float32 chain, closed-form eigenvalues), ppg[i] (int32) =
 * round-half-even(magnitude * num_points / sum) with the first min(deficit, #zeros) zero entries raised to 1
 * (gauss_to_pc.py:73-90; the sum is reduced in a fixed order: bit-identical re-runs).  workspace:
 * g2pc_ppg_workspace_bytes(n), 8-byte aligned. */
int64_t g2pc_ppg_workspace_bytes(int64_t n);
int g2pc_points_per_gaussian(const float* cov, const float* contrib, int64_t n, double num_points, double* magnitudes,
                             int32_t* ppg, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- N5: statistical outlier removal of the point cloud (s9_clean.cu, --clean_pointcloud) ------------------------ */
/* Replaces Open3D's PointCloud::remove_statistical_outlier(nb_neighbors=20, std_ratio) behind the reference's
 * mesh_handler.clean_point_cloud (mesh_handler.py:89-94, called at gauss_to_pc.py:743-759).  Compact the cloud with
 * keep as the extra_mask of g2pc_cull_select, then g2pc_gather_rows. */
#define G2PC_SOR_K_MAX 32 /* largest nb_neighbors */

/* avg (n float64) = mean of the sqrt of the k' = min(k, n) smallest squared distances of every point to the cloud (the
 * point itself included, d2 = (dx*dx + dy*dy) + dz*dz in float64 of the float32 coordinates, summed in ascending order):
 * exact, not approximate.  xyz (n,3) f32; 1 <= k <= G2PC_SOR_K_MAX.  status: one int32, set to the number of points with a
 * non-finite coordinate (their avg is NaN and they are nobody's neighbour).  workspace: g2pc_knn_workspace_bytes(n),
 * 256-byte aligned. */
int64_t g2pc_knn_workspace_bytes(int64_t n);
int g2pc_knn_mean_dist(const float* xyz, int64_t n, int32_t k, double* avg, int32_t* status, void* workspace,
                       int64_t workspace_bytes, void* stream);
/* The neighbour lists of a cloud, for the normal orientation (N7).  ids (n,k int32), d2 (n,k float64, or NULL): the k' =
 * min(k, n - 1) nearest OTHER points of every row by ascending (d2, id) (d2 as for g2pc_knn_mean_dist, ties of d2 to the
 * smaller row id; exact), in slots 0..k'-1; slots k'..k-1 hold id -1 and d2 +inf.  A row with a non-finite coordinate
 * gets id -1 and d2 NaN everywhere and is nobody's neighbour; status counts such rows.  1 <= k <= G2PC_ORIENT_K_MAX.
 * workspace: g2pc_knn_workspace_bytes(n), 256-byte aligned. */
#define G2PC_ORIENT_K_MAX 31 /* largest k of g2pc_knn_ids: k + the point itself fit the 32-entry list of N5 */
int g2pc_knn_ids(const float* xyz, int64_t n, int32_t k, int32_t* ids, double* d2, int32_t* status, void* workspace,
                 int64_t workspace_bytes, void* stream);
/* stats (3 float64): mean = (sum of avg over avg > 0) / n, std = sqrt((sum of (avg - mean)^2 over avg > 0) / (n - 1)),
 * threshold = mean + std_ratio * std, each sum reduced in a fixed order (bit-identical re-runs); keep (n uint8) =
 * avg > 0 && avg < threshold.  std_ratio > 0.  workspace: g2pc_sor_workspace_bytes(n), 8-byte aligned.  n == 0 writes
 * nothing. */
int64_t g2pc_sor_workspace_bytes(int64_t n);
int g2pc_sor_mask(const double* avg, int64_t n, double std_ratio, uint8_t* keep, double* stats, void* workspace,
                  int64_t workspace_bytes, void* stream);

/* ---- N6: Poisson mesh of an oriented point cloud (s10_mesh.cu, g2pc/mesh.py, mesh_pc.py) ------------------------- */
/* Replaces Open3D's create_from_point_cloud_poisson + density trim + filter_smooth_laplacian behind the reference's
 * mesh_handler.generate_mesh (mesh_handler.py:23-40), with this project's own rules (DESIGN.md §2).  Order of calls:
 * splat -> vcycle (until the residual is small enough) -> iso -> extract_count -> extract_emit -> gather -> trim -> smooth
 * -> normals.  Grid: R = 2^depth nodes per axis, 2 <= depth <= G2PC_MESH_DEPTH_MAX; node index (k*R + j)*R + i. */
#define G2PC_MESH_DEPTH_MAX 10
#define G2PC_MESH_FRAME_WORDS 8 /* float64: origin x y z, h, L, mean of B, largest extent, R */

/* frame (G2PC_MESH_FRAME_WORDS float64): L = 1.1 x the largest extent of the finite points, origin = bounding-box
 * centre - L/2, h = L/R (h = 0: zero extent, nothing is splatted).  B (R^3 int64, zeroed here): every point with a
 * usable normal adds llrint(w * n_a / |n| * 2^32) at node - e_a and subtracts it at node + e_a for the 8 trilinear
 * weights w of its dual cell and the 3 axes a (exact integer atomics).  cell (n uint32): linear index of the point's
 * dual cell in the (R-1)^3 lattice, 0x7FFFFFFF when it was not splatted.  status (2 int32): points skipped for a zero or
 * non-finite normal, points with a non-finite coordinate.  normals (n,3) in normal_dtype (G2PC_F32 / G2PC_F64).
 * workspace: g2pc_mesh_splat_workspace_bytes(n), 256-byte aligned. */
int64_t g2pc_mesh_splat_workspace_bytes(int64_t n);
int g2pc_mesh_splat(const float* xyz, const void* normals, int normal_dtype, int64_t n, int32_t depth, double* frame,
                    int64_t* B, uint32_t* cell, int32_t* status, void* workspace, int64_t workspace_bytes, void* stream);

/* One multigrid V-cycle of (sum of the 6 neighbours - 6 chi) = b with mirrored ghosts (homogeneous Neumann),
 * b = (B - mean B) * h * 2^-33 read from B: red-black Gauss-Seidel (2 + 2 sweeps), fused residual + 8-cell restriction,
 * trilinear prolongation, 4^3 coarsest level.  chi: R^3 float32; first != 0 zeroes chi and writes norms[1] = |b|^2; every
 * call writes norms[0] = |r|^2 after the cycle (fixed-order float64 sums).  workspace:
 * g2pc_mesh_solve_workspace_bytes(depth), 256-byte aligned (the coarse levels). */
int64_t g2pc_mesh_solve_workspace_bytes(int32_t depth);
int g2pc_mesh_vcycle(const int64_t* B, const double* frame, int32_t depth, float* chi, int32_t first, double* norms,
                     void* workspace, int64_t workspace_bytes, void* stream);

/* Subtracts the mean of chi from chi, then iso (3 float64): iso[0] = that mean, iso[1] = mean over the splatted points
 * of the trilinear chi at the point (the splat's weights), iso[2] = their count.  Fixed-order float64 sums.
 * workspace: g2pc_mesh_iso_workspace_bytes(), 8-byte aligned. */
int64_t g2pc_mesh_iso_workspace_bytes(void);
int g2pc_mesh_iso(const float* xyz, const uint32_t* cell, int64_t n, const double* frame, int32_t depth, float* chi,
                  double* iso, void* workspace, int64_t workspace_bytes, void* stream);

/* Marching tetrahedra over the (R-1)^3 cubes of the node lattice, 6 Kuhn tetrahedra per cube; a node is inside iff
 * chi < iso[1].  extract_count writes counts (2 int64) = vertices m, triangles t; extract_emit (same workspace, after
 * extract_count) writes vkey (m int64, node*8 + d for the crossed edge (node, node + d), d = 1..7 bit 0 = x, ascending),
 * vt (m float64, t = (iso - chi_a) / (chi_b - chi_a)), vpos (m,3 float64), faces (t,3 int32, ascending (cube, tetrahedron,
 * triangle), counter-clockwise seen from chi > iso).  node_scratch: 5 bytes per node (B's memory may be reused).
 * workspace: g2pc_mesh_extract_workspace_bytes(depth), 256-byte aligned. */
int64_t g2pc_mesh_extract_workspace_bytes(int32_t depth);
int g2pc_mesh_extract_count(const float* chi, int32_t depth, const double* iso, int64_t* counts, void* workspace,
                            int64_t workspace_bytes, void* stream);
int g2pc_mesh_extract_emit(const float* chi, int32_t depth, const double* frame, const double* iso, void* node_scratch,
                           int64_t node_scratch_bytes, const void* workspace, int64_t workspace_bytes, int64_t* vkey,
                           double* vt, double* vpos, int32_t* faces, void* stream);

/* Per vertex: density = (1-t) W_a + t W_b and colour = floor(((1-t) C_a + t C_b) / density + 0.5) clamped to 0..255
 * (0 where density is 0), W / C = sums of w / w * colour over the points of the 8 dual cells around the node (cells in
 * ascending index, points in ascending input index, sequential float64).  colours (n,3 int32) and vcolours (m,3 uint8)
 * may both be NULL.  cell_scratch: 4 bytes per dual cell.  workspace: g2pc_mesh_gather_workspace_bytes(n), 256-byte
 * aligned. */
int64_t g2pc_mesh_gather_workspace_bytes(int64_t n);
int g2pc_mesh_gather(const float* xyz, const int32_t* colours, const uint32_t* cell, int64_t n, const double* frame,
                     int32_t depth, const int64_t* vkey, const double* vt, int64_t m, void* cell_scratch,
                     int64_t cell_scratch_bytes, double* density, uint8_t* vcolours, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* threshold = numpy's linear 10 % quantile of the densities; keep (m uint8) = !(density < threshold); triangles with a
 * removed vertex are dropped and the kept vertices re-indexed in order.  Outputs (capacity m / t) are compacted: counts
 * (2 int64) = kept vertices, kept triangles.  workspace: g2pc_mesh_trim_workspace_bytes(m, t), 256-byte aligned. */
int64_t g2pc_mesh_trim_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_trim(const double* density, const double* vpos, const uint8_t* vcolours, int64_t m, const int32_t* faces,
                   int64_t t, uint8_t* keep, double* threshold, int64_t* counts, double* density_out, double* vpos_out,
                   uint8_t* vcolours_out, int32_t* faces_out, void* workspace, int64_t workspace_bytes, void* stream);

/* `iterations` Jacobi steps v += (sum w_j v_j / sum w_j - v) / 2, w_j = 1 / (|v - v_j| + 1e-12) over the distinct one-ring
 * neighbours in ascending index (float64; a vertex without neighbours stays).  vpos (m,3 float64) in place.
 * workspace: g2pc_mesh_smooth_workspace_bytes(m, t), 256-byte aligned. */
int64_t g2pc_mesh_smooth_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_smooth(double* vpos, int64_t m, const int32_t* faces, int64_t t, int32_t iterations, void* workspace,
                     int64_t workspace_bytes, void* stream);

/* vertices (m,3 float32) = vpos rounded; normals (m,3 float32) = normalised sum of cross(p1 - p0, p2 - p0) over the
 * incident triangles in ascending order (float64; zero stays zero).  workspace: g2pc_mesh_normals_workspace_bytes(m, t),
 * 256-byte aligned. */
int64_t g2pc_mesh_normals_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_normals(const double* vpos, int64_t m, const int32_t* faces, int64_t t, float* vertices, float* normals,
                      void* workspace, int64_t workspace_bytes, void* stream);

/* ---- N6b: narrow-band levels of the Poisson mesh (s12_mesh_band.cu, g2pc/mesh.py band_depth) ------------------- */
/* One or two levels D = depth + 1 .. G2PC_MESH_BAND_DEPTH_MAX above the dense solve, stored only in bricks of
 * G2PC_MESH_BRICK^3 nodes within G2PC_MESH_BAND_MARGIN bricks of the points (rules in DESIGN.md §2, N6b).  Level D:
 * R = 2^D, NB = R / 8 bricks per axis, brick map (NB^3 int32: slot or -1; slots in ascending linear brick index), brick
 * list (slot -> brick), node storage slot * 512 + (lz * 8 + ly) * 8 + lx.  parent_map / parent_chi: the level below
 * (parent_map NULL: the dense level, chi mean-free after g2pc_mesh_iso).  Order of calls per level: bricks (host reads
 * counts) -> list -> splat -> ghosts -> cg_start, then cg_step 1, 2, ... (one host read of scalars per call); at the
 * finest level: iso -> extract_count -> extract_emit -> gather, then g2pc_mesh_trim / _smooth / _normals. */
#define G2PC_MESH_BAND_DEPTH_MAX 12
#define G2PC_MESH_BRICK 8
#define G2PC_MESH_BAND_MARGIN 1
#define G2PC_MESH_CG_WORDS 5 /* float64: |c|^2, p.q, |r|^2, r.z (two slots) */

/* band_frame (G2PC_MESH_FRAME_WORDS): the dense frame with h = L / R and R of level D.  map: NB^3 int32.  counts
 * (2 int64): active bricks, seed bricks lost to the nesting rule (must be 0).  cell: the dense splat's cell (its
 * CELL_NONE marks the points that are not splatted).  workspace: g2pc_mesh_band_bricks_workspace_bytes(depth). */
int64_t g2pc_mesh_band_bricks_workspace_bytes(int32_t depth);
int g2pc_mesh_band_bricks(const float* xyz, const uint32_t* cell, int64_t n, const double* frame, int32_t depth,
                          const int32_t* parent_map, double* band_frame, int32_t* map, int64_t* counts, void* workspace,
                          int64_t workspace_bytes, void* stream);
/* list: counts[0] int32, slot -> linear brick index. */
int g2pc_mesh_band_list(const int32_t* map, int32_t depth, int32_t* list, void* stream);
/* B (nbricks * 512 int64, zeroed here): the dense splat's terms at level D on band storage.  status (1 int32): terms
 * whose node is not in the band (0 when the nesting rule held). */
int g2pc_mesh_band_splat(const float* xyz, const void* normals, int normal_dtype, const uint32_t* cell, int64_t n,
                         const double* band_frame, int32_t depth, const int32_t* map, int64_t nbricks, int64_t* B,
                         int32_t* status, void* stream);
/* Per band node: ghost (float64, may be NULL) = sum of s P(parent chi) over the in-grid neighbours outside the band,
 * chi = s P(parent chi) (the initial guess), rhs = (float)(ghost - B h 2^-33), s = 1/8. */
int g2pc_mesh_band_ghosts(const float* parent_chi, const int32_t* parent_map, int32_t depth, const int32_t* map,
                          const int32_t* list, int64_t nbricks, const int64_t* B, const double* band_frame,
                          double* ghost, float* chi, float* rhs, void* stream);
/* Jacobi-preconditioned conjugate gradients on (count x chi - sum of the active in-grid neighbours) = rhs.  cg_start
 * (re)starts from chi (residual from chi, direction = preconditioned residual); cg_step with iteration t = 1, 2, ...
 * (counted from the last start) does one step.  scalars (G2PC_MESH_CG_WORDS float64): [0] |rhs|^2, [2] |r|^2 after
 * either call.  workspace: g2pc_mesh_band_cg_workspace_bytes(nbricks), kept between the calls. */
int64_t g2pc_mesh_band_cg_workspace_bytes(int64_t nbricks);
int g2pc_mesh_band_cg_start(const float* rhs, int32_t depth, const int32_t* map, const int32_t* list, int64_t nbricks,
                            float* chi, double* scalars, void* workspace, int64_t workspace_bytes, void* stream);
int g2pc_mesh_band_cg_step(const float* rhs, int32_t depth, const int32_t* map, const int32_t* list, int64_t nbricks,
                           float* chi, int32_t iteration, double* scalars, void* workspace, int64_t workspace_bytes,
                           void* stream);
/* iso (3 float64): 0, mean of trilinear chi over the splatted points, their count.  workspace:
 * g2pc_mesh_band_iso_workspace_bytes(). */
int64_t g2pc_mesh_band_iso_workspace_bytes(void);
int g2pc_mesh_band_iso(const float* xyz, const uint32_t* cell, int64_t n, const double* band_frame, int32_t depth,
                       const int32_t* map, const float* chi, double* iso, void* workspace, int64_t workspace_bytes,
                       void* stream);
/* Marching tetrahedra over the cubes whose 8 corners are in the band; keys node * 8 + d (global node, int64); vertices
 * in ascending (storage index, d), triangles in ascending (storage index of the cube, tetrahedron, triangle).
 * node_scratch: 5 bytes per band node.  workspace: g2pc_mesh_band_extract_workspace_bytes(nbricks). */
int64_t g2pc_mesh_band_extract_workspace_bytes(int64_t nbricks);
int g2pc_mesh_band_extract_count(const float* chi, int32_t depth, const int32_t* map, const int32_t* list,
                                 int64_t nbricks, const double* iso, int64_t* counts, void* workspace,
                                 int64_t workspace_bytes, void* stream);
int g2pc_mesh_band_extract_emit(const float* chi, int32_t depth, const int32_t* map, const int32_t* list,
                                int64_t nbricks, const double* band_frame, const double* iso, void* node_scratch,
                                int64_t node_scratch_bytes, const void* workspace, int64_t workspace_bytes,
                                int64_t* vkey, double* vt, double* vpos, int32_t* faces, void* stream);
/* g2pc_mesh_gather at level D with int64 dual cells (no dense cell table).  workspace:
 * g2pc_mesh_band_gather_workspace_bytes(n). */
int64_t g2pc_mesh_band_gather_workspace_bytes(int64_t n);
int g2pc_mesh_band_gather(const float* xyz, const int32_t* colours, const uint32_t* cell, int64_t n,
                          const double* band_frame, int32_t depth, const int64_t* vkey, const double* vt, int64_t m,
                          double* density, uint8_t* vcolours, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- N9: decimation by parallel quadric edge collapse (s13_decimate.cu, g2pc/mesh.py decimate) ----------------- */
/* Rules in DESIGN.md §2, N9.  vpos (m,3 float64), faces (t,3 int32, no face uses a vertex twice).  Order of calls:
 * prepare once, then per round select (host reads counts) -> apply into a second face buffer, until the target is
 * reached or no edge is selected; then finish.  quadrics: m x 10 float64 (A00 A01 A02 A11 A12 A22 b0 b1 b2 c). */
/* quadrics: the area-weighted plane quadrics summed over each vertex's faces in ascending id; free_flags (m uint8): 1 iff
 * the vertex has 1..128 faces, every edge at it is used by exactly two of them and they form one closed fan.
 * workspace: g2pc_mesh_decimate_prepare_workspace_bytes(m, t). */
int64_t g2pc_mesh_decimate_prepare_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_decimate_prepare(const double* vpos, int64_t m, const int32_t* faces, int64_t t, double* quadrics,
                               uint8_t* free_flags, void* workspace, int64_t workspace_bytes, void* stream);
/* Candidate edges and the 2-ring minimum selection.  counts (3 int64): unique edges, candidates, selected edges.  The
 * workspace (g2pc_mesh_decimate_round_workspace_bytes(m, t)) carries the selection to the apply call of the same round
 * with the same m and t. */
int64_t g2pc_mesh_decimate_round_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_decimate_select(const double* vpos, int64_t m, const int32_t* faces, int64_t t, const double* quadrics,
                              const uint8_t* free_flags, int64_t* counts, void* workspace, int64_t workspace_bytes,
                              void* stream);
/* Collapses the k (<= selected = counts[2] of the select call) selected edges with the smallest keys: vpos, quadrics,
 * colour_sums (m,3 int64, may be NULL), merged (m int32), density_sums (m float64, may be NULL) and alive (m uint8) in
 * place; faces_out (t - 2k, 3) = the surviving faces remapped, in their order; kept (1 int64) = their count.  applied
 * (k uint64 keys, ascending) and applied_ab (k x 2 int32: survivor a, removed b) may be NULL. */
int g2pc_mesh_decimate_apply(double* vpos, int64_t m, const int32_t* faces, int64_t t, double* quadrics,
                             int64_t* colour_sums, int32_t* merged, double* density_sums, uint8_t* alive,
                             int64_t selected, int64_t k, int32_t* faces_out, int64_t* kept, uint64_t* applied,
                             int32_t* applied_ab, void* workspace, int64_t workspace_bytes, void* stream);
/* The alive vertices in their order: vpos_out, colours_out = floor(sum / merged + 1/2) (NULL with colour_sums),
 * densities_out = sum / merged (NULL with density_sums); faces_out = faces renumbered; counts (1 int64) = alive vertices.
 * workspace: g2pc_mesh_decimate_finish_workspace_bytes(m). */
int64_t g2pc_mesh_decimate_finish_workspace_bytes(int64_t m);
int g2pc_mesh_decimate_finish(const double* vpos, int64_t m, const int32_t* faces, int64_t t, const uint8_t* alive,
                              const int64_t* colour_sums, const int32_t* merged, const double* density_sums,
                              double* vpos_out, uint8_t* colours_out, double* densities_out, int32_t* faces_out,
                              int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream);

/* ---- N11: connected-component filter of a triangle mesh (s15_components.cu, g2pc/mesh.py remove_components) ------ */
/* Rules in DESIGN.md §2, N11.  m vertices (1..2^31-2), faces (t,3 int32, 3 t < 2^31 - 1, indices in 0..m-1; a face may
 * use a vertex twice).  Order of calls: label (host reads counts[0]) -> select (host reads counts) -> compact into
 * buffers of the kept sizes. */
/* Two vertices are connected when a face uses both.  labels (m int32) = the smallest vertex of each vertex's component;
 * sizes (m int32, indexed by label) = triangles per component (0 for an unused vertex); counts (2 int64): components
 * with at least one triangle, the largest size. */
int g2pc_mesh_components_label(const int32_t* faces, int64_t m, int64_t t, int32_t* labels, int32_t* sizes,
                               int64_t* counts, void* stream);
/* keep (m uint8) = 1 iff the vertex's component has size >= max(1, min_triangles) and, when 0 < keep_largest <
 * components (counts[0] of the label call), rank < keep_largest in (size descending, label ascending).  0 turns a
 * parameter off.  counts (3 int64): kept vertices, kept triangles, kept components.  The workspace
 * (g2pc_mesh_components_select_workspace_bytes(m, t)) carries the selection to the compact call with the same m, t. */
int64_t g2pc_mesh_components_select_workspace_bytes(int64_t m, int64_t t);
int g2pc_mesh_components_select(const int32_t* faces, int64_t m, int64_t t, const int32_t* labels, const int32_t* sizes,
                                int64_t components, int64_t min_triangles, int64_t keep_largest, uint8_t* keep,
                                int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream);
/* The kept vertices (vpos (m,3 float64), vcolours (m,3 uint8, may be NULL), density (m float64)) and faces (renumbered)
 * in their order into the *_out buffers, which hold the kept counts of the select call. */
int g2pc_mesh_components_compact(const double* vpos, const uint8_t* vcolours, const double* density, int64_t m,
                                 const int32_t* faces, int64_t t, const uint8_t* keep, double* vpos_out,
                                 uint8_t* vcolours_out, double* density_out, int32_t* faces_out, const void* workspace,
                                 int64_t workspace_bytes, void* stream);

/* ---- N12: closing small holes of a triangle mesh (s16_holes.cu, g2pc/mesh.py fill_holes) ------------------------- */
/* Rules in DESIGN.md §2, N12.  m vertices (1..2^31-2), faces (t,3 int32, 1 <= t, 3 t < 2^31 - 1, indices in 0..m-1, no
 * face uses a vertex twice).  Order of calls, all with one workspace (g2pc_mesh_holes_workspace_bytes(m, t)) and the
 * same m, t: find (host reads counts) -> plan (host reads counts) -> fill into buffers of m + added vertices and
 * t + added faces. */
int64_t g2pc_mesh_holes_workspace_bytes(int64_t m, int64_t t);
/* A half-edge is on the boundary when its undirected edge is used by exactly one face.  labels (m int32) = the smallest
 * vertex of each vertex's boundary set, -1 off the boundary; succ (m int32) = the target of the vertex's boundary
 * half-edge where it has exactly one, else -1; lengths (m int32, indexed by label) = vertices per set, 0 at an index
 * that is no label.  counts (3 int64): boundary half-edges, holes, pinched sets. */
int g2pc_mesh_holes_find(const int32_t* faces, int64_t m, int64_t t, int32_t* labels, int32_t* succ, int32_t* lengths,
                         int64_t* counts, void* workspace, int64_t workspace_bytes, void* stream);
/* filled (m uint8, indexed by label) = 1 iff the set is a hole of length <= max_hole_edges (3..1024) that is not a lone
 * triangle.  counts (5 int64): added vertices, added faces, filled, too long, lone triangles. */
int g2pc_mesh_holes_plan(int64_t m, int64_t t, const int32_t* labels, const int32_t* succ, const int32_t* lengths,
                         int64_t max_hole_edges, uint8_t* filled, int64_t* counts, void* workspace,
                         int64_t workspace_bytes, void* stream);
/* The input mesh (vcolours and density may be NULL, each with its output) copied into the *_out buffers, then the
 * centres from index m and the added faces from index t, in ascending label order.  added_* are plan's counts. */
int g2pc_mesh_holes_fill(const double* vpos, const uint8_t* vcolours, const double* density, int64_t m,
                         const int32_t* faces, int64_t t, const int32_t* succ, const int32_t* lengths,
                         const uint8_t* filled, int64_t added_vertices, int64_t added_faces, double* vpos_out,
                         uint8_t* vcolours_out, double* density_out, int32_t* faces_out, const void* workspace,
                         int64_t workspace_bytes, void* stream);

/* ---- N7: consistent orientation of point-cloud normals (s11_orient.cu, g2pc/orient.py) -------------------------- */
/* Hoppe et al. 1992 (the rule behind Open3D's orient_normals_consistent_tangent_plane) with this project's own rules
 * (DESIGN.md §2): k-NN graph, edge weight 1 - |n_i . n_j|, minimum spanning forest, sign propagated from one seed per
 * tree (its largest z) so that the seed's normal points to +z.  Order of calls: g2pc_orient_prepare, g2pc_knn_ids on the
 * m usable points, g2pc_orient_edges, g2pc_orient_round for round = 0, 1, ... until a round hooks nothing (one host read
 * of its counts per round), g2pc_orient_finish. */

/* The usable rows (finite coordinate; finite, non-zero float64 normal length), ascending: rows[0..m), their points
 * uxyz (m,3 float32) and unit normals unh (m,3 float64, n / sqrt((nx*nx + ny*ny) + nz*nz) without FMA).  Every buffer has
 * room for n rows; count (one int64) = m.  workspace: g2pc_orient_prepare_workspace_bytes(n), 256-byte aligned. */
int64_t g2pc_orient_prepare_workspace_bytes(int64_t n);
int g2pc_orient_prepare(const float* xyz, const void* normals, int normal_dtype, int64_t n, int32_t* rows, float* uxyz,
                        double* unh, int64_t* count, void* workspace, int64_t workspace_bytes, void* stream);

/* The undirected edges of the k-NN graph of g2pc_knn_ids(uxyz, m, k): edges (E uint64, min << 32 | max) ascending and
 * unique; keys (c uint64): keys[e] = (float32 bits of max(0, 1 - |dot|)) << 32 | e for e < E, UINT64_MAX after;
 * flips (E uint8) = dot < 0, dot = (ax*bx + ay*by) + az*bz of the unit normals in float64 without FMA.  Capacity of
 * every buffer: c = m * min(k, m - 1) entries (below 2^32).  count (one int64) = E.  workspace:
 * g2pc_orient_edges_workspace_bytes(m, k), 256-byte aligned. */
int64_t g2pc_orient_edges_workspace_bytes(int64_t m, int32_t k);
int g2pc_orient_edges(const int32_t* ids, int64_t m, int32_t k, const double* unh, uint64_t* edges, uint64_t* keys,
                      uint8_t* flips, int64_t* count, void* workspace, int64_t workspace_bytes, void* stream);

/* One Borůvka round over the keys: every component hooks along its smallest outgoing key (in a mutual pair the smaller
 * representative stays the root) and mst[e] = 1 for each edge used.  comp (m int32): representative of each point;
 * rel (m uint8): XOR of the flip bits along the tree path to it.  Round 0 initialises comp, rel and mst (c bytes) and
 * needs active = c; later rounds take active = counts[1] of the round before.  counts (2 int64) = components hooked,
 * active edges left.  The workspace carries the active edges from round to round: the same buffer for every round,
 * g2pc_orient_round_workspace_bytes(m, c), 256-byte aligned. */
int64_t g2pc_orient_round_workspace_bytes(int64_t m, int64_t c);
int g2pc_orient_round(const uint64_t* edges, const uint64_t* keys, const uint8_t* flips, int64_t m, int64_t c,
                      int32_t round_index, int64_t active, int32_t* comp, uint8_t* rel, uint8_t* mst, int64_t* counts,
                      void* workspace, int64_t workspace_bytes, void* stream);

/* out (n,3, the normals' dtype) = normals, with the rows rows[v] of every flipped point v negated: flip(v) = rel(v) ^
 * rel(s) ^ (unh[s].z < 0), s = the seed of v's component (largest z of uxyz, then smallest index).  seed (m int32) and
 * seed_rel (m uint8, rel(v) ^ rel(s)) may be NULL.  stats (2 int64) = components, flipped points.  workspace:
 * g2pc_orient_finish_workspace_bytes(m), 256-byte aligned. */
int64_t g2pc_orient_finish_workspace_bytes(int64_t m);
int g2pc_orient_finish(const float* uxyz, const double* unh, const int32_t* rows, int64_t m, const void* normals,
                       int normal_dtype, int64_t n, const int32_t* comp, const uint8_t* rel, void* out, int32_t* seed,
                       uint8_t* seed_rel, int64_t* stats, void* workspace, int64_t workspace_bytes, void* stream);

/* Normals turned toward the camera that saw each Gaussian (gauss_to_mesh.py; rules in DESIGN.md §2).  means (m,3
 * float32), normals (m,3 float32 or float64, normal_dtype), ids (m int32): the original Gaussian row of each row;
 * cam_of (n int32): the colour stage's first_frame, INT32_MAX = never raised a maximum; cams (ncam,3 float32): camera
 * centres in camera-index order.  Row r with f = cam_of[ids[r]]: invalid when ids[r] is outside [0, n) or f is outside
 * [0, ncam) and not INT32_MAX; unseen when f == INT32_MAX; otherwise dot = (nx*dx + ny*dy) + nz*dz, d = cams[f] - means[r],
 * in float64 of the stored values without FMA.  out (m,3, the normals' dtype) = the row negated when dot < 0 (flipped),
 * the row unchanged otherwise (dot == 0 or NaN: undecided).  counts (4 int64) = flipped, unseen, undecided, invalid.
 * The normals are not modified.  m = 0 launches nothing and writes nothing. */
int g2pc_face_cameras(const float* means, const void* normals, int normal_dtype, const int32_t* ids, int64_t m,
                      const int32_t* cam_of, int64_t n, const float* cams, int64_t ncam, void* out, int64_t* counts,
                      void* stream);

/* ---- S3-S6: colour stage, renderer_type=python semantics (gauss_render.py:101-465) ------------------------------ */
/* Replaces GaussPythonRenderer.__call__/render (gauss_render.py:266-465) and — as the native op boundary — the role
 * of _C.rasterize_gaussians (rasterize_points.cu:36-145) in the per-camera loop of gauss_to_pc.py:437-454.
 * One camera (a "frame") = preprocess -> depth_sort -> build_tree -> multisplit -> blend -> accumulate
 * (-> compose_image).  No call waits for the device: every size the later stages need is read from the device-side
 * frame header; a frame that does not fit the caller's buffers poisons the header (see G2PC_HDR_POISON). */
typedef struct {
    float view[16];  /* world_view_transform, row-vector convention p_view = [p,1] * V (camera_handler.py:46), row-major */
    float proj[16];  /* projection_matrix as stored by Camera (already transposed, camera_handler.py:48), row-major */
    float campos[3]; /* camera centre (SH view directions) */
    float tan_fovx, tan_fovy, focal_x, focal_y;
    int32_t width, height;
} g2pc_camera_t;

typedef struct {
    int32_t r0, c0, w, h;    /* first row / column and size of the leaf tile in pixels */
    int32_t inst_begin;      /* offset of the leaf's list in inst_gid */
    int32_t inst_count;      /* Gaussians whose rect overlaps the leaf */
    int32_t pix_offset;      /* offset of the leaf's pixels in the concatenated leaf-colour buffer */
    int32_t node;            /* index of the quadtree node */
} g2pc_leaf_t;

#define G2PC_MAX_LEVELS 12
/* frame header (int32 words, device memory, written by g2pc_build_tree) */
#define G2PC_HDR_NUM_LEAVES 0
#define G2PC_HDR_TOTAL_INST 1     /* sum of the leaves' instance counts, low word */
#define G2PC_HDR_TOTAL_PIX 2
#define G2PC_HDR_NEED_DEEPER 3    /* a tile at the deepest tabulated level still has to split: tabulate more levels */
#define G2PC_HDR_LEAF_OVERFLOW 4  /* more leaves than max_leaves */
#define G2PC_HDR_CAP_OVERFLOW 5   /* instance / leaf-pixel / multisplit-matrix / row-list capacity too small for this
                                     frame */
#define G2PC_HDR_POISON 6         /* snapshot of the shared failure word at the end of this frame's build_tree: 0 = no
                                     frame has failed, else 1 + the LOWEST frame number that did not fit */
#define G2PC_HDR_FRAME 7          /* frame number of the header's contents */
#define G2PC_HDR_TOTAL_INST_HI 8
#define G2PC_HDR_ROW_INST 9       /* entries of the multisplit's row lists (written by the multisplit; saturates at
                                     2^31 - 1) */
#define G2PC_HDR_WORDS 16
#define G2PC_WORK_COUNTERS 4      /* int32 work-distribution counters cleared by g2pc_build_tree */
/* device-side statistics (uint64 words, accumulated by g2pc_blend when `stats` is not NULL) */
#define G2PC_STAT_WARP_GAUSSIANS 0  /* (warp, Gaussian) iterations executed: x 128 = (pixel, Gaussian) pairs */
#define G2PC_STAT_WORDS 4

/* The failure word `fail` (one uint32 in device memory, shared by the frames in flight, initialised to 0xFFFFFFFF):
 * build_tree lowers it to 1 + frame when the frame does not fit; build_tree, multisplit and blend of frame f do nothing
 * iff f + 1 >= *fail.  Frames may be enqueued on two streams (the front-end of frame f + 1 overlaps the blend of frame
 * f), so a later frame can fail first: earlier frames still complete.  The caller resets the word after growing its
 * buffers and replays from the failed frame. */

/* Quadtree tables (host-built, g2pc/quadtree.py): `tables` = 6 int32 arrays of n1 = 2^num_levels - 1 entries each,
 * concatenated: x start, x end (inclusive), x flags, y start, y end, y flags; level l at offset 2^l - 1.
 * 2-D node index = (4^l - 1)/3 + iy * 2^l + ix.  level_mask: bit l set iff level l has nodes small enough to be
 * leaves.  clean_mask: bit l set iff level l has no dropped / degenerate node on either axis (then the membership of
 * an interval is exactly its looked-up node range and the kernels skip the per-node table checks). */

/* Once per renderer: geom (n x 48 bytes, 16-byte aligned) = {x,y,z,S00} {S01,S02,S11,S12} {S22,log2(opacity),0,0}
 * from xyz (n,3), cov (n,3,3), opacity (n) — the coalesced 16-byte-load form the per-camera kernel reads. */
int g2pc_pack_geometry(const float* xyz, const float* cov, const float* opacity, int64_t n, void* geom, void* stream);

/* S3.  Per Gaussian: projection (projection_ndc, gauss_render.py:151-168), EWA covariance (build_covariance_2d
 * :101-148), radius / rect (:171-193), conic = inverse(cov2d) (:349) pre-scaled by -0.5*log2(e), colour (given, or SH
 * deg <= 3 evaluated towards the camera: eval_sh :43-99 + 0.5, clamped at 0), and tile-membership counting on the
 * leaf-candidate levels.  colours (n,3) f32 or NULL · shs (n,3,sh_stride) f32 channel-major or NULL.
 * proj: n x 48 bytes (3 float4: {mx,my,c00',c01'} {c11',log2(opacity),r,g} {b,depth,radius,valid}).
 * node_cnt: one uint32 per 2-D node, zero on entry (g2pc_build_tree clears it again).  depth_key (n) uint32:
 * bits(-z_view), 0xFFFFFFFF if behind the camera.  val (n) uint64: (node range at the first candidate level, 8 bits per
 * bound: xlo | xhi<<8 | ylo<<16 | yhi<<24) << 32 | Gaussian index.
 * luts (uint16, 4-byte aligned): per level [x lo (W)][x hi+1 (W)][y lo (H)][y hi+1 (H)] — node range of an interval as
 * a lookup over pixel coordinates, lo[floor(min)] .. hi1[ceil(max)] - 1 (g2pc/quadtree.py QuadtreeTables.pixel_luts). */
int g2pc_preprocess(const void* geom, const float* colours, const float* shs, int32_t sh_stride, int32_t sh_degree,
                    int64_t n, const g2pc_camera_t* cam_host, const int32_t* tables, const uint16_t* luts,
                    int32_t num_levels, uint32_t level_mask, uint32_t clean_mask, void* proj, uint32_t* node_cnt,
                    uint32_t* depth_key, uint64_t* val, void* stream);

/* S3 for a batch of cameras: the same outputs as num_cameras calls of g2pc_preprocess, bit for bit, with the scene read
 * once per batch instead of once per camera.  cams_host: num_cameras (1..G2PC_PREPROCESS_MAX_CAMERAS) cameras of one
 * resolution, which share tables / luts / masks.  proj, node_cnt, depth_key, val: host arrays of num_cameras device
 * pointers, camera c's outputs as g2pc_preprocess describes them.  The cameras whose node histograms do not fit the
 * shared memory together go to further launches (one camera per launch when even one histogram does not fit). */
#define G2PC_PREPROCESS_MAX_CAMERAS 8
int g2pc_preprocess_cameras(const void* geom, const float* colours, const float* shs, int32_t sh_stride,
                            int32_t sh_degree, int64_t n, const g2pc_camera_t* cams_host, int32_t num_cameras,
                            const int32_t* tables, const uint16_t* luts, int32_t num_levels, uint32_t level_mask,
                            uint32_t clean_mask, void* const* proj, uint32_t* const* node_cnt,
                            uint32_t* const* depth_key, uint64_t* const* val, void* stream);

/* S4a.  val_sorted[k] = val of the k-th nearest Gaussian (stable radix sort of depth_key: ties keep index order, the
 * reference's torch.sort is unstable there, gauss_render.py:340-344).  cub::DeviceRadixSort (library call). */
int64_t g2pc_depth_sort_workspace_bytes(int64_t n);
int g2pc_depth_sort(const uint32_t* depth_key, const uint64_t* val, int64_t n, uint64_t* val_sorted, void* workspace,
                    int64_t workspace_bytes, void* stream);

/* S4b.  Resolve the quadtree (one CTA): node states, node_leaf (int32 per node: leaf id, -1 none, -2 split), leaves in
 * the reference's BFS order with list / pixel offsets, leaf_order (heaviest leaf first, the blend's launch order), the
 * frame header; clears node_cnt and work_counters.  inst_capacity (uint32 ids) / pix_capacity (pixels) /
 * matrix_capacity (uint32 words, >= ms_chunks * leaves): sizes of the caller's buffers, checked here. */
int g2pc_build_tree(const int32_t* tables, int32_t num_levels, int32_t max_gaussians_per_tile, uint32_t* node_cnt,
                    uint8_t* node_state, int32_t* node_leaf, g2pc_leaf_t* leaves, int32_t* leaf_order,
                    int32_t max_leaves, int64_t inst_capacity, int64_t pix_capacity, int64_t matrix_capacity,
                    int32_t ms_chunks, int32_t frame, int32_t* header, uint32_t* fail, int32_t* work_counters,
                    void* stream);

/* S4c.  Stable multisplit of the depth-ordered stream into the leaves' lists: inst_gid[leaf.inst_begin ..
 * + leaf.inst_count) = Gaussian ids overlapping the leaf, nearest first.
 * Base-level leaves (cells of the first leaf-candidate level, 2^base x 2^base): the stream is split by rows into row
 * lists of 64-bit entries, then each row list by columns into the leaves' lists.  workspace:
 * g2pc_multisplit_workspace_bytes(n, row_capacity, 2^base, 2^base) bytes, 256-byte aligned, holding row_capacity
 * row-list entries.  A frame whose row lists need more (at most the base level's instances when that level is clean) sets
 * HDR_CAP_OVERFLOW and HDR_ROW_INST in `header`, lowers `fail` and is skipped like a frame build_tree refused.
 * Leaves below the base level (num_levels > base + 1 only): three more kernels (count, scan, scatter); one CTA per
 * chunk of S x C consecutive sorted entries, walked in S sub-steps of C = g2pc_multisplit_chunk(leaf_cap) entries
 * (S grows with n: a few waves of CTAs on the GPU); matrix: g2pc_multisplit_rows(n, leaf_cap) x leaves uint32 scratch
 * (pass that row count as ms_chunks to g2pc_build_tree, which checks the capacity; NULL and 0 rows without such levels).
 * leaf_cap = max_leaves given to g2pc_build_tree. */
int32_t g2pc_multisplit_chunk(int32_t leaf_cap);           /* C: entries per sub-step (0: too many leaves) */
int32_t g2pc_multisplit_rows(int64_t n, int32_t leaf_cap); /* rows of `matrix` needed: one per chunk */
int64_t g2pc_multisplit_workspace_bytes(int64_t n, int64_t row_capacity, int32_t grid_w, int32_t grid_h);
int g2pc_multisplit(const uint64_t* val_sorted, int64_t n, const void* proj, int32_t width, int32_t height,
                    const int32_t* tables, int32_t num_levels, uint32_t level_mask, uint32_t clean_mask,
                    const int32_t* node_leaf, const g2pc_leaf_t* leaves, int32_t* header, const uint32_t* fail,
                    int32_t frame, int32_t leaf_cap, uint32_t* matrix, int64_t row_capacity, void* workspace,
                    int64_t workspace_bytes, uint32_t* inst_gid, void* stream);

/* S5.  Front-to-back blend of every leaf (gauss_render.py:337-369) + per-Gaussian maximum contribution / arg-max pixel
 * (:371-385) published as cam_best[g] = max((bits(contribution) << 32) | ~leaf_pixel_index).
 * The leaf count comes from `header` (device).  max_leaf_width / max_leaf_height: upper bounds of the leaves' w and h
 * (every leaf fits in max_leaf_width x max_leaf_height); they size the split of a leaf into work items.
 * max_contrib (n) f32: the running maxima of the earlier cameras (read-only here; contributions that cannot beat
 * them skip the bookkeeping).  leaf_colour: (pix_capacity,3) f32.  owner: uint32 per image pixel (zero on entry):
 * 1 + index of the last leaf pixel covering it.  work_counters: cleared by g2pc_build_tree (persistent CTAs pull
 * (leaf, slab) items, heaviest leaf first).
 * t_stop: a warp stops walking its leaf's list once ALL of its 128 pixels have transmittance T < t_stop; every
 * contribution it skips is then < t_stop and their sum per pixel is < t_stop.  t_stop = 0 selects FLT_MIN (only
 * contributions that underflow are dropped: the strict-parity setting); the reference's CUDA back-end stops each pixel
 * at T < 1e-4 (forward.cu:415).  stats: G2PC_STAT_WORDS uint64 or NULL. */
int g2pc_blend(const g2pc_leaf_t* leaves, const int32_t* leaf_order, const int32_t* header, const uint32_t* fail,
               int32_t frame, int32_t max_leaf_width, int32_t max_leaf_height, const uint32_t* inst_gid, const void* proj,
               uint64_t* cam_best,
               const float* max_contrib, float* leaf_colour, uint32_t* owner, int32_t width, int32_t height,
               float background, float t_stop, int32_t* work_counters, uint64_t* stats, void* stream);

/* Pixel-to-thread mapping of g2pc_blend: 1 (default) = a warp owns a compact block of <= 32 quads (e.g. 20 x 6 pixels),
 * 0 = a warp owns a strip of full rows.  Results do not depend on it up to the t_stop tolerance. */
void g2pc_blend_set_compact(int on);

/* Footprint cull of g2pc_blend: 1 (default) = when t_stop > FLT_MIN, a warp skips the Gaussians whose alpha is below
 * eps = min(2^-26, t_stop / list length) over its whole pixel rectangle (transmittance bit-identical, each pixel's colour
 * moves by < t_stop x max |colour|); 0 = never.  t_stop = 0 (FLT_MIN) never culls. */
void g2pc_blend_set_cull(int on);

/* S6.  Fold one camera into the per-Gaussian accumulators (gauss_render.py:387-395; the role of
 * GaussianRasterizer.update_max_contributions, gaussian_pointcloud_rasterization/__init__.py:142-152):
 * where the camera's best contribution beats max_contrib[g] (strict >) store it and the blended colour of the winning
 * pixel.  Clears cam_best.  first_frame (n) int32 or NULL: set to `frame` where the maximum was raised (the multi-GPU
 * merge needs the index of the camera that first reached each maximum, g2pc/dist.py). */
int g2pc_accumulate(uint64_t* cam_best, const float* leaf_colour, int64_t n, float* max_contrib, float* colours,
                    int32_t* first_frame, int32_t frame, void* stream);

/* Rendered image (H,W,3) f32, flipped left-right like the reference (gauss_render.py:402); clears `owner`. */
int g2pc_compose_image(uint32_t* owner, const float* leaf_colour, int32_t width, int32_t height, float background,
                       float* image, void* stream);

/* ---- colour stage, renderer_type=cuda semantics: the reference's CUDA rasterizer restated (16x16 tiles) ---------- */
/* Replaces _C.rasterize_gaussians (gaussian-pointcloud-rasterization/ext.cpp:15-17, rasterize_points.cu:36-145 ->
 * CudaRasterizer::Rasterizer::forward, rasterizer_impl.cu:197-352: preprocessCUDA forward.cu:153-271, duplicateWithKeys /
 * radix sort / identifyTileRanges rasterizer_impl.cu:69-137,285-326, renderCUDA forward.cu:303-497) and the accumulator
 * updates of GaussianRasterizer.forward (gaussian_pointcloud_rasterization/__init__.py:126-158).
 * One camera = tiles_preprocess -> depth_sort -> tiles_build -> multisplit_grid -> tiles_blend -> tiles_accumulate.
 * The depth-ordered lists are built per SUPER-TILE of 2x2 tiles (32x32 pixels; grid SW x SH = ceil(ceil(W/16)/2) x
 * ceil(ceil(H/16)/2)); the blend of a tile walks its super-tile's list and skips the entries whose tile rect (packed into
 * the projection record) does not contain the tile, so every tile sees exactly the reference's per-tile list. */
typedef struct {
    float viewmatrix[16];  /* world->view, row-vector convention, z forward (camera_handler.py:75,91), row-major */
    float projmatrix[16];  /* viewmatrix @ projection (camera_handler.py:100), row-major */
    float campos[3];
    float tan_fovx, tan_fovy;
    int32_t width, height;
} g2pc_raster_t;

/* preprocessCUDA: near cull z_view <= 0.2, EWA covariance + 0.3, conic, radius = ceil(3 sqrt(lambda_max)), tile rect
 * (16x16 tiles), colour given or SH deg <= 3 (sh_layout 0: (n,3,stride) channel-major as the loader yields it,
 * gauss_dataloader.py:42-44; 1: (n,stride,3) coefficient-major as forward.cu:31 reads it).  Outputs as g2pc_preprocess
 * (proj records — the last word holds the packed TILE rect; depth_key = bits(z_view); val = packed SUPER-TILE rect << 32 |
 * index; node_cnt (SW*SH, zeroed by the caller / by tiles_build) = Gaussians per super-tile); radii (n) int32 or NULL. */
int g2pc_tiles_preprocess(const void* geom, const float* colours, const float* shs, int32_t sh_stride,
                          int32_t sh_degree, int32_t sh_layout, int64_t n, const g2pc_raster_t* rs_host, void* proj,
                          uint32_t* node_cnt, uint32_t* depth_key, uint64_t* val, int32_t* radii, void* stream);

/* List table: every super-tile of the SW x SH grid is a leaf (leaf index = super-tile index, row-major; max_leaves >=
 * SW*SH); list offsets, launch order, frame header / poison as g2pc_build_tree; clears node_cnt and work_counters. */
int g2pc_tiles_build(uint32_t* node_cnt, int32_t width, int32_t height, g2pc_leaf_t* leaves, int32_t* leaf_order,
                     int32_t max_leaves, int64_t inst_capacity, int64_t matrix_capacity, int32_t ms_rows, int32_t frame,
                     int32_t* header, uint32_t* fail, int32_t* work_counters, void* stream);

/* The base-level split of g2pc_multisplit over a flat grid (grid_w x grid_h = SW x SH here, each <= 256; the packed
 * range is the rect in grid cells, leaf = cell index).  workspace: g2pc_multisplit_workspace_bytes(n, row_capacity,
 * grid_w, grid_h) bytes; row-list overflow as g2pc_multisplit. */
int g2pc_multisplit_grid(const uint64_t* val_sorted, int64_t n, int32_t grid_w, int32_t grid_h,
                         const g2pc_leaf_t* leaves, int32_t* header, const uint32_t* fail, int32_t frame,
                         int64_t row_capacity, void* workspace, int64_t workspace_bytes, uint32_t* inst_gid,
                         void* stream);

/* renderCUDA: per pixel front-to-back blend (power > 0 and alpha < 1/255 skipped, the pixel stops before T < 1e-4),
 * out_color (3,H,W) = C + T*bg, out_depth / out_invdepth (H,W) = sum depth*alpha*T / sum alpha*T/depth, written for
 * pixels inside the image whose mask (H*W int32 or NULL) is non-zero; cam_best[g] = max((bits(alpha*T) << 32) |
 * ~pixel_id) (deterministic arg-max: lowest pixel id among equals); cam_dist (n uint32, pre-filled with the bits of
 * FLT_MAX, or NULL): bits of the minimum surface distance (see s7_tiles.cu header). */
int g2pc_tiles_blend(const g2pc_leaf_t* leaves, const int32_t* leaf_order, const int32_t* header, const uint32_t* fail,
                     int32_t frame, const uint32_t* inst_gid, const void* proj, uint64_t* cam_best, uint32_t* cam_dist,
                     const int32_t* mask, float* out_color, float* out_depth, float* out_invdepth, int32_t width,
                     int32_t height, const float* background3_host, int32_t* work_counters, uint64_t* stats,
                     void* stream);

/* g2pc_tiles_blend (cam_dist must be NULL) that also writes, for every pixel inside the image, out_T (H,W) f32 = the final
 * transmittance and out_zmed (H,W) f32 = the view depth of the first blended Gaussian after which T < 0.5, 0 when T never
 * drops below 0.5; both 0 where the mask is 0. */
int g2pc_tiles_blend_fusion(const g2pc_leaf_t* leaves, const int32_t* leaf_order, const int32_t* header,
                            const uint32_t* fail, int32_t frame, const uint32_t* inst_gid, const void* proj,
                            uint64_t* cam_best, uint32_t* cam_dist, const int32_t* mask, float* out_color,
                            float* out_depth, float* out_invdepth, int32_t width, int32_t height,
                            const float* background3_host, int32_t* work_counters, uint64_t* stats, float* out_T,
                            float* out_zmed, void* stream);

/* Accumulator update of one camera (__init__.py:128-158): where the camera's contribution beats max_contrib (strict >)
 * store it and the FINAL colour of its arg-max pixel; total_contrib += contribution; min_dist = min(min_dist, cam_dist).
 * Clears cam_best / re-arms cam_dist.  Optional per-camera outputs of the op (n each): cam_contrib f32, cam_pixel i32,
 * cam_surface f32. */
int g2pc_tiles_accumulate(uint64_t* cam_best, uint32_t* cam_dist, const float* out_color, int32_t width, int32_t height,
                          int64_t n, float* max_contrib, float* total_contrib, float* colours, float* min_dist,
                          int32_t* first_frame, int32_t frame, float* cam_contrib, int32_t* cam_pixel,
                          float* cam_surface, void* stream);

int g2pc_fill_u32(uint32_t* v, uint32_t value, int64_t n, void* stream);

/* ---- N10: TSDF fusion of rendered depth (s14_tsdf.cu, g2pc/tsdf.py, gauss_to_mesh.py --mesh_method tsdf) --------- */
/* Frame words (8 doubles, the layout g2pc_mesh_splat writes) of a 2^depth grid over the finite points xyz (n,3) f32:
 * L = 1.1 x the largest extent, centred on the bounding box, h = L / R.  workspace: g2pc_tsdf_frame_workspace_bytes(n),
 * 4-byte aligned. */
int64_t g2pc_tsdf_frame_workspace_bytes(int64_t n);
int g2pc_tsdf_frame(const float* xyz, int64_t n, int32_t depth, double* frame, void* workspace, int64_t workspace_bytes,
                    void* stream);

/* Integrate one camera into the grid (R^3 voxels, node index (k*R + j)*R + i): tsdf f32, weight f32, colour (3, R^3)
 * f32.  zmed / transmittance (H,W) f32 and image (3,H,W) f32 are g2pc_tiles_blend_fusion's outputs for the camera
 * rs_host, mask (H*W) int32 or NULL, background3_host its background.  One thread per voxel: skipped when the view
 * depth z <= 0.2, the nearest pixel is outside the image or masked, z_med = 0 there, or z_med - z < -mu with
 * mu = float(trunc_voxels * h); otherwise tsdf, colour += (min(1, sdf / mu), un-blended pixel colour) as running means
 * and weight += 1 (DESIGN.md §2, N10).  Does nothing when frame_index is skipped by the failure word fail. */
int g2pc_tsdf_integrate(const double* frame, int32_t depth, double trunc_voxels, const float* zmed,
                        const float* transmittance, const float* image, const int32_t* mask, int32_t width,
                        int32_t height, const g2pc_raster_t* rs_host, const float* background3_host,
                        const uint32_t* fail, int32_t frame_index, float* tsdf, float* weight, float* colour,
                        void* stream);

/* After g2pc_mesh_extract_emit on the tsdf grid (iso 0): keep[v] (m u8) = both ends of vertex v's edge have weight > 0,
 * density[v] = (1-t) w_a + t w_b (f64), vcolours[v] (m,3 u8, NULL with colour NULL) = floor(255 ((1-t) c_a + t c_b) +
 * 1/2) clamped; a triangle is kept iff its three vertices are; then the kept vertices (density, vpos, colours) and
 * triangles (re-indexed) are compacted in order into the *_out arrays, counts (2 int64) = kept vertices, triangles.
 * workspace: g2pc_tsdf_compact_workspace_bytes(m, t), 256-byte aligned. */
int64_t g2pc_tsdf_compact_workspace_bytes(int64_t m, int64_t t);
int g2pc_tsdf_gather_compact(const float* weight, const float* colour, int32_t depth, const int64_t* vkey,
                             const double* vt, const double* vpos, int64_t m, const int32_t* faces, int64_t t,
                             uint8_t* keep, double* density, uint8_t* vcolours, int64_t* counts, double* density_out,
                             double* vpos_out, uint8_t* vcolours_out, int32_t* faces_out, void* workspace,
                             int64_t workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* G2PC_H */
