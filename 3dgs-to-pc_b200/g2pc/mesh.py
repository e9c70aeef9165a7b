"""Poisson mesh of an oriented point cloud on the device (N6): the reference's mesh_handler.generate_mesh
(mesh_handler.py:23-40: Open3D outlier removal, Poisson reconstruction, 10 % density trim, Laplacian smoothing) with
this project's own rules, written down in DESIGN.md §2 and restated in float64 by tests/f64ref_mesh.py.

Steps: statistical outlier removal (g2pc/outliers.py) -> g2pc_mesh_splat -> g2pc_mesh_vcycle until |r| <= 1e-5 |b| or 40
cycles -> g2pc_mesh_iso -> g2pc_mesh_extract_count / _emit (marching tetrahedra) -> g2pc_mesh_gather (density, colour)
-> g2pc_mesh_trim -> g2pc_mesh_smooth -> g2pc_mesh_normals.  Host reads: the frame and skip counts after the splat, the
residual once per cycle, the vertex / triangle counts before and after the trim.

With band_depth (N6b, s12_mesh_band.cu): after the dense solve and iso, per level depth + 1 .. band_depth
g2pc_mesh_band_bricks (host reads the brick count) -> _list -> memory check -> _splat -> _ghosts -> _cg until
|r| <= 1e-6 |b| (one host read per iteration); then g2pc_mesh_band_iso / _extract_count / _extract_emit / _gather at
band_depth and the same trim, smoothing and normals.

With target_triangles (N9, s13_decimate.cu): between the smoothing and the normals, decimate(): g2pc_mesh_decimate_prepare,
then per round _select (host reads the counts) -> _apply until the target is met or nothing is selected, then _finish.

With min_component_triangles / keep_largest_components (N11, s15_components.cu): between the trim and the smoothing,
remove_components(): g2pc_mesh_components_label (host reads the component count) -> _select (host reads the kept counts)
-> _compact.

With max_hole_edges (N12, s16_holes.cu): after the component filter and before the smoothing, fill_holes():
g2pc_mesh_holes_find (host reads the boundary counts) -> _plan (host reads the added counts) -> _fill.
"""
import collections
import math
import warnings

import numpy as np
import torch

from . import capi, outliers

DEPTH_MIN, DEPTH_MAX = 2, 10  # G2PC_MESH_DEPTH_MAX in include/g2pc.h
BAND_DEPTH_MAX = 12  # G2PC_MESH_BAND_DEPTH_MAX
BRICK = 8  # G2PC_MESH_BRICK: nodes per brick edge
BAND_MARGIN = 1  # G2PC_MESH_BAND_MARGIN: bricks of band around the seed bricks
CG_WORDS = 5  # G2PC_MESH_CG_WORDS
MAX_CG_ITERATIONS = 2000
# The band solve stops 10x below the dense target: conjugate gradients leave their error in smooth modes, where
# |r| / |b| = 1e-5 still lets chi move by up to 2.4e-4 of its range (DESIGN.md §2, N6b).
BAND_TOLERANCE = 1e-6
# new device bytes per band node: B, chi, rhs while the ghosts are formed, then chi, rhs and the CG vectors r, p, q;
# with return_debug B, the ghost sums and a copy of the initial chi stay alive as well
BAND_BYTES_PER_NODE = max(8 + 4 + 4, 4 + 4 + 12)
BAND_DEBUG_BYTES_PER_NODE = 8 + 8 + 4 + 4 + 4 + 12
FRAME_WORDS = 8
MAX_CYCLES = 40
TOLERANCE = 1e-5
NB_NEIGHBORS = 20
MAX_HOLE_EDGES = 1024  # the longest hole fill_holes() closes: bounds each loop's walk and a centre's valence

Mesh = collections.namedtuple("Mesh", ["vertices", "faces", "colours", "normals", "densities"])


def splat(points, normals, depth):
    """frame (8,) float64, B (R^3,) int64, cell (n,) int32 (dual cell, 0x7FFFFFFF when not splatted), status (2,) int32
    (skipped normals, non-finite points).  points (n,3) float32, normals (n,3) float32 / float64, contiguous CUDA."""
    dev, n, R = points.device, points.shape[0], 1 << depth
    frame = torch.empty((FRAME_WORDS,), dtype=torch.float64, device=dev)
    B = torch.empty((R ** 3,), dtype=torch.int64, device=dev)
    cell = torch.empty((n,), dtype=torch.int32, device=dev)
    status = torch.empty((2,), dtype=torch.int32, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_splat_workspace_bytes(n), dev)
    capi.call("g2pc_mesh_splat", capi.ptr(points), capi.ptr(normals), capi.dtype_code(normals), n, depth,
              capi.ptr(frame), capi.ptr(B), capi.ptr(cell), capi.ptr(status), capi.ptr(ws), ws.numel(),
              capi.stream_ptr(dev))
    return frame, B, cell, status


def solve(B, frame, depth, max_cycles=MAX_CYCLES, tol=TOLERANCE):
    """chi (R^3,) float32 (not yet mean-free), cycles, |r| / |b| (0 when b = 0)."""
    dev = B.device
    chi = torch.empty((1 << (3 * depth),), dtype=torch.float32, device=dev)
    norms = torch.zeros((2,), dtype=torch.float64, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_solve_workspace_bytes(depth), dev)
    st = capi.stream_ptr(dev)
    ratio, cycles = 0.0, 0
    for c in range(max_cycles):
        capi.call("g2pc_mesh_vcycle", capi.ptr(B), capi.ptr(frame), depth, capi.ptr(chi), int(c == 0), capi.ptr(norms),
                  capi.ptr(ws), ws.numel(), st)
        rr, bb = norms.tolist()
        cycles = c + 1
        if bb == 0.0:
            break
        ratio = math.sqrt(rr / bb)
        if ratio <= tol:
            break
    return chi, cycles, ratio


def iso_value(points, cell, frame, depth, chi):
    """Subtracts the mean of chi in place; returns iso (3,) float64 on the device: (that mean, iso, used points)."""
    dev = points.device
    iso = torch.empty((3,), dtype=torch.float64, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_iso_workspace_bytes(), dev)
    capi.call("g2pc_mesh_iso", capi.ptr(points), capi.ptr(cell), points.shape[0], capi.ptr(frame), depth, capi.ptr(chi),
              capi.ptr(iso), capi.ptr(ws), ws.numel(), capi.stream_ptr(dev))
    return iso


def extract(chi, depth, frame, iso, node_scratch):
    """Marching tetrahedra: vkey (m,) int64, vt (m,) float64, vpos (m,3) float64, faces (t,3) int32.  node_scratch: a
    CUDA tensor of at least 5 bytes per node (its contents are overwritten)."""
    dev = chi.device
    ws = capi.workspace(capi.load().g2pc_mesh_extract_workspace_bytes(depth), dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    st = capi.stream_ptr(dev)
    capi.call("g2pc_mesh_extract_count", capi.ptr(chi), depth, capi.ptr(iso), capi.ptr(counts), capi.ptr(ws),
              ws.numel(), st)
    m, t = counts.tolist()
    if m >= 2 ** 31 - 1 or 3 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the surface has {m} vertices and {t} triangles: more than int32 indices can address")
    vkey = torch.empty((m,), dtype=torch.int64, device=dev)
    vt = torch.empty((m,), dtype=torch.float64, device=dev)
    vpos = torch.empty((m, 3), dtype=torch.float64, device=dev)
    faces = torch.empty((t, 3), dtype=torch.int32, device=dev)
    if m:
        capi.call("g2pc_mesh_extract_emit", capi.ptr(chi), depth, capi.ptr(frame), capi.ptr(iso),
                  capi.ptr(node_scratch), node_scratch.numel() * node_scratch.element_size(), capi.ptr(ws), ws.numel(),
                  capi.ptr(vkey), capi.ptr(vt), capi.ptr(vpos), capi.ptr(faces), st)
    return vkey, vt, vpos, faces


def gather(points, colours, cell, frame, depth, vkey, vt, cell_scratch):
    """density (m,) float64 and colours (m,3) uint8 (None when colours is None) of every vertex.  colours (n,3) int32."""
    dev, n, m = points.device, points.shape[0], vkey.shape[0]
    dens = torch.empty((m,), dtype=torch.float64, device=dev)
    vcol = torch.empty((m, 3), dtype=torch.uint8, device=dev) if colours is not None else None
    ws = capi.workspace(capi.load().g2pc_mesh_gather_workspace_bytes(n), dev)
    capi.call("g2pc_mesh_gather", capi.ptr(points), capi.ptr(colours), capi.ptr(cell), n, capi.ptr(frame), depth,
              capi.ptr(vkey), capi.ptr(vt), m, capi.ptr(cell_scratch),
              cell_scratch.numel() * cell_scratch.element_size(), capi.ptr(dens), capi.ptr(vcol), capi.ptr(ws),
              ws.numel(), capi.stream_ptr(dev))
    return dens, vcol


def trim(dens, vpos, vcol, faces):
    """Removes the vertices below numpy's linear 10 % density quantile and every triangle that uses one.  Returns
    (dens, vpos, vcol, faces) of the kept mesh, the keep mask (m,) uint8 and the threshold (1,) float64."""
    dev, m, t = dens.device, dens.shape[0], faces.shape[0]
    keep = torch.empty((m,), dtype=torch.uint8, device=dev)
    thr = torch.empty((1,), dtype=torch.float64, device=dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    outs = [torch.empty_like(dens), torch.empty_like(vpos), torch.empty_like(vcol) if vcol is not None else None,
            torch.empty_like(faces)]
    ws = capi.workspace(capi.load().g2pc_mesh_trim_workspace_bytes(m, t), dev)
    capi.call("g2pc_mesh_trim", capi.ptr(dens), capi.ptr(vpos), capi.ptr(vcol), m, capi.ptr(faces), t, capi.ptr(keep),
              capi.ptr(thr), capi.ptr(counts), *[capi.ptr(o) for o in outs], capi.ptr(ws), ws.numel(),
              capi.stream_ptr(dev))
    mk, tk = counts.tolist()
    d, p, c, f = outs
    return d[:mk], p[:mk], (c[:mk] if c is not None else None), f[:tk], keep, thr


def smooth(vpos, faces, iterations):
    """`iterations` Jacobi steps of the weighted Laplacian (lambda = 1/2) on vpos (m,3) float64, in place."""
    m, t = vpos.shape[0], faces.shape[0]
    if m == 0 or iterations == 0:
        return vpos
    ws = capi.workspace(capi.load().g2pc_mesh_smooth_workspace_bytes(m, t), vpos.device)
    capi.call("g2pc_mesh_smooth", capi.ptr(vpos), m, capi.ptr(faces), t, int(iterations), capi.ptr(ws), ws.numel(),
              capi.stream_ptr(vpos.device))
    return vpos


def vertex_normals(vpos, faces):
    """vertices (m,3) float32 and area-weighted unit normals (m,3) float32."""
    dev, m, t = vpos.device, vpos.shape[0], faces.shape[0]
    v = torch.empty((m, 3), dtype=torch.float32, device=dev)
    nrm = torch.empty((m, 3), dtype=torch.float32, device=dev)
    if m:
        ws = capi.workspace(capi.load().g2pc_mesh_normals_workspace_bytes(m, t), dev)
        capi.call("g2pc_mesh_normals", capi.ptr(vpos), m, capi.ptr(faces), t, capi.ptr(v), capi.ptr(nrm), capi.ptr(ws),
                  ws.numel(), capi.stream_ptr(dev))
    return v, nrm


def band_bricks(pts, cell, frame, depth, parent_map):
    """Level `depth` of the band: band frame (8,) float64, brick map (NB^3,) int32, brick list (k,) int32, and the
    count of seed bricks the nesting rule dropped.  Reads the counts once."""
    dev, n, NB = pts.device, pts.shape[0], 1 << (depth - 3)
    bframe = torch.empty((FRAME_WORDS,), dtype=torch.float64, device=dev)
    bmap = torch.empty((NB ** 3,), dtype=torch.int32, device=dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_band_bricks_workspace_bytes(depth), dev)
    st = capi.stream_ptr(dev)
    capi.call("g2pc_mesh_band_bricks", capi.ptr(pts), capi.ptr(cell), n, capi.ptr(frame), depth, capi.ptr(parent_map),
              capi.ptr(bframe), capi.ptr(bmap), capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
    del ws
    k, lost = counts.tolist()
    blist = torch.empty((k,), dtype=torch.int32, device=dev)
    if k:
        capi.call("g2pc_mesh_band_list", capi.ptr(bmap), depth, capi.ptr(blist), st)
    return bframe, bmap, blist, lost


def band_splat(pts, nrm, cell, bframe, depth, bmap, nbricks):
    """B (nbricks * 512,) int64 on band storage, and the count of terms that fell outside the band (0 when nested)."""
    dev = pts.device
    B = torch.empty((nbricks * BRICK ** 3,), dtype=torch.int64, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    capi.call("g2pc_mesh_band_splat", capi.ptr(pts), capi.ptr(nrm), capi.dtype_code(nrm), capi.ptr(cell),
              pts.shape[0], capi.ptr(bframe), depth, capi.ptr(bmap), nbricks, capi.ptr(B), capi.ptr(status),
              capi.stream_ptr(dev))
    return B, status


def band_ghosts(parent_chi, parent_map, depth, bmap, blist, B, bframe, with_ghosts=False):
    """(ghost sums (float64, None unless with_ghosts), initial chi (float32), right-hand side (float32)) per band node."""
    dev, nodes = B.device, B.shape[0]
    ghost = torch.empty((nodes,), dtype=torch.float64, device=dev) if with_ghosts else None
    chi = torch.empty((nodes,), dtype=torch.float32, device=dev)
    rhs = torch.empty((nodes,), dtype=torch.float32, device=dev)
    capi.call("g2pc_mesh_band_ghosts", capi.ptr(parent_chi), capi.ptr(parent_map), depth, capi.ptr(bmap),
              capi.ptr(blist), blist.shape[0], capi.ptr(B), capi.ptr(bframe), capi.ptr(ghost), capi.ptr(chi),
              capi.ptr(rhs), capi.stream_ptr(dev))
    return ghost, chi, rhs


def band_solve(rhs, chi, depth, bmap, blist, max_iterations=MAX_CG_ITERATIONS, tol=BAND_TOLERANCE):
    """Jacobi-preconditioned CG on chi (in place): (iterations, |r| / |rhs|).  One host read per iteration.  When the
    recurrence says the target is met, the residual is recomputed from chi (a restart) and the solve continues if the
    recomputed one is above it."""
    dev = rhs.device
    sc = torch.zeros((CG_WORDS,), dtype=torch.float64, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_band_cg_workspace_bytes(blist.shape[0]), dev)
    st = capi.stream_ptr(dev)
    args = (capi.ptr(rhs), depth, capi.ptr(bmap), capi.ptr(blist), blist.shape[0], capi.ptr(chi))
    tail = (capi.ptr(sc), capi.ptr(ws), ws.numel(), st)
    total, it, ratio, cc = 0, 0, 0.0, None
    while True:
        if it == 0:
            capi.call("g2pc_mesh_band_cg_start", *args, *tail)
        else:
            capi.call("g2pc_mesh_band_cg_step", *args, it, *tail)
        c2, _, rr = sc[:3].tolist()
        cc = c2 if cc is None else cc
        if cc == 0.0:
            return total, 0.0
        ratio = math.sqrt(rr / cc)
        if ratio <= tol and it > 0:
            it = 0  # confirm with a fresh residual
            continue
        if ratio <= tol or total >= max_iterations:
            return total, ratio
        it += 1
        total += 1


def band_iso(pts, cell, bframe, depth, bmap, chi):
    dev = pts.device
    iso = torch.empty((3,), dtype=torch.float64, device=dev)
    ws = capi.workspace(capi.load().g2pc_mesh_band_iso_workspace_bytes(), dev)
    capi.call("g2pc_mesh_band_iso", capi.ptr(pts), capi.ptr(cell), pts.shape[0], capi.ptr(bframe), depth,
              capi.ptr(bmap), capi.ptr(chi), capi.ptr(iso), capi.ptr(ws), ws.numel(), capi.stream_ptr(dev))
    return iso


def band_extract(chi, depth, bmap, blist, bframe, iso, smoothing=False):
    """Marching tetrahedra over the covered cubes of the band: vkey, vt, vpos, faces as extract().  smoothing: the
    mesh goes on to g2pc_mesh_smooth, whose one-ring lists hold 6 entries per triangle in int32."""
    dev, k = chi.device, blist.shape[0]
    ws = capi.workspace(capi.load().g2pc_mesh_band_extract_workspace_bytes(k), dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    st = capi.stream_ptr(dev)
    capi.call("g2pc_mesh_band_extract_count", capi.ptr(chi), depth, capi.ptr(bmap), capi.ptr(blist), k, capi.ptr(iso),
              capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
    m, t = counts.tolist()
    if m >= 2 ** 31 - 1 or 3 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the surface at band_depth {depth} has {m} vertices and {t} triangles: more than int32 "
                             f"indices can address; use a smaller band_depth")
    if smoothing and 6 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the surface at band_depth {depth} has {t} triangles: the Laplacian smoothing's one-ring "
                             f"lists (6 per triangle) exceed int32; use a smaller band_depth or laplacian_iters=0")
    # extraction scratch and mesh, then the larger of the trim's and the smoothing's buffers
    check_memory(5 * chi.shape[0] + 40 * m + 12 * t + max(52 * m + 20 * t, 96 * t + 24 * m), dev,
                 f"the band surface at depth {depth} ({m} vertices, {t} triangles)")
    vkey = torch.empty((m,), dtype=torch.int64, device=dev)
    vt = torch.empty((m,), dtype=torch.float64, device=dev)
    vpos = torch.empty((m, 3), dtype=torch.float64, device=dev)
    faces = torch.empty((t, 3), dtype=torch.int32, device=dev)
    if m:
        scratch = torch.empty((5 * chi.shape[0],), dtype=torch.uint8, device=dev)
        capi.call("g2pc_mesh_band_extract_emit", capi.ptr(chi), depth, capi.ptr(bmap), capi.ptr(blist), k,
                  capi.ptr(bframe), capi.ptr(iso), capi.ptr(scratch), scratch.numel(), capi.ptr(ws), ws.numel(),
                  capi.ptr(vkey), capi.ptr(vt), capi.ptr(vpos), capi.ptr(faces), st)
    return vkey, vt, vpos, faces


def band_gather(points, colours, cell, bframe, depth, vkey, vt):
    """gather() at a band level (int64 dual cells)."""
    dev, n, m = points.device, points.shape[0], vkey.shape[0]
    dens = torch.empty((m,), dtype=torch.float64, device=dev)
    vcol = torch.empty((m, 3), dtype=torch.uint8, device=dev) if colours is not None else None
    ws = capi.workspace(capi.load().g2pc_mesh_band_gather_workspace_bytes(n), dev)
    capi.call("g2pc_mesh_band_gather", capi.ptr(points), capi.ptr(colours), capi.ptr(cell), n, capi.ptr(bframe), depth,
              capi.ptr(vkey), capi.ptr(vt), m, capi.ptr(dens), capi.ptr(vcol), capi.ptr(ws), ws.numel(),
              capi.stream_ptr(dev))
    return dens, vcol


def check_memory(need, dev, what, remedy="use a smaller band_depth"):
    """Raises G2pcError when `what` needs more than the device's free bytes (after emptying PyTorch's cache)."""
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info(dev)
    if need > free:
        raise capi.G2pcError(f"{what} needs {need} bytes, but only {free} bytes of device memory are free: {remedy}")


def check_target(target_triangles):
    """Refuses a triangle target that is not an integer >= 1 (bool included)."""
    if isinstance(target_triangles, bool) or not isinstance(target_triangles, (int, np.integer)) or target_triangles < 1:
        raise capi.G2pcError(f"target_triangles must be an integer >= 1, got {target_triangles!r}")


def decimate(vpos, faces, target_triangles, colours=None, densities=None, return_debug=False, stats=None):
    """Decimation by parallel quadric edge collapse (DESIGN.md §2, N9) to target_triangles or target_triangles - 1
    triangles.  vpos (m,3) float64, faces (t,3) int32 (no face uses a vertex twice), colours (m,3) uint8 or None,
    densities (m,) float64 or None, all CUDA.  Returns (vpos, faces, colours, densities) of the decimated mesh: the
    surviving vertices in their order, a merged vertex with the rounded mean colour and the mean density of the original
    vertices merged into it.  Boundary, non-manifold and unused vertices never move and are never removed.  When no edge
    can collapse before the target is met, returns what was reached with a RuntimeWarning.  target_triangles >= t returns
    the input tensors themselves and runs no kernel.

    stats: a dict that receives rounds, collapses (per round) and reached (the target was met).  return_debug: also a
    dict with quadrics and free (after the preparation) and rounds: per round a dict of edges, candidates, selected
    (counts), keys (the applied keys, ascending) and ab (their survivor / removed vertex pairs), then vpos, quadrics,
    colour_sums, merged, density_sums and faces after the round."""
    check_target(target_triangles)
    for name, x in (("vpos", vpos), ("faces", faces), ("colours", colours), ("densities", densities)):
        if x is not None and not (torch.is_tensor(x) and x.is_cuda):
            raise capi.G2pcError(f"{name} must be a CUDA tensor (the decimation has no CPU path)")
    if vpos.dim() != 2 or vpos.shape[1] != 3 or vpos.dtype != torch.float64:
        raise capi.G2pcError(f"vpos must be (m, 3) float64, got {tuple(vpos.shape)} {vpos.dtype}")
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype != torch.int32:
        raise capi.G2pcError(f"faces must be (t, 3) int32, got {tuple(faces.shape)} {faces.dtype}")
    m, t, dev = vpos.shape[0], faces.shape[0], vpos.device
    if colours is not None and (colours.shape != (m, 3) or colours.dtype != torch.uint8):
        raise capi.G2pcError(f"colours must be (m, 3) uint8, got {tuple(colours.shape)} {colours.dtype}")
    if densities is not None and (densities.shape != (m,) or densities.dtype != torch.float64):
        raise capi.G2pcError(f"densities must be (m,) float64, got {tuple(densities.shape)} {densities.dtype}")
    if any(x is not None and x.device != dev for x in (faces, colours, densities)):
        raise capi.G2pcError("vpos, faces, colours and densities must be on one device")
    if m >= 2 ** 31 - 1 or 3 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the mesh has {m} vertices and {t} triangles: more than the decimation's int32 lists "
                             f"(3 entries per triangle) can hold")
    if m and not bool(torch.isfinite(vpos).all()):
        raise capi.G2pcError("a vertex position is not finite")
    if t:
        f = faces.long()
        lo, hi, rep = torch.stack([f.min(), f.max(), ((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) |
                                                       (f[:, 0] == f[:, 2])).sum()]).tolist()
        del f
        if lo < 0 or hi >= m:
            raise capi.G2pcError(f"face indices must be in 0..{m - 1}, got {lo}..{hi}")
        if rep:
            raise capi.G2pcError(f"{rep} face(s) use a vertex twice")
    target = int(target_triangles)
    if target >= t:
        if stats is not None:
            stats.update(rounds=0, collapses=[], reached=True)
        out = (vpos, faces, colours, densities)
        return (out, {"rounds": []}) if return_debug else out
    lib = capi.load()
    round_bytes = lib.g2pc_mesh_decimate_round_workspace_bytes(m, t)
    # positions, Q (80 B), flags, alive, merge counts, colour and density sums per vertex; two face buffers; the round
    # workspace (sorted incidence and edge keys)
    check_memory(m * (24 + 80 + 1 + 1 + 4 + 24 + 8) + 2 * 12 * t + round_bytes, dev,
                 f"decimating {m} vertices and {t} triangles", remedy="decimate a smaller mesh")
    st = capi.stream_ptr(dev)
    p = vpos.clone()
    Q = torch.empty((m, 10), dtype=torch.float64, device=dev)
    free = torch.empty((m,), dtype=torch.uint8, device=dev)
    ws = capi.workspace(lib.g2pc_mesh_decimate_prepare_workspace_bytes(m, t), dev)
    capi.call("g2pc_mesh_decimate_prepare", capi.ptr(p), m, capi.ptr(faces), t, capi.ptr(Q), capi.ptr(free),
              capi.ptr(ws), ws.numel(), st)
    del ws
    alive = torch.ones((m,), dtype=torch.uint8, device=dev)
    merged = torch.ones((m,), dtype=torch.int32, device=dev)
    csum = colours.to(torch.int64).contiguous() if colours is not None else None
    dsum = densities.clone() if densities is not None else None
    debug = {"quadrics": Q.clone(), "free": free.clone(), "rounds": []} if return_debug else None
    ws = capi.workspace(round_bytes, dev)
    counts = torch.zeros((4,), dtype=torch.int64, device=dev)  # edges, candidates, selected; faces kept by apply
    bufs = [torch.empty_like(faces), torch.empty((max(t - 2, 1), 3), dtype=torch.int32, device=dev)]
    cur, collapses = faces, []
    while t > target:
        capi.call("g2pc_mesh_decimate_select", capi.ptr(p), m, capi.ptr(cur), t, capi.ptr(Q), capi.ptr(free),
                  capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
        E, C, S, kept = counts.tolist()
        if collapses and kept != t:
            raise capi.G2pcError(f"round {len(collapses)} kept {kept} triangles, expected {t}")
        if S == 0:
            warnings.warn(f"the decimation stopped at {t} triangles, above the target of {target}: no edge can "
                          f"collapse (boundary, non-manifold or locked by the link and fold-over checks)",
                          RuntimeWarning, stacklevel=2)
            break
        k = min(S, (t - target + 1) // 2)
        nxt = bufs[len(collapses) % 2][:t - 2 * k]
        keys = torch.empty((k,), dtype=torch.int64, device=dev) if return_debug else None
        ab = torch.empty((k, 2), dtype=torch.int32, device=dev) if return_debug else None
        capi.call("g2pc_mesh_decimate_apply", capi.ptr(p), m, capi.ptr(cur), t, capi.ptr(Q), capi.ptr(csum),
                  capi.ptr(merged), capi.ptr(dsum), capi.ptr(alive), S, k, capi.ptr(nxt), capi.ptr(counts[3:]),
                  capi.ptr(keys), capi.ptr(ab), capi.ptr(ws), ws.numel(), st)
        t -= 2 * k
        cur = nxt
        collapses.append(k)
        if return_debug:
            debug["rounds"].append({"edges": E, "candidates": C, "selected": S, "keys": keys, "ab": ab,
                                    "vpos": p.clone(), "quadrics": Q.clone(), "merged": merged.clone(),
                                    "colour_sums": csum.clone() if csum is not None else None,
                                    "density_sums": dsum.clone() if dsum is not None else None,
                                    "faces": nxt.clone()})
    del ws
    if stats is not None:
        stats.update(rounds=len(collapses), collapses=collapses, reached=t <= target)
    vout = torch.empty((m, 3), dtype=torch.float64, device=dev)
    cout = torch.empty((m, 3), dtype=torch.uint8, device=dev) if colours is not None else None
    dout = torch.empty((m,), dtype=torch.float64, device=dev) if densities is not None else None
    fout = torch.empty((t, 3), dtype=torch.int32, device=dev)
    fin = torch.empty((1,), dtype=torch.int64, device=dev)
    ws = capi.workspace(lib.g2pc_mesh_decimate_finish_workspace_bytes(m), dev)
    capi.call("g2pc_mesh_decimate_finish", capi.ptr(p), m, capi.ptr(cur), t, capi.ptr(alive), capi.ptr(csum),
              capi.ptr(merged), capi.ptr(dsum), capi.ptr(vout), capi.ptr(cout), capi.ptr(dout), capi.ptr(fout),
              capi.ptr(fin), capi.ptr(ws), ws.numel(), st)
    mk = int(fin.item())
    out = (vout[:mk], fout, cout[:mk] if cout is not None else None, dout[:mk] if dout is not None else None)
    return (out, debug) if return_debug else out


def decimate_mesh(mesh, target_triangles, stats=None):
    """decimate() of a Mesh (its float32 vertices taken as float64), with the normals recomputed by vertex_normals.
    A target of at least the mesh's triangle count returns the mesh itself."""
    check_target(target_triangles)
    if target_triangles >= mesh.faces.shape[0]:
        if stats is not None:
            stats.update(rounds=0, collapses=[], reached=True)
        return mesh
    vpos, faces, vcol, dens = decimate(mesh.vertices.to(torch.float64), mesh.faces.contiguous(), target_triangles,
                                       mesh.colours, mesh.densities, stats=stats)
    v, vn = vertex_normals(vpos, faces)
    return Mesh(v, faces, vcol, vn, dens)


def check_component_params(min_triangles, keep_largest, need_one=True):
    """Refuses a component-filter parameter that is neither None nor an integer >= 1 (bool included), and, with need_one,
    two Nones."""
    for name, x in (("min_triangles", min_triangles), ("keep_largest", keep_largest)):
        if x is not None and (isinstance(x, bool) or not isinstance(x, (int, np.integer)) or x < 1):
            raise capi.G2pcError(f"{name} must be None or an integer >= 1, got {x!r}")
    if need_one and min_triangles is None and keep_largest is None:
        raise capi.G2pcError("give min_triangles, keep_largest or both")


def remove_components(vpos, faces, colours=None, densities=None, min_triangles=None, keep_largest=None, stats=None,
                      return_debug=False):
    """Removes the small connected components of a triangle mesh (DESIGN.md §2, N11).  Two vertices are connected when a
    face uses both; a component's size is its number of triangles.  A component is kept iff its size is >= 1, >=
    min_triangles (when given) and its rank is < keep_largest (when given; ranked by size descending, ties to the smaller
    label, a component's smallest vertex index).  vpos (m,3) float64, faces (t,3) int32, colours (m,3) uint8 or None,
    densities (m,) float64 or None, all CUDA.  Returns (vpos, faces, colours, densities) of the kept vertices and faces,
    in their order, with the faces renumbered; the values are copied unchanged.  Raises G2pcError when nothing is kept.

    stats: a dict that receives components (with at least one triangle), kept, largest (size), removed_triangles and
    removed_vertices.  return_debug: also a dict with labels (m,) int32, keep (m,) uint8 and sizes (m,) int32 (triangles
    per label, 0 at an index that is no label)."""
    check_component_params(min_triangles, keep_largest)
    for name, x in (("vpos", vpos), ("faces", faces), ("colours", colours), ("densities", densities)):
        if x is not None and not (torch.is_tensor(x) and x.is_cuda):
            raise capi.G2pcError(f"{name} must be a CUDA tensor (the component filter has no CPU path)")
    if vpos.dim() != 2 or vpos.shape[1] != 3 or vpos.dtype != torch.float64:
        raise capi.G2pcError(f"vpos must be (m, 3) float64, got {tuple(vpos.shape)} {vpos.dtype}")
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype != torch.int32:
        raise capi.G2pcError(f"faces must be (t, 3) int32, got {tuple(faces.shape)} {faces.dtype}")
    m, t, dev = vpos.shape[0], faces.shape[0], vpos.device
    if colours is not None and (colours.shape != (m, 3) or colours.dtype != torch.uint8):
        raise capi.G2pcError(f"colours must be (m, 3) uint8, got {tuple(colours.shape)} {colours.dtype}")
    if densities is not None and (densities.shape != (m,) or densities.dtype != torch.float64):
        raise capi.G2pcError(f"densities must be (m,) float64, got {tuple(densities.shape)} {densities.dtype}")
    if any(x is not None and x.device != dev for x in (faces, colours, densities)):
        raise capi.G2pcError("vpos, faces, colours and densities must be on one device")
    if m >= 2 ** 31 - 1 or 3 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the mesh has {m} vertices and {t} triangles: more than the component filter's int32 "
                             f"indices can address")
    if t:
        lo, hi = torch.stack([faces.min(), faces.max()]).tolist()
        if lo < 0 or hi >= m:
            raise capi.G2pcError(f"face indices must be in 0..{m - 1}, got {lo}..{hi}")
    if t == 0:
        raise capi.G2pcError("no component is kept: the mesh has no triangle (the largest component has 0)")
    vpos, faces = vpos.contiguous(), faces.contiguous()
    colours = colours.contiguous() if colours is not None else None
    lib = capi.load()
    ws_bytes = lib.g2pc_mesh_components_select_workspace_bytes(m, t)
    # labels, sizes, keep, a density scratch when there are no densities, the select workspace, and outputs as large
    # as the input mesh
    check_memory(m * (4 + 4 + 1) + (8 * m if densities is None else 0) + ws_bytes + m * (24 + 8 + 3) + 12 * t, dev,
                 f"the component filter of {m} vertices and {t} triangles", remedy="filter a smaller mesh")
    st = capi.stream_ptr(dev)
    labels = torch.empty((m,), dtype=torch.int32, device=dev)
    sizes = torch.empty((m,), dtype=torch.int32, device=dev)
    counts = torch.empty((3,), dtype=torch.int64, device=dev)
    capi.call("g2pc_mesh_components_label", capi.ptr(faces), m, t, capi.ptr(labels), capi.ptr(sizes),
              capi.ptr(counts), st)
    components, largest = counts[:2].tolist()
    keep = torch.empty((m,), dtype=torch.uint8, device=dev)
    ws = capi.workspace(ws_bytes, dev)
    capi.call("g2pc_mesh_components_select", capi.ptr(faces), m, t, capi.ptr(labels), capi.ptr(sizes), components,
              int(min_triangles or 0), int(keep_largest or 0), capi.ptr(keep), capi.ptr(counts), capi.ptr(ws),
              ws.numel(), st)
    mk, tk, kept = counts.tolist()
    if stats is not None:
        stats.update(components=components, kept=kept, largest=largest, removed_triangles=t - tk,
                     removed_vertices=m - mk)
    if tk == 0:
        raise capi.G2pcError(f"no component is kept: the largest of the {components} component(s) has {largest} "
                             f"triangle(s) (min_triangles {min_triangles}, keep_largest {keep_largest})")
    dens = densities.contiguous() if densities is not None else torch.empty((m,), dtype=torch.float64, device=dev)
    vout = torch.empty((mk, 3), dtype=torch.float64, device=dev)
    cout = torch.empty((mk, 3), dtype=torch.uint8, device=dev) if colours is not None else None
    dout = torch.empty((mk,), dtype=torch.float64, device=dev)
    fout = torch.empty((tk, 3), dtype=torch.int32, device=dev)
    capi.call("g2pc_mesh_components_compact", capi.ptr(vpos), capi.ptr(colours), capi.ptr(dens), m, capi.ptr(faces), t,
              capi.ptr(keep), capi.ptr(vout), capi.ptr(cout), capi.ptr(dout), capi.ptr(fout), capi.ptr(ws), ws.numel(),
              st)
    out = (vout, fout, cout, dout if densities is not None else None)
    return (out, {"labels": labels, "keep": keep, "sizes": sizes}) if return_debug else out


def remove_components_mesh(mesh, min_triangles=None, keep_largest=None, stats=None):
    """remove_components() of a Mesh.  Its float32 vertices and normals are carried over unchanged: the kept vertices'
    normals need no recomputation, because a vertex normal reads only the vertex's own faces, and they all stay."""
    check_component_params(min_triangles, keep_largest)
    # The compaction copies float64 words bit for bit, so each vertex's float32 position and normal (24 bytes) travel
    # together as one float64 triple.
    packed = torch.cat([mesh.vertices.to(torch.float32), mesh.normals.to(torch.float32)], 1).contiguous()
    vn, faces, vcol, dens = remove_components(packed.view(torch.float64), mesh.faces.contiguous(), mesh.colours,
                                              mesh.densities, min_triangles, keep_largest, stats=stats)
    vn = vn.view(torch.float32)
    return Mesh(vn[:, :3].contiguous(), faces, vcol, vn[:, 3:].contiguous(), dens)


def filter_components(vpos, faces, vcol, dens, min_triangles, keep_largest, stats, timings, debug):
    """The component filter of a mesher's trimmed mesh when min_triangles or keep_largest is given, else the mesh as it
    is.  debug (a dict or None) receives component_labels."""
    if min_triangles is None and keep_largest is None:
        return vpos, faces, vcol, dens
    with capi.phase(timings, "components"):
        out, cdbg = remove_components(vpos, faces, vcol, dens, min_triangles, keep_largest, stats=stats,
                                      return_debug=True)
    if debug is not None:
        debug["component_labels"] = cdbg["labels"]
    return out


def check_max_hole_edges(max_hole_edges):
    """Refuses a hole length that is not an integer in 3..MAX_HOLE_EDGES (bool included)."""
    x = max_hole_edges
    if isinstance(x, bool) or not isinstance(x, (int, np.integer)) or not 3 <= x <= MAX_HOLE_EDGES:
        raise capi.G2pcError(f"max_hole_edges must be an integer in 3..{MAX_HOLE_EDGES}, got {x!r}")


def fill_holes(vpos, faces, colours=None, densities=None, max_hole_edges=64, stats=None, return_debug=False):
    """Closes the holes of a triangle mesh whose boundary loop has at most max_hole_edges edges (DESIGN.md §2, N12).  A
    half-edge is on the boundary when its undirected edge is used by exactly one face; a boundary set (vertices joined
    by boundary half-edges, labelled by its smallest vertex) is a hole when each of its vertices has exactly one
    outgoing and one incoming boundary half-edge, else it is pinched and stays open.  A hole of 3 edges gets one face
    (unless its three half-edges belong to one face: a lone triangle), a longer one a fan around a new centre vertex
    (the mean position, colour and density of its loop).  Every new face runs the opposite way to its boundary edge.

    vpos (m,3) float64, faces (t,3) int32 (no face uses a vertex twice), colours (m,3) uint8 or None, densities (m,)
    float64 or None, all CUDA; max_hole_edges an integer in 3..1024.  Returns (vpos, faces, colours, densities): the
    input vertices and faces unchanged and in their order, then the centres and the new faces in ascending label order.
    When nothing is filled, the input tensors themselves.

    stats: a dict that receives boundary_edges, holes, filled, too_long, lone_triangles, pinched, added_vertices and
    added_triangles.  return_debug: also a dict with labels (m,) int32 (-1 off the boundary), succ (m,) int32 (the
    target of a vertex's only outgoing boundary half-edge, else -1), lengths (m,) int32 (vertices per label, 0 at an
    index that is no label) and filled (m,) uint8 (per label)."""
    check_max_hole_edges(max_hole_edges)
    for name, x in (("vpos", vpos), ("faces", faces), ("colours", colours), ("densities", densities)):
        if x is not None and not (torch.is_tensor(x) and x.is_cuda):
            raise capi.G2pcError(f"{name} must be a CUDA tensor (the hole filling has no CPU path)")
    if vpos.dim() != 2 or vpos.shape[1] != 3 or vpos.dtype != torch.float64:
        raise capi.G2pcError(f"vpos must be (m, 3) float64, got {tuple(vpos.shape)} {vpos.dtype}")
    if faces.dim() != 2 or faces.shape[1] != 3 or faces.dtype != torch.int32:
        raise capi.G2pcError(f"faces must be (t, 3) int32, got {tuple(faces.shape)} {faces.dtype}")
    m, t, dev = vpos.shape[0], faces.shape[0], vpos.device
    if colours is not None and (colours.shape != (m, 3) or colours.dtype != torch.uint8):
        raise capi.G2pcError(f"colours must be (m, 3) uint8, got {tuple(colours.shape)} {colours.dtype}")
    if densities is not None and (densities.shape != (m,) or densities.dtype != torch.float64):
        raise capi.G2pcError(f"densities must be (m,) float64, got {tuple(densities.shape)} {densities.dtype}")
    if any(x is not None and x.device != dev for x in (faces, colours, densities)):
        raise capi.G2pcError("vpos, faces, colours and densities must be on one device")
    if m >= 2 ** 31 - 1 or 3 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the mesh has {m} vertices and {t} triangles: more than the hole filling's int32 lists "
                             f"(3 half-edges per triangle) can hold")
    if t:
        f = faces.long()
        lo, hi, rep = torch.stack([f.min(), f.max(), ((f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) |
                                                       (f[:, 0] == f[:, 2])).sum()]).tolist()
        del f
        if lo < 0 or hi >= m:
            raise capi.G2pcError(f"face indices must be in 0..{m - 1}, got {lo}..{hi}")
        if rep:
            raise capi.G2pcError(f"{rep} face(s) use a vertex twice")
    st_keys = ("boundary_edges", "holes", "filled", "too_long", "lone_triangles", "pinched", "added_vertices",
               "added_triangles")
    if t == 0:  # no edge, no boundary
        if stats is not None:
            stats.update(dict.fromkeys(st_keys, 0))
        out = (vpos, faces, colours, densities)
        if return_debug:
            return out, {"labels": torch.full((m,), -1, dtype=torch.int32, device=dev),
                         "succ": torch.full((m,), -1, dtype=torch.int32, device=dev),
                         "lengths": torch.zeros((m,), dtype=torch.int32, device=dev),
                         "filled": torch.zeros((m,), dtype=torch.uint8, device=dev)}
        return out
    fcont = faces.contiguous()
    lib = capi.load()
    ws_bytes = lib.g2pc_mesh_holes_workspace_bytes(m, t)
    # labels, succ, lengths, filled and the workspace (sorted edge keys, per-vertex degrees, flags and ranks)
    check_memory(m * (4 + 4 + 4 + 1) + ws_bytes, dev, f"the hole search of {m} vertices and {t} triangles",
                 remedy="fill the holes of a smaller mesh")
    st = capi.stream_ptr(dev)
    labels = torch.empty((m,), dtype=torch.int32, device=dev)
    succ = torch.empty((m,), dtype=torch.int32, device=dev)
    lengths = torch.empty((m,), dtype=torch.int32, device=dev)
    filled = torch.empty((m,), dtype=torch.uint8, device=dev)
    counts = torch.empty((5,), dtype=torch.int64, device=dev)
    ws = capi.workspace(ws_bytes, dev)
    capi.call("g2pc_mesh_holes_find", capi.ptr(fcont), m, t, capi.ptr(labels), capi.ptr(succ), capi.ptr(lengths),
              capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
    boundary, holes, pinched = counts[:3].tolist()
    capi.call("g2pc_mesh_holes_plan", m, t, capi.ptr(labels), capi.ptr(succ), capi.ptr(lengths), int(max_hole_edges),
              capi.ptr(filled), capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
    av, af, nfilled, too_long, lone = counts.tolist()
    if stats is not None:
        stats.update(boundary_edges=boundary, holes=holes, filled=nfilled, too_long=too_long, lone_triangles=lone,
                     pinched=pinched, added_vertices=av, added_triangles=af)
    debug = {"labels": labels, "succ": succ, "lengths": lengths, "filled": filled}
    if nfilled == 0:
        out = (vpos, faces, colours, densities)
        return (out, debug) if return_debug else out
    M, T = m + av, t + af
    if M >= 2 ** 31 - 1 or 3 * T >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the filled mesh would have {M} vertices and {T} triangles: more than int32 lists "
                             f"(3 entries per triangle) can hold")
    check_memory(M * (24 + (3 if colours is not None else 0) + (8 if densities is not None else 0)) + 12 * T, dev,
                 f"the filled mesh of {M} vertices and {T} triangles", remedy="fill the holes of a smaller mesh")
    vcont = vpos.contiguous()
    ccont = colours.contiguous() if colours is not None else None
    dcont = densities.contiguous() if densities is not None else None
    vout = torch.empty((M, 3), dtype=torch.float64, device=dev)
    cout = torch.empty((M, 3), dtype=torch.uint8, device=dev) if colours is not None else None
    dout = torch.empty((M,), dtype=torch.float64, device=dev) if densities is not None else None
    fout = torch.empty((T, 3), dtype=torch.int32, device=dev)
    capi.call("g2pc_mesh_holes_fill", capi.ptr(vcont), capi.ptr(ccont), capi.ptr(dcont), m, capi.ptr(fcont), t,
              capi.ptr(succ), capi.ptr(lengths), capi.ptr(filled), av, af, capi.ptr(vout), capi.ptr(cout),
              capi.ptr(dout), capi.ptr(fout), capi.ptr(ws), ws.numel(), st)
    out = (vout, fout, cout, dout)
    return (out, debug) if return_debug else out


def fill_holes_mesh(mesh, max_hole_edges, stats=None):
    """fill_holes() of a Mesh, its float32 positions taken as float64.  Vertices on no filled loop keep their stored
    normals bit for bit; the vertices of the filled loops and the centres get vertex_normals() of the filled mesh
    (area-weighted).  A mesh with nothing to fill is returned as it is."""
    check_max_hole_edges(max_hole_edges)
    vpos = mesh.vertices.to(torch.float64)
    (p, faces, vcol, dens), dbg = fill_holes(vpos, mesh.faces, mesh.colours, mesh.densities, max_hole_edges,
                                             stats=stats, return_debug=True)
    if p is vpos:
        return mesh
    m = vpos.shape[0]
    labels = dbg["labels"].long()
    on_loop = (labels >= 0) & (dbg["filled"][labels.clamp(min=0)] != 0)
    v, vn = vertex_normals(p, faces)
    normals = torch.cat([torch.where(on_loop[:, None], vn[:m], mesh.normals.to(torch.float32)), vn[m:]])
    return Mesh(v, faces, vcol, normals, dens)


def close_holes(vpos, faces, vcol, dens, max_hole_edges, stats, timings, debug, smoothing):
    """fill_holes() of a mesher's mesh before the smoothing when max_hole_edges is given, else the mesh as it is.
    debug (a dict or None) receives hole_labels.  smoothing: the mesh goes on to g2pc_mesh_smooth, whose one-ring lists
    hold 6 entries per triangle in int32."""
    if max_hole_edges is None:
        return vpos, faces, vcol, dens
    with capi.phase(timings, "holes"):
        out, hdbg = fill_holes(vpos, faces, vcol, dens, max_hole_edges, stats=stats, return_debug=True)
    if debug is not None:
        debug["hole_labels"] = hdbg["labels"]
    t = out[1].shape[0]
    if smoothing and 6 * t >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the filled surface has {t} triangles: the Laplacian smoothing's one-ring lists (6 per "
                             f"triangle) exceed int32; use a smaller depth or laplacian_iters=0")
    return out


def poisson_mesh(points, normals, colours=None, depth=10, laplacian_iters=10, std_ratio=3.0, return_debug=False,
                 timings=None, band_depth=None, band_stats=None, target_triangles=None, min_component_triangles=None,
                 keep_largest_components=None, component_stats=None, max_hole_edges=None, hole_stats=None):
    """Mesh of an oriented point cloud.  points (n,3) float32 CUDA; normals (n,3) float32 / float64 (outward for an
    outward-facing mesh); colours (n,3) in 0..255 or None.  Returns Mesh(vertices (m,3) float32, faces (t,3) int32,
    colours (m,3) uint8 or None, normals (m,3) float32, densities (m,) float64).  With return_debug also a dict: chi
    (R^3 float32, mean-free), iso, B (R^3 int64), frame, cycles, ratio (final |r| / |b|), skipped (points whose normal is
    zero or not finite), keep (vertex trim mask), threshold.  `timings`: a dict that receives CUDA event pairs per phase
    (clean, splat, solve, extract, gather_trim, smooth, normals).

    band_depth: None meshes the dense level `depth`.  An integer in depth + 1 .. 12 adds the narrow-band levels
    depth + 1 .. band_depth (DESIGN.md §2, N6b: bricks of 8^3 nodes around the points, boundary values from the level
    below) and extracts the mesh at band_depth; depth 10 with band_depth 12 is the reference's Poisson depth 12.  Its
    debug dict adds "levels": one dict per band level (depth, frame, map, bricks, B, ghost, chi0, rhs, chi, iterations,
    ratio), and chi / iso are those of band_depth ("dense_chi", "dense_iso" the dense level's); its timings add
    band<D>_bricks, band<D>_splat, band<D>_solve per level.  band_stats: a list that receives one dict per band level
    (depth, bricks, nodes, iterations, ratio: host values), with or without return_debug.

    target_triangles: None keeps every triangle.  An integer >= 1 decimates the smoothed mesh to target_triangles or
    target_triangles - 1 triangles (decimate(), DESIGN.md §2, N9) before the normals are computed; timings add
    "decimate".

    min_component_triangles, keep_largest_components: None and None keep every component.  Otherwise the trimmed mesh
    goes through remove_components() (DESIGN.md §2, N11) before the smoothing; timings add "components", the debug dict
    component_labels (per vertex of the trimmed mesh) and component_stats (a dict) receives remove_components' stats.

    max_hole_edges: None leaves the holes open.  An integer in 3..1024 closes the holes of at most that many edges with
    fill_holes() (DESIGN.md §2, N12) after the component filter and before the smoothing; timings add "holes", the debug
    dict hole_labels (per vertex of the mesh before the fill) and hole_stats (a dict) receives fill_holes' stats."""
    capi.check_cloud(points, normals, colours, what="Poisson meshing")
    if target_triangles is not None:
        check_target(target_triangles)
    check_component_params(min_component_triangles, keep_largest_components, need_one=False)
    if max_hole_edges is not None:
        check_max_hole_edges(max_hole_edges)
    if int(depth) != depth or not DEPTH_MIN <= depth <= DEPTH_MAX:
        raise capi.G2pcError(f"depth must be an integer in {DEPTH_MIN}..{DEPTH_MAX} (the dense int64 right-hand side "
                             f"alone is 69 GB at depth 11), got {depth}")
    if band_depth is not None and (int(band_depth) != band_depth or not depth < band_depth <= BAND_DEPTH_MAX):
        raise capi.G2pcError(f"band_depth must be None or an integer in {int(depth) + 1}..{BAND_DEPTH_MAX}, got "
                             f"{band_depth}")
    if int(laplacian_iters) != laplacian_iters or laplacian_iters < 0:
        raise capi.G2pcError(f"laplacian_iters must be an integer >= 0, got {laplacian_iters}")
    if points.shape[0] == 0:
        raise capi.G2pcError("the point cloud is empty")
    depth, dev = int(depth), points.device
    with capi.phase(timings, "clean"):
        pts, cols, nrm = outliers.remove_statistical_outliers(points, colours, normals, NB_NEIGHBORS, std_ratio)
        pts, nrm = pts.contiguous(), nrm.contiguous()
        cols = cols.contiguous() if cols is not None else None
    if pts.shape[0] == 0:
        raise capi.G2pcError("no point is left after the outlier removal")
    with capi.phase(timings, "splat"):
        frame, B, cell, status = splat(pts, nrm, depth)
        host = torch.cat([frame, status.to(torch.float64)]).tolist()
    extent, skipped, bad = host[6], int(host[FRAME_WORDS]), int(host[FRAME_WORDS + 1])
    if bad:
        raise capi.G2pcError(f"{bad} point(s) have a non-finite coordinate")
    if not extent > 0.0:
        raise capi.G2pcError("the point cloud has zero extent: every point is at the same place")
    if skipped == pts.shape[0]:
        raise capi.G2pcError("no point has a usable normal (all are zero or not finite)")
    with capi.phase(timings, "solve"):
        chi, cycles, ratio = solve(B, frame, depth)
        iso = iso_value(pts, cell, frame, depth, chi)
    if ratio > TOLERANCE:
        warnings.warn(f"the Poisson solve stopped after {cycles} V-cycles at |r| / |b| = {ratio:.2e}, above the "
                      f"{TOLERANCE:g} target: the surface may be displaced", RuntimeWarning, stacklevel=2)
    debug = {}
    if return_debug:
        debug = {"B": B.clone(), "frame": frame, "cycles": cycles, "ratio": ratio, "skipped": skipped}
    if band_depth is not None:
        del B
        dense = {"chi": chi}  # handed over, so that the band levels can free it
        del chi
        return _band_mesh(pts, nrm, cols, cell, frame, dense, iso, depth, int(band_depth), laplacian_iters, debug,
                          return_debug, timings, band_stats, target_triangles,
                          (min_component_triangles, keep_largest_components, component_stats),
                          (max_hole_edges, hole_stats))
    with capi.phase(timings, "extract"):
        # B is dead after the solve: its memory holds the node lists of the extraction and the cell lists of the gather
        vkey, vt, vpos, faces = extract(chi, depth, frame, iso, B)
    if vkey.shape[0] == 0:
        raise capi.G2pcError("no surface: the indicator function does not cross its iso-value")
    with capi.phase(timings, "gather_trim"):
        dens, vcol = gather(pts, cols.to(torch.int32) if cols is not None else None, cell, frame, depth, vkey, vt, B)
        dens, vpos, vcol, faces, keep, thr = trim(dens, vpos, vcol, faces)
    vpos, faces, vcol, dens = filter_components(vpos, faces, vcol, dens, min_component_triangles,
                                                 keep_largest_components, component_stats, timings,
                                                 debug if return_debug else None)
    vpos, faces, vcol, dens = close_holes(vpos, faces, vcol, dens, max_hole_edges, hole_stats, timings,
                                          debug if return_debug else None, smoothing=laplacian_iters > 0)
    with capi.phase(timings, "smooth"):
        smooth(vpos, faces, laplacian_iters)
    smoothed = vpos
    if target_triangles is not None:
        with capi.phase(timings, "decimate"):
            vpos, faces, vcol, dens = decimate(vpos, faces, target_triangles, vcol, dens)
    with capi.phase(timings, "normals"):
        v, vn = vertex_normals(vpos, faces)
    out = Mesh(v, faces, vcol, vn, dens)
    if return_debug:
        debug.update(chi=chi, iso=iso, keep=keep, threshold=thr, vkey=vkey, vpos_smoothed=smoothed)
        return out, debug
    return out


def _band_mesh(pts, nrm, cols, cell, frame, dense, iso, depth, band_depth, laplacian_iters, debug, return_debug,
               timings, band_stats, target_triangles, components, holes):
    """The band levels depth + 1 .. band_depth after the dense solve, then the mesh at band_depth.  dense: {"chi": the
    dense level's chi}, emptied here.  components: poisson_mesh's (min_component_triangles, keep_largest_components,
    component_stats); holes: its (max_hole_edges, hole_stats)."""
    dev = pts.device
    parent_chi, parent_map = dense.pop("chi"), None
    if return_debug:
        debug.update(dense_chi=parent_chi, dense_iso=iso, levels=[])
    for D in range(depth + 1, band_depth + 1):
        with capi.phase(timings, f"band{D}_bricks"):
            bframe, bmap, blist, lost = band_bricks(pts, cell, frame, D, parent_map)
        k = blist.shape[0]
        if lost:
            raise capi.G2pcError(f"{lost} seed brick(s) at depth {D} are not nested in the level below")
        if k == (1 << (D - 3)) ** 3:
            raise capi.G2pcError(f"the band at depth {D} covers the whole grid (no boundary): mesh at a dense depth "
                                 f"of at least {D} instead")
        check_memory(k * BRICK ** 3 * (BAND_DEBUG_BYTES_PER_NODE if return_debug else BAND_BYTES_PER_NODE), dev,
                     f"the band at depth {D} ({k} bricks, {k * BRICK ** 3} nodes)")
        with capi.phase(timings, f"band{D}_splat"):
            B, status = band_splat(pts, nrm, cell, bframe, D, bmap, k)
            ghost, bchi, rhs = band_ghosts(parent_chi, parent_map, D, bmap, blist, B, bframe, with_ghosts=return_debug)
        outside = int(status.item())
        if outside:
            raise capi.G2pcError(f"{outside} splat term(s) at depth {D} fall outside the band")
        parent_chi = parent_map = None  # the level below is dead once the ghosts are known
        level = {"depth": D, "frame": bframe, "map": bmap, "bricks": blist}
        if return_debug:
            level.update(B=B, ghost=ghost, chi0=bchi.clone(), rhs=rhs)
        del B, ghost
        with capi.phase(timings, f"band{D}_solve"):
            its, ratio = band_solve(rhs, bchi, D, bmap, blist)
        del rhs
        if ratio > BAND_TOLERANCE:
            warnings.warn(f"the band solve at depth {D} stopped after {its} iterations at |r| / |b| = {ratio:.2e}, "
                          f"above the {BAND_TOLERANCE:g} target: the surface may be displaced", RuntimeWarning,
                          stacklevel=3)
        level.update(chi=bchi, iterations=its, ratio=ratio, nodes=k * BRICK ** 3)
        if band_stats is not None:
            band_stats.append({"depth": D, "bricks": k, "nodes": k * BRICK ** 3, "iterations": its, "ratio": ratio})
        if return_debug:
            debug["levels"].append(level)
        parent_chi, parent_map = bchi, bmap
    with capi.phase(timings, "extract"):
        biso = band_iso(pts, cell, bframe, band_depth, bmap, bchi)
        vkey, vt, vpos, faces = band_extract(bchi, band_depth, bmap, blist, bframe, biso,
                                             smoothing=laplacian_iters > 0)
    if vkey.shape[0] == 0:
        raise capi.G2pcError("no surface: the indicator function does not cross its iso-value in the band")
    if not return_debug:
        del bchi, bmap, blist, parent_chi, parent_map
    with capi.phase(timings, "gather_trim"):
        dens, vcol = band_gather(pts, cols.to(torch.int32) if cols is not None else None, cell, bframe, band_depth,
                                 vkey, vt)
        dens, vpos, vcol, faces, keep, thr = trim(dens, vpos, vcol, faces)
    vpos, faces, vcol, dens = filter_components(vpos, faces, vcol, dens, *components, timings,
                                                 debug if return_debug else None)
    vpos, faces, vcol, dens = close_holes(vpos, faces, vcol, dens, *holes, timings, debug if return_debug else None,
                                          smoothing=laplacian_iters > 0)
    with capi.phase(timings, "smooth"):
        smooth(vpos, faces, laplacian_iters)
    smoothed = vpos
    if target_triangles is not None:
        with capi.phase(timings, "decimate"):
            vpos, faces, vcol, dens = decimate(vpos, faces, target_triangles, vcol, dens)
    with capi.phase(timings, "normals"):
        v, vn = vertex_normals(vpos, faces)
    out = Mesh(v, faces, vcol, vn, dens)
    if return_debug:
        debug.update(chi=bchi, iso=biso, keep=keep, threshold=thr, vkey=vkey, vpos_smoothed=smoothed, cell=cell,
                     points=pts, normals=nrm, colours=cols)
        return out, debug
    return out


def write_mesh_ply(path, mesh):
    """Binary little-endian PLY: vertices `float x y z nx ny nz` + `uchar red green blue` (255 when the mesh has no
    colours), faces `list uchar int vertex_indices`."""
    v = mesh.vertices.detach().cpu().numpy().astype("<f4")
    n = mesh.normals.detach().cpu().numpy().astype("<f4")
    m = v.shape[0]
    c = mesh.colours.detach().cpu().numpy().astype(np.uint8) if mesh.colours is not None else np.full((m, 3), 255,
                                                                                                       np.uint8)
    f = mesh.faces.detach().cpu().numpy().astype("<i4")
    vrec = np.empty(m, dtype=[("p", "<f4", 3), ("n", "<f4", 3), ("c", "u1", 3)])
    vrec["p"], vrec["n"], vrec["c"] = v, n, c
    frec = np.empty(f.shape[0], dtype=[("k", "u1"), ("i", "<i4", 3)])
    frec["k"], frec["i"] = 3, f
    header = ("ply\nformat binary_little_endian 1.0\n"
              f"element vertex {m}\nproperty float x\nproperty float y\nproperty float z\n"
              "property float nx\nproperty float ny\nproperty float nz\n"
              "property uchar red\nproperty uchar green\nproperty uchar blue\n"
              f"element face {f.shape[0]}\nproperty list uchar int vertex_indices\nend_header\n")
    with open(path, "wb") as fh:
        fh.write(header.encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())


def read_mesh_ply(path):
    """(vertices (m,3) f32, normals (m,3) f32, colours (m,3) u8, faces (t,3) i32) of a file written by write_mesh_ply."""
    with open(path, "rb") as fh:
        lines = []
        while True:
            line = fh.readline()
            if not line:
                raise ValueError(f"{path}: unterminated PLY header")
            lines.append(line.decode("ascii").strip())
            if lines[-1] == "end_header":
                break
        counts = {t[1]: int(t[2]) for t in (ln.split() for ln in lines) if t and t[0] == "element"}
        if "format binary_little_endian 1.0" not in lines:
            raise ValueError(f"{path}: not a binary little-endian PLY")
        m, t = counts.get("vertex", 0), counts.get("face", 0)
        vrec = np.frombuffer(fh.read(27 * m), dtype=[("p", "<f4", 3), ("n", "<f4", 3), ("c", "u1", 3)], count=m)
        frec = np.frombuffer(fh.read(13 * t), dtype=[("k", "u1"), ("i", "<i4", 3)], count=t)
    if t and not (frec["k"] == 3).all():
        raise ValueError(f"{path}: a face is not a triangle")
    return vrec["p"].copy(), vrec["n"].copy(), vrec["c"].copy(), frec["i"].copy()
