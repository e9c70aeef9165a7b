"""Poisson mesh of an oriented point cloud on the device (N6): the reference's mesh_handler.generate_mesh
(mesh_handler.py:23-40: Open3D outlier removal, Poisson reconstruction, 10 % density trim, Laplacian smoothing) with
this project's own rules, written down in DESIGN.md §2 and restated in float64 by tests/f64ref_mesh.py.

Steps: statistical outlier removal (g2pc/outliers.py) -> g2pc_mesh_splat -> g2pc_mesh_vcycle until |r| <= 1e-5 |b| or 40
cycles -> g2pc_mesh_iso -> g2pc_mesh_extract_count / _emit (marching tetrahedra) -> g2pc_mesh_gather (density, colour)
-> g2pc_mesh_trim -> g2pc_mesh_smooth -> g2pc_mesh_normals.  Host reads: the frame and skip counts after the splat, the
residual once per cycle, the vertex / triangle counts before and after the trim.
"""
import collections
import math
import warnings

import numpy as np
import torch

from . import capi, outliers

DEPTH_MIN, DEPTH_MAX = 2, 10  # G2PC_MESH_DEPTH_MAX in include/g2pc.h
FRAME_WORDS = 8
MAX_CYCLES = 40
TOLERANCE = 1e-5
NB_NEIGHBORS = 20

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


def poisson_mesh(points, normals, colours=None, depth=10, laplacian_iters=10, std_ratio=3.0, return_debug=False,
                 timings=None):
    """Mesh of an oriented point cloud.  points (n,3) float32 CUDA; normals (n,3) float32 / float64 (outward for an
    outward-facing mesh); colours (n,3) in 0..255 or None.  Returns Mesh(vertices (m,3) float32, faces (t,3) int32,
    colours (m,3) uint8 or None, normals (m,3) float32, densities (m,) float64).  With return_debug also a dict: chi
    (R^3 float32, mean-free), iso, B (R^3 int64), frame, cycles, ratio (final |r| / |b|), skipped (points whose normal is
    zero or not finite), keep (vertex trim mask), threshold.  `timings`: a dict that receives CUDA event pairs per phase
    (clean, splat, solve, extract, gather_trim, smooth, normals)."""
    capi.check_cloud(points, normals, colours, what="Poisson meshing")
    if int(depth) != depth or not DEPTH_MIN <= depth <= DEPTH_MAX:
        raise capi.G2pcError(f"depth must be an integer in {DEPTH_MIN}..{DEPTH_MAX} (the dense int64 right-hand side "
                             f"alone is 69 GB at depth 11), got {depth}")
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
    with capi.phase(timings, "extract"):
        # B is dead after the solve: its memory holds the node lists of the extraction and the cell lists of the gather
        vkey, vt, vpos, faces = extract(chi, depth, frame, iso, B)
    if vkey.shape[0] == 0:
        raise capi.G2pcError("no surface: the indicator function does not cross its iso-value")
    with capi.phase(timings, "gather_trim"):
        dens, vcol = gather(pts, cols.to(torch.int32) if cols is not None else None, cell, frame, depth, vkey, vt, B)
        dens, vpos, vcol, faces, keep, thr = trim(dens, vpos, vcol, faces)
    with capi.phase(timings, "smooth"):
        smooth(vpos, faces, laplacian_iters)
    with capi.phase(timings, "normals"):
        v, vn = vertex_normals(vpos, faces)
    out = Mesh(v, faces, vcol, vn, dens)
    if return_debug:
        debug.update(chi=chi, iso=iso, keep=keep, threshold=thr, vkey=vkey, vpos_smoothed=vpos)
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
