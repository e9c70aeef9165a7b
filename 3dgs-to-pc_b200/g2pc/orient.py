"""Consistent orientation of point-cloud normals on the device (N7): Hoppe et al. 1992, the rule behind Open3D's
orient_normals_consistent_tangent_plane, with this project's own rules (DESIGN.md §2), restated in float64 by
tests/f64ref_orient.py.

Steps: g2pc_orient_prepare (usable points, unit normals) -> g2pc_knn_ids (k nearest other points) -> g2pc_orient_edges
(undirected k-NN edges, keys, flip bits) -> g2pc_orient_round until a round hooks nothing (Borůvka with sign parity) ->
g2pc_orient_finish (seed per component, flips, output).  Host reads: the usable count after the prepare, the two round
counts once per round, the stats at the end.

face_cameras turns the normals of Gaussians toward the camera that saw each one best (g2pc_face_cameras, one pass, no
neighbour graph); gauss_to_mesh.py orients its surface cloud that way.
"""
import collections

import torch

from . import capi

K_MAX = 31  # G2PC_ORIENT_K_MAX in include/g2pc.h
K_DEFAULT = 10

OrientStats = collections.namedtuple("OrientStats", ["components", "flipped", "skipped", "rounds"])
FaceCameraStats = collections.namedtuple("FaceCameraStats", ["flipped", "unseen", "undecided", "invalid"])


def knn_ids(xyz, k):
    """ids (n,k) int32 and d2 (n,k) float64: the k' = min(k, n - 1) nearest other points of every row by ascending (d2,
    id), then id -1 / d2 inf; and the device int32 count of rows with a non-finite coordinate."""
    n, dev = xyz.shape[0], xyz.device
    ids = torch.empty((n, k), dtype=torch.int32, device=dev)
    d2 = torch.empty((n, k), dtype=torch.float64, device=dev)
    status = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = capi.workspace(capi.load().g2pc_knn_workspace_bytes(n), dev)
    capi.call("g2pc_knn_ids", capi.ptr(xyz), n, int(k), capi.ptr(ids), capi.ptr(d2), capi.ptr(status), capi.ptr(ws),
              ws.numel(), capi.stream_ptr(dev))
    return ids, d2, status


def orient_normals(points, normals, k=K_DEFAULT, return_debug=False, timings=None):
    """Normals with a consistent sign.  points (n,3) float32 CUDA; normals (n,3) float32 / float64 CUDA (not modified).
    Returns (oriented normals: the input's dtype, values and magnitudes, with the sign of every flipped row negated;
    OrientStats(components, flipped, skipped, rounds)).  A point is used when its coordinate is finite and its normal
    finite and non-zero; the others (`skipped`) are returned unchanged.  With return_debug also a dict over the m usable
    points, in row order: rows (m,) int64 (their row in the input), ids (m,k) int32 and d2 (m,k) float64 (neighbours as
    usable-point indices), edges (E,2) int64 (the k-NN graph's edges, ascending), mst (m - components,) int64 (the
    spanning forest's edge numbers, ascending), rel (m,) uint8 (flip parity to the component's seed), seed (m,) int32
    (the seed of each point's component).  `timings`: a dict that receives CUDA event pairs per phase (prepare, knn,
    edges, rounds, finish)."""
    capi.check_cloud(points, normals, what="orienting normals")
    if isinstance(k, bool) or int(k) != k or not 1 <= k <= K_MAX:
        raise capi.G2pcError(f"k must be an integer in 1..{K_MAX}, got {k}")
    k, dev, n = int(k), points.device, points.shape[0]
    pts, nrm = points.contiguous(), normals.contiguous()
    lib, st = capi.load(), capi.stream_ptr(dev)
    with capi.phase(timings, "prepare"):
        rows = torch.empty((n,), dtype=torch.int32, device=dev)
        uxyz = torch.empty((n, 3), dtype=torch.float32, device=dev)
        unh = torch.empty((n, 3), dtype=torch.float64, device=dev)
        count = torch.empty((1,), dtype=torch.int64, device=dev)
        ws = capi.workspace(lib.g2pc_orient_prepare_workspace_bytes(n), dev)
        capi.call("g2pc_orient_prepare", capi.ptr(pts), capi.ptr(nrm), capi.dtype_code(nrm), n, capi.ptr(rows),
                  capi.ptr(uxyz), capi.ptr(unh), capi.ptr(count), capi.ptr(ws), ws.numel(), st)
        del ws
        m = int(count.item())
    with capi.phase(timings, "knn"):
        ids, d2, _ = knn_ids(uxyz[:m], k) if m else (torch.empty((0, k), dtype=torch.int32, device=dev),
                                                     torch.empty((0, k), dtype=torch.float64, device=dev), None)
    kp = min(k, m - 1) if m > 1 else 0
    c = m * kp
    with capi.phase(timings, "edges"):
        edges = torch.empty((max(c, 1),), dtype=torch.int64, device=dev)
        keys = torch.empty((max(c, 1),), dtype=torch.int64, device=dev)
        flips = torch.empty((max(c, 1),), dtype=torch.uint8, device=dev)
        ecount = torch.zeros((1,), dtype=torch.int64, device=dev)
        if c:
            ws = capi.workspace(lib.g2pc_orient_edges_workspace_bytes(m, k), dev)
            capi.call("g2pc_orient_edges", capi.ptr(ids), m, k, capi.ptr(unh), capi.ptr(edges), capi.ptr(keys),
                      capi.ptr(flips), capi.ptr(ecount), capi.ptr(ws), ws.numel(), st)
            del ws
    comp = torch.empty((max(m, 1),), dtype=torch.int32, device=dev)
    rel = torch.empty((max(m, 1),), dtype=torch.uint8, device=dev)
    mst = torch.empty((max(c, 1),), dtype=torch.uint8, device=dev)
    rounds = 0
    with capi.phase(timings, "rounds"):
        if m:
            counts = torch.empty((2,), dtype=torch.int64, device=dev)
            ws = capi.workspace(lib.g2pc_orient_round_workspace_bytes(m, c), dev)
            active = c
            while True:
                capi.call("g2pc_orient_round", capi.ptr(edges), capi.ptr(keys), capi.ptr(flips), m, c, rounds, active,
                          capi.ptr(comp), capi.ptr(rel), capi.ptr(mst), capi.ptr(counts), capi.ptr(ws), ws.numel(), st)
                rounds += 1
                hooked, active = counts.tolist()  # the one host read of a round
                if hooked == 0 or active == 0:
                    break
            del ws
    with capi.phase(timings, "finish"):
        out = torch.empty_like(nrm)
        seed = torch.empty((max(m, 1),), dtype=torch.int32, device=dev) if return_debug else None
        srel = torch.empty((max(m, 1),), dtype=torch.uint8, device=dev) if return_debug else None
        stats = torch.empty((2,), dtype=torch.int64, device=dev)
        ws = capi.workspace(lib.g2pc_orient_finish_workspace_bytes(m), dev)
        capi.call("g2pc_orient_finish", capi.ptr(uxyz), capi.ptr(unh), capi.ptr(rows), m, capi.ptr(nrm),
                  capi.dtype_code(nrm), n, capi.ptr(comp), capi.ptr(rel), capi.ptr(out), capi.ptr(seed), capi.ptr(srel),
                  capi.ptr(stats), capi.ptr(ws), ws.numel(), st)
        components, flipped = stats.tolist()
    info = OrientStats(components, flipped, n - m, rounds)
    if not return_debug:
        return out, info
    E = int(ecount.item())
    e = edges[:E]
    debug = {"rows": rows[:m].to(torch.int64), "ids": ids, "d2": d2,
             "edges": torch.stack([e >> 32, e & 0xFFFFFFFF], 1),
             "mst": torch.nonzero(mst[:E]).flatten(), "rel": srel[:m], "seed": seed[:m]}
    return out, info, debug


def face_cameras(means, normals, ids, cam_of, cam_centres):
    """Normals turned toward the camera that gave each Gaussian its maximum contribution (rules in DESIGN.md §2).

    means (m,3) float32 and normals (m,3) float32 / float64 (not modified) of m Gaussians; ids (m,) int32: the original
    row of each (Gaussians.ids); cam_of (N,) int32: the colour stage's first_frame over the original rows, INT32_MAX
    where no camera raised a maximum; cam_centres (ncam,3) float32 in camera-index order; all CUDA tensors.  Returns
    (normals: the input's dtype and values, with every row whose normal points away from its camera negated,
    FaceCameraStats(flipped, unseen, undecided, invalid)).  Unseen rows (no camera) and undecided rows (normal
    perpendicular to the view direction, or not finite) keep their sign.  Raises G2pcError when a row's id or camera index
    is out of range."""
    capi.check_cloud(means, normals, what="turning normals toward the cameras")
    capi.require_cuda(ids, cam_of, cam_centres)
    m, dev = means.shape[0], means.device
    if ids is None or ids.dtype != torch.int32 or tuple(ids.shape) != (m,):
        raise capi.G2pcError(f"ids must be ({m},) int32 like the means")
    if cam_of is None or cam_of.dtype != torch.int32 or cam_of.dim() != 1:
        raise capi.G2pcError("cam_of must be a 1-D int32 tensor")
    if cam_centres is None or cam_centres.dtype != torch.float32 or cam_centres.dim() != 2 or cam_centres.shape[1] != 3:
        raise capi.G2pcError("cam_centres must be (ncam, 3) float32")
    if len({str(t.device) for t in (means, ids, cam_of, cam_centres)}) > 1:
        raise capi.G2pcError("means, ids, cam_of and cam_centres are on different devices")
    nrm = normals.contiguous()
    out = torch.empty_like(nrm)
    counts = torch.zeros((4,), dtype=torch.int64, device=dev)
    if m:
        capi.call("g2pc_face_cameras", capi.ptr(means.contiguous()), capi.ptr(nrm), capi.dtype_code(nrm),
                  capi.ptr(ids.contiguous()), m, capi.ptr(cam_of.contiguous()), cam_of.shape[0],
                  capi.ptr(cam_centres.contiguous()), cam_centres.shape[0], capi.ptr(out), capi.ptr(counts),
                  capi.stream_ptr(dev))
    stats = FaceCameraStats(*counts.tolist())
    if stats.invalid:
        raise capi.G2pcError(f"{stats.invalid} row(s) have a Gaussian id outside [0, {cam_of.shape[0]}) or a camera index "
                             f"outside [0, {cam_centres.shape[0]})")
    return out, stats
