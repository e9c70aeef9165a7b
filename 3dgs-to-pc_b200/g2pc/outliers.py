"""Statistical outlier removal of a point cloud on the device (--clean_pointcloud).

The reference cleans the finished cloud with Open3D's remove_statistical_outlier(nb_neighbors=20, std_ratio)
(mesh_handler.py:89-94).  Here: g2pc_knn_mean_dist (exact k-nearest-neighbour mean distances), g2pc_sor_mask (cloud
statistics and keep rule), then the existing compaction, g2pc_cull_select with the keep mask as its extra mask and
g2pc_gather_rows.  One host read: the kept count and the non-finite-point count, together.
"""
import torch

from . import capi

K_MAX = 32  # G2PC_SOR_K_MAX in include/g2pc.h


def mean_distances(xyz, k):
    """avg (n,) float64: mean distance of every point to its k nearest points (itself included), and the device int32
    count of points with a non-finite coordinate."""
    n = xyz.shape[0]
    avg = torch.empty((n,), dtype=torch.float64, device=xyz.device)
    status = torch.empty((1,), dtype=torch.int32, device=xyz.device)
    ws = capi.workspace(capi.load().g2pc_knn_workspace_bytes(n), xyz.device)
    capi.call("g2pc_knn_mean_dist", capi.ptr(xyz), n, int(k), capi.ptr(avg), capi.ptr(status), capi.ptr(ws),
              ws.numel(), capi.stream_ptr(xyz.device))
    return avg, status


def sor_mask(avg, std_ratio):
    """keep (n,) uint8 and stats (3,) float64 = (mean, std, threshold) of the per-point mean distances."""
    n = avg.shape[0]
    keep = torch.empty((n,), dtype=torch.uint8, device=avg.device)
    stats = torch.full((3,), float("nan"), dtype=torch.float64, device=avg.device)
    ws = capi.workspace(capi.load().g2pc_sor_workspace_bytes(n), avg.device)
    capi.call("g2pc_sor_mask", capi.ptr(avg), n, float(std_ratio), capi.ptr(keep), capi.ptr(stats), capi.ptr(ws),
              ws.numel(), capi.stream_ptr(avg.device))
    return keep, stats


def remove_statistical_outliers(points, colours, normals, nb_neighbors=20, std_ratio=10.0, return_debug=False):
    """Keep point i iff 0 < avg[i] < mean + std_ratio * std (Open3D's rule).  points (n,3) float32 CUDA; colours (n,3)
    or None, returned as clamp(colours, 0, 255) truncated to int32 like the reference's Open3D round trip; normals (n,3)
    or None (None stays None).  The kept rows keep their order.  With return_debug, also returns
    {"avg", "keep", "stats"}."""
    capi.check_cloud(points, normals, colours)
    k = int(nb_neighbors)
    if not 1 <= k <= K_MAX:
        raise capi.G2pcError(f"nb_neighbors must be in 1..{K_MAX}, got {nb_neighbors}")
    if not float(std_ratio) > 0.0:
        raise capi.G2pcError(f"std_ratio must be > 0, got {std_ratio}")
    n, dev = points.shape[0], points.device
    if colours is not None:
        colours = torch.clamp(colours, min=0, max=255).to(torch.int32)  # mesh_handler.py:45 of the reference
    xyz = points.contiguous()
    avg, status = mean_distances(xyz, k)
    keep, stats = sor_mask(avg, std_ratio)

    index = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
    count = torch.zeros((1,), dtype=torch.int64, device=dev)
    ws = capi.workspace(capi.load().g2pc_cull_workspace_bytes(n), dev)
    st = capi.stream_ptr(dev)
    capi.call("g2pc_cull_select", None, 0.0, None, 0.0, None, None, None, None, None, capi.ptr(keep), 0, n, n,
              capi.ptr(index), capi.ptr(count), capi.ptr(ws), ws.numel(), st)
    m, bad = torch.cat([count, status.to(torch.int64)]).tolist()  # the one host read
    if bad:
        raise capi.G2pcError(f"{bad} point(s) have a non-finite coordinate; the outlier statistics are undefined")
    it = iter(capi.gather_rows(index, m, [t for t in (xyz, colours, normals) if t is not None]))
    out = tuple(next(it) if t is not None else None for t in (xyz, colours, normals))
    if return_debug:
        return out + ({"avg": avg, "keep": keep, "stats": stats},)
    return out
