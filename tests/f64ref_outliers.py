"""Plain float64 restatement of Open3D's statistical outlier removal (PointCloud::RemoveStatisticalOutliers, behind
the reference's mesh_handler.clean_point_cloud): the yardstick of the --clean_pointcloud kernels.  Inputs are the
float32 coordinates the kernels see, upcast; sums run in the sequential order of Open3D's std::accumulate."""
import math

import numpy as np


def knn_mean_distances(xyz, k, query=None):
    """Open3D's per-point mean distance (RemoveStatisticalOutliers): for each query row i, the k' = min(k, n) smallest
    d2 = (dx*dx + dy*dy) + dz*dz over all points j (i itself included), dx = x_i - x_j in float64 of the float32
    coordinates, then (sqrt(d2_0) + sqrt(d2_1) + ...) / k' summed left to right in ascending order.  Candidates come
    from a cKDTree queried with k + 8 and are re-ranked on d2 recomputed as above (only the multiset of the k smallest
    values matters, so ties at the k-th slot are harmless).  query: row indices (default: every row)."""
    from scipy.spatial import cKDTree
    p = np.asarray(xyz, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    n = p.shape[0]
    rows = np.arange(n) if query is None else np.asarray(query, dtype=np.int64)
    if n == 0 or rows.size == 0:
        return np.zeros(rows.size)
    kp, kq = min(k, n), min(k + 8, n)
    _, nb = cKDTree(p).query(p[rows], k=kq, workers=-1)
    nb = np.asarray(nb).reshape(rows.size, kq)
    return _mean_of_smallest(p[rows], p[nb], kp)


def _mean_of_smallest(q, cand, kp):
    d = q[:, None, :] - cand
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    d2.sort(axis=1)
    s = np.sqrt(d2[:, :kp])
    acc = np.zeros(q.shape[0])
    for j in range(kp):  # left to right per row, as std::accumulate
        acc = acc + s[:, j]
    return acc / kp


def knn_mean_distances_brute(xyz, k):
    """The same quantity from all pairs (small clouds only): the pin of knn_mean_distances."""
    p = np.asarray(xyz, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    n = p.shape[0]
    if n == 0:
        return np.zeros(0)
    return _mean_of_smallest(p, np.broadcast_to(p[None], (n, n, 3)), min(k, n))


def sor_statistics(avg, std_ratio):
    """(mean, std, threshold) of Open3D's rule: plain sequential sums over avg > 0, divided by the count of points that
    have a neighbour (n), Bessel's correction; NaN where Open3D divides 0 by 0."""
    vals = [float(v) for v in np.asarray(avg, dtype=np.float64)]
    n = len(vals)
    if n == 0:
        return math.nan, math.nan, math.nan
    total = 0.0
    for v in vals:
        if v > 0:
            total += v
    mean = total / n
    sq = 0.0
    for v in vals:
        if v > 0:
            sq += (v - mean) * (v - mean)
    std = math.sqrt(sq / (n - 1)) if n > 1 else math.nan
    return mean, std, mean + std_ratio * std


def sor_keep(avg, threshold):
    avg = np.asarray(avg, dtype=np.float64)
    return (avg > 0) & (avg < threshold)


def statistical_outliers(xyz, k, std_ratio):
    """Open3D's remove_statistical_outlier(nb_neighbors=k, std_ratio) restated.
    Returns (avg, keep mask, (mean, std, threshold))."""
    avg = knn_mean_distances(xyz, k)
    stats = sor_statistics(avg, std_ratio)
    return avg, sor_keep(avg, stats[2]), stats
