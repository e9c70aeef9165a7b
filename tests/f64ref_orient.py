"""Plain float64 restatement of the normal orientation (N7, g2pc/orient.py; rules in DESIGN.md §2): the yardstick of
g2pc_knn_ids and the s11_orient.cu kernels.  Neighbours by a cKDTree re-ranked on the exact d2, edges and keys in numpy,
Kruskal with union-find on the keys, rel by breadth-first search from each component's seed."""
import collections

import numpy as np

import f64ref_mesh


def _d2(q, c):
    d = q[:, None, :] - c
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def _rank(p, rows, cand, k):
    """ids (len(rows), k) int32 and d2 float64 of the k' smallest (d2, j) over the candidate lists (j != row, -1 pads)."""
    n = p.shape[0]
    kp = min(k, n - 1)
    ids = np.full((rows.size, k), -1, np.int32)
    d2 = np.full((rows.size, k), np.inf)
    for r, (i, c) in enumerate(zip(rows, cand)):
        c = np.unique(np.asarray(c, np.int64))
        c = c[(c != i) & (c >= 0) & (c < n)]
        d = _d2(p[i][None], p[c])[0]
        o = np.lexsort((c, d))[:kp]
        ids[r, :o.size], d2[r, :o.size] = c[o], d[o]
    return ids, d2


def knn_ids(xyz, k, query=None):
    """The k' = min(k, n - 1) nearest other points of every query row by ascending (d2, j), d2 = (dx*dx + dy*dy) + dz*dz
    in float64 of the float32 coordinates; slots k'.. hold -1 / inf.  Candidates: every point within the distance of a
    cKDTree's k'-th neighbour (with a relative slack), so every tie at the k-th slot is among them."""
    from scipy.spatial import cKDTree
    p = np.asarray(xyz, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    n = p.shape[0]
    rows = np.arange(n) if query is None else np.asarray(query, dtype=np.int64)
    if n <= 1 or rows.size == 0:
        return np.full((rows.size, k), -1, np.int32), np.full((rows.size, k), np.inf)
    kq = min(k + 1, n)
    tree = cKDTree(p)
    dist, _ = tree.query(p[rows], k=kq, workers=-1)
    r = np.asarray(dist).reshape(rows.size, kq)[:, -1]
    cand = tree.query_ball_point(p[rows], r * (1 + 1e-9) + 1e-300, workers=-1)
    return _rank(p, rows, cand, k)


def knn_ids_brute(xyz, k):
    """The same lists from all pairs (small clouds only): the pin of knn_ids."""
    p = np.asarray(xyz, dtype=np.float32).astype(np.float64).reshape(-1, 3)
    n = p.shape[0]
    if n <= 1:
        return np.full((n, k), -1, np.int32), np.full((n, k), np.inf)
    return _rank(p, np.arange(n), [np.arange(n)] * n, k)


def edges_and_keys(ids, nh):
    """edges (E,2) int64 ascending by (min, max), keys (E,) uint64, weights (E,) float32, flips (E,) bool."""
    ids = np.asarray(ids, np.int64)
    m = ids.shape[0]
    i = np.repeat(np.arange(m), ids.shape[1])
    j = ids.reshape(-1)
    ok = j >= 0
    a, b = np.minimum(i[ok], j[ok]), np.maximum(i[ok], j[ok])
    packed = np.unique(a << 32 | b)
    edges = np.stack([packed >> 32, packed & 0xFFFFFFFF], 1)
    u, v = nh[edges[:, 0]], nh[edges[:, 1]]
    dot = (u[:, 0] * v[:, 0] + u[:, 1] * v[:, 1]) + u[:, 2] * v[:, 2]
    w = np.maximum(0.0, 1.0 - np.abs(dot)).astype(np.float32)
    keys = w.view(np.uint32).astype(np.uint64) << np.uint64(32) | np.arange(edges.shape[0], dtype=np.uint64)
    return edges, keys, w, dot < 0


def kruskal(m, edges, keys):
    """Edge numbers of the minimum spanning forest on the (unique) keys, ascending, and the component root of every
    point (union-find)."""
    parent = list(range(m))

    def find(x):
        while parent[x] != x:
            parent[x] = parent[parent[x]]
            x = parent[x]
        return x

    chosen = []
    for e in np.argsort(keys, kind="stable"):
        a, b = find(int(edges[e, 0])), find(int(edges[e, 1]))
        if a != b:
            parent[max(a, b)] = min(a, b)
            chosen.append(int(e))
    return np.sort(np.asarray(chosen, np.int64)), np.array([find(x) for x in range(m)], np.int64)


def seeds_and_rel(xyz, m, edges, flips, mst, root):
    """seed (m,) of every point's component (largest z, then smallest index) and rel (m,) uint8: XOR of the flip bits
    along the forest path to that seed (breadth-first search from it)."""
    z = np.asarray(xyz, np.float32)[:, 2].astype(np.float64)
    order = np.lexsort((np.arange(m), -z))  # largest z first, then smallest index
    seed_of_root = {}
    for v in order:
        seed_of_root.setdefault(int(root[v]), int(v))
    seed = np.array([seed_of_root[int(r)] for r in root], np.int64)
    adj = collections.defaultdict(list)
    for e in mst:
        a, b = int(edges[e, 0]), int(edges[e, 1])
        adj[a].append((b, int(flips[e])))
        adj[b].append((a, int(flips[e])))
    rel = np.zeros(m, np.uint8)
    for s in set(seed_of_root.values()):
        queue = collections.deque([s])
        seen = {s}
        while queue:
            x = queue.popleft()
            for y, f in adj[x]:
                if y not in seen:
                    seen.add(y)
                    rel[y] = rel[x] ^ f
                    queue.append(y)
    return seed, rel


def orient(points, normals, k=10, brute=False):
    """The whole rule.  Returns (oriented normals: the input with the flipped rows negated, dict of rows, ids, d2, edges,
    keys, weights, flips, mst, seed, rel, flip, components, skipped)."""
    p = np.asarray(points, np.float32)
    nrm = np.asarray(normals)
    ok, nh_all = f64ref_mesh.usable_normals(nrm)
    ok &= np.isfinite(p).all(1)
    rows = np.nonzero(ok)[0]
    up, nh = p[rows], nh_all[rows]
    m = rows.size
    ids, d2 = (knn_ids_brute if brute else knn_ids)(up, k)
    edges, keys, w, flips = edges_and_keys(ids, nh) if m else (np.zeros((0, 2), np.int64),) + (np.zeros(0),) * 3
    mst, root = kruskal(m, edges, keys)
    seed, rel = seeds_and_rel(up, m, edges, flips, mst, root)
    flip = (rel ^ (nh[seed, 2] < 0)).astype(bool) if m else np.zeros(0, bool)
    out = nrm.copy()
    out[rows[flip]] = -out[rows[flip]]
    info = dict(rows=rows, ids=ids, d2=d2, edges=edges, keys=keys, weights=w, flips=flips, mst=mst, seed=seed, rel=rel,
                flip=flip, components=len(set(root.tolist())), skipped=int(p.shape[0] - m))
    return out, info
