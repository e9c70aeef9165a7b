"""Independent restatement of the hole filling (DESIGN.md §2, N12) with numpy and scipy.

Boundary half-edges: the undirected edges used once, by np.unique counts.  Boundary sets: scipy's connected_components
over the boundary half-edges, each set named by its smallest vertex.  Loops: walked from the label through succ, one
step per column over all holes at once.  Centre sums: sequential float64 additions in loop order, one numpy add per
loop position (each is correctly rounded, as __dadd_rn is), never numpy's pairwise reductions."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


def boundary_half_edges(m, faces):
    """(u, v, face) of every boundary half-edge, in half-edge order (3 face + corner)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    u, v = f.ravel(), np.roll(f, -1, axis=1).ravel()
    key = np.minimum(u, v) * m + np.maximum(u, v)
    _, inv, cnt = np.unique(key, return_inverse=True, return_counts=True)
    b = cnt[inv.ravel()] == 1
    return u[b], v[b], (np.arange(u.shape[0]) // 3)[b]


def find(m, faces):
    """labels (-1 off the boundary), succ (-1 unless exactly one outgoing boundary half-edge), lengths and pinched (both
    indexed by label), the face of each vertex's only outgoing boundary half-edge, and the boundary half-edge count."""
    bu, bv, bf = boundary_half_edges(m, faces)
    outdeg = np.bincount(bu, minlength=m)
    indeg = np.bincount(bv, minlength=m)
    adj = coo_matrix((np.ones(bu.shape[0], np.int8), (bu, bv)), shape=(m, m))
    _, comp = connected_components(adj, directed=False)
    smallest = np.full(comp.max() + 1, m, np.int64)
    np.minimum.at(smallest, comp, np.arange(m))
    on = (outdeg + indeg) > 0
    labels = np.where(on, smallest[comp], -1).astype(np.int32)
    one = outdeg[bu] == 1
    succ = np.full(m, -1, np.int32)
    succ[bu[one]] = bv[one]
    bface = np.full(m, -1, np.int64)
    bface[bu[one]] = bf[one]
    lengths = np.bincount(labels[on], minlength=m).astype(np.int32)
    pinched = np.zeros(m, bool)
    pinched[labels[on & ((outdeg != 1) | (indeg != 1))]] = True
    return labels, succ, lengths, pinched, bface, int(bu.shape[0])


def walk(succ, starts, L):
    """(k, max L) vertex matrix of the loops from `starts`; entries past a loop's length repeat its start."""
    W = int(L.max()) if L.shape[0] else 0
    loops = np.empty((starts.shape[0], W), np.int64)
    cur = starts.astype(np.int64)
    for k in range(W):
        loops[:, k] = np.where(k < L, cur, starts)
        cur = np.where(k + 1 < L, succ[cur], cur)
    return loops


def fill_holes(vpos, faces, colours=None, densities=None, max_hole_edges=64):
    """((vpos, faces, colours, densities), info) of the filled mesh (the inputs themselves when nothing is filled).
    info: labels, succ, lengths, filled (uint8, per label) and the stats of mesh.fill_holes."""
    vpos = np.asarray(vpos, np.float64)
    faces = np.asarray(faces, np.int32).reshape(-1, 3)
    m, t = vpos.shape[0], faces.shape[0]
    labels, succ, lengths, pinched, bface, nb = find(m, faces)
    roots = np.flatnonzero(labels == np.arange(m))
    hole = roots[~pinched[roots]]
    L = lengths[hole].astype(np.int64)
    too_long = L > max_hole_edges
    lone = np.zeros(hole.shape[0], bool)
    tri = ~too_long & (L == 3)
    s1 = succ[hole[tri]]
    s2 = succ[s1]
    lone[tri] = (bface[s1] == bface[hole[tri]]) & (bface[s2] == bface[hole[tri]])
    fill = ~too_long & ~lone
    filled = np.zeros(m, np.uint8)
    filled[hole[fill]] = 1
    starts, Lf = hole[fill], L[fill]  # ascending labels
    fan = Lf >= 4
    info = dict(labels=labels, succ=succ, lengths=lengths, filled=filled, boundary_edges=nb,
                holes=int(hole.shape[0]), filled_holes=int(fill.sum()), too_long=int(too_long.sum()),
                lone_triangles=int(lone.sum()), pinched=int(pinched[roots].sum()), added_vertices=int(fan.sum()),
                added_triangles=int(np.where(fan, Lf, 1).sum()))
    if not fill.any():
        return (vpos, faces, colours, densities), info
    loops = walk(succ, starts, Lf)
    W = loops.shape[1]
    cen = np.cumsum(fan) - 1 + m  # centre index of each fan hole
    A = np.stack([np.roll(loops, -1, 1), loops, np.broadcast_to(cen[:, None], loops.shape)], -1)  # (v(k+1), v(k), c)
    t3 = Lf == 3
    A[t3, 0] = loops[t3][:, [0, 2, 1]]
    F = np.concatenate([faces.astype(np.int64), A[np.arange(W) < np.where(t3, 1, Lf)[:, None]]]).astype(np.int32)
    fl, Lfan = loops[fan], Lf[fan]

    def seq_sum(x):  # x: (k, W, ...) in loop order; sequential from the first entry
        s = x[:, 0].copy()
        for k in range(1, W):
            live = (k < Lfan).reshape((-1,) + (1,) * (x.ndim - 2))
            s = np.where(live, s + x[:, k], s)
        return s

    Pc = seq_sum(vpos[fl]) / Lfan[:, None].astype(np.float64)
    P = np.concatenate([vpos, Pc])
    C = D = None
    if colours is not None:
        colours = np.asarray(colours, np.uint8)
        cs = (colours[fl].astype(np.int64) * (np.arange(W) < Lfan[:, None])[:, :, None]).sum(1)
        C = np.concatenate([colours, ((2 * cs + Lfan[:, None]) // (2 * Lfan[:, None])).astype(np.uint8)])
    if densities is not None:
        densities = np.asarray(densities, np.float64)
        D = np.concatenate([densities, seq_sum(densities[fl]) / Lfan.astype(np.float64)])
    return (P, F, C, D), info


STATS = ("boundary_edges", "holes", "filled", "too_long", "lone_triangles", "pinched", "added_vertices",
         "added_triangles")


def stats_of(info):
    """The stats dict mesh.fill_holes fills, from fill_holes' info."""
    return {k: info["filled_holes" if k == "filled" else k] for k in STATS}


def euler(m, faces):
    """V - E + F of the vertices the faces use."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    e = np.unique(np.sort(np.stack([f.ravel(), np.roll(f, -1, 1).ravel()], 1), 1), axis=0).shape[0]
    return np.unique(f).shape[0] - e + f.shape[0]
