"""Independent restatement of the connected-component filter (DESIGN.md §2, N11) with scipy and numpy.

labels: scipy.sparse.csgraph.connected_components on the vertex adjacency (an edge between the first vertex of every
face and each of the other two), each component named by its smallest vertex.  sizes: np.bincount of the faces' labels.
Ranking (size descending, label ascending) and the stable compaction in numpy."""
import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components


class NothingKept(ValueError):
    pass


def labels_of(m, faces):
    """(m,) int32: the smallest vertex index of each vertex's component."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    rows = np.r_[f[:, 0], f[:, 0]]
    cols = np.r_[f[:, 1], f[:, 2]]
    adj = coo_matrix((np.ones(rows.shape[0], np.int8), (rows, cols)), shape=(m, m))
    _, comp = connected_components(adj, directed=False)
    smallest = np.full(comp.max() + 1 if m else 0, m, np.int64)
    np.minimum.at(smallest, comp, np.arange(m))
    return smallest[comp].astype(np.int32)


def sizes_of(m, faces, labels):
    """(m,) int32 indexed by label: triangles per component (0 at an index that is no label or an unused vertex)."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    return np.bincount(labels[f[:, 0]], minlength=m).astype(np.int32)


def keep_of(labels, sizes, min_triangles=None, keep_largest=None):
    """(m,) bool keep mask, and the kept component labels in rank order."""
    m = labels.shape[0]
    roots = np.flatnonzero((labels == np.arange(m)) & (sizes > 0))
    order = np.lexsort((roots, -sizes[roots].astype(np.int64)))  # size descending, then label ascending
    ranked = roots[order]
    ok = np.ones(ranked.shape[0], bool)
    if min_triangles is not None:
        ok &= sizes[ranked] >= min_triangles
    if keep_largest is not None:
        ok &= np.arange(ranked.shape[0]) < keep_largest
    kept = ranked[ok]
    keep_label = np.zeros(m, bool)
    keep_label[kept] = True
    return keep_label[labels], kept


def remove_components(vpos, faces, colours=None, densities=None, min_triangles=None, keep_largest=None):
    """((vpos, faces, colours, densities), info) of the kept mesh; raises NothingKept (with the largest size) when no
    component is kept.  info: labels, sizes, keep, components, kept, largest, removed_triangles, removed_vertices."""
    vpos = np.asarray(vpos)
    faces = np.asarray(faces, np.int32).reshape(-1, 3)
    m, t = vpos.shape[0], faces.shape[0]
    labels = labels_of(m, faces)
    sizes = sizes_of(m, faces, labels)
    keep, kept = keep_of(labels, sizes, min_triangles, keep_largest)
    roots = (labels == np.arange(m)) & (sizes > 0)
    largest = int(sizes.max()) if m else 0
    fkeep = keep[faces[:, 0]] if t else np.zeros(0, bool)
    info = dict(labels=labels, sizes=sizes, keep=keep, components=int(roots.sum()), kept=int(kept.shape[0]),
                largest=largest, removed_triangles=int(t - fkeep.sum()), removed_vertices=int(m - keep.sum()))
    if not fkeep.any():
        raise NothingKept(f"no component is kept: the largest has {largest} triangle(s)")
    vmap = np.cumsum(keep) - 1
    out = (vpos[keep], vmap[faces[fkeep]].astype(np.int32), None if colours is None else np.asarray(colours)[keep],
           None if densities is None else np.asarray(densities)[keep])
    return out, info
