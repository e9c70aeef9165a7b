"""Plain numpy / scipy float64 restatement of the Poisson mesher's rules (DESIGN.md §2, N6): frame, splat, direct
Neumann solve, iso-value, marching tetrahedra, density / colour gathers, density trim, Laplacian smoothing and vertex
normals.  Written from the stated rules, not from the kernels: loops are vectorised with numpy, and every sum the
kernels promise to evaluate in a fixed sequential order is evaluated in that order here (np.add.at applies its updates
in index order; segmented sums run rank by rank), so those results can be compared bit for bit."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

CELL_NONE = 0x7FFFFFFF
PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


# ---- frame and splat ------------------------------------------------------------------------------------------------
def frame(points, depth):
    """dict(origin (3,), h, L, extent, R) of the finite points."""
    p = np.asarray(points, np.float32)
    p = p[np.isfinite(p).all(1)]
    R = 1 << depth
    if p.shape[0] == 0:
        return dict(origin=np.zeros(3), h=0.0, L=0.0, extent=0.0, R=R)
    mn, mx = p.min(0).astype(np.float64), p.max(0).astype(np.float64)
    ext = float(np.max(mx - mn))
    L = 1.1 * ext
    origin = (mn + mx) * 0.5 - L * 0.5
    return dict(origin=origin, h=L / R, L=L, extent=ext, R=R)


def point_cells(points, fr):
    """i0 (n,3) int64 and f (n,3) float64 of every point."""
    R = fr["R"]
    u = (np.asarray(points, np.float32).astype(np.float64) - fr["origin"]) / fr["h"] - 0.5
    fl = np.clip(np.floor(u), 0.0, float(R - 2))
    f = np.clip(u - fl, 0.0, 1.0)
    return fl.astype(np.int64), f


def corner_weights(f):
    """(n,8) trilinear weights, corner o: bit 0 = x; w = (wx * wy) * wz."""
    w = np.empty((f.shape[0], 8))
    for o in range(8):
        ax = [f[:, a] if (o >> a) & 1 else 1.0 - f[:, a] for a in range(3)]
        w[:, o] = (ax[0] * ax[1]) * ax[2]
    return w


def usable_normals(normals):
    """(mask of points whose normal has a finite non-zero float64 length, unit normals)."""
    n = np.asarray(normals).astype(np.float64)
    with np.errstate(all="ignore"):
        s = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
        ok = (s > 0) & np.isfinite(s)
        nh = n / s[:, None]
    return ok, nh


def _splat_terms(points, normals, depth):
    """(cell (n,) int64 dual-cell index or CELL_NONE, skipped count, frame, [(nodes, q)]): every integer term the splat
    adds to B, in (corner, axis, side) order."""
    fr = frame(points, depth)
    R = fr["R"]
    p = np.asarray(points, np.float32)
    finite = np.isfinite(p).all(1)
    ok, nh = usable_normals(normals)
    skipped = int((finite & ~ok).sum())
    use = finite & ok & (fr["h"] > 0)
    cell = np.full(p.shape[0], CELL_NONE, np.int64)
    terms = []
    if not use.any():
        return cell, skipped, fr, terms
    idx = np.nonzero(use)[0]
    i0, f = point_cells(p[idx], fr)
    cell[idx] = (i0[:, 2] * (R - 1) + i0[:, 1]) * (R - 1) + i0[:, 0]
    w = corner_weights(f)
    stride = np.array([1, R, R * R])
    for o in range(8):
        c = i0 + np.array([o & 1, (o >> 1) & 1, o >> 2])
        node = (c[:, 2] * R + c[:, 1]) * R + c[:, 0]
        for a in range(3):
            q = np.rint((w[:, o] * nh[idx, a]) * 4294967296.0).astype(np.int64)
            lo, hi = c[:, a] > 0, c[:, a] < R - 1
            terms.append((node[lo] - stride[a], q[lo]))
            terms.append((node[hi] + stride[a], -q[hi]))
    return cell, skipped, fr, terms


def splat(points, normals, depth):
    """(B (R^3,) int64, cell (n,) int64 dual-cell index or CELL_NONE, skipped count, frame)."""
    cell, skipped, fr, terms = _splat_terms(points, normals, depth)
    B = np.zeros(fr["R"] ** 3, np.int64)
    for node, q in terms:
        np.add.at(B, node, q)
    return B, cell, skipped, fr


def splat_sparse(points, normals, depth):
    """(nodes (k,) int64 ascending, values (k,) int64, cell, skipped, frame): the non-zero entries of splat's B without
    the dense R^3 array.  B is an integer sum, so grouping its terms by node gives the same values in any order."""
    cell, skipped, fr, terms = _splat_terms(points, normals, depth)
    if not terms:
        return np.zeros(0, np.int64), np.zeros(0, np.int64), cell, skipped, fr
    node = np.concatenate([t[0] for t in terms])
    q = np.concatenate([t[1] for t in terms])
    del terms
    order = np.argsort(node, kind="stable")
    node, q = node[order], q[order]
    del order
    start = np.r_[0, np.nonzero(np.diff(node))[0] + 1]
    vals = np.add.reduceat(q, start)
    nodes = node[start]
    nz = vals != 0
    return nodes[nz], vals[nz], cell, skipped, fr


# ---- solve and iso --------------------------------------------------------------------------------------------------
def rhs(B, fr):
    """b = (B - mean B) * h * 2^-33 (the mean of B from its exact integer sum)."""
    mean = float(int(B.sum())) / float(B.size)
    return (B.astype(np.float64) - mean) * (fr["h"] * 2.0 ** -33)


def neumann_laplacian(R):
    """(sum of the in-grid neighbours - their count x chi) on an R^3 grid, node (k R + j) R + i."""
    t = sp.diags([np.ones(R - 1), np.r_[-1.0, -2.0 * np.ones(R - 2), -1.0], np.ones(R - 1)], [-1, 0, 1])
    eye = sp.identity(R)
    return (sp.kron(sp.kron(eye, eye), t) + sp.kron(sp.kron(eye, t), eye) + sp.kron(sp.kron(t, eye), eye)).tocsc()


def solve_direct(b, R):
    """Mean-free chi of the Neumann system.  Up to 32^3 nodes: node 0 pinned to 0 (b is mean-free, so the system is
    consistent), a sparse direct solve of the rest, then the mean subtracted.  Above that the direct factorisation of a
    3-D grid fills in too much (64^3 takes minutes): conjugate gradients on the mean-free system instead, to a relative
    residual of 1e-13, far below the float32 solve it checks."""
    A = neumann_laplacian(R)
    if R <= 32:
        x = np.zeros(R ** 3)
        x[1:] = spla.spsolve(A[1:, 1:], b[1:])
    else:
        x, info = spla.cg(-A, -(b - b.mean()), rtol=1e-13, atol=0.0, maxiter=20 * R ** 2)
        assert info == 0, info
    return x - x.mean()


def solve_dct(b, R):
    """Exact mean-free chi of the Neumann system, computed in place in b's memory (b (R^3,) float64 is overwritten).
    The orthonormal DCT-II along each axis diagonalises the 1-D operator with mirrored ghosts, eigenvalue
    2 cos(pi k / R) - 2 for mode k, so the 3-D operator has the sum over the axes; the k = 0 mode (the null space, the
    mean) is set to 0."""
    import scipy.fft as sfft
    x = b.reshape(R, R, R)
    sfft.dctn(x, type=2, norm="ortho", overwrite_x=True, workers=-1)
    lam = 2.0 * np.cos(np.pi * np.arange(R) / R) - 2.0
    plane = lam[:, None] + lam[None, :]
    for k in range(R):
        x[k] /= plane + lam[k] if k else np.where(plane == 0.0, 1.0, plane)
    x[0, 0, 0] = 0.0
    sfft.idctn(x, type=2, norm="ortho", overwrite_x=True, workers=-1)
    return b


def residual_ratio(chi, b, R):
    r = b - neumann_laplacian(R) @ np.asarray(chi, np.float64)
    return float(np.linalg.norm(r) / np.linalg.norm(b))


def residual_ratio_slabs(chi, b, R, slab=64):
    """residual_ratio with a numpy stencil, `slab` z-layers at a time: no sparse matrix, and no temporary larger than
    one slab."""
    c = np.asarray(chi).reshape(R, R, R)
    bb = np.asarray(b).reshape(R, R, R)
    cnt_ij = np.full((R, R), 6.0)
    cnt_ij[:, 0] -= 1
    cnt_ij[:, -1] -= 1
    cnt_ij[0, :] -= 1
    cnt_ij[-1, :] -= 1
    rr = bsq = 0.0
    for k0 in range(0, R, slab):
        k1 = min(k0 + slab, R)
        x = c[k0:k1].astype(np.float64)
        s = np.zeros_like(x)
        s[:, :, 1:] += x[:, :, :-1]
        s[:, :, :-1] += x[:, :, 1:]
        s[:, 1:, :] += x[:, :-1, :]
        s[:, :-1, :] += x[:, 1:, :]
        s[1:] += x[:-1]
        s[:-1] += x[1:]
        cnt = np.repeat(cnt_ij[None], k1 - k0, 0)
        if k0 > 0:
            s[0] += c[k0 - 1]
        else:
            cnt[0] -= 1
        if k1 < R:
            s[-1] += c[k1]
        else:
            cnt[-1] -= 1
        r = bb[k0:k1] - (s - cnt * x)
        rr += float(np.vdot(r, r))
        bsq += float(np.vdot(bb[k0:k1], bb[k0:k1]))
    return float(np.sqrt(rr) / np.sqrt(bsq))


def trilinear(points, fr, chi):
    """Trilinear chi at the points with the splat's weights, corners summed in order o = 0..7."""
    R = fr["R"]
    i0, f = point_cells(points, fr)
    w = corner_weights(f)
    chi = np.asarray(chi).astype(np.float64)
    v = np.zeros(i0.shape[0])
    for o in range(8):
        c = i0 + np.array([o & 1, (o >> 1) & 1, o >> 2])
        v = v + w[:, o] * chi[(c[:, 2] * R + c[:, 1]) * R + c[:, 0]]
    return v


def iso_value(points, cell, fr, chi):
    used = np.asarray(cell) != CELL_NONE
    return float(trilinear(np.asarray(points)[used], fr, chi).sum() / used.sum())


# ---- marching tetrahedra ------------------------------------------------------------------------------------------
def tet_corners(p):
    a, b, _ = PERMS[p]
    return [0, 1 << a, (1 << a) | (1 << b), 7]


def _xyz(corner):
    return np.array([corner & 1, (corner >> 1) & 1, corner >> 2])


def tet_triangles(p, inside):
    """Triangles of Kuhn tetrahedron p for the corner inside-bits `inside` (8-bit cube mask): a list of triangles, each
    three (lower corner, upper corner) pairs.  One corner alone on its side: the triangle on its three edges.  Two and
    two (inside i0 < i1, outside o0 < o1 in tetrahedron order): the quad i0o0, i0o1, i1o1, i1o0 cut along i0o0-i1o1.  A
    triangle whose normal (right-hand rule over the edge midpoints) does not point towards the outside is reversed
    (its last two entries swap)."""
    v = tet_corners(p)
    ins = [q for q in range(4) if (inside >> v[q]) & 1]
    outs = [q for q in range(4) if not (inside >> v[q]) & 1]
    if len(ins) in (1, 3):
        apex, rest = (ins[0], outs) if len(ins) == 1 else (outs[0], ins)
        tris = [[(apex, r) for r in rest]]
    elif len(ins) == 2:
        (i0, i1), (o0, o1) = ins, outs
        tris = [[(i0, o0), (i0, o1), (i1, o1)], [(i0, o0), (i1, o1), (i1, o0)]]
    else:
        return []
    out = []
    for tri in tris:
        mids = [_xyz(v[a]) + _xyz(v[b]) for a, b in tri]
        normal = np.cross(mids[1] - mids[0], mids[2] - mids[0])
        if normal @ (_xyz(v[outs[0]]) - _xyz(v[ins[0]])) < 0:
            tri = [tri[0], tri[2], tri[1]]
        out.append([(min(v[a], v[b]), max(v[a], v[b])) for a, b in tri])
    return out


_TABLE = [[tet_triangles(p, m) for m in range(256)] for p in range(6)]


def _slab(chi, R, k0, k1):
    """(k0, k1, chi[k0 : k1 + 1] as float64 (z, y, x)): the layers the vertices of node layers [k0, k1) and the cubes
    with lowest corner in [k0, k1) read."""
    k0 = 0 if k0 is None else int(k0)
    k1 = R if k1 is None else int(k1)
    assert 0 <= k0 < k1 <= R
    c = np.asarray(chi).reshape(R, R, R)[k0:min(k1 + 1, R)].astype(np.float64)
    return k0, k1, c


def crossed_edges(chi, R, iso, k0=None, k1=None):
    """(vkey (m,) int64 ascending, vt (m,)) of the lattice edges crossed by the iso-surface whose first node lies in
    z-layers [k0, k1) (default: all); a node is inside iff chi < iso."""
    k0, k1, c = _slab(chi, R, k0, k1)
    inside = c < iso
    nk = k1 - k0
    keys = []
    for d in range(1, 8):
        dx, dy, dz = d & 1, (d >> 1) & 1, d >> 2
        top = min(nk, c.shape[0] - dz)
        crossed = inside[:top, :R - dy, :R - dx] != inside[dz:top + dz, dy:, dx:]
        k, j, i = np.nonzero(crossed)
        keys.append((((k + k0) * R + j) * R + i) * 8 + d)
    vkey = np.sort(np.concatenate(keys)).astype(np.int64)
    node, d = vkey >> 3, vkey & 7
    flat = c.reshape(-1)
    ii, jj, kk = node % R, (node // R) % R, node // (R * R) - k0
    ib, jb, kb = ii + (d & 1), jj + ((d >> 1) & 1), kk + (d >> 2)
    ca, cb = flat[(kk * R + jj) * R + ii], flat[(kb * R + jb) * R + ib]
    return vkey, (iso - ca) / (cb - ca)


def marching_tetrahedra(chi, R, iso, origin=(0.0, 0.0, 0.0), h=1.0, k0=None, k1=None):
    """(vkey (m,) int64 ascending, vt (m,), vpos (m,3), faces (t,3) int64) on the node lattice of chi (R^3, node
    (k R + j) R + i); a node is inside iff chi < iso; node positions origin + (i + 1/2) h.  With k0 / k1, one z-slab:
    the vertices whose node lies in layers [k0, k1) and the triangles of the cubes whose lowest corner does, the faces
    then as triples of vertex keys (global vertex indices need the whole grid)."""
    slab = k0 is not None or k1 is not None
    vkey, t = crossed_edges(chi, R, iso, k0, k1)
    k0, k1, c = _slab(chi, R, k0, k1)
    node, d = vkey >> 3, vkey & 7
    ii, jj, kk = node % R, (node // R) % R, node // (R * R)
    ib, jb, kb = ii + (d & 1), jj + ((d >> 1) & 1), kk + (d >> 2)
    origin = np.asarray(origin, np.float64)
    vpos = np.empty((vkey.size, 3))
    for a, (lo, hi) in enumerate(((ii, ib), (jj, jb), (kk, kb))):
        pa = origin[a] + (lo + 0.5) * h
        pb = origin[a] + (hi + 0.5) * h
        vpos[:, a] = pa + t * (pb - pa)
    # cubes: 8-bit inside mask per cube origin (k, j, i) <= R - 2
    inside = c < iso
    nc = min(k1, R - 1) - k0
    m = np.zeros((max(nc, 0), R - 1, R - 1), np.uint8)
    for o in range(8):
        dx, dy, dz = o & 1, (o >> 1) & 1, o >> 2
        m |= inside[dz:nc + dz, dy:R - 1 + dy, dx:R - 1 + dx].astype(np.uint8) << o
    k, j, i = np.nonzero((m != 0) & (m != 255))
    mask = m[k, j, i]
    cube_node = ((k + k0) * R + j) * R + i
    rows = []  # (cube node, tetrahedron, triangle, 3 edge keys)
    for p in range(6):
        for case in np.unique(mask):
            tris = _TABLE[p][case]
            sel = cube_node[mask == case]
            for ti, tri in enumerate(tris):
                ek = []
                for lo, hi in tri:
                    off = (lo & 1) + ((lo >> 1) & 1) * R + (lo >> 2) * R * R
                    ek.append((sel + off) * 8 + (hi ^ lo))
                rows.append(np.stack([sel, np.full_like(sel, p), np.full_like(sel, ti)] + ek, 1))
    if rows and slab:
        rows = np.concatenate(rows)
        faces = rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))][:, 3:6]
    elif rows:
        rows = np.concatenate(rows)
        rows = rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))]
        faces = np.searchsorted(vkey, rows[:, 3:6])
        assert (vkey[faces] == rows[:, 3:6]).all()
    else:
        faces = np.zeros((0, 3), np.int64)
    return vkey, t, vpos, faces


# ---- densities, colours, trim ---------------------------------------------------------------------------------------
def _segment_sums(seg, vals, nseg):
    """Sequential float64 sums of vals per segment, in the given order of the entries."""
    out = np.zeros((nseg,) + vals.shape[1:])
    if seg.size == 0:
        return out
    start = np.r_[0, np.nonzero(np.diff(seg))[0] + 1]
    rank = np.arange(seg.size) - np.repeat(start, np.diff(np.r_[start, seg.size]))
    for r in range(int(rank.max()) + 1):
        sel = rank == r
        out[seg[sel]] = out[seg[sel]] + vals[sel]
    return out


def vertex_density_colour(points, colours, cell, fr, vkey, vt):
    """density (m,) and colours (m,3) uint8 (None without colours): node sums over the 8 dual cells around the node,
    cells in ascending index, points in ascending input index."""
    R = fr["R"]
    used = np.nonzero(np.asarray(cell) != CELL_NONE)[0]
    i0, f = point_cells(np.asarray(points)[used], fr)
    w = corner_weights(f)
    cid = np.asarray(cell)[used]
    nodes, cells, pidx, ws, cols = [], [], [], [], []
    col = None if colours is None else np.asarray(colours).astype(np.float64)[used]
    for o in range(8):
        c = i0 + np.array([o & 1, (o >> 1) & 1, o >> 2])
        nodes.append((c[:, 2] * R + c[:, 1]) * R + c[:, 0])
        cells.append(cid)
        pidx.append(used)
        ws.append(w[:, o])
        if col is not None:
            cols.append(w[:, o, None] * col)
    nodes, cells, pidx, ws = map(np.concatenate, (nodes, cells, pidx, ws))
    order = np.lexsort((pidx, cells, nodes))
    nodes, ws = nodes[order], ws[order]
    uniq, seg = np.unique(nodes, return_inverse=True)
    W = _segment_sums(seg, ws, uniq.size)
    C = _segment_sums(seg, np.concatenate(cols)[order], uniq.size) if col is not None else None
    node_a = vkey >> 3
    d = vkey & 7
    ia, ja, ka = node_a % R, (node_a // R) % R, node_a // (R * R)
    node_b = ((ka + (d >> 2)) * R + ja + ((d >> 1) & 1)) * R + ia + (d & 1)

    def look(tab, nd):
        pos = np.searchsorted(uniq, nd)
        pos = np.minimum(pos, uniq.size - 1)
        hit = uniq[pos] == nd
        out = np.zeros((nd.size,) + tab.shape[1:])
        out[hit] = tab[pos[hit]]
        return out

    s = 1.0 - vt
    dens = s * look(W, node_a) + vt * look(W, node_b)
    if C is None:
        return dens, None
    num = s[:, None] * look(C, node_a) + vt[:, None] * look(C, node_b)
    with np.errstate(all="ignore"):
        c = np.floor(num / dens[:, None] + 0.5)
    c = np.where(dens[:, None] > 0, np.clip(c, 0, 255), 0)
    return dens, c.astype(np.uint8)


def trim_mask(dens):
    """keep = not (density < numpy's linear 10 % quantile)."""
    thr = np.quantile(dens, 0.1)
    return ~(dens < thr), thr


def trim(dens, vpos, vcol, faces):
    keep, thr = trim_mask(dens)
    fk = keep[faces].all(1) if faces.size else np.zeros(0, bool)
    remap = np.cumsum(keep) - 1
    return (dens[keep], vpos[keep], None if vcol is None else vcol[keep], remap[faces[fk]], keep, thr)


# ---- smoothing and normals ----------------------------------------------------------------------------------------
def one_ring(faces, m):
    """(u, v) of the distinct directed one-ring edges, sorted by (u, v): unique packed keys u << 32 | v (vertex indices
    are below 2^31, so the key order is the pair order)."""
    f = np.asarray(faces, np.int64)
    a = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    b = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    e = np.unique(np.concatenate([a << 32 | b, b << 32 | a]))
    return e >> 32, e & 0xFFFFFFFF


def smooth(vpos, faces, iterations, lam=0.5):
    v = np.asarray(vpos, np.float64).copy()
    m = v.shape[0]
    u, nb = one_ring(faces, m)
    has = np.zeros(m, bool)
    has[u] = True
    for _ in range(iterations):
        d = v[u] - v[nb]
        w = 1.0 / (np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) + 1e-12)
        sw = np.zeros(m)
        s = np.zeros((m, 3))
        np.add.at(sw, u, w)
        np.add.at(s, u, w[:, None] * v[nb])
        new = v.copy()
        new[has] = v[has] + lam * (s[has] / sw[has, None] - v[has])
        v = new
    return v


def vertex_normals(vpos, faces):
    v = np.asarray(vpos, np.float64)
    f = np.asarray(faces, np.int64)
    n = np.zeros_like(v)
    if f.size:
        cr = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
        np.add.at(n, f.reshape(-1), np.repeat(cr, 3, axis=0))
    s = np.sqrt((n[:, 0] * n[:, 0] + n[:, 1] * n[:, 1]) + n[:, 2] * n[:, 2])
    out = np.zeros_like(n)
    nz = s > 0
    out[nz] = n[nz] / s[nz, None]
    return out


# ---- mesh topology helpers (tests) ----------------------------------------------------------------------------------
def edge_use(faces):
    """{undirected edge: count}, and whether every directed edge occurs at most once (consistent orientation)."""
    f = np.asarray(faces, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und = np.sort(d, 1)
    _, counts = np.unique(und, axis=0, return_counts=True)
    _, dcounts = np.unique(d, axis=0, return_counts=True)
    return counts, bool((dcounts == 1).all())


def euler_characteristic(faces, m=None):
    f = np.asarray(faces, np.int64)
    V = np.unique(f).size if m is None else m
    E = np.unique(np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), 1), axis=0).shape[0]
    return V - E + f.shape[0]


def components(faces):
    from scipy.sparse.csgraph import connected_components
    f = np.asarray(faces, np.int64)
    used = np.unique(f)
    idx = np.searchsorted(used, f)
    e = np.concatenate([idx[:, [0, 1]], idx[:, [1, 2]]])
    g = sp.coo_matrix((np.ones(e.shape[0]), (e[:, 0], e[:, 1])), shape=(used.size, used.size))
    return connected_components(g, directed=False)[0]


def signed_volume(vpos, faces):
    v = np.asarray(vpos, np.float64)
    f = np.asarray(faces, np.int64)
    return float(np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6.0)
