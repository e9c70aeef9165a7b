"""Plain numpy / scipy float64 restatement of the Poisson mesher's narrow-band levels (DESIGN.md §2, N6b): brick map
and list with the nesting rule, band splat, ghosts and initial guess, the band solve, iso-value, marching tetrahedra over
the covered cubes, and the density / colour gather.  Written from the rules, not the kernels, and built on f64ref_mesh
(its splat terms, trilinear weights, tetrahedron table and gathers).  Sums the kernels evaluate in a fixed order are
evaluated in that order here, so those results compare bit for bit."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import f64ref_mesh as fm

BRICK, MARGIN, S = 8, 1, 0.125
BRICK_NODES = BRICK ** 3
DIRECT_MAX = 100_000  # active nodes up to which the band solve is a sparse direct one (CG to 1e-12 above)


def band_frame(points, D):
    """The frame of level D: the dense frame's origin and L, h = L / 2^D (f64ref_mesh.frame at depth D)."""
    return fm.frame(points, D)


# ---- bricks ---------------------------------------------------------------------------------------------------------
def seed_nodes(points, normals, D):
    """Sorted unique global nodes the splat writes at level D (q = 0 terms included)."""
    _, _, _, terms = fm._splat_terms(points, normals, D)
    if not terms:
        return np.zeros(0, np.int64)
    return np.unique(np.concatenate([t[0] for t in terms]))


def _brick_of(nodes, R):
    NB = R // BRICK
    i, j, k = nodes % R, (nodes // R) % R, nodes // (R * R)
    return ((k // BRICK) * NB + j // BRICK) * NB + i // BRICK


def bricks(points, normals, D, parent_map=None):
    """(map (NB^3,) int32, list (k,) int32, lost seed bricks) of level D; parent_map None: the level below is dense."""
    R = 1 << D
    NB = R // BRICK
    seed = np.zeros((NB, NB, NB), bool)
    seed.reshape(-1)[_brick_of(seed_nodes(points, normals, D), R)] = True
    near = np.zeros_like(seed)
    p = np.pad(seed, MARGIN)
    for dz in range(2 * MARGIN + 1):
        for dy in range(2 * MARGIN + 1):
            for dx in range(2 * MARGIN + 1):
                near |= p[dz:dz + NB, dy:dy + NB, dx:dx + NB]
    nested = np.ones_like(seed)
    if parent_map is not None:
        NBc, Rc = NB // 2, R // 2
        act_c = (np.asarray(parent_map) >= 0).reshape(NBc, NBc, NBc)
        b = np.arange(NB)
        lo, hi = np.maximum(4 * b - 1, 0) // BRICK, np.minimum(4 * b + 4, Rc - 1) // BRICK
        # per axis the coarse bricks lo..hi (at most two); nested iff all are active
        for cz in (lo, hi):
            for cy in (lo, hi):
                for cx in (lo, hi):
                    nested &= act_c[cz[:, None, None], cy[None, :, None], cx[None, None, :]]
    keep = (near & nested).reshape(-1)
    lost = int((seed & ~nested).sum())
    bmap = np.full(NB ** 3, -1, np.int32)
    blist = np.nonzero(keep)[0].astype(np.int32)
    bmap[blist] = np.arange(blist.size, dtype=np.int32)
    return bmap, blist, lost


def storage(bmap, R, i, j, k):
    """Storage index of global nodes (arrays, in grid) or -1; bmap None: dense indexing."""
    if bmap is None:
        return (k * R + j) * R + i
    NB = R // BRICK
    s = np.asarray(bmap)[((k // BRICK) * NB + j // BRICK) * NB + i // BRICK].astype(np.int64)
    loc = ((k % BRICK) * BRICK + j % BRICK) * BRICK + i % BRICK
    return np.where(s >= 0, s * BRICK_NODES + loc, -1)


def node_ijk(blist, R):
    """Global (i, j, k) of every band storage index."""
    NB = R // BRICK
    b = np.repeat(np.asarray(blist, np.int64), BRICK_NODES)
    loc = np.tile(np.arange(BRICK_NODES), len(blist))
    return ((b % NB) * BRICK + loc % 8, ((b // NB) % NB) * BRICK + (loc // 8) % 8, (b // (NB * NB)) * BRICK + loc // 64)


# ---- splat, ghosts ------------------------------------------------------------------------------------------------
def band_B(points, normals, D, bmap, nbricks):
    """(B (nbricks * 512,) int64, terms outside the band)."""
    R = 1 << D
    _, _, _, terms = fm._splat_terms(points, normals, D)
    B = np.zeros(nbricks * BRICK_NODES, np.int64)
    outside = 0
    for node, q in terms:
        u = storage(bmap, R, node % R, (node // R) % R, node // (R * R))
        nz = q != 0
        outside += int(((u < 0) & nz).sum())
        np.add.at(B, u[(u >= 0) & nz], q[(u >= 0) & nz])
    return B, outside


def prolong(chi_c, map_c, Rc, i, j, k):
    """s P(chi_c) at fine nodes (arrays): per axis lo = i >> 1 (3/4) and lo +- 1 towards i (1/4, clamped); corners
    o = 0..7 summed in order with w = (wx * wy) * wz, then times s."""
    chi_c = np.asarray(chi_c)
    lo, hi = [], []
    for p in (i, j, k):
        l = p >> 1
        lo.append(l)
        hi.append(np.clip(l + np.where(p & 1, 1, -1), 0, Rc - 1))
    v = np.zeros(np.shape(i))
    for o in range(8):
        x = hi[0] if o & 1 else lo[0]
        y = hi[1] if o & 2 else lo[1]
        z = hi[2] if o & 4 else lo[2]
        w = ((0.25 if o & 1 else 0.75) * (0.25 if o & 2 else 0.75)) * (0.25 if o & 4 else 0.75)
        u = storage(map_c, Rc, x, y, z)
        assert (u >= 0).all(), "prolongation reads an inactive coarse node"
        v = v + w * chi_c[u].astype(np.float64)
    return S * v


def ghosts(chi_c, map_c, D, bmap, blist, B, h):
    """(ghost sums, chi0 float32, rhs float32) per band node."""
    R = 1 << D
    i, j, k = node_ijk(blist, R)
    g = np.zeros(i.size)
    for e in range(6):
        p = [i.copy(), j.copy(), k.copy()]
        p[e >> 1] += 1 if e & 1 else -1
        ing = (p[e >> 1] >= 0) & (p[e >> 1] <= R - 1)
        q = [np.clip(a, 0, R - 1) for a in p]
        ghost = ing & (storage(bmap, R, *q) < 0)
        if ghost.any():
            val = np.zeros(i.size)
            val[ghost] = prolong(chi_c, map_c, R // 2, q[0][ghost], q[1][ghost], q[2][ghost])
            g = np.where(ghost, g + val, g)
    chi0 = prolong(chi_c, map_c, R // 2, i, j, k).astype(np.float32)
    b = B.astype(np.float64) * (h * 2.0 ** -33)
    return g, chi0, (g - b).astype(np.float32)


# ---- solve ------------------------------------------------------------------------------------------------------
def operator(bmap, blist, D):
    """M = count x chi - sum of the active in-grid neighbours on the band (csr), and the counts."""
    R = 1 << D
    i, j, k = node_ijk(blist, R)
    n = i.size
    rows, cols = [], []
    cnt = np.zeros(n)
    for e in range(6):
        p = [i.copy(), j.copy(), k.copy()]
        p[e >> 1] += 1 if e & 1 else -1
        ing = (p[e >> 1] >= 0) & (p[e >> 1] <= R - 1)
        cnt += ing
        u = storage(bmap, R, *[np.clip(a, 0, R - 1) for a in p])
        sel = ing & (u >= 0)
        rows.append(np.nonzero(sel)[0])
        cols.append(u[sel])
    r, c = np.concatenate(rows), np.concatenate(cols)
    A = sp.csr_matrix((-np.ones(r.size), (r, c)), shape=(n, n)) + sp.diags(cnt)
    return A.tocsr(), cnt


def solve(rhs, bmap, blist, D, x0=None):
    """float64 chi of M chi = rhs on the band."""
    A, cnt = operator(bmap, blist, D)
    c = np.asarray(rhs, np.float64)
    if c.size <= DIRECT_MAX:
        return spla.spsolve(A.tocsc(), c)
    x, info = spla.cg(A, c, x0=None if x0 is None else np.asarray(x0, np.float64), rtol=1e-12, atol=0.0,
                      maxiter=20000, M=sp.diags(1.0 / cnt))
    assert info == 0, info
    return x


def residual_ratio(chi, rhs, bmap, blist, D):
    A, _ = operator(bmap, blist, D)
    c = np.asarray(rhs, np.float64)
    return float(np.linalg.norm(c - A @ np.asarray(chi, np.float64)) / np.linalg.norm(c))


# ---- iso, extraction, gather --------------------------------------------------------------------------------------
def iso_value(points, cell, fr, bmap, chi):
    """Mean over the splatted points of trilinear chi (corners in order o)."""
    R = fr["R"]
    used = np.asarray(cell) != fm.CELL_NONE
    i0, f = fm.point_cells(np.asarray(points)[used], fr)
    w = fm.corner_weights(f)
    chi = np.asarray(chi).astype(np.float64)
    v = np.zeros(i0.shape[0])
    for o in range(8):
        c = i0 + np.array([o & 1, (o >> 1) & 1, o >> 2])
        u = storage(bmap, R, c[:, 0], c[:, 1], c[:, 2])
        assert (u >= 0).all()
        v = v + w[:, o] * chi[u]
    return float(v.sum() / used.sum())


def marching_tetrahedra(chi, bmap, blist, fr, iso):
    """(vkey, vt, vpos, faces) over the covered cubes (all 8 corners active): vertices in ascending (storage index, d)
    for the crossed edges some covered cube holds, triangles in ascending (storage index of the cube, tetrahedron,
    triangle), node positions origin + (i + 1/2) h."""
    R = fr["R"]
    chi = np.asarray(chi).astype(np.float64)
    i, j, k = node_ijk(blist, R)
    n = i.size

    def look(dx, dy, dz):
        x, y, z = i + dx, j + dy, k + dz
        ing = (x >= 0) & (y >= 0) & (z >= 0) & (x < R) & (y < R) & (z < R)
        u = storage(bmap, R, np.clip(x, 0, R - 1), np.clip(y, 0, R - 1), np.clip(z, 0, R - 1))
        return np.where(ing, u, -1)

    act = {}
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                act[(dx, dy, dz)] = look(dx, dy, dz)
    inside = np.zeros(n, np.int64)
    for o in range(8):
        u = act[(o & 1, (o >> 1) & 1, o >> 2)]
        inside |= ((u >= 0) & (chi[np.maximum(u, 0)] < iso)).astype(np.int64) << o
    cov = np.zeros((8, n), bool)
    for lo in range(8):
        ok = np.ones(n, bool)
        for o in range(8):
            d = ((o & 1) - (lo & 1), ((o >> 1) & 1) - ((lo >> 1) & 1), (o >> 2) - (lo >> 2))
            ok &= act[d] >= 0
        cov[lo] = ok
    vmask = np.zeros(n, np.int64)
    for d in range(1, 8):
        held = np.zeros(n, bool)
        for lo in range(8):
            if not lo & d:
                held |= cov[lo]
        crossed = ((inside >> d) & 1) != (inside & 1)
        vmask |= (held & crossed).astype(np.int64) << d
    # vertices
    us, ds = [], []
    for d in range(1, 8):
        sel = np.nonzero((vmask >> d) & 1)[0]
        us.append(sel)
        ds.append(np.full(sel.size, d))
    u, d = np.concatenate(us), np.concatenate(ds)
    order = np.argsort(u * 8 + d, kind="stable")
    u, d = u[order], d[order]
    vid = u * 8 + d  # storage-order vertex ids (ascending)
    ia, ja, ka = i[u], j[u], k[u]
    ib, jb, kb = ia + (d & 1), ja + ((d >> 1) & 1), ka + (d >> 2)
    ca, cb = chi[u], chi[storage(bmap, R, ib, jb, kb)]
    t = (iso - ca) / (cb - ca)
    vkey = (((ka * R + ja) * R + ia) * 8 + d).astype(np.int64)
    vpos = np.empty((u.size, 3))
    for a, (lo_, hi_) in enumerate(((ia, ib), (ja, jb), (ka, kb))):
        pa = fr["origin"][a] + (lo_ + 0.5) * fr["h"]
        pb = fr["origin"][a] + (hi_ + 0.5) * fr["h"]
        vpos[:, a] = pa + t * (pb - pa)
    # triangles
    cube = np.nonzero(cov[0] & (inside != 0) & (inside != 255))[0]
    rows = []
    for p in range(6):
        for case in np.unique(inside[cube]):
            sel = cube[inside[cube] == case]
            for ti, tri in enumerate(fm._TABLE[p][case]):
                ek = []
                for lo_, hi_ in tri:
                    pn = storage(bmap, R, i[sel] + (lo_ & 1), j[sel] + ((lo_ >> 1) & 1), k[sel] + (lo_ >> 2))
                    ek.append(pn * 8 + (hi_ ^ lo_))
                rows.append(np.stack([sel, np.full_like(sel, p), np.full_like(sel, ti)] + ek, 1))
    if rows:
        rows = np.concatenate(rows)
        rows = rows[np.lexsort((rows[:, 2], rows[:, 1], rows[:, 0]))]
        faces = np.searchsorted(vid, rows[:, 3:6])
        assert (vid[faces] == rows[:, 3:6]).all()
    else:
        faces = np.zeros((0, 3), np.int64)
    return vkey, t, vpos, faces


def band_cells(points, cell, fr):
    """int64 dual cell of every splatted point at the band level (CELL_NONE for the others: only its != test is
    read)."""
    R = fr["R"]
    out = np.full(len(cell), fm.CELL_NONE, np.int64)
    used = np.asarray(cell) != fm.CELL_NONE
    i0, _ = fm.point_cells(np.asarray(points)[used], fr)
    out[used] = (i0[:, 2] * (R - 1) + i0[:, 1]) * (R - 1) + i0[:, 0]
    return out


def vertex_density_colour(points, colours, cell, fr, vkey, vt):
    """f64ref_mesh's gather at the band level (its node sums only need the points' dual cells at that level)."""
    return fm.vertex_density_colour(points, colours, band_cells(points, cell, fr), fr, vkey, vt)


# ---- the whole band pipeline (tests) ----------------------------------------------------------------------------
def band_levels(points, normals, depth, band_depth, dense_chi):
    """Every level's (map, list, lost, B, ghost, chi0, rhs, chi) with float64 solves, each level fed the level
    below's float64 chi."""
    out = []
    chi_c, map_c = np.asarray(dense_chi, np.float64), None
    for D in range(depth + 1, band_depth + 1):
        fr = band_frame(points, D)
        bmap, blist, lost = bricks(points, normals, D, map_c)
        B, outside = band_B(points, normals, D, bmap, blist.size)
        g, chi0, rhs = ghosts(chi_c, map_c, D, bmap, blist, B, fr["h"])
        chi = solve(rhs.astype(np.float64), bmap, blist, D, chi0)
        out.append(dict(depth=D, frame=fr, map=bmap, bricks=blist, lost=lost, B=B, outside=outside, ghost=g, chi0=chi0,
                        rhs=rhs, chi=chi))
        chi_c, map_c = chi, bmap
    return out
