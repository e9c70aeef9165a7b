"""Plain numpy / scipy float64 restatement of the decimation's rules (DESIGN.md §2, N9): plane quadrics, free flags,
unique edges and candidates, the 2-ring minimum selection, the collapses and the final compaction.  Written from the
stated rules, not from the kernels: every float64 expression is evaluated in the order the rules state (numpy never
fuses a multiply and an add), and the quadric sums run in ascending face id (np.add.at applies its updates in index
order), so the results can be compared with the kernels bit for bit."""
import numpy as np
import scipy.sparse as sp
from scipy.sparse.csgraph import connected_components

FAN_MAX = 128
KEY_NONE = np.uint64(0xFFFFFFFFFFFFFFFF)
LOW = np.uint64(0xFFFFFFFF)


def dot3(a, b):
    return (a[:, 0] * b[:, 0] + a[:, 1] * b[:, 1]) + a[:, 2] * b[:, 2]


def face_normals(p0, p1, p2):
    """cross(p1 - p0, p2 - p0) per row."""
    u, w = p1 - p0, p2 - p0
    return np.stack([u[:, 1] * w[:, 2] - u[:, 2] * w[:, 1], u[:, 2] * w[:, 0] - u[:, 0] * w[:, 2],
                     u[:, 0] * w[:, 1] - u[:, 1] * w[:, 0]], 1)


def quadrics(p, f):
    """(m,10) Q_v = sum over v's faces in ascending id of [n n^T, -n (n . p0); (n . p0)^2] / (2 |n|); |n| = 0 adds 0."""
    p, f = np.asarray(p, np.float64), np.asarray(f, np.int64)
    Q = np.zeros((p.shape[0], 10))
    if f.size == 0:
        return Q
    p0 = p[f[:, 0]]
    n = face_normals(p0, p[f[:, 1]], p[f[:, 2]])
    ln = np.sqrt(dot3(n, n))
    ok = ln > 0
    n, p0, s = n[ok], p0[ok], 2.0 * ln[ok]
    d = dot3(n, p0)
    K = np.stack([n[:, 0] * n[:, 0], n[:, 0] * n[:, 1], n[:, 0] * n[:, 2], n[:, 1] * n[:, 1], n[:, 1] * n[:, 2],
                  n[:, 2] * n[:, 2], -(n[:, 0] * d), -(n[:, 1] * d), -(n[:, 2] * d), d * d], 1) / s[:, None]
    np.add.at(Q, f[ok].reshape(-1), np.repeat(K, 3, axis=0))
    return Q


def free_flags(f, m, fan_max=FAN_MAX):
    """free (m,) bool: 1..fan_max incident faces, every edge at the vertex used by exactly two of them, and one closed
    fan (the link, a graph on the neighbours with one edge per face, is connected).  fan_max=None: no cap."""
    f = np.asarray(f, np.int64)
    free = np.zeros(m, bool)
    if f.size == 0:
        return free
    V = np.concatenate([f[:, 0], f[:, 1], f[:, 2]])
    X = np.concatenate([f[:, 1], f[:, 2], f[:, 0]])
    Y = np.concatenate([f[:, 2], f[:, 0], f[:, 1]])
    nf = np.bincount(V, minlength=m)
    kx, ky = V << 32 | X, V << 32 | Y
    uniq, cnt = np.unique(np.concatenate([kx, ky]), return_counts=True)
    bad = np.zeros(m, bool)
    bad[uniq[cnt != 2] >> 32] = True
    ix, iy = np.searchsorted(uniq, kx), np.searchsorted(uniq, ky)
    g = sp.coo_matrix((np.ones(ix.size), (ix, iy)), shape=(uniq.size, uniq.size))
    _, lab = connected_components(g, directed=False)
    owner = uniq >> 32
    comp = np.bincount(np.unique(owner << 32 | lab) >> 32, minlength=m)
    free = (nf >= 1) & ~bad & (comp == 1)
    if fan_max is not None:
        free &= nf <= fan_max
    return free


def cost(q, v):
    """max(0, v^T A v + 2 b^T v + c) per row: Av_i = (A_i0 v0 + A_i1 v1) + A_i2 v2, then (v . Av + 2 (b . v)) + c."""
    A = [[q[:, 0], q[:, 1], q[:, 2]], [q[:, 1], q[:, 3], q[:, 4]], [q[:, 2], q[:, 4], q[:, 5]]]
    Av = np.stack([(A[i][0] * v[:, 0] + A[i][1] * v[:, 1]) + A[i][2] * v[:, 2] for i in range(3)], 1)
    r = (dot3(v, Av) + 2.0 * dot3(q[:, 6:9], v)) + q[:, 9]
    return np.where(r > 0.0, r, 0.0)


def place(Q, p, a, b):
    """(v (k,3), cost (k,)) of the merged vertex of edges (a, b)."""
    q = Q[a] + Q[b]
    pa, pb = p[a], p[b]
    A00, A01, A02, A11, A12, A22 = (q[:, i] for i in range(6))
    C00 = A11 * A22 - A12 * A12
    C01 = A02 * A12 - A01 * A22
    C02 = A01 * A12 - A02 * A11
    C11 = A00 * A22 - A02 * A02
    C12 = A01 * A02 - A00 * A12
    C22 = A00 * A11 - A01 * A01
    det = (A00 * C00 + A01 * C01) + A02 * C02
    nA = np.abs(A00)
    for x in (A01, A02, A11, A12, A22):
        nA = np.maximum(nA, np.abs(x))
    C = [[C00, C01, C02], [C01, C11, C12], [C02, C12, C22]]
    mid = (pa + pb) * 0.5
    with np.errstate(all="ignore"):
        s = np.stack([(-((C[i][0] * q[:, 6] + C[i][1] * q[:, 7]) + C[i][2] * q[:, 8])) / det for i in range(3)], 1)
        d, e = s - mid, pb - pa
        ok = (np.abs(det) > 1e-12 * ((nA * nA) * nA)) & (dot3(d, d) <= dot3(e, e))
    v, c = pa.copy(), cost(q, pa)
    for alt in (pb, mid):
        ca = cost(q, alt)
        better = ca < c
        v[better], c[better] = alt[better], ca[better]
    okv = np.where(ok[:, None], s, 0.0)
    v[ok], c[ok] = okv[ok], cost(q, okv)[ok]
    return v, c


def incidence(f, m):
    """(ptr (m+1,), faces of each vertex in ascending id)."""
    V = np.asarray(f, np.int64).reshape(-1)
    F = np.repeat(np.arange(f.shape[0]), 3)
    order = np.lexsort((F, V))
    return np.searchsorted(V[order], np.arange(m + 1)), F[order]


def select(p, f, Q, free):
    """One round's selection: dict(ea, eb (E,) edge endpoints by id, key (E,) uint64 (KEY_NONE: not a candidate),
    edges, candidates, selected (counts), sel (selected keys, ascending))."""
    p, f = np.asarray(p, np.float64), np.asarray(f, np.int64)
    m, t = p.shape[0], f.shape[0]
    assert m < 1 << 21, "face keys pack three 21-bit indices"
    a3 = f.reshape(-1)
    b3 = f[:, [1, 2, 0]].reshape(-1)
    K = np.minimum(a3, b3) << 32 | np.maximum(a3, b3)
    F = np.repeat(np.arange(t), 3)
    order = np.argsort(K, kind="stable")
    ek, ev = K[order], F[order]
    head = np.r_[True, ek[1:] != ek[:-1]]
    starts = np.nonzero(head)[0]
    E = starts.size
    runs = np.diff(np.r_[starts, ek.size])
    ea, eb = ek[starts] >> 32, ek[starts] & 0xFFFFFFFF
    key = np.full(E, KEY_NONE, np.uint64)
    cand = free[ea] & free[eb] & (runs == 2)
    idx = np.nonzero(cand)[0]
    f1, f2 = ev[starts[idx]], ev[starts[idx] + 1]
    a, b = ea[idx], eb[idx]
    c, d = f[f1].sum(1) - a - b, f[f2].sum(1) - a - b
    # link condition: exactly c and d in common, and {a,c,d}, {b,c,d} not both faces
    rows = np.concatenate([a3, b3])
    cols = np.concatenate([b3, a3])
    adj = sp.csr_matrix((np.ones(rows.size), (rows, cols)), shape=(m, m))
    adj.data[:] = 1.0
    common = np.asarray(adj[a].multiply(adj[b]).sum(1)).reshape(-1) if idx.size else np.zeros(0)
    fs = np.sort(f, 1)
    fkeys = np.unique(fs[:, 0] << 42 | fs[:, 1] << 21 | fs[:, 2])

    def has(x, y, z):
        s3 = np.sort(np.stack([x, y, z], 1), 1)
        q = s3[:, 0] << 42 | s3[:, 1] << 21 | s3[:, 2]
        pos = np.minimum(np.searchsorted(fkeys, q), fkeys.size - 1)
        return fkeys[pos] == q

    ok = (c != d) & (common == 2) & ~(has(a, c, d) & has(b, c, d))
    v, cst = place(Q, p, a, b)
    # fold-over: every face of a or b other than f1, f2 keeps dot(n_old, n_new) > 0 with the endpoint at v
    ptr, inc = incidence(f, m)
    j = np.concatenate([np.arange(idx.size), np.arange(idx.size)])
    u = np.concatenate([a, b])
    lens = ptr[u + 1] - ptr[u]
    jr = np.repeat(j, lens)
    ur = np.repeat(u, lens)
    g = inc[np.repeat(ptr[u], lens) + (np.arange(lens.sum()) - np.repeat(np.cumsum(lens) - lens, lens))]
    use = (g != f1[jr]) & (g != f2[jr])
    jr, ur, g = jr[use], ur[use], g[use]
    old = [p[f[g, s]] for s in range(3)]
    new = [np.where((f[g, s] == ur)[:, None], v[jr], old[s]) for s in range(3)]
    flip = ~(dot3(face_normals(*old), face_normals(*new)) > 0.0)
    ok &= np.bincount(jr[flip], minlength=idx.size) == 0
    kk = cst.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32) | idx.astype(np.uint64)
    key[idx[ok]] = kk[ok]
    M1 = np.full(m, KEY_NONE, np.uint64)
    ci = idx[ok]
    np.minimum.at(M1, ea[ci], key[ci])
    np.minimum.at(M1, eb[ci], key[ci])
    M2 = M1.copy()
    np.minimum.at(M2, ea, M1[eb])
    np.minimum.at(M2, eb, M1[ea])
    sel = (key != KEY_NONE) & (key == M2[ea]) & (key == M2[eb])
    return dict(ea=ea, eb=eb, key=key, edges=E, candidates=int(ok.sum()), selected=int(sel.sum()),
                sel=np.sort(key[sel]))


def decimate(vpos, faces, target, colours=None, densities=None, check=False):
    """(vpos, faces, colours, densities, info) with info = dict(quadrics, free (after the preparation), rounds (per
    round: edges, candidates, selected, keys, ab, vpos, quadrics, merged, colour_sums, density_sums, faces), reached).
    check: assert each round that the free flags are unchanged (without the fan cap), that no endpoint of a selected
    edge lies in the closed neighbourhood of another's, and that each collapse removes two faces."""
    p = np.array(vpos, np.float64)
    f = np.array(faces, np.int64).reshape(-1, 3)
    m, t = p.shape[0], f.shape[0]
    if target >= t:
        return vpos, faces, colours, densities, dict(rounds=[], reached=True)
    Q = quadrics(p, f)
    free = free_flags(f, m)
    topo0 = free_flags(f, m, fan_max=None)
    info = dict(quadrics=Q.copy(), free=free.copy(), rounds=[], reached=False)
    alive = np.ones(m, bool)
    merged = np.ones(m, np.int64)
    csum = None if colours is None else np.asarray(colours).astype(np.int64)
    dsum = None if densities is None else np.array(densities, np.float64)
    while t > target:
        s = select(p, f, Q, free)
        if s["selected"] == 0:
            break
        k = min(s["selected"], (t - target + 1) // 2)
        keys = s["sel"][:k]
        ids = (keys & LOW).astype(np.int64)
        a, b = s["ea"][ids], s["eb"][ids]
        if check:
            ptr, inc = incidence(f, m)
            owner = np.full(m, -1)
            owner[a], owner[b] = np.arange(k), np.arange(k)
            for u in (a, b):
                for j in range(k):
                    nb = f[inc[ptr[u[j]]:ptr[u[j] + 1]]].reshape(-1)
                    assert ((owner[nb] == -1) | (owner[nb] == j)).all()
        v, _ = place(Q, p, a, b)
        p[a] = v
        Q[a] = Q[a] + Q[b]
        merged[a] += merged[b]
        if csum is not None:
            csum[a] += csum[b]
        if dsum is not None:
            dsum[a] = dsum[a] + dsum[b]
        alive[b] = False
        vmap = np.arange(m)
        vmap[b] = a
        nf = vmap[f]
        keep = (nf[:, 0] != nf[:, 1]) & (nf[:, 1] != nf[:, 2]) & (nf[:, 0] != nf[:, 2])
        f = nf[keep]
        if check:
            assert f.shape[0] == t - 2 * k
            topo = free_flags(f, m, fan_max=None)
            assert (topo[alive] == topo0[alive]).all()
        t = f.shape[0]
        info["rounds"].append(dict(edges=s["edges"], candidates=s["candidates"], selected=s["selected"], keys=keys,
                                   ab=np.stack([a, b], 1), vpos=p.copy(), quadrics=Q.copy(), merged=merged.copy(),
                                   colour_sums=None if csum is None else csum.copy(),
                                   density_sums=None if dsum is None else dsum.copy(), faces=f.copy()))
    info["reached"] = t <= target
    keep = np.nonzero(alive)[0]
    pos = np.cumsum(alive) - 1
    n = merged[keep]
    cols = None if csum is None else ((2 * csum[keep] + n[:, None]) // (2 * n[:, None])).astype(np.uint8)
    dens = None if dsum is None else dsum[keep] / n
    return p[keep], pos[f], cols, dens, info


# ---- hand meshes ----------------------------------------------------------------------------------------------------
def tetrahedron():
    v = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64)
    return v, np.array([[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]])


def octahedron():
    v = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    f = [[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]]
    return v, np.array(f)


def icosphere(subdivisions=3):
    t = (1.0 + 5.0 ** 0.5) / 2.0
    v = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    f = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
         [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
         [8, 6, 7], [9, 8, 1]]
    v = [np.array(x, np.float64) / np.linalg.norm(x) for x in v]
    for _ in range(subdivisions):
        mid, nf = {}, []

        def midpoint(i, j):
            key = (min(i, j), max(i, j))
            if key not in mid:
                x = v[i] + v[j]
                v.append(x / np.linalg.norm(x))
                mid[key] = len(v) - 1
            return mid[key]

        for a, b, c in f:
            ab, bc, ca = midpoint(a, b), midpoint(b, c), midpoint(c, a)
            nf += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        f = nf
    return np.array(v), np.array(f)


def torus(nu=24, nv=12, R=2.0, r=0.7):
    u, w = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    th, ph = 2 * np.pi * u / nu, 2 * np.pi * w / nv
    v = np.stack([(R + r * np.cos(ph)) * np.cos(th), (R + r * np.cos(ph)) * np.sin(th), r * np.sin(ph)], -1)
    idx = lambda i, j: (i % nu) * nv + (j % nv)
    f = []
    for i in range(nu):
        for j in range(nv):
            f += [[idx(i, j), idx(i + 1, j), idx(i + 1, j + 1)], [idx(i, j), idx(i + 1, j + 1), idx(i, j + 1)]]
    return v.reshape(-1, 3), np.array(f)


def grid(n=12, bump=0.0):
    """An open (n+1)^2-vertex grid in z = bump * sin(x) sin(y)."""
    y, x = np.meshgrid(np.arange(n + 1), np.arange(n + 1), indexing="ij")
    v = np.stack([x, y, bump * np.sin(x * 0.7) * np.sin(y * 0.5)], -1).reshape(-1, 3).astype(np.float64)
    idx = lambda i, j: i * (n + 1) + j
    f = []
    for i in range(n):
        for j in range(n):
            f += [[idx(i, j), idx(i, j + 1), idx(i + 1, j + 1)], [idx(i, j), idx(i + 1, j + 1), idx(i + 1, j)]]
    return v, np.array(f)


def boundary_edges(f):
    """Directed boundary edges (used once, and not in the other direction) as a sorted (k,2) array."""
    f = np.asarray(f, np.int64)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    und = np.sort(d, 1)
    u, inv, cnt = np.unique(und, axis=0, return_inverse=True, return_counts=True)
    return np.sort(d[cnt[inv.reshape(-1)] == 1], 0)
