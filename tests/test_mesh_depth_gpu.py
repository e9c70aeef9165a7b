"""GPU: the Poisson mesher at depths 8..10 (10 is the default of every way into it) against the float64 restatement
f64ref_mesh, stage by stage through the C ABI, each stage fed the kernel's own upstream values.

At R = 1024 the index widths change: vertex keys node * 8 + d pass 2^31 from z-layer 256 and 2^32 from layer 512, node
indices reach 2^30 and dual-cell ids 1023^3 - 1.  So the splat is compared bit for bit at depths 8..10 (sparse: the
non-zero entries of B), the float32 multigrid solve against the exact DCT solve with a geometric bound on the surface
it gives, the extraction, gathers and trim bit for bit over the whole grid at depths 8 and 9 and on z-slabs around
layers 0, 256, 512 and 1023 at depth 10, and smoothing and normals bit for bit.  Every test prints its GPU and host
times and the host's peak RSS."""
import hashlib
import resource
import time

import numpy as np
import pytest
import torch

import clouds
import f64ref_mesh as fm
from test_mesh_gpu import _cloud, _fr
from util import gpu, same

pytestmark = pytest.mark.gpu
SURFACE_N = 1_000_000  # points of the splat clouds that sample a surface
DEPTH10_SLABS = [(0, 3), (254, 259), (510, 515), (1021, 1024)]
CHI_TOL = 2e-5  # |chi_gpu - chi_exact| <= CHI_TOL * range(chi_exact), as at depth 4..6 (test_mesh_gpu)
T_TOL = 0.01  # |t_gpu - t_exact| in units of h on edges crossed in both fields, but for at most ODD_MAX of them
ODD_MAX = 1e-4  # edges crossed in only one field, and edges beyond T_TOL, each as a fraction of the crossed edges


def _rss_gb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20


def _log(tag, t_gpu, t_host, extra=""):
    print(f"[{tag}] gpu {t_gpu:.2f} s, host {t_host:.2f} s, host peak RSS {_rss_gb():.1f} GB{extra}")


def _sync_time(t0):
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def _rot(f):
    """Each triangle rolled so that its smallest entry comes first (the orientation is kept)."""
    f = np.asarray(f, np.int64)
    if f.size == 0:
        return f
    s = np.argmin(f, 1)
    return np.stack([f[np.arange(f.shape[0]), (s + q) % 3] for q in range(3)], 1)


# ---- splat ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth", [8, 9, 10])
@pytest.mark.parametrize("name", ["sphere", "two_spheres", "plane", "node_planes", "cube_faces", "copies",
                                  "bad_normals"])
def test_splat_bit_identical_deep(lib, name, depth):
    from g2pc import mesh
    p, n = _cloud(name, np.random.default_rng(100 + len(name)), depth, SURFACE_N)
    t0 = time.perf_counter()
    frame, B, cell, status = mesh.splat(gpu(p), gpu(n), depth)
    nz = torch.nonzero(B).squeeze(1)
    vals = B[nz].cpu().numpy()
    nz = nz.cpu().numpy()
    del B
    t_gpu = _sync_time(t0)
    f, cell, st = frame.cpu().numpy(), cell.cpu().numpy().astype(np.int64), status.cpu().numpy()
    t0 = time.perf_counter()
    nodes, vals_o, cell_o, skipped_o, fr = fm.splat_sparse(p, n, depth)
    t_host = time.perf_counter() - t0
    _log(f"splat {name} depth {depth}", t_gpu, t_host, f", {nodes.size} non-zero nodes, max |B| {np.abs(vals_o).max():.3e}")
    R = 1 << depth
    assert np.array_equal(nz, nodes) and np.array_equal(vals, vals_o)
    assert np.array_equal(cell, cell_o) and st[0] == skipped_o and st[1] == 0, st
    used = cell_o != fm.CELL_NONE
    assert (cell_o[used] < (R - 1) ** 3).all()
    assert f[0:3].tobytes() == fr["origin"].tobytes() and f[3] == fr["h"] and f[4] == fr["L"]
    assert f[5] == float(int(vals_o.sum())) / R ** 3 and f[6] == fr["extent"] and f[7] == R
    if name == "copies":
        assert np.abs(vals_o).max() > 2 ** 49
    if name == "bad_normals":
        assert skipped_o == 70
    if depth == 10 and name in ("sphere", "cube_faces"):
        assert nodes.max() >= 2 ** 29 and cell_o[used].max() >= 2 ** 29  # the upper half of the node / cell range


# ---- solve ----------------------------------------------------------------------------------------------------------
def _solve_cloud(name, rng):
    if name == "sphere":
        return clouds.sphere(2_000_000, rng)
    if name == "torus":
        p, n, _ = clouds.torus(1_000_000, rng)
        return p, n
    if name == "small_surface":  # a sphere of 0.05 x the box, and a tight 30-point cluster in the far corner
        p, n = clouds.sphere(200_000, rng, 0.05)
        q = clouds.clusters(rng, [[0.95, 0.95, 0.95]], [30], 5e-4)
        return np.r_[p, q], np.r_[n, rng.normal(size=q.shape).astype(np.float32)]
    raise KeyError(name)


def _host_b(B, frame):
    """b = (B - mean B) h 2^-33 in float64, copied from the device in slices (no host copy of the int64 B)."""
    total = int(B.sum().item())
    mean = float(total) / float(B.numel())
    scale = frame[3] * 2.0 ** -33
    b = np.empty(B.numel())
    step = 1 << 26
    for s in range(0, B.numel(), step):
        b[s:s + step] = (B[s:s + step].cpu().numpy().astype(np.float64) - mean) * scale
    return b


def _edge_ends(vkey, R):
    node = vkey >> 3
    d = vkey & 7
    i, j, k = node % R, (node // R) % R, node // (R * R)
    return node, ((k + (d >> 2)) * R + j + ((d >> 1) & 1)) * R + i + (d & 1)


@pytest.mark.parametrize("depth", [7, 8, 9, 10])
@pytest.mark.parametrize("name", ["sphere", "torus", "small_surface"])
def test_solve_against_dct(lib, name, depth):
    """Converges in < 40 cycles to |r| <= 1e-5 |b| (recomputed on the host in float64); chi within CHI_TOL of its range
    of the exact solution; and the surface it gives.  With e = max |d chi| + |d iso|: on an edge crossed in both fields
    |t_gpu - t_exact| |chi_b - chi_a| <= e (t_gpu D_gpu = t_exact D_exact + d iso - d chi_a with D = chi_b - chi_a,
    0 <= t_gpu <= 1), and an edge crossed in only one field has an end whose exact chi lies within e of the exact iso.
    An edge nearly tangent to the surface (small |chi_b - chi_a|) turns a small chi error into a large move along the
    edge: at depths 9 and 10 a few such edges move by more than T_TOL = 0.01 h (up to 0.044 h measured), so T_TOL and
    the count of one-sided edges are each held for all but ODD_MAX of the crossed edges."""
    from g2pc import mesh
    rng = np.random.default_rng(40 + depth)
    p, n = _solve_cloud(name, rng)
    if name == "small_surface" and depth == 7:
        from g2pc import outliers
        kept, _, _ = outliers.remove_statistical_outliers(gpu(p), None, gpu(n), mesh.NB_NEIGHBORS, 3.0)
        assert (kept.cpu().numpy() > 0.9).all(1).sum() == 30  # the cluster survives the mesher's outlier removal
    R = 1 << depth
    t0 = time.perf_counter()
    P, N = gpu(p), gpu(n)
    frame, B, cell, _ = mesh.splat(P, N, depth)
    chi, cycles, ratio = mesh.solve(B, frame, depth)
    t_solve = _sync_time(t0)
    f = frame.cpu().numpy()
    fr = _fr(f, depth)
    t0 = time.perf_counter()
    b = _host_b(B, f)
    del B
    host_ratio = fm.residual_ratio_slabs(chi.cpu().numpy(), b, R)
    t_host = time.perf_counter() - t0
    t0 = time.perf_counter()
    iso_g = float(mesh.iso_value(P, cell, frame, depth, chi)[1].item())  # chi made mean-free in place
    cg = chi.cpu().numpy()
    del chi
    t_gpu = t_solve + _sync_time(t0)
    t0 = time.perf_counter()
    x = fm.solve_dct(b, R)  # in place: b is gone
    cell = cell.cpu().numpy().astype(np.int64)
    iso_x = fm.iso_value(p, cell, fr, x)
    dchi = 0.0
    for s in range(0, x.size, 1 << 26):
        dchi = max(dchi, float(np.abs(cg[s:s + (1 << 26)].astype(np.float64) - x[s:s + (1 << 26)]).max()))
    rng_x = float(x.max() - x.min())
    diso = abs(iso_g - iso_x)
    bound = (dchi + diso) * (1 + 1e-9)
    both = one_sided = crossed = beyond = 0
    tmax = 0.0
    slab = 64
    for k0 in range(0, R, slab):
        k1 = min(k0 + slab, R)
        kg, tg = fm.crossed_edges(cg, R, iso_g, k0, k1)
        kx, tx = fm.crossed_edges(x, R, iso_x, k0, k1)
        common, ig, ix = np.intersect1d(kg, kx, assume_unique=True, return_indices=True)
        crossed += kx.size
        both += common.size
        if common.size:
            dt = np.abs(tg[ig] - tx[ix])
            tmax = max(tmax, float(dt.max()))
            beyond += int((dt > T_TOL).sum())
            a, e = _edge_ends(common, R)
            assert (dt * np.abs(x[e] - x[a]) <= bound).all(), k0
        odd = np.setxor1d(kg, kx, assume_unique=True)
        one_sided += odd.size
        if odd.size:
            a, e = _edge_ends(odd, R)
            near = np.minimum(np.abs(x[a] - iso_x), np.abs(x[e] - iso_x))
            assert (near <= bound).all(), (k0, float(near.max()), bound)
    t_host += time.perf_counter() - t0
    _log(f"solve {name} depth {depth}", t_gpu, t_host,
         f", {cycles} cycles, ratio {ratio:.2e} (host {host_ratio:.2e}), max |chi - dct| / range {dchi / rng_x:.2e}, "
         f"|iso - iso_dct| / range {diso / rng_x:.2e}, {crossed} crossed edges, max |t - t_dct| {tmax:.2e} h, "
         f"{beyond} beyond {T_TOL} h, {one_sided} crossed in one field only")
    assert cycles < mesh.MAX_CYCLES and ratio <= mesh.TOLERANCE
    assert abs(host_ratio - ratio) <= 1e-3 * ratio and dchi <= CHI_TOL * rng_x
    assert crossed > 0 and beyond <= ODD_MAX * crossed and one_sided <= ODD_MAX * crossed


# ---- extraction, gathers, trim, smoothing, normals ------------------------------------------------------------------
def _mesh_cloud(name, rng):
    if name == "sphere":  # its surface crosses z-layers 256 and 512 at depth 10
        return clouds.sphere(2_000_000, rng)
    if name == "cube_faces":  # the box faces with the longest extent along z: surface next to the bottom and the top
        p, n = _cloud("cube_faces", rng, 10, SURFACE_N)
        return np.ascontiguousarray(p[:, [1, 2, 0]]), np.ascontiguousarray(n[:, [1, 2, 0]])
    raise KeyError(name)


_RUNS = {}
# the box faces at depth 10 give 43 M vertices and 87 M triangles (the field crosses its iso far from the data): the
# restatement's one-ring lists of that mesh alone would take tens of GB, so their smoothing is checked at 8 and 9 only
SMOOTH_CASES = [("sphere", 8), ("sphere", 9), ("sphere", 10), ("cube_faces", 8), ("cube_faces", 9)]


def _smooth_iters(depth):
    return 1 if depth == 10 else 3


def _run(name, depth):
    """Every stage through the C ABI, each fed the previous one's output, kept on the host (computed once per cloud
    and depth)."""
    if (name, depth) in _RUNS:
        return _RUNS[name, depth]
    from g2pc import mesh
    rng = np.random.default_rng(60 + depth)
    p, n = _mesh_cloud(name, rng)
    colours = rng.integers(0, 256, p.shape)
    t0 = time.perf_counter()
    out = _device_run(p, n, colours, depth)
    t_gpu = time.perf_counter() - t0
    out.update(p=p, colours=colours, t_gpu=t_gpu)
    _RUNS[name, depth] = out
    print(f"[stages {name} depth {depth}] gpu {t_gpu:.2f} s (with copies to the host), {out['cycles']} cycles, "
          f"ratio {out['ratio']:.2e}, {out['vkey'].size} vertices, {out['faces'].shape[0]} triangles, "
          f"{out['tfaces'].shape[0]} after the trim")
    return out


def _device_run(p, n, colours, depth):
    from g2pc import mesh
    pts, nrm, col = gpu(p), gpu(n), gpu(colours, np.int32)
    frame, B, cell, _ = mesh.splat(pts, nrm, depth)
    chi, cycles, ratio = mesh.solve(B, frame, depth)
    iso = mesh.iso_value(pts, cell, frame, depth, chi)
    out = dict(frame=frame.cpu().numpy(), cell=cell.cpu().numpy().astype(np.int64), cycles=cycles, ratio=ratio,
               chi=chi.cpu().numpy(), iso=iso.cpu().numpy())
    vkey, vt, vpos, faces = mesh.extract(chi, depth, frame, iso, B)
    del chi
    dens, vcol = mesh.gather(pts, col, cell, frame, depth, vkey, vt, B)
    del B
    out.update(vkey=vkey.cpu().numpy(), vt=vt.cpu().numpy(), vpos=vpos.cpu().numpy(), faces=faces.cpu().numpy(),
               dens=dens.cpu().numpy(), vcol=vcol.cpu().numpy())
    d2, p2, c2, f2, keep, thr = mesh.trim(dens, vpos, vcol, faces)
    out.update(keep=keep.cpu().numpy().astype(bool), thr=float(thr.item()), tdens=d2.cpu().numpy(),
               tpos=p2.cpu().numpy(), tcol=c2.cpu().numpy(), tfaces=f2.cpu().numpy())
    mesh.smooth(p2, f2, _smooth_iters(depth))
    v, vn = mesh.vertex_normals(p2, f2)
    out.update(spos=p2.cpu().numpy(), verts=v.cpu().numpy(), normals=vn.cpu().numpy())
    return out


@pytest.mark.parametrize("depth", [8, 9, 10])
@pytest.mark.parametrize("name", ["sphere", "cube_faces"])
def test_extraction_gather_trim_deep(lib, name, depth):
    """Fed the kernel's chi and iso: vertex keys, t, positions, triangles, densities and colours bit for bit (whole grid
    at depths 8 and 9; at depth 10 the z-slabs of DEPTH10_SLABS, where keys pass 2^31 and 2^32); the trim's keep mask,
    threshold and kept mesh bit for bit over the whole mesh."""
    s = _run(name, depth)
    p, colours = s["p"], s["colours"]
    fr = _fr(s["frame"], depth)
    R = 1 << depth
    chi = s.pop("chi")  # the last user of the dense field
    t0 = time.perf_counter()
    iso = s["iso"][1]
    iso_o = fm.iso_value(p, s["cell"], fr, chi)
    assert abs(iso - iso_o) <= 1e-12 * abs(iso_o)
    gk, gt, gp = s["vkey"], s["vt"], s["vpos"]
    gf = gk[s["faces"].astype(np.int64)]  # triangles as vertex-key triples
    if depth < 10:
        vkey, vt, vpos, faces = fm.marching_tetrahedra(chi, R, iso, fr["origin"], fr["h"])
        assert np.array_equal(gk, vkey) and same(gt, vt) and same(gp, vpos)
        assert np.array_equal(_rot(s["faces"]), _rot(faces))
        sel = slice(None)
    else:
        layer = (gk >> 3) // (R * R)
        cube_layer = (gf >> 3).min(1) // (R * R)  # every triangle has an edge whose lower end is its cube's corner 0
        sel = np.zeros(gk.size, bool)
        counts = []
        for k0, k1 in DEPTH10_SLABS:
            vkey, vt, vpos, fkeys = fm.marching_tetrahedra(chi, R, iso, fr["origin"], fr["h"], k0, k1)
            vs = (layer >= k0) & (layer < k1)
            fs = (cube_layer >= k0) & (cube_layer < k1)
            assert np.array_equal(gk[vs], vkey), (k0, k1)
            assert same(gt[vs], vt) and same(gp[vs], vpos), (k0, k1)
            assert np.array_equal(_rot(gf[fs]), _rot(fkeys)), (k0, k1)
            sel |= vs
            counts.append((k0, k1, vkey.size, fkeys.shape[0]))
        print(f"[depth 10 slabs {name}] (k0, k1, vertices, triangles): {counts}")
        if name == "sphere":
            assert gk[sel].max() >= 2 ** 32 and ((gk[sel] >= 2 ** 31) & (gk[sel] < 2 ** 32)).any()
        vkey, vt = gk[sel], gt[sel]
    del chi
    dens, vcol = fm.vertex_density_colour(p, colours, s["cell"], fr, vkey, vt)
    assert same(s["dens"][sel], dens) and np.array_equal(s["vcol"][sel], vcol)
    # the trim is global: on the kernel's densities (equal to the restatement's wherever those were computed)
    d2, p2, c2, f2, keep, thr = fm.trim(s["dens"], gp, s["vcol"], s["faces"].astype(np.int64))
    assert thr == np.quantile(s["dens"], 0.1) and s["thr"] == thr and np.array_equal(s["keep"], keep)
    assert same(s["tdens"], d2) and same(s["tpos"], p2) and np.array_equal(s["tcol"], c2)
    assert np.array_equal(s["tfaces"].astype(np.int64), f2)
    _log(f"extract / gather / trim {name} depth {depth}", s["t_gpu"], time.perf_counter() - t0,
         f", {int(sel.sum()) if depth == 10 else gk.size} vertices compared, threshold {thr:.6e}")
    if (name, depth) not in SMOOTH_CASES:
        del _RUNS[name, depth]


@pytest.mark.parametrize("name,depth", SMOOTH_CASES)
def test_smoothing_and_normals_deep(lib, name, depth):
    """Bit for bit: both kernels and the restatement evaluate every operation in float64 with round-to-nearest and no
    FMA, neighbours and incident triangles in ascending order."""
    s = _run(name, depth)
    t0 = time.perf_counter()
    sm = fm.smooth(s["tpos"], s["tfaces"], _smooth_iters(depth))
    assert same(s["spos"], sm)
    nr = fm.vertex_normals(s["spos"], s["tfaces"])
    assert same(s["normals"], nr.astype(np.float32)) and same(s["verts"], s["spos"].astype(np.float32))
    _log(f"smooth x{_smooth_iters(depth)} / normals {name} depth {depth}", s["t_gpu"], time.perf_counter() - t0,
         f", {sm.shape[0]} vertices, max move {np.abs(sm - s['tpos']).max() / s['frame'][3]:.3f} h")
    del _RUNS[name, depth]


def test_unconverged_solve_is_reported(lib, monkeypatch):
    """poisson_mesh warns when the solve stops at its cycle cap above the tolerance (here a cap of 1 cycle)."""
    from g2pc import mesh
    p, n = clouds.sphere(50_000, np.random.default_rng(2))
    full = mesh.solve
    monkeypatch.setattr(mesh, "solve", lambda B, frame, depth: full(B, frame, depth, max_cycles=1))
    with pytest.warns(RuntimeWarning, match="stopped after 1 V-cycles"):
        mesh.poisson_mesh(gpu(p), gpu(n), depth=6)


def test_determinism_depth10(lib):
    rng = np.random.default_rng(70)
    p, n = clouds.sphere(2_000_000, rng)
    colours = rng.integers(0, 256, p.shape)
    t0 = time.perf_counter()
    runs = []
    for _ in range(2):
        out = _device_run(p, n, colours, 10)
        runs.append({k: (v.dtype.str, v.shape, hashlib.sha256(v.tobytes()).hexdigest()) if isinstance(v, np.ndarray)
                     else v for k, v in out.items()})
        del out
    t_gpu = time.perf_counter() - t0
    assert runs[0] == runs[1]
    _log("determinism depth 10", t_gpu, 0.0, f", {runs[0]['vkey'][1][0]} vertices")


# ---- the trim, smoothing and normals entry points on hand-built inputs ----------------------------------------------
def _trim_case(dens, faces, vcol=True):
    from g2pc import mesh
    rng = np.random.default_rng(dens.size)
    m = dens.size
    vpos = rng.normal(size=(m, 3))
    col = rng.integers(0, 256, (m, 3)).astype(np.uint8)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    d2, p2, c2, f2, keep, thr = mesh.trim(gpu(dens), gpu(vpos), gpu(col) if vcol else None, gpu(faces, np.int32))
    o = fm.trim(dens, vpos, col if vcol else None, faces)
    assert float(thr.item()) == o[5] == np.quantile(dens, 0.1), (m, float(thr.item()), o[5])
    assert np.array_equal(keep.cpu().numpy().astype(bool), o[4])
    assert same(d2.cpu().numpy(), o[0]) and same(p2.cpu().numpy(), o[1])
    assert np.array_equal(f2.cpu().numpy().astype(np.int64), o[3])
    if vcol:
        assert np.array_equal(c2.cpu().numpy(), o[2])
    return o


def _branches_differ(d):
    """Whether numpy's two forms of the linear quantile, a + (b - a) g and b - (b - a)(1 - g), round differently here."""
    s = np.sort(d)
    vi = (d.size - 1) * 0.1
    lo = int(np.floor(vi))
    a, b, g = s[lo], s[min(lo + 1, d.size - 1)], vi - lo
    return a + (b - a) * g != b - (b - a) * (1 - g)


def test_trim_edge_cases(lib):
    """m = 1, 2, 10, 11, 12, 21 (integral virtual index at 11 and 21, g >= 0.5 at 10 and 2 vs 12); equal densities;
    ties exactly at the threshold; zero densities; no triangles; triangles on removed vertices only."""
    rng = np.random.default_rng(3)
    for m in (1, 2, 10, 11, 12, 21):
        d = rng.random(m)
        faces = rng.integers(0, m, (2 * m, 3))
        _trim_case(d, faces)
        _trim_case(d, np.zeros((0, 3)))
        _trim_case(d, faces, vcol=False)
    # m = 10 takes the g >= 0.5 branch (g = 0.9): a case where the two branches round differently
    seed = next(s for s in range(1000) if _branches_differ(np.random.default_rng(s).random(10)))
    _trim_case(np.random.default_rng(seed).random(10), rng.integers(0, 10, (15, 3)))
    _trim_case(np.full(37, 0.25), rng.integers(0, 37, (50, 3)))  # all equal: every vertex kept
    ties = np.r_[np.full(4, 0.5), np.full(3, 0.125), np.linspace(0.6, 0.9, 4)]  # m = 11: threshold = sorted[1]
    o = _trim_case(rng.permutation(ties), rng.integers(0, 11, (20, 3)))
    assert o[5] == 0.125 and o[4].all()  # vertices exactly at the threshold are kept
    o = _trim_case(np.r_[np.zeros(5), rng.random(16)], rng.integers(0, 21, (30, 3)))  # zero densities
    assert o[5] == 0.0 and o[4].all()
    d = np.r_[np.zeros(3), np.ones(18)]
    d[:3] = [0.0, 5e-324, 1e-300]  # m = 21: threshold = sorted[2] = 1e-300, below it a subnormal and 0
    o = _trim_case(d, [[0, 1, 2], [2, 1, 0], [0, 0, 1], [3, 4, 5], [1, 5, 6]])  # triangles on removed vertices
    assert not o[4][:2].any() and o[3].shape[0] == 1


def _smooth_abi(vpos, faces, iterations):
    from g2pc import capi, mesh
    v = gpu(vpos)
    f = gpu(np.asarray(faces, np.int64).reshape(-1, 3), np.int32)
    m, t = v.shape[0], f.shape[0]
    ws = capi.workspace(capi.load().g2pc_mesh_smooth_workspace_bytes(m, t), v.device)
    capi.call("g2pc_mesh_smooth", capi.ptr(v), m, capi.ptr(f), t, int(iterations), capi.ptr(ws), ws.numel(),
              capi.stream_ptr(v.device))
    return v.cpu().numpy()


def test_smooth_edge_cases(lib):
    """Isolated vertices stay; duplicate triangles (and both orientations of one) count each neighbour once; coincident
    neighbours get weight 1e12; 0, 1 and 7 iterations (odd counts end in the workspace buffer)."""
    rng = np.random.default_rng(5)
    v = rng.normal(size=(40, 3))
    v[7] = v[3]  # coincident neighbours
    v[8] = v[3]
    f = rng.integers(0, 30, (50, 3))  # vertices 30..39 isolated
    f = np.r_[f, [[3, 7, 8], [3, 7, 8], [8, 7, 3], [3, 7, 8]], f[:10], f[:5, ::-1]]
    for it in (0, 1, 2, 7):
        got = _smooth_abi(v, f, it)
        want = fm.smooth(v, f, it)
        assert same(got, want), it
        assert same(got[30:], v[30:])
    got = _smooth_abi(v, np.zeros((0, 3)), 3)  # no triangles: nothing moves
    assert same(got, v)


def test_normals_edge_cases(lib):
    """Zero-area triangles add nothing; two opposite triangles cancel to a zero normal; a vertex of no triangle gets 0."""
    from g2pc import mesh
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [2, 0, 0], [3, 0, 0], [5, 5, 5], [0.5, 0.5, 1e-9], [9, 9, 9]])
    f = np.array([[0, 1, 2], [0, 2, 1],  # cancel: vertices 0, 1, 2 end at zero
                  [1, 3, 4], [3, 3, 5],  # zero area: collinear, and a repeated vertex
                  [0, 1, 6], [6, 6, 6]])
    vp = gpu(v)
    verts, nrm = mesh.vertex_normals(vp, gpu(f, np.int32))
    want = fm.vertex_normals(v, f)
    assert same(nrm.cpu().numpy(), want.astype(np.float32)) and same(verts.cpu().numpy(), v.astype(np.float32))
    got = nrm.cpu().numpy()
    assert (got[[2, 3, 4, 5, 7]] == 0).all() and (got[[0, 1, 6]] != 0).any(1).all()
