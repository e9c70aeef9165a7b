"""GPU: the Poisson mesher's narrow-band levels (s12_mesh_band.cu through g2pc/mesh.py) against the float64
restatement f64ref_mesh_band, stage by stage, each stage fed the kernel's own upstream outputs.

Bit for bit: brick maps, brick lists, the lost-seed count, band B, ghosts, initial guess and right-hand side, the
extraction (keys, triangles, t, positions), densities, colours, trim mask and threshold.  The float32 conjugate-gradient
solve against a float64 solve with the same right-hand side, within CHI_TOL of chi's range; the iso-value to 1e-12.
End to end: closed surfaces, topology, distance to the true surface and to the dense depth-10 mesh, repeatability on
poisoned memory, refusals, and a 10 M-point shell at (10, 12).  Each test prints its solver iterations."""
import os
import time

import numpy as np
import pytest
import torch
from scipy.spatial import cKDTree

import clouds
import f64ref_mesh as fm
import f64ref_mesh_band as fb
from sanitizer_harness import assert_repeatable, check_target
from util import gpu, same

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "mesh_band_sanitizer_target.py")
CHI_TOL = 2e-5  # |chi_gpu - chi_f64| <= CHI_TOL * range(chi_f64), same ghosts and right-hand side: measured <= 7.7e-6


def _small_pair(rng, n=20_000, r=0.01):
    """Two small spheres one unit apart: the grid spans the pair, so each sphere's band stays small at depth 12."""
    a, na = clouds.sphere(n, rng, r, (0.0, 0.0, 0.0))
    b, nb = clouds.sphere(n // 2, rng, r * 0.8, (1.0, 0.3, -0.2))
    return np.r_[a, b], np.r_[na, nb]


def _cloud(name, rng):
    if name == "sphere":
        return clouds.sphere(20_000, rng, 1.0, (0.1, -0.2, 0.05))
    if name == "torus":
        p, n, _ = clouds.torus(20_000, rng)
        return p, n
    if name == "small_pair":
        return _small_pair(rng)
    if name == "plane":  # a square of the plane z = 0.1 inside a far cluster's frame
        p = clouds.plane(40_000, rng, 0.0, 0.05, 0.1)
        q = clouds.sphere(2_000, rng, 0.01, (1.0, 1.0, 1.0))
        return np.r_[p, q[0]], np.r_[np.tile(np.float32([0, 0, 1]), (p.shape[0], 1)), q[1]]
    if name == "box_face":  # the six faces of a small box, normals outward
        s = 0.02
        p = rng.uniform(-s, s, (30_000, 3))
        ax = rng.integers(0, 3, p.shape[0])
        sg = np.sign(rng.normal(size=p.shape[0]))
        p[np.arange(p.shape[0]), ax] = sg * s
        nrm = np.zeros_like(p)
        nrm[np.arange(p.shape[0]), ax] = sg
        q = clouds.sphere(2_000, rng, 0.01, (1.0, 0.5, 0.5))
        return np.r_[p.astype(np.float32), q[0]], np.r_[nrm.astype(np.float32), q[1]]
    raise ValueError(name)


def _np(t):
    return t.cpu().numpy()


STAGE_CASES = [(5, 7, "sphere"), (7, 9, "torus"), (10, 11, "small_pair"), (10, 12, "small_pair"), (10, 12, "plane"),
               (10, 12, "box_face")]


@pytest.mark.parametrize("depth,band_depth,name", STAGE_CASES)
def test_stages_against_restatement(lib, depth, band_depth, name):
    from g2pc import mesh
    rng = np.random.default_rng(depth * 100 + band_depth)
    p, n = _cloud(name, rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    t0 = time.perf_counter()
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=depth, band_depth=band_depth, return_debug=True,
                               laplacian_iters=3)
    torch.cuda.synchronize()
    t_gpu = time.perf_counter() - t0
    pts, nrm, cell = _np(dbg["points"]), _np(dbg["normals"]), _np(dbg["cell"]).astype(np.int64)
    parent_chi, parent_map = _np(dbg["dense_chi"]), None
    for lv in dbg["levels"]:
        D = lv["depth"]
        fr = fb.band_frame(pts, D)
        f = _np(lv["frame"])
        assert f[3] == fr["h"] and f[7] == 1 << D and f[0:3].tobytes() == fr["origin"].tobytes()
        bmap, blist, lost = fb.bricks(pts, nrm, D, parent_map)
        assert lost == 0
        assert same(_np(lv["map"]), bmap) and same(_np(lv["bricks"]), blist)
        B, outside = fb.band_B(pts, nrm, D, bmap, blist.size)
        assert outside == 0 and same(_np(lv["B"]), B)
        g, chi0, rhs = fb.ghosts(parent_chi, parent_map, D, bmap, blist, B, fr["h"])
        assert same(_np(lv["ghost"]), g) and same(_np(lv["chi0"]), chi0) and same(_np(lv["rhs"]), rhs)
        chi = _np(lv["chi"])
        ratio = fb.residual_ratio(chi, rhs, bmap, blist, D)
        msg = (f"[{name} ({depth}, {band_depth}) level {D}] {blist.size} bricks, {blist.size * 512} nodes, "
               f"{lv['iterations']} CG iterations, ratio {lv['ratio']:.2e} (f64 {ratio:.2e})")
        assert ratio <= 1.5 * mesh.BAND_TOLERANCE and lv["ratio"] <= mesh.BAND_TOLERANCE, msg
        if blist.size * 512 <= 3_000_000:
            ref = fb.solve(rhs.astype(np.float64), bmap, blist, D, chi0)
            err = np.abs(chi - ref).max() / (ref.max() - ref.min())
            msg += f", |chi - chi_f64| / range {err:.2e}"
            assert err <= CHI_TOL, msg
        print(msg)
        parent_chi, parent_map = chi, bmap
    # iso, extraction, gathers, trim at band_depth, from the kernel's chi
    fr = fb.band_frame(pts, band_depth)
    iso = _np(dbg["iso"])
    iso_ref = fb.iso_value(pts, cell, fr, parent_map, parent_chi)
    assert iso[0] == 0.0 and abs(iso[1] - iso_ref) <= 1e-12 * max(abs(iso_ref), 1e-300) + 1e-300
    lv = dbg["levels"][-1]
    vkey, vt, vpos, faces = fb.marching_tetrahedra(parent_chi, parent_map, _np(lv["bricks"]), fr, iso[1])
    assert vkey.size > 0 and faces.shape[0] > 0
    gk, gt, gp, gf = mesh.band_extract(lv["chi"], band_depth, lv["map"], lv["bricks"], lv["frame"], dbg["iso"])
    assert same(_np(dbg["vkey"]), vkey) and same(_np(gk), vkey) and same(_np(gt), vt) and same(_np(gp), vpos)
    assert same(_np(gf).astype(np.int64), faces)
    cols = _np(dbg["colours"]).astype(np.int32)
    gd, gc = mesh.band_gather(dbg["points"], dbg["colours"].to(torch.int32), dbg["cell"], lv["frame"], band_depth, gk, gt)
    dens, vcol = fb.vertex_density_colour(pts, cols, cell, fr, vkey, vt)
    assert same(_np(gd), dens) and same(_np(gc), vcol)
    # trim, smoothing (3 steps) and normals of the kernel's mesh against f64ref_mesh's, bit for bit
    d_k, p_k, c_k, f_k, keep, thr = fm.trim(dens, vpos, vcol, faces)
    assert same(_np(dbg["keep"]).astype(bool), keep) and _np(dbg["threshold"])[0] == thr
    assert same(_np(m.densities), d_k) and same(_np(m.colours), c_k) and same(_np(m.faces).astype(np.int64), f_k)
    if p_k.shape[0] <= 2_000_000:
        sm = fm.smooth(p_k, f_k, 3)
        assert same(_np(dbg["vpos_smoothed"]), sm)
        assert same(_np(m.vertices), sm.astype(np.float32))
        assert same(_np(m.normals), fm.vertex_normals(sm, f_k).astype(np.float32))
    # the per-level report without return_debug
    stats = []
    mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=depth, band_depth=band_depth, laplacian_iters=0, band_stats=stats)
    assert [(s["depth"], s["bricks"], s["iterations"], s["ratio"]) for s in stats] == \
        [(lv["depth"], int(lv["bricks"].shape[0]), lv["iterations"], lv["ratio"]) for lv in dbg["levels"]]
    print(f"[{name} ({depth}, {band_depth})] gpu {t_gpu:.2f} s, {vkey.size} vertices, {faces.shape[0]} triangles")


def _closed(vpos, faces):
    counts, oriented = fm.edge_use(faces)
    return bool((counts == 2).all()) and oriented


def _component_euler(faces):
    """Euler characteristic of every connected component of the triangles, in ascending order."""
    from scipy.sparse.csgraph import connected_components
    import scipy.sparse as sp
    f = np.asarray(faces, np.int64)
    used, idx = np.unique(f, return_inverse=True)
    idx = idx.reshape(f.shape)
    e = np.concatenate([idx[:, [0, 1]], idx[:, [1, 2]]])
    g = sp.coo_matrix((np.ones(e.shape[0]), (e[:, 0], e[:, 1])), shape=(used.size, used.size))
    _, lab = connected_components(g, directed=False)
    return sorted(fm.euler_characteristic(f[lab[idx[:, 0]] == c]) for c in range(lab.max() + 1))


def _untrimmed(dbg, band_depth):
    """(positions, triangles) of the band extraction before the density trim, from the run's own chi and iso."""
    from g2pc import mesh
    lv = dbg["levels"][-1]
    _, _, vpos, faces = mesh.band_extract(lv["chi"], band_depth, lv["map"], lv["bricks"], lv["frame"], dbg["iso"])
    return _np(vpos), _np(faces)


def test_end_to_end(lib):
    from g2pc import mesh
    rng = np.random.default_rng(21)
    for band in (11, 12):
        p, n = _small_pair(rng)
        m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), depth=10, band_depth=band, laplacian_iters=0, return_debug=True)
        v, f = _untrimmed(dbg, band)
        h = float(_np(dbg["levels"][-1]["frame"])[3])
        # each sphere is its own closed component of Euler characteristic 2
        assert _component_euler(f) == [2, 2] and fm.signed_volume(v, f) > 0 and _closed(v, f)
        da = np.abs(np.linalg.norm(v, axis=1) - 0.01)
        db = np.abs(np.linalg.norm(v - np.array([1.0, 0.3, -0.2]), axis=1) - 0.008)
        dist = np.minimum(da, db)
        print(f"[pair (10, {band})] max distance to the spheres {dist.max() / h:.3f} h, iterations "
              f"{[lv['iterations'] for lv in dbg['levels']]}")
        assert dist.max() <= 2 * h
        if band == 12:
            _, d10 = mesh.poisson_mesh(gpu(p), gpu(n), depth=10, laplacian_iters=0, return_debug=True)
            B10 = d10["B"]
            _, _, a, _ = mesh.extract(d10["chi"], 10, d10["frame"], d10["iso"], B10)
            h10 = 4 * h
            a, b = _np(a), v
            sym = max(cKDTree(a).query(b)[0].max(), cKDTree(b).query(a)[0].max())
            print(f"[pair] depth 12 vs dense depth 10: {sym / h10:.3f} h10")
            assert sym <= 2 * h10
    # a small torus beside a far cluster at (10, 11): the torus has genus 1, the cluster's sphere genus 0
    p, n, _ = clouds.torus(100_000, rng, 0.02, 0.007)
    q, qn = clouds.sphere(5_000, rng, 0.005, (1.0, 1.0, 1.0))
    _, dbg = mesh.poisson_mesh(gpu(np.r_[p, q]), gpu(np.r_[n, qn]), depth=10, band_depth=11, laplacian_iters=0,
                               return_debug=True)
    v, f = _untrimmed(dbg, 11)
    assert _component_euler(f) == [0, 2] and _closed(v, f) and fm.signed_volume(v, f) > 0
    # band_depth=None is the dense path, byte for byte
    p, n = clouds.sphere(50_000, rng)
    a = mesh.poisson_mesh(gpu(p), gpu(n), depth=7)
    b = mesh.poisson_mesh(gpu(p), gpu(n), depth=7, band_depth=None)
    for x, y in zip(a, b):
        assert (x is None and y is None) or same(_np(x), _np(y))


def _band_run(p, n, c):
    from g2pc import mesh
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=10, band_depth=12, laplacian_iters=2, return_debug=True)
    out = [_np(t) for t in m] + [_np(dbg["chi"]), _np(dbg["iso"]), _np(dbg["keep"])]
    return out + [lv["iterations"] for lv in dbg["levels"]]


def test_repeatable_on_poisoned_memory(lib):
    rng = np.random.default_rng(31)
    p, n = _small_pair(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    assert_repeatable(lambda: _band_run(p, n, c), byte=0xFF, large_bytes=1 << 30, large_blocks=2)


def test_refusals(lib, monkeypatch):
    from g2pc import capi, mesh
    p, n = _small_pair(np.random.default_rng(41), 4_000)
    P, N = gpu(p), gpu(n)
    for depth, band in ((8, 8), (8, 7), (10, 13), (8, 9.5)):
        with pytest.raises(capi.G2pcError, match="band_depth"):
            mesh.poisson_mesh(P, N, depth=depth, band_depth=band)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 20, 80 << 30))
    with pytest.raises(capi.G2pcError, match="bytes"):
        mesh.poisson_mesh(P, N, depth=8, band_depth=10)


def test_scale_10m_shell(lib):
    """10 M points on a sphere shell of radius 0.5 beside a far cluster: 44.7 M vertices at depth 12 (measured 5.1 s,
    peak 18.2 GiB on an H100).  The unit sphere filling the frame gives 5.0e8 triangles, more than the smoothing's int32
    one-ring lists address (6 t < 2^31): band_extract refuses it as soon as the triangle count is known."""
    from g2pc import mesh
    rng = np.random.default_rng(3)
    p, n = clouds.sphere(10_000_000, rng, 0.5, noise=1e-3)
    q, qn = clouds.sphere(20_000, rng, 0.02, (1.5, 1.5, 1.5))
    p, n = np.r_[p, q], np.r_[n, qn]
    P, N = gpu(p), gpu(n)
    del p, n
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m = mesh.poisson_mesh(P, N, depth=10, band_depth=12)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"[10M shell, (10, 12)] {dt:.2f} s, peak {peak:.2f} GiB, {m.vertices.shape[0]} vertices, "
          f"{m.faces.shape[0]} faces")
    assert dt < 120.0 and m.faces.shape[0] > 0 and int(m.faces.max()) < m.vertices.shape[0]


def test_mesh_pc_band(lib, tmp_path):
    import mesh_pc
    from g2pc import mesh
    from gauss_dataloader import save_xyz_to_ply
    p, n = clouds.sphere(200_000, np.random.default_rng(51), 1.0)
    cloud = str(tmp_path / "cloud.ply")
    save_xyz_to_ply(torch.from_numpy(p), cloud, rgb_colors=torch.full(p.shape, 128.0), normals_points=torch.from_numpy(n),
                    quiet=True)
    out = str(tmp_path / "mesh.ply")
    mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "10", "--band_depth", "11",
                  "--quiet"])
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert v.shape[0] > 0 and f.shape[0] > 0 and f.min() >= 0 and f.max() < v.shape[0]
    assert np.isfinite(v).all() and np.isfinite(nn).all()


def test_gauss_to_mesh_band(lib, tmp_path):
    """gauss_to_mesh.py at --poisson_depth 8 --band_depth 10 on the flat-Gaussian sphere seen from outside: a cloud
    sampled from Gaussians, normals turned toward the cameras, through the band levels.  The written mesh equals the
    library's on the returned surface cloud, faces outward, and lies no further from the sphere than the dense depth-10
    mesh of the same cloud plus 2 h10 (100 k surface points are about 5 h10 apart at depth 10, so both meshes bulge
    between them)."""
    import gauss_to_mesh
    from g2pc import mesh, sampler
    from test_gauss_mesh_gpu import _opaque, _outside, _write_scene
    from test_orient_gpu import _surface_distance, _tangent_scene
    rng = np.random.default_rng(41)
    ply, tj = _write_scene(tmp_path, _opaque(_tangent_scene("sphere", 20_000, rng), rng), *_outside())
    cloud, out = str(tmp_path / "cloud.ply"), str(tmp_path / "mesh.ply")
    sampler.reset_call_counter(0)
    surf, m = gauss_to_mesh.main(["--input_path", ply, "--transform_path", tj, "--output_path", cloud,
                                  "--mesh_output_path", out, "--num_points", "200000", "--poisson_depth", "8",
                                  "--band_depth", "10", "--colour_quality", "original", "--quiet"])
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert f.shape[0] > 0 and f.min() >= 0 and f.max() < v.shape[0] and np.isfinite(nn).all()
    ref = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=8, band_depth=10, std_ratio=3.0)
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(c, _np(ref.colours))
    h10 = fm.frame(surf.points.cpu().numpy(), 10)["h"]
    spread = float(_surface_distance(surf.points.cpu().numpy().astype(np.float64), "sphere").max() / h10)
    dist = float(_surface_distance(v.astype(np.float64), "sphere").max() / h10)
    dense = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=10, std_ratio=3.0)
    d10 = float(_surface_distance(_np(dense.vertices).astype(np.float64), "sphere").max() / h10)
    print(f"[gauss_to_mesh (8, 10)] {surf.points.shape[0]} surface points (up to {spread:.2f} h10 off the sphere), "
          f"{v.shape[0]} vertices, max distance {dist:.2f} h10; dense depth 10 on the same cloud: "
          f"{dense.vertices.shape[0]} vertices, {d10:.2f} h10")
    assert fm.signed_volume(v, f) > 0 and dist <= d10 + 2.0


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_band_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "MESH_BAND_TARGET_OK", tool, tmp_path, timeout=600)
