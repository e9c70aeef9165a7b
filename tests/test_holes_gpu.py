"""GPU: the hole filling (s16_holes.cu, DESIGN.md §2, N12) bit for bit against its restatement (tests/f64ref_holes.py)
on hand meshes, trimmed Poisson meshes, TSDF meshes and 1 M-triangle adversarial meshes; the meshers' composition
(filling inside poisson_mesh / fuse_mesh is smooth(fill_holes(...)) of the unfilled mesh) on the dense, band and TSDF
paths; nothing fillable changes nothing; fill then decimate; repeatability on poisoned memory; the refusals; a
10 M-triangle grid; the three commands; and compute-sanitizer."""
import os
import time

import numpy as np
import pytest
import torch

import clouds
import f64ref_holes as fh
from sanitizer_harness import assert_repeatable, check_target
from test_holes_cpu import HAND, grid
from util import gpu, same

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "holes_sanitizer_target.py")


def _np(t):
    return None if t is None else t.cpu().numpy()


def _compare(v, f, H, cols=None, dens=None):
    """fill_holes() on the device against the restatement: labels, succ, lengths, filled mask, stats and outputs."""
    from g2pc import mesh
    v, f = np.asarray(v, np.float64), np.asarray(f, np.int32)
    stats = {}
    (gv, gf, gc, gd), dbg = mesh.fill_holes(gpu(v), gpu(f), None if cols is None else gpu(cols),
                                            None if dens is None else gpu(dens), H, stats=stats, return_debug=True)
    (rv, rf, rc, rd), info = fh.fill_holes(v, f, cols, dens, H)
    assert (_np(dbg["labels"]) == info["labels"]).all()
    assert (_np(dbg["succ"]) == info["succ"]).all()
    assert (_np(dbg["lengths"]) == info["lengths"]).all()
    assert (_np(dbg["filled"]) == info["filled"]).all()
    assert stats == fh.stats_of(info)
    assert same(_np(gv), rv) and same(_np(gf), rf)
    assert (gc is None) == (cols is None) and (gd is None) == (dens is None)
    if cols is not None:
        assert same(_np(gc), rc)
    if dens is not None:
        assert same(_np(gd), rd)
    return info


@pytest.mark.parametrize("name", sorted(HAND))
def test_hand_meshes(lib, name):
    v, f = HAND[name]()
    rng = np.random.default_rng(1)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, v.shape[0])
    for H in (3, 4, 5, 12, 16, 1024):
        _compare(v, f, H, cols, dens)
        _compare(v, f, H)


def test_nothing_filled_returns_the_inputs(lib):
    from g2pc import mesh
    v, f = HAND["tetrahedron"]()
    V, F = gpu(v), gpu(f, np.int32)
    out = mesh.fill_holes(V, F, max_hole_edges=64)
    assert out[0] is V and out[1] is F and out[2] is None and out[3] is None
    v, f = grid(6)
    V, F = gpu(v), gpu(f, np.int32)
    stats = {}
    out = mesh.fill_holes(V, F, max_hole_edges=23, stats=stats)
    assert out[0] is V and out[1] is F and stats["too_long"] == 1


def _sphere_with_clumps(rng, n=20_000):
    p, nn = clouds.sphere(n, rng)
    parts = [(p, nn)] + [clouds.sphere(600, rng, 0.2, c) for c in ((1.7, 0.0, 0.0), (-1.2, 1.2, 0.3))]
    return np.concatenate([a for a, _ in parts]), np.concatenate([b for _, b in parts])


@pytest.mark.parametrize("depth", [5, 6, 7])
def test_poisson_meshes(lib, depth):
    from g2pc import mesh
    rng = np.random.default_rng(depth)
    p, n = _sphere_with_clumps(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=depth, laplacian_iters=0, return_debug=True)
    v, f, col, dens = _np(dbg["vpos_smoothed"]), _np(m.faces), _np(m.colours), _np(m.densities)
    for H in (3, 8, 64, 1024):
        info = _compare(v, f, H, col, dens)
    _compare(v, f, 32)
    print(f"[trimmed Poisson, depth {depth}] {f.shape[0]} triangles: {fh.stats_of(info)}")
    assert info["holes"] >= 1


def _tsdf_scene(laplacian_iters=0):
    from test_tsdf_gpu import _scene_and_cameras
    d, cov, cams = _scene_and_cameras(with_masks=False)
    return (d["xyz"], d["opacities"], cov, cams), dict(colours=d["colours"].float(), depth=6,
                                                       laplacian_iters=laplacian_iters)


def _adversarial(name, rng):
    if name == "grid_many_holes":  # ~1 M triangles, holes of 4 and 8 edges, ids permuted
        n = 700
        skip = {(i, j) for i in range(1, n - 1, 3) for j in range(1, n - 1, 3) if (i + j) % 2}
        skip |= {(i + a, j + b) for i in range(2, n - 3, 9) for j in range(2, n - 3, 9) for a in (0, 1) for b in (0, 1)}
        v, f = _grid_fast(n, skip)
        perm = rng.permutation(v.shape[0])
        inv = np.empty_like(perm)
        inv[perm] = np.arange(perm.shape[0])
        return v[inv], perm[f].astype(np.int32), 8
    if name == "descending_loop":  # ids descend along the rows: every union hooks a root that is not the minimum yet
        n = 700
        v, f = _grid_fast(n, {(i, j) for i in range(200, 450) for j in range(300, 302)})
        return v[::-1].copy(), (v.shape[0] - 1) - f, 1024
    if name == "one_long_loop":  # a 1 x 500 000 strip: one loop of 1 000 002 edges
        v, f = _strip(500_000)
        perm = rng.permutation(v.shape[0])
        inv = np.empty_like(perm)
        inv[perm] = np.arange(perm.shape[0])
        return v[inv], perm[f].astype(np.int32), 16
    n = 700  # many pinched vertices: pairs of missing cells that touch at a corner
    skip = {(i + a, i2 + a) for i in range(1, n - 3, 4) for i2 in range(1, n - 3, 4) for a in (0, 1)}
    v, f = _grid_fast(n, skip)
    return v, f, 1024


def _grid_fast(n, skip):
    x, y = np.meshgrid(np.arange(n + 1), np.arange(n + 1))
    v = np.stack([x.ravel(), y.ravel(), np.sin(x.ravel() * 0.1) * np.cos(y.ravel() * 0.07)], 1).astype(np.float64)
    j, i = np.meshgrid(np.arange(n), np.arange(n), indexing="ij")
    keep = np.ones((n, n), bool)
    for (a, b) in skip:
        keep[b, a] = False
    i, j = i[keep], j[keep]
    a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i + 1, (j + 1) * (n + 1) + i
    f = np.stack([np.stack([a, b, c], 1), np.stack([a, c, d], 1)], 1).reshape(-1, 3)
    return v, f.astype(np.int32)


def _strip(n):
    v = np.stack([np.arange(n + 1).repeat(2), np.tile([0.0, 1.0], n + 1), np.zeros(2 * (n + 1))], 1)
    i = np.arange(n)
    a, b, c, d = 2 * i, 2 * i + 2, 2 * i + 3, 2 * i + 1
    return v, np.stack([np.stack([a, b, c], 1), np.stack([a, c, d], 1)], 1).reshape(-1, 3).astype(np.int32)


@pytest.mark.parametrize("name", ["grid_many_holes", "descending_loop", "one_long_loop", "many_pinched"])
def test_adversarial_meshes(lib, name):
    rng = np.random.default_rng(7)
    v, f, H = _adversarial(name, rng)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, v.shape[0])
    info = _compare(v, f.astype(np.int32), H, cols, dens)
    print(f"[{name}] {f.shape[0]} triangles: {fh.stats_of(info)}")
    if name == "grid_many_holes":
        assert info["filled_holes"] > 10_000 and info["pinched"] > 1000
    elif name == "descending_loop":
        assert info["filled_holes"] == 1 and info["added_triangles"] == 504
    elif name == "one_long_loop":
        assert info["holes"] == 1 and info["too_long"] == 1 and info["boundary_edges"] == 1_000_002
    else:
        assert info["pinched"] > 20_000 and info["filled_holes"] == 0


def _spy_smooth(monkeypatch):
    """Records the mesh every g2pc_mesh_smooth call receives."""
    from g2pc import mesh
    seen, real = [], mesh.smooth

    def spy(vpos, faces, iterations):
        seen.append((vpos.clone(), faces.clone()))
        return real(vpos, faces, iterations)
    monkeypatch.setattr(mesh, "smooth", spy)
    return seen


def _assert_composition(run, monkeypatch, H, iters, compare_hs=(), check_unfillable=True):
    """run(**kw) -> Mesh: the run with max_hole_edges=H equals smooth(fill_holes(...)) of the run without it.  With
    compare_hs, the mesh the smoothing received is also checked against the restatement at each of those H.  With
    check_unfillable, a run with a max_hole_edges below the shortest hole equals the run without it, bit for bit."""
    from g2pc import mesh
    seen = _spy_smooth(monkeypatch)
    m0 = run()
    v0, f0 = seen[-1]
    for h in compare_hs:
        info = _compare(_np(v0), _np(f0), h, _np(m0.colours), _np(m0.densities))
        print(f"[unfilled mesh, H = {h}] {f0.shape[0]} triangles: {fh.stats_of(info)}")
    lengths = fh.find(v0.shape[0], _np(f0))[2]
    shortest = int(lengths[lengths > 0].min())
    if check_unfillable and shortest > 3:  # nothing fillable with the flag given
        stats = {}
        m1 = run(max_hole_edges=shortest - 1, hole_stats=stats)
        assert stats["filled"] == 0 and stats["holes"] >= 1
        for a, b in zip(m0, m1):
            assert (a is None and b is None) or same(_np(a), _np(b))
    stats, timings = {}, {}
    m, dbg = run(max_hole_edges=H, hole_stats=stats, timings=timings, return_debug=True)
    assert "holes" in timings and dbg["hole_labels"].shape[0] == v0.shape[0]
    monkeypatch.undo()
    vf, ff, cf, df = mesh.fill_holes(v0, f0, m0.colours, m0.densities, H)
    vf = vf.clone()
    mesh.smooth(vf, ff, iters)
    v, vn = mesh.vertex_normals(vf, ff)
    for a, b in zip(m, (v, ff, cf, vn, df)):
        assert (a is None and b is None) or same(_np(a), _np(b))
    if "vpos_smoothed" in dbg:
        assert same(_np(dbg["vpos_smoothed"]), _np(vf))
    print(f"[composition] {stats}")
    assert stats["filled"] >= 1
    return stats


def test_dense_path_composition(lib, monkeypatch):
    from g2pc import mesh
    rng = np.random.default_rng(21)
    p, n = _sphere_with_clumps(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    _assert_composition(lambda **kw: mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7, **kw), monkeypatch, 64, 10)


def test_band_path_composition(lib, monkeypatch):
    from g2pc import mesh
    from test_mesh_band_gpu import _small_pair
    p, n = _small_pair(np.random.default_rng(11), 8_000)
    _assert_composition(lambda **kw: mesh.poisson_mesh(gpu(p), gpu(n), depth=6, band_depth=8, **kw), monkeypatch,
                        64, 10, check_unfillable=False)


def test_tsdf_composition(lib, monkeypatch):
    from g2pc import tsdf
    args, kw = _tsdf_scene(laplacian_iters=3)
    _assert_composition(lambda **k: tsdf.fuse_mesh(*args, **kw, **k), monkeypatch, 256, 3, compare_hs=(3, 16, 256))


def test_closed_surface_changes_nothing(lib):
    """The flag given and nothing fillable on a closed surface (the meshers' runs are checked in the composition
    tests)."""
    from g2pc import mesh
    v, f = HAND["tetrahedron"]()
    out = mesh.fill_holes(gpu(v), gpu(f, np.int32), max_hole_edges=1024)
    assert same(_np(out[0]), v) and same(_np(out[1]), f.astype(np.int32))


def test_fill_then_decimate(lib):
    from g2pc import mesh
    rng = np.random.default_rng(22)
    p, n = _sphere_with_clumps(rng)
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), depth=7, min_component_triangles=200, return_debug=True)
    v, f = dbg["vpos_smoothed"], m.faces
    stats = {}
    vf, ff, _, _ = mesh.fill_holes(v, f, max_hole_edges=64, stats=stats)
    target = f.shape[0] // 20
    _, d0 = mesh.decimate(v, f, target, return_debug=True)
    _, d1 = mesh.decimate(vf, ff, target, return_debug=True)
    locked0 = int((d0["free"] == 0).sum())
    locked1 = int((d1["free"] == 0).sum())
    print(f"[fill then decimate] {stats}, locked {locked0} -> {locked1}")
    assert stats["filled"] >= 1 and locked1 < locked0


def _repeat_run(v, f, cols, dens):
    from g2pc import mesh
    (gv, gf, gc, gd), dbg = mesh.fill_holes(gpu(v), gpu(f), gpu(cols), gpu(dens), 12, return_debug=True)
    return [_np(gv), _np(gf), _np(gc), _np(gd)] + [_np(dbg[k]) for k in ("labels", "succ", "lengths", "filled")]


def test_repeatable_on_poisoned_memory(lib):
    rng = np.random.default_rng(3)
    v, f, _ = _adversarial("grid_many_holes", rng)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, v.shape[0])
    assert_repeatable(lambda: _repeat_run(v, f, cols, dens), byte=0xFF, large_bytes=1 << 28, large_blocks=2)


def test_refusals(lib, monkeypatch):
    from g2pc import capi, mesh
    v, f = HAND["annulus"]()
    V, F = gpu(v), gpu(f, np.int32)
    for bad in (2, 1025, True, 4.0, None):
        with pytest.raises(capi.G2pcError, match="3..1024"):
            mesh.fill_holes(V, F, max_hole_edges=bad)
    with pytest.raises(capi.G2pcError, match="3..1024"):
        mesh.poisson_mesh(gpu(clouds.sphere(1000, np.random.default_rng(0))[0]),
                          gpu(clouds.sphere(1000, np.random.default_rng(0))[1]), depth=5, max_hole_edges=2)
    for bad in (-1, v.shape[0]):
        Fb = F.clone()
        Fb[2, 1] = bad
        with pytest.raises(capi.G2pcError, match="face indices"):
            mesh.fill_holes(V, Fb, max_hole_edges=8)
    Fb = F.clone()
    Fb[3, 2] = Fb[3, 0]
    with pytest.raises(capi.G2pcError, match="use a vertex twice"):
        mesh.fill_holes(V, Fb, max_hole_edges=8)
    with pytest.raises(capi.G2pcError, match="float64"):
        mesh.fill_holes(V.float(), F, max_hole_edges=8)
    with pytest.raises(capi.G2pcError, match="int32"):
        mesh.fill_holes(V, F.long(), max_hole_edges=8)
    with pytest.raises(capi.G2pcError, match="colours"):
        mesh.fill_holes(V, F, colours=gpu(np.zeros((3, 3), np.uint8)), max_hole_edges=8)
    with pytest.raises(capi.G2pcError, match="densities"):
        mesh.fill_holes(V, F, densities=gpu(np.zeros(3)), max_hole_edges=8)
    with pytest.raises(capi.G2pcError, match="CUDA"):
        mesh.fill_holes(V, F.cpu(), max_hole_edges=8)
    out = mesh.fill_holes(V, F[:0], max_hole_edges=8)
    assert out[1].shape[0] == 0
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 10, 80 << 30))
    with pytest.raises(capi.G2pcError, match="bytes"):
        mesh.fill_holes(V, F, max_hole_edges=8)


def test_ten_million_triangles(lib):
    """A 2237 x 2237 grid (10 M triangles) with 100 k single-cell holes."""
    from g2pc import mesh
    n = 2237
    odd = np.arange(1, n - 1, 2)  # cells at odd (i, j) never touch each other
    pick = np.random.default_rng(8).choice(odd.shape[0] ** 2, 100_000, replace=False)
    cells = np.stack([odd[pick % odd.shape[0]], odd[pick // odd.shape[0]]], 1)
    v, f = _grid_fast(n, set(map(tuple, cells.tolist())))
    V, F = gpu(v), gpu(f)
    mesh.fill_holes(V, F, max_hole_edges=8)  # warm-up
    torch.cuda.synchronize()
    stats = {}
    t0 = time.perf_counter()
    gv, gf, _, _ = mesh.fill_holes(V, F, max_hole_edges=8, stats=stats)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"[10M grid] {f.shape[0]} triangles, {stats} in {dt:.2f} s")
    assert f.shape[0] >= 9_800_000 and stats["filled"] == cells.shape[0] == 100_000 and dt < 10.0
    assert gf.shape[0] == f.shape[0] + 4 * 100_000 and gv.shape[0] == v.shape[0] + 100_000


def test_mesh_pc_flag(lib, tmp_path, capsys):
    import mesh_pc
    from g2pc import mesh
    from gauss_dataloader import save_xyz_to_ply
    p, n = _sphere_with_clumps(np.random.default_rng(52))
    cloud = str(tmp_path / "cloud.ply")
    save_xyz_to_ply(torch.from_numpy(p), cloud, rgb_colors=torch.full(p.shape, 128.0),
                    normals_points=torch.from_numpy(n), quiet=True)
    out = str(tmp_path / "mesh.ply")
    mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "7", "--max_hole_edges", "64"])
    line = [x for x in capsys.readouterr().out.splitlines() if x.startswith("Closed holes")][0]
    found, filled = int(line.split()[2]), int(line.split()[5])
    assert filled <= found
    P, N, C = mesh_pc.load_cloud(cloud)
    ref = mesh.poisson_mesh(P, N, C, depth=7, max_hole_edges=64)
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(nn, _np(ref.normals))


@pytest.mark.parametrize("method", ["poisson", "tsdf"])
def test_gauss_to_mesh_flag(lib, tmp_path, method):
    from g2pc import mesh
    from test_gauss_mesh_gpu import _mesh_cmd, _opaque, _outside, _write_scene
    from test_orient_gpu import _tangent_scene
    rng = np.random.default_rng(41)
    ply, tj = _write_scene(tmp_path, _opaque(_tangent_scene("sphere", 20_000, rng), rng), *_outside())
    extra = ["--max_hole_edges", "128"]
    if method == "tsdf":
        extra += ["--mesh_method", "tsdf", "--tsdf_depth", "6"]
    _, out, surf, m = _mesh_cmd(tmp_path, ply, tj, method, extra)
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert same(v, _np(m.vertices)) and same(f, _np(m.faces))
    if method == "poisson":
        ref = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=7, std_ratio=3.0, max_hole_edges=128)
        assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(c, _np(ref.colours))


def test_prune_mesh_round_trip(lib, tmp_path):
    import prune_mesh
    from g2pc import mesh
    p, n = _sphere_with_clumps(np.random.default_rng(53))
    c = np.random.default_rng(54).uniform(0, 255, p.shape).astype(np.float32)
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7)
    src, out = str(tmp_path / "mesh.ply"), str(tmp_path / "filled.ply")
    mesh.write_mesh_ply(src, m)
    prune_mesh.main(["--input_path", src, "--min_component_triangles", "200", "--max_hole_edges", "64",
                     "--mesh_output_path", out, "--quiet"])
    prune_mesh.main(["--input_path", src, "--min_component_triangles", "200", "--mesh_output_path",
                     str(tmp_path / "pruned.ply"), "--quiet"])
    v0, n0, c0, f0 = mesh.read_mesh_ply(str(tmp_path / "pruned.ply"))
    (rv, rf, rc, _), info = fh.fill_holes(v0.astype(np.float64), f0, c0, None, 64)
    v, nn, cc, f = mesh.read_mesh_ply(out)
    assert info["filled_holes"] >= 1
    assert same(v, rv.astype(np.float32)) and same(f, rf) and same(cc, rc)
    labels, filled = info["labels"], info["filled"]
    off = ~((labels >= 0) & (filled[np.maximum(labels, 0)] == 1))
    assert same(nn[:v0.shape[0]][off], n0[off])  # vertices on no filled loop keep their normals
    _, ref_n = mesh.vertex_normals(gpu(rv), gpu(rf))
    assert same(nn[:v0.shape[0]][~off], _np(ref_n)[:v0.shape[0]][~off]) and same(nn[v0.shape[0]:],
                                                                                 _np(ref_n)[v0.shape[0]:])


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_holes_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "HOLES_TARGET_OK", tool, tmp_path, timeout=600)
