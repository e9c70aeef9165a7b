"""GPU: the decimation kernels (s13_decimate.cu) bit for bit against the float64 restatement (tests/f64ref_decimate.py,
DESIGN.md §2, N9) round by round on hand meshes and Poisson meshes, at the end on a 1 M-triangle mesh; the mesher with
target_triangles end to end; repeatability on poisoned memory; the refusals; a 10 M-triangle mesh; the three commands;
and compute-sanitizer."""
import os
import time
import warnings

import numpy as np
import pytest
import torch

import clouds
import f64ref_decimate as fd
import f64ref_mesh as fm
from sanitizer_harness import assert_repeatable, check_target
from util import gpu, same

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "decimate_sanitizer_target.py")


def _np(t):
    return None if t is None else t.cpu().numpy()


def _attributes(m, rng):
    return rng.integers(0, 256, (m, 3)).astype(np.uint8), rng.uniform(0.5, 2.0, m)


def _compare(v, f, target, cols=None, dens=None, rounds=True):
    """decimate() on the device against the restatement: the preparation, every round (when `rounds`) and the result."""
    from g2pc import mesh
    v, f = np.asarray(v, np.float64), np.asarray(f, np.int32)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        (gv, gf, gc, gd), dbg = mesh.decimate(gpu(v), gpu(f), target, None if cols is None else gpu(cols),
                                              None if dens is None else gpu(dens), return_debug=True)
    rv, rf, rc, rd, info = fd.decimate(v, f, target, cols, dens, check=rounds)
    assert len(dbg["rounds"]) == len(info["rounds"])
    stopped = [x for x in w if issubclass(x.category, RuntimeWarning) and "decimation stopped" in str(x.message)]
    assert bool(stopped) == (not info["reached"])
    if info["rounds"]:
        assert same(_np(dbg["quadrics"]), info["quadrics"]) and same(_np(dbg["free"]).astype(bool), info["free"])
    if rounds:
        for i, (g, r) in enumerate(zip(dbg["rounds"], info["rounds"])):
            assert (g["edges"], g["candidates"], g["selected"]) == (r["edges"], r["candidates"], r["selected"]), i
            assert (_np(g["keys"]).view(np.uint64) == r["keys"]).all(), i
            assert (_np(g["ab"]) == r["ab"]).all(), i
            assert same(_np(g["vpos"]), r["vpos"]) and same(_np(g["quadrics"]), r["quadrics"]), i
            assert (_np(g["merged"]) == r["merged"]).all() and (_np(g["faces"]) == r["faces"]).all(), i
            if cols is not None:
                assert (_np(g["colour_sums"]) == r["colour_sums"]).all(), i
            if dens is not None:
                assert same(_np(g["density_sums"]), r["density_sums"]), i
    assert same(_np(gv), rv) and (_np(gf) == rf).all()
    if cols is not None:
        assert same(_np(gc), rc)
    if dens is not None:
        assert same(_np(gd), rd)
    return rv, rf, info


def _pyramid():
    ring = np.array([[2, 0], [0, 1], [-1, 0], [0, -1], [0.2, -0.2]], float)
    v = np.zeros((7, 3))
    v[1:6, :2] = ring
    v[6] = [0, 0, -3]
    return v, np.array([x for i in range(5) for x in ([0, 1 + i, 1 + (i + 1) % 5], [1 + i, 6, 1 + (i + 1) % 5])])


def _hand(name):
    if name == "flat_grid":
        return fd.grid(10, 0.0)
    if name == "grid":
        return fd.grid(14, 0.5)
    if name == "pyramid":
        return _pyramid()
    if name == "pinch":
        v, f = fd.octahedron()
        return np.r_[v, v[1:] + [2.0, 0, 0]], np.r_[f, np.where(f == 0, 0, f + 5)]
    if name == "zero_area":
        v, f = fd.icosphere(2)
        a, b, c = f[0]
        v = np.r_[v, (v[[a]] + v[[b]]) * 0.5]
        k = v.shape[0] - 1
        return v, np.r_[f[1:], [[a, b, k], [b, c, k], [c, a, k]]]
    return getattr(fd, name)()


@pytest.mark.parametrize("name", ["tetrahedron", "octahedron", "icosphere", "torus", "grid", "flat_grid", "pyramid",
                                  "pinch", "zero_area"])
def test_hand_meshes(lib, name):
    v, f = _hand(name)
    cols, dens = _attributes(v.shape[0], np.random.default_rng(1))
    for target in (max(1, f.shape[0] // 4), f.shape[0] // 2 + 1):
        _compare(v, f, target, cols, dens)


@pytest.mark.parametrize("depth", [5, 6, 7])
@pytest.mark.parametrize("name", ["sphere", "two_spheres", "plane", "cube_faces"])
def test_poisson_meshes(lib, name, depth):
    """The smoothed float64 Poisson mesh of the mesher's test clouds (plane and cube_faces carry the trim's holes and
    boundaries), with its colours and densities, decimated to 30 %."""
    from g2pc import mesh
    from test_mesh_gpu import _cloud
    rng = np.random.default_rng(depth)
    p, n = _cloud(name, rng, depth)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=depth, laplacian_iters=3, return_debug=True)
    v, f = _np(dbg["vpos_smoothed"]), _np(m.faces)
    rv, rf, info = _compare(v, f, max(1, int(0.3 * f.shape[0])), _np(m.colours), _np(m.densities))
    print(f"[{name} depth {depth}] {f.shape[0]} -> {rf.shape[0]} triangles, {len(info['rounds'])} rounds, "
          f"{int((~info['free']).sum())} of {v.shape[0]} vertices locked")


def _mt_sphere(R, radius, centre):
    g = np.arange(R) + 0.5
    chi = np.empty((R, R, R))
    for k in range(R):
        chi[k] = np.sqrt((g[None, :] - centre[0]) ** 2 + (g[:, None] - centre[1]) ** 2 + (g[k] - centre[2]) ** 2)
    chi -= radius
    _, _, vpos, faces = fm.marching_tetrahedra(chi.reshape(-1), R, 0.0)
    return vpos, faces


def test_million_triangles_at_the_end(lib):
    v, f = _mt_sphere(224, 100.3, (111.7, 112.2, 111.9))
    assert f.shape[0] >= 1_000_000
    cols, dens = _attributes(v.shape[0], np.random.default_rng(2))
    t0 = time.perf_counter()
    rv, rf, info = _compare(v, f, f.shape[0] // 10, cols, dens, rounds=False)
    print(f"[MT sphere] {f.shape[0]} -> {rf.shape[0]} triangles in {len(info['rounds'])} rounds "
          f"({time.perf_counter() - t0:.1f} s with the restatement)")


def test_poisson_mesh_end_to_end(lib):
    """poisson_mesh(target_triangles=) on a sphere cloud whose x < 0 half is red and x > 0 half blue.  The density trim
    leaves small holes, whose boundary vertices are locked: the decimated mesh keeps the undecimated mesh's Euler
    characteristic, boundary edge count and consistent orientation, has a positive volume, every vertex lies within 2 h
    of the sphere, and the halves keep their colours."""
    from g2pc import mesh
    rng = np.random.default_rng(5)
    p, n = clouds.sphere(200_000, rng)
    c = np.where(p[:, :1] < 0, [[255, 0, 0]], [[0, 0, 255]]).astype(np.float32)
    full = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=8)
    timings = {}
    target = full.faces.shape[0] // 3
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=8, target_triangles=target, timings=timings)
    assert "decimate" in timings
    v, f, col = _np(m.vertices).astype(np.float64), _np(m.faces), _np(m.colours)
    f0 = _np(full.faces)
    assert f.shape[0] in (target - 1, target)
    counts, oriented = fm.edge_use(f)
    assert oriented and (counts <= 2).all()
    assert fm.euler_characteristic(f, v.shape[0]) == fm.euler_characteristic(f0, full.vertices.shape[0])
    assert fd.boundary_edges(f).shape[0] == fd.boundary_edges(f0).shape[0]
    assert fm.signed_volume(v, f) > 0
    h = fm.frame(p, 8)["h"]
    dist = np.abs(np.linalg.norm(v, axis=1) - 1.0)
    assert dist.max() <= 2 * h
    far = np.abs(v[:, 0]) > 0.1
    assert (col[far & (v[:, 0] < 0)] == [255, 0, 0]).all() and (col[far & (v[:, 0] > 0)] == [0, 0, 255]).all()
    print(f"[poisson_mesh sphere depth 8] {f0.shape[0]} -> {f.shape[0]} triangles, max distance {dist.max() / h:.2f} h")


def test_band_path_decimates(lib):
    from g2pc import mesh
    from test_mesh_band_gpu import _small_pair
    p, n = _small_pair(np.random.default_rng(11), 8_000)
    full = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, band_depth=8)
    target = full.faces.shape[0] // 3
    timings = {}
    m = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, band_depth=8, target_triangles=target, timings=timings)
    assert "decimate" in timings and m.faces.shape[0] in (target - 1, target)


def test_target_at_least_t_returns_the_input(lib):
    from g2pc import mesh
    v, f = fd.icosphere(2)
    V, F = gpu(v), gpu(f, np.int32)
    C, D = gpu(np.zeros((v.shape[0], 3), np.uint8)), gpu(np.ones(v.shape[0]))
    for target in (f.shape[0], f.shape[0] + 1, 10 ** 9):
        out = mesh.decimate(V, F, target, C, D)
        assert all(a is b for a, b in zip(out, (V, F, C, D)))
    m = mesh.Mesh(V.float(), F, C, V.float(), D)
    assert mesh.decimate_mesh(m, f.shape[0]) is m


def _repeat_run(v, f, cols, dens):
    from g2pc import mesh
    (gv, gf, gc, gd), dbg = mesh.decimate(gpu(v), gpu(f, np.int32), f.shape[0] // 5, gpu(cols), gpu(dens),
                                          return_debug=True)
    return [_np(gv), _np(gf), _np(gc), _np(gd), len(dbg["rounds"])]


def test_repeatable_on_poisoned_memory(lib):
    v, f = _mt_sphere(64, 25.3, (31.7, 32.2, 31.9))
    cols, dens = _attributes(v.shape[0], np.random.default_rng(3))
    assert_repeatable(lambda: _repeat_run(v, f, cols, dens), byte=0xFF, large_bytes=1 << 28, large_blocks=2)


def test_refusals(lib, monkeypatch):
    from g2pc import capi, mesh
    v, f = fd.icosphere(1)
    V, F = gpu(v), gpu(f, np.int32)
    for bad in (0, -3, 2.5, True):
        with pytest.raises(capi.G2pcError, match="target_triangles"):
            mesh.decimate(V, F, bad)
    with pytest.raises(capi.G2pcError, match="target_triangles"):
        mesh.poisson_mesh(gpu(clouds.sphere(1000, np.random.default_rng(0))[0]),
                          gpu(clouds.sphere(1000, np.random.default_rng(0))[1]), depth=5, target_triangles=0)
    Vn = V.clone()
    Vn[3, 1] = float("nan")
    with pytest.raises(capi.G2pcError, match="finite"):
        mesh.decimate(Vn, F, 10)
    for bad in (-1, v.shape[0]):
        Fb = F.clone()
        Fb[5, 2] = bad
        with pytest.raises(capi.G2pcError, match="face indices"):
            mesh.decimate(V, Fb, 10)
    Fr = F.clone()
    Fr[2, 1] = Fr[2, 0]
    with pytest.raises(capi.G2pcError, match="twice"):
        mesh.decimate(V, Fr, 10)
    with pytest.raises(capi.G2pcError, match="float64"):
        mesh.decimate(V.float(), F, 10)
    with pytest.raises(capi.G2pcError, match="int32"):
        mesh.decimate(V, F.long(), 10)
    with pytest.raises(capi.G2pcError, match="colours"):
        mesh.decimate(V, F, 10, colours=gpu(np.zeros((3, 3), np.uint8)))
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 10, 80 << 30))
    with pytest.raises(capi.G2pcError, match="bytes"):
        mesh.decimate(V, F, 10)


def test_ten_million_triangles(lib):
    """A 10.4 M-triangle torus with radial noise to 1 M triangles: the ceiling only catches rounds that stall."""
    from g2pc import mesh
    nu, nv = 4000, 1300
    v, f = _torus_fast(nu, nv)
    V, F = gpu(v), gpu(f, np.int32)
    del v, f
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gv, gf, _, _ = mesh.decimate(V, F, 1_000_000, stats=stats)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"[10M torus] {F.shape[0]} -> {gf.shape[0]} triangles in {stats['rounds']} rounds, {dt:.2f} s; collapses "
          f"per round {stats['collapses'][:6]} ... {stats['collapses'][-3:]}")
    assert stats["reached"] and gf.shape[0] in (999_999, 1_000_000) and dt < 60.0


def _torus_fast(nu, nv, R=2.0, r=0.7, noise=1e-3):
    rng = np.random.default_rng(7)
    th = 2 * np.pi * np.arange(nu)[:, None] / nu
    ph = 2 * np.pi * np.arange(nv)[None, :] / nv
    rr = r + noise * r * rng.standard_normal((nu, nv))
    v = np.stack([(R + rr * np.cos(ph)) * np.cos(th), (R + rr * np.cos(ph)) * np.sin(th), rr * np.sin(ph)], -1)
    i, j = np.meshgrid(np.arange(nu), np.arange(nv), indexing="ij")
    a, b = i * nv + j, ((i + 1) % nu) * nv + j
    c, d = ((i + 1) % nu) * nv + (j + 1) % nv, i * nv + (j + 1) % nv
    f = np.stack([np.stack([a, b, c], -1), np.stack([a, c, d], -1)], 2).reshape(-1, 3)
    return v.reshape(-1, 3), f


def test_mesh_pc_target(lib, tmp_path):
    import mesh_pc
    from g2pc import mesh
    from gauss_dataloader import save_xyz_to_ply
    p, n = clouds.sphere(100_000, np.random.default_rng(52), 1.0)
    cloud = str(tmp_path / "cloud.ply")
    save_xyz_to_ply(torch.from_numpy(p), cloud, rgb_colors=torch.full(p.shape, 128.0),
                    normals_points=torch.from_numpy(n), quiet=True)
    out = str(tmp_path / "mesh.ply")
    P, N, C = mesh_pc.load_cloud(cloud)
    target = mesh.poisson_mesh(P, N, C, depth=8).faces.shape[0] // 3
    mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "8", "--target_triangles",
                  str(target), "--quiet"])
    v, nn, c, f = mesh.read_mesh_ply(out)
    ref = mesh.poisson_mesh(P, N, C, depth=8, target_triangles=target)
    assert f.shape[0] in (target - 1, target) and f.max() < v.shape[0] and np.isfinite(nn).all()
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces))
    assert fm.signed_volume(v.astype(np.float64), f) > 0


def test_gauss_to_mesh_target(lib, tmp_path):
    """gauss_to_mesh.py --target_triangles on the flat-Gaussian sphere seen from outside: the mesh is the library's
    decimated mesh of the returned surface cloud, has fewer triangles than the undecimated one (the target, unless the
    trim's locked hole boundaries stop it first, with a warning), and faces the cameras (positive volume)."""
    import gauss_to_mesh
    from g2pc import mesh, sampler
    from test_gauss_mesh_gpu import _opaque, _outside, _write_scene
    from test_orient_gpu import _tangent_scene
    rng = np.random.default_rng(41)
    ply, tj = _write_scene(tmp_path, _opaque(_tangent_scene("sphere", 20_000, rng), rng), *_outside())
    cloud, out = str(tmp_path / "cloud.ply"), str(tmp_path / "mesh.ply")
    sampler.reset_call_counter(0)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        surf, m = gauss_to_mesh.main(["--input_path", ply, "--transform_path", tj, "--output_path", cloud,
                                      "--mesh_output_path", out, "--num_points", "200000", "--poisson_depth", "7",
                                      "--target_triangles", "3000", "--colour_quality", "original", "--quiet"])
    v, nn, c, f = mesh.read_mesh_ply(out)
    full = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=7, std_ratio=3.0)
    stopped = any("decimation stopped" in str(x.message) for x in w)
    print(f"[gauss_to_mesh depth 7] {full.faces.shape[0]} -> {f.shape[0]} triangles (target 3000)")
    assert f.shape[0] in (2999, 3000) or (stopped and f.shape[0] < full.faces.shape[0])
    ref = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=7, std_ratio=3.0, target_triangles=3000)
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(c, _np(ref.colours))
    counts, oriented = fm.edge_use(f)
    assert oriented and fm.signed_volume(v.astype(np.float64), f) > 0


def test_decimate_mesh_round_trip(lib, tmp_path):
    import decimate_mesh
    from g2pc import mesh
    p, n = clouds.sphere(50_000, np.random.default_rng(53), 1.0)
    c = np.random.default_rng(54).uniform(0, 255, p.shape).astype(np.float32)
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7)
    src, out = str(tmp_path / "mesh.ply"), str(tmp_path / "small.ply")
    mesh.write_mesh_ply(src, m)
    target = m.faces.shape[0] // 4
    decimate_mesh.main(["--input_path", src, "--target_triangles", str(target), "--mesh_output_path", out, "--quiet"])
    v0, n0, c0, f0 = mesh.read_mesh_ply(src)
    ref = mesh.decimate_mesh(mesh.Mesh(gpu(v0), gpu(f0), gpu(c0), gpu(n0), None), target)
    v, nn, cc, f = mesh.read_mesh_ply(out)
    assert f.shape[0] in (target - 1, target)
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(cc, _np(ref.colours))
    assert same(nn, _np(ref.normals))


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_decimate_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "DECIMATE_TARGET_OK", tool, tmp_path, timeout=600)
