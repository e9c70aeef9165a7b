"""GPU: the component filter (s15_components.cu, DESIGN.md §2, N11) bit for bit against its restatement
(tests/f64ref_components.py) on hand meshes, Poisson meshes and adversarial union-find graphs; the invariance of the
meshers (a filtered mesh is the unfiltered one restricted to the kept components) on the dense, band and TSDF paths;
filter then decimate; the defaults; repeatability on poisoned memory; the refusals; a 10 M-triangle mesh; the three
commands; and compute-sanitizer."""
import os
import time

import numpy as np
import pytest
import torch

import clouds
import f64ref_components as fc
from sanitizer_harness import assert_repeatable, check_target
from test_components_cpu import HAND
from util import gpu, same

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "components_sanitizer_target.py")


def _np(t):
    return None if t is None else t.cpu().numpy()


def _compare(v, f, min_t=None, K=None, cols=None, dens=None):
    """remove_components() on the device against the restatement: labels, sizes, keep mask, stats and outputs."""
    from g2pc import mesh
    v, f = np.asarray(v, np.float64), np.asarray(f, np.int32)
    stats = {}
    (gv, gf, gc, gd), dbg = mesh.remove_components(gpu(v), gpu(f), None if cols is None else gpu(cols),
                                                   None if dens is None else gpu(dens), min_t, K, stats=stats,
                                                   return_debug=True)
    (rv, rf, rc, rd), info = fc.remove_components(v, f, cols, dens, min_t, K)
    assert (_np(dbg["labels"]) == info["labels"]).all()
    assert (_np(dbg["sizes"]) == info["sizes"]).all()
    assert (_np(dbg["keep"]).astype(bool) == info["keep"]).all()
    assert stats == {k: info[k] for k in ("components", "kept", "largest", "removed_triangles", "removed_vertices")}
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
    for min_t, K in ((1, None), (2, None), (None, 1), (None, 2), (3, 2), (None, 100)):
        try:
            fc.remove_components(v, f, min_triangles=min_t, keep_largest=K)
        except fc.NothingKept:
            continue
        _compare(v, f, min_t, K, cols, dens)
        _compare(v, f, min_t, K)


def _sphere_with_clumps(rng, n=20_000):
    """The unit sphere and four small spheres around it: pieces that the mesher makes into small components."""
    p, nn = clouds.sphere(n, rng)
    parts = [(p, nn)]
    for c in ((1.7, 0.0, 0.0), (-1.2, 1.2, 0.3), (0.0, -1.1, -1.3), (0.4, 0.5, 1.6)):
        parts.append(clouds.sphere(600, rng, 0.2, c))
    return np.concatenate([a for a, _ in parts]), np.concatenate([b for _, b in parts])


@pytest.mark.parametrize("depth", [5, 6, 7])
def test_poisson_meshes(lib, depth):
    from g2pc import mesh
    rng = np.random.default_rng(depth)
    p, n = _sphere_with_clumps(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=depth, laplacian_iters=3, return_debug=True)
    v, f, col, dens = _np(dbg["vpos_smoothed"]), _np(m.faces), _np(m.colours), _np(m.densities)
    info = _compare(v, f, 20, None, col, dens)
    _compare(v, f, None, 2, col, dens)
    _compare(v, f, 5, 3)
    print(f"[sphere with clumps, depth {depth}] {f.shape[0]} triangles, {info['components']} components, largest "
          f"{info['largest']}")
    assert info["components"] >= 2


def _strip(t):
    return np.stack([np.arange(t), np.arange(t) + 1, np.arange(t) + 2], 1)


def _adversarial(name, t=1_000_000):
    rng = np.random.default_rng(7)
    if name == "permuted_strip":  # long hook chains
        perm = rng.permutation(t + 2)
        f = perm[_strip(t)]
    elif name == "fan":  # every union meets vertex 0
        f = np.stack([np.zeros(t, np.int64), np.arange(t) + 1, np.arange(t) + 2], 1)
    elif name == "disjoint":  # t components of one triangle, listed in random order
        f = np.arange(3 * t).reshape(t, 3)[rng.permutation(t)]
    else:  # descending ids along the strip
        f = (t + 1) - _strip(t)
    m = int(f.max()) + 1
    return rng.normal(size=(m, 3)), f.astype(np.int32)


@pytest.mark.parametrize("name", ["permuted_strip", "fan", "disjoint", "descending_strip"])
def test_adversarial_graphs(lib, name):
    v, f = _adversarial(name)
    rng = np.random.default_rng(2)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    info = _compare(v, f, 1, None, cols)
    _compare(v, f, None, 1000 if name == "disjoint" else 1)
    if name == "disjoint":
        assert info["components"] == f.shape[0]
    else:
        assert info["components"] == 1 and info["labels"].max() == 0


def _restrict(mesh_out, min_t, K):
    """The mesh restricted to the components the rules keep, computed on the host from its faces."""
    v, f, c, n, d = (_np(x) for x in (mesh_out.vertices, mesh_out.faces, mesh_out.colours, mesh_out.normals,
                                      mesh_out.densities))
    labels = fc.labels_of(v.shape[0], f)
    keep, _ = fc.keep_of(labels, fc.sizes_of(v.shape[0], f, labels), min_t, K)
    vmap = np.cumsum(keep) - 1
    fk = f[keep[f[:, 0]]]
    return v[keep], vmap[fk].astype(np.int32), None if c is None else c[keep], n[keep], d[keep]


def _assert_restricted(full, filtered, min_t, K):
    rv, rf, rc, rn, rd = _restrict(full, min_t, K)
    assert same(_np(filtered.vertices), rv) and same(_np(filtered.faces), rf) and same(_np(filtered.normals), rn)
    assert same(_np(filtered.densities), rd)
    assert (filtered.colours is None) == (rc is None) and (rc is None or same(_np(filtered.colours), rc))


@pytest.mark.parametrize("min_t, K", [(5000, None), (None, 1), (10, 2)])
def test_dense_path_is_the_restriction(lib, min_t, K):
    from g2pc import mesh
    rng = np.random.default_rng(21)
    p, n = _sphere_with_clumps(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    full = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7)
    stats, timings = {}, {}
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7, min_component_triangles=min_t,
                               keep_largest_components=K, component_stats=stats, timings=timings, return_debug=True)
    assert "components" in timings and dbg["component_labels"].shape[0] == stats["removed_vertices"] + \
        m.vertices.shape[0]
    assert stats["removed_triangles"] > 0 and stats["removed_triangles"] == full.faces.shape[0] - m.faces.shape[0]
    _assert_restricted(full, m, min_t, K)


def test_band_path_is_the_restriction(lib):
    from g2pc import mesh
    from test_mesh_band_gpu import _small_pair
    p, n = _small_pair(np.random.default_rng(11), 8_000)
    full = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, band_depth=8)
    stats = {}
    m = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, band_depth=8, keep_largest_components=1, component_stats=stats)
    print(f"[band 6 -> 8] {stats}")
    assert stats["components"] >= 2 and stats["kept"] == 1
    _assert_restricted(full, m, None, 1)


def _tsdf_scene():
    from test_tsdf_gpu import _scene_and_cameras
    d, cov, cams = _scene_and_cameras(with_masks=False)
    return (d["xyz"], d["opacities"], cov, cams), dict(colours=d["colours"].float(), depth=6, laplacian_iters=3)


def test_tsdf_is_the_restriction(lib):
    from g2pc import tsdf
    args, kw = _tsdf_scene()
    full = tsdf.fuse_mesh(*args, **kw)
    stats, timings = {}, {}
    m, dbg = tsdf.fuse_mesh(*args, keep_largest_components=1, component_stats=stats, timings=timings,
                            return_debug=True, **kw)
    print(f"[tsdf depth 6] {stats}")
    assert "components" in timings and "component_labels" in dbg
    assert stats["components"] >= 2 and stats["kept"] == 1
    _assert_restricted(full, m, None, 1)
    m2 = tsdf.fuse_mesh(*args, min_component_triangles=stats["largest"], **kw)
    for a, b in zip(m, m2):
        assert same(_np(a), _np(b))


def test_filter_then_decimate(lib):
    """poisson_mesh(min_component_triangles=, target_triangles=) is decimate() of the filtered, smoothed mesh."""
    from g2pc import mesh
    rng = np.random.default_rng(22)
    p, n = _sphere_with_clumps(rng)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    kw = dict(depth=7, min_component_triangles=40)
    m1, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), return_debug=True, **kw)
    target = m1.faces.shape[0] // 3
    vp, fp, cp, dp = mesh.decimate(dbg["vpos_smoothed"], m1.faces, target, m1.colours, m1.densities)
    v, vn = mesh.vertex_normals(vp, fp)
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), target_triangles=target, **kw)
    for a, b in zip(m, (v, fp, cp, vn, dp)):
        assert same(_np(a), _np(b))


def test_keep_largest_one_is_the_sphere(lib):
    from g2pc import mesh
    rng = np.random.default_rng(23)
    p, n = _sphere_with_clumps(rng)
    full = mesh.poisson_mesh(gpu(p), gpu(n), depth=7)
    labels = fc.labels_of(full.vertices.shape[0], _np(full.faces))
    assert np.unique(labels[_np(full.faces)[:, 0]]).shape[0] >= 2
    stats = {}
    m = mesh.poisson_mesh(gpu(p), gpu(n), depth=7, keep_largest_components=1, component_stats=stats)
    v, f = _np(m.vertices).astype(np.float64), _np(m.faces)
    assert np.unique(fc.labels_of(v.shape[0], f)).shape[0] == 1 and stats["kept"] == 1
    r = np.linalg.norm(v, axis=1)
    assert r.min() > 0.8 and r.max() < 1.2  # the unit sphere's, not a clump's (those lie beyond 1.3)


def test_defaults_change_nothing(lib):
    from g2pc import mesh, tsdf
    rng = np.random.default_rng(24)
    p, n = _sphere_with_clumps(rng)
    timings = {}
    a, da = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, timings=timings, return_debug=True)
    b = mesh.poisson_mesh(gpu(p), gpu(n), depth=6, min_component_triangles=None, keep_largest_components=None,
                          component_stats={})
    assert "components" not in timings and "component_labels" not in da
    for x, y in zip(a, b):
        assert (x is None and y is None) or same(_np(x), _np(y))
    args, kw = _tsdf_scene()
    timings = {}
    a = tsdf.fuse_mesh(*args, timings=timings, **kw)
    b = tsdf.fuse_mesh(*args, min_component_triangles=None, keep_largest_components=None, **kw)
    assert "components" not in timings
    for x, y in zip(a, b):
        assert same(_np(x), _np(y))


def _repeat_run(v, f, cols, dens):
    from g2pc import mesh
    (gv, gf, gc, gd), dbg = mesh.remove_components(gpu(v), gpu(f), gpu(cols), gpu(dens), 2, 500, return_debug=True)
    return [_np(gv), _np(gf), _np(gc), _np(gd), _np(dbg["labels"]), _np(dbg["sizes"]), _np(dbg["keep"])]


def _mixed(rng, strips=2000, singles=50_000):
    """Strips of random lengths and single triangles, vertex ids permuted."""
    lengths = rng.integers(1, 200, strips)
    f = [off + _strip(L) for off, L in zip(np.r_[0, np.cumsum(lengths + 2)[:-1]], lengths)]
    base = int((lengths + 2).sum())
    f.append(base + np.arange(3 * singles).reshape(-1, 3))
    f = np.concatenate(f)
    perm = rng.permutation(base + 3 * singles)
    return rng.normal(size=(perm.shape[0], 3)), perm[f].astype(np.int32)


def test_repeatable_on_poisoned_memory(lib):
    rng = np.random.default_rng(3)
    v, f = _mixed(rng)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, v.shape[0])
    assert_repeatable(lambda: _repeat_run(v, f, cols, dens), byte=0xFF, large_bytes=1 << 28, large_blocks=2)


def test_refusals(lib, monkeypatch):
    from g2pc import capi, mesh
    v, f = HAND["ties"]()
    V, F = gpu(v), gpu(f, np.int32)
    for bad in (0, -3, 2.5, True):
        with pytest.raises(capi.G2pcError, match="integer >= 1"):
            mesh.remove_components(V, F, min_triangles=bad)
        with pytest.raises(capi.G2pcError, match="integer >= 1"):
            mesh.remove_components(V, F, keep_largest=bad)
    with pytest.raises(capi.G2pcError, match="give min_triangles"):
        mesh.remove_components(V, F)
    with pytest.raises(capi.G2pcError, match="integer >= 1"):
        mesh.poisson_mesh(gpu(clouds.sphere(1000, np.random.default_rng(0))[0]),
                          gpu(clouds.sphere(1000, np.random.default_rng(0))[1]), depth=5, keep_largest_components=0)
    for bad in (-1, v.shape[0]):
        Fb = F.clone()
        Fb[2, 1] = bad
        with pytest.raises(capi.G2pcError, match="face indices"):
            mesh.remove_components(V, Fb, min_triangles=1)
    with pytest.raises(capi.G2pcError, match="float64"):
        mesh.remove_components(V.float(), F, min_triangles=1)
    with pytest.raises(capi.G2pcError, match="int32"):
        mesh.remove_components(V, F.long(), min_triangles=1)
    with pytest.raises(capi.G2pcError, match="colours"):
        mesh.remove_components(V, F, colours=gpu(np.zeros((3, 3), np.uint8)), min_triangles=1)
    with pytest.raises(capi.G2pcError, match="densities"):
        mesh.remove_components(V, F, densities=gpu(np.zeros(3)), min_triangles=1)
    with pytest.raises(capi.G2pcError, match="CUDA"):
        mesh.remove_components(V, F.cpu(), min_triangles=1)
    stats = {}
    with pytest.raises(capi.G2pcError, match="largest of the 6 component.s. has 5 triangle"):
        mesh.remove_components(V, F, min_triangles=6, stats=stats)
    assert stats["kept"] == 0 and stats["removed_triangles"] == f.shape[0]
    with pytest.raises(capi.G2pcError, match="no triangle"):
        mesh.remove_components(V, F[:0], min_triangles=1)
    monkeypatch.setattr(torch.cuda, "mem_get_info", lambda *a: (1 << 10, 80 << 30))
    with pytest.raises(capi.G2pcError, match="bytes"):
        mesh.remove_components(V, F, min_triangles=1)


def test_ten_million_triangles(lib):
    """10 M triangles in strips of random lengths, ids permuted: the ceiling only catches pathological chains."""
    from g2pc import mesh
    rng = np.random.default_rng(8)
    lengths = rng.integers(1, 20_000, 1000)
    lengths = lengths * -(-10_000_000 // int(lengths.sum()))
    offs = np.r_[0, np.cumsum(lengths + 2)[:-1]]
    t, m = int(lengths.sum()), int((lengths + 2).sum())
    strip_of = np.repeat(np.arange(lengths.shape[0]), lengths)
    i = np.arange(t) - np.repeat(np.r_[0, np.cumsum(lengths)[:-1]], lengths)
    base = offs[strip_of] + i
    perm = rng.permutation(m)
    f = perm[np.stack([base, base + 1, base + 2], 1)].astype(np.int32)
    V, F = gpu(rng.normal(size=(m, 3))), gpu(f)
    min_t = int(np.sort(lengths)[lengths.shape[0] // 2])
    stats = {}
    mesh.remove_components(V, F, min_triangles=1)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gv, gf, _, _ = mesh.remove_components(V, F, min_triangles=min_t, keep_largest=300, stats=stats)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"[10M strips] {t} triangles, {stats} in {dt:.2f} s")
    assert t >= 10_000_000 and stats["components"] == lengths.shape[0] and dt < 10.0
    keep = lengths >= min_t
    kept_sizes = np.sort(lengths[keep])[::-1][:300]
    assert stats["kept"] == kept_sizes.shape[0] and gf.shape[0] == int(kept_sizes.sum())


def test_mesh_pc_flags(lib, tmp_path, capsys):
    import mesh_pc
    from g2pc import mesh
    from gauss_dataloader import save_xyz_to_ply
    p, n = _sphere_with_clumps(np.random.default_rng(52))
    cloud = str(tmp_path / "cloud.ply")
    save_xyz_to_ply(torch.from_numpy(p), cloud, rgb_colors=torch.full(p.shape, 128.0),
                    normals_points=torch.from_numpy(n), quiet=True)
    out = str(tmp_path / "mesh.ply")
    mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "7",
                  "--min_component_triangles", "30", "--keep_largest_components", "2"])
    assert "component(s) found" in capsys.readouterr().out
    P, N, C = mesh_pc.load_cloud(cloud)
    ref = mesh.poisson_mesh(P, N, C, depth=7, min_component_triangles=30, keep_largest_components=2)
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(nn, _np(ref.normals))


@pytest.mark.parametrize("method", ["poisson", "tsdf"])
def test_gauss_to_mesh_flags(lib, tmp_path, method):
    from g2pc import mesh
    from test_gauss_mesh_gpu import _mesh_cmd, _opaque, _outside, _write_scene
    from test_orient_gpu import _tangent_scene
    rng = np.random.default_rng(41)
    ply, tj = _write_scene(tmp_path, _opaque(_tangent_scene("sphere", 20_000, rng), rng), *_outside())
    extra = ["--keep_largest_components", "1", "--min_component_triangles", "10"]
    if method == "tsdf":
        extra += ["--mesh_method", "tsdf", "--tsdf_depth", "6"]
    _, out, surf, m = _mesh_cmd(tmp_path, ply, tj, method, extra)
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert same(v, _np(m.vertices)) and same(f, _np(m.faces))
    assert np.unique(fc.labels_of(v.shape[0], f)[f[:, 0]]).shape[0] == 1
    if method == "poisson":
        ref = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=7, std_ratio=3.0,
                                keep_largest_components=1, min_component_triangles=10)
        assert same(v, _np(ref.vertices)) and same(f, _np(ref.faces)) and same(c, _np(ref.colours))


def test_prune_mesh_round_trip(lib, tmp_path):
    import prune_mesh
    from g2pc import mesh
    p, n = _sphere_with_clumps(np.random.default_rng(53))
    c = np.random.default_rng(54).uniform(0, 255, p.shape).astype(np.float32)
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7)
    src, out = str(tmp_path / "mesh.ply"), str(tmp_path / "pruned.ply")
    mesh.write_mesh_ply(src, m)
    prune_mesh.main(["--input_path", src, "--keep_largest_components", "2", "--min_component_triangles", "20",
                     "--mesh_output_path", out, "--quiet"])
    v0, n0, c0, f0 = mesh.read_mesh_ply(src)
    (rv, rf, rc, rn), info = fc.remove_components(v0, f0, c0, n0, 20, 2)
    v, nn, cc, f = mesh.read_mesh_ply(out)
    assert info["removed_triangles"] > 0
    assert same(v, rv) and same(f, rf) and same(cc, rc) and same(nn, rn)


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_components_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "COMPONENTS_TARGET_OK", tool, tmp_path, timeout=600)
