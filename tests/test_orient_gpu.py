"""GPU: the normal orientation (g2pc_knn_ids in s9_clean.cu, the s11_orient.cu kernels, g2pc/orient.py, mesh_pc.py
--orient_normals) against the float64 restatement f64ref_orient.

Every output is integer or an exact float64 / float32 expression of the inputs, so everything is compared bit for bit:
the neighbour ids and d2, the edges, the spanning-forest edge set, rel, the seeds, the stats and the output normals."""
import os
import time
import zlib

import numpy as np
import pytest
import torch

import clouds
import f64ref_mesh as fm
import f64ref_orient as fo
from sanitizer_harness import assert_repeatable, check_target
from util import gpu, same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "orient_sanitizer_target.py")
K_MAX = 31


def _cloud(name, rng):
    """(points float32, normals float32 with random signs)"""
    u = lambda n, lo=0.0, hi=1.0: clouds.uniform(n, rng, lo, hi)
    if name == "sphere_floaters":
        p, n = clouds.sphere(15_000, rng, noise=1e-3)
        p = np.r_[p, u(300, -3.0, 3.0)]
        n = np.r_[n, rng.normal(size=(300, 3)).astype(np.float32)]
    elif name == "plane":
        p = clouds.plane(12_000, rng, -2.0, 2.0, 0.5)
        n = np.tile(np.float32([0, 0, 1]), (p.shape[0], 1)) + u(p.shape[0], -0.1, 0.1)
    elif name == "lattice":  # ties at every slot
        p = clouds.lattice(20)
        n = rng.normal(size=p.shape).astype(np.float32)
    elif name == "clusters":  # 1e-4 clusters beside sparse points
        p = np.concatenate([clouds.clusters(rng, [0.3, -0.4], [8_000, 4_000], 1e-4), u(2_000)])
        n = rng.normal(size=p.shape).astype(np.float32)
    elif name == "dup_runs":  # runs of exact copies around k
        p = clouds.dup_runs(3_000, rng, (9, 10, 11, 12, 30, 31, 32, 33, 100), 5)
        n = rng.normal(size=p.shape).astype(np.float32)
    elif name == "far":  # +-1e4 coordinates
        p = clouds.clusters(rng, clouds.FAR[:3], [3_000] * 3, 1.0)
        n = rng.normal(size=p.shape).astype(np.float32)
    elif name.startswith("small"):
        p = u(int(name[5:]))
        n = rng.normal(size=p.shape).astype(np.float32)
    else:
        raise KeyError(name)
    s = np.where(rng.random(p.shape[0]) < 0.5, -1.0, 1.0).astype(np.float32)
    return p.astype(np.float32), (n * s[:, None]).astype(np.float32)


CLOUDS = ["sphere_floaters", "plane", "lattice", "clusters", "dup_runs", "far", "small1", "small2", "small10",
          "small11", "small31", "small32"]


@pytest.mark.parametrize("k", [1, 10, K_MAX])
@pytest.mark.parametrize("name", CLOUDS)
def test_knn_ids_bit_identical(lib, name, k):
    from g2pc import orient
    p, _ = _cloud(name, np.random.default_rng(zlib.crc32(name.encode())))
    ids, d2, status = orient.knn_ids(gpu(p), k)
    want_i, want_d = fo.knn_ids(p, k)
    got_i, got_d = ids.cpu().numpy(), d2.cpu().numpy()
    bad = np.nonzero((got_i != want_i).any(1))[0]
    if bad.size:
        print(f"[{name} k={k}] {bad.size} rows differ; first {bad[:3]}: got {got_i[bad[:3]]} want {want_i[bad[:3]]}")
    assert int(status.item()) == 0 and np.array_equal(got_i, want_i) and same(got_d, want_d)


def _check_against_restatement(p, n, k, tag):
    from g2pc import orient
    out, st, dbg = orient.orient_normals(gpu(p), gpu(n), k=k, return_debug=True)
    want, info = fo.orient(p, n, k=k)
    got = {key: v.cpu().numpy() for key, v in dbg.items()}
    assert np.array_equal(got["rows"], info["rows"]), tag
    assert np.array_equal(got["ids"], info["ids"]) and same(got["d2"], info["d2"]), tag
    assert np.array_equal(got["edges"], info["edges"].reshape(-1, 2)), tag
    assert np.array_equal(got["mst"], info["mst"]), tag
    assert np.array_equal(got["seed"].astype(np.int64), info["seed"]), tag
    assert np.array_equal(got["rel"], info["rel"]), tag
    assert (st.components, st.flipped, st.skipped) == (info["components"], int(info["flip"].sum()), info["skipped"]), \
        (tag, st, info["components"], int(info["flip"].sum()), info["skipped"])
    o = out.cpu().numpy()
    assert same(o, want), tag
    print(f"[{tag}] {p.shape[0]} points: {st.components} component(s), {st.flipped} flipped, {st.skipped} skipped, "
          f"{st.rounds} rounds")
    return o


@pytest.mark.parametrize("name", CLOUDS)
def test_orientation_bit_identical(lib, name):
    rng = np.random.default_rng(zlib.crc32(name.encode()) + 1)
    p, n = _cloud(name, rng)
    _check_against_restatement(p, n, 10, name)


@pytest.mark.parametrize("k", [1, 31])
def test_orientation_other_k(lib, k):
    p, n = _cloud("sphere_floaters", np.random.default_rng(k))
    _check_against_restatement(p, n, k, f"sphere k={k}")


def test_unusable_rows_and_float64(lib):
    rng = np.random.default_rng(21)
    p, n = clouds.sphere(8_000, rng, noise=1e-3)
    n = n.astype(np.float64) * rng.uniform(1e-3, 1e3, (n.shape[0], 1))
    n *= np.where(rng.random(n.shape[0]) < 0.5, -1.0, 1.0)[:, None]
    n[:40] = 0.0
    n[40:50, 1] = np.nan
    n[50:60, 2] = -np.inf
    p[60, 0] = np.inf
    o = _check_against_restatement(p, n, 10, "unusable f64")
    assert o.dtype == np.float64 and same(o[:61], n[:61])  # untouched rows
    assert (np.abs(o) == np.abs(n))[61:].all()
    o32 = _check_against_restatement(p, n.astype(np.float32), 10, "unusable f32")
    assert o32.dtype == np.float32


def _run_to_host(p, n):
    from g2pc import orient
    out, st, dbg = orient.orient_normals(gpu(p), gpu(n), return_debug=True)
    return [out.cpu().numpy()] + [dbg[k].cpu().numpy() for k in sorted(dbg)] + [np.array(st)]


def test_determinism_on_poisoned_memory(lib):
    rng = np.random.default_rng(9)
    p, n = clouds.sphere(200_000, rng, noise=1e-3)
    n *= np.where(rng.random(n.shape[0]) < 0.5, -1.0, 1.0).astype(np.float32)[:, None]
    assert_repeatable(lambda: _run_to_host(p, n), byte=0xFF, large_bytes=1 << 30, large_blocks=2)


def test_refusals(lib):
    from g2pc import capi, orient
    p, n = clouds.sphere(500, np.random.default_rng(1), noise=1e-3)
    P, N = gpu(p), gpu(n)
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P.cpu(), N.cpu())
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P, N.cpu())
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P, None)
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P.double(), N)
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P, N.half())
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P, N[:100])
    with pytest.raises(capi.G2pcError):
        orient.orient_normals(P[:, :2].contiguous(), N[:, :2].contiguous())
    for k in (0, -1, K_MAX + 1, 2.5):
        with pytest.raises(capi.G2pcError):
            orient.orient_normals(P, N, k=k)
    with pytest.raises(capi.G2pcError):  # the C ABI refuses k above the cap on its own
        capi.call("g2pc_knn_ids", capi.ptr(P), 500, K_MAX + 1, None, None, None, None, 0, capi.stream_ptr(DEV))
    e = torch.zeros((0, 3), device=DEV)
    out, st = orient.orient_normals(e, e)
    assert out.shape == (0, 3) and tuple(st)[:3] == (0, 0, 0)


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_orient_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "ORIENT_TARGET_OK", tool, tmp_path, timeout=600)


# ---- end to end: Gaussians tangent to a surface, sampled by the CLI, meshed by mesh_pc.py ----------------------------
def _tangent_scene(kind, n, rng):
    """Flat Gaussians tangent to a unit sphere or a torus (R 1, r 0.35); each smallest-scale axis gets a random sign
    through its quaternion."""
    from scipy.spatial.transform import Rotation
    from g2pc import synth
    if kind == "sphere":
        nrm = rng.normal(size=(n, 3))
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        xyz = nrm.copy()
    else:
        u, v = rng.uniform(0, 2 * np.pi, n), rng.uniform(0, 2 * np.pi, n)
        c = np.stack([np.cos(u), np.sin(u), np.zeros(n)], 1)
        nrm = np.cos(v)[:, None] * c + np.sin(v)[:, None] * np.array([0, 0, 1.0])
        xyz = c + 0.35 * nrm
    a = np.cross(nrm, rng.normal(size=(n, 3)))
    a /= np.linalg.norm(a, axis=1, keepdims=True)
    b = np.cross(nrm, a)
    s = np.where(rng.random(n) < 0.5, -1.0, 1.0)[:, None]
    R = np.stack([a * s, b, nrm * s], 2)  # columns: two tangents and the normal; det stays +1
    q = Rotation.from_matrix(R).as_quat()[:, [3, 0, 1, 2]]  # (r, x, y, z)
    sc = synth.make_scene(n, seed=int(rng.integers(1 << 30)))
    sc["xyz"] = torch.from_numpy(xyz.astype(np.float32))
    sc["rots"] = torch.from_numpy(q.astype(np.float64))
    tangent = rng.uniform(0.008, 0.016, (n, 1))  # varied sizes and opacities: the sampler bins Gaussians by point count
    sc["scales"] = torch.from_numpy(np.log(np.c_[tangent, tangent, np.full((n, 1), 1e-4)]).astype(np.float64))
    sc["opacities"] = torch.from_numpy(rng.uniform(0.5, 0.95, n).astype(np.float32))
    return sc


def _surface_distance(v, kind):
    if kind == "sphere":
        return np.abs(np.linalg.norm(v, axis=1) - 1.0)
    ring = np.linalg.norm(v[:, :2], axis=1)
    return np.abs(np.hypot(ring - 1.0, v[:, 2]) - 0.35)


def _untrimmed_surface(points, normals, depth):
    """The mesher's surface before its 10 % density trim (which cuts holes): clean, splat, solve, iso, extraction."""
    from g2pc import mesh, outliers
    pts, _, nrm = outliers.remove_statistical_outliers(points, None, normals, mesh.NB_NEIGHBORS, 3.0)
    pts, nrm = pts.contiguous(), nrm.contiguous()
    frame, B, cell, _ = mesh.splat(pts, nrm, depth)
    chi, _, _ = mesh.solve(B, frame, depth)
    iso = mesh.iso_value(pts, cell, frame, depth, chi)
    _, _, vpos, faces = mesh.extract(chi, depth, frame, iso, B)
    return vpos.cpu().numpy(), faces.cpu().numpy()


def _topology(vpos, faces):
    counts, oriented = fm.edge_use(faces)
    return bool(len(faces) and (counts == 2).all() and oriented), fm.euler_characteristic(faces), \
        fm.signed_volume(vpos, faces)


@pytest.mark.parametrize("kind", ["sphere", "torus"])
def test_mesh_pc_orient_end_to_end(lib, tmp_path, kind):
    """The command's mesh (trimmed, smoothed) faces outward and lies within 2h of the surface; the surface before the
    trim, from the same oriented normals, is closed with the shape's Euler characteristic and faces outward."""
    import gauss_to_pc as g2p
    import mesh_pc
    from g2pc import mesh, orient, sampler
    from test_io_cpu import write_gaussian_ply
    sc = _tangent_scene(kind, 20_000, np.random.default_rng(31))
    ply = str(tmp_path / "scene.ply")
    write_gaussian_ply(ply, sc)
    cloud = str(tmp_path / "cloud.ply")
    sampler.reset_call_counter(0)
    g2p.main(["--input_path", ply, "--output_path", cloud, "--num_points", "200000", "--no_render_colours", "--quiet"])
    points, normals, _ = mesh_pc.load_cloud(cloud)
    h = fm.frame(points.cpu().numpy(), 7)["h"]
    results = {}
    for tag, flag in (("--orient_normals", ["--orient_normals"]), ("normals as given", [])):
        out = str(tmp_path / f"mesh{len(flag)}.ply")
        try:
            mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "7", "--quiet"] + flag)
            v, _, _, f = mesh.read_mesh_ply(out)
            v = v.astype(np.float64)
            vol, dist = fm.signed_volume(v, f), float(_surface_distance(v, kind).max() / h)
            nrm = orient.orient_normals(points, normals)[0] if flag else normals
            closed, chi, vol0 = _topology(*_untrimmed_surface(points, nrm, 7))
            results[tag] = (vol, dist, closed, chi, vol0)
            print(f"[{kind}, {tag}] command: {v.shape[0]} vertices, {f.shape[0]} triangles, volume {vol:.4f}, max "
                  f"distance {dist:.2f} h; before the trim: closed {closed}, Euler {chi}, volume {vol0:.4f}")
        except Exception as e:  # without the flag the mesher may find no surface; that is only reported
            if flag:
                raise
            print(f"[{kind}, {tag}] no mesh: {type(e).__name__}: {e}")
    vol, dist, closed, chi, vol0 = results["--orient_normals"]
    assert vol > 0 and dist <= 2.0
    assert closed and chi == (2 if kind == "sphere" else 0) and vol0 > 0


def test_scale_c3_cloud(lib):
    """A 10 M-point cloud sampled like C3, k = 10: the neighbour lists of a 20 k subset bit-identical to the restatement
    over all 10 M points; every spanning-forest edge joins two output normals with a non-negative dot product (the
    parity of the whole forest); time and peak memory printed."""
    from g2pc import orient, synth
    pc = synth.sampled_cloud(3_000_000, 10_000_000, 1236, DEV)
    pts, nrm = pc.points, pc.normals
    del pc
    orient.orient_normals(pts[:1000].contiguous(), nrm[:1000].contiguous())  # warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out, st, dbg = orient.orient_normals(pts, nrm, k=10, return_debug=True)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    m = dbg["rows"].shape[0]
    print(f"[10M] {pts.shape[0]} points ({m} usable), {dt:.3f} s with debug outputs, peak {peak:.2f} GiB above the "
          f"inputs, {st.components} components, {st.flipped} flipped, {st.rounds} rounds")
    assert m > 9_000_000 and dbg["mst"].shape[0] == m - st.components
    e = dbg["edges"][dbg["mst"]]
    o = out[dbg["rows"]].double()
    o = o / o.norm(dim=1, keepdim=True)
    dot = (o[e[:, 0], 0] * o[e[:, 1], 0] + o[e[:, 0], 1] * o[e[:, 1], 1]) + o[e[:, 0], 2] * o[e[:, 1], 2]
    assert int((dot < 0).sum()) == 0
    up = pts[dbg["rows"]].cpu().numpy()
    sub = np.random.default_rng(4).choice(m, 20_000, replace=False)
    want_i, want_d = fo.knn_ids(up, 10, query=sub)
    assert np.array_equal(dbg["ids"][torch.from_numpy(sub).to(DEV)].cpu().numpy(), want_i)
    assert same(dbg["d2"][torch.from_numpy(sub).to(DEV)].cpu().numpy(), want_d)
