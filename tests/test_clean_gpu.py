"""GPU: statistical outlier removal (--clean_pointcloud, g2pc_knn_mean_dist + g2pc_sor_mask + the cull compaction)
against the float64 restatement of Open3D's rule (f64ref_outliers.statistical_outliers).

The per-point mean distances are exact: the kernel evaluates the same float64 operations in the same order as the
oracle, so they must be bit-identical.  The cloud statistics are reduced in a fixed order on the device and
sequentially in the oracle, so they agree to 1e-12 relative; a point whose avg lies within 1e-12 * threshold of the
threshold may then be kept by one and not the other (counted and printed; none are expected)."""
import os
import time
import zlib

import numpy as np
import pytest
import torch

import clouds
import f64ref_outliers
from sanitizer_harness import assert_repeatable, check_target
from util import same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "clean_sanitizer_target.py")
K_MAX = 32
BAND = 1e-12


def _scene(name, rng):
    u = lambda n: clouds.uniform(n, rng)
    if name == "sampled":
        from g2pc import synth
        return synth.sampled_cloud(60_000, 200_000, 71, DEV).points.cpu().numpy()
    if name == "cube":
        return u(100_000)
    if name == "plane":
        return clouds.plane(100_000, rng, -2.0, 2.0, 0.5, jitter=1e-6)
    if name == "dense_sparse":
        return np.concatenate([clouds.clusters(rng, [0.3], [50_000], 1e-4), u(5_000)])
    if name == "isolated":
        return np.concatenate([u(20_000), np.float32([[1e3, 1e3, 1e3], [-1e3, 0, 0], [0, 1e3, -1e3], [2e3, 2e3, 2e3]])])
    if name == "far_clusters":
        return clouds.clusters(rng, clouds.FAR, [5_000] * 4, 1e-3)
    if name == "dup_runs":
        return clouds.dup_runs(3_000, rng, (18, 19, 20, 21, 30, 31, 32, 33, 40), 7)
    if name == "lattice":  # every point on an octree cell boundary
        return clouds.lattice(32)
    if name.startswith("small"):
        return u(int(name[5:]))
    raise KeyError(name)


SCENES = ["sampled", "cube", "plane", "dense_sparse", "isolated", "far_clusters", "dup_runs", "lattice", "small1",
          "small5", "small19", "small31"]


def _avg(p, k):
    from g2pc import outliers
    xyz = torch.from_numpy(np.ascontiguousarray(p, dtype=np.float32)).to(DEV)
    avg, status = outliers.mean_distances(xyz, k)
    assert int(status.item()) == 0
    return avg.cpu().numpy()


def _ulps(a, b):
    ia, ib = a.view(np.int64), b.view(np.int64)
    return np.abs(ia - ib)


@pytest.mark.parametrize("k", [1, 2, 20, K_MAX])
@pytest.mark.parametrize("scene", SCENES)
def test_mean_distances_bit_identical(lib, scene, k):
    rng = np.random.default_rng(zlib.crc32(f"{scene}/{k}".encode()))
    p = _scene(scene, rng)
    got = _avg(p, k)
    want = f64ref_outliers.knn_mean_distances(p, k)
    diff = got.tobytes() != want.tobytes()
    if diff:
        bad = np.nonzero(got != want)[0]
        print(f"[{scene} k={k}] {bad.size} of {p.shape[0]} differ, max {_ulps(got, want).max()} ulp; first "
              f"{bad[:5]} got {got[bad[:5]]} want {want[bad[:5]]}")
    assert not diff


def _check_keep(keep, avg, thr, tag):
    rule = (avg > 0) & (avg < thr)
    band = np.abs(avg - thr) <= BAND * abs(thr)
    off = (keep != rule) & ~band
    print(f"[{tag}] kept {int(keep.sum())} of {avg.size}; {int(band.sum())} point(s) within the threshold band")
    assert not off.any(), f"{int(off.sum())} keep decisions differ outside the band"


@pytest.mark.parametrize("scene", ["sampled", "isolated", "dup_runs", "small1", "small5"])
def test_statistics_and_keep_mask(lib, scene):
    from g2pc import outliers
    p = _scene(scene, np.random.default_rng(3))
    avg_o, keep_o, (mean, std, thr) = f64ref_outliers.statistical_outliers(p, 20, 10.0)
    xyz = torch.from_numpy(p).to(DEV)
    avg, _ = outliers.mean_distances(xyz, 20)
    keep, stats = outliers.sor_mask(avg, 10.0)
    s = stats.cpu().numpy()
    if p.shape[0] == 1:
        assert s[0] == 0.0 and np.isnan(s[1]) and np.isnan(s[2]) and int(keep.sum()) == 0
        return
    for got, want in zip(s, (mean, std, thr)):
        assert abs(got - want) <= 1e-12 * abs(want), (s, (mean, std, thr))
    _check_keep(keep.cpu().numpy().astype(bool), avg_o, thr, scene)


def test_output_rows(lib):
    from g2pc import outliers
    rng = np.random.default_rng(8)
    p = np.concatenate([rng.random((20_000, 3)), rng.uniform(5, 50, (40, 3))]).astype(np.float32)
    n = p.shape[0]
    cols = torch.from_numpy(rng.uniform(-60.0, 320.0, (n, 3)).astype(np.float32)).to(DEV)
    cols[:3] = torch.tensor([[-0.5, 255.0, 255.9], [0.99, 254.99, 1e9], [-1e9, 0.0, 128.5]], device=DEV)
    nrm = torch.from_numpy(rng.normal(size=(n, 3)).astype(np.float32)).to(DEV)
    xyz = torch.from_numpy(p).to(DEV)
    pts, c, nn, dbg = outliers.remove_statistical_outliers(xyz, cols, nrm, 20, 3.0, return_debug=True)
    _, keep_o, _ = f64ref_outliers.statistical_outliers(p, 20, 3.0)
    keep = dbg["keep"].cpu().numpy().astype(bool)
    assert np.array_equal(keep, keep_o) and not keep[20_000:].all()
    assert pts.dtype == torch.float32 and same(pts.cpu().numpy(), p[keep])
    want_c = np.clip(cols.cpu().numpy(), 0, 255).astype(np.int32)[keep]
    assert c.dtype == torch.int32 and np.array_equal(c.cpu().numpy(), want_c)
    assert same(nn.cpu().numpy(), nrm.cpu().numpy()[keep])
    pts2, c2, nn2 = outliers.remove_statistical_outliers(xyz, None, None, 20, 3.0)
    assert c2 is None and nn2 is None and torch.equal(pts2, pts)
    import mesh_handler
    pts3, c3, nn3 = mesh_handler.clean_point_cloud(xyz, cols, None, std_ratio=3.0)
    assert nn3 is None and torch.equal(pts3, pts) and torch.equal(c3, c)
    # an empty cloud comes back empty
    e = torch.zeros((0, 3), device=DEV)
    pe, ce, ne = outliers.remove_statistical_outliers(e, e, None)
    assert pe.shape == (0, 3) and ce.shape == (0, 3) and ce.dtype == torch.int32 and ne is None


def _clean_to_host(xyz, cols, nrm):
    from g2pc import outliers
    out = outliers.remove_statistical_outliers(xyz, cols, nrm, 20, 10.0, return_debug=True)
    return [t.cpu().numpy() for t in out[:3]] + [out[3][k].cpu().numpy() for k in ("avg", "stats", "keep")]


def test_scale_c3_cloud(lib):
    """A 10 M-point cloud sampled like C3: avg on a 20 k subset bit-identical to the oracle over all 10 M points, the
    statistics recomputed on the host from the kernel's avg, the keep rule, and three bit-identical runs (the last one
    on poisoned allocator memory)."""
    from g2pc import synth
    pc = synth.sampled_cloud(3_000_000, 10_000_000, 1236, DEV)
    host = [t.cpu() for t in (pc.points, pc.colours, pc.normals)]
    del pc
    n = host[0].shape[0]
    assert n > 9_000_000
    pts, _, _, avg, s, keep = assert_repeatable(lambda: _clean_to_host(*[t.to(DEV) for t in host]), byte=0x5A,
                                                large_bytes=1 << 30)
    keep = keep.astype(bool)
    p = host[0].numpy()
    sub = np.random.default_rng(4).choice(n, 20_000, replace=False)
    want = f64ref_outliers.knn_mean_distances(p, 20, query=sub)
    assert same(avg[sub], want), f"{int((avg[sub] != want).sum())} of 20000 differ"
    mean, std, thr = f64ref_outliers.sor_statistics(avg, 10.0)
    for got, w in zip(s, (mean, std, thr)):
        assert abs(got - w) <= 1e-12 * abs(w), (s, (mean, std, thr))
    _check_keep(keep, avg, thr, "10M")
    assert same(pts, p[keep])


@pytest.mark.parametrize("case", ["copies", "tiny_cube"])
def test_bounded_work(lib, case):
    """Degenerate clouds finish within 10 s (a bound on the work, not a performance claim)."""
    from g2pc import outliers
    rng = np.random.default_rng(12)
    sparse = rng.uniform(-1.0, 1.0, (1000, 3)).astype(np.float32)
    if case == "copies":
        dense = np.repeat(np.float32([[0.25, -0.5, 0.125]]), 1_000_000, 0)
    else:
        dense = (np.float32(0.1) + rng.uniform(0, 1e-5, (1_000_000, 3))).astype(np.float32)
    p = np.concatenate([dense, sparse])
    xyz = torch.from_numpy(p).to(DEV)
    outliers.remove_statistical_outliers(xyz[:1000], None, None)  # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    _, _, _, dbg = outliers.remove_statistical_outliers(xyz, None, None, return_debug=True)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print(f"[{case}] clean of {p.shape[0]} points: {dt:.3f} s")
    assert dt < 10.0
    avg = dbg["avg"].cpu().numpy()
    if case == "copies":
        assert (avg[:1_000_000] == 0).all() and not dbg["keep"].cpu().numpy()[:1_000_000].any()
        # the k nearest of a scattered point hold at most k copies: the oracle over 20 copies + the sparse points
        want = f64ref_outliers.knn_mean_distances(np.concatenate([dense[:20], sparse]), 20)[20:]
        assert same(avg[1_000_000:], want)
    else:
        sub = np.concatenate([np.arange(0, 1_000_000, 997), np.arange(1_000_000, p.shape[0])])
        want = f64ref_outliers.knn_mean_distances(p, 20, query=sub)
        assert same(avg[sub], want)


def test_cli_clean(lib, tmp_path):
    """g2p.main with and without --clean_pointcloud on the same scene and seed: the cleaned PLY's records are the
    uncleaned PLY's records selected by the oracle's keep mask; --no_calculate_normals writes no normal properties."""
    import gauss_dataloader as gd
    import gauss_to_pc as g2p
    from g2pc import sampler, synth
    from test_io_cpu import write_gaussian_ply
    sc = synth.make_scene(20_000, seed=23, sh_degree=3)
    ply = str(tmp_path / "scene.ply")
    write_gaussian_ply(ply, sc)
    outs = {}
    for tag, extra in (("raw", []), ("clean", ["--clean_pointcloud"]), ("raw_nn", ["--no_calculate_normals"]),
                       ("clean_nn", ["--no_calculate_normals", "--clean_pointcloud"])):
        outs[tag] = str(tmp_path / f"{tag}.ply")
        sampler.reset_call_counter(0)
        g2p.main(["--input_path", ply, "--output_path", outs[tag], "--num_points", "150000", "--no_render_colours",
                  "--quiet"] + extra)
    for raw, clean in (("raw", "clean"), ("raw_nn", "clean_nn")):
        v, c = gd.read_ply_vertices(outs[raw]), gd.read_ply_vertices(outs[clean])
        assert v.dtype == c.dtype
        p = np.stack([v["x"], v["y"], v["z"]], 1)
        avg, keep, (_, _, thr) = f64ref_outliers.statistical_outliers(p, 20, 10.0)
        assert int((np.abs(avg - thr) <= BAND * thr).sum()) == 0
        assert 0 < int(keep.sum()) < p.shape[0] or keep.all()
        assert same(c, v[keep])
    with open(outs["clean_nn"], "rb") as f:
        head = f.read(400).split(b"end_header")[0]
    assert b"nx" not in head and b"red" in head
    with open(outs["clean"], "rb") as f:
        assert b"property float nx" in f.read(400)


def test_errors(lib):
    from g2pc import capi, outliers
    p = torch.rand((100, 3), device=DEV)
    with pytest.raises(capi.G2pcError):
        outliers.remove_statistical_outliers(p.cpu(), None, None)
    for bad in (float("nan"), float("inf"), -float("inf")):
        q = p.clone()
        q[17, 1] = bad
        with pytest.raises(capi.G2pcError, match="non-finite"):
            outliers.remove_statistical_outliers(q, None, None)
    for k in (0, -1, K_MAX + 1):
        with pytest.raises(capi.G2pcError):
            outliers.remove_statistical_outliers(p, None, None, nb_neighbors=k)
    for r in (0.0, -1.0, float("nan")):
        with pytest.raises(capi.G2pcError):
            outliers.remove_statistical_outliers(p, None, None, std_ratio=r)
    with pytest.raises(capi.G2pcError):
        outliers.remove_statistical_outliers(p.double(), None, None)
    with pytest.raises(capi.G2pcError):  # the C ABI refuses k above the cap on its own
        capi.call("g2pc_knn_mean_dist", capi.ptr(p), 100, K_MAX + 1, None, None, None, 0, capi.stream_ptr(DEV))


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_clean_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "CLEAN_TARGET_OK", tool, tmp_path, timeout=600)
