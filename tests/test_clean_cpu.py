"""CPU: the float64 restatement of Open3D's statistical outlier removal (f64ref_outliers.statistical_outliers),
pinned against all pairs on small and degenerate clouds, and the CLI accepting --clean_pointcloud without Open3D."""
import numpy as np
import pytest

import clouds
import f64ref_outliers

K = 20


def _clouds():
    rng = np.random.default_rng(5)
    u = lambda n: clouds.uniform(n, rng)
    out = {f"n{n}": u(n) for n in (0, 1, 2, K - 1, K, K + 1)}
    for run in (K - 2, K - 1, K):  # exact duplicates
        out[f"dup{run}"] = np.concatenate([np.repeat(u(1), run, 0), u(40), np.repeat(u(1), run, 0)])
    out["lattice"] = clouds.lattice(5)  # 6 neighbours at 1, 12 at sqrt 2, 8 at sqrt 3: ties at the 20th slot
    out["plane"] = clouds.plane(300, rng, 0.0, 1.0, 0.25)
    t = rng.random(200).astype(np.float32)
    out["line"] = np.stack([t, 2 * t, np.full_like(t, -1)], 1).astype(np.float32)
    return out


@pytest.mark.parametrize("name", sorted(_clouds()))
def test_restatement_matches_all_pairs(name):
    p = _clouds()[name]
    a = f64ref_outliers.knn_mean_distances(p, K)
    b = f64ref_outliers.knn_mean_distances_brute(p, K)
    assert a.shape == (p.shape[0],) and a.tobytes() == b.tobytes()


def test_keep_rule_edges():
    # N = 0: nothing; N = 1: avg 0, NaN statistics, nothing kept
    avg, keep, stats = f64ref_outliers.statistical_outliers(np.zeros((0, 3), np.float32), K, 10.0)
    assert avg.size == 0 and keep.size == 0
    avg, keep, stats = f64ref_outliers.statistical_outliers(np.ones((1, 3), np.float32), K, 10.0)
    assert avg[0] == 0.0 and np.isnan(stats[1]) and not keep.any()
    # a run of >= k exact copies has avg 0 and is removed; k - 1 copies are not
    p = _clouds()[f"dup{K}"]
    avg, keep, _ = f64ref_outliers.statistical_outliers(p, K, 10.0)
    assert (avg[:K] == 0).all() and not keep[:K].any() and keep[K:].any()
    p = _clouds()[f"dup{K - 1}"]
    avg, keep, _ = f64ref_outliers.statistical_outliers(p, K, 10.0)
    assert (avg[:K - 1] > 0).all()
    # avg == 0 points are left out of the sums but counted in n
    mean, std, thr = f64ref_outliers.sor_statistics([0.0, 1.0, 3.0], 1.0)
    assert mean == 4.0 / 3 and std == np.sqrt(((1 - mean) ** 2 + (3 - mean) ** 2) / 2) and thr == mean + std


def test_far_point_is_an_outlier():
    rng = np.random.default_rng(9)
    p = np.concatenate([rng.random((500, 3)), [[1e3, 1e3, 1e3]]]).astype(np.float32)
    _, keep, _ = f64ref_outliers.statistical_outliers(p, K, 3.0)
    assert keep[:500].all() and not keep[500]


def test_cli_accepts_clean_without_open3d(tmp_path):
    import gauss_to_pc as g2p
    args = g2p.config_parser(["--input_path", str(tmp_path / "s.ply"), "--no_render_colours", "--clean_pointcloud"])
    assert args.clean_pointcloud
    with pytest.raises(AttributeError):
        g2p.config_parser(["--input_path", str(tmp_path / "s.ply"), "--no_render_colours", "--generate_mesh"])


def test_clean_refuses_host_tensors():
    import torch
    import mesh_handler
    from g2pc import capi
    with pytest.raises(capi.G2pcError):
        mesh_handler.clean_point_cloud(torch.zeros((4, 3)), None, None)
    with pytest.raises(NotImplementedError if _has_open3d() else ImportError):
        mesh_handler.generate_mesh(torch.zeros((4, 3)), None, None, str("unused.ply"))


def _has_open3d():
    try:
        import open3d  # noqa: F401
        return True
    except ImportError:
        return False
