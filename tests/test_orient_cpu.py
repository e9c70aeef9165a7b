"""CPU: the float64 restatement of the normal orientation (f64ref_orient) against brute force, scipy's minimum spanning
tree and shapes whose outward side is known; mesh_pc.py's --orient_normals flag."""
import numpy as np
import pytest

import clouds
import f64ref_orient as fo


def _negate_some(n, rng):
    return np.where(rng.random(n.shape[0]) < 0.5, -1.0, 1.0).astype(n.dtype)[:, None] * n


@pytest.mark.parametrize("k", [1, 3, 10, 31])
def test_knn_ids_against_brute_force(k):
    rng = np.random.default_rng(k)
    cases = [rng.random((n, 3)).astype(np.float32) for n in (0, 1, 2, k, k + 1, 300)]
    cases += [clouds.lattice(5), clouds.lattice(4) * np.float32(0.5),
              clouds.dup_runs(200, rng, (k - 1, k, k + 1, k + 2, 2 * k), 3), np.zeros((40, 3), np.float32),
              np.repeat(np.float32([[1.0, 2.0, 3.0]]), k + 1, 0)]
    for p in cases:
        ids, d2 = fo.knn_ids(p, k)
        bi, bd = fo.knn_ids_brute(p, k)
        assert ids.shape == (p.shape[0], k) and np.array_equal(ids, bi) and np.array_equal(d2, bd), p.shape
        kp = max(min(k, p.shape[0] - 1), 0)
        assert (ids[:, kp:] == -1).all() and (ids[:, :kp] >= 0).all()
        assert (ids[:, :kp] != np.arange(p.shape[0])[:, None]).all()  # never the point itself


def test_ties_go_to_the_smaller_index():
    p = clouds.lattice(3)  # the centre (13) has 6 neighbours at d2 = 1, 12 at 2, 8 at 3
    ids, d2 = fo.knn_ids(p, 10)
    c = ids[13]
    assert list(c[:6]) == [4, 10, 12, 14, 16, 22] and (d2[13, :6] == 1).all()
    assert list(c[6:]) == [1, 3, 5, 7] and (d2[13, 6:] == 2).all()
    same = np.zeros((12, 3), np.float32)  # all identical: the k smallest other indices
    ids, d2 = fo.knn_ids(same, 5)
    assert list(ids[0]) == [1, 2, 3, 4, 5] and list(ids[7]) == [0, 1, 2, 3, 4] and (d2 == 0).all()


def test_mst_weight_matches_scipy():
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    rng = np.random.default_rng(2)
    for p, n in (clouds.sphere(2000, rng, noise=1e-3), clouds.torus(3000, rng)[:2]):
        n = _negate_some(n, rng)
        _, info = fo.orient(p, n, k=10)
        e, w, mst = info["edges"], info["weights"].astype(np.float64), info["mst"]
        m = p.shape[0]
        # scipy drops zero weights as missing edges: shift every weight by 1 (every spanning forest has m - c edges)
        g = coo_matrix((w + 1.0, (e[:, 0], e[:, 1])), shape=(m, m))
        want = minimum_spanning_tree(g).sum()
        assert mst.size == m - info["components"]
        assert abs((w[mst] + 1.0).sum() - want) <= 1e-9 * want
        assert len(np.unique(info["keys"])) == e.shape[0]


def _outward(out, p, centres):
    return np.einsum("ij,ij->i", out.astype(np.float64), p.astype(np.float64) - centres)


def test_sphere_and_torus_point_outward():
    rng = np.random.default_rng(4)
    p, n = clouds.sphere(3000, rng, 1.0, (0.3, -0.2, 0.1), noise=1e-3)
    out, info = fo.orient(p, _negate_some(n, rng), k=10)
    assert info["components"] == 1 and (_outward(out, p, np.float64([0.3, -0.2, 0.1])) > 0).all()
    p, n, ring = clouds.torus(6000, rng)
    out, info = fo.orient(p, _negate_some(n, rng), k=10)
    assert info["components"] == 1 and (_outward(out, p, ring) > 0).all()


def test_two_far_spheres_are_two_components():
    rng = np.random.default_rng(6)
    a, na = clouds.sphere(1500, rng, 0.6, (-50, 0, 0), noise=1e-3)
    b, nb = clouds.sphere(1500, rng, 0.5, (50, 0.2, 0), noise=1e-3)
    p, n = np.r_[a, b], _negate_some(np.r_[na, nb], rng)
    out, info = fo.orient(p, n, k=10)
    assert info["components"] == 2
    centres = np.r_[np.tile([-50.0, 0, 0], (1500, 1)), np.tile([50.0, 0.2, 0], (1500, 1))]
    assert (_outward(out, p, centres) > 0).all()
    assert len(set(info["seed"][:1500])) == 1 and len(set(info["seed"][1500:])) == 1


def test_unusable_rows_and_magnitudes():
    rng = np.random.default_rng(8)
    p, n = clouds.sphere(500, rng, noise=1e-3)
    n = n.astype(np.float64) * rng.uniform(1e-3, 1e3, (500, 1))
    n[:5] = 0.0
    n[5:8, 1] = np.nan
    n[8:10, 2] = np.inf
    p[10, 0] = np.nan
    out, info = fo.orient(p, _negate_some(n, rng), k=10)
    assert info["skipped"] == 11 and out.dtype == np.float64
    same = np.isnan(out[:11]) == np.isnan(n[:11])
    assert same.all()
    assert (np.abs(out[11:]) == np.abs(n[11:])).all()
    assert (_outward(out[11:], p[11:], np.zeros(3)) > 0).all()


def test_mesh_pc_flag_parses():
    import mesh_pc
    assert mesh_pc.config_parser(["--input_path", "a.ply"]).orient_normals is False
    assert mesh_pc.config_parser(["--input_path", "a.ply", "--orient_normals"]).orient_normals is True
