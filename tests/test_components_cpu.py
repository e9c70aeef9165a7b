"""CPU: the restatement of the component filter (tests/f64ref_components.py, DESIGN.md §2, N11) on hand meshes, and the
component flags of mesh_pc.py, gauss_to_mesh.py and prune_mesh.py, refused before any file is opened."""
import os

import numpy as np
import pytest

import f64ref_components as fc

TET = np.array([[0, 1, 2], [0, 3, 1], [1, 3, 2], [2, 3, 0]])


def two_tetrahedra():
    """Vertices 0..3 and 4..7, the second one's faces listed first."""
    return np.random.default_rng(0).normal(size=(8, 3)), np.r_[TET + 4, TET]


def bowtie():
    """Two faces that share vertex 0 only."""
    return np.random.default_rng(1).normal(size=(5, 3)), np.array([[0, 1, 2], [0, 3, 4]])


def with_isolated():
    """A tetrahedron on vertices 1, 3, 5, 6; vertices 0, 2, 4 and 7 are used by no face."""
    ids = np.array([1, 3, 5, 6])
    return np.random.default_rng(2).normal(size=(8, 3)), ids[TET]


def degenerate():
    """Faces that use a vertex twice or thrice: [2, 2, 3] joins 2 and 3, [5, 5, 5] is a component of size 1 on its own."""
    return np.random.default_rng(3).normal(size=(6, 3)), np.array([[0, 1, 0], [2, 2, 3], [5, 5, 5], [1, 1, 1]])


def pieces(sizes, rng=None):
    """Disjoint triangle fans with the given triangle counts, their vertex blocks in the order given."""
    v, f, base = [], [], 0
    for s in sizes:
        n = s + 2
        f += [[base, base + i + 1, base + i + 2] for i in range(s)]
        base += n
    return np.random.default_rng(4).normal(size=(base, 3)), np.array(f)


HAND = {"two_tetrahedra": two_tetrahedra, "bowtie": bowtie, "with_isolated": with_isolated, "degenerate": degenerate,
        "ties": lambda: pieces([3, 5, 2, 5, 5, 1])}


def test_two_tetrahedra():
    v, f = two_tetrahedra()
    (p, ff, _, _), info = fc.remove_components(v, f, min_triangles=1)
    assert (info["labels"] == [0, 0, 0, 0, 4, 4, 4, 4]).all()
    assert info["sizes"][0] == 4 and info["sizes"][4] == 4 and info["components"] == 2
    assert ff.shape == (8, 3) and (p == v).all() and (ff == f).all()
    (p, ff, _, _), info = fc.remove_components(v, f, keep_largest=1)
    assert info["kept"] == 1 and (p == v[:4]).all() and (ff == TET).all()  # tie: the smaller label wins


def test_bowtie_is_one_component():
    v, f = bowtie()
    (p, ff, _, _), info = fc.remove_components(v, f, keep_largest=1)
    assert (info["labels"] == 0).all() and info["sizes"][0] == 2 and info["components"] == 1
    assert ff.shape[0] == 2 and p.shape[0] == 5


def test_isolated_vertices_are_removed():
    v, f = with_isolated()
    (p, ff, _, _), info = fc.remove_components(v, f, min_triangles=1)
    assert info["removed_vertices"] == 4 and info["removed_triangles"] == 0 and info["components"] == 1
    assert (p == v[[1, 3, 5, 6]]).all() and (ff == TET).all()
    assert info["labels"][0] == 0 and info["sizes"][0] == 0 and info["labels"][3] == 1


def test_degenerate_faces():
    v, f = degenerate()
    (p, ff, _, _), info = fc.remove_components(v, f, min_triangles=1)
    assert list(info["labels"]) == [0, 0, 2, 2, 4, 5]
    assert info["sizes"][0] == 2 and info["sizes"][2] == 1 and info["sizes"][5] == 1 and info["sizes"][4] == 0
    assert info["components"] == 3 and p.shape[0] == 5 and (ff == [[0, 1, 0], [2, 2, 3], [4, 4, 4], [1, 1, 1]]).all()
    (p, ff, _, _), info = fc.remove_components(v, f, min_triangles=2)
    assert (ff == [[0, 1, 0], [1, 1, 1]]).all() and p.shape[0] == 2


def test_ties_at_the_kth_size_go_to_the_smaller_label():
    v, f = pieces([3, 5, 2, 5, 5, 1])
    labels = fc.labels_of(v.shape[0], f)
    starts = [0, 5, 12, 16, 23, 30]
    assert sorted(set(labels.tolist())) == starts
    _, kept = fc.keep_of(labels, fc.sizes_of(v.shape[0], f, labels), keep_largest=2)
    assert list(kept) == [5, 16]
    (_, ff, _, _), info = fc.remove_components(v, f, keep_largest=4)
    assert info["kept"] == 4 and ff.shape[0] == 5 + 5 + 5 + 3


def test_k_larger_than_the_component_count():
    v, f = pieces([3, 5, 2])
    (p, ff, _, _), info = fc.remove_components(v, f, keep_largest=10)
    assert info["kept"] == 3 and (p == v).all() and (ff == f).all()


def test_both_parameters():
    v, f = pieces([3, 5, 2, 5, 5, 1])
    (_, ff, _, _), info = fc.remove_components(v, f, min_triangles=3, keep_largest=5)
    assert info["kept"] == 4 and ff.shape[0] == 18  # the 2 and the 1 fail min_triangles, the rank does not bind
    (_, ff, _, _), info = fc.remove_components(v, f, min_triangles=3, keep_largest=2)
    assert info["kept"] == 2 and ff.shape[0] == 10


def test_attributes_travel_with_their_vertices():
    v, f = pieces([1, 4])
    cols = np.arange(v.shape[0] * 3, dtype=np.uint8).reshape(-1, 3)
    dens = np.arange(v.shape[0], dtype=np.float64) + 0.5
    (p, ff, c, d), _ = fc.remove_components(v, f, cols, dens, min_triangles=2)
    assert (p == v[3:]).all() and (c == cols[3:]).all() and (d == dens[3:]).all() and ff.min() == 0


def test_everything_removed_raises():
    v, f = pieces([3, 5])
    with pytest.raises(fc.NothingKept, match="largest has 5"):
        fc.remove_components(v, f, min_triangles=6)
    with pytest.raises(fc.NothingKept, match="largest has 0"):
        fc.remove_components(v, np.zeros((0, 3), np.int32), min_triangles=1)


# ---- arguments ------------------------------------------------------------------------------------------------------
def test_component_parameter_refusals():
    from g2pc import capi, mesh
    for bad in (0, -1, 1.5, True, "3"):
        with pytest.raises(capi.G2pcError, match="integer >= 1"):
            mesh.check_component_params(bad, None)
        with pytest.raises(capi.G2pcError, match="integer >= 1"):
            mesh.check_component_params(None, bad)
    with pytest.raises(capi.G2pcError, match="give min_triangles, keep_largest or both"):
        mesh.check_component_params(None, None)
    mesh.check_component_params(None, None, need_one=False)
    mesh.check_component_params(1, np.int64(3))


def test_remove_components_needs_cuda_tensors():
    import torch
    from g2pc import capi, mesh
    v, f = bowtie()
    with pytest.raises(capi.G2pcError, match="CUDA"):
        mesh.remove_components(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), min_triangles=1)
    with pytest.raises(capi.G2pcError, match="give min_triangles"):
        mesh.remove_components(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)))


def test_mesh_pc_component_flags(tmp_path):
    import mesh_pc
    missing = str(tmp_path / "missing.ply")
    base = ["--input_path", missing]
    a = mesh_pc.config_parser(base)
    assert a.min_component_triangles is None and a.keep_largest_components is None
    a = mesh_pc.config_parser(base + ["--min_component_triangles", "100", "--keep_largest_components", "2"])
    assert a.min_component_triangles == 100 and a.keep_largest_components == 2
    for flag in ("--min_component_triangles", "--keep_largest_components"):
        for bad in ("0", "-5", "1.5", "x"):
            with pytest.raises(SystemExit):
                mesh_pc.config_parser(base + [flag, bad])
    assert not os.path.exists(missing)


@pytest.mark.parametrize("method", ["poisson", "tsdf"])
def test_gauss_to_mesh_component_flags(tmp_path, method):
    import gauss_to_pc as g2p
    base = ["--input_path", str(tmp_path / "missing.ply"), "--transform_path", str(tmp_path / "missing.json"),
            "--mesh_method", method]
    a = g2p.config_parser(base, mesh=True)
    assert a.min_component_triangles is None and a.keep_largest_components is None
    a = g2p.config_parser(base + ["--min_component_triangles", "50", "--keep_largest_components", "1"], mesh=True)
    assert a.min_component_triangles == 50 and a.keep_largest_components == 1
    for bad in ("0", "-2"):
        with pytest.raises(AttributeError, match="Minimum component triangles"):
            g2p.config_parser(base + ["--min_component_triangles", bad], mesh=True)
        with pytest.raises(AttributeError, match="Largest components"):
            g2p.config_parser(base + ["--keep_largest_components", bad], mesh=True)
    with pytest.raises(SystemExit):
        g2p.config_parser(base + ["--keep_largest_components", "2.5"], mesh=True)
    for flag in ("--min_component_triangles", "--keep_largest_components"):
        with pytest.raises(SystemExit):  # gauss_to_pc.py itself has no component flags
            g2p.config_parser(base[:4] + [flag, "5"])
    assert not os.path.exists(str(tmp_path / "missing.ply"))


def test_prune_mesh_arguments(tmp_path):
    import prune_mesh
    missing = str(tmp_path / "missing.ply")
    a = prune_mesh.config_parser(["--input_path", missing, "--min_component_triangles", "10"])
    assert a.min_component_triangles == 10 and a.keep_largest_components is None
    assert a.mesh_output_path == "pruned_mesh.ply"
    a = prune_mesh.config_parser(["--input_path", missing, "--keep_largest_components", "3"])
    assert a.keep_largest_components == 3
    for argv in (["--input_path", missing], ["--min_component_triangles", "10"],
                 ["--input_path", missing, "--min_component_triangles", "0"],
                 ["--input_path", missing, "--keep_largest_components", "-1"],
                 ["--input_path", missing, "--keep_largest_components", "two"]):
        with pytest.raises(SystemExit):
            prune_mesh.config_parser(argv)
    assert not os.path.exists(missing)
