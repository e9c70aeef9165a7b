"""CPU: the restatement of the hole filling (tests/f64ref_holes.py, DESIGN.md §2, N12) on hand meshes, and the hole flag
of mesh_pc.py, gauss_to_mesh.py and prune_mesh.py, refused before any file is opened."""
import os

import numpy as np
import pytest
from scipy.spatial import ConvexHull

import f64ref_holes as fh


def _outward(p, f):
    """The hull's triangles wound counter-clockwise seen from outside (the hull contains the origin)."""
    f = np.asarray(f, np.int64)
    n = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    flip = (n * p[f].mean(1)).sum(1) < 0
    f[flip] = f[flip][:, [0, 2, 1]]
    return f


def octahedron():
    p = np.array([[1, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], np.float64)
    f = np.array([[0, 2, 4], [2, 1, 4], [1, 3, 4], [3, 0, 4], [2, 0, 5], [1, 2, 5], [3, 1, 5], [0, 3, 5]])
    return p, f


def icosahedron():
    g = (1 + 5 ** 0.5) / 2
    p = np.array([[a, b * g, 0] for a in (-1, 1) for b in (-1, 1)] + [[0, a, b * g] for a in (-1, 1) for b in (-1, 1)] +
                 [[b * g, 0, a] for a in (-1, 1) for b in (-1, 1)], np.float64)
    return p, _outward(p, ConvexHull(p).simplices)


def sphere(n=600):
    """A closed triangulated sphere: the hull of n Fibonacci points."""
    i = np.arange(n) + 0.5
    z = 1 - 2 * i / n
    r = np.sqrt(1 - z * z)
    a = np.pi * (1 + 5 ** 0.5) * i
    p = np.stack([r * np.cos(a), r * np.sin(a), z], 1)
    return p, _outward(p, ConvexHull(p).simplices)


def without_stars(f, centres):
    """The faces that use none of `centres`: a hole around each (the centres are left unused)."""
    return f[~np.isin(f, centres).any(1)]


def grid(n, skip=()):
    """(n+1)^2 vertices, n^2 unit cells of two counter-clockwise triangles each (normal +z); cells in `skip` left out."""
    x, y = np.meshgrid(np.arange(n + 1), np.arange(n + 1))
    p = np.stack([x.ravel(), y.ravel(), np.zeros(x.size)], 1).astype(np.float64)
    f = []
    for j in range(n):
        for i in range(n):
            if (i, j) in skip:
                continue
            a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i + 1, (j + 1) * (n + 1) + i
            f += [[a, b, c], [a, c, d]]
    return p, np.array(f, np.int64).reshape(-1, 3)


def octahedron_open():
    p, f = octahedron()
    return p, f[1:]


def icosahedron_open():
    p, f = icosahedron()
    return p, without_stars(f, [0])


def cube_open():
    """A cube of 12 triangles without its top and bottom squares: two 4-edge holes."""
    p = np.array([[x, y, z] for z in (-1, 1) for y in (-1, 1) for x in (-1, 1)], np.float64)
    f = _outward(p, ConvexHull(p).simplices)
    n = np.cross(p[f[:, 1]] - p[f[:, 0]], p[f[:, 2]] - p[f[:, 0]])
    return p, f[np.abs(n[:, 2]) < 0.5]


def sphere_punched(k=6):
    p, f = sphere()
    centres = [0, 120, 250, 380, 480, 599][:k]
    return p, without_stars(f, centres)


def annulus():
    return grid(3, skip={(1, 1)})


def pinched():
    """Two cells missing that touch at a corner: one boundary set through that corner."""
    return grid(4, skip={(1, 1), (2, 2)})


def lone_triangle():
    return np.random.default_rng(5).normal(size=(3, 3)), np.array([[0, 1, 2]])


def lone_quad():
    return np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float64), np.array([[0, 1, 2], [0, 2, 3]])


def same_direction():
    """Two faces that both use the half-edge 0 -> 1: the edge is used twice, so it is not on the boundary."""
    return np.random.default_rng(6).normal(size=(4, 3)), np.array([[0, 1, 2], [0, 1, 3]])


def tetrahedron():
    p = np.array([[1, 1, 1], [1, -1, -1], [-1, 1, -1], [-1, -1, 1]], np.float64)
    return p, _outward(p, ConvexHull(p).simplices)


HAND = {"octahedron_open": octahedron_open, "icosahedron_open": icosahedron_open, "cube_open": cube_open,
        "sphere_punched": sphere_punched, "grid_4": lambda: grid(4), "annulus": annulus, "pinched": pinched,
        "lone_triangle": lone_triangle, "lone_quad": lone_quad, "same_direction": same_direction,
        "tetrahedron": tetrahedron}


def closed(f):
    """Every directed edge once and its reverse present."""
    f = np.asarray(f, np.int64)
    d = np.stack([f.ravel(), np.roll(f, -1, 1).ravel()], 1)
    u = np.unique(d, axis=0)
    return u.shape[0] == d.shape[0] and np.unique(np.r_[d, d[:, ::-1]], axis=0).shape[0] == d.shape[0]


def volume(p, f):
    a, b, c = p[f[:, 0]], p[f[:, 1]], p[f[:, 2]]
    return float((a * np.cross(b, c)).sum() / 6)


def test_octahedron_one_face():
    p, f = octahedron_open()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=3)
    assert info["holes"] == 1 and info["filled_holes"] == 1 and info["added_triangles"] == 1
    assert P.shape[0] == 6 and F.shape[0] == 8 and closed(F)
    assert list(np.roll(F[-1], -int(np.argmin(F[-1])))) == [0, 2, 4]  # the removed face, wound as it was
    assert fh.euler(6, F) == 2 and volume(P, F) > 0


def test_icosahedron_star_is_a_fan():
    p, f = icosahedron_open()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=5)
    assert info["lengths"][info["labels"][f[0, 0]]] == 5 and info["added_vertices"] == 1
    assert P.shape[0] == 13 and F.shape[0] == 20 and closed(F) and volume(P, F) > 0
    assert (F[-5:, 2] == 12).all()
    ring = np.flatnonzero(info["labels"] >= 0)
    assert ring.shape[0] == 5 and np.allclose(P[12], p[ring].mean(0), rtol=0, atol=1e-15)
    _, info = fh.fill_holes(p, f, max_hole_edges=4)
    assert info["too_long"] == 1 and info["filled_holes"] == 0


def test_cube_two_faces():
    p, f = cube_open()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=4)
    assert info["holes"] == 2 and info["filled_holes"] == 2 and info["added_vertices"] == 2
    assert closed(F) and fh.euler(P.shape[0], F) == 2 and volume(P, F) > 0
    assert np.array_equal(np.sort(P[8:, 2]), [-1.0, 1.0]) and (P[8:, :2] == 0).all()


@pytest.mark.parametrize("k", [1, 3, 6])
def test_punched_sphere_comes_out_closed(k):
    p, f = sphere_punched(k)
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=16)
    assert info["holes"] == k and info["filled_holes"] == k and info["pinched"] == 0
    assert closed(F) and fh.euler(P.shape[0], F) == 2 and volume(P, F) > 0
    assert fh.euler(p.shape[0], f) + k == 2


@pytest.mark.parametrize("n", [2, 4, 7])
def test_grid_outer_loop(n):
    p, f = grid(n)
    for H in (4 * n - 1, 4 * n):
        (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=H)
        assert info["holes"] == 1 and info["boundary_edges"] == 4 * n
        if H < 4 * n:
            assert info["too_long"] == 1 and F is not None and np.array_equal(F, f)
        else:
            assert info["filled_holes"] == 1 and F.shape[0] == f.shape[0] + 4 * n and closed(F)
            assert fh.euler(P.shape[0], F) == 2  # a pillow: the grid and its fan, back to back


def test_annulus_two_loops():
    p, f = annulus()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=4)
    assert info["holes"] == 2 and info["filled_holes"] == 1 and info["too_long"] == 1
    assert info["labels"][5] == 5 and info["lengths"][5] == 4 and info["lengths"][0] == 12
    assert np.array_equal(P[16], [1.5, 1.5, 0.0])
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=12)
    assert info["filled_holes"] == 2 and closed(F)


def test_pinched_stays_open():
    p, f = pinched()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=1024)
    assert info["pinched"] == 1 and info["holes"] == 1  # the outer loop is a hole, the touching pair is not
    assert info["lengths"][6] == 7 and (info["succ"][12] == -1)
    assert F.shape[0] == f.shape[0] + 16 and info["filled"][6] == 0


def test_lone_triangle_and_quad():
    p, f = lone_triangle()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=3)
    assert info["lone_triangles"] == 1 and info["filled_holes"] == 0 and F is not None and F.shape[0] == 1
    p, f = lone_quad()
    (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=4)
    assert info["filled_holes"] == 1 and F.shape[0] == 6 and closed(F) and np.array_equal(P[4], [0.5, 0.5, 0.0])


def test_edge_used_twice_in_one_direction_is_not_boundary():
    p, f = same_direction()
    u, v, _ = fh.boundary_half_edges(4, f)
    assert sorted(zip(u.tolist(), v.tolist())) == [(1, 2), (1, 3), (2, 0), (3, 0)]
    (_, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=8)
    assert info["pinched"] == 1 and info["holes"] == 0 and F.shape[0] == 2


def test_closed_mesh_returns_the_inputs():
    p, f = tetrahedron()
    cols = np.zeros((4, 3), np.uint8)
    out, info = fh.fill_holes(p, f, cols, None, max_hole_edges=3)
    assert out[0] is not None and np.array_equal(out[1], f) and info["boundary_edges"] == 0
    assert (info["labels"] == -1).all() and (info["succ"] == -1).all()


@pytest.mark.parametrize("name", sorted(HAND))
def test_euler_rises_by_filled(name):
    p, f = HAND[name]()
    for H in (3, 4, 16, 1024):
        (P, F, _, _), info = fh.fill_holes(p, f, max_hole_edges=H)
        assert fh.euler(P.shape[0], F) == fh.euler(p.shape[0], f) + info["filled_holes"]
        assert info["holes"] == info["filled_holes"] + info["too_long"] + info["lone_triangles"]
        assert F.shape[0] == f.shape[0] + info["added_triangles"] and P.shape[0] == p.shape[0] + info["added_vertices"]


def test_centre_values():
    p, f = lone_quad()
    cols = np.array([[0, 0, 0], [255, 1, 2], [255, 2, 2], [0, 0, 1]], np.uint8)
    dens = np.array([0.1, 0.2, 0.3, 0.4])
    (P, F, C, D), _ = fh.fill_holes(p, f, cols, dens, max_hole_edges=4)
    assert list(C[4]) == [(2 * 510 + 4) // 8, (2 * 3 + 4) // 8, (2 * 5 + 4) // 8]
    assert D[4] == (((0.1 + 0.2) + 0.3) + 0.4) / 4
    assert [list(x) for x in F[2:]] == [[1, 0, 4], [2, 1, 4], [3, 2, 4], [0, 3, 4]]


# ---- arguments ------------------------------------------------------------------------------------------------------
def test_max_hole_edges_refusals():
    from g2pc import capi, mesh
    for bad in (2, 1025, 0, -4, 3.0, True, "8", None):
        with pytest.raises(capi.G2pcError, match="3..1024"):
            mesh.check_max_hole_edges(bad)
    mesh.check_max_hole_edges(3)
    mesh.check_max_hole_edges(np.int64(1024))


def test_fill_holes_needs_cuda_tensors():
    import torch
    from g2pc import capi, mesh
    p, f = lone_quad()
    with pytest.raises(capi.G2pcError, match="CUDA"):
        mesh.fill_holes(torch.from_numpy(p), torch.from_numpy(f.astype(np.int32)), max_hole_edges=4)
    with pytest.raises(capi.G2pcError, match="3..1024"):
        mesh.fill_holes(torch.from_numpy(p), torch.from_numpy(f.astype(np.int32)), max_hole_edges=2)


def test_mesh_pc_hole_flag(tmp_path):
    import mesh_pc
    missing = str(tmp_path / "missing.ply")
    base = ["--input_path", missing]
    assert mesh_pc.config_parser(base).max_hole_edges is None
    assert mesh_pc.config_parser(base + ["--max_hole_edges", "64"]).max_hole_edges == 64
    for bad in ("2", "1025", "-5", "1.5", "x"):
        with pytest.raises(SystemExit):
            mesh_pc.config_parser(base + ["--max_hole_edges", bad])
    assert not os.path.exists(missing)


@pytest.mark.parametrize("method", ["poisson", "tsdf"])
def test_gauss_to_mesh_hole_flag(tmp_path, method):
    import gauss_to_pc as g2p
    base = ["--input_path", str(tmp_path / "missing.ply"), "--transform_path", str(tmp_path / "missing.json"),
            "--mesh_method", method]
    assert g2p.config_parser(base, mesh=True).max_hole_edges is None
    assert g2p.config_parser(base + ["--max_hole_edges", "1024"], mesh=True).max_hole_edges == 1024
    for bad in ("2", "0", "-1", "1025"):
        with pytest.raises(AttributeError, match="Maximum hole edges"):
            g2p.config_parser(base + ["--max_hole_edges", bad], mesh=True)
    with pytest.raises(SystemExit):
        g2p.config_parser(base + ["--max_hole_edges", "8.5"], mesh=True)
    with pytest.raises(SystemExit):  # gauss_to_pc.py itself has no hole flag
        g2p.config_parser(base[:4] + ["--max_hole_edges", "8"])
    assert not os.path.exists(str(tmp_path / "missing.ply"))


def test_prune_mesh_hole_flag(tmp_path):
    import prune_mesh
    missing = str(tmp_path / "missing.ply")
    a = prune_mesh.config_parser(["--input_path", missing, "--max_hole_edges", "32"])
    assert a.max_hole_edges == 32 and a.min_component_triangles is None and a.keep_largest_components is None
    a = prune_mesh.config_parser(["--input_path", missing, "--min_component_triangles", "5", "--max_hole_edges", "3"])
    assert a.max_hole_edges == 3 and a.min_component_triangles == 5
    assert prune_mesh.config_parser(["--input_path", missing, "--keep_largest_components", "1"]).max_hole_edges is None
    for argv in (["--input_path", missing], ["--max_hole_edges", "10"],
                 ["--input_path", missing, "--max_hole_edges", "2"],
                 ["--input_path", missing, "--max_hole_edges", "1025"],
                 ["--input_path", missing, "--max_hole_edges", "many"]):
        with pytest.raises(SystemExit):
            prune_mesh.config_parser(argv)
    assert not os.path.exists(missing)
