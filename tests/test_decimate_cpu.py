"""CPU: the float64 restatement of the decimation (tests/f64ref_decimate.py, DESIGN.md §2, N9) on hand meshes and
marching-tetrahedra spheres, and the argument checks of decimate(), mesh_pc.py, gauss_to_mesh.py and decimate_mesh.py
(no GPU)."""
import os

import numpy as np
import pytest

import f64ref_decimate as fd
import f64ref_mesh as fm


def _closed_checks(v0, f0, v, f):
    counts, oriented = fm.edge_use(f)
    assert (counts == 2).all() and oriented
    assert fm.euler_characteristic(f, v.shape[0]) == fm.euler_characteristic(f0, v0.shape[0])
    assert fm.components(f) == fm.components(f0)
    assert np.sign(fm.signed_volume(v, f)) == np.sign(fm.signed_volume(v0, f0))


def test_tetrahedron_is_unchanged():
    v, f = fd.tetrahedron()
    p, ff, _, _, info = fd.decimate(v, f, 2, check=True)
    assert not info["reached"] and info["rounds"] == [] and info["free"].all()
    assert (ff == f).all() and (p == v).all()


@pytest.mark.parametrize("name", ["octahedron", "icosphere", "torus"])
def test_closed_meshes_stay_closed(name):
    v, f = getattr(fd, name)()
    target = f.shape[0] // 4
    p, ff, _, _, info = fd.decimate(v, f, target, check=True)
    _closed_checks(v, f, p, ff)
    if info["reached"]:
        assert ff.shape[0] in (target - 1, target)
    else:  # the octahedron: every edge of the 4-face tetrahedron-like remainder fails the link condition
        assert name == "octahedron" and ff.shape[0] == 4
    if name == "torus":
        assert fm.euler_characteristic(ff, p.shape[0]) == 0  # genus 1


def test_open_grid_keeps_its_boundary():
    v, f = fd.grid(12, 0.5)
    colours = (np.arange(v.shape[0] * 3).reshape(-1, 3) % 256).astype(np.uint8)
    p, ff, c, _, info = fd.decimate(v, f, 60, colours=colours, check=True)
    assert ff.shape[0] in (59, 60)
    locked = ~info["free"]
    assert locked.sum() == 48  # the boundary loop of the 13 x 13 grid
    alive = np.ones(v.shape[0], bool)
    for r in info["rounds"]:
        alive[r["ab"][:, 1]] = False
        assert not locked[r["ab"]].any()
    assert alive[locked].all()
    new_index = np.cumsum(alive) - 1
    assert (p[new_index[locked]] == v[locked]).all() and (c[new_index[locked]] == colours[locked]).all()
    assert (fd.boundary_edges(ff) == np.sort(new_index[fd.boundary_edges(f)], 0)).all()


def test_bowtie_and_pinched_vertices_are_locked():
    # two triangles sharing one vertex (an open bowtie), and two octahedra sharing a vertex (a pinch of two closed fans,
    # where the counts alone cannot tell: 8 faces, 8 neighbours, every edge used twice)
    assert not fd.free_flags(np.array([[0, 1, 2], [0, 3, 4]]), 5)[0]
    v, f = fd.octahedron()
    f2 = np.where(f == 0, 0, f + 5)  # the second octahedron shares vertex 0
    flags = fd.free_flags(np.r_[f, f2], 11)
    assert not flags[0] and flags[1:].all()


def test_zero_area_faces():
    v, f = fd.icosphere(2)
    v = np.r_[v, v[f[0]].mean(0, keepdims=True)]
    # split face 0 into three around its centroid, and then make one of them zero-area by moving the centroid onto
    # the edge's midpoint
    a, b, c = f[0]
    k = v.shape[0] - 1
    v[k] = (v[a] + v[b]) * 0.5
    f = np.r_[f[1:], [[a, b, k], [b, c, k], [c, a, k]]]
    Q = fd.quadrics(v, f)
    assert np.isfinite(Q).all()
    p, ff, _, _, info = fd.decimate(v, f, f.shape[0] // 3, check=True)
    assert np.isfinite(p).all() and ff.shape[0] in (f.shape[0] // 3 - 1, f.shape[0] // 3)
    _closed_checks(v, f, p, ff)


def test_flat_plane_uses_the_fallback():
    """Every quadric of a flat grid has rank 1 (A = n n^T / 2|n| sums of one normal), so no minimiser is taken: every
    collapse lands on a, b or the midpoint, all of cost 0, and the tie goes to a."""
    v, f = fd.grid(10, 0.0)
    p, ff, _, _, info = fd.decimate(v, f, 40, check=True)
    assert (p[:, 2] == 0.0).all()
    for r in info["rounds"]:
        assert (r["keys"] >> np.uint64(32) == 0).all()  # cost 0
    # with all costs 0 every collapse keeps a where it was
    q = v.copy()
    for r in info["rounds"]:
        assert (r["vpos"][r["ab"][:, 0]] == q[r["ab"][:, 0]]).all()
        q = r["vpos"]


def test_fold_over_is_refused():
    """A closed pyramid: a fan around b in z = 0 whose ring has a reflex corner, over an apex.  Collapsing b into a
    keeps the link condition but turns the face (b, 4, 5) over, so the edge is no candidate."""
    ring = np.array([[2, 0], [0, 1], [-1, 0], [0, -1], [0.2, -0.2]], float)
    v = np.zeros((7, 3))
    v[1:6, :2] = ring
    v[6] = [0, 0, -3]
    f = np.array([x for i in range(5) for x in ([0, 1 + i, 1 + (i + 1) % 5], [1 + i, 6, 1 + (i + 1) % 5])])
    Q, free = fd.quadrics(v, f), fd.free_flags(f, 7)
    assert free.all()
    s = fd.select(v, f, Q, free)
    e = int(np.nonzero((s["ea"] == 0) & (s["eb"] == 1))[0][0])
    pv, _ = fd.place(Q, v, np.array([0]), np.array([1]))
    n = lambda p0, p1, p2: np.cross(p1 - p0, p2 - p0)
    assert n(v[0], v[4], v[5]) @ n(pv[0], v[4], v[5]) <= 0  # the premise: the move folds face (0, 4, 5)
    assert s["key"][e] == fd.KEY_NONE
    assert s["candidates"] > 0


def test_cost_ties_go_by_edge_id():
    """On a flat grid every candidate costs 0, so keys are edge ids: the smallest candidate id is selected, and every
    selected edge has the smallest candidate id among the candidates at and next to its endpoints."""
    v, f = fd.grid(8, 0.0)
    Q, free = fd.quadrics(v, f), fd.free_flags(f, v.shape[0])
    s = fd.select(v, f, Q, free)
    cand = np.nonzero(s["key"] != fd.KEY_NONE)[0]
    assert (s["key"][cand] == cand.astype(np.uint64)).all()
    assert s["sel"][0] == cand.min()
    nbr = {}
    for x, y in zip(s["ea"], s["eb"]):
        nbr.setdefault(x, {x}).add(y)
        nbr.setdefault(y, {y}).add(x)
    for key in s["sel"]:
        e = int(key)
        near = nbr[s["ea"][e]] | nbr[s["eb"][e]]
        at = [c for c in cand if s["ea"][c] in near or s["eb"][c] in near]
        assert e == min(at)


def _mt_sphere(R=32, radius=11.3, centre=(15.7, 16.2, 15.9)):
    g = np.arange(R) + 0.5
    z, y, x = np.meshgrid(g, g, g, indexing="ij")
    chi = np.sqrt((x - centre[0]) ** 2 + (y - centre[1]) ** 2 + (z - centre[2]) ** 2) - radius
    _, _, vpos, faces = fm.marching_tetrahedra(chi.reshape(-1), R, 0.0)
    return vpos, faces, np.asarray(centre), radius


def test_marching_tetrahedra_sphere_to_a_quarter():
    """h = 1: every vertex stays within 0.5 h of the analytic sphere and the volume within 2 %."""
    v, f, c, r = _mt_sphere()
    target = f.shape[0] // 4
    p, ff, _, _, info = fd.decimate(v, f, target, check=True)
    assert info["reached"] and ff.shape[0] in (target - 1, target)
    _closed_checks(v, f, p, ff)
    dist = np.abs(np.linalg.norm(p - c, axis=1) - r)
    vol, vol0 = fm.signed_volume(p, ff), 4.0 / 3.0 * np.pi * r ** 3
    print(f"[MT sphere R=32] {f.shape[0]} -> {ff.shape[0]} triangles in {len(info['rounds'])} rounds, max distance "
          f"{dist.max():.3f} h, volume {vol / vol0 - 1:+.4f}")
    assert dist.max() <= 0.5 and abs(vol / vol0 - 1.0) <= 0.02


# ---- arguments ------------------------------------------------------------------------------------------------------
def test_target_refusals():
    from g2pc import capi, mesh
    for bad in (0, -1, 1.5, True, "3", None):
        with pytest.raises(capi.G2pcError, match="target_triangles"):
            mesh.check_target(bad)
    mesh.check_target(1)
    mesh.check_target(np.int64(7))


def test_decimate_needs_cuda_tensors():
    import torch
    from g2pc import capi, mesh
    v, f = fd.octahedron()
    with pytest.raises(capi.G2pcError, match="CUDA"):
        mesh.decimate(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32)), 4)


def test_mesh_pc_target_triangles(tmp_path):
    import mesh_pc
    missing = str(tmp_path / "missing.ply")
    base = ["--input_path", missing]
    assert mesh_pc.config_parser(base).target_triangles is None
    assert mesh_pc.config_parser(base + ["--target_triangles", "1000"]).target_triangles == 1000
    for bad in ("0", "-5", "1.5", "x"):
        with pytest.raises(SystemExit):
            mesh_pc.config_parser(base + ["--target_triangles", bad])
    assert not os.path.exists(missing)


def test_gauss_to_mesh_target_triangles(tmp_path):
    import gauss_to_pc as g2p
    base = ["--input_path", str(tmp_path / "missing.ply"), "--transform_path", str(tmp_path / "missing.json")]
    assert g2p.config_parser(base, mesh=True).target_triangles is None
    assert g2p.config_parser(base + ["--target_triangles", "500"], mesh=True).target_triangles == 500
    for bad in ("0", "-2"):
        with pytest.raises(AttributeError, match="Target triangles"):
            g2p.config_parser(base + ["--target_triangles", bad], mesh=True)
    with pytest.raises(SystemExit):
        g2p.config_parser(base + ["--target_triangles", "2.5"], mesh=True)
    with pytest.raises(SystemExit):  # gauss_to_pc.py itself has no --target_triangles
        g2p.config_parser(base + ["--target_triangles", "500"])


def test_decimate_mesh_arguments(tmp_path):
    import decimate_mesh
    missing = str(tmp_path / "missing.ply")
    a = decimate_mesh.config_parser(["--input_path", missing, "--target_triangles", "10"])
    assert a.target_triangles == 10 and a.mesh_output_path == "decimated_mesh.ply"
    for argv in (["--input_path", missing], ["--target_triangles", "10"],
                 ["--input_path", missing, "--target_triangles", "0"],
                 ["--input_path", missing, "--target_triangles", "ten"]):
        with pytest.raises(SystemExit):
            decimate_mesh.config_parser(argv)
    assert not os.path.exists(missing)
