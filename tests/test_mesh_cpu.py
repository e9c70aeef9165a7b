"""CPU: the float64 restatement of the Poisson mesher (f64ref_mesh): marching tetrahedra on analytic signed distances,
the 16 sign patterns of every Kuhn tetrahedron, the density-quantile trim, the mesh PLY round trip and mesh_pc.py's
argument checks."""
import numpy as np
import pytest
import torch

import clouds
import f64ref_mesh as fm

R = 32


def _cell_centres(R):
    """x, y, z of the centres of the R^3 unit cells in chi's order (x fastest), float64."""
    z, y, x = (clouds.lattice(R).astype(np.float64) + 0.5).T
    return x, y, z


def _sphere_sdf(R, c, r):
    x, y, z = _cell_centres(R)
    return np.sqrt((x - c[0]) ** 2 + (y - c[1]) ** 2 + (z - c[2]) ** 2) - r


def _check_closed(faces):
    counts, oriented = fm.edge_use(faces)
    assert (counts == 2).all() and oriented


def test_sphere_closed_genus0_volume():
    r = 11.3
    vkey, vt, vpos, faces = fm.marching_tetrahedra(_sphere_sdf(R, (16.1, 15.8, 16.3), r), R, 0.0)
    assert faces.shape[0] > 1000 and np.all(np.diff(vkey) > 0)
    _check_closed(faces)
    assert fm.euler_characteristic(faces) == 2
    vol = fm.signed_volume(vpos, faces)
    assert vol > 0 and abs(vol - 4.0 / 3.0 * np.pi * r ** 3) <= 0.02 * 4.0 / 3.0 * np.pi * r ** 3
    # every vertex on its lattice edge, strictly crossing
    assert ((vt >= 0) & (vt <= 1)).all()


def test_torus_genus1():
    x, y, z = _cell_centres(R)
    q = np.sqrt((x - 16) ** 2 + (y - 16) ** 2) - 9.0
    vkey, vt, vpos, faces = fm.marching_tetrahedra(np.sqrt(q ** 2 + (z - 16) ** 2) - 3.5, R, 0.0)
    _check_closed(faces)
    assert fm.euler_characteristic(faces) == 0 and fm.components(faces) == 1


def test_two_spheres_two_components():
    chi = np.minimum(_sphere_sdf(R, (9, 9, 16), 6.2), _sphere_sdf(R, (23, 22, 16), 5.7))
    _, _, vpos, faces = fm.marching_tetrahedra(chi, R, 0.0)
    _check_closed(faces)
    assert fm.components(faces) == 2 and fm.euler_characteristic(faces) == 4 and fm.signed_volume(vpos, faces) > 0


def test_inside_out_sphere_has_negative_volume():
    _, _, vpos, faces = fm.marching_tetrahedra(-_sphere_sdf(R, (16, 16, 16), 10.0), R, 0.0)
    assert fm.signed_volume(vpos, faces) < 0


@pytest.mark.parametrize("p", range(6))
def test_every_sign_pattern_of_a_tetrahedron(p):
    """The triangles of each of the 16 inside/outside patterns use exactly the crossing edges (each once in a single
    triangle, each triangle edge twice in a quad), and every triangle has every outside corner strictly in front of it
    and every inside corner strictly behind it (counter-clockwise seen from outside)."""
    v = fm.tet_corners(p)
    xyz = lambda c: np.array([c & 1, (c >> 1) & 1, c >> 2], float)
    for pattern in range(16):
        inside = 0
        for q in range(4):
            if (pattern >> q) & 1:
                inside |= 1 << v[q]
        tris = fm.tet_triangles(p, inside)
        k = bin(pattern).count("1")
        assert len(tris) == {0: 0, 1: 1, 2: 2, 3: 1, 4: 0}[k]
        crossing = {(min(v[a], v[b]), max(v[a], v[b])) for a in range(4) for b in range(a + 1, 4)
                    if ((pattern >> a) & 1) != ((pattern >> b) & 1)}
        used = [e for t in tris for e in t]
        assert set(used) == crossing
        for t in tris:
            pts = [(xyz(a) + xyz(b)) / 2 for a, b in t]
            n = np.cross(pts[1] - pts[0], pts[2] - pts[0])
            for q in range(4):
                s = n @ (xyz(v[q]) - pts[0])
                assert (s < 0) if (pattern >> q) & 1 else (s > 0), (p, pattern, q)


@pytest.mark.parametrize("case", ["ties", "runs", "distinct", "one", "two", "all_equal"])
def test_trim_follows_numpy_linear_quantile(case):
    rng = np.random.default_rng(4)
    d = {"ties": np.repeat(rng.random(7), 13), "runs": np.r_[np.zeros(5), np.full(30, 0.5), rng.random(40)],
         "distinct": rng.random(1001), "one": np.array([0.3]), "two": np.array([0.1, 0.9]),
         "all_equal": np.full(50, 2.0)}[case]
    keep, thr = fm.trim_mask(d)
    s = np.sort(d)
    vi = (d.size - 1) * 0.1
    lo = int(np.floor(vi))
    hi = min(lo + 1, d.size - 1)
    g = vi - lo
    want = s[hi] - (s[hi] - s[lo]) * (1 - g) if g >= 0.5 else s[lo] + (s[hi] - s[lo]) * g
    assert thr == want and np.array_equal(keep, ~(d < want))
    # the trim drops every triangle that uses a removed vertex and keeps the order of the rest
    faces = rng.integers(0, d.size, (60, 3))
    dens, vpos, _, f2, keep2, _ = fm.trim(d, np.arange(d.size * 3.0).reshape(-1, 3), None, faces)
    kept = np.nonzero(keep2)[0]
    assert np.array_equal(kept[f2], faces[keep2[faces].all(1)])


def test_smoothing_and_normals_on_a_tetrahedron():
    v = np.array([[0.0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [5, 5, 5]])
    f = np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]])
    s = fm.smooth(v, f, 1)
    assert np.array_equal(s[4], v[4])  # a vertex without neighbours does not move
    d = np.linalg.norm(v[:4, None] - v[None, :4], axis=2) + 1e-12
    w = np.where(np.eye(4, dtype=bool), 0.0, 1.0 / d)
    want = v[:4] + 0.5 * ((w @ v[:4]) / w.sum(1, keepdims=True) - v[:4])
    assert np.abs(s[:4] - want).max() < 1e-15
    n = fm.vertex_normals(v, f)
    assert np.allclose(n[4], 0) and np.allclose(np.linalg.norm(n[:4], axis=1), 1)
    assert (np.einsum("ij,ij->i", n[:4], v[:4] - v[:4].mean(0)) > 0).all()  # outward


def test_mesh_ply_round_trip(tmp_path):
    from g2pc import mesh
    rng = np.random.default_rng(1)
    m = mesh.Mesh(torch.from_numpy(rng.random((7, 3)).astype(np.float32)), torch.tensor([[0, 1, 2], [2, 3, 6]],
                                                                                        dtype=torch.int32),
                  torch.from_numpy(rng.integers(0, 256, (7, 3)).astype(np.uint8)),
                  torch.from_numpy(rng.normal(size=(7, 3)).astype(np.float32)), torch.from_numpy(rng.random(7)))
    path = str(tmp_path / "m.ply")
    mesh.write_mesh_ply(path, m)
    v, n, c, f = mesh.read_mesh_ply(path)
    assert np.array_equal(v, m.vertices.numpy()) and np.array_equal(n, m.normals.numpy())
    assert np.array_equal(c, m.colours.numpy()) and np.array_equal(f, m.faces.numpy())
    import gauss_dataloader as gd  # the vertex element reads like any other cloud
    rec = gd.read_ply_vertices(path)
    assert np.array_equal(np.stack([rec["x"], rec["y"], rec["z"]], 1), m.vertices.numpy())
    mesh.write_mesh_ply(path, m._replace(colours=None))
    assert (mesh.read_mesh_ply(path)[2] == 255).all()


def test_mesh_pc_arguments(tmp_path):
    import mesh_pc
    a = mesh_pc.config_parser(["--input_path", "c.ply"])
    assert a.poisson_depth == 10 and a.laplacian_iterations == 10 and a.mesh_output_path == "mesh.ply" and not a.quiet
    a = mesh_pc.config_parser(["--input_path", "c.ply", "--mesh_output_path", "o.ply", "--poisson_depth", "7",
                               "--laplacian_iterations", "0", "--quiet"])
    assert (a.poisson_depth, a.laplacian_iterations, a.mesh_output_path, a.quiet) == (7, 0, "o.ply", True)
    for bad in (["--poisson_depth", "1"], ["--poisson_depth", "11"], ["--laplacian_iterations", "-1"]):
        with pytest.raises(SystemExit):
            mesh_pc.config_parser(["--input_path", "c.ply"] + bad)
    with pytest.raises(SystemExit):
        mesh_pc.config_parser([])
    # a cloud without normals is refused before any device work
    import gauss_dataloader as gd
    path = str(tmp_path / "no_normals.ply")
    gd.save_xyz_to_ply(torch.rand(10, 3), path)
    with pytest.raises(ValueError, match="nx"):
        mesh_pc.load_cloud(path)


def test_splat_restatement_conserves_and_skips():
    """Interior splats cancel exactly: B sums to 0 when no contribution leaves the grid; zero / non-finite normals are
    counted as skipped."""
    rng = np.random.default_rng(2)
    p = np.r_[rng.uniform(-1, 1, (500, 3)), [[-3, -3, -3], [3, 3, 3]]].astype(np.float32)
    n = rng.normal(size=p.shape)
    n[:3] = [[0, 0, 0], [np.nan, 1, 0], [np.inf, 0, 0]]
    B, cell, skipped, fr = fm.splat(p, n, 4)
    assert skipped == 3 and (cell[:3] == fm.CELL_NONE).all() and (cell[3:] != fm.CELL_NONE).all()
    assert fr["L"] == 1.1 * 6.0 and fr["h"] == fr["L"] / 16
    # the direct solve satisfies its system
    b = fm.rhs(B, fr)
    chi = fm.solve_direct(b, 16)
    assert fm.residual_ratio(chi, b, 16) < 1e-10 and abs(chi.mean()) < 1e-12 * np.abs(chi).max()
