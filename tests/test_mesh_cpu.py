"""CPU: the float64 restatement of the Poisson mesher (f64ref_mesh): marching tetrahedra on analytic signed distances,
the 16 sign patterns of every Kuhn tetrahedron, the density-quantile trim, the mesh PLY round trip and mesh_pc.py's
argument checks."""
import numpy as np
import pytest
import torch

import clouds
import f64ref_mesh as fm
from util import same

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


@pytest.mark.parametrize("R", [4, 8, 16, 32, 64])
def test_dct_solve_against_sparse_solve(R):
    """The DCT solve against spsolve (R <= 32) and conjugate gradients to 1e-13 (R = 64), on a splatted sphere's b and
    on white noise made mean-free."""
    rng = np.random.default_rng(R)
    p, n = clouds.sphere(4_000, rng, 0.8, (0.1, 0.0, -0.1))
    B, _, _, fr = fm.splat(p, n, R.bit_length() - 1)
    noise = rng.normal(size=R ** 3)
    for b in (fm.rhs(B, fr), noise - noise.mean()):
        x = fm.solve_direct(b, R)
        y = fm.solve_dct(b.copy(), R)
        assert np.abs(y - x).max() <= 1e-11 * (x.max() - x.min()), R
        assert abs(y.mean()) <= 1e-13 * np.abs(y).max()
        assert fm.residual_ratio(y, b, R) < 1e-12


@pytest.mark.parametrize("name", ["sphere", "two_spheres", "plane", "node_planes", "cube_faces", "copies",
                                  "bad_normals"])
def test_sparse_splat_equals_dense(name):
    from test_mesh_gpu import _cloud
    rng = np.random.default_rng(len(name))
    for depth in range(2, 7):
        p, n = _cloud(name, rng, depth)
        B, cell, skipped, fr = fm.splat(p, n, depth)
        nodes, vals, cell_s, skipped_s, fr_s = fm.splat_sparse(p, n, depth)
        nz = np.nonzero(B)[0]
        assert np.array_equal(nodes, nz) and np.array_equal(vals, B[nz]), (name, depth)
        assert np.array_equal(cell_s, cell) and skipped_s == skipped and fr_s["h"] == fr["h"], (name, depth)


def _bumpy_field(R, rng):
    """A sphere's signed distance plus smooth noise on an R^3 grid, float32, with nodes exactly at the iso 0."""
    x, y, z = _cell_centres(R)
    f = np.sqrt((x - R * 0.47) ** 2 + (y - R * 0.52) ** 2 + (z - R * 0.5) ** 2) - R * 0.37
    f = f + 1.5 * np.sin(x * 0.41) * np.cos(y * 0.37 + z * 0.23)
    f = f.astype(np.float32)
    f[rng.choice(f.size, 200, replace=False)] = 0.0
    return f


def test_slab_extraction_matches_whole_grid():
    """Slabs over partitions of k with edges at several offsets give, concatenated, the whole grid's vertices, and its
    triangles as vertex-key triples."""
    R = 64
    rng = np.random.default_rng(6)
    chi = _bumpy_field(R, rng)
    origin, h = np.array([-1.0, 0.5, 2.0]), 0.03
    vkey, vt, vpos, faces = fm.marching_tetrahedra(chi, R, 0.0, origin, h)
    assert faces.shape[0] > 1000
    for edges in ([0, 64], [0, 1, 2, 31, 32, 33, 63, 64], [0, 7, 20, 21, 50, 62, 64], list(range(0, 65, 16))):
        parts = [fm.marching_tetrahedra(chi, R, 0.0, origin, h, k0, k1) for k0, k1 in zip(edges[:-1], edges[1:])]
        assert np.array_equal(np.concatenate([q[0] for q in parts]), vkey), edges
        assert same(np.concatenate([q[1] for q in parts]), vt) and same(np.concatenate([q[2] for q in parts]), vpos)
        assert np.array_equal(np.concatenate([q[3] for q in parts]), vkey[faces]), edges
        ek = [fm.crossed_edges(chi, R, 0.0, k0, k1) for k0, k1 in zip(edges[:-1], edges[1:])]
        assert np.array_equal(np.concatenate([q[0] for q in ek]), vkey) and same(np.concatenate([q[1] for q in ek]), vt)


def test_slab_residual_equals_sparse_residual():
    rng = np.random.default_rng(8)
    for R, slab in ((16, 3), (32, 32), (32, 7)):
        b = rng.normal(size=R ** 3)
        b -= b.mean()
        chi = fm.solve_dct(b.copy(), R).astype(np.float32)
        want = fm.residual_ratio(chi, b, R)
        assert abs(fm.residual_ratio_slabs(chi, b, R, slab) - want) <= 1e-12 * want, (R, slab)


def test_one_ring_packed_keys_sorted_and_distinct():
    rng = np.random.default_rng(12)
    f = rng.integers(0, 50, (300, 3))
    f = np.r_[f, f[:20], f[:5, ::-1]]
    u, v = fm.one_ring(f, 50)
    e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    want = np.unique(np.concatenate([e, e[:, ::-1]]), axis=0)
    assert np.array_equal(np.stack([u, v], 1), want)
