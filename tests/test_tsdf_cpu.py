"""CPU: the float64 restatement of TSDF fusion (N10) on hand cases, the gather's rule on every tetrahedron, a sphere
fused from exact depth maps, and gauss_to_mesh.py's --mesh_method flags (defaults and refusals before any loading)."""
import math

import numpy as np
import pytest

import f64ref_mesh as fm
import f64ref_tsdf as ft

F32 = np.float32


def _camera(eye, target=(0.0, 0.0, 0.0), W=64, H=48, f=40.0):
    import camera_handler as ch
    from g2pc import synth
    return ch.get_camera("cuda", synth.look_at_c2w(eye, target, up=(0.0, 1.0, 0.0)), [W, H, f, f])


def _frame(R, lo=-1.0, h=None):
    h = 2.0 / R if h is None else h
    return dict(origin=np.full(3, lo), h=h, L=h * R, extent=h * R / 1.1, R=R)


def _run(fr, rs, zmed, T=None, image=None, mask=None, trunc=4.0):
    H, W = zmed.shape
    T = np.zeros((H, W), F32) if T is None else T
    image = np.full((3, H, W), 0.5, F32) if image is None else image
    g = ft.new_grid(fr["R"])
    upd = ft.integrate(g, fr, trunc, zmed, T, image, mask, rs._viewmatrix_host, rs._projmatrix_host, rs._bg_host)
    return g, upd


def test_plane_zero_crossing_within_rounding():
    """A camera on the +z axis looking down at a plane of view depth 2: along every observed voxel column the tsdf
    changes sign where the plane is, to float rounding."""
    R = 32
    fr = _frame(R)
    rs = _camera((0.0, 0.0, 2.0))
    zmed = np.full((48, 64), 2.0, F32)  # the plane z = 0 in world
    g, upd = _run(fr, rs, zmed)
    tsdf = g["tsdf"].reshape(R, R, R)
    w = g["weight"].reshape(R, R, R)
    x, y, z = ft.voxel_centres(fr)
    zv, *_ = ft.project(fr, rs._viewmatrix_host, rs._projmatrix_host, 64, 48)
    sdf = (F32(2.0) - zv.astype(F32)).reshape(R, R, R)
    mu = F32(4.0 * fr["h"])
    seen = upd.reshape(R, R, R)
    assert seen.any()
    assert np.array_equal(tsdf[seen], np.minimum(F32(1), sdf[seen] / mu))
    # column through the centre: the sign changes between the layers around z = 0 (|dz| = h / 2 either side)
    col, wc = tsdf[:, R // 2, R // 2], w[:, R // 2, R // 2]
    cross = np.nonzero((col[:-1] > 0) != (col[1:] > 0))[0]
    zs = fr["origin"][2] + (np.arange(R) + 0.5) * fr["h"]
    assert wc[R // 2 - 1] > 0 and wc[R // 2] > 0
    k = int(cross[-1])
    t = col[k] / (col[k] - col[k + 1])
    zc = zs[k] + t * (zs[k + 1] - zs[k])
    assert abs(zc) < 1e-5, zc
    assert (w[: R // 2 - 4 - 1] == 0).all()  # more than mu behind the plane: never updated


def test_skips_behind_near_and_half_pixels():
    R = 16
    fr = _frame(R, lo=-4.0, h=0.5)
    rs = _camera((0.0, 0.0, 0.0), target=(0.0, 0.0, -1.0), W=32, H=32, f=16.0)
    zmed = np.full((32, 32), 1.0, F32)
    g, upd = _run(fr, rs, zmed, trunc=100.0)
    zv, fx, fy, px, py = ft.project(fr, rs._viewmatrix_host, rs._projmatrix_host, 32, 32)
    assert not upd[zv <= 0.2].any() and (zv <= 0.2).any()  # behind the camera and inside the near plane
    inside = (fx >= 0) & (fx < 32) & (fy >= 0) & (fy < 32) & (zv > 0.2)
    assert np.array_equal(upd, inside)



def test_half_pixel_coordinates_round_up():
    """A voxel that projects exactly onto pixel coordinates (15.5, 15.5): floor(p + 1/2) puts it in pixel (16, 16), not
    in one of its three other neighbours.  Only one pixel carries a depth per run, so the voxel is updated iff it is
    that pixel."""
    import camera_handler as ch
    from g2pc import synth
    # origin camera looking down -z, 32 x 32, f = 16: pixel = 15.5 + 16 x / z_view (x right, y down); z_view = 2
    rs = ch.get_camera("cuda", synth.look_at_c2w((0.0, 0.0, 0.0), (0.0, 0.0, -1.0), up=(0.0, 1.0, 0.0)),
                       [32, 32, 16.0, 16.0])
    fr = dict(origin=np.array([-0.5, -0.5, -2.5]), h=1.0, R=2)  # voxel centres x, y in {0, 1}, z in {-2, -1}
    zv, fx, fy, px, py = ft.project(fr, rs._viewmatrix_host, rs._projmatrix_host, 32, 32)
    i000 = 0  # centre (0, 0, -2): pixel (15.5, 15.5) exactly
    assert (px[i000], py[i000]) == (15.5, 15.5) and (fx[i000], fy[i000]) == (16.0, 16.0)
    for pix, want in (((16, 16), True), ((15, 15), False), ((15, 16), False), ((16, 15), False)):
        zmed = np.zeros((32, 32), F32)
        zmed[pix[1], pix[0]] = 2.0
        g, upd = _run(fr, rs, zmed, T=np.zeros((32, 32), F32), image=np.full((3, 32, 32), 0.5, F32))
        assert bool(upd[i000]) is want, pix


def test_masked_pixels_and_zero_median_are_skipped():
    R = 16
    fr = _frame(R)
    rs = _camera((0.0, 0.0, 3.0))
    zmed = np.full((48, 64), 3.0, F32)
    zmed[:, :32] = 0.0
    mask = np.ones(48 * 64, np.int32)
    mask.reshape(48, 64)[:24] = 0
    g, upd = _run(fr, rs, zmed, mask=mask)
    _, fx, fy, _, _ = ft.project(fr, rs._viewmatrix_host, rs._projmatrix_host, 64, 48)
    assert upd.any()
    assert not upd[fx < 32].any() and not upd[fy < 24].any()


def test_sdf_exactly_minus_mu_is_integrated():
    """sdf = -mu exactly takes -1 (sdf < -mu is skipped, sdf = -mu is not)."""
    R = 8
    fr = _frame(R, lo=-1.0, h=0.25)
    rs = _camera((0.0, 0.0, 4.0))
    zv, fx, fy, _, _ = ft.project(fr, rs._viewmatrix_host, rs._projmatrix_host, 64, 48)
    mu = F32(2.0 * fr["h"])
    vox = int(np.argmin(np.abs(fx - 32) + np.abs(fy - 24) + np.abs(zv - 4.0)))
    target = F32(zv[vox]) - mu  # z_med that puts this voxel at sdf = -mu exactly
    assert target - F32(zv[vox]) == -mu
    zmed = np.full((48, 64), target, F32)
    g, upd = _run(fr, rs, zmed, trunc=2.0)
    assert upd[vox] and g["tsdf"][vox] == F32(-1.0)
    below = (zmed.reshape(-1)[0] - zv.astype(F32)) < -mu
    assert not upd[below].any()


@pytest.mark.parametrize("p", range(6))
def test_gather_keeps_exactly_the_observed_tetrahedra(p):
    """Every sign pattern of Kuhn tetrahedron p and every set of unobserved corners: a triangle survives the gather iff
    all four corners of its tetrahedron are observed, because each triangle has a vertex on an edge at every corner."""
    corners = fm.tet_corners(p)
    for signs in range(16):
        inside = sum(1 << corners[q] for q in range(4) if (signs >> q) & 1)
        tris = fm.tet_triangles(p, inside)
        for unobs in range(16):
            observed = {corners[q] for q in range(4) if not (unobs >> q) & 1}
            for tri in tris:
                kept = all(a in observed and b in observed for a, b in tri)
                assert kept == (len(observed) == 4), (p, signs, unobs, tri)
            if tris:
                touched = {c for tri in tris for e in tri for c in e}
                assert touched == set(corners)


def _sphere_cameras(inside=False, count=24):
    from g2pc import synth
    cams = []
    for i in range(count):
        z = 1 - 2 * (i + 0.5) / count
        a = math.pi * (1 + 5 ** 0.5) * i
        r = math.sqrt(1 - z * z)
        d = (r * math.cos(a), r * math.sin(a), z)
        if inside:
            cams.append(_camera((0.0, 0.0, 0.0), target=d, W=96, H=96, f=48.0))
        else:
            cams.append(_camera(tuple(3.0 * c for c in d), W=96, H=96, f=60.0))
    return cams


def _fuse_sphere(inside):
    R = 64
    rng = np.random.default_rng(0)
    p = rng.normal(size=(4000, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    fr = ft.frame(p.astype(F32), 6)
    g = ft.new_grid(R)
    for rs in _sphere_cameras(inside):
        zmed, T, image = ft.sphere_images(rs)
        ft.integrate(g, fr, 4.0, zmed, T, image, None, rs._viewmatrix_host, rs._projmatrix_host, rs._bg_host)
    return fr, g


def test_sphere_from_outside():
    fr, g = _fuse_sphere(False)
    v, f, c, d, keep = ft.mesh(g, fr)
    counts, oriented = fm.edge_use(f)
    chi, vol = fm.euler_characteristic(f), fm.signed_volume(v, f)
    dist = np.abs(np.linalg.norm(v, axis=1) - 1.0).max() / fr["h"]
    print(f"sphere from outside: {v.shape[0]} vertices, {f.shape[0]} triangles, Euler {chi}, volume {vol:.4f}, "
          f"max distance {dist:.3f} h, {int((~keep).sum())} vertices dropped by the gather")
    assert (counts == 2).all() and oriented and chi == 2 and vol > 0 and dist <= 1.0
    # running float32 means of one colour stay within rounding of it: 255 x = (51, 153, 229.5)
    assert (np.abs(c.astype(int) - np.array([51, 153, 229.5])) <= 0.5).all()


def test_sphere_from_the_centre_faces_inward():
    fr, g = _fuse_sphere(True)
    v, f, *_ = ft.mesh(g, fr)
    counts, oriented = fm.edge_use(f)
    vol = fm.signed_volume(v, f)
    print(f"sphere from the centre: {v.shape[0]} vertices, Euler {fm.euler_characteristic(f)}, volume {vol:.4f}")
    assert (counts == 2).all() and oriented and vol < 0


# ---- command flags ---------------------------------------------------------------------------------------------------
def _argv(tmp_path, *extra):
    return ["--input_path", str(tmp_path / "missing.ply"), "--transform_path", str(tmp_path / "missing.json"),
            *extra]


def test_flag_defaults(tmp_path):
    import gauss_to_mesh
    import gauss_to_pc as g2p
    args = gauss_to_mesh.config_parser(_argv(tmp_path))
    assert (args.mesh_method, args.tsdf_depth, args.tsdf_trunc) == ("poisson", 9, 4.0)
    assert (args.poisson_depth, args.laplacian_iterations, args.band_depth, args.target_triangles) == (10, 10, None, None)
    args = gauss_to_mesh.config_parser(_argv(tmp_path, "--mesh_method", "tsdf", "--tsdf_depth", "10", "--tsdf_trunc",
                                             "2.5", "--target_triangles", "1000"))
    assert (args.mesh_method, args.tsdf_depth, args.tsdf_trunc, args.target_triangles) == ("tsdf", 10, 2.5, 1000)
    assert gauss_to_mesh.config_parser(_argv(tmp_path, "--mesh_method", "tsdf", "--tsdf_depth", "2")).tsdf_depth == 2
    # --poisson_depth has no effect with tsdf, so it is not range-checked there
    assert gauss_to_mesh.config_parser(_argv(tmp_path, "--mesh_method", "tsdf", "--poisson_depth", "12")).poisson_depth == 12
    # gauss_to_pc.py has none of these flags
    assert not hasattr(g2p.config_parser(_argv(tmp_path)), "mesh_method")
    with pytest.raises(SystemExit):
        g2p.config_parser(_argv(tmp_path, "--mesh_method", "tsdf"))


@pytest.mark.parametrize("extra", [
    ["--mesh_method", "tsdf", "--band_depth", "11"],
    ["--mesh_method", "tsdf", "--band_depth", "5"],
    ["--mesh_method", "tsdf", "--tsdf_depth", "1"],
    ["--mesh_method", "tsdf", "--tsdf_depth", "11"],
    ["--mesh_method", "tsdf", "--tsdf_trunc", "0"],
    ["--mesh_method", "tsdf", "--tsdf_trunc", "-1"],
    ["--mesh_method", "tsdf", "--renderer_type", "python"],
])
def test_refusals_before_loading(tmp_path, extra):
    import gauss_to_mesh
    with pytest.raises(AttributeError):
        gauss_to_mesh.main(_argv(tmp_path, *extra))


def test_unknown_method_refused(tmp_path):
    import gauss_to_mesh
    with pytest.raises(SystemExit):
        gauss_to_mesh.config_parser(_argv(tmp_path, "--mesh_method", "marching_cubes"))
