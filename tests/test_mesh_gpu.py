"""GPU: the Poisson mesher (s10_mesh.cu through the C ABI, g2pc/mesh.py, mesh_pc.py) against the float64 restatement
f64ref_mesh.

Integer and fixed-order float64 results are compared bit for bit: B, the dual cells and the skip count of the splat; the
vertex keys, triangles, positions, densities, colours and the trim mask of the extraction when it is fed the kernel's own
chi and iso.  The float32 multigrid solve is compared with a sparse direct solve within a stated fraction of chi's
range; the iso-value, the smoothed positions and the normals within stated tolerances."""
import os
import time

import numpy as np
import pytest
import torch

import clouds
import f64ref_mesh as fm
from sanitizer_harness import assert_repeatable, check_target
from util import gpu, same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "mesh_sanitizer_target.py")
CHI_TOL = 2e-5  # |chi_gpu - chi_direct| <= CHI_TOL * range(chi_direct), both mean-free: measured <= 3.4e-6 (DESIGN.md §2)


def _cloud(name, rng, depth, n=20_000):
    """Splat test cloud `name`; n is the size of the clouds that sample a surface (sphere, two spheres, plane, node
    planes, box faces)."""
    if name == "sphere":
        return clouds.sphere(n, rng)
    if name == "two_spheres":
        a, na = clouds.sphere(n // 2, rng, 0.6, (-1, 0, 0))
        b, nb = clouds.sphere(n // 2, rng, 0.5, (1, 0.2, 0))
        return np.r_[a, b], np.r_[na, nb]
    if name == "plane":
        p = clouds.plane(n, rng, -1.0, 1.0, 0.1)
        return p, np.tile(np.float32([0, 0, 1]), (p.shape[0], 1))
    if name == "node_planes":  # bbox [0, 1]^3: points on the (float32-rounded) node planes, f = 0 and f = 1
        R = 1 << depth
        h, o = 1.1 / R, 0.5 - 0.55
        g = o + (np.arange(R) + 0.5) * h
        g = g[(g >= 0) & (g <= 1)]
        p = rng.uniform(0, 1, (n, 3))
        for a in range(3):
            p[a::3, a] = rng.choice(g, p[a::3, a].shape)
        p = np.r_[p, [[0, 0, 0], [1, 1, 1]]].astype(np.float32)
        return p, rng.normal(size=p.shape).astype(np.float32)
    if name == "cube_faces":  # every point on a face of its bounding box, the largest extent along x
        p = rng.uniform(-1, 1, (n, 3)) * np.array([2.0, 1.0, 0.5])
        ax = rng.integers(0, 3, p.shape[0])
        p[np.arange(p.shape[0]), ax] = np.sign(rng.normal(size=p.shape[0])) * np.array([2.0, 1.0, 0.5])[ax]
        return p.astype(np.float32), rng.normal(size=p.shape).astype(np.float32)
    if name == "copies":  # 1 M exact copies: a single node collects 1 M x 2^32
        p = np.r_[np.repeat(np.float32([[0.3, -0.2, 0.1]]), 1_000_000, 0), rng.uniform(-1, 1, (100, 3))]
        n = np.r_[np.repeat(np.float32([[0.0, 0.6, 0.8]]), 1_000_000, 0), rng.normal(size=(100, 3))]
        return p.astype(np.float32), n.astype(np.float32)
    if name == "bad_normals":
        p, n = clouds.sphere(5_000, rng)
        n = n.astype(np.float64) * rng.uniform(1e-3, 1e3, (n.shape[0], 1))
        n[:50] = 0.0
        n[50:60, 1] = np.nan
        n[60:70, 2] = np.inf
        return p, n
    raise KeyError(name)


@pytest.mark.parametrize("name", ["sphere", "two_spheres", "plane", "node_planes", "cube_faces", "copies",
                                  "bad_normals"])
def test_splat_bit_identical(lib, name):
    from g2pc import mesh
    rng = np.random.default_rng(len(name))
    for depth in range(2, 8):
        p, n = _cloud(name, rng, depth)
        frame, B, cell, status = mesh.splat(gpu(p), gpu(n), depth)
        B_o, cell_o, skipped_o, fr = fm.splat(p, n, depth)
        f = frame.cpu().numpy()
        assert f[0:3].tobytes() == fr["origin"].tobytes() and f[3] == fr["h"] and f[4] == fr["L"], (name, depth)
        assert same(B.cpu().numpy(), B_o), (name, depth)
        assert np.array_equal(cell.cpu().numpy().astype(np.int64), cell_o), (name, depth)
        st = status.cpu().numpy()
        assert st[0] == skipped_o and st[1] == 0, (name, depth, st)
        assert f[5] == float(int(B_o.sum())) / B_o.size
    if name == "bad_normals":
        assert skipped_o == 70
    if name == "copies":
        assert np.abs(B_o).max() > 2 ** 49  # far beyond int32, well inside int64


def _stages(p, n, depth, colours=None):
    """The mesher's stages one by one through the C ABI, keeping what each one produced."""
    from g2pc import mesh
    pts, nrm = gpu(p), gpu(n)
    col = gpu(colours, np.int32) if colours is not None else None
    frame, B, cell, status = mesh.splat(pts, nrm, depth)
    B_host = B.cpu().numpy()
    chi, cycles, ratio = mesh.solve(B, frame, depth)
    iso = mesh.iso_value(pts, cell, frame, depth, chi)
    vkey, vt, vpos, faces = mesh.extract(chi, depth, frame, iso, B)
    dens, vcol = mesh.gather(pts, col, cell, frame, depth, vkey, vt, B)
    out = dict(frame=frame.cpu().numpy(), B=B_host, cell=cell.cpu().numpy().astype(np.int64), cycles=cycles,
               ratio=ratio, chi=chi.cpu().numpy(), iso=iso.cpu().numpy(), vkey=vkey.cpu().numpy(), vt=vt.cpu().numpy(),
               vpos=vpos.cpu().numpy(), faces=faces.cpu().numpy(), dens=dens.cpu().numpy(),
               vcol=None if vcol is None else vcol.cpu().numpy())
    d2, p2, c2, f2, keep, thr = mesh.trim(dens, vpos, vcol, faces)
    out.update(keep=keep.cpu().numpy().astype(bool), thr=float(thr.item()), tdens=d2.cpu().numpy(),
               tpos=p2.cpu().numpy(), tfaces=f2.cpu().numpy())
    mesh.smooth(p2, f2, 3)
    v, vn = mesh.vertex_normals(p2, f2)
    out.update(spos=p2.cpu().numpy(), verts=v.cpu().numpy(), normals=vn.cpu().numpy())
    return out


def _fr(frame, depth):
    return dict(origin=frame[0:3].copy(), h=frame[3], L=frame[4], extent=frame[6], R=1 << depth)


@pytest.mark.parametrize("depth", [4, 5, 6])
def test_solve_against_direct(lib, depth):
    rng = np.random.default_rng(depth)
    p, n = clouds.sphere(20_000, rng)
    s = _stages(p, n, depth)
    fr = _fr(s["frame"], depth)
    b = fm.rhs(s["B"], fr)
    x = fm.solve_direct(b, 1 << depth)
    chi = s["chi"].astype(np.float64)
    chi -= chi.mean()
    err = np.abs(chi - x).max() / (x.max() - x.min())
    print(f"[depth {depth}] cycles {s['cycles']} ratio {s['ratio']:.2e} max |chi - direct| / range {err:.2e}")
    assert s["ratio"] <= 1e-5 and err <= CHI_TOL


@pytest.mark.parametrize("depth", [2, 3, 7])
def test_residual_ratio(lib, depth):
    from g2pc import mesh
    p, n = clouds.sphere(50_000, np.random.default_rng(7))
    frame, B, cell, _ = mesh.splat(gpu(p), gpu(n), depth)
    chi, cycles, ratio = mesh.solve(B, frame, depth)
    b = fm.rhs(B.cpu().numpy(), _fr(frame.cpu().numpy(), depth))
    host = fm.residual_ratio(chi.cpu().numpy(), b, 1 << depth)
    print(f"[depth {depth}] cycles {cycles} ratio {ratio:.2e} (host recomputation {host:.2e})")
    assert ratio <= 1e-5 and cycles < 40 and abs(host - ratio) <= 1e-3 * ratio + 1e-7


@pytest.mark.parametrize("name,depth", [("sphere", 6), ("two_spheres", 7), ("torus", 7)])
def test_extraction_against_restatement(lib, name, depth):
    rng = np.random.default_rng(11)
    if name == "torus":
        p, n, _ = clouds.torus(60_000, rng)
    else:
        p, n = _cloud(name, rng, depth)
    colours = rng.integers(0, 256, p.shape)
    s = _stages(p, n, depth, colours)
    fr = _fr(s["frame"], depth)
    R = 1 << depth
    # iso against the restatement over the kernel's mean-free chi
    iso_o = fm.iso_value(p, s["cell"], fr, s["chi"])
    assert abs(s["iso"][1] - iso_o) <= 1e-12 * abs(iso_o)
    iso = s["iso"][1]
    vkey, vt, vpos, faces = fm.marching_tetrahedra(s["chi"], R, iso, fr["origin"], fr["h"])
    assert np.array_equal(s["vkey"], vkey)
    assert same(s["vt"], vt) and same(s["vpos"], vpos)
    rot = lambda f: np.stack([np.roll(r, -int(np.argmin(r))) for r in f]) if len(f) else f
    assert np.array_equal(rot(s["faces"].astype(np.int64)), rot(faces))
    dens, vcol = fm.vertex_density_colour(p, colours, s["cell"], fr, vkey, vt)
    assert same(s["dens"], dens) and np.array_equal(s["vcol"], vcol)
    d2, p2, c2, f2, keep, thr = fm.trim(dens, vpos, vcol, faces)
    assert np.array_equal(s["keep"], keep) and s["thr"] == thr
    assert same(s["tdens"], d2) and same(s["tpos"], p2) and np.array_equal(s["tfaces"], f2)
    sm = fm.smooth(p2, f2, 3)
    assert np.abs(s["spos"] - sm).max() <= 1e-12 * fr["L"]
    nr = fm.vertex_normals(s["spos"], f2)
    assert np.abs(s["normals"] - nr).max() <= 1e-6
    assert same(s["verts"], s["spos"].astype(np.float32))


def _closed_checks(vpos, faces, h, centre=None, radius=None):
    counts, oriented = fm.edge_use(faces)
    assert (counts == 2).all() and oriented
    if radius is not None:
        assert np.abs(np.linalg.norm(vpos - centre, axis=1) - radius).max() <= 2 * h


def test_end_to_end_shapes(lib):
    rng = np.random.default_rng(5)
    depth = 7
    p, n = clouds.sphere(200_000, rng, 1.0, (0.2, -0.1, 0.3))
    s = _stages(p, n, depth)
    _closed_checks(s["vpos"], s["faces"], s["frame"][3], np.array([0.2, -0.1, 0.3]), 1.0)
    assert fm.euler_characteristic(s["faces"]) == 2 and fm.signed_volume(s["vpos"], s["faces"]) > 0
    flipped = _stages(p, -n, depth)
    assert fm.signed_volume(flipped["vpos"], flipped["faces"]) < 0
    p, n, _ = clouds.torus(200_000, rng)
    s = _stages(p, n, depth)
    _closed_checks(s["vpos"], s["faces"], s["frame"][3])
    assert fm.euler_characteristic(s["faces"]) == 0 and fm.components(s["faces"]) == 1
    a, na = clouds.sphere(100_000, rng, 0.6, (-1, 0, 0))
    b, nb = clouds.sphere(100_000, rng, 0.5, (1, 0.2, 0))
    s = _stages(np.r_[a, b], np.r_[na, nb], depth)
    _closed_checks(s["vpos"], s["faces"], s["frame"][3])
    assert fm.components(s["faces"]) == 2
    # the whole pipeline: every triangle after the trim indexes a kept vertex, the normals are unit or zero
    from g2pc import mesh
    m = mesh.poisson_mesh(gpu(p), gpu(n), gpu(rng.uniform(0, 255, p.shape).astype(np.float32)), depth=depth)
    assert int(m.faces.max()) < m.vertices.shape[0] and m.colours.dtype == torch.uint8
    ln = torch.linalg.norm(m.normals.double(), dim=1)
    assert bool(((ln - 1).abs() < 1e-5).logical_or(ln == 0).all())


def _run_to_host(p, n, c):
    from g2pc import mesh
    m, dbg = mesh.poisson_mesh(gpu(p), gpu(n), gpu(c), depth=7, laplacian_iters=4, return_debug=True)
    out = [t.cpu().numpy() for t in m]
    out += [dbg[k].cpu().numpy() for k in ("chi", "iso", "B", "keep", "threshold")] + [dbg["cycles"], dbg["ratio"]]
    return out


def test_determinism_on_poisoned_memory(lib):
    rng = np.random.default_rng(9)
    p, n = clouds.sphere(200_000, rng, noise=1e-3)
    c = rng.uniform(0, 255, p.shape).astype(np.float32)
    assert_repeatable(lambda: _run_to_host(p, n, c), byte=0xFF, large_bytes=1 << 30, large_blocks=2)


def test_refusals(lib):
    from g2pc import capi, mesh
    p, n = clouds.sphere(2_000, np.random.default_rng(1))
    P, N = gpu(p), gpu(n)
    for d in (1, 11):
        with pytest.raises(capi.G2pcError):
            mesh.poisson_mesh(P, N, depth=d)
    with pytest.raises(capi.G2pcError):
        mesh.poisson_mesh(P[:0], N[:0], depth=5)
    with pytest.raises(capi.G2pcError, match="usable normal"):
        mesh.poisson_mesh(P, torch.zeros_like(N), depth=5)
    with pytest.raises(capi.G2pcError):
        mesh.poisson_mesh(P.cpu(), N.cpu(), depth=5)
    with pytest.raises(capi.G2pcError):
        mesh.poisson_mesh(P, None, depth=5)
    q = P.clone()
    q[5, 0] = float("nan")
    with pytest.raises(capi.G2pcError, match="non-finite"):
        mesh.poisson_mesh(q, N, depth=5)
    with pytest.raises(capi.G2pcError):  # copies of one point: the outlier removal keeps none of them
        mesh.poisson_mesh(P[:1].repeat(100, 1), N[:100], depth=5)
    frame, B, _, _ = mesh.splat(P[:1].repeat(100, 1).contiguous(), N[:100], 5)  # zero extent: nothing is splatted
    f = frame.cpu().numpy()
    assert f[3] == 0.0 and f[6] == 0.0 and int(B.abs().sum()) == 0
    with pytest.raises(capi.G2pcError):  # the C ABI refuses depths outside 2..10 on its own
        capi.call("g2pc_mesh_vcycle", None, None, 11, None, 1, None, None, 0, capi.stream_ptr(DEV))


def test_scale_10m_depth10(lib):
    from g2pc import mesh
    rng = np.random.default_rng(3)
    p, n = clouds.sphere(10_000_000, rng, noise=2e-3)
    P, N = gpu(p), gpu(n)
    del p, n
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    m, dbg = mesh.poisson_mesh(P, N, depth=10, return_debug=True)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"[10M, depth 10] {dt:.2f} s, peak {peak:.2f} GiB, {m.vertices.shape[0]} vertices, {m.faces.shape[0]} faces, "
          f"{dbg['cycles']} cycles, ratio {dbg['ratio']:.2e}")
    assert dt < 60.0 and m.faces.shape[0] > 0 and int(m.faces.max()) < m.vertices.shape[0]
    assert dbg["cycles"] < mesh.MAX_CYCLES and dbg["ratio"] <= mesh.TOLERANCE


def test_mesh_pc_command(lib, tmp_path):
    import gauss_to_pc as g2p
    import mesh_pc
    from g2pc import mesh, sampler, synth
    from test_io_cpu import write_gaussian_ply
    sc = synth.make_scene(20_000, seed=23, sh_degree=3)
    ply = str(tmp_path / "scene.ply")
    write_gaussian_ply(ply, sc)
    cloud = str(tmp_path / "cloud.ply")
    sampler.reset_call_counter(0)
    g2p.main(["--input_path", ply, "--output_path", cloud, "--num_points", "150000", "--no_render_colours", "--quiet"])
    out = str(tmp_path / "mesh.ply")
    mesh_pc.main(["--input_path", cloud, "--mesh_output_path", out, "--poisson_depth", "7", "--quiet"])
    v, nn, c, f = mesh.read_mesh_ply(out)
    assert v.shape[0] > 0 and f.shape[0] > 0 and f.min() >= 0 and f.max() < v.shape[0]
    assert np.isfinite(v).all() and np.isfinite(nn).all()


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_mesh_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "MESH_TARGET_OK", tool, tmp_path, timeout=600)
