"""GPU: gauss_to_mesh.py — g2pc_face_cameras (s11_orient.cu) against the float64 restatement f64ref_face_cameras, the
surface stage of convert_gaussians_to_pc against a recomputation from the renderer's accumulators, and the command end
to end: the topology and the facing of its meshes, its point cloud unchanged from gauss_to_pc.py's, its mesh equal to
g2pc.mesh's on the returned cloud, repeatable runs, and the whole command under compute-sanitizer."""
import math
import os

import numpy as np
import pytest
import torch

import f64ref_mesh as fm
import f64ref_face_cameras as fo
from sanitizer_harness import assert_repeatable, check_target
from test_orient_gpu import _surface_distance, _tangent_scene, _topology, _untrimmed_surface
from util import gpu, same

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))
TARGET = os.path.join(HERE, "gauss_mesh_sanitizer_target.py")
INT32_MAX = 2 ** 31 - 1


# ---- the kernel ---------------------------------------------------------------------------------------------------
def _random_rows(m, ncam, rng, dtype):
    """m rows of N = m + m // 3 Gaussians: random ids, 5 % of the Gaussians unseen, 1 % zero and 0.5 % NaN normals, and
    3 % of the rows sitting exactly on their camera's centre (dot 0)."""
    N = m + m // 3
    ids = rng.permutation(N)[:m].astype(np.int32)
    cam_of = rng.integers(0, ncam, N).astype(np.int32)
    cam_of[rng.random(N) < 0.05] = INT32_MAX
    cams = (rng.normal(size=(ncam, 3)) * 4).astype(np.float32)
    means = rng.normal(size=(m, 3)).astype(np.float32)
    nrm = rng.normal(size=(m, 3)).astype(dtype)
    nrm[rng.random(m) < 0.01] = 0.0
    nrm[rng.random(m) < 0.005, 1] = np.nan
    on_cam = (rng.random(m) < 0.03) & (cam_of[ids] != INT32_MAX)
    means[on_cam] = cams[cam_of[ids[on_cam]]]
    return means, nrm, ids, cam_of, cams


def _kernel(means, nrm, ids, cam_of, cams):
    from g2pc import orient
    N = gpu(nrm)
    out, st = orient.face_cameras(gpu(means), N, gpu(ids), gpu(cam_of), gpu(cams))
    return out.cpu().numpy(), np.array(st, np.int64), N


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
@pytest.mark.parametrize("ncam", [1, 200, 10_000])
@pytest.mark.parametrize("m", [1, 31, 257, 1025, 1_000_000, 3_000_000])
def test_kernel_bit_identical(lib, m, ncam, dtype):
    rng = np.random.default_rng(m * 7 + ncam)
    rows = _random_rows(m, ncam, rng, dtype)
    got, counts, _ = _kernel(*rows)
    want, wcounts = fo.face_cameras(*rows)
    assert same(got, want) and np.array_equal(counts, wcounts), (counts, wcounts)


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_hand_cases(lib, dtype):
    from g2pc import capi
    means, nrm, ids, cam_of, cams, flip, counts = fo.face_camera_hand_cases(dtype)
    with pytest.raises(capi.G2pcError, match="4 row"):  # the hand cases hold 4 invalid rows
        _kernel(means, nrm, ids, cam_of, cams)
    ok = np.r_[np.ones(10, bool), np.zeros(4, bool)]  # without them: the restatement's outputs and counts, bit for bit
    got, c, _ = _kernel(means[ok], nrm[ok], ids[ok], cam_of, cams)
    want, wc = fo.face_cameras(means[ok], nrm[ok], ids[ok], cam_of, cams)
    assert same(got, want) and np.array_equal(c, wc) and tuple(c) == (3, 1, 5, 0)


def test_invalid_input_unchanged_and_negation(lib):
    from g2pc import capi, orient
    rng = np.random.default_rng(5)
    means, nrm, ids, cam_of, cams = _random_rows(50_000, 64, rng, np.float32)
    for bad_ids, bad_cam in ((cam_of.shape[0] + 7, None), (-3, None), (None, 64), (None, -2)):
        i, c = ids.copy(), cam_of.copy()
        if bad_ids is not None:
            i[123] = bad_ids
        else:
            c[i[123]] = bad_cam
        with pytest.raises(capi.G2pcError):
            _kernel(means, nrm, i, c, cams)
    got, counts, N = _kernel(means, nrm, ids, cam_of, cams)
    assert same(N.cpu().numpy(), nrm)  # the input is not modified
    neg, ncounts, _ = _kernel(means, -nrm, ids, cam_of, cams)
    _, wc = fo.face_cameras(means, nrm, ids, cam_of, cams)
    und = np.zeros(ids.shape[0], bool)  # the undecided rows: seen, dot 0 or NaN
    f = cam_of[ids]
    seen = f != INT32_MAX
    d = cams[f[seen]].astype(np.float64) - means[seen]
    with np.errstate(invalid="ignore"):
        dot = (nrm[seen, 0] * d[:, 0] + nrm[seen, 1] * d[:, 1]) + nrm[seen, 2] * d[:, 2]
    und[seen] = ~((dot < 0) | (dot > 0))
    assert int(und.sum()) == counts[2] > 0 and int((~seen).sum()) == counts[1] > 0
    kept = und | ~seen  # undecided and unseen rows keep the sign they are given
    assert same(neg[~kept], got[~kept]) and same(neg[kept], -nrm[kept])
    assert ncounts[1:].tolist() == counts[1:].tolist() and tuple(counts) == tuple(wc)
    e = torch.zeros((0, 3), device=DEV)
    out, st = orient.face_cameras(e, e, torch.zeros((0,), dtype=torch.int32, device=DEV), gpu(cam_of), gpu(cams))
    assert out.shape == (0, 3) and tuple(st) == (0, 0, 0, 0)


# ---- the surface stage --------------------------------------------------------------------------------------------
def _settings(num_points, prioritise=True, res=360):
    import gauss_to_pc as g2p
    return g2p.GaussPointCloudSettings(
        renderer_type="cuda", num_points=num_points, prioritise_visible_gaussians=prioritise,
        mahalanobis_distance_std=2.0, camera_skip_rate=0, render_colours=True, min_opacity=0.0, bounding_box_min=None,
        bounding_box_max=None, calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True,
        colour_resolution=res, max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05,
        surface_distance_std=None, generate_mesh=True, quiet=True, device=DEV)


def _recompute_surface(d, cams, intr, res):
    """Surface ids, first_frame and camera centres from a renderer of our own (the colour stage is deterministic)."""
    import camera_handler as ch
    import gauss_render as gr
    from gauss_handler import Gaussians
    G = Gaussians(d["xyz"], d["scales"], d["rots"], d["colours"].clone() * 255, d["opacities"])
    R = gr.get_renderer("cuda", G.xyz, torch.unsqueeze(torch.clone(G.opacities), 1), G.colours, G.covariances,
                        visible_gaussian_threshold=0.05, calculate_surface_distance=True)
    ff = torch.full((G.xyz.shape[0],), INT32_MAX, dtype=torch.int32, device=DEV)
    R.first_frame = ff
    centres = []
    for c2w, k in zip(cams, intr):
        cam = ch.get_camera("cuda", c2w, k, colour_resolution=res, sh_degree=3, white_bkgd=True)
        centres.append(cam._campos_host)
        R(cam)
    R.flush()
    dist = R.gaussian_min_surface_distance
    mean = float(torch.std_mean(dist[dist < torch.finfo(torch.float).max])[1])
    surf = dist.cpu().numpy() < np.float32(mean)
    keep = np.nonzero(R.gaussian_max_contribution.cpu().numpy() > np.float32(0.05))[0]
    kept = G.fused_cull(max_contribution=R.gaussian_max_contribution, visibility_threshold=0.05)
    assert np.array_equal(kept.cpu().numpy(), keep)
    valid = G.validate_covariances().cpu().numpy()
    ids = keep[valid][surf[keep][valid]]
    return ids, ff.cpu().numpy(), np.float32(centres)


@pytest.mark.parametrize("prioritise", [True, False])
def test_surface_stage(lib, prioritise):
    import gauss_to_pc as g2p
    from g2pc import sampler, synth
    sc = synth.make_scene(20_000, seed=77)
    d = {k: v.to(DEV) for k, v in sc.items()}
    cams, intr = synth.make_cameras(12)
    P, res = 400_000, 360
    sampler.reset_call_counter(0)
    _, surf = g2p.convert_gaussians_to_pc(d["xyz"], d["scales"], d["rots"], d["colours"].clone() * 255, d["opacities"],
                                          d["shs"], {f"c{i}": c for i, c in enumerate(cams)},
                                          {f"c{i}": k for i, k in enumerate(intr)}, None, _settings(P, prioritise, res))
    info = g2p.LAST_SURFACE_STATS
    ids, ff, centres = _recompute_surface(d, cams, intr, res)
    got = info["ids"].cpu().numpy()
    assert np.array_equal(got, ids) and 0 < ids.size < 20_000
    assert same(info["first_frame"].cpu().numpy(), ff)
    assert same(info["cam_centres"].cpu().numpy(), centres)
    f = ff[ids]
    assert ((f >= 0) & (f < len(cams))).all()  # every surface Gaussian was seen: it raised a maximum
    st = info["face_cameras"]
    assert st.unseen == 0 and st.invalid == 0 and st.flipped > 0
    want = min(P // 2, 25 * ids.size)
    n = surf.points.shape[0]
    print(f"[prioritise={prioritise}] {ids.size} surface Gaussians, {n} surface points (target {want}), {st}")
    assert abs(n - want) <= 0.03 * want
    assert surf.normals is not None and surf.normals.shape == surf.points.shape


# ---- the command end to end ---------------------------------------------------------------------------------------
def _inside_cameras(count=14):
    """Cameras at the origin looking out along a Fibonacci sphere of directions, 90 degrees of view each."""
    from g2pc import synth
    cams, intr = [], []
    for i in range(count):
        z = 1 - 2 * (i + 0.5) / count
        a = math.pi * (1 + 5 ** 0.5) * i
        r = math.sqrt(1 - z * z)
        cams.append(synth.look_at_c2w((0.0, 0.0, 0.0), (r * math.cos(a), r * math.sin(a), z)))
        intr.append([480, 480, 240.0, 240.0])
    return cams, intr


def _write_scene(tmp_path, sc, cams, intr):
    from test_io_cpu import write_gaussian_ply, write_transforms_json
    ply, tj = str(tmp_path / "scene.ply"), str(tmp_path / "transforms.json")
    write_gaussian_ply(ply, sc)
    write_transforms_json(tj, cams, intr)
    return ply, tj


def _mesh_cmd(tmp_path, ply, tj, tag, extra=(), depth=7):
    import gauss_to_mesh
    from g2pc import sampler
    cloud, out = str(tmp_path / f"cloud_{tag}.ply"), str(tmp_path / f"mesh_{tag}.ply")
    sampler.reset_call_counter(0)
    surf, m = gauss_to_mesh.main(["--input_path", ply, "--transform_path", tj, "--output_path", cloud,
                                  "--mesh_output_path", out, "--num_points", "200000", "--poisson_depth", str(depth),
                                  "--colour_quality", "original", "--quiet", *extra])
    return cloud, out, surf, m


def _outside():
    """A 3-turn spiral climbing from 3 below to 3 above the equator: every part of the shapes is seen nearly face-on."""
    from g2pc import synth
    cams, intr = synth.make_cameras(48, radius=4.0, height=3.0, turns=3.0)
    return cams, [[640, 360, 533.3, 533.3]] * len(cams)


def _opaque(sc, rng):
    """A Gaussian's best view is then a front view: from outside a closed surface, a view of a Gaussian's back crosses
    the surface first, and almost no light gets through.  (Flat Gaussians give the same peak alpha from both sides.)"""
    sc["opacities"] = torch.from_numpy(rng.uniform(0.9, 0.99, sc["xyz"].shape[0]).astype(np.float32))
    return sc


@pytest.mark.parametrize("kind", ["sphere", "torus"])
def test_cameras_outside(lib, tmp_path, kind):
    from g2pc import mesh
    rng = np.random.default_rng(41)
    ply, tj = _write_scene(tmp_path, _opaque(_tangent_scene(kind, 20_000, rng), rng), *_outside())
    _, out, surf, _ = _mesh_cmd(tmp_path, ply, tj, kind)
    v, _, _, f = mesh.read_mesh_ply(out)
    h = fm.frame(surf.points.cpu().numpy(), 7)["h"]
    closed, chi, vol0 = _topology(*_untrimmed_surface(surf.points, surf.normals, 7))
    dist = float(_surface_distance(v.astype(np.float64), kind).max() / h)
    print(f"[{kind}, outside] {surf.points.shape[0]} surface points; mesh {v.shape[0]} vertices, max distance "
          f"{dist:.2f} h; before the trim: closed {closed}, Euler {chi}, volume {vol0:.4f}")
    assert closed and chi == (2 if kind == "sphere" else 0) and vol0 > 0
    assert fm.signed_volume(v, f) > 0 and dist <= 2.0


def test_cameras_inside(lib, tmp_path):
    """Seen from its centre, the sphere's mesh faces inward, toward the cameras; the neighbour-graph orientation (N7),
    which seeds every component at its topmost point with +z, faces it outward."""
    from g2pc import mesh, orient
    ply, tj = _write_scene(tmp_path, _tangent_scene("sphere", 20_000, np.random.default_rng(42)), *_inside_cameras())
    _, out, surf, _ = _mesh_cmd(tmp_path, ply, tj, "inside")
    v, n, _, f = mesh.read_mesh_ply(out)
    closed, chi, vol0 = _topology(*_untrimmed_surface(surf.points, surf.normals, 7))
    toward = float((np.einsum("ij,ij->i", n.astype(np.float64), v.astype(np.float64)) < 0).mean())
    hoppe = orient.orient_normals(surf.points, surf.normals)[0]
    h_closed, _, h_vol = _topology(*_untrimmed_surface(surf.points, hoppe, 7))
    print(f"[sphere, inside] facing the cameras: closed {closed}, Euler {chi}, volume {vol0:.4f}, {100 * toward:.2f} % "
          f"of vertex normals toward the centre; orient_normals (N7) on the same cloud: closed {h_closed}, volume "
          f"{h_vol:.4f}")
    assert closed and vol0 < 0 and toward >= 0.99
    assert h_vol > 0


def test_colours_follow_the_surface(lib, tmp_path):
    from g2pc import mesh, synth
    rng = np.random.default_rng(43)
    sc = _opaque(_tangent_scene("sphere", 20_000, rng), rng)
    up = sc["xyz"][:, 2] > 0
    dc = 0.5 / synth.SH_C0
    sc["shs"][:, :, 0] = torch.where(up[:, None], torch.tensor([dc, -dc, -dc], dtype=torch.float64),
                                     torch.tensor([-dc, -dc, dc], dtype=torch.float64))
    ply, tj = _write_scene(tmp_path, sc, *_outside())
    _, out, _, _ = _mesh_cmd(tmp_path, ply, tj, "colour")
    v, _, c, _ = mesh.read_mesh_ply(out)
    red = c[:, 0].astype(int) > c[:, 2].astype(int)
    top, bottom = v[:, 2] > 0.1, v[:, 2] < -0.1
    print(f"red above z = 0.1: {red[top].mean():.4f}; blue below z = -0.1: {(~red[bottom]).mean():.4f}")
    assert red[top].mean() > 0.9 and (~red[bottom]).mean() > 0.9


def test_cloud_unchanged_and_mesh_equals_library(lib, tmp_path):
    """The point cloud is byte-identical to gauss_to_pc.py's for the same flags, although meshing makes the renderer
    track surface distances and the first camera of every maximum; the mesh is g2pc.mesh's on the returned cloud."""
    import gauss_to_pc as g2p
    from g2pc import mesh, sampler, synth
    sc = synth.make_scene(30_000, seed=5)
    ply, tj = _write_scene(tmp_path, sc, *synth.make_cameras(8))
    for flags in ([], ["--clean_pointcloud"], ["--no_prioritise_visible_gaussians"]):
        tag = "_".join(f.strip("-") for f in flags) or "default"
        cloud, out, surf, m = _mesh_cmd(tmp_path, ply, tj, tag, flags, depth=8)
        ref = str(tmp_path / f"ref_{tag}.ply")
        sampler.reset_call_counter(0)
        g2p.main(["--input_path", ply, "--transform_path", tj, "--output_path", ref, "--num_points", "200000",
                  "--colour_quality", "original", "--quiet", *flags])
        assert open(cloud, "rb").read() == open(ref, "rb").read(), tag
        lib_mesh = str(tmp_path / f"lib_{tag}.ply")
        mesh.write_mesh_ply(lib_mesh, mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=8,
                                                        laplacian_iters=10, std_ratio=3.0))
        assert open(out, "rb").read() == open(lib_mesh, "rb").read(), tag
        print(f"[{tag}] cloud {os.path.getsize(cloud)} bytes identical; mesh {m.vertices.shape[0]} vertices identical")


def test_determinism_on_poisoned_memory(lib, tmp_path):
    from g2pc import synth
    ply, tj = _write_scene(tmp_path, synth.make_scene(30_000, seed=6), *synth.make_cameras(8))
    runs = iter(range(3))

    def run():
        _, out, _, _ = _mesh_cmd(tmp_path, ply, tj, f"run{next(runs)}", depth=8)
        return [np.frombuffer(open(out, "rb").read(), np.uint8)]

    assert_repeatable(run, byte=0xFF, large_bytes=1 << 30, large_blocks=2)


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_gauss_to_mesh_under_compute_sanitizer(lib, tool, tmp_path):
    check_target(TARGET, "GAUSS_MESH_TARGET_OK", tool, tmp_path, timeout=900)
