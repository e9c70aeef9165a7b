"""The batched preprocess (g2pc_preprocess_cameras: one pass over the scene for up to 8 cameras) writes exactly what one
g2pc_preprocess per camera writes, byte for byte, and the colour stage / point cloud built on it are the same bits with
config.PREPROCESS_CAMERAS at 1 and at its default — across partial batches, getters called mid-batch and frames that
poison and replay in the middle of a batch."""
import ctypes
import os

import numpy as np
import pytest
import torch

from util import scene_to

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
HERE = os.path.dirname(os.path.abspath(__file__))


def _renderer(sc, shs=True, sh_degree=3):
    import gauss_render as gr
    from oracle import gaussians as og
    cov = og.build_covariance(sc["scales"], sc["rots"])
    d = scene_to(sc, DEV)
    R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov.to(DEV),
                        shs=d["shs"].float() if shs else None, visible_gaussian_threshold=0.05)
    if shs:
        R.sh_degree = sh_degree
    return R


def _cameras(n, res, poses=None):
    import camera_handler as ch
    from g2pc import synth
    cams, intr = poses if poses is not None else synth.make_cameras(n)
    return [ch.get_camera("python", c.to(DEV), k, colour_resolution=res) for c, k in zip(cams, intr)]


def _outputs(R, t):
    n = max(R._n, 1)
    return dict(proj=torch.empty((n, 12), dtype=torch.float32, device=DEV),
                depth_key=torch.empty((n,), dtype=torch.int32, device=DEV),
                val=torch.empty((n,), dtype=torch.int64, device=DEV),
                node_cnt=torch.zeros((t["qt"].nodes_2d,), dtype=torch.int32, device=DEV))


def _scene_args(R):
    from g2pc import capi
    return (capi.ptr(R._geom), capi.ptr(R._colour_f32) if R.shs is None else None, capi.ptr(R.shs),
            int(R.shs.shape[-1]) if R.shs is not None else 0, R.sh_degree, R._n)


def _single(R, t, cam):
    from g2pc import capi
    o = _outputs(R, t)
    c = R._camera_struct(cam)
    capi.call("g2pc_preprocess", *_scene_args(R), ctypes.byref(c), capi.ptr(t["tables"]), capi.ptr(t["luts"]),
              t["qt"].num_levels, t["level_mask"], t["clean_mask"], capi.ptr(o["proj"]), capi.ptr(o["node_cnt"]),
              capi.ptr(o["depth_key"]), capi.ptr(o["val"]), capi.stream_ptr(DEV))
    return o


def _batched(R, t, cams):
    from g2pc import capi
    k = len(cams)
    outs = [_outputs(R, t) for _ in cams]
    ptrs = lambda key: (ctypes.c_void_p * k)(*[capi.ptr(o[key]) for o in outs])
    cs = (capi.Camera * k)(*[R._camera_struct(c) for c in cams])
    capi.call("g2pc_preprocess_cameras", *_scene_args(R), cs, k, capi.ptr(t["tables"]), capi.ptr(t["luts"]),
              t["qt"].num_levels, t["level_mask"], t["clean_mask"], ptrs("proj"), ptrs("node_cnt"), ptrs("depth_key"),
              ptrs("val"), capi.stream_ptr(DEV))
    return outs


def _check_batch(R, cams, extra_levels=0):
    """Every camera's four outputs of one batched call against the single-camera kernel, on the raw bytes."""
    R._extra_levels = extra_levels
    t = R._get_tables(int(cams[0].image_width), int(cams[0].image_height))
    want = [_single(R, t, c) for c in cams]
    got = _batched(R, t, cams)
    torch.cuda.synchronize()
    for ci, (w, g) in enumerate(zip(want, got)):
        for key in ("proj", "depth_key", "val", "node_cnt"):
            assert torch.equal(w[key].view(torch.uint8), g[key].view(torch.uint8)), f"camera {ci}: {key} differs"
    return t, want


@pytest.fixture(scope="module")
def scene():
    from g2pc import synth
    return synth.make_scene(20000 + 77, seed=4242, sh_degree=3)  # not a multiple of any CTA size


@pytest.mark.parametrize("k", [1, 2, 3, 4, 8])
def test_kernel_matches_single_camera_mixed_poses(lib, scene, k):
    R = _renderer(scene)
    cams = _cameras(8, 1280)[:k]  # synth.make_cameras: poses all around the scene
    t, want = _check_batch(R, cams)
    assert int(t["pre_cnt"][0][0].numel()) == t["qt"].nodes_2d
    assert all(int((w["depth_key"] != -1).sum()) > 0 for w in want)


@pytest.mark.parametrize("sh", [None, 0, 1, 2, 3])
def test_kernel_sh_degrees_and_dc_colours(lib, scene, sh):
    R = _renderer(scene, shs=sh is not None, sh_degree=sh or 0)
    _check_batch(R, _cameras(4, 720))


@pytest.mark.parametrize("res,extra", [
    (720, 0), (1280, 1), (1920, 0),
    (1920, 2),   # 21845-word histograms: one camera per launch
    (1920, 3),   # 87381 nodes: no shared-memory histogram, global atomics, one camera per launch
])
def test_kernel_resolutions_and_table_sets(lib, scene, res, extra):
    R = _renderer(scene)
    t, _ = _check_batch(R, _cameras(4, res), extra_levels=extra)
    assert (t["qt"].nodes_2d > 24 * 1024) == (extra == 3)


def test_kernel_edge_cameras(lib):
    """Cameras inside the scene, a camera that sees only Gaussians behind it, and one that sees nothing, in one batch
    with an ordinary pose."""
    import edge_scenes as es
    from g2pc import synth
    sc, c_in, k_in, _, _ = es.inside(n_shell=1500, seed=11, res=(96, 64))
    R = _renderer(sc, sh_degree=0)
    turn = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0]))  # at the origin looking down +z: the probes are behind it
    away = turn.clone()
    away[2, 3] = 1e4  # the whole scene behind the camera
    poses = ([c_in[0], turn, away, synth.make_cameras(1)[0][0]], [k_in[0]] * 4)
    _, want = _check_batch(R, _cameras(4, None, poses))
    assert bool((want[2]["depth_key"] == -1).all()) and int(want[2]["node_cnt"].sum()) == 0
    assert all(int((w["depth_key"] != -1).sum()) > 0 for w in (want[0], want[1]))


# ---- colour stage ---------------------------------------------------------------------------------------------------
def _colour_run(sc, cams, k, monkeypatch, inst_cap=None, getter_after=None, exact_growth=False):
    from g2pc import config, frames
    monkeypatch.setattr(config, "PREPROCESS_CAMERAS", k)
    R = _renderer(sc)
    R.first_frame = torch.full((R._n,), torch.iinfo(torch.int32).max, dtype=torch.int32, device=DEV)
    R.async_mode = True
    failed = []
    if inst_cap is not None:
        R._inst_cap = inst_cap
    if exact_growth:
        # grow the lists to exactly what the failing frame needed: every later frame with more instances poisons too
        R._grow_inst_cap = lambda h: setattr(R, "_inst_cap", max(R._inst_cap, frames.total_instances(h)))
    position = {}
    launch_batch, recover = R._launch_batch, R._recover

    def _launch_batch(batch):
        for j, (f, _, _) in enumerate(batch):
            position[f] = j
        launch_batch(batch)

    def _recover(h):
        failed.append((h[frames.capi.HDR_POISON] - 1, position.get(h[frames.capi.HDR_POISON] - 1)))
        recover(h)

    R._launch_batch, R._recover = _launch_batch, _recover
    for i, c in enumerate(cams):
        R(c)
        if getter_after is not None and i == getter_after:
            R.get_gaussian_colours()
    R.flush()
    return R, failed


def _same_colour_stage(a, b):
    assert torch.equal(a.gaussian_max_contribution, b.gaussian_max_contribution)
    assert torch.equal(a.gaussian_colours, b.gaussian_colours)
    assert torch.equal(a.first_frame, b.first_frame)


@pytest.fixture(scope="module")
def colour_scene():
    from g2pc import synth
    return synth.make_scene(60000, seed=1244, sh_degree=3)


def test_colour_stage_partial_batches(lib, colour_scene, monkeypatch):
    from g2pc import config
    k = config.PREPROCESS_CAMERAS
    assert k > 1
    cams = _cameras(7, 720)  # 7 cameras, batches of 4 + 3
    R1, _ = _colour_run(colour_scene, cams, 1, monkeypatch)
    Rk, _ = _colour_run(colour_scene, cams, k, monkeypatch)
    assert Rk._batch == -(-7 // k) and R1._batch == 7
    _same_colour_stage(R1, Rk)


def test_colour_stage_getter_mid_batch(lib, colour_scene, monkeypatch):
    from g2pc import config
    cams = _cameras(7, 720)
    R1, _ = _colour_run(colour_scene, cams, 1, monkeypatch)
    Rk, _ = _colour_run(colour_scene, cams, config.PREPROCESS_CAMERAS, monkeypatch, getter_after=4)
    _same_colour_stage(R1, Rk)


def test_colour_stage_poison_and_replay_mid_batch(lib, colour_scene, monkeypatch):
    from g2pc import config
    k = config.PREPROCESS_CAMERAS
    cams = _cameras(7, 720)
    # order the cameras by their instance counts, so that with lists grown to exactly one frame's need the next frame
    # poisons again: the first frame of a batch and frames in the middle of one both fail and replay
    R0, _ = _colour_run(colour_scene, cams, 1, monkeypatch)
    counts = []
    for c in cams:
        R0.async_mode = False
        R0(c)
        counts.append(R0.last_stats["total_instances"])
    cams = [cams[i] for i in np.argsort(counts, kind="stable")]
    R1, _ = _colour_run(colour_scene, cams, 1, monkeypatch)
    Rk, failed = _colour_run(colour_scene, cams, k, monkeypatch, inst_cap=1024, exact_growth=True)
    assert Rk.replays >= 1
    assert any(pos == 0 for _, pos in failed), failed
    assert any(pos not in (None, 0) for _, pos in failed), failed
    _same_colour_stage(R1, Rk)


# ---- end to end ----------------------------------------------------------------------------------------------------
def _cloud(sc, k, ncams, res, points, monkeypatch):
    import gauss_to_pc as g2p
    from g2pc import config, sampler, synth
    monkeypatch.setattr(config, "PREPROCESS_CAMERAS", k)
    cams, intr = synth.make_cameras(ncams)
    d = scene_to(sc, DEV)
    st = g2p.GaussPointCloudSettings(
        renderer_type="python", num_points=points, prioritise_visible_gaussians=True, mahalanobis_distance_std=2.0,
        camera_skip_rate=0, render_colours=True, min_opacity=0.0, bounding_box_min=None, bounding_box_max=None,
        calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True, colour_resolution=res,
        max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05, surface_distance_std=None,
        generate_mesh=False, quiet=True, device=DEV)
    sampler.reset_call_counter(0)
    pc, _ = g2p.convert_gaussians_to_pc(d["xyz"], d["scales"], d["rots"], d["colours"].clone(), d["opacities"],
                                        d["shs"], {f"c{i}": c for i, c in enumerate(cams)},
                                        {f"c{i}": q for i, q in enumerate(intr)}, None, st, render_shs=True)
    return pc


@pytest.mark.parametrize("n,ncams,res,points", [
    (100_000, 4, 720, 400_000),      # bench.py's `tiny` workload
    (1_000_000, 9, 720, 2_000_000),  # two full batches and a partial one
])
def test_point_cloud_is_byte_identical(lib, monkeypatch, n, ncams, res, points):
    from g2pc import config, synth
    sc = synth.make_scene(n, seed=1234 + 9, sh_degree=3)
    a = _cloud(sc, 1, ncams, res, points, monkeypatch)
    b = _cloud(sc, config.PREPROCESS_CAMERAS, ncams, res, points, monkeypatch)
    assert a.points.shape[0] > 0
    for name in ("points", "colours", "normals"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_batched_frames_under_compute_sanitizer(lib, tool, tmp_path):
    from sanitizer_harness import check_target
    first = check_target(os.path.join(HERE, "preprocess_batch_sanitizer_target.py"), "PREPROCESS_BATCH_TARGET_OK", tool,
                         tmp_path, timeout=900, repeat_racecheck=True)
    if first is not None:
        assert first["max_contribution"].max() > 0
