"""Tiny run of the python colour back-end with the batched preprocess (6 cameras in async mode: a batch of
config.PREPROCESS_CAMERAS, then a partial one), meant to be executed under compute-sanitizer
(tests/test_preprocess_batch_gpu.py): memcheck over the batched preprocess and the frames that read its per-camera
outputs, racecheck over its per-camera shared-memory histograms.  Without the sanitizer the harness runs it directly
(G2PC_TARGET_POISON / G2PC_TARGET_OUT as in sanitizer_target.py)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
import camera_handler as ch  # noqa: E402
import gauss_handler as gh  # noqa: E402
import gauss_render as gr  # noqa: E402
from g2pc import synth  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    sc = synth.make_scene(1500, seed=37, sh_degree=3)
    d = {k: v.to(dev) for k, v in sc.items()}
    G = gh.Gaussians(d["xyz"], d["scales"], d["rots"], d["colours"], d["opacities"], shs=d["shs"])
    cams, intr = synth.make_cameras(6)
    R = gr.get_renderer("python", G.xyz, G.opacities.unsqueeze(1), G.colours, G.covariances, shs=G.shs,
                        visible_gaussian_threshold=0.05)
    R.async_mode = True
    for c, k in zip(cams, intr):
        R(ch.get_camera("python", c.to(dev), k, colour_resolution=180))
    R.flush()
    outputs = dict(max_contribution=R.gaussian_max_contribution, colours=R.get_gaussian_colours())
    return outputs, (R._batch, int((R.gaussian_max_contribution > 0).sum()))


target_main("PREPROCESS_BATCH_TARGET_OK", run, large_bytes=256 << 20)
