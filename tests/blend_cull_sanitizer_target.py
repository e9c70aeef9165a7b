"""A default-mode frame sequence of the python back-end (t_stop = config.BLEND_T_STOP, so the blend's footprint cull is
on), meant to be executed under compute-sanitizer (tests/test_blend_cull_gpu.py): memcheck over the blend and the
kernels around it, racecheck over the blend's shared-memory staging while warps walk different subsets of a chunk.

Without the sanitizer the same G2PC_TARGET_POISON / G2PC_TARGET_OUT protocol as sanitizer_target.py applies."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
import camera_handler as ch  # noqa: E402
import gauss_render as gr  # noqa: E402
from g2pc import capi, config, synth  # noqa: E402
from oracle import gaussians as og  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    capi.load().g2pc_blend_set_cull(1)
    sc = synth.make_scene(4000, seed=33, sh_degree=3)
    d = {k: v.to(dev) for k, v in sc.items()}
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(dev)
    R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov, shs=d["shs"],
                        visible_gaussian_threshold=0.05)
    assert R.t_stop == config.BLEND_T_STOP > 0
    R.async_mode = True
    cams, intr = synth.make_cameras(3)
    for c, k in zip(cams, intr):
        R(ch.get_camera("python", c.to(dev), k, colour_resolution=240))
    R.flush()
    mc = R.gaussian_max_contribution
    assert float(mc.max()) > 0
    outputs = {"max_contribution": mc, "colours": R.get_gaussian_colours()}
    return outputs, (int((mc > 0).sum()), R.executed_pairs())


target_main("BLEND_CULL_TARGET_OK", run, large_bytes=256 << 20)
