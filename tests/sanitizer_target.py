"""Tiny run of both colour back-ends + the sampler, meant to be executed under compute-sanitizer
(tests/test_sanitizer_gpu.py): memcheck over every g2pc kernel, racecheck over the shared-memory protocols of the blend
(TMA / cp.async staging buffers, s_best merge) and the multisplit bit matrix.

Without the sanitizer (tests/test_sanitizer_gpu.py runs it directly when the tool does not support the GPU):
  G2PC_TARGET_POISON=<byte>   every block PyTorch's caching allocator hands out afterwards starts filled with <byte>
  G2PC_TARGET_OUT=<file.npz>  every output of the run is saved there, for bit-for-bit comparison between runs"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
import camera_handler as ch  # noqa: E402
import gauss_handler as gh  # noqa: E402
import gauss_render as gr  # noqa: E402
import gauss_to_pc as g2p  # noqa: E402
from g2pc import synth  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    outputs = {}
    sc = synth.make_scene(1500, seed=31, sh_degree=3)
    d = {k: v.to(dev) for k, v in sc.items()}
    G = gh.Gaussians(d["xyz"], d["scales"], d["rots"], d["colours"], d["opacities"], shs=d["shs"])
    G.calculate_normals()
    cams, intr = synth.make_cameras(2)
    for rtype in ("python", "cuda"):
        R = gr.get_renderer(rtype, G.xyz, G.opacities.unsqueeze(1), G.colours, G.covariances, shs=G.shs,
                            visible_gaussian_threshold=0.05, surface_distance_std=2.0 if rtype == "cuda" else None,
                            calculate_surface_distance=rtype == "cuda")
        R.async_mode = True
        for c, k in zip(cams, intr):
            R(ch.get_camera(rtype, c.to(dev), k, colour_resolution=180))
        R.flush()
        mc = R.gaussian_max_contribution
        assert float(mc.max()) > 0
        outputs[rtype + "_max_contribution"] = mc
        outputs[rtype + "_colours"] = R.get_gaussian_colours()
        if rtype == "cuda":
            outputs["cuda_total_contribution"] = R.gaussian_total_contribution
            outputs["cuda_min_surface_distance"] = R.gaussian_min_surface_distance
    G.colours = G.colours * 255
    idx = G.fused_cull(max_contribution=mc, visibility_threshold=0.01)
    G.validate_covariances()
    pts, cols, nrm = g2p.generate_pointcloud(G, 20000, quiet=True)
    outputs.update(cull_index=idx, points=pts, point_colours=cols, point_normals=nrm)
    return outputs, (pts.shape[0], idx.shape[0])


target_main("SANITIZER_TARGET_OK", run, large_bytes=256 << 20)
