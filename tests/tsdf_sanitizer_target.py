"""Tiny gauss_to_mesh.py --mesh_method tsdf run, meant to be executed under compute-sanitizer (tests/test_tsdf_gpu.py):
memcheck and racecheck over the colour stage, the culls, the sampling, the fusion blend, the integration, the
extraction, the gather and compaction, smoothing and normals.

Without the sanitizer (the test runs it directly when the tool does not support the GPU):
  G2PC_TARGET_POISON=<byte>   every block PyTorch's caching allocator hands out afterwards starts filled with <byte>
  G2PC_TARGET_OUT=<file.npz>  every output of the run is saved there, for bit-for-bit comparison between runs"""
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import gauss_to_mesh  # noqa: E402
from g2pc import sampler, synth  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402
from test_io_cpu import write_gaussian_ply, write_transforms_json  # noqa: E402


def run():
    with tempfile.TemporaryDirectory() as tmp:
        ply, tj = os.path.join(tmp, "scene.ply"), os.path.join(tmp, "transforms.json")
        write_gaussian_ply(ply, synth.make_scene(3000, seed=8))
        write_transforms_json(tj, *synth.make_cameras(3))
        sampler.reset_call_counter(0)
        _, m = gauss_to_mesh.main(["--input_path", ply, "--transform_path", tj, "--output_path",
                                   os.path.join(tmp, "pc.ply"), "--mesh_output_path", os.path.join(tmp, "mesh.ply"),
                                   "--num_points", "30000", "--colour_quality", "tiny", "--mesh_method", "tsdf",
                                   "--tsdf_depth", "5", "--quiet"])
        cloud = np.frombuffer(open(os.path.join(tmp, "pc.ply"), "rb").read(), np.uint8)
    return (dict(cloud=torch.from_numpy(cloud.copy()), vertices=m.vertices, faces=m.faces, colours=m.colours,
                 densities=m.densities),
            (m.vertices.shape[0], m.faces.shape[0]))


target_main("TSDF_TARGET_OK", run)
