"""Tiny gauss_to_mesh.py run, meant to be executed under compute-sanitizer (tests/test_gauss_mesh_gpu.py): memcheck and
racecheck over the colour stage with first_frame and surface distances, the culls, both samplings, g2pc_face_cameras and
the mesher.

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
import gauss_to_pc as g2p  # noqa: E402
from g2pc import sampler, synth  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402
from test_io_cpu import write_gaussian_ply, write_transforms_json  # noqa: E402


def run():
    with tempfile.TemporaryDirectory() as tmp:
        ply, tj = os.path.join(tmp, "scene.ply"), os.path.join(tmp, "transforms.json")
        write_gaussian_ply(ply, synth.make_scene(3000, seed=8))
        write_transforms_json(tj, *synth.make_cameras(3))
        sampler.reset_call_counter(0)
        surf, m = gauss_to_mesh.main(["--input_path", ply, "--transform_path", tj, "--output_path",
                                      os.path.join(tmp, "pc.ply"), "--mesh_output_path", os.path.join(tmp, "mesh.ply"),
                                      "--num_points", "30000", "--colour_quality", "tiny", "--poisson_depth", "5",
                                      "--quiet"])
        cloud = np.frombuffer(open(os.path.join(tmp, "pc.ply"), "rb").read(), np.uint8)
    st = g2p.LAST_SURFACE_STATS
    return (dict(cloud=torch.from_numpy(cloud.copy()), points=surf.points, normals=surf.normals, vertices=m.vertices,
                 faces=m.faces, first_frame=st["first_frame"], ids=st["ids"],
                 face_cameras=torch.tensor(list(st["face_cameras"]))),
            (m.vertices.shape[0], m.faces.shape[0], tuple(st["face_cameras"])))


target_main("GAUSS_MESH_TARGET_OK", run)
