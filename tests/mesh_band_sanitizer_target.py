"""Tiny Poisson mesh with two narrow-band levels, meant to be executed under compute-sanitizer
(tests/test_mesh_band_gpu.py): memcheck and racecheck over the brick map, band splat, ghosts, conjugate gradients,
band iso-value, extraction and gather.

Without the sanitizer (the test runs it directly when the tool does not support the GPU):
  G2PC_TARGET_POISON=<byte>   every block PyTorch's caching allocator hands out afterwards starts filled with <byte>
  G2PC_TARGET_OUT=<file.npz>  every output of the run is saved there, for bit-for-bit comparison between runs"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from g2pc import mesh  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    rng = np.random.default_rng(3)
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = np.concatenate([0.2 * d, 0.05 * d[:300] + 1.0]).astype(np.float32)  # a far cluster keeps the band narrow
    d = np.concatenate([d, d[:300]])
    cols = rng.uniform(0, 255, p.shape).astype(np.float32)
    m, dbg = mesh.poisson_mesh(torch.from_numpy(p).to(dev), torch.from_numpy(d.astype(np.float32)).to(dev),
                               torch.from_numpy(cols).to(dev), depth=5, band_depth=7, laplacian_iters=2,
                               return_debug=True)
    outputs = dict(m._asdict(), **{k: dbg[k] for k in ("chi", "iso", "keep", "threshold")})
    return outputs, (m.vertices.shape[0], m.faces.shape[0], [lv["iterations"] for lv in dbg["levels"]])


target_main("MESH_BAND_TARGET_OK", run)
