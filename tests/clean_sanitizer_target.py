"""Tiny statistical-outlier clean, meant to be executed under compute-sanitizer (tests/test_clean_gpu.py): memcheck and
racecheck over the k-NN index build, the query kernel, the statistics and the compaction.

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

from g2pc import outliers  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    rng = np.random.default_rng(3)
    p = np.concatenate([rng.random((3000, 3)), np.repeat(rng.random((1, 3)), 25, 0), [[40.0, 40.0, 40.0]],
                        0.5 + 1e-6 * rng.random((500, 3))]).astype(np.float32)
    xyz = torch.from_numpy(p).to(dev)
    cols = torch.from_numpy(rng.uniform(-10, 300, p.shape).astype(np.float32)).to(dev)
    nrm = torch.from_numpy(rng.normal(size=p.shape).astype(np.float32)).to(dev)
    pts, c, n, dbg = outliers.remove_statistical_outliers(xyz, cols, nrm, 20, 3.0, return_debug=True)
    return dict(points=pts, colours=c, normals=n, **dbg), (pts.shape[0],)


target_main("CLEAN_TARGET_OK", run)
