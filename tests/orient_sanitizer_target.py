"""Tiny normal orientation, meant to be executed under compute-sanitizer (tests/test_orient_gpu.py): memcheck and
racecheck over the usable-point compaction, the k-NN id lists, the edge build, every Borůvka round and the finish.

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

from g2pc import orient  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    rng = np.random.default_rng(3)
    d = rng.normal(size=(3000, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    p = np.concatenate([d, np.repeat(rng.random((1, 3)), 25, 0), [[40.0, 40.0, 40.0]],
                        0.5 + 1e-6 * rng.random((500, 3))]).astype(np.float32)
    n = rng.normal(size=p.shape).astype(np.float32)
    n[:3000] = d * np.where(rng.random(3000) < 0.5, -1.0, 1.0)[:, None]
    n[5] = 0.0
    n[6, 1] = np.nan
    out, st, dbg = orient.orient_normals(torch.from_numpy(p).to(dev), torch.from_numpy(n).to(dev), return_debug=True)
    return dict(normals=out, stats=torch.tensor(list(st)), **dbg), (st.components, st.flipped)


target_main("ORIENT_TARGET_OK", run)
