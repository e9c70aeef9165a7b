"""Small decimation, meant to be executed under compute-sanitizer (tests/test_decimate_gpu.py): memcheck and racecheck
over the preparation, the selection, the collapses and the compaction of every round.

Without the sanitizer (the test runs it directly when the tool does not support the GPU):
  G2PC_TARGET_POISON=<byte>   every block PyTorch's caching allocator hands out afterwards starts filled with <byte>
  G2PC_TARGET_OUT=<file.npz>  every output of the run is saved there, for bit-for-bit comparison between runs"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import f64ref_decimate as fd  # noqa: E402
from g2pc import mesh  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    v, f = fd.icosphere(3)
    g, gf = fd.grid(16, 0.4)
    v, f = np.r_[v, g], np.r_[f, gf + v.shape[0]]  # a closed part and an open one
    rng = np.random.default_rng(3)
    cols = rng.integers(0, 256, (v.shape[0], 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, v.shape[0])
    (p, ff, c, d), dbg = mesh.decimate(torch.from_numpy(v).to(dev), torch.from_numpy(f.astype(np.int32)).to(dev),
                                       f.shape[0] // 4, torch.from_numpy(cols).to(dev), torch.from_numpy(dens).to(dev),
                                       return_debug=True)
    outputs = {"vpos": p, "faces": ff, "colours": c, "densities": d}
    return outputs, (p.shape[0], ff.shape[0], len(dbg["rounds"]))


target_main("DECIMATE_TARGET_OK", run)
