"""Small component filter, meant to be executed under compute-sanitizer (tests/test_components_gpu.py): memcheck and
racecheck over the union-find, the size count, the ranking sort, the selection and the compaction.

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

from g2pc import mesh  # noqa: E402
from sanitizer_harness import target_main  # noqa: E402


def run():
    dev = "cuda:0"
    rng = np.random.default_rng(3)
    lengths = rng.integers(1, 60, 300)
    f = [off + np.stack([np.arange(L), np.arange(L) + 1, np.arange(L) + 2], 1)
         for off, L in zip(np.r_[0, np.cumsum(lengths + 2)[:-1]], lengths)]
    m = int((lengths + 2).sum()) + 50  # 50 vertices no face uses
    f = rng.permutation(m)[np.concatenate(f)].astype(np.int32)
    v = rng.normal(size=(m, 3))
    cols = rng.integers(0, 256, (m, 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, m)
    (p, ff, c, d), dbg = mesh.remove_components(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev),
                                                torch.from_numpy(cols).to(dev), torch.from_numpy(dens).to(dev),
                                                min_triangles=5, keep_largest=100, return_debug=True)
    outputs = {"vpos": p, "faces": ff, "colours": c, "densities": d, "labels": dbg["labels"], "sizes": dbg["sizes"],
               "keep": dbg["keep"]}
    return outputs, (p.shape[0], ff.shape[0])


target_main("COMPONENTS_TARGET_OK", run)
