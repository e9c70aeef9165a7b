"""Small hole filling, meant to be executed under compute-sanitizer (tests/test_holes_gpu.py): memcheck and racecheck
over the edge sort, the boundary degrees, the union-find, the plan scans and the loop walks.

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
    n = 40  # a 40 x 40 grid with single and 2 x 2 holes, a pinched pair and 30 vertices no face uses
    skip = {(i, j) for i in range(1, n - 1, 4) for j in range(1, n - 1, 4)}
    skip |= {(i + a, j + b) for i in (3, 19) for j in (3, 27) for a in (0, 1) for b in (0, 1)} | {(10, 14), (11, 15)}
    f = []
    for j in range(n):
        for i in range(n):
            if (i, j) not in skip:
                a, b, c, d = j * (n + 1) + i, j * (n + 1) + i + 1, (j + 1) * (n + 1) + i + 1, (j + 1) * (n + 1) + i
                f += [[a, b, c], [a, c, d]]
    m = (n + 1) ** 2 + 30
    f = rng.permutation(m)[np.array(f)].astype(np.int32)
    v = rng.normal(size=(m, 3))
    cols = rng.integers(0, 256, (m, 3)).astype(np.uint8)
    dens = rng.uniform(0.5, 2.0, m)
    (p, ff, c, d), dbg = mesh.fill_holes(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev),
                                         torch.from_numpy(cols).to(dev), torch.from_numpy(dens).to(dev),
                                         max_hole_edges=8, return_debug=True)
    outputs = {"vpos": p, "faces": ff, "colours": c, "densities": d, "labels": dbg["labels"], "succ": dbg["succ"],
               "lengths": dbg["lengths"], "filled": dbg["filled"]}
    return outputs, (p.shape[0], ff.shape[0])


target_main("HOLES_TARGET_OK", run)
