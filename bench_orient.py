"""Time the normal orientation (g2pc.orient.orient_normals, k = 10) on a C3-sized point cloud.

    python bench_orient.py [--runs 5] [--points 10000000]

The cloud is sampled from the synthetic 3 M-Gaussian scene the way C3 samples its own, with the Gaussians' own colours
(--no_render_colours), and its normals are the sampler's (each takes its sign from its Gaussian's rotation).  One
warm-up, then `--runs` timed runs with CUDA events around the whole call (its host reads included) and around each
phase (prepare, k-NN, edges, Borůvka rounds, finish); the median and the spread (min..max) are printed with the number
of rounds, the peak memory above the inputs and the card's name and power limit, read in the same run.  One JSON line on
stdout; nothing is written to disk.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from bench_clean import DEV, card, spread, timed_runs  # noqa: E402

PHASES = ("prepare", "knn", "edges", "rounds", "finish")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--points", type=int, default=10_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_orient.py needs a CUDA device")
    from g2pc import build, orient, synth
    build.build()
    name, power = card()
    pc = synth.sampled_cloud(3_000_000, args.points, 1236, DEV)
    pts, nrm = pc.points, pc.normals
    del pc
    torch.cuda.empty_cache()
    stats = orient.orient_normals(pts, nrm, k=10)[1]  # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    total, phases = timed_runs(lambda timings: orient.orient_normals(pts, nrm, k=10, timings=timings), PHASES, args.runs)
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    res = {"metric": "normal orientation (k = 10), whole call", "card": name, "power_limit": power,
           "points": int(pts.shape[0]), "runs": args.runs, **spread(total, 2),
           "phase_median_ms": {p: round(float(np.median(v)), 2) for p, v in phases.items()},
           "rounds": stats.rounds, "components": stats.components, "flipped": stats.flipped, "skipped": stats.skipped,
           "peak_gib_above_inputs": round(peak, 2)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
