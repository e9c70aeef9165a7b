"""Time the statistical outlier removal (--clean_pointcloud) on C3- and C4-sized point clouds.

    python bench_clean.py [--runs 5] [--sizes 10000000,50000000] [--no-cpu]

The clouds are sampled from the synthetic 3 M-Gaussian scene the way C3 / C4 sample theirs, with the Gaussians' own
colours (--no_render_colours): the colour stage does not move any point.  Every size is warmed up once, then timed
`--runs` times with CUDA events around the whole clean (k-NN, statistics, compaction, its one host read); the median
and the spread (min..max) are printed with the card's name and power limit, read in the same run.  The CPU comparator
is scipy's cKDTree (k = 20, every host core) on the 10 M cloud: tree build + query, then the same statistics in numpy.
It is NOT Open3D (not installed), only a CPU k-d tree doing the same search.  One JSON line on stdout; nothing is
written to disk.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

DEV = "cuda:0"


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # the number is still reported, marked as missing its power limit
        out = f"unknown ({type(e).__name__})"
    return name, out


def timed_runs(call, phases, runs):
    """`runs` calls of call(timings), each between two device synchronisations, with the peak-memory statistics reset
    first.  Returns the CUDA-event time of every whole call and, for each name in `phases`, the sum of the event pairs
    the call put under that name in `timings`, per run (ms)."""
    torch.cuda.reset_peak_memory_stats()
    total, per_phase = [], {p: [] for p in phases}
    for _ in range(runs):
        timings = {}
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        call(timings)
        b.record()
        torch.cuda.synchronize()
        total.append(a.elapsed_time(b))
        for p in phases:
            per_phase[p].append(sum(s.elapsed_time(e) for s, e in timings[p]))
    return total, per_phase


def spread(ms, digits):
    """Median and range of a list of times, rounded to `digits` decimals."""
    return {"median_ms": round(float(np.median(ms)), digits), "min_ms": round(min(ms), digits),
            "max_ms": round(max(ms), digits)}


def time_clean(pc, runs):
    from g2pc import outliers
    clean = lambda timings=None: outliers.remove_statistical_outliers(pc.points, pc.colours, pc.normals, 20, 10.0)
    kept = int(clean()[0].shape[0])  # warm-up
    ms, _ = timed_runs(clean, (), runs)
    # the k-NN kernels alone (index build + queries), same warm state
    knn, _ = timed_runs(lambda timings: outliers.mean_distances(pc.points, 20), (), runs)
    return {"points": int(pc.points.shape[0]), "kept": kept, **spread(ms, 2), "runs": runs,
            "knn_median_ms": round(float(np.median(knn)), 2)}


def cpu_ckdtree(points):
    from scipy.spatial import cKDTree
    p = points.cpu().numpy().astype(np.float64)
    t0 = time.perf_counter()
    tree = cKDTree(p)
    t1 = time.perf_counter()
    d, _ = tree.query(p, k=20, workers=-1)
    avg = np.sqrt(d * d).mean(axis=1)  # statistics as numpy (timing only)
    pos = avg > 0
    mean = avg[pos].sum() / avg.size
    std = np.sqrt(((avg[pos] - mean) ** 2).sum() / (avg.size - 1))
    keep = pos & (avg < mean + 10.0 * std)
    t2 = time.perf_counter()
    return {"impl": "scipy cKDTree (not Open3D)", "points": int(p.shape[0]), "host_cores": os.cpu_count(),
            "build_s": round(t1 - t0, 2), "query_and_stats_s": round(t2 - t1, 2), "total_s": round(t2 - t0, 2),
            "kept": int(keep.sum())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--sizes", default="10000000,50000000")
    ap.add_argument("--no-cpu", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clean.py needs a CUDA device")
    from g2pc import build, synth
    build.build()
    name, power = card()
    res = {"metric": "statistical outlier removal (k = 20, std_ratio = 10), whole clean", "card": name,
           "power_limit": power, "gpu": []}
    cpu_done = False
    for n in [int(s) for s in args.sizes.split(",")]:
        pc = synth.sampled_cloud(3_000_000, n, 1234 + (2 if n <= 10_000_000 else 3), DEV)
        r = time_clean(pc, args.runs)
        res["gpu"].append(r)
        print(f"[clean] {r}", file=sys.stderr)
        if not args.no_cpu and not cpu_done and n <= 10_000_000:
            res["cpu"] = cpu_ckdtree(pc.points)
            print(f"[cpu] {res['cpu']}", file=sys.stderr)
            cpu_done = True
        del pc
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
