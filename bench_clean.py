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


def sampled_cloud(num_points, seed):
    import gauss_to_pc as g2p
    from g2pc import sampler, synth
    sc = {k: v.to(DEV) for k, v in synth.make_scene(3_000_000, seed=seed).items()}
    st = g2p.GaussPointCloudSettings(
        renderer_type="python", num_points=num_points, prioritise_visible_gaussians=True, mahalanobis_distance_std=2.0,
        camera_skip_rate=0, render_colours=False, min_opacity=0.0, bounding_box_min=None, bounding_box_max=None,
        calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True, colour_resolution=None,
        max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05, surface_distance_std=None,
        generate_mesh=False, quiet=True, device=DEV)
    sampler.reset_call_counter(0)
    pc, _ = g2p.convert_gaussians_to_pc(sc["xyz"], sc["scales"], sc["rots"], sc["colours"].clone() * 255,
                                        sc["opacities"], sc["shs"], None, None, None, st)
    del sc
    return pc


def time_clean(pc, runs):
    from g2pc import outliers
    clean = lambda: outliers.remove_statistical_outliers(pc.points, pc.colours, pc.normals, 20, 10.0)
    out = clean()  # warm-up
    kept = int(out[0].shape[0])
    del out
    ms = []
    for _ in range(runs):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = clean()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
        del out
    # the k-NN kernels alone (index build + queries), same warm state
    from g2pc import outliers as o
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    knn = []
    for _ in range(runs):
        torch.cuda.synchronize()
        a.record()
        o.mean_distances(pc.points, 20)
        b.record()
        torch.cuda.synchronize()
        knn.append(a.elapsed_time(b))
    return {"points": int(pc.points.shape[0]), "kept": kept, "median_ms": round(float(np.median(ms)), 2),
            "min_ms": round(min(ms), 2), "max_ms": round(max(ms), 2), "runs": runs,
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
    from g2pc import build
    build.build()
    name, power = card()
    res = {"metric": "statistical outlier removal (k = 20, std_ratio = 10), whole clean", "card": name,
           "power_limit": power, "gpu": []}
    cpu_done = False
    for n in [int(s) for s in args.sizes.split(",")]:
        pc = sampled_cloud(n, seed=1234 + (2 if n <= 10_000_000 else 3))
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
