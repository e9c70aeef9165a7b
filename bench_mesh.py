"""Time the Poisson mesher (g2pc/mesh.py) on a C3-sized point cloud at depths 8, 9 and 10.

    python bench_mesh.py [--runs 5] [--depths 8,9,10] [--points 10000000]

The cloud is sampled from the synthetic 3 M-Gaussian scene the way C3 samples its cloud, with the Gaussians' own colours
(--no_render_colours).  The sampler's normals have an arbitrary sign, so they are flipped to point away from the origin
(the scene's centre): the surface is then one shell seen from outside.  Every depth is warmed up once, then timed
`--runs` times with CUDA events around the whole mesh and around each phase (clean, splat, solve, extract, gather+trim,
smooth, normals); medians and the spread are printed with the multigrid cycles, the final residual ratio, the peak of
torch.cuda.max_memory_allocated, the vertex and face counts, and the card's name and power limit read in the same run.
There is no CPU comparator: Open3D, whose Poisson reconstruction the reference calls, is not installed.  One JSON line on
stdout; nothing is written to disk.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "3dgs-to-pc_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

DEV = "cuda:0"
PHASES = ["clean", "splat", "solve", "extract", "gather_trim", "smooth", "normals"]


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
    nrm = pc.normals.to(torch.float32)
    flip = (nrm * pc.points).sum(1, keepdim=True) < 0
    return pc.points.contiguous(), torch.where(flip, -nrm, nrm).contiguous(), pc.colours


def time_depth(points, normals, colours, depth, runs):
    from g2pc import mesh
    m, dbg = mesh.poisson_mesh(points, normals, colours, depth=depth, return_debug=True)  # warm-up, solver report
    nv, nf, cycles, ratio = int(m.vertices.shape[0]), int(m.faces.shape[0]), dbg["cycles"], dbg["ratio"]
    del m, dbg
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    total, phases = [], {p: [] for p in PHASES}
    for _ in range(runs):
        timings = {}
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        m = mesh.poisson_mesh(points, normals, colours, depth=depth, timings=timings)
        b.record()
        torch.cuda.synchronize()
        total.append(a.elapsed_time(b))
        for p in PHASES:
            phases[p].append(sum(s.elapsed_time(e) for s, e in timings[p]))
        assert (int(m.vertices.shape[0]), int(m.faces.shape[0])) == (nv, nf)
        del m
    med = lambda v: round(float(np.median(v)), 1)
    return {"depth": depth, "points": int(points.shape[0]), "median_ms": med(total), "min_ms": round(min(total), 1),
            "max_ms": round(max(total), 1), "runs": runs, "phase_median_ms": {p: med(v) for p, v in phases.items()},
            "cycles": cycles, "residual_ratio": float(f"{ratio:.3g}"), "vertices": nv, "faces": nf,
            "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "peak_above_inputs_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--depths", default="8,9,10")
    ap.add_argument("--points", type=int, default=10_000_000)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh.py needs a CUDA device")
    from g2pc import build
    build.build()
    name, power = card()
    res = {"metric": "Poisson mesh (clean + splat + multigrid + marching tetrahedra + trim + 10 smoothing steps)",
           "card": name, "power_limit": power, "cpu": "none: Open3D is not installed, no CPU comparator", "gpu": []}
    points, normals, colours = sampled_cloud(args.points, seed=1236)
    for d in [int(s) for s in args.depths.split(",")]:
        r = time_depth(points, normals, colours, d, args.runs)
        res["gpu"].append(r)
        print(f"[mesh] {r}", file=sys.stderr)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
