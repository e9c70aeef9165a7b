"""Time gauss_to_mesh.py's device part on a C4-like scene, phase by phase.

    python bench_gauss_mesh.py [--runs 5] [--gaussians 3000000] [--cameras 200] [--points 10000000] [--depth 10]

The scene is the synthetic 3 M-Gaussian scene of the other benchmarks, rendered from 200 cameras at 1280 x 720 with
surface distances and the first camera of every maximum, sampled into 10 M points, then the surface cloud of the
Gaussians on a predicted surface, its normals turned toward their cameras, meshed at depth 10.  What is timed is
convert_gaussians_to_pc (with generate_mesh) plus g2pc.mesh.poisson_mesh: from the scene on the device to the mesh on the
device, without the loaders and the PLY writers.  One warm-up run, then `--runs` runs, each between two device
synchronisations with CUDA events around the whole and around every phase; the median and the range are printed with
the card's name and power limit, read in the same run, and the peak of max_memory_allocated.  One JSON line on stdout;
nothing is written to disk.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_clean import DEV, card, spread, timed_runs

PHASES = ("colour", "cull", "sample", "surface_select", "face_cameras", "surface_sample", "clean", "splat", "solve",
          "extract", "gather_trim", "smooth", "normals")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--depth", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gauss_mesh.py needs a CUDA device")
    import gauss_to_pc as g2p
    from g2pc import build, mesh, sampler, synth
    build.build()
    name, power = card()
    sc = {k: v.to(DEV) for k, v in synth.make_scene(args.gaussians, seed=1234).items()}
    cams, intr = synth.make_cameras(args.cameras)  # 1920 x 1080 poses, rendered 1280 px wide (--colour_quality high)
    transforms = {f"c{i}": c for i, c in enumerate(cams)}
    intrinsics = {f"c{i}": k for i, k in enumerate(intr)}
    settings = g2p.GaussPointCloudSettings(
        renderer_type="cuda", num_points=args.points, prioritise_visible_gaussians=True, mahalanobis_distance_std=2.0,
        camera_skip_rate=0, render_colours=True, min_opacity=0.0, bounding_box_min=None, bounding_box_max=None,
        calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True, colour_resolution=1280,
        max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05, surface_distance_std=None,
        generate_mesh=True, quiet=True, device=DEV)
    sizes = {}

    def call(timings):
        sampler.reset_call_counter(0)
        pc, surf = g2p.convert_gaussians_to_pc(sc["xyz"], sc["scales"], sc["rots"], sc["colours"].clone() * 255,
                                               sc["opacities"], sc["shs"], transforms, intrinsics, None, settings,
                                               timings=timings)
        m = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=args.depth, laplacian_iters=10,
                              std_ratio=3.0, timings=timings)
        sizes.update(points=int(pc.points.shape[0]), surface_gaussians=int(g2p.LAST_SURFACE_STATS["ids"].shape[0]),
                     surface_points=int(surf.points.shape[0]),
                     face_cameras=g2p.LAST_SURFACE_STATS["face_cameras"]._asdict(),
                     vertices=int(m.vertices.shape[0]), triangles=int(m.faces.shape[0]))

    call({})  # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    total, per_phase = timed_runs(call, PHASES, args.runs)
    peak = torch.cuda.max_memory_allocated()
    res = {"metric": "gauss_to_mesh device part (colour stage .. mesh), C4-like scene", "card": name,
           "power_limit": power, "gaussians": args.gaussians, "cameras": args.cameras, "resolution": "1280x720",
           "num_points": args.points, "depth": args.depth, "runs": args.runs, "total": spread(total, 1),
           "phases_median_ms": {p: round(float(np.median(v)), 2) for p, v in per_phase.items()},
           "peak_allocated_gib": round(peak / 2 ** 30, 2), "scene_allocated_gib": round(base / 2 ** 30, 2), **sizes}
    print(f"[gauss_mesh] {res}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
