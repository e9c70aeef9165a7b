"""Time gauss_to_mesh.py --mesh_method tsdf's device part on the C3-like scene, phase by phase, next to the Poisson path.

    python bench_tsdf.py [--runs 3] [--gaussians 3000000] [--cameras 200] [--depths 9 10] [--poisson_depth 10]

The scene is the synthetic 3 M-Gaussian scene of the other benchmarks, rendered from 200 cameras at 1280 x 720.  For
each tsdf depth what is timed is convert_gaussians_to_pc (mesh_method="tsdf": colour stage, culls, the 10 M-point
cloud) plus g2pc.tsdf.fuse_mesh, from the scene on the device to the mesh on the device, without the loaders and the
PLY writers.  Phases of fuse_mesh: frame (outlier removal of the means, grid frame), fusion render (every camera's
projection, sort, lists and fusion blend), integration (the g2pc_tsdf_integrate launches, CUDA events around each),
extract, gather (gather and compaction), smooth and normals.  Events are put around every entry point of the fusion
phase to split it, which adds a little host time to it.  Then bench_gauss_mesh.py's Poisson path on the same scene at
--poisson_depth.  One warm-up run per configuration, then `--runs` runs between device synchronisations; medians and
ranges, the peak of max_memory_allocated and the mesh sizes are printed with the card's name and power limit, read in
the same run.  One JSON line on stdout; nothing is written to disk.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_clean import DEV, card, spread, timed_runs

TSDF_PHASES = ("colour", "cull", "sample", "frame", "fusion", "g2pc_tsdf_integrate", "extract", "gather", "smooth",
               "normals")
POISSON_PHASES = ("colour", "cull", "sample", "surface_select", "face_cameras", "surface_sample", "clean", "splat",
                  "solve", "extract", "gather_trim", "smooth", "normals")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--depths", type=int, nargs="+", default=[9, 10])
    ap.add_argument("--poisson_depth", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_tsdf.py needs a CUDA device")
    import gauss_to_pc as g2p
    from g2pc import build, capi, mesh, sampler, synth, tsdf
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

    def convert(timings, method):
        sampler.reset_call_counter(0)
        return g2p.convert_gaussians_to_pc(sc["xyz"], sc["scales"], sc["rots"], sc["colours"].clone() * 255,
                                           sc["opacities"], sc["shs"], transforms, intrinsics, None, settings,
                                           timings=timings, mesh_method=method)

    def run_tsdf(depth):
        def call(timings):
            pc, scene = convert(timings, "tsdf")
            capi.TIMING = timings
            try:
                m = tsdf.fuse_mesh(scene.xyz, scene.opacities, scene.covariances, scene.cameras, colours=scene.colours,
                                   shs=scene.shs, depth=depth, laplacian_iters=10, timings=timings)
            finally:
                capi.TIMING = None
            sizes[f"tsdf{depth}"] = dict(gaussians_rendered=int(scene.xyz.shape[0]), vertices=int(m.vertices.shape[0]),
                                         triangles=int(m.faces.shape[0]))
        return call

    def run_poisson(timings):
        pc, surf = convert(timings, "poisson")
        m = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=args.poisson_depth, laplacian_iters=10,
                              std_ratio=3.0, timings=timings)
        sizes["poisson"] = dict(vertices=int(m.vertices.shape[0]), triangles=int(m.faces.shape[0]))

    res = {"metric": "gauss_to_mesh device part (colour stage .. mesh), C3-like scene", "card": name,
           "power_limit": power, "gaussians": args.gaussians, "cameras": args.cameras, "resolution": "1280x720",
           "num_points": args.points, "runs": args.runs}
    for depth in args.depths:
        call = run_tsdf(depth)
        call({})  # warm-up
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        total, per_phase = timed_runs(call, TSDF_PHASES, args.runs)
        med = {p: round(float(np.median(v)), 2) for p, v in per_phase.items()}
        integ = med.pop("g2pc_tsdf_integrate")
        med["fusion_render"] = round(med.pop("fusion") - integ, 2)
        med["integration"] = integ
        med["integration_per_camera"] = round(integ / args.cameras, 3)
        res[f"tsdf_depth{depth}"] = {"total": spread(total, 1), "phases_median_ms": med,
                                     "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
                                     **sizes[f"tsdf{depth}"]}
        torch.cuda.empty_cache()
    run_poisson({})  # warm-up
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    total, per_phase = timed_runs(run_poisson, POISSON_PHASES, args.runs)
    res[f"poisson_depth{args.poisson_depth}"] = {
        "total": spread(total, 1), "phases_median_ms": {p: round(float(np.median(v)), 2) for p, v in per_phase.items()},
        "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2), **sizes["poisson"]}
    print(f"[tsdf] {res}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
