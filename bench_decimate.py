"""Time g2pc.mesh.decimate on the depth-10 scene mesh, to 10 % and to 1 % of its triangles.

    python bench_decimate.py [--runs 3] [--gaussians 3000000] [--cameras 200] [--points 10000000] [--depth 10]
                             [--fractions 0.1,0.01]

The mesh is made the way bench_gauss_mesh.py makes it: the synthetic 3 M-Gaussian scene, 200 cameras at 1280 x 720,
10 M points, the surface cloud with its normals turned toward their cameras, meshed at depth 10.  Its float64 vertices,
faces, colours and densities are then decimated to each fraction of its triangle count: one warm-up run, then `--runs`
runs, each between two device synchronisations, timed with CUDA events around the whole call and around every entry
point (prepare, select, apply, finish, summed over the rounds).  Printed per fraction: the median and range, the rounds,
the fraction of the surviving vertices collapsed in each round, and the peak of max_memory_allocated; with the card's
name and power limit, read in the same run.  One JSON line on stdout; nothing is written to disk.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_clean import DEV, card, spread

ENTRY_POINTS = ("g2pc_mesh_decimate_prepare", "g2pc_mesh_decimate_select", "g2pc_mesh_decimate_apply",
                "g2pc_mesh_decimate_finish")


def scene_mesh(args):
    import gauss_to_pc as g2p
    from g2pc import mesh, sampler, synth
    sc = {k: v.to(DEV) for k, v in synth.make_scene(args.gaussians, seed=1234).items()}
    cams, intr = synth.make_cameras(args.cameras)
    settings = g2p.GaussPointCloudSettings(
        renderer_type="cuda", num_points=args.points, prioritise_visible_gaussians=True, mahalanobis_distance_std=2.0,
        camera_skip_rate=0, render_colours=True, min_opacity=0.0, bounding_box_min=None, bounding_box_max=None,
        calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True, colour_resolution=1280,
        max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05, surface_distance_std=None,
        generate_mesh=True, quiet=True, device=DEV)
    sampler.reset_call_counter(0)
    _, surf = g2p.convert_gaussians_to_pc(sc["xyz"], sc["scales"], sc["rots"], sc["colours"].clone() * 255,
                                          sc["opacities"], sc["shs"], {f"c{i}": c for i, c in enumerate(cams)},
                                          {f"c{i}": k for i, k in enumerate(intr)}, None, settings)
    del sc
    m, dbg = mesh.poisson_mesh(surf.points, surf.normals, surf.colours, depth=args.depth, laplacian_iters=10,
                               std_ratio=3.0, return_debug=True)
    return dbg["vpos_smoothed"], m.faces, m.colours, m.densities


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--fractions", default="0.1,0.01")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_decimate.py needs a CUDA device")
    from g2pc import build, capi, mesh
    build.build()
    name, power = card()
    vpos, faces, colours, dens = scene_mesh(args)
    torch.cuda.empty_cache()
    m, t = int(vpos.shape[0]), int(faces.shape[0])
    res = {"metric": "decimate the depth-10 scene mesh", "card": name, "power_limit": power, "depth": args.depth,
           "vertices": m, "triangles": t, "runs": args.runs, "fractions": {}}
    for frac in (float(x) for x in args.fractions.split(",")):
        target = max(1, int(frac * t))
        stats = {}
        mesh.decimate(vpos, faces, target, colours, dens, stats=stats)  # warm-up
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        total, per_entry, out_t = [], {e: [] for e in ENTRY_POINTS}, 0
        for _ in range(args.runs):
            capi.TIMING = {}
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = mesh.decimate(vpos, faces, target, colours, dens, stats=stats)
            b.record()
            torch.cuda.synchronize()
            total.append(a.elapsed_time(b))
            for e in ENTRY_POINTS:
                per_entry[e].append(sum(x.elapsed_time(y) for x, y in capi.TIMING.get(e, [])))
            out_t = int(out[1].shape[0])
            del out
        capi.TIMING = None
        peak = torch.cuda.max_memory_allocated()
        alive, per_round = m, []
        for k in stats["collapses"]:
            per_round.append(round(k / alive, 4))
            alive -= k
        res["fractions"][str(frac)] = {
            "target": target, "triangles_out": out_t, "reached": stats["reached"], "rounds": stats["rounds"],
            "total": spread(total, 1), "entry_points_median_ms": {e[19:]: round(float(np.median(v)), 2)
                                                                  for e, v in per_entry.items()},
            "collapsed_fraction_per_round": per_round,
            "peak_allocated_gib": round(peak / 2 ** 30, 2), "mesh_allocated_gib": round(base / 2 ** 30, 2)}
    print(f"[decimate] {res}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
