"""Time g2pc.mesh.fill_holes on the depth-10 scene mesh, and its effect on a decimation to 1 %.

    python bench_holes.py [--runs 5] [--gaussians 3000000] [--cameras 200] [--points 10000000] [--depth 10]
                          [--fraction 0.01] [--skip_decimate]

The mesh is bench_decimate.scene_mesh's: the synthetic 3 M-Gaussian scene, 200 cameras at 1280 x 720, 10 M points, the
surface cloud meshed at depth 10, smoothed.  Its float64 vertices, faces, colours and densities are filled with
max_hole_edges 16, 64 and 256: one warm-up run each, then `--runs` runs, each between two device synchronisations, timed
with CUDA events around the whole call and around every entry point (find, plan, fill).  Printed per setting: the median
and range, the counts of the stats, the peak of max_memory_allocated and the algorithmic bytes from the shapes.  Then
the mesh is decimated to `--fraction` of its triangles once as it is and once after filling at max_hole_edges 64: the
rounds, the time and the triangles reached.  With the card's name and power limit, read in the same run.  One JSON line
on stdout; nothing is written to disk.
"""
import argparse
import json
import sys
import time

import numpy as np
import torch

from bench_clean import card, spread
from bench_decimate import scene_mesh

ENTRY_POINTS = ("g2pc_mesh_holes_find", "g2pc_mesh_holes_plan", "g2pc_mesh_holes_fill")
SETTINGS = (16, 64, 256)


def algorithmic_bytes(m, t, M, T, boundary):
    """The least DRAM traffic of one call, from the shapes.  The faces (12 B per triangle) are read to build the keys
    and the 3 t keys and payloads (12 B each) are written; the radix sort reads and writes keys and payloads once per
    pass (8 passes at most); the two passes over the sorted keys read them (8 B) and the payload (4 B), and gather the
    two ends of each half-edge (8 B).  Per vertex the degrees, succ, labels, lengths and flags are written and read a few
    times (about 64 B); the fill copies the input mesh (35 B per vertex, 12 B per triangle) and writes the added part."""
    e = 3 * t
    sort = 8 * 2 * 12 * e
    passes = 12 * t + 12 * e + sort + 2 * (12 * e) + 2 * 8 * boundary
    return {"sort_bytes": sort, "edge_passes_bytes": passes - sort, "vertex_bytes": 64 * m,
            "total_bytes": passes + 64 * m + 2 * (35 * m + 12 * t) + 35 * (M - m) + 12 * (T - t)}


def _decimate(vpos, faces, colours, dens, target):
    from g2pc import mesh
    stats = {}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = mesh.decimate(vpos, faces, target, colours, dens, stats=stats)
    torch.cuda.synchronize()
    return {"seconds": round(time.perf_counter() - t0, 2), "rounds": stats["rounds"], "reached": stats["reached"],
            "triangles": int(out[1].shape[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--fraction", type=float, default=0.01)
    ap.add_argument("--skip_decimate", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_holes.py needs a CUDA device")
    from g2pc import build, capi, mesh
    build.build()
    name, power = card()
    vpos, faces, colours, dens = scene_mesh(args)
    torch.cuda.empty_cache()
    m, t = int(vpos.shape[0]), int(faces.shape[0])
    res = {"metric": "fill small holes of the depth-10 scene mesh", "card": name, "power_limit": power,
           "depth": args.depth, "vertices": m, "triangles": t, "runs": args.runs, "settings": {}}
    for H in SETTINGS:
        stats = {}
        mesh.fill_holes(vpos, faces, colours, dens, H)  # warm-up
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        total, per_entry, out = [], {e: [] for e in ENTRY_POINTS}, None
        for _ in range(args.runs):
            out = None
            capi.TIMING = {}
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = mesh.fill_holes(vpos, faces, colours, dens, H, stats=stats)
            b.record()
            torch.cuda.synchronize()
            total.append(a.elapsed_time(b))
            for e in ENTRY_POINTS:
                per_entry[e].append(sum(x.elapsed_time(y) for x, y in capi.TIMING.get(e, [])))
        capi.TIMING = None
        peak = torch.cuda.max_memory_allocated()
        M, T = int(out[0].shape[0]), int(out[1].shape[0])
        del out
        ab = algorithmic_bytes(m, t, M, T, stats["boundary_edges"])
        med = float(np.median(total))
        res["settings"][f"max_hole_edges {H}"] = {
            "total": spread(total, 2), "entry_points_median_ms": {e[16:]: round(float(np.median(v)), 2)
                                                                  for e, v in per_entry.items()},
            **stats, "algorithmic_bytes": ab, "algorithmic_gb_per_s": round(ab["total_bytes"] / (med * 1e-3) / 1e9, 1),
            "peak_allocated_gib": round(peak / 2 ** 30, 2), "mesh_allocated_gib": round(base / 2 ** 30, 2)}
    if not args.skip_decimate:
        target = max(1, int(t * args.fraction))
        res["decimate"] = {"target": target, "plain": _decimate(vpos, faces, colours, dens, target)}
        vf, ff, cf, df = mesh.fill_holes(vpos, faces, colours, dens, 64)
        torch.cuda.empty_cache()
        res["decimate"]["filled_64"] = _decimate(vf, ff, cf, df, target)
    print(f"[holes] {res}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
