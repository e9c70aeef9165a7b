"""Time g2pc.mesh.remove_components on the depth-10 scene mesh.

    python bench_components.py [--runs 5] [--gaussians 3000000] [--cameras 200] [--points 10000000] [--depth 10]

The mesh is bench_decimate.scene_mesh's: the synthetic 3 M-Gaussian scene, 200 cameras at 1280 x 720, 10 M points, the
surface cloud meshed at depth 10, smoothed.  Its float64 vertices, faces, colours and densities are filtered with
min_triangles 100, min_triangles 1000 and keep_largest 1: one warm-up run each, then `--runs` runs, each between two
device synchronisations, timed with CUDA events around the whole call and around every entry point (label, select,
compact).  Printed per setting: the median and range, the components found and kept, the triangles removed and the peak
of max_memory_allocated; with the card's name and power limit, read in the same run, and the algorithmic bytes of the
filter computed from the shapes.  One JSON line on stdout; nothing is written to disk.
"""
import argparse
import json
import sys

import numpy as np
import torch

from bench_clean import card, spread
from bench_decimate import scene_mesh

ENTRY_POINTS = ("g2pc_mesh_components_label", "g2pc_mesh_components_select", "g2pc_mesh_components_compact")
SETTINGS = (("min_triangles 100", 100, None), ("min_triangles 1000", 1000, None), ("keep_largest 1", None, 1))


def algorithmic_bytes(m, t, mk, tk):
    """The least DRAM traffic of one call, from the shapes.  Faces (12 B per triangle) are read by four passes: the
    unions, the size count, the triangle flags and the face compaction.  Per vertex, the parent / label array is written
    once, read and written by the compression, and read with the sizes by the component count and the keep pass
    (4 + 8 + 8 + 8 B); the keep pass writes a byte and a flag (5 B), the scan reads the flags and writes the map (8 B).
    The compaction reads the map and writes 12 B per kept triangle, and moves 24 + 3 + 8 B per kept vertex."""
    per_pass = 12 * t
    per_vertex = 4 + 8 + 8 + 8 + 5 + 8
    return {"faces_bytes_per_pass": per_pass, "face_passes": 4, "label_bytes_per_vertex": per_vertex,
            "total_bytes": 4 * per_pass + per_vertex * m + 4 * 2 * t + 12 * tk + 2 * 35 * mk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--depth", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_components.py needs a CUDA device")
    from g2pc import build, capi, mesh
    build.build()
    name, power = card()
    vpos, faces, colours, dens = scene_mesh(args)
    torch.cuda.empty_cache()
    m, t = int(vpos.shape[0]), int(faces.shape[0])
    res = {"metric": "remove small components of the depth-10 scene mesh", "card": name, "power_limit": power,
           "depth": args.depth, "vertices": m, "triangles": t, "runs": args.runs, "settings": {}}
    for label, min_t, K in SETTINGS:
        stats = {}
        mesh.remove_components(vpos, faces, colours, dens, min_t, K)  # warm-up
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        total, per_entry, out = [], {e: [] for e in ENTRY_POINTS}, None
        for _ in range(args.runs):
            capi.TIMING = {}
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = mesh.remove_components(vpos, faces, colours, dens, min_t, K, stats=stats)
            b.record()
            torch.cuda.synchronize()
            total.append(a.elapsed_time(b))
            for e in ENTRY_POINTS:
                per_entry[e].append(sum(x.elapsed_time(y) for x, y in capi.TIMING.get(e, [])))
        capi.TIMING = None
        peak = torch.cuda.max_memory_allocated()
        mk, tk = int(out[0].shape[0]), int(out[1].shape[0])
        del out
        ab = algorithmic_bytes(m, t, mk, tk)
        med = float(np.median(total))
        res["settings"][label] = {
            "total": spread(total, 2), "entry_points_median_ms": {e[21:]: round(float(np.median(v)), 2)
                                                                  for e, v in per_entry.items()},
            "components": stats["components"], "kept": stats["kept"], "largest": stats["largest"],
            "removed_triangles": stats["removed_triangles"], "removed_vertices": stats["removed_vertices"],
            "algorithmic_bytes": ab, "algorithmic_gb_per_s": round(ab["total_bytes"] / (med * 1e-3) / 1e9, 1),
            "peak_allocated_gib": round(peak / 2 ** 30, 2), "mesh_allocated_gib": round(base / 2 ** 30, 2)}
    print(f"[components] {res}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
