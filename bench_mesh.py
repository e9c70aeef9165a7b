"""Time the Poisson mesher (g2pc/mesh.py) on a C3-sized point cloud at depths 8, 9 and 10.

    python bench_mesh.py [--runs 5] [--depths 8,9,10] [--points 10000000] [--band_depths 11,12]

The cloud is sampled from the synthetic 3 M-Gaussian scene the way C3 samples its cloud, with the Gaussians' own colours
(--no_render_colours).  The sampler's normals have an arbitrary sign, so they are flipped to point away from the origin
(the scene's centre): the surface is then one shell seen from outside.  Every depth is warmed up once, then timed
`--runs` times with CUDA events around the whole mesh and around each phase (clean, splat, solve, extract, gather+trim,
smooth, normals); medians and the spread are printed with the multigrid cycles, the final residual ratio, the peak of
torch.cuda.max_memory_allocated, the vertex and face counts, and the card's name and power limit read in the same run.
There is no CPU comparator: Open3D, whose Poisson reconstruction the reference calls, is not installed.  One JSON line on
stdout; nothing is written to disk.

--band_depths times the narrow-band levels on the same cloud: the dense solve at depth 10, then band levels 11 ..
band_depth, with per-phase times (the band phases per level), bricks and nodes per level, conjugate-gradient
iterations and the peak of torch.cuda.max_memory_allocated.  A band the device cannot hold is reported with the memory
check's message instead of times.
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

PHASES = ["clean", "splat", "solve", "extract", "gather_trim", "smooth", "normals"]


def time_depth(points, normals, colours, depth, runs):
    from g2pc import mesh
    m, dbg = mesh.poisson_mesh(points, normals, colours, depth=depth, return_debug=True)  # warm-up, solver report
    nv, nf, cycles, ratio = int(m.vertices.shape[0]), int(m.faces.shape[0]), dbg["cycles"], dbg["ratio"]
    del m, dbg
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()

    def run(timings):
        m = mesh.poisson_mesh(points, normals, colours, depth=depth, timings=timings)
        assert (int(m.vertices.shape[0]), int(m.faces.shape[0])) == (nv, nf)

    total, phases = timed_runs(run, PHASES, runs)
    return {"depth": depth, "points": int(points.shape[0]), **spread(total, 1), "runs": runs,
            "phase_median_ms": {p: round(float(np.median(v)), 1) for p, v in phases.items()},
            "cycles": cycles, "residual_ratio": float(f"{ratio:.3g}"), "vertices": nv, "faces": nf,
            "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
            "peak_above_inputs_gib": round((torch.cuda.max_memory_allocated() - base) / 2 ** 30, 2)}


def time_band(points, normals, colours, band_depth, runs):
    from g2pc import capi, mesh
    torch.cuda.empty_cache()
    stats = []
    try:  # warm-up and solver report
        m = mesh.poisson_mesh(points, normals, colours, depth=10, band_depth=band_depth, band_stats=stats)
    except capi.G2pcError as e:  # the levels that fitted before the refusal are still reported
        return {"depth": 10, "band_depth": band_depth, "levels": stats, "refused": str(e)}
    levels = [dict(s, ratio=float(f"{s['ratio']:.3g}")) for s in stats]
    nv, nf = int(m.vertices.shape[0]), int(m.faces.shape[0])
    del m
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    phases = PHASES + [f"band{d}_{p}" for d in range(11, band_depth + 1) for p in ("bricks", "splat", "solve")]

    def run(timings):
        m = mesh.poisson_mesh(points, normals, colours, depth=10, band_depth=band_depth, timings=timings)
        assert (int(m.vertices.shape[0]), int(m.faces.shape[0])) == (nv, nf)

    total, ph = timed_runs(run, phases, runs)
    return {"depth": 10, "band_depth": band_depth, "points": int(points.shape[0]), **spread(total, 1), "runs": runs,
            "phase_median_ms": {p: round(float(np.median(v)), 1) for p, v in ph.items()}, "levels": levels,
            "vertices": nv, "faces": nf, "peak_allocated_gib": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--depths", default="8,9,10")
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--band_depths", default="", help="comma-separated band depths (11, 12) above a dense depth 10")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mesh.py needs a CUDA device")
    from g2pc import build, synth
    build.build()
    name, power = card()
    res = {"metric": "Poisson mesh (clean + splat + multigrid + marching tetrahedra + trim + 10 smoothing steps)",
           "card": name, "power_limit": power, "cpu": "none: Open3D is not installed, no CPU comparator", "gpu": []}
    pc = synth.sampled_cloud(3_000_000, args.points, 1236, DEV)
    nrm = pc.normals.to(torch.float32)
    flip = (nrm * pc.points).sum(1, keepdim=True) < 0
    points, normals, colours = pc.points.contiguous(), torch.where(flip, -nrm, nrm).contiguous(), pc.colours
    del pc, nrm, flip
    for d in [int(s) for s in args.depths.split(",") if s]:
        r = time_depth(points, normals, colours, d, args.runs)
        res["gpu"].append(r)
        print(f"[mesh] {r}", file=sys.stderr)
        torch.cuda.empty_cache()
    for b in [int(s) for s in args.band_depths.split(",") if s]:
        r = time_band(points, normals, colours, b, args.runs)
        res.setdefault("band", []).append(r)
        print(f"[band] {r}", file=sys.stderr)
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
