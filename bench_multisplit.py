#!/usr/bin/env python
"""bench_multisplit.py — the colour stage's list build alone (g2pc_multisplit / g2pc_multisplit_grid, csrc/s4_tree.cu).

    python bench_multisplit.py [--cameras 20] [--repeats 3] [--shapes c3,c4,big]

Shapes: c3 = 3 M Gaussians at 1280 x 720, python back-end (quadtree leaves); c4 = the same scene at 1280 x 720 through
the CUDA back-end (super-tile grid); big = 6 M Gaussians at 1920 x 1080, python back-end, where count-driven splits below
the base level are common.  For each shape the renderer runs every camera once (warm-up: capacities grow, frames
replay), then --repeats passes over the cameras in async mode with every multisplit launch bracketed by CUDA events; the
median pass is reported as microseconds per camera (one frame slot: the frames do not overlap), with the last camera's row-list entries (0 where the build has no
row lists), final list entries and, for the python back-end, the quadtree's num_levels and base level.  The card's name,
power limit and SM clock are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.join(ROOT, "3dgs-to-pc_b200")
for p in (ROOT, PKG):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

SHAPES = {
    "c3": dict(n=3_000_000, res=1280, renderer="python"),
    "c4": dict(n=3_000_000, res=1280, renderer="cuda"),
    "big": dict(n=6_000_000, res=1920, renderer="python"),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock, max_clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_clock": clock, "sm_max_clock": max_clock}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({type(e).__name__})"}


def run_shape(shape, cameras, repeats, dev):
    from g2pc import capi, config, synth
    from oracle import gaussians as og
    import camera_handler as ch
    import gauss_render as gr
    sc = synth.make_scene(shape["n"], seed=1234 + 2, sh_degree=0)
    xyz, op, col = sc["xyz"].to(dev), sc["opacities"].to(dev), sc["colours"].to(dev)
    cov = og.build_covariance(sc["scales"], sc["rots"]).contiguous().to(dev)
    config.FRAME_SLOTS = 1  # kernel times are only the multisplit's when the frames do not overlap
    R = gr.get_renderer(shape["renderer"], xyz, op.unsqueeze(1), col, cov, visible_gaussian_threshold=0.05)
    poses, intr = synth.make_cameras(cameras)
    cams = [ch.get_camera(shape["renderer"], c.to(dev), k, colour_resolution=shape["res"]) for c, k in zip(poses, intr)]
    R.async_mode = True
    for c in cams:
        R(c)
    R.flush()
    name = "g2pc_multisplit" if shape["renderer"] == "python" else "g2pc_multisplit_grid"
    per_cam = []
    for _ in range(repeats):
        capi.TIMING = {}
        for c in cams:
            R(c)
        R.flush()
        torch.cuda.synchronize()
        ev = capi.TIMING.get(name, [])
        capi.TIMING = None
        per_cam.append(1000.0 * sum(a.elapsed_time(b) for a, b in ev) / max(len(ev), 1))
    h = R._slots[R._last_slot]["hdr"].tolist()
    row_word = getattr(capi, "HDR_ROW_INST", None)
    out = {"us_per_camera": round(float(np.median(per_cam)), 1), "passes_us": [round(x, 1) for x in per_cam],
           "cameras": cameras, "row_list_entries": h[row_word] if row_word is not None else 0,
           "list_entries": R.last_stats.get("total_instances"), "replays": R.replays}
    if shape["renderer"] == "python":
        t = R._last_tables
        out.update(num_levels=t["qt"].num_levels, base_level=t["base_level"], num_leaves=R.last_stats["num_leaves"])
    del R
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, default=20)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--shapes", default="c3,c4,big")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multisplit.py needs a CUDA device")
    from g2pc import build, capi
    build.build()
    capi.load()
    res = {"card": card()}
    for s in args.shapes.split(","):
        res[s] = run_shape(SHAPES[s], args.cameras, args.repeats, "cuda:0")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
