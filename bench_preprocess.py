#!/usr/bin/env python
"""bench_preprocess.py — the colour stage's preprocess alone (csrc/s3_preprocess.cu) at C3's shapes, K cameras per launch.

    python bench_preprocess.py [--gaussians 3000000] [--cameras 200] [--res 1280] [--repeats 3] [--lib PATH ...]
                               [--no-timing]

C3: 3 M Gaussians, SH degree 3, 200 cameras at 1280 x 720.  For K = 1, 2, 4 and 8 the 200 cameras are projected in
launches of K (K = 1: g2pc_preprocess; K > 1: g2pc_preprocess_cameras), timed with CUDA events over all cameras after a
warm-up pass; the median of --repeats passes is reported.  Algorithmic bytes per (Gaussian, camera): the 240-byte scene
row (48 B packed geometry + 192 B SH) once per launch, i.e. 240 / K, plus the 60 bytes written (48 B record, 4 B key,
8 B value).  GB/s is set against MEASURED_PEAKS.json's hbm_gbs when that file exists, else the H100 SXM data sheet's
3.35 TB/s (labelled).  --lib PATH (repeatable) times the preprocess of another build of libg2pc.so in the same session
(e.g. the parent commit's, to compare kernels on one card; K = 1 only when it has no g2pc_preprocess_cameras).
Also: the peak max_memory_allocated of the whole colour stage (python back-end, async mode) at config.PREPROCESS_CAMERAS
= 1 and at the default, each in a fresh process (--memory-k K), with the scene alone as the baseline.  The card's name
and power limit are read in the same run.  Prints one JSON line."""
import argparse
import ctypes
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clock}
    except Exception as e:
        return {"name": torch.cuda.get_device_name(0), "power_limit": f"unknown ({type(e).__name__})"}


def peak_gbs():
    try:
        return float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]), "measured HBM peak"
    except Exception:
        return 3350.0, "H100 SXM data sheet (not measured)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gaussians", type=int, default=3_000_000)
    ap.add_argument("--cameras", type=int, default=200)
    ap.add_argument("--res", type=int, default=1280)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1234 + 2)
    ap.add_argument("--lib", action="append", default=[], help="another build of libg2pc.so to time in this session")
    ap.add_argument("--memory-k", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--no-timing", action="store_true", help="colour-stage memory only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_preprocess.py needs a CUDA device")
    from g2pc import build, capi, config, synth
    build.build()
    capi.load()
    import camera_handler as ch
    import gauss_handler as gh
    import gauss_render as gr

    dev = "cuda:0"
    sc = synth.make_scene(args.gaussians, seed=args.seed, sh_degree=3)
    d = {k: v.to(dev) for k, v in sc.items()}
    G = gh.Gaussians(d["xyz"], d["scales"], d["rots"], d["colours"], d["opacities"], shs=d["shs"])
    poses, intr = synth.make_cameras(args.cameras)
    cams = [ch.get_camera("python", c, k, colour_resolution=args.res) for c, k in zip(poses, intr)]

    if args.memory_k:
        # one process per K: nothing of an earlier renderer can still be allocated
        config.PREPROCESS_CAMERAS = args.memory_k
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        R = gr.get_renderer("python", G.xyz, G.opacities.unsqueeze(1), G.colours, G.covariances, shs=G.shs,
                            visible_gaussian_threshold=0.05)
        R.async_mode = True
        for c in cams:
            R(c)
        R.flush()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated()
        print(json.dumps({"K": args.memory_k, "scene_gib": round(base / 2**30, 3), "peak_gib": round(peak / 2**30, 3),
                          "above_scene_gib": round((peak - base) / 2**30, 3)}))
        return
    memory = {}
    for k in sorted({1, config.PREPROCESS_CAMERAS}):
        out = subprocess.run([sys.executable, os.path.abspath(__file__), "--memory-k", str(k), "--gaussians",
                              str(args.gaussians), "--cameras", str(args.cameras), "--res", str(args.res), "--seed",
                              str(args.seed)], capture_output=True, text=True)
        lines = [x for x in out.stdout.splitlines() if x.startswith("{")]
        memory[f"K={k}"] = json.loads(lines[-1]) if lines else {"failed": out.stderr[-500:]}
    if args.no_timing:
        print(json.dumps({"bench": "preprocess memory", "gaussians": args.gaussians, "cameras": args.cameras,
                          "res": args.res, "card": card(), "colour_stage_memory": memory}))
        return

    # ---- the preprocess alone ------------------------------------------------------------------------------------------
    R = gr.get_renderer("python", G.xyz, G.opacities.unsqueeze(1), G.colours, G.covariances, shs=G.shs,
                        visible_gaussian_threshold=0.05)
    W, H = int(cams[0].image_width), int(cams[0].image_height)
    t = R._get_tables(W, H)
    qt = t["qt"]
    n = R._n
    kmax = capi.PREPROCESS_MAX_CAMERAS
    outs = [dict(proj=torch.empty((n, 12), dtype=torch.float32, device=dev),
                 depth_key=torch.empty((n,), dtype=torch.int32, device=dev),
                 val=torch.empty((n,), dtype=torch.int64, device=dev),
                 node_cnt=torch.zeros((qt.nodes_2d,), dtype=torch.int32, device=dev)) for _ in range(kmax)]
    structs = [R._camera_struct(c) for c in cams]
    scene = (capi.ptr(R._geom), None, capi.ptr(R.shs), int(R.shs.shape[-1]), R.sh_degree, n)
    tab = (capi.ptr(t["tables"]), capi.ptr(t["luts"]), qt.num_levels, t["level_mask"], t["clean_mask"])
    st = capi.stream_ptr(dev)

    def ptrs(key, k):
        return (ctypes.c_void_p * k)(*[capi.ptr(o[key]) for o in outs[:k]])

    def one_pass(lib, K):
        arrays = {key: ptrs(key, K) for key in ("proj", "node_cnt", "depth_key", "val")}
        for c0 in range(0, len(structs), K):
            k = min(K, len(structs) - c0)
            if K == 1:
                o = outs[0]
                status = lib.g2pc_preprocess(*scene, ctypes.byref(structs[c0]), *tab, capi.ptr(o["proj"]),
                                             capi.ptr(o["node_cnt"]), capi.ptr(o["depth_key"]), capi.ptr(o["val"]), st)
            else:
                cs = (capi.Camera * k)(*structs[c0:c0 + k])
                status = lib.g2pc_preprocess_cameras(*scene, cs, k, *tab, arrays["proj"], arrays["node_cnt"],
                                                     arrays["depth_key"], arrays["val"], st)
            capi.check(status, "preprocess")

    def load(path):
        lib = ctypes.CDLL(path)
        for name in ("g2pc_preprocess", "g2pc_preprocess_cameras"):
            if hasattr(lib, name):
                getattr(lib, name).argtypes, getattr(lib, name).restype = capi.SIGNATURES[name]
        return lib

    gbs_peak, peak_src = peak_gbs()
    rows = []
    for path in [capi.LIB_PATH] + [os.path.abspath(x) for x in args.lib]:
        lib = load(path)
        for K in ((1, 2, 4, 8) if hasattr(lib, "g2pc_preprocess_cameras") else (1,)):
            one_pass(lib, K)  # warm-up
            times = []
            for _ in range(args.repeats):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                one_pass(lib, K)
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b))
            ms = float(np.median(times))
            per_cam = ms / len(structs)
            alg = n * (240.0 / K + 60.0)  # bytes per camera
            gbs = alg / (per_cam * 1e-3) / 1e9
            rows.append({"lib": os.path.relpath(path, ROOT), "K": K, "ms_per_camera": round(per_cam, 4),
                         "ms_all_cameras": round(ms, 2), "spread_ms": [round(min(times), 2), round(max(times), 2)],
                         "alg_bytes_per_gaussian_camera": round(240.0 / K + 60.0, 1), "alg_GBps": round(gbs, 1),
                         "frac_of_peak": round(gbs / gbs_peak, 3)})
    print(json.dumps({"bench": "preprocess", "gaussians": n, "cameras": len(structs), "resolution": [W, H],
                      "sh_degree": 3, "card": card(), "peak_GBps": gbs_peak, "peak_source": peak_src,
                      "results": rows, "colour_stage_memory": memory,
                      "preprocess_cameras_default": config.PREPROCESS_CAMERAS}))


if __name__ == "__main__":
    main()
