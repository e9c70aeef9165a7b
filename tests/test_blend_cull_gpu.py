"""Footprint cull of the python back-end's blend (csrc/s5_blend.cu, g2pc_blend_set_cull): a warp skips the Gaussians
whose alpha is below eps = min(2^-26, t_stop / list length) over its whole pixel rectangle.

  * predicate soundness (host, no GPU): the predicate restated in f32 on warp rectangles of both mappings and on
    random, needle (cond 1e10, every angle), degenerate (det <= 0), non-finite, clamped-opacity, edge-centred and huge
    splats: every pair it skips has a float64 (and a kernel-order f32) alpha below eps at every pixel of the rectangle;
    degenerate and non-finite records are never skipped;
  * cull on vs off at the same t_stop, colours 0 and background 1 (the leaf colour IS the transmittance): leaf colours
    bit for bit and cam_best bit for bit for every Gaussian whose maximum is >= 2^-26, on the hand-built leaf tables of
    test_blend_mapping_gpu (both mappings), the needle / disc / huge / ties / opacity edge scenes and one 1280x720 frame
    of a 3 M-Gaussian C3 scene;
  * with real colours every leaf pixel and every recorded colour (maximum > 1e-5) moves by <= t_stop x max |colour|;
  * t_stop = 0: cull on and off are byte-identical with equal executed pairs;
  * convert_gaussians_to_pc at C3's settings on a smaller scene: points, normals and the kept-Gaussian set identical;
  * compute-sanitizer memcheck / racecheck of a default-mode frame sequence (blend_cull_sanitizer_target.py).
"""
import math
import os

import numpy as np
import pytest
import torch

import edge_scenes as es
import f64ref as fr
import test_blend_mapping_gpu as bm
from util import scene_to

DEV = "cuda:0"
K = fr.K_EXP2
F32 = np.float32
EPS_MAX = 2.0 ** -26


# ---- the predicate, restated on the host -----------------------------------------------------------------------------
def _fma(a, b, c):
    """f32 fused multiply-add (the f64 product of two f32 values is exact)."""
    f64 = np.float64
    return (np.asarray(a, f64) * np.asarray(b, f64) + np.asarray(c, f64)).astype(F32)


def host_negligible(rec, rect, log2eps):
    """cull_negligible of s5_blend.cu for records rec (m, >= 6) f32 {mx, my, K a, K b, K c, log2 o} and one rectangle
    (x0, x1, y0, y1) of pixel coordinates."""
    x0, x1, y0, y1 = (F32(v) for v in rect)
    with np.errstate(all="ignore"):
        mx, my, a, b, c, L = (rec[:, i].astype(F32) for i in range(6))
        dx0, dx1, dy0, dy1 = x0 - mx, x1 - mx, y0 - my, y1 - my
        inside = (dx0 <= 0) & (dx1 >= 0) & (dy0 <= 0) & (dy1 >= 0)
        Dx, Dy = np.maximum(np.abs(dx0), np.abs(dx1)), np.maximum(np.abs(dy0), np.abs(dy1))
        S = np.abs(L) + np.abs(a) * Dx * Dx + np.abs(b) * Dx * Dy + np.abs(c) * Dy * Dy
        ry, rx = F32(-0.5) * b / c, F32(-0.5) * b / a

        def q(dx, dy):
            return -_fma(dx, _fma(a, dx, b * dy), c * dy * dy)

        def clamp(v, lo, hi):  # fminf / fmaxf: a NaN operand yields the other one
            return np.fmin(np.fmax(v, lo), hi)

        qmin = np.fmin(np.fmin(q(dx0, clamp(ry * dx0, dy0, dy1)), q(dx1, clamp(ry * dx1, dy0, dy1))),
                       np.fmin(q(clamp(rx * dy0, dx0, dx1), dy0), q(clamp(rx * dy1, dx0, dx1), dy1)))
        kappa = L - F32(log2eps)
        return ((S + np.abs(rx) + np.abs(ry) < np.inf) & (a < 0) & (c < 0) & (F32(4) * a * c > b * b) & ~inside &
                (qmin > kappa + _fma(S, F32(2.0 ** -16), F32(2.0 ** -12))))


def _max_alpha(rec, rect):
    """Largest alpha over the rectangle's pixels: float64 from the f32 record, and the kernel's f32 evaluation order."""
    x0, x1, y0, y1 = rect
    px, py = np.meshgrid(np.arange(x0, x1 + 1, dtype=np.float64), np.arange(y0, y1 + 1, dtype=np.float64))
    px, py = px.reshape(1, -1), py.reshape(1, -1)
    r = rec.astype(np.float64)
    mx, my, a, b, c, L = (r[:, i:i + 1] for i in range(6))
    dx, dy = px - mx, py - my
    e64 = L + a * dx * dx + b * dx * dy + c * dy * dy
    rf = rec.astype(F32)
    dxf, dyf = (px.astype(F32) - rf[:, 0:1]), (py.astype(F32) - rf[:, 1:2])
    Bq = dyf * rf[:, 3:4]
    Cq = _fma(dyf * dyf, rf[:, 4:5], rf[:, 5:6])
    e32 = _fma(dxf, _fma(dxf, rf[:, 2:3], Bq), Cq)
    with np.errstate(all="ignore"):
        return (np.minimum(0.99, np.exp2(e64)).max(axis=1),
                np.minimum(0.99, np.exp2(e32.astype(np.float64))).max(axis=1))


def _conic_records(rng, m, cx, cy, sx, sy, theta, opacity):
    """Records of 2-D Gaussians with axis sigmas sx, sy rotated by theta around (cx, cy)."""
    c, s = np.cos(theta), np.sin(theta)
    s00 = c * c * sx ** 2 + s * s * sy ** 2
    s11 = s * s * sx ** 2 + c * c * sy ** 2
    s01 = c * s * (sx ** 2 - sy ** 2)
    det = s00 * s11 - s01 ** 2
    rec = np.zeros((m, 6))
    rec[:, 0], rec[:, 1] = cx, cy
    rec[:, 2], rec[:, 3], rec[:, 4] = K * s11 / det, K * 2.0 * (-s01) / det, K * s00 / det
    rec[:, 5] = np.log2(opacity)
    return rec.astype(F32)


# warp rectangles: compact blocks of a 40 x 23 leaf (C3), of a 45 x 26 leaf (C2), a 4-px single-row block, row strips of
# 64-px and 160-px leaves, a 1-row strip
RECTS = [(640, 659, 360, 365), (660, 679, 378, 382), (720, 739, 405, 410), (100, 103, 7, 7), (0, 63, 0, 1),
         (320, 479, 100, 100), (1279, 1279, 700, 719)]


def _adversarial(rng, rect):
    x0, x1, y0, y1 = rect
    w, h = x1 - x0 + 1, y1 - y0 + 1
    xc, yc = 0.5 * (x0 + x1), 0.5 * (y0 + y1)
    out = []
    m = 4000  # ordinary splats around the rectangle, 0.3 .. 60 px, opacities up to the 0.99 clamp and above
    out.append(_conic_records(rng, m, xc + rng.uniform(-3, 3, m) * (w + 40), yc + rng.uniform(-3, 3, m) * (h + 40),
                              np.exp(rng.uniform(np.log(0.3), np.log(60), m)), np.exp(rng.uniform(np.log(0.3), np.log(60), m)),
                              rng.uniform(0, np.pi, m), rng.choice([0.002, 0.3, 0.99, 1.0], m)))
    ang = np.radians(np.arange(0.0, 180.0, 0.5))  # cond 1e10 needles at every angle, near and far
    for sx in (1e3, 10.0):
        for d in (0.0, 5.0, 40.0):
            out.append(_conic_records(rng, ang.size, x1 + d + 0.5, yc + d, np.full(ang.size, sx), np.full(ang.size, sx * 1e-5),
                                      ang, np.full(ang.size, 0.99)))
    m = 400  # splats larger than the leaf
    out.append(_conic_records(rng, m, xc + rng.uniform(-400, 400, m), yc + rng.uniform(-400, 400, m),
                              rng.uniform(60, 400, m), rng.uniform(60, 400, m), rng.uniform(0, np.pi, m), 0.5))
    m = 200  # means exactly on an edge or a corner of the rectangle
    e = _conic_records(rng, m, xc, yc, rng.uniform(0.3, 3, m), rng.uniform(0.3, 3, m), rng.uniform(0, np.pi, m), 1e-12)
    e[:, 0] = rng.choice([x0, x1, xc], m)
    e[:, 1] = np.where(e[:, 0] == xc, rng.choice([y0, y1], m), rng.uniform(y0, y1, m))
    out.append(e)
    return np.concatenate(out), e.shape[0]


def _degenerate(rect):
    """det P = 0 and < 0, non-positive diagonals, NaN / Inf in every field: never skipped."""
    x0, x1, y0, y1 = rect
    far = (x1 + 500.0, y1 + 500.0)
    base = np.array([*far, -1.0, 0.0, -1.0, -1.0], dtype=F32)
    assert host_negligible(base[None], rect, -26.0).all()  # skipped as it stands: each defect below is what keeps it
    rows = []
    for b in (2.0, -2.0, 3.0, -5.0):        # 4ac - b^2 = 0, 0, -5, -21
        r = base.copy(); r[3] = b; rows.append(r)
    for a, c in ((0.0, -1.0), (-1.0, 0.0), (1.0, -1.0), (-1.0, 1.0)):
        r = base.copy(); r[2], r[4], r[3] = a, c, 0.0; rows.append(r)
    for i in range(6):
        for v in (np.nan, np.inf, -np.inf):
            r = base.copy(); r[i] = v; rows.append(r)
    return np.asarray(rows, dtype=F32)


@pytest.mark.parametrize("log2eps", [-26.0, math.log2(1e-6) - math.log2(5000.0)])
def test_predicate_sound_against_f64(log2eps):
    """Every (rectangle, record) pair the predicate skips has alpha < eps at every pixel, in float64 and in the kernel's
    f32 order; degenerate and non-finite records and means on the rectangle are never skipped."""
    rng = np.random.default_rng(2601)
    eps = 2.0 ** log2eps
    kept = total = 0
    for rect in RECTS:
        rec, n_edge = _adversarial(rng, rect)
        skip = host_negligible(rec, rect, log2eps)
        a64, a32 = _max_alpha(rec[skip], rect)
        assert (a64 < eps).all(), f"{rect}: {int((a64 >= eps).sum())} skipped pairs reach eps in f64 (max {a64.max():.3e})"
        assert (a32 < eps).all(), f"{rect}: {int((a32 >= eps).sum())} skipped pairs reach eps in f32"
        assert not skip[-n_edge:].any(), f"{rect}: a splat centred on the rectangle's boundary was skipped"
        assert not host_negligible(_degenerate(rect), rect, log2eps).any(), f"{rect}: a degenerate record was skipped"
        kept += int((~skip).sum())
        total += skip.size
    print(f"[cull predicate] log2 eps {log2eps:.2f}: {total} adversarial pairs, kept {kept / total:.3f}")
    assert kept < total  # the test exercises both outcomes


# ---- the kernel, cull on vs off ------------------------------------------------------------------------------------
@pytest.fixture
def cull(lib):
    """g2pc_blend_set_cull is process-wide state: every test leaves it at the default (on)."""
    yield lambda on: lib.g2pc_blend_set_cull(int(on))
    lib.g2pc_blend_set_cull(1)


def _blend(S, bound, t_stop):
    """g2pc_blend + g2pc_accumulate + g2pc_compose_image on a hand-built frame; leaf colours, image, cam_best, the
    accumulated colours and the executed (pixel, Gaussian) pairs."""
    from g2pc import capi
    stats = torch.zeros(capi.STAT_WORDS, dtype=torch.int64, device=DEV)
    st = capi.stream_ptr(torch.device(DEV))
    n, L, W, H = S["proj"].shape[0], S["leaves"].shape[0], S["W"], S["H"]
    t = {k: torch.as_tensor(S[k], device=DEV) for k in ("leaves", "order", "gid")}
    proj = torch.as_tensor(S["proj"] if n else np.zeros((1, 12), F32), device=DEV)
    hdr = torch.zeros(capi.HDR_WORDS, dtype=torch.int32, device=DEV)
    hdr[capi.HDR_NUM_LEAVES] = L
    fail = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    work = torch.zeros(capi.WORK_COUNTERS, dtype=torch.int32, device=DEV)
    cam_best = torch.zeros(max(n, 1), dtype=torch.int64, device=DEV)
    mc = torch.zeros(max(n, 1), dtype=torch.float32, device=DEV)
    lc = torch.full((3 * max(S["total_pix"], 1),), float("nan"), dtype=torch.float32, device=DEV)
    owner = torch.zeros(W * H, dtype=torch.int32, device=DEV)
    capi.call("g2pc_blend", capi.ptr(t["leaves"]), capi.ptr(t["order"]), capi.ptr(hdr), capi.ptr(fail), 0, bound[0],
              bound[1], capi.ptr(t["gid"]), capi.ptr(proj), capi.ptr(cam_best), capi.ptr(mc), capi.ptr(lc),
              capi.ptr(owner), W, H, S["bg"], float(t_stop), capi.ptr(work), capi.ptr(stats), st)
    best = cam_best.clone()
    colours = torch.zeros((max(n, 1), 3), dtype=torch.float32, device=DEV)
    capi.call("g2pc_accumulate", capi.ptr(cam_best), capi.ptr(lc), n, capi.ptr(mc), capi.ptr(colours), None, 0, st)
    image = torch.empty((H, W, 3), dtype=torch.float32, device=DEV)
    capi.call("g2pc_compose_image", capi.ptr(owner), capi.ptr(lc), W, H, S["bg"], capi.ptr(image), st)
    torch.cuda.synchronize()
    return dict(lc=lc.cpu().numpy().reshape(-1, 3)[:S["total_pix"]], image=image.cpu().numpy(),
                best=best.cpu().numpy().view(np.uint64)[:n], colours=colours.cpu().numpy()[:n],
                pairs=int(stats[capi.STAT_WARP_GAUSSIANS]) * 128)


def _frames():
    S1, _ = bm._shape_grid()
    S2, _ = bm._early_exit()
    rng = np.random.default_rng(2602)
    wide = [bm._frame(rng, [wh, wh], [L for L in bm.LENGTHS if wh[0] * wh[1] * L <= 600_000][-2:], wh[0])
            for wh in bm.WIDE]
    return [("shapes", S1), ("early", S2)] + [(f"{S['W']}x{S['leaves'][0, 3]}", S) for S in wide]


def _dark(S):
    """The same frame with every record colour 0 and background 1: a leaf pixel's colour is its transmittance."""
    D = dict(S)
    D["proj"] = S["proj"].copy()
    D["proj"][:, 6:9] = 0.0
    D["bg"] = 1.0
    return D


@pytest.mark.gpu
def test_cull_leaf_tables(lib, mapping, cull):
    """Hand-built leaf tables (every width 2..64, wide and short leaves, list lengths around the chunk and sub-step
    edges, early-exit leaves), both mappings: T bit for bit with colours 0; the colour bound with real colours; fewer
    pairs; t_stop = 0 byte-identical."""
    from g2pc import config
    t_stop = config.BLEND_T_STOP
    for name, S in _frames():
        bound = (int(S["leaves"][:, 2].max()), int(S["leaves"][:, 3].max()))
        cmax = float(np.abs(S["proj"][:, 6:9]).max(initial=0.0))
        for compact in (1, 0):
            mapping(compact)
            what = f"{name} {'compact' if compact else 'strips'}"
            runs = {}
            for on in (0, 1):
                cull(on)
                runs[on] = (_blend(_dark(S), bound, t_stop), _blend(S, bound, t_stop), _blend(S, bound, 0.0))
            (d0, c0, s0), (d1, c1, s1) = runs[0], runs[1]
            assert np.array_equal(d0["lc"].view(np.uint32), d1["lc"].view(np.uint32)), f"{what}: T differs"
            v0 = bm._decode(d0["best"])[0]
            big = v0 >= EPS_MAX
            assert np.array_equal(d0["best"][big], d1["best"][big]), f"{what}: cam_best differs"
            dc = np.abs(c0["lc"] - c1["lc"]).max(initial=0.0)
            assert dc <= t_stop * cmax, f"{what}: leaf colour moved by {dc:.3e}"
            seen = bm._decode(c0["best"])[0] > 1e-5
            da = np.abs(c0["colours"][seen] - c1["colours"][seen]).max(initial=0.0)
            assert da <= t_stop * cmax, f"{what}: recorded colour moved by {da:.3e}"
            assert d1["pairs"] <= d0["pairs"] and c1["pairs"] <= c0["pairs"]
            for k in ("lc", "image", "best", "colours"):
                assert np.array_equal(np.asarray(s0[k]).view(np.uint8), np.asarray(s1[k]).view(np.uint8)), f"{what}: strict {k}"
            assert s0["pairs"] == s1["pairs"], f"{what}: strict pairs {s0['pairs']} vs {s1['pairs']}"
            print(f"[blend cull] {what}: pairs {c0['pairs']:.3e} -> {c1['pairs']:.3e} "
                  f"({c1['pairs'] / max(c0['pairs'], 1):.3f}), leaf colour moved {dc:.2e}, recorded colour {da:.2e}")


@pytest.fixture
def mapping(lib):
    yield lambda compact: lib.g2pc_blend_set_compact(int(compact))
    lib.g2pc_blend_set_compact(1)


def _edge_families():
    sc, cams, intr = es.huge(res=(320, 200))
    yield "huge", sc, cams, intr
    yield "ties", *es.ties()
    sc, cams, intr = es.opacity()
    yield "opacity", sc, cams[:40], intr[:40]
    for kind in ("needle", "disc"):
        sc = es.badly_conditioned(kind)
        sc["xyz"][:, 2] -= 3.0
        c2w, k = es.origin_camera(256, 192, 230.0)
        yield kind, sc, [c2w], [k]


def _render(sc, cams, intr, dark, **kw):
    import camera_handler as ch
    import gauss_render as gr
    from oracle import gaussians as og
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    col = torch.zeros_like(d["colours"]) if dark else d["colours"]
    R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), col, cov, **kw)
    imgs = [R(ch.get_camera("python", c.to(DEV), k))[0].cpu().numpy() for c, k in zip(cams, intr)]
    return imgs, R.gaussian_max_contribution.cpu().numpy(), R.gaussian_colours.cpu().numpy(), R.executed_pairs()


@pytest.mark.gpu
def test_cull_edge_scenes(lib, cull):
    """needle / disc / huge / ties / opacity families through the renderer at the default t_stop: images (= T with
    colours 0) bit for bit, maxima and their colours bit for bit where the maximum is >= 2^-26; real colours within
    t_stop x max |colour|."""
    from g2pc import config
    for name, sc, cams, intr in _edge_families():
        cmax = float(sc["colours"].abs().max())
        out = {}
        for on in (0, 1):
            cull(on)
            out[on] = (_render(sc, cams, intr, True), _render(sc, cams, intr, False))
        (d0, c0), (d1, c1) = out[0], out[1]
        for a, b in zip(d0[0], d1[0]):
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), f"{name}: T differs"
        big = d0[1] >= EPS_MAX
        assert np.array_equal(d0[1][big], d1[1][big]) and np.array_equal(c0[1][big], c1[1][big]), f"{name}: maxima"
        seen = c0[1] > 1e-5
        da = float(np.abs(c0[2][seen] - c1[2][seen]).max(initial=0.0))
        assert da <= config.BLEND_T_STOP * cmax, f"{name}: recorded colour moved by {da:.3e}"
        di = max(float(np.abs(a - b).max()) for a, b in zip(c0[0], c1[0]))
        assert di <= config.BLEND_T_STOP * cmax, f"{name}: image moved by {di:.3e}"
        assert c1[3] <= c0[3]
        print(f"[blend cull] {name}: pairs {c0[3]:.3e} -> {c1[3]:.3e}, image moved {di:.2e}, recorded colour {da:.2e}")


@pytest.mark.gpu
def test_cull_c3_frame(lib, cull):
    """One 1280x720 frame of a 3 M-Gaussian scene with C3's seed and camera rig: T bit for bit, maxima bit for bit
    where >= 2^-26, the image within t_stop x max |colour|, and the kept fraction of the pairs."""
    import camera_handler as ch
    import gauss_render as gr
    from g2pc import config, synth
    from oracle import gaussians as og
    sc = synth.make_scene(3_000_000, seed=1234 + 2, sh_degree=0)
    cams, intr = synth.make_cameras(200)
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    cmax = float(sc["colours"].abs().max())
    cam = ch.get_camera("python", cams[0].to(DEV), intr[0], colour_resolution=1280)
    out = {}
    for on in (0, 1):
        cull(on)
        res = []
        for col in (torch.zeros_like(d["colours"]), d["colours"]):
            R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), col, cov)
            img = R(cam)[0].cpu().numpy()
            res.append((img, R.gaussian_max_contribution.cpu().numpy(), R.executed_pairs()))
            del R
        out[on] = res
    (t0, c0), (t1, c1) = out[0], out[1]
    assert np.array_equal(t0[0].view(np.uint32), t1[0].view(np.uint32)), "T differs"
    big = t0[1] >= EPS_MAX
    assert np.array_equal(t0[1][big], t1[1][big])
    di = float(np.abs(c0[0] - c1[0]).max())
    assert di <= config.BLEND_T_STOP * cmax, f"image moved by {di:.3e}"
    assert c1[2] < c0[2]
    print(f"[blend cull] C3 frame 1280x720, 3M Gaussians: pairs {c0[2]:.4e} -> {c1[2]:.4e} "
          f"(kept {c1[2] / c0[2]:.4f}), image moved {di:.2e}")


@pytest.mark.gpu
def test_cull_end_to_end(lib, cull):
    """convert_gaussians_to_pc at C3's settings (300 k Gaussians, 24 cameras): points, normals and the kept-Gaussian
    set byte-identical, colours within 255 t_stop max |colour|, fewer executed pairs."""
    import bench
    import gauss_to_pc as g2p
    from g2pc import config, sampler, synth
    wl = dict(bench.WORKLOADS["c3"], n=300_000, cams=24, points=1_000_000)
    sc = synth.make_scene(wl["n"], seed=wl["seed"], sh_degree=wl["sh"])
    cams, intr = synth.make_cameras(wl["cams"])
    tr = {f"cam{i:04d}": c for i, c in enumerate(cams)}
    ki = {f"cam{i:04d}": k for i, k in enumerate(intr)}
    d = scene_to(sc, DEV)
    out = {}
    for on in (0, 1):
        cull(on)
        st = bench.settings_for(wl, g2p, DEV)
        sampler.reset_call_counter(0)
        pc, _ = g2p.convert_gaussians_to_pc(d["xyz"], d["scales"], d["rots"], d["colours"].clone(), d["opacities"],
                                            d["shs"], tr, ki, None, st, render_shs=True)
        pairs = int(g2p.LAST_RENDER_STATS["stats"][0].item()) * 128
        out[on] = (pc.points.cpu().numpy(), pc.normals.cpu().numpy(), pc.colours.cpu().numpy(), pairs)
    (p0, n0, c0, q0), (p1, n1, c1, q1) = out[0], out[1]
    assert np.array_equal(p0.view(np.uint8), p1.view(np.uint8)), "points differ"
    assert np.array_equal(n0.view(np.uint8), n1.view(np.uint8)), "normals differ"
    # point colours are 255 x the Gaussian's recorded colour; SH colours are clamped at 0 only, so max |colour| is read
    # from the cloud (at least 1)
    dc = float(np.abs(c0 - c1).max())
    assert dc <= 255.0 * config.BLEND_T_STOP * max(1.0, float(np.abs(c0).max()) / 255.0), f"colours moved by {dc:.3e}"
    assert q1 < q0
    print(f"[blend cull] end to end C3 settings, 300k Gaussians / 24 cameras: {p0.shape[0]} points, pairs "
          f"{q0:.3e} -> {q1:.3e} ({q1 / q0:.3f}), colours moved {dc:.2e}")


@pytest.mark.gpu
@pytest.mark.parametrize("tool", ["memcheck", "racecheck"])
def test_cull_under_compute_sanitizer(lib, tool, tmp_path):
    """memcheck / racecheck of a default-mode (t_stop = 1e-6, cull on) frame sequence."""
    from sanitizer_harness import check_target
    target = os.path.join(os.path.dirname(os.path.abspath(__file__)), "blend_cull_sanitizer_target.py")
    first = check_target(target, "BLEND_CULL_TARGET_OK", tool, tmp_path, timeout=900, repeat_racecheck=True)
    if first is not None:
        assert first["max_contribution"].shape[0] > 0
