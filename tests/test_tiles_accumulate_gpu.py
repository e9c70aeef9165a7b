"""CUDA back-end (renderer_type="cuda", csrc/s7_tiles.cu) against float64 beyond one unmasked camera: per-pixel masks,
the per-Gaussian accumulators over several cameras, the two culls built on them and the SH colours of the projection
records.  Every blend is checked stage-wise: tests/f64ref.py is fed the kernel's own records (tests/tiles_harness.py).

Tolerances: image, depth and inverse depth within 2e-5 (depths relative to max(1, |depth|)) on pixels without a skip /
stop decision in the float32 band, exactly 0 on masked pixels; per-camera and accumulated maxima within 2e-5, arg-max
pixels and winning cameras equal unless declared near-ties (within 1e-6); total contribution within ncams * 2e-5;
surface distances defined on the same Gaussians and within 5e-5 relative; cull decisions exact outside a 2e-5 band;
SH record colours within 2e-6 + 8 u sum|term|.
"""
import numpy as np
import pytest
import torch

import edge_scenes as es
import f64ref as fr
import tiles_harness as th
from util import scene_to

pytestmark = pytest.mark.gpu
DEV = th.DEV
U = fr.U32
FLT_MAX = float(np.finfo(np.float32).max)
MASK_SIZES = [(200, 113), (65, 17), (48, 32)]


# ---- scenes and masks ----------------------------------------------------------------------------------------------
def _edge_scene(W, H, n_field, seed=21):
    """The `huge` field (long per-tile lists) in front of the origin camera, plus small splats centred in the right and
    bottom tile column / row and just outside the image, whose lists hold nothing else of theirs."""
    sc, cams, intr = es.huge(n_field=n_field, n_huge=2, seed=seed, res=(W, H))
    f = intr[0][2]
    rng = np.random.default_rng(seed)
    cx, cy = (W - 1) / 2.0, (H - 1) / 2.0
    pts = []
    for px in np.linspace(W - min(W, 16) + 2, W + 3, 5):
        for py in np.linspace(0, H - 1, 5):
            pts.append((px, py))
    for py in np.linspace(H - min(H, 16) + 1, H + 3, 4):
        for px in np.linspace(0, W - 1, 6):
            pts.append((px, py))
    pts = np.asarray(pts)
    z = rng.uniform(2.0, 5.0, pts.shape[0])
    # origin camera: view x = world x, view y = -world y, view z = -world z; pixel = c + f * view / view z
    xyz = np.stack([(pts[:, 0] - cx) * z / f, -(pts[:, 1] - cy) * z / f, -z], 1)
    m = xyz.shape[0]
    probe = es._finish(xyz, np.log(np.full((m, 3), 0.6 / f)) + np.log(z)[:, None], rng.normal(size=(m, 4)),
                       rng.uniform(0.3, 0.9, m), seed)
    probe["colours"] = torch.as_tensor(rng.uniform(0, 1, (m, 3)))
    out = {k: torch.cat([sc[k], probe[k]]) for k in ("xyz", "scales", "rots", "opacities", "colours")}
    out["shs"] = torch.zeros((out["xyz"].shape[0], 3, 1), dtype=torch.float64)
    return out, cams[0], intr[0]


def _masks(W, H):
    """name -> (H, W) int32 mask (1 = keep)."""
    ys, xs = np.mgrid[0:H, 0:W]
    out = {"ones": np.ones((H, W), np.int32), "zeros": np.zeros((H, W), np.int32),
           "checker": ((xs + ys) % 2).astype(np.int32)}
    for name, cols, rows in (("lines_a", (15, 32), (16, 31)), ("lines_b", (16, 31), (15, 32))):
        m = np.ones((H, W), np.int32)
        m[:, [c for c in cols if c < W]] = 0
        m[[r for r in rows if r < H], :] = 0
        out[name] = m
    # whole tiles: the right and bottom tile column / row (partial unless the size is a multiple of 16), one interior
    # tile and the first tile of the second super-tile column
    m = np.ones((H, W), np.int32)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    m[:, (gx - 1) * 16:] = 0
    m[(gy - 1) * 16:, :] = 0
    if gx > 3 and gy > 1:
        m[0:16, 32:48] = 0
    if gx > 2 and gy > 2:
        m[16:32, 16:32] = 0
    out["tiles"] = m
    return out


def _camera(c2w, k, mask=None, white=True, sh_degree=3, uint8=False):
    import camera_handler as ch
    mt = None
    if mask is not None:
        mt = torch.as_tensor(mask.astype(np.uint8) * 255 if uint8 else mask, device=DEV)
    return ch.get_camera("cuda", c2w.to(DEV), k, mask=mt, white_bkgd=white, sh_degree=sh_degree)


# ---- per-camera check ----------------------------------------------------------------------------------------------
def _check_camera(name, o, W, H, mask=None, bg=(1.0, 1.0, 1.0)):
    """One camera's outputs against the f64 blend of its own records; returns the f64 result and the counts."""
    f = fr.tiles_blend(o["rec"], o["ok"], W, H, list(bg), mask=mask)
    good = np.isfinite(f["image"][0])
    n_taint = int((~good).sum())
    assert n_taint <= max(4, int(2e-2 * W * H)), f"{name}: {n_taint} pixels with a decision in the f32 band"
    e = {}
    e["image"] = float(np.abs(o["image"] - f["image"])[:, good].max(initial=0.0))
    for key in ("depth", "invdepth"):
        e[key] = float((np.abs(o[key] - f[key])[good] / np.maximum(1.0, np.abs(f[key][good]))).max(initial=0.0))
    for key, v in e.items():
        assert v < 2e-5, f"{name}: {key} vs f64 {v:.2e}"
    if mask is not None:
        off = np.asarray(mask).reshape(H, W) == 0
        assert not o["image"][:, off].any() and not o["depth"][off].any() and not o["invdepth"][off].any(), \
            f"{name}: a masked pixel was written"
    clean = ~f["taint"]
    e["contrib"] = float(np.abs(o["contrib"] - f["contrib"])[clean].max(initial=0.0))
    assert e["contrib"] < 2e-5, f"{name}: max contribution vs f64 {e['contrib']:.2e}"
    seen = clean & (f["contrib"] > 0)
    differ = seen & (o["pixel"] != f["pixel"])
    near = f["contrib"] - f["second"] < 1e-6
    assert not (differ & ~near).any(), f"{name}: {int((differ & ~near).sum())} arg-max pixels differ on a clear maximum"
    ks = o["surface"] < FLT_MAX
    st = f["surf_taint"]
    cover = int((ks != np.isfinite(f["surface"]))[~st].sum())
    assert cover == 0, f"{name}: surface distance defined on {cover} Gaussians on one side only " \
                       f"(kernel {int(ks[~st].sum())}, f64 {int(np.isfinite(f['surface'])[~st].sum())})"
    fin = ks & ~st
    e["surface"] = float((np.abs(o["surface"] - f["surface"])[fin] / np.maximum(1.0, f["surface"][fin])).max(initial=0.0))
    assert e["surface"] < 5e-5, f"{name}: surface distance vs f64 {e['surface']:.2e}"
    cnt = dict(taint_px=n_taint, near_ties=int(differ.sum()), surf_taint=int(st.sum()), rounds=f["rounds_max"],
               list_max=f["list_max"])
    return f, cnt, e


# ---- masks ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wh", MASK_SIZES)
def test_masks_vs_f64(lib, wh):
    """Masks on images with partial edge tiles (200x113, 65x17) and exact ones (48x32): all ones is bit-identical to no
    mask, all zeros renders nothing, and a checkerboard, single masked columns / rows on tile and super-tile edges,
    whole masked tiles (the right and bottom partial ones included, on lists of several 256-entry rounds) and a 0/255
    uint8 mask agree with the f64 blend.  A tile whose inside pixels are all masked leaves before round 0 and records no
    surface distance."""
    W, H = wh
    sc, c2w, k = _edge_scene(W, H, n_field=900 if W * H > 10000 else 1500)
    masks = _masks(W, H)

    def run(mask, uint8=False):
        R, _, _ = th.cuda_setup(sc)
        o = th.tiles_camera(R, _camera(c2w, k, mask, uint8=uint8))
        R.flush()
        acc = [R.gaussian_max_contribution, R.gaussian_total_contribution, R.gaussian_colours,
               R.gaussian_min_surface_distance]
        return o, [a.cpu().numpy() for a in acc]

    o_none, acc_none = run(None)
    o_ones, acc_ones = run(masks["ones"])
    for key in ("image", "depth", "invdepth", "radii", "contrib", "pixel", "surface"):
        assert np.array_equal(o_none[key], o_ones[key]), f"all-ones mask changed {key}"
    for a, b in zip(acc_none, acc_ones):
        assert np.array_equal(a, b), "all-ones mask changed an accumulator"
    o_zero, acc_zero = run(masks["zeros"])
    assert not o_zero["image"].any() and not o_zero["depth"].any() and not o_zero["invdepth"].any()
    assert not o_zero["contrib"].any() and not acc_zero[0].any() and not acc_zero[1].any() and not acc_zero[2].any()
    n_fin = int((acc_zero[3] < FLT_MAX).sum())
    assert n_fin == 0, f"all-zeros mask: {n_fin} Gaussians received a surface distance"
    report = []
    f, cnt, e = _check_camera(f"{W}x{H} none", o_none, W, H)
    report.append(("none", cnt, e))
    for name in ("checker", "lines_a", "lines_b", "tiles"):
        o, _ = run(masks[name])
        f, cnt, e = _check_camera(f"{W}x{H} {name}", o, W, H, mask=masks[name])
        report.append((name, cnt, e))
        if name == "tiles":
            assert f["rounds_max"] >= 3, f"whole-tile mask scene: only {f['rounds_max']} rounds"
            o8, _ = run(masks[name], uint8=True)
            for key in ("image", "depth", "invdepth", "contrib", "pixel", "surface"):
                assert np.array_equal(o8[key], o[key]), f"uint8 0/255 mask differs from the 0/1 mask in {key}"
    for name, cnt, e in report:
        print(f"[accumulate masks {W}x{H} {name}] list max {cnt['list_max']} ({cnt['rounds']} rounds): "
              f"{cnt['taint_px']} pixels excluded by the taint band, {cnt['surf_taint']} surface distances tainted, "
              f"arg-max near-ties {cnt['near_ties']}; worst " + ", ".join(f"{a} {b:.1e}" for a, b in e.items()))


# ---- accumulation over cameras and the two culls --------------------------------------------------------------------
def _cross_scene():
    """A shell of 2500 Gaussians seen by five spiral poses, then pose 0 again with a black background and pose 2 again
    with whole tiles and a checkerboard band masked: 7 overlapping cameras of 160x90."""
    from g2pc import synth
    sc = synth.make_scene(2500, seed=31, sh_degree=0)
    sc["scales"] = sc["scales"] + 1.0  # larger splats: more overlap between cameras and longer lists
    cams, _ = synth.make_cameras(5)
    W, H = 160, 90
    k = [W, H, 200.0, 200.0]
    m = _masks(W, H)["tiles"]
    m[40:60, :] &= _masks(W, H)["checker"][40:60, :]
    views = [(cams[0], True, None), (cams[0], False, None), (cams[1], True, None), (cams[2], True, None),
             (cams[3], True, None), (cams[2], True, m), (cams[4], True, None)]
    return sc, k, views


def _render_cross(sc, k, views, async_replay=False, per_camera=True):
    R, _, _ = th.cuda_setup(sc)
    R.first_frame = torch.full((R._n,), -1, dtype=torch.int32, device=DEV)
    if async_replay:
        R.async_mode = True
        R._inst_cap = 16
    outs = []
    for c2w, white, mask in views:
        rs = _camera(c2w, k, mask, white=white)
        if per_camera:
            outs.append(th.tiles_camera(R, rs))
        else:
            R(rs)
    R.flush()
    if async_replay:
        assert R.replays >= 1, "the tiny instance buffer did not force a replay"
    return R, outs


def test_cross_camera_accumulators_and_culls_vs_f64(lib):
    """Seven overlapping cameras: the per-camera blends against f64, then the fold over cameras (strict > so the first
    camera keeps an exact tie, the colour from that camera's final image with its T * bg, f64 total, minimum surface
    distance, the winning camera index) and the two culls against f64; async mode with a forced replay gives the same
    accumulators bit for bit."""
    sc, k, views = _cross_scene()
    W, H = k[0], k[1]
    R, outs = _render_cross(sc, k, views)
    per, taint_px, near_px = [], 0, 0
    for i, (o, (_, white, mask)) in enumerate(zip(outs, views)):
        bg = (1.0, 1.0, 1.0) if white else (0.0, 0.0, 0.0)
        f, cnt, _ = _check_camera(f"camera {i}", o, W, H, mask=mask, bg=bg)
        per.append(f)
        taint_px += cnt["taint_px"]
        near_px += cnt["near_ties"]
    acc = fr.accumulate(per)
    kmax = R.gaussian_max_contribution.cpu().numpy()
    ktot = R.gaussian_total_contribution.cpu().numpy()
    kcol = R.gaussian_colours.cpu().numpy()
    kdist = R.gaussian_min_surface_distance.cpu().numpy()
    kfirst = R.first_frame.cpu().numpy()
    clean = ~acc["taint"]
    exact = clean & ~acc["near_tie"]
    assert np.abs(kmax - acc["max"])[clean].max() < 2e-5, "accumulated maximum vs f64"
    assert np.abs(ktot - acc["total"])[clean].max() < len(views) * 2e-5, "total contribution vs f64"
    wrong = exact & (kfirst != acc["winner"])
    assert not wrong.any(), f"{int(wrong.sum())} Gaussians credited to another camera than the f64 winner"
    colour_ok = exact & ~acc["pixel_tie"] & np.isfinite(acc["colour"]).all(axis=1)
    cerr = np.abs(kcol - acc["colour"]).max(axis=1)[colour_ok]
    assert cerr.max() < 2e-5, f"accumulated colour vs f64: {cerr.max():.2e}"
    # the repeated pose: exact ties keep camera 0 and its white-background colour
    c0, c1 = outs[0]["contrib"], outs[1]["contrib"]
    tie = (c0 > 0) & (c0 == c1) & (kfirst == 0)
    assert tie.sum() > 100 and not ((c0 > 0) & (c0 == c1) & (kfirst == 1)).any(), "exact ties not kept by camera 0"
    img0, img1 = outs[0]["image"].reshape(3, -1), outs[1]["image"].reshape(3, -1)
    pix = outs[0]["pixel"][tie]
    assert np.array_equal(kcol[tie], img0[:, pix].T), "a tie took another colour than camera 0's image"
    carries_bg = int((np.abs(img0[:, pix] - img1[:, pix]).max(axis=0) > 1e-3).sum())
    assert carries_bg > 0, "no tied arg-max pixel where the background shows"
    sfin = np.isfinite(acc["surface"])
    st = acc["surf_taint"]
    assert int(((kdist < FLT_MAX) != sfin)[~st].sum()) == 0, "accumulated surface distance coverage"
    serr = (np.abs(kdist - acc["surface"])[sfin & ~st] / np.maximum(1.0, acc["surface"][sfin & ~st])).max()
    assert serr < 5e-5, f"accumulated surface distance vs f64: {serr:.2e}"

    # culls: visibility at 0.05, surface distance below mean(finite) * std
    R.visible_gaussian_threshold = 0.05
    vis = R.get_visible_gaussians().cpu().numpy()
    band = np.abs(acc["max"] - 0.05) <= 2e-5
    want = acc["max"] > 0.05
    bad = (vis != want) & ~band & clean
    assert not bad.any(), f"{int(bad.sum())} visibility decisions differ from f64 outside the band"
    vis_flips = int(((vis != want) & (band | ~clean)).sum())
    # tainted distances are not pinned by f64: the mean takes the kernel's value for them
    dref = np.where(st, np.where(kdist < FLT_MAX, kdist.astype(np.float64), np.inf), acc["surface"])
    surf_flips = {}
    for std in (2.0, 0.5):
        R.surface_distance_std = std
        got = R.get_gaussians_with_low_surface_distance().cpu().numpy()
        thr = dref[np.isfinite(dref)].mean() * std
        want = dref < thr
        band = np.abs(dref - thr) <= 2e-5 * max(1.0, thr)
        bad = (got != want) & ~band & ~st
        assert not bad.any(), f"std {std}: {int(bad.sum())} surface-cull decisions differ from f64 outside the band"
        surf_flips[std] = int(((got != want) & (band | st)).sum())
        assert 0 < int(want.sum()) < int(np.isfinite(dref).sum()), f"std {std}: the cull keeps all or nothing"

    # async with a forced replay: the same accumulators bit for bit
    Ra, _ = _render_cross(sc, k, views, async_replay=True, per_camera=False)
    for name in ("gaussian_max_contribution", "gaussian_total_contribution", "gaussian_colours",
                 "gaussian_min_surface_distance", "first_frame"):
        assert torch.equal(getattr(R, name), getattr(Ra, name)), f"async replay changed {name}"
    print(f"[accumulate cameras] {len(views)} cameras {W}x{H}: {taint_px} pixels excluded by the taint band, "
          f"{int(acc['taint'].sum())} Gaussians tainted, per-camera arg-max near-ties {near_px}, cross-camera near-ties "
          f"{int((acc['near_tie'] & clean).sum())}, exact ties kept by camera 0 {int(tie.sum())} ({carries_bg} showing "
          f"the background); cull flips in the band: visibility {vis_flips}, surface std 2.0 {surf_flips[2.0]}, "
          f"std 0.5 {surf_flips[0.5]}")


# ---- SH ------------------------------------------------------------------------------------------------------------
def _sh_scene(stride, seed=41):
    """Gaussians on the six axes, the twelve face diagonals and the eight cube diagonals from the origin (where SH
    terms cancel or vanish exactly), plus random directions; coefficients large enough that r + 0.5 < 0 is common."""
    rng = np.random.default_rng(seed + stride)
    dirs = []
    for a in range(3):
        for s in (-1.0, 1.0):
            v = np.zeros(3); v[a] = s; dirs.append(3.0 * v)
    for a in range(3):
        for b in range(a + 1, 3):
            for sa in (-1.0, 1.0):
                for sb in (-1.0, 1.0):
                    v = np.zeros(3); v[a] = sa; v[b] = sb; dirs.append(2.0 * v)
    for sx in (-1.0, 1.0):
        for sy in (-1.0, 1.0):
            for sz in (-1.0, 1.0):
                dirs.append(2.0 * np.array([sx, sy, sz]))
    r = rng.normal(size=(200, 3))
    dirs += list(3.0 * r / np.linalg.norm(r, axis=1, keepdims=True))
    xyz = np.asarray(dirs)
    n = xyz.shape[0]
    sc = es._finish(xyz, np.log(np.full((n, 3), 0.03)), np.tile([1.0, 0, 0, 0], (n, 1)), np.full(n, 0.5), seed)
    shs = rng.normal(0.0, 0.6, (n, 3, stride))
    shs[:, :, 0] = rng.normal(0.0, 2.0, (n, 3))
    sc["shs"] = torch.as_tensor(shs)
    return sc


def _axis_cameras():
    """Six cameras at the origin looking along +-x, +-y, +-z (exact 0 / +-1 rotations, camera centre exactly 0)."""
    from g2pc import synth
    out = []
    for a in range(3):
        for s in (-1.0, 1.0):
            t = [0.0, 0.0, 0.0]; t[a] = s
            up = (0.0, 1.0, 0.0) if a == 2 else (0.0, 0.0, 1.0)
            out.append(synth.look_at_c2w((0.0, 0.0, 0.0), t, up))
    return out, [128, 96, 32.0, 32.0]  # tan(fov / 2) = 2 in x: the diagonals are in view


@pytest.mark.parametrize("stride", [1, 4, 9, 16])
def test_sh_record_colours_vs_f64(lib, stride):
    """SH colours of the projection records for every camera degree up to the scene's, channel-major (sh_layout 0,
    through get_renderer) and coefficient-major (sh_layout 1, GaussianRasterizer), against the f64 polynomial of the
    real spherical harmonics; a camera degree above what the stride holds raises G2pcError."""
    import gauss_render as gr
    from g2pc import capi
    from g2pc.rasterizer import GaussianRasterizer
    from oracle import gaussians as og
    sc = _sh_scene(stride)
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    shs32 = sc["shs"].float()
    cams, k = _axis_cameras()
    deg_max = int(round(stride ** 0.5)) - 1
    n = sc["xyz"].shape[0]
    xyz = sc["xyz"].numpy().astype(np.float64)
    worst, clamped, seen_all = 0.0, 0, np.zeros(n, dtype=bool)

    def renderer(layout):
        if layout == 0:
            return gr.get_renderer("cuda", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov, shs=d["shs"])
        return GaussianRasterizer(d["xyz"], None, d["opacities"], shs=shs32.permute(0, 2, 1).contiguous().to(DEV),
                                  cov3D_precomp=cov, sh_layout=1)

    for deg in range(deg_max + 1):
        for layout in (0, 1):
            R = renderer(layout)
            for c2w in cams:
                rs = _camera(c2w, k, sh_degree=deg)
                R(rs)
                sl = R._slots[R._last_slot]
                ok = sl["depth_key"].cpu().numpy().view(np.uint32) != 0xFFFFFFFF
                rec = sl["proj"].cpu().numpy()
                campos = np.asarray(rs._campos_host, dtype=np.float64)
                dirs = xyz - campos[None, :]
                dirs /= np.linalg.norm(dirs, axis=1, keepdims=True)
                coef = shs32.numpy() if layout == 0 else shs32.permute(0, 2, 1).numpy()
                want, bound = fr.sh_colour(deg, coef, dirs, layout)
                err = np.abs(rec[:, 6:9].astype(np.float64) - want)[ok]
                allow = 2e-6 + 8 * U * bound[ok]
                bad = err > allow
                assert not bad.any(), f"deg {deg} layout {layout}: {int(bad.sum())} colours off, worst " \
                                      f"{(err / allow).max():.2f} of allowed"
                worst = max(worst, float((err / allow).max(initial=0.0)))
                clamped += int((want[ok] == 0).sum())
                seen_all |= ok
    assert seen_all[:26].all(), "an axis or diagonal Gaussian was never in view"
    assert clamped > 0, "no colour hit the clamp at 0"
    if deg_max < 3:
        for layout in (0, 1):
            with pytest.raises(capi.G2pcError):
                renderer(layout)(_camera(cams[0], k, sh_degree=deg_max + 1))
    print(f"[accumulate sh stride {stride}] degrees 0..{deg_max}, both layouts, 6 axis cameras: worst err / allowed "
          f"{worst:.2f}, {clamped} colours clamped at 0")
