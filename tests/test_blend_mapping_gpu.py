"""How the python back-end's blend (csrc/s5_blend.cu) hands pixels to threads, checked against float64.

The parity tests run the blend only through the renderer at max_tile_size = 60, which reaches a handful of leaf shapes.
Here g2pc_blend -> g2pc_accumulate -> g2pc_compose_image are driven through the C ABI on hand-built leaf tables:
  * every leaf width 2..64 at 13 heights (every quads-per-row value 1..16 and every block shape of the compact mapping),
    wide, short leaves (more blocks across than the 60-px leaves have) and a 1-row leaf, under a tight and a loose
    leaf-size bound;
  * list lengths around the 128-id chunks, the 3-slot TMA ring and the 32-Gaussian stop check (0 .. ~2000);
  * leaves whose front splats are opaque, so every warp stops in chunk 0 or 1, interleaved in the launch order with
    ordinary leaves, so that persistent CTAs take an ordinary item with the same buffers right after an early exit;
  * splats centred between two pixels of one quad, between two quads and between four pixels (exact ties: the lowest
    pixel wins) and just beyond a leaf's right edge (next to the padding pixels of the last quad);
  * both pixel mappings (compact blocks, row strips) at t_stop = 0 (FLT_MIN) and at config.BLEND_T_STOP.
The float64 reference is f64ref.leaf_blend fed the same records and lists.  Renderer-level cases: max_tile_size raised to
the image width on 163x7 and 1280x13 images (one wide, short leaf), and a frame of more than 4096 leaves (build_tree's
launch order is then the BFS order instead of the heaviest-first sort).
"""
import numpy as np
import pytest
import torch

import edge_scenes as es
import f64ref as fr
from util import scene_to

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
K = fr.K_EXP2
FLT_MIN = float(np.finfo(np.float32).tiny)
HEIGHTS = (2, 3, 5, 6, 7, 8, 12, 13, 23, 31, 32, 33, 60)
LENGTHS = (0, 1, 31, 32, 33, 127, 128, 129, 255, 256, 257, 385, 1999)
WIDE = [(163, 2), (163, 7), (168, 7), (320, 4), (1280, 13), (4096, 2), (161, 1)]
PAIR_BUDGET = 120_000  # pixels x list length per leaf of the shape grid (bounds the f64 blend's time)


@pytest.fixture
def mapping(lib):
    """g2pc_blend_set_compact is process-wide state: every test leaves it at the default (compact blocks)."""
    yield lambda compact: lib.g2pc_blend_set_compact(int(compact))
    lib.g2pc_blend_set_compact(1)


# ---- hand-built frames ---------------------------------------------------------------------------------------------
def _splats(rng, r0, c0, w, h, m):
    """m records around the leaf in the python back-end layout {mx, my, K a, K 2b} {K c, log2 o, r, g} {b, depth, radius,
    valid}, conic (a, b, c) of a random 2-D Gaussian pre-scaled by K = -0.5 log2(e)."""
    sx = rng.uniform(0.6, 0.4 * w + 1.0, m)
    sy = rng.uniform(0.6, 0.4 * h + 1.0, m)
    rho = rng.uniform(-0.7, 0.7, m)
    det = (sx * sy) ** 2 * (1.0 - rho ** 2)
    rec = np.zeros((m, 12))
    rec[:, 0] = c0 + rng.uniform(-1.5, w + 0.5, m)
    rec[:, 1] = r0 + rng.uniform(-1.5, h + 0.5, m)
    rec[:, 2], rec[:, 3], rec[:, 4] = K * sy ** 2 / det, K * 2.0 * (-rho * sx * sy) / det, K * sx ** 2 / det
    rec[:, 5] = np.log2(rng.uniform(0.02, 0.6, m))
    rec[:, 6:9] = rng.uniform(0.0, 1.0, (m, 3))
    rec[:, 9] = np.arange(m)
    rec[:, 10], rec[:, 11] = 3.0, 1.0
    return rec


def _round(rec, x, y, s, opacity):
    """Make `rec` an axis-aligned round splat at (x, y): its values at pixels mirrored about it are equal in f32."""
    rec[0], rec[1], rec[2], rec[3], rec[4], rec[5] = x, y, K / s ** 2, 0.0, K / s ** 2, np.log2(opacity)


def _place(shapes, width):
    """Leaves of the given (w, h) on shelves of an image `width` pixels wide, without overlap: (r0, c0) each, W, H."""
    x = y = shelf = 0
    out = []
    for w, h in shapes:
        if x + w > width:
            y, x, shelf = y + shelf, 0, 0
        out.append((y, x))
        x, shelf = x + w, max(shelf, h)
    return out, width, y + shelf


def _frame(rng, shapes, lengths, width, bg=1.0, early=(), order=None):
    """One frame: leaf table (BFS order = list order), launch order (heaviest first unless given), 16-byte aligned lists
    of fresh splats per leaf.  The first entry of a list is a tie splat (between two pixels of a quad, two quads or
    four pixels, in rotation), the second, on leaves whose width is not a multiple of 4, a splat just beyond the right
    edge (0.2 px from the padding pixel).  early: (leaf, k0) pairs whose entries k0 .. k0 + 5 become opaque splats
    larger than the leaf (T < 1e-8 after them)."""
    pos, W, H = _place(shapes, width)
    early = dict(early)
    recs, lists, leaves, ties = [], [], [], []
    n = beg = pix = 0
    for i, ((w, h), (r0, c0), m) in enumerate(zip(shapes, pos, lengths)):
        rec = _splats(rng, r0, c0, w, h, m)
        kind = i % 3
        k0 = early.get(i, m)
        if k0 >= 1 and (kind < 2 and w >= (3 if kind == 0 else 5) or kind == 2 and h >= 2):
            if kind == 0:    # pixels 1 and 2 of a quad (one thread)
                _round(rec[0], c0 + 4 * ((w - 3) // 8) + 1.5, r0 + h // 2, rng.uniform(0.8, 2.5), 0.9)
            elif kind == 1:  # pixel 3 of one quad and pixel 0 of the next (two threads)
                _round(rec[0], c0 + 4 * ((w - 5) // 8) + 3.5, r0 + h // 2, rng.uniform(0.8, 2.5), 0.9)
            else:            # four pixels on two rows (two warps / blocks where a block boundary falls between them)
                _round(rec[0], c0 + w // 2 - 0.5, r0 + h // 2 - 0.5, rng.uniform(0.8, 2.5), 0.9)
            ties.append(n)
        if m >= 2 and w % 4:
            _round(rec[1], c0 + w - 0.2, r0 + h // 2, 0.7, 0.8)
        if i in early:
            for k in range(k0, k0 + 6):
                _round(rec[k], c0 + 0.5 * w, r0 + 0.5 * h, 4.0 * max(w, h) + 4.0, 0.995)
        recs.append(rec)
        lists.append(np.arange(n, n + m))
        leaves.append((r0, c0, w, h, beg, m, pix, i))
        n, beg, pix = n + m, beg + (m + 3) // 4 * 4, pix + w * h
    proj = np.concatenate(recs).astype(np.float32) if n else np.zeros((0, 12), np.float32)
    gid = np.zeros(beg + 4, dtype=np.int32)  # + one 16-byte unit: the TMA copies whole units
    for lf, ids in zip(leaves, lists):
        gid[lf[4]:lf[4] + lf[5]] = ids
    leaves = np.asarray(leaves, dtype=np.int32)
    if order is None:
        order = np.argsort(-leaves[:, 5], kind="stable")
    return dict(leaves=leaves, lists=lists, proj=proj, gid=gid, order=np.asarray(order, dtype=np.int32), W=W, H=H,
                bg=bg, total_pix=pix, ties=np.asarray(ties, dtype=np.int64),
                tight=(int(leaves[:, 2].max()), int(leaves[:, 3].max())))


def _reference(S):
    """float64: leaf colours and final transmittance, the image, and per Gaussian the maximum contribution over its
    leaves (strict > in BFS order: the lowest concatenated leaf-pixel index among exact ties), that pixel, and the
    largest contribution at any other pixel (how far the arg-max is from a tie)."""
    proj, n = S["proj"], S["proj"].shape[0]
    cols, Ts, G, V, P, S2 = [], [], [], [], [], []
    img = np.full((S["H"], S["W"], 3), S["bg"], dtype=np.float64)
    Timg = np.ones((S["H"], S["W"]))
    for (r0, c0, w, h, _, m, pix, _), ids in zip(S["leaves"], S["lists"]):
        col, con, T = fr.leaf_blend(r0, c0, w, h, ids, proj, bg=S["bg"], transmittance=True)
        cols.append(col)
        Ts.append(T)
        img[r0:r0 + h, c0:c0 + w] = col.reshape(h, w, 3)
        Timg[r0:r0 + h, c0:c0 + w] = T.reshape(h, w)
        if m:
            ar = np.arange(m)
            am = con.argmax(axis=0)  # first (lowest) pixel among exact ties
            v = con[am, ar]
            other = con.copy()
            other[am, ar] = -1.0
            G.append(ids); V.append(v); P.append(pix + am); S2.append(other.max(axis=0) if w * h > 1 else 0 * v)
    best, bpix, second = np.zeros(n), np.full(n, -1, dtype=np.int64), np.zeros(n)
    if G:
        G, V, P, S2 = (np.concatenate(a) for a in (G, V, P, S2))
        o = np.lexsort((P, -V, G))
        G, V, P, S2 = G[o], V[o], P[o], S2[o]
        first = np.r_[True, G[1:] != G[:-1]]
        best[G[first]], bpix[G[first]], second[G[first]] = V[first], P[first], S2[first]
        nxt = np.flatnonzero(first[:-1] & ~first[1:])  # Gaussians listed in several leaves: best of the others
        second[G[nxt]] = np.maximum(second[G[nxt]], V[nxt + 1])
    return dict(colour=np.concatenate(cols), T=np.concatenate(Ts), image=img[:, ::-1], T_image=Timg[:, ::-1],
                best=best, pix=bpix, second=second)


def _run(S, bound, t_stop, preset=None):
    """g2pc_blend (leaf colours pre-filled with NaN, work counters zeroed, fail word 0xFFFFFFFF), then g2pc_accumulate
    and g2pc_compose_image on the frame's buffers."""
    from g2pc import capi
    st = capi.stream_ptr(torch.device(DEV))
    n, L = S["proj"].shape[0], S["leaves"].shape[0]
    W, H, bg = S["W"], S["H"], S["bg"]
    leaves = torch.as_tensor(S["leaves"], device=DEV)
    order = torch.as_tensor(S["order"], device=DEV)
    gid = torch.as_tensor(S["gid"], device=DEV)
    proj = torch.as_tensor(S["proj"] if n else np.zeros((1, 12), np.float32), device=DEV)
    hdr = torch.zeros(capi.HDR_WORDS, dtype=torch.int32, device=DEV)
    hdr[capi.HDR_NUM_LEAVES] = L
    fail = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    work = torch.zeros(capi.WORK_COUNTERS, dtype=torch.int32, device=DEV)
    cam_best = torch.zeros(max(n, 1), dtype=torch.int64, device=DEV)
    mc = torch.zeros(max(n, 1), dtype=torch.float32, device=DEV)
    if preset is not None:
        mc[:n] = torch.as_tensor(preset, device=DEV)
    lc = torch.full((3 * max(S["total_pix"], 1),), float("nan"), dtype=torch.float32, device=DEV)
    owner = torch.zeros(W * H, dtype=torch.int32, device=DEV)
    capi.call("g2pc_blend", capi.ptr(leaves), capi.ptr(order), capi.ptr(hdr), capi.ptr(fail), 0, bound[0], bound[1],
              capi.ptr(gid), capi.ptr(proj), capi.ptr(cam_best), capi.ptr(mc), capi.ptr(lc), capi.ptr(owner), W, H, bg,
              float(t_stop), capi.ptr(work), None, st)
    best = cam_best.clone()
    colours = torch.zeros((max(n, 1), 3), dtype=torch.float32, device=DEV)
    capi.call("g2pc_accumulate", capi.ptr(cam_best), capi.ptr(lc), n, capi.ptr(mc), capi.ptr(colours), None, 0, st)
    image = torch.empty((H, W, 3), dtype=torch.float32, device=DEV)
    capi.call("g2pc_compose_image", capi.ptr(owner), capi.ptr(lc), W, H, bg, capi.ptr(image), st)
    torch.cuda.synchronize()
    assert int(cam_best.abs().sum()) == 0 and int(owner.abs().sum()) == 0, "accumulate / compose must clear their input"
    best = best.cpu().numpy().view(np.uint64)[:n]
    return dict(lc=lc.cpu().numpy().reshape(-1, 3)[:S["total_pix"]], image=image.cpu().numpy(), best=best,
                mc=mc.cpu().numpy()[:n], colours=colours.cpu().numpy()[:n])


def _decode(best):
    """cam_best -> (f32 contribution, concatenated leaf-pixel index; -1 where nothing was recorded)."""
    v = (best >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    p = np.where(best == 0, -1, 0xFFFFFFFF - (best & np.uint64(0xFFFFFFFF)).astype(np.int64))
    return v, p


def _check_f64(S, ref, out, what):
    """Strict stop: every leaf pixel written; colours, image and maxima within 2e-5 of f64; the arg-max pixel equal
    unless the f64 runner-up is within 1e-6 (exact ties always: the lowest pixel); accumulate copied what blend
    recorded."""
    lc = out["lc"]
    unwritten = ~np.isfinite(lc).all(axis=1)
    assert not unwritten.any(), f"{what}: {int(unwritten.sum())} of {lc.shape[0]} leaf pixels never written"
    e_col = np.abs(lc - ref["colour"]).max() if lc.size else 0.0
    e_img = np.abs(out["image"] - ref["image"]).max()
    assert e_col < 2e-5 and e_img < 2e-5, f"{what}: leaf colours {e_col:.2e}, image {e_img:.2e} vs f64"
    kv, kp = _decode(out["best"])
    e_max = np.abs(kv - ref["best"]).max() if kv.size else 0.0
    assert e_max < 2e-5, f"{what}: per-Gaussian maximum {e_max:.2e} vs f64"
    seen = kv > 0
    clear = ref["best"] - ref["second"] >= 1e-6
    bad = seen & clear & (kp != ref["pix"])
    assert not bad.any(), f"{what}: {int(bad.sum())} arg-max pixels differ on a clear maximum"
    ties = S["ties"]
    assert (ref["second"][ties] == ref["best"][ties]).all(), "tie splats must tie exactly in f64"
    assert np.array_equal(kp[ties], ref["pix"][ties]), \
        f"{what}: {int((kp[ties] != ref['pix'][ties]).sum())} of {ties.size} exact ties not resolved to the lowest pixel"
    assert np.array_equal(out["mc"], np.where(seen, kv, 0.0).astype(np.float32))
    assert np.array_equal(out["colours"][seen], lc[kp[seen]]) and (out["colours"][~seen] == 0).all()
    return int((seen & ~clear & (kp != ref["pix"])).sum())


def _check_stop(strict, tol, what):
    """Default stop against the strict run of the same mapping (test_tolerance_stop_within_contract's rules)."""
    assert np.isfinite(tol["lc"]).all(), f"{what}: leaf pixels never written"
    m0, m1 = _decode(strict["best"])[0], _decode(tol["best"])[0]
    assert np.abs(m0 - m1).max(initial=0) < 1e-5, f"{what}: maxima moved by the stop"
    assert np.abs(strict["lc"] - tol["lc"]).max(initial=0) < 1e-5
    assert np.abs(strict["image"] - tol["image"]).max() < 1e-5
    seen = m0 > 1e-5
    assert np.abs(strict["colours"][seen] - tol["colours"][seen]).max(initial=0) < 1e-5


def _check_strict_gt(S, bound, t_stop, out, what):
    """cam_best records a Gaussian only where it beats the running maximum (strict >): preset to the kernel's own
    maximum nothing is recorded, preset one ulp lower the same winner is."""
    kv = _decode(out["best"])[0].astype(np.float32)
    again = _run(S, bound, t_stop, preset=kv)
    assert not again["best"].any(), f"{what}: {int((again['best'] != 0).sum())} recorded at an equal maximum"
    lower = np.where(kv > 0, np.nextafter(kv, np.float32(0)), np.float32(0))
    below = _run(S, bound, t_stop, preset=lower)
    assert np.array_equal(below["best"], out["best"]), f"{what}: winners differ one ulp below the maximum"


def _compare_mappings(ref, a, b, what):
    """Compact blocks vs row strips, strict stop: every pixel runs the same f32 operations and the packed atomicMax does
    not depend on order, so the outputs are identical, except where a warp of one mapping stopped earlier at FLT_MIN:
    Gaussians whose maximum is below FLT_MIN and pixels whose final T is below FLT_MIN."""
    va, vb = _decode(a["best"])[0], _decode(b["best"])[0]
    dg = a["best"] != b["best"]
    g_ok = (va < FLT_MIN) & (vb < FLT_MIN)
    assert not (dg & ~g_ok).any(), f"{what}: cam_best differs for {int((dg & ~g_ok).sum())} Gaussians"
    dp = (a["lc"] != b["lc"]).any(axis=1)
    assert not (dp & ~(ref["T"] < FLT_MIN)).any(), f"{what}: {int((dp & ~(ref['T'] < FLT_MIN)).sum())} leaf colours differ"
    di = (a["image"] != b["image"]).any(axis=2)
    assert not (di & ~(ref["T_image"] < FLT_MIN)).any(), f"{what}: image differs"
    return int(dg.sum()), int(dp.sum())


def _all_configs(lib, mapping, S, ref, bound, what):
    from g2pc import config
    strict = {}
    for compact in (1, 0):
        mapping(compact)
        name = f"{what} {'compact' if compact else 'strips'} bound {bound}"
        s = _run(S, bound, 0.0)
        near = _check_f64(S, ref, s, name + " t_stop 0")
        _check_strict_gt(S, bound, 0.0, s, name + " t_stop 0")
        t = _run(S, bound, config.BLEND_T_STOP)
        _check_stop(s, t, name + f" t_stop {config.BLEND_T_STOP}")
        _check_strict_gt(S, bound, config.BLEND_T_STOP, t, name + f" t_stop {config.BLEND_T_STOP}")
        strict[compact] = (s, near)
    dg, dp = _compare_mappings(ref, strict[1][0], strict[0][0], what)
    pairs = sum(int(l[2]) * int(l[3]) * int(l[5]) for l in S["leaves"])
    print(f"[blend mapping] {what} bound {bound}: {len(S['lists'])} leaves, {S['proj'].shape[0]} splats, "
          f"{pairs:.3e} pixel x Gaussian pairs, {S['ties'].size} exact ties; arg-max on f64 near-ties differing: "
          f"compact {strict[1][1]}, strips {strict[0][1]}; compact vs strips below FLT_MIN: {dg} Gaussians, {dp} pixels")


_CACHE = {}


def _shape_grid():
    if "shapes" not in _CACHE:
        rng = np.random.default_rng(1301)
        shapes = [(w, h) for h in HEIGHTS for w in range(2, 65)]
        lengths = []
        for i, (w, h) in enumerate(shapes):
            k = i % len(LENGTHS)
            while k > 0 and w * h * LENGTHS[k] > PAIR_BUDGET:
                k -= 1
            lengths.append(LENGTHS[k])
        S = _frame(rng, shapes, lengths, 1024)
        _CACHE["shapes"] = (S, _reference(S))
    return _CACHE["shapes"]


def _early_exit():
    if "early" not in _CACHE:
        rng = np.random.default_rng(1302)
        kinds = [(40, 23), (20, 11), (37, 13), (64, 33), (9, 6), (17, 31)]
        shapes, lengths, early = [], [], []
        for i in range(480):
            shapes.append(kinds[i % len(kinds)])
            if i % 2 == 0:  # stops in chunk 0 (k0 = 0: first check after 32) or chunk 1 (k0 = 130: check after 160)
                lengths.append(int(rng.integers(260, 520)))
                early.append((i, 0 if i % 4 == 0 else 130))
            else:
                lengths.append(int(rng.integers(1, 200)))
        # launch order: early-exit and ordinary leaves alternate, so CTAs move from one kind straight to the other
        S = _frame(rng, shapes, lengths, 1024, bg=0.25, early=early, order=np.arange(len(shapes)))
        _CACHE["early"] = (S, _reference(S))
    return _CACHE["early"]


@pytest.mark.parametrize("bound", ["tight", "loose"])
@pytest.mark.parametrize("scene", ["shapes", "early"])
def test_blend_mappings_vs_f64(lib, mapping, scene, bound):
    """Every leaf shape up to 64 px (list lengths 0 .. 1999 in rotation, bounded by PAIR_BUDGET), or early-exit leaves
    interleaved with ordinary ones (background 0.25): both mappings, both stop settings, against f64."""
    S, ref = _shape_grid() if scene == "shapes" else _early_exit()
    w, h = S["tight"]
    _all_configs(lib, mapping, S, ref, (w, h) if bound == "tight" else (w + 37, 2 * h + 5), scene)


@pytest.mark.parametrize("wh", WIDE)
def test_wide_short_leaves(lib, mapping, wh):
    """Leaves wider than 160 px with few rows have more blocks across than the 60-px leaves the slab count was first
    sized for: every block must be rendered, under the tightest bound (the leaf's own size) and a loose one."""
    w, h = wh
    rng = np.random.default_rng(1303 + w + h)
    lens = [L for L in LENGTHS if w * h * L <= 600_000][-2:]  # the longest two lists the budget allows
    S = _frame(rng, [wh, wh], lens, w)
    ref = _reference(S)
    for bound in ((w, h), (w + 37, 2 * h + 5)):
        _all_configs(lib, mapping, S, ref, bound, f"{w}x{h}")


# ---- through the renderer ------------------------------------------------------------------------------------------
def _renderer_vs_f64(R, cam, what):
    """Python back-end, strict stop: image and maxima against the f64 leaf blend of the kernel's records and lists
    (test_edges_gpu.test_python_blend_vs_f64_and_tie_order's rules); the recorded colour is the f64 colour of the f64
    arg-max pixel unless the f64 runner-up at another pixel is within 1e-6 (broad, faint splats)."""
    img = R(cam)[0].cpu().numpy()
    proj, leaves = R.debug_last_camera()
    Wd = img.shape[1]
    n = proj.shape[0]
    best, bestpix, second = np.zeros(n), np.full(n, -1, dtype=np.int64), np.zeros(n)
    fimg = np.ones(img.shape)
    for (r0, c0, w, h, gids) in leaves:
        col, con = fr.leaf_blend(r0, c0, w, h, gids, proj)
        ys, xs = np.meshgrid(np.arange(r0, r0 + h), np.arange(c0, c0 + w), indexing="ij")
        fimg[ys.reshape(-1), Wd - 1 - xs.reshape(-1)] = col
        if len(gids):
            ar = np.arange(len(gids))
            am = con.argmax(axis=0)
            v = con[am, ar]
            other = con.copy()
            other[am, ar] = -1.0
            s = other.max(axis=0) if w * h > 1 else 0 * v
            up = v > best[gids]  # strict > over leaves in BFS order, first pixel inside a leaf
            second[gids] = np.where(up, np.maximum(best[gids], s), np.maximum(second[gids], v))
            best[gids[up]], bestpix[gids[up]] = v[up], (ys.reshape(-1) * Wd + xs.reshape(-1))[am[up]]
    derr = np.abs(img - fimg).max()
    assert derr < 2e-5, f"{what}: image vs f64 {derr:.2e}"
    kmax = R.gaussian_max_contribution.cpu().numpy()
    merr = np.abs(kmax - best).max()
    assert merr < 2e-5, f"{what}: maxima vs f64 {merr:.2e}"
    seen = best > 1e-5
    want = fimg[bestpix[seen] // Wd, Wd - 1 - bestpix[seen] % Wd]
    off = np.abs(R.gaussian_colours.cpu().numpy()[seen] - want).max(axis=1) > 2e-5
    near = (best - second < 1e-6)[seen]
    assert not (off & ~near).any(), f"{what}: {int((off & ~near).sum())} arg-max colours off on a clear maximum"
    return img, kmax, len(leaves), derr, merr, int(off.sum())


@pytest.mark.parametrize("wh", [(163, 7), (1280, 13)])
def test_renderer_max_tile_at_image_width(lib, mapping, wh):
    """max_tile_size raised to the image width: the whole image is one wide, short leaf."""
    import camera_handler as ch
    import gauss_render as gr
    from oracle import gaussians as og
    W, H = wh
    sc, _, _ = es.huge(n_field=300, n_huge=1, res=(W, H))
    c2w, k = es.origin_camera(W, H, 0.9 * max(W, H))
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    out = []
    for compact in (1, 0):
        mapping(compact)
        R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov)
        R.t_stop = 0.0
        R.max_tile_size = W
        r = _renderer_vs_f64(R, ch.get_camera("python", c2w.to(DEV), k), f"{W}x{H} compact={compact}")
        assert r[2] == 1, f"expected one leaf, got {r[2]}"
        out.append(r)
        print(f"[blend mapping renderer] {W}x{H} max_tile_size {W} compact={compact}: {r[2]} leaf, image err "
              f"{r[3]:.1e}, max err {r[4]:.1e}, arg-max colours off on f64 near-ties {r[5]}")
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])


def _cap_scene(W=1280, H=720, z=4.0):
    """A dense grid of small splats (4 px apart) over one quarter of the image in front of one large background
    splat: the base leaves under the grid split twice by count, the others stay whole."""
    f = 0.9 * W
    us, vs = np.meshgrid(np.arange(2.0, W / 4, 4.0), np.arange(2.0, H, 4.0))
    xy = np.stack([(us.reshape(-1) - 0.5 * W) * z / f, (vs.reshape(-1) - 0.5 * H) * z / f], 1)
    m = xy.shape[0]
    xyz = np.concatenate([np.c_[xy, np.full(m, -z)], [[0.0, 0.0, -12.0]]])
    ls = np.concatenate([np.log(np.full((m, 3), 0.5 * z / f)), np.log([[40.0, 40.0, 1.0]])])
    rng = np.random.default_rng(1304)
    sc = es._finish(xyz, ls, np.tile([1.0, 0, 0, 0], (m + 1, 1)), np.r_[rng.uniform(0.2, 0.8, m), 0.5], 1304)
    return sc, es.origin_camera(W, H, f)


def test_renderer_above_sort_cap(lib, mapping):
    """More than 4096 leaves: build_tree's launch order falls back to BFS order, and the leaf table selects a smaller
    multisplit chunk.  Image, maxima and arg-max colours against f64 in both mappings."""
    import camera_handler as ch
    import gauss_render as gr
    from oracle import gaussians as og
    sc, (c2w, k) = _cap_scene()
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    out = []
    for compact in (1, 0):
        mapping(compact)
        R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov)
        R.t_stop = 0.0
        R.max_gaussians_per_tile = 18
        r = _renderer_vs_f64(R, ch.get_camera("python", c2w.to(DEV), k), f"sort cap compact={compact}")
        t = R._last_tables
        nl = R.last_stats["num_leaves"]
        assert nl > 4096, f"only {nl} leaves"
        assert t["chunk"] == int(lib.g2pc_multisplit_chunk(t["leaf_cap"])) == 64, (t["leaf_cap"], t["chunk"])
        out.append(r)
        print(f"[blend mapping renderer] sort cap compact={compact}: {nl} leaves (table {t['leaf_cap']}, multisplit "
              f"C = {t['chunk']}), image err {r[3]:.1e}, max err {r[4]:.1e}, arg-max colours off on f64 near-ties {r[5]}")
    assert np.array_equal(out[0][0], out[1][0]) and np.array_equal(out[0][1], out[1][1])
