"""GPU tests of the kernels on adversarial scenes and edge shapes (tests/edge_scenes.py) against plain float64
references (tests/f64ref.py).

Rules, per stage:
  * a float output may be off the f64 value by at most max(c * u * scale, 4 x the float32 oracle's own error): never
    materially worse than the reference's arithmetic;
  * a decision on a threshold must agree with f64 outside a stated band; inside the band flips are counted, printed
    and bounded;
  * integer structure (lists, orders, tie-breaks) is exact;
  * blends are checked stage-wise: the f64 blend is fed the kernel's own projection records and lists.
"""
import numpy as np
import pytest
import torch

import edge_scenes as es
import f64ref as fr
import tiles_harness as th
from util import scene_to

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
U = fr.U32


def _not_worse(name, got, ref32, ref64, scale, c=64.0):
    """|got - f64| <= max(c u scale, 4 |f32 oracle - f64|) elementwise; returns the worst ratio."""
    got, ref32, ref64 = (np.asarray(a, dtype=np.float64) for a in (got, ref32, ref64))
    err = np.abs(got - ref64)
    allow = np.maximum(c * U * np.asarray(scale, dtype=np.float64), 4.0 * np.abs(ref32 - ref64))
    bad = err > allow
    ratio = float((err / np.maximum(allow, 1e-300)).max()) if err.size else 0.0
    assert not bad.any(), f"{name}: {int(bad.sum())} values worse than allowed, worst ratio {ratio:.2f}"
    return ratio


# ---- per-Gaussian kernels ------------------------------------------------------------------------------------------
def test_eigvals_ascending_on_diagonal_inputs(lib):
    """Exactly diagonal covariances take the closed form's p1 == 0 branch; the result must still be ascending (the
    header's contract) and equal the diagonal, through g2pc_eigvals_sym3.  The magnitudes kernel calls the same
    g2pc_eig3_sym (common.cuh); its formula is symmetric in the eigenvalues, so only its values are checked here."""
    import gauss_handler as gh
    cov = es.diagonal_covariances()
    ev = gh.eigvals_sym3(torch.as_tensor(cov, device=DEV)).cpu().numpy()
    want = np.sort(np.diagonal(cov, axis1=1, axis2=2), axis=1)
    assert np.array_equal(ev, want), f"diag(3,1,2) -> {ev[0]}"
    assert (np.diff(ev, axis=1) >= 0).all()
    # the same matrices rotated by an exact permutation stay diagonal; a random rotation leaves the diagonal branch
    sc = es.badly_conditioned("disc", n=513)
    G = gh.Gaussians(*(scene_to(sc, DEV)[k] for k in ("xyz", "scales", "rots", "colours", "opacities")))
    ev2 = gh.eigvals_sym3(G.covariances).cpu().numpy()
    assert (np.diff(ev2, axis=1) >= 0).all(), "eigenvalues not ascending"
    m = cov.shape[0]
    z = torch.zeros((m, 3), device=DEV)
    G = gh.Gaussians(z, z.double(), torch.tensor([[1.0, 0, 0, 0]], device=DEV).repeat(m, 1).double(), z.double(),
                     torch.full((m,), 0.5, device=DEV))
    G.covariances = torch.as_tensor(cov, device=DEV)
    _, mags = G.points_per_gaussian(1000, torch.full((m,), 0.5, device=DEV))
    want_m = fr.magnitudes(cov, np.full(cov.shape[0], 0.5))
    rel = np.abs(mags.cpu().numpy() - want_m) / want_m
    assert rel.max() < 5e-6, f"magnitudes of diagonal covariances: rel err {rel.max():.2e}"


@pytest.mark.parametrize("kind", ["needle", "disc"])
@pytest.mark.parametrize("n", es.SHAPES_N)
def test_per_gaussian_kernels_vs_f64(lib, kind, n):
    """cov_build (f32 / f64 inputs, scale_modifier 1, 0.5, 1.7), normals, eigvals_sym3, magnitudes and the
    non-positive-definite flag on cond(Sigma) 1e6 .. 1e10, at Gaussian counts with partial 256-row tiles."""
    import gauss_handler as gh
    from oracle import gaussians as og
    sc = es.badly_conditioned(kind, n=n)
    d = scene_to(sc, DEV)
    worst = {}
    for mod in (1.0, 0.5, 1.7):
        c64 = fr.covariance(sc["scales"].numpy(), sc["rots"].numpy(), mod)
        c32o = og.build_covariance(sc["scales"], sc["rots"], mod).numpy()
        scale = np.abs(c64).max(axis=(1, 2), keepdims=True) * np.ones((1, 3, 3))
        for dt in (torch.float64, torch.float32):
            got = gh.build_covariance_from_scaling_rotation(d["scales"].to(dt), mod, d["rots"].to(dt)).cpu().numpy()
            ref64 = c64 if dt == torch.float64 else fr.covariance(sc["scales"].float().double().numpy(),
                                                                   sc["rots"].float().double().numpy(), mod)
            ref32 = c32o if dt == torch.float64 else og.build_covariance(sc["scales"].float(), sc["rots"].float(),
                                                                         mod).numpy()
            worst[f"cov mod={mod} {dt}"] = _not_worse("covariance", got, ref32, ref64, scale, c=16)
    G = gh.Gaussians(d["xyz"], d["scales"], d["rots"], d["colours"], d["opacities"])
    G.calculate_normals()
    nrm64 = fr.normals(sc["scales"].numpy(), sc["rots"].numpy())
    nrm_s = np.abs(nrm64).max(axis=1, keepdims=True) * np.ones((1, 3))
    worst["normals"] = _not_worse("normals", G.normals.cpu().numpy(), og.calculate_normals(sc["scales"], sc["rots"]).numpy(),
                                  nrm64, nrm_s, c=4)
    # eigenvalues of the kernel's own f32 matrices against f64 eigvalsh; the f32 oracle is LAPACK's general solver
    cov32 = G.covariances.cpu().numpy()
    ev = gh.eigvals_sym3(G.covariances).cpu().numpy().astype(np.float64)
    ev64 = fr.eigvalsh(cov32)
    ev32 = np.sort(torch.linalg.eigvals(torch.as_tensor(cov32)).real.numpy(), axis=1)
    assert (np.diff(ev, axis=1) >= 0).all(), "eigenvalues not ascending"
    lmax = np.abs(ev64).max(axis=1, keepdims=True) * np.ones((1, 3))
    # the closed form's absolute error is ~0.1 u lambda_max (1e-8 relative on needles): 4 u lambda_max is the fixed arm
    worst["eigvals"] = _not_worse("eigvals", ev, ev32, ev64, lmax, c=4)
    # non_posdef_covariances(eps): flag = any(eig <= eps).  The closed form's smallest eigenvalue carries an absolute
    # error of up to ~1e-8 * lambda_max on needles: inside that band of eps the flag is undetermined, outside exact.
    flips_total = 0
    for eps in (1e-10, 1e-8, 1e-7):
        got = G.non_posdef_covariances(G.covariances, epsilon=eps).cpu().numpy()
        want = (ev64 <= eps).any(axis=1)
        band = np.abs(ev64[:, 0] - eps) <= 1e-7 * lmax[:, 0]
        assert np.array_equal(got[~band], want[~band]), f"non-posdef flag wrong outside the band (eps {eps})"
        flips_total += int((got != want).sum())
    assert flips_total <= max(4, int(0.05 * n)), f"{flips_total} non-posdef flips inside the band"
    # magnitudes are taken after validate_covariances (+5e-7 I, eigen-clamp), as in the pipeline: on the raw needles
    # the smallest eigenvalue may round below zero and its square root is NaN in every implementation
    G.validate_covariances()
    assert G.covariances.shape[0] == n
    cov32 = G.covariances.cpu().numpy()
    ev64 = fr.eigvalsh(cov32)
    lmax = np.abs(ev64).max(axis=1, keepdims=True) * np.ones((1, 3))
    m64 = fr.magnitudes(cov32, sc["opacities"].numpy())
    _, m = G.points_per_gaussian(10 * n, d["opacities"])
    mo = og.gaussian_magnitudes(torch.as_tensor(cov32), sc["opacities"]).numpy()
    # magnitude = sqrt(area): the smallest eigenvalue enters through a * b products, so its relative error matters
    # only as far as it moves the area; same rule against the f32 oracle (LAPACK eigvals)
    # the magnitude's sensitivity to an eigenvalue error of the closed form's size (256 u lambda_max) is allowed on top
    sens = np.zeros(n)
    for sgn in ((1, 1, 1), (-1, 1, 1), (1, -1, 1), (-1, -1, 1)):
        pert = ev64 + np.asarray(sgn)[None, :] * 256 * U * lmax
        sens = np.maximum(sens, np.abs(fr.magnitudes_from_eig(pert, sc["opacities"].numpy()) - m64))
    mk = m.cpu().numpy()
    allow = np.maximum(256 * U * m64 + sens, 4 * np.abs(mo - m64))  # f32 powf / sqrtf chain: a few ulp per step
    bad = np.abs(mk - m64) > allow
    assert not bad.any(), f"magnitudes: {int(bad.sum())} worse than allowed, e.g. {mk[bad][:3]} vs f64 {m64[bad][:3]}"
    worst["magnitudes"] = float((np.abs(mk - m64) / allow).max())
    print(f"[edge per-gaussian] {kind} n={n}: worst err / allowed " +
          ", ".join(f"{k} {v:.2f}" for k, v in worst.items()) + f"; non-posdef flips in band {flips_total}")


def test_cholesky_ladder_levels_and_samples(lib):
    """The per-Gaussian regularise-and-retry ladder (Sigma + k 1e-6 I, k = 0, 1, 2): the level each covariance needs is
    predicted in f64 for inputs clearly on one side of each step, the status words G2PC_ST_CHOLREG / G2PC_ST_CHOLFAIL
    must equal the predicted counts, and the samples x = mu + L eps (kernel's eps) must match f64 Cholesky of the
    regularised matrix at the predicted level."""
    from g2pc import capi, config, sampler
    import gauss_to_pc as g2p
    rng = np.random.default_rng(5)
    rows = []
    for lam_min, count in ((1e-4, 40), (-4e-7, 30), (-1.5e-6, 20), (-6e-6, 10)):
        for _ in range(count):
            q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
            ev = np.array([lam_min, rng.uniform(1e-4, 1e-3), rng.uniform(1e-3, 1e-2)])
            rows.append((q * ev) @ q.T)
    cov = np.asarray(rows, dtype=np.float32)
    cov = 0.5 * (cov + cov.transpose(0, 2, 1))
    lvl, L, margin = fr.cholesky_ladder(cov)
    n = cov.shape[0]
    assert (margin > 64 * U).all(), "inputs chosen too close to a ladder step"
    xyz = torch.as_tensor(rng.uniform(-1, 1, (n, 3)), dtype=torch.float32, device=DEV)
    k, seed, call = 8, 77, 5
    dummy = torch.zeros((n, 3), dtype=torch.float32, device=DEV)
    pts, _, _, total, status, _ = g2p._single_bin_run(k, xyz, torch.as_tensor(cov, device=DEV), dummy, None,
                                                      float("inf"), 1, False, seed, call, cull_mode=capi.CULL_EPS_NORM)
    st = status.tolist()
    want_reg, want_fail = int(((lvl > 0) & (lvl < 3)).sum()), int((lvl == 3).sum())
    print(f"[edge cholesky] levels {np.bincount(lvl, minlength=4).tolist()}, status reg {st[capi.ST_CHOLREG]} "
          f"fail {st[capi.ST_CHOLFAIL]}")
    assert st[capi.ST_CHOLREG] == want_reg and st[capi.ST_CHOLFAIL] == want_fail
    t = int(total.item())
    okg = np.nonzero(lvl < 3)[0]
    assert t == k * okg.shape[0]
    got = pts[:t].view(okg.shape[0], k, 3).cpu().numpy().astype(np.float64)
    eps = sampler.dump_eps(torch.as_tensor(okg, device=DEV), k, 0, seed, call).cpu().numpy().astype(np.float64)
    want = xyz.cpu().numpy()[okg][:, None, :] + np.einsum("gij,kgj->gki", L[okg], eps)
    err = np.abs(got - want)
    assert err.max() < 2e-5, f"samples differ from f64 Cholesky at the predicted level: {err.max():.2e}"


# ---- projection ----------------------------------------------------------------------------------------------------
def test_preprocess_camera_inside_both_backends(lib):
    """Camera inside the cloud: probes at exact view depths around both near culls and behind the camera.  The
    in-front / near-cull decisions are exact (the view depth is exact in f32 for this camera); mean, conic and radius
    against f64 under the not-worse-than-f32 rule, radius ceil flips only where its argument is within 1e-5 of an
    integer."""
    import camera_handler as ch
    import gauss_render as gr
    from g2pc.rasterizer import GaussianRasterizer
    from oracle import gaussians as og, render as orr, render_cuda as orc
    sc, cams, intr, pidx, pdep = es.inside()
    cov = og.build_covariance(sc["scales"], sc["rots"])
    d = scene_to(sc, DEV)
    xyz, c32 = sc["xyz"].numpy(), cov.numpy()
    # python back-end: in front <=> z_view <= -1e-6 (f32 compare)
    R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov.to(DEV))
    R.t_stop = 0.0
    R(ch.get_camera("python", cams[0].to(DEV), intr[0]))
    proj, _ = R.debug_last_camera()
    ocam = orr.Camera(cams[0], intr[0])
    f = fr.project_python(xyz, c32, ocam)
    vis = proj[:, 11] > 0
    assert np.array_equal(vis, f["z"] <= np.float32(-1e-6)), "python back-end in-front decision"
    assert np.array_equal(vis[pidx], pdep >= np.float32(1e-6))
    o = orr.project(sc["xyz"], cov, ocam)
    sel = vis & (f["z"] < -1e-4) & np.isfinite(f["mx"])
    W, H = ocam.image_width, ocam.image_height
    worst = {}
    for key, col in (("mx", 0), ("my", 1)):
        worst[key] = _not_worse(key, proj[sel, col], o[key].numpy()[sel], f[key][sel],
                                np.maximum(np.abs(f[key][sel]), max(W, H)), c=64)
    oconic = torch.inverse(o["cov2d"]).numpy()
    cs = np.abs(f["conic"][sel]).max(axis=(1, 2))
    for name, col, a, b in (("c00", 2, 0, 0), ("c11", 4, 1, 1)):
        worst[name] = _not_worse(name, proj[sel, col] / fr.K_EXP2, oconic[sel, a, b], f["conic"][sel, a, b], cs, c=256)
    arg = f["sqrt_lmax"][sel]
    band = np.abs(arg - np.round(arg)) <= 1e-5 * arg
    rad64 = 3.0 * np.ceil(arg)
    flips_py = int((proj[sel, 10] != rad64).sum())
    assert np.array_equal(proj[sel, 10][~band], rad64[~band]), "python back-end radius != 3 ceil(sqrt(lambda_max))"
    # CUDA back-end: ok <=> z_view > 0.2 (f32 compare) and a non-empty tile rect
    rs = ch.get_camera("cuda", cams[0].to(DEV), intr[0])
    Rc = GaussianRasterizer(d["xyz"], None, d["opacities"], colors_precomp=d["colours"].float(), cov3D_precomp=cov.to(DEV))
    _, radii, _, _ = Rc(rs)
    rec = Rc._slots[Rc._last_slot]["proj"].cpu().numpy()
    keyok = Rc._slots[Rc._last_slot]["depth_key"].cpu().numpy().view(np.uint32) != 0xFFFFFFFF
    ors = orc.RasterSettings(cams[0], intr[0])
    g = fr.preprocess_cuda(xyz, c32, ors)
    near = g["z"] > np.float32(0.2)
    assert not (keyok & ~near).any(), "CUDA back-end kept a Gaussian at or before the near plane"
    assert np.array_equal(keyok[pidx], pdep > np.float32(0.2)), "CUDA back-end near cull on the probes"
    oc = orc.preprocess(xyz, c32, ors)
    okc = keyok & np.isfinite(g["px"])
    worst["px"] = _not_worse("px", rec[okc, 0], oc["px"][okc], g["px"][okc], np.maximum(np.abs(g["px"][okc]), ors.image_width))
    arg = g["three_sigma"][okc]
    band = np.abs(arg - np.round(arg)) <= 1e-5 * arg
    flips_cu = int((rec[okc, 10] != np.ceil(arg)).sum())
    assert np.array_equal(rec[okc, 10][~band], np.ceil(arg)[~band]), "CUDA back-end radius != ceil(3 sqrt(lambda_max))"
    assert np.array_equal(radii.cpu().numpy()[okc], rec[okc, 10].astype(np.int32))
    print(f"[edge inside] python: {int(vis.sum())} in front, radius flips in band {flips_py}; cuda: {int(keyok.sum())} "
          f"kept, radius flips in band {flips_cu}; worst err / allowed " + ", ".join(f"{k} {v:.2f}" for k, v in worst.items()))


# ---- opacity edges -------------------------------------------------------------------------------------------------
def test_opacity_clamp_and_alpha_skip(lib):
    """Gaussian i alone on the optical axis of camera i, centred on a pixel centre (power exactly 0): with T = 1 its
    maximum contribution is its alpha.  The python back-end has no alpha skip, so it reports the kernel's f32 alpha
    min(0.99, exp2(log2 o)) for every opacity; the CUDA back-end must report exactly that alpha when alpha >= 1/255
    and 0 when alpha < 1/255, and nothing may exceed the 0.99 clamp."""
    import camera_handler as ch
    import gauss_render as gr
    from g2pc.rasterizer import GaussianRasterizer
    from oracle import gaussians as og
    sc, cams, intr = es.opacity()
    cov = og.build_covariance(sc["scales"], sc["rots"]).to(DEV)
    d = scene_to(sc, DEV)
    n = len(cams)
    Rp = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov)
    Rp.t_stop = 0.0
    Rc = GaussianRasterizer(d["xyz"], None, d["opacities"], colors_precomp=d["colours"].float(), cov3D_precomp=cov)
    W = intr[0][0]
    for i, (c2w, k) in enumerate(zip(cams, intr)):
        Rp(ch.get_camera("python", c2w.to(DEV), k))
        Rc(ch.get_camera("cuda", c2w.to(DEV), k))
        if i == 0:
            rec = Rc._slots[Rc._last_slot]["proj"].cpu().numpy()
            assert rec[0, 0] == (W - 1) / 2 and rec[0, 1] == (k[1] - 1) / 2, "probe not on a pixel centre"
    a_py = Rp.gaussian_max_contribution.cpu().numpy()
    a_cu = Rc.gaussian_max_contribution.cpu().numpy()
    o = sc["opacities"].numpy().astype(np.float64)
    thr = np.float32(1.0 / 255.0)
    assert a_py.max() <= np.float32(0.99) and a_cu.max() <= np.float32(0.99), "alpha above the 0.99 clamp"
    # f64: alpha = min(0.99, o); the kernel's exp2(log2 o) is off by a few ulp
    rel = np.abs(a_py - np.minimum(o, 0.99)) / np.minimum(o, 0.99)
    assert rel.max() < 2e-6, f"python back-end alpha vs f64: {rel.max():.2e}"
    want_cu = np.where(a_py >= thr, a_py, np.float32(0))
    assert np.array_equal(a_cu, want_cu), \
        f"CUDA back-end alpha skip: {int((a_cu != want_cu).sum())} of {n} differ from keep iff alpha >= 1/255"
    on_thr = int((a_py == thr).sum())
    # only an alpha of exactly 1/255 separates `alpha < 1/255` from `alpha <= 1/255`: the sweep must reach it
    assert on_thr > 0, "no f32 alpha of the sweep equals 1/255: widen alpha_sweep()"
    flips = int(((a_cu > 0) != (o >= 1.0 / 255.0)).sum())
    print(f"[edge opacity] {n} opacities: f32 alpha exactly 1/255 for {on_thr}; skip decisions differing from f64 "
          f"o >= 1/255 (all within {es.alpha_sweep().shape[0] // 2} ulp): {flips}")


# ---- blends, stage-wise --------------------------------------------------------------------------------------------
def _cuda_setup(sc, cams, intr, surf=True):
    return th.cuda_setup(sc, surf)


def _tiles_camera(R, rs):
    o = th.tiles_camera(R, rs)
    return tuple(o[k] for k in ("image", "depth", "rec", "ok", "contrib", "pixel", "surface"))


@pytest.mark.parametrize("family", ["huge", "ties", "inside"])
def test_tiles_blend_vs_f64(lib, family):
    """CUDA back-end blend fed its own records against the f64 blend: images and per-Gaussian maxima within 2e-5, the
    arg-max pixel equal (lowest id among exact ties), surface distances over several 256-entry rounds; skip / stop
    decisions inside the f32 band are counted and their pixels excluded."""
    import camera_handler as ch
    scene = {"huge": es.huge, "ties": es.ties, "inside": lambda: es.inside()[:3]}[family]
    sc, cams, intr = scene()
    R, d, cov = _cuda_setup(sc, cams, intr)
    rs = ch.get_camera("cuda", cams[0].to(DEV), intr[0])
    W, H = int(rs.image_width), int(rs.image_height)
    img, dep, rec, ok, contrib, pix, surf = _tiles_camera(R, rs)
    f = fr.tiles_blend(rec, ok, W, H, [1.0, 1.0, 1.0])
    good = np.isfinite(f["image"])
    derr = np.abs(img - f["image"])[good]
    n_taint_px = int((~good[0]).sum())
    assert n_taint_px <= max(4, int(2e-2 * W * H)), f"{n_taint_px} pixels with a decision in the f32 band"
    assert derr.max() < 2e-5, f"image vs f64: {derr.max():.2e}"
    dd = np.abs(dep - f["depth"])[good[0]] / np.maximum(1.0, np.abs(f["depth"][good[0]]))
    assert dd.max() < 5e-5, f"depth vs f64: {dd.max():.2e}"
    clean = ~f["taint"]
    cerr = np.abs(contrib - f["contrib"])[clean]
    assert cerr.max() < 2e-5, f"max contribution vs f64: {cerr.max():.2e}"
    # arg-max: equal pixel unless the f64 runner-up (another pixel) is within 1e-6 of the maximum (declared near-tie)
    seen = clean & (f["contrib"] > 0)
    differ = seen & (pix != f["pixel"])
    near = f["contrib"] - f["second"] < 1e-6
    assert not (differ & ~near).any(), f"{int((differ & ~near).sum())} arg-max pixels differ on a clear maximum"
    near_ties = int(differ.sum())
    if family == "ties":
        front = sc["xyz"].shape[0] - 2  # the splat centred between two pixels
        assert f["pixel"][front] == (H // 2 - 1) * W + (W // 2 - 1), "the front splat should tie four pixels"
        assert pix[front] == f["pixel"][front], f"exact tie resolved to pixel {pix[front]}, want {f['pixel'][front]}"
    fin = (surf < 3e38) & np.isfinite(f["surface"]) & ~f["surf_taint"]
    serr = np.abs(surf - f["surface"])[fin] / np.maximum(1.0, np.abs(f["surface"][fin]))
    assert int(((surf < 3e38) != np.isfinite(f["surface"]))[~f["surf_taint"]].sum()) == 0, "surface distance coverage"
    assert fin.sum() == 0 or serr.max() < 5e-5, f"surface distance vs f64: {serr.max():.2e}"
    if family == "huge":
        assert f["list_max"] > 1000 and f["rounds_max"] >= 4, (f["list_max"], f["rounds_max"])
    print(f"[edge tiles {family}] {W}x{H}: longest list {f['list_max']} ({f['rounds_max']} rounds), decisions in band "
          f"skip {f['skip_band']} stop {f['stop_band']} -> {n_taint_px} pixels excluded; image err {derr.max():.1e}, "
          f"contrib err {cerr.max():.1e}, arg-max differing {near_ties} of {int((seen & near).sum())} near-ties, surface err {serr.max() if fin.any() else 0:.1e}")


@pytest.mark.parametrize("family", ["huge", "ties"])
def test_accumulators_async_idempotent_and_rerun_exact(lib, family):
    """On the huge and ties scenes: three passes over the same camera leave the maximum, its colour and the minimum
    surface distance of one pass unchanged (strict > / min updates); with async_mode and a tiny instance buffer (the
    frame is replayed) the accumulators equal the synchronous run bit for bit, and a fresh renderer reproduces them."""
    import camera_handler as ch
    sc, cams, intr = {"huge": es.huge, "ties": es.ties}[family]()
    out = []
    for mode, passes in (("sync", 1), ("sync", 3), ("async", 3), ("async", 3)):
        R, d, cov = _cuda_setup(sc, cams, intr)
        if mode == "async":
            R.async_mode = True
            R._inst_cap = 16
        for _ in range(passes):
            R(ch.get_camera("cuda", cams[0].to(DEV), intr[0]))
        R.flush()
        if mode == "async":
            assert R.replays >= 1, "the tiny instance buffer did not force a replay"
        out.append((R.gaussian_max_contribution.clone(), R.gaussian_colours.clone(),
                    R.gaussian_min_surface_distance.clone(), R.gaussian_total_contribution.clone()))
    for a, b in zip(out[0][:3], out[1][:3]):
        assert torch.equal(a, b), "a second pass over the same camera changed an accumulator"
    for a, b in zip(out[1], out[2]):
        assert torch.equal(a, b)
    for a, b in zip(out[2], out[3]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("family", ["huge", "ties", "inside"])
def test_python_blend_vs_f64_and_tie_order(lib, family):
    """Python back-end: per-leaf lists are depth-ordered with exact ties by index, and the blend fed the kernel's
    records and lists matches the f64 leaf blend (image and max contributions within 2e-5, the colour of the arg-max
    pixel — lowest pixel id among exact ties)."""
    import camera_handler as ch
    import gauss_render as gr
    from oracle import gaussians as og
    sc, cams, intr = {"huge": es.huge, "ties": es.ties, "inside": lambda: es.inside()[:3]}[family]()
    cov = og.build_covariance(sc["scales"], sc["rots"])
    d = scene_to(sc, DEV)
    R = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov.to(DEV))
    R.t_stop = 0.0
    img, _, _, _ = R(ch.get_camera("python", cams[0].to(DEV), intr[0]))
    img = img.cpu().numpy()
    proj, leaves = R.debug_last_camera()
    Wd = img.shape[1]
    depth = proj[:, 9]
    n = proj.shape[0]
    best = np.zeros(n)
    bestpix = np.full(n, -1, dtype=np.int64)
    fimg = np.full(img.shape, 1.0)
    ties_seen = 0
    for (r0, c0, w, h, gids) in leaves:
        order = np.lexsort((gids, -depth[gids]))
        assert np.array_equal(gids[order], gids), "leaf list not depth-ordered with ties by index"
        ties_seen += int((np.diff(depth[gids]) == 0).sum())
        col, con = fr.leaf_blend(r0, c0, w, h, gids, proj)
        ys, xs = np.meshgrid(np.arange(r0, r0 + h), np.arange(c0, c0 + w), indexing="ij")
        fimg[ys.reshape(-1), Wd - 1 - xs.reshape(-1)] = col
        pid = (ys * Wd + xs).reshape(-1)
        for j, g in enumerate(gids):
            # leaves in BFS order, strict > across leaves, first pixel (row-major) inside a leaf
            v = con[:, j].max()
            if v > best[g]:
                best[g], bestpix[g] = v, pid[int(np.argmax(con[:, j]))]
    derr = np.abs(img - fimg)
    assert derr.max() < 2e-5, f"image vs f64: {derr.max():.2e}"
    kmax = R.gaussian_max_contribution.cpu().numpy()
    assert np.abs(kmax - best).max() < 2e-5
    # the recorded colour is the blended colour at the arg-max pixel (f64 image, lowest pixel id among exact ties)
    kcol = R.gaussian_colours.cpu().numpy()
    seen = best > 1e-5
    ys, xs = bestpix[seen] // Wd, bestpix[seen] % Wd
    want = fimg[ys, Wd - 1 - xs]
    cerr = np.abs(kcol[seen] - want).max(axis=1)
    n_off = int((cerr > 2e-5).sum())
    assert n_off <= max(1, int(1e-3 * seen.sum())), f"{n_off} arg-max colours off"
    if family == "ties":
        assert ties_seen > 0
        front = n - 2
        assert cerr[np.nonzero(seen)[0] == front].max() < 2e-5, "exact tie not resolved to the lowest pixel id"
    print(f"[edge python blend {family}] leaves {len(leaves)}, exact depth ties in lists {ties_seen}, image err "
          f"{derr.max():.1e}, colours off {n_off}")


# ---- shapes --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wh", es.SHAPES_WH)
def test_small_and_thin_images(lib, wh):
    """Partial / one-pixel-wide tiles, super-tiles and quadtree leaves: CUDA back-end against the f64 blend fed its
    records, python back-end leaf list against the quadtree oracle fed the kernel's floats (exact) and its blend
    against f64."""
    import camera_handler as ch
    import gauss_render as gr
    from oracle import gaussians as og, render as orr
    W, H = wh
    sc, _, _ = es.huge(n_field=300, n_huge=1, res=(W, H))
    c2w, k = es.origin_camera(W, H, 0.9 * max(W, H))
    R, d, cov = _cuda_setup(sc, [c2w], [k])
    rs = ch.get_camera("cuda", c2w.to(DEV), k)
    img, dep, rec, ok, contrib, pix, surf = _tiles_camera(R, rs)
    f = fr.tiles_blend(rec, ok, W, H, [1.0, 1.0, 1.0])
    good = np.isfinite(f["image"])
    assert np.abs(img - f["image"])[good].max() < 2e-5
    assert np.abs(contrib - f["contrib"])[~f["taint"]].max() < 2e-5
    Rp = gr.get_renderer("python", d["xyz"], d["opacities"].unsqueeze(1), d["colours"], cov.to(DEV))
    Rp.t_stop = 0.0
    if min(W, H) < 2:
        # known divergence: the reference's quadtree drops nodes one pixel wide (gauss_render.py:297) and renders only
        # the background; this back-end has no leaf-candidate level to tabulate and refuses the camera
        from g2pc import capi
        with pytest.raises(capi.G2pcError, match="level_mask"):
            Rp(ch.get_camera("python", c2w.to(DEV), k))
        print(f"[edge shapes] {W}x{H}: cuda list max {f['list_max']}, python back-end refuses the camera")
        return
    pimg, _, _, _ = Rp(ch.get_camera("python", c2w.to(DEV), k))
    proj, kleaves = Rp.debug_last_camera()
    vid = np.nonzero(proj[:, 11] > 0)[0]
    f32 = np.float32
    mx, my, rad = proj[vid, 0], proj[vid, 1], proj[vid, 10]
    rx0, rx1 = np.clip(mx - rad, f32(0), f32(W - 1)), np.clip(mx + rad, f32(0), f32(W - 1))
    ry0, ry1 = np.clip(my - rad, f32(0), f32(H - 1)), np.clip(my + rad, f32(0), f32(H - 1))
    oleaves, _ = orr.quadtree_leaves(W, H, rx0, ry0, rx1, ry1, Rp.max_tile_size, Rp.max_gaussians_per_tile)
    assert [tuple(a[:4]) for a in oleaves] == [tuple(a[:4]) for a in kleaves], "leaf list"
    pimg = pimg.cpu().numpy()
    fimg = np.ones_like(pimg, dtype=np.float64)
    for (r0, c0, w, h, members), (_, _, _, _, gids) in zip(oleaves, kleaves):
        assert np.array_equal(np.sort(vid[members]), np.sort(gids)), "per-leaf index set"
        col, _ = fr.leaf_blend(r0, c0, w, h, gids, proj)
        ys, xs = np.meshgrid(np.arange(r0, r0 + h), np.arange(c0, c0 + w), indexing="ij")
        fimg[ys.reshape(-1), W - 1 - xs.reshape(-1)] = col
    assert np.abs(pimg - fimg).max() < 2e-5
    print(f"[edge shapes] {W}x{H}: cuda list max {f['list_max']}, python leaves {len(kleaves)}")


def test_super_tile_sort_cap_fallback(lib):
    """More than 8192 super-tiles (CUDA back-end, 4096x2304) switch the list table to launch order instead of the
    heaviest-first sort.  The blend must not depend on the order tiles run in: image, per-Gaussian maxima and arg-max
    pixels against the f64 blend of the kernel's records, as under the cap."""
    import camera_handler as ch
    # CUDA back-end: a handful of splats, most tiles empty
    W, H = 4096, 2304
    rng = np.random.default_rng(3)
    m = 40
    z = rng.uniform(3, 5, m)
    xyz = np.stack([rng.uniform(-0.5, 0.5, m) * z, rng.uniform(-0.3, 0.3, m) * z, -z], 1)
    sc = es._finish(xyz, np.log(rng.uniform(0.002, 0.01, (m, 3))), rng.normal(size=(m, 4)), rng.uniform(0.3, 0.9, m), 3)
    c2w, k = es.origin_camera(W, H, 0.9 * W)
    R, d, cov = _cuda_setup(sc, [c2w], [k], surf=False)
    assert R._res_tables(W, H)["ntiles"] > 8192
    img, dep, rec, ok, contrib, pix, surf = _tiles_camera(R, ch.get_camera("cuda", c2w.to(DEV), k))
    f = fr.tiles_blend(rec, ok, W, H, [1.0, 1.0, 1.0], surface=False)
    good = np.isfinite(f["image"])
    assert np.abs(img - f["image"])[good].max() < 2e-5
    assert np.abs(contrib - f["contrib"])[~f["taint"]].max() < 2e-5
    assert np.array_equal(pix[~f["taint"] & (f["contrib"] > 0)], f["pixel"][~f["taint"] & (f["contrib"] > 0)])
    print(f"[edge sort cap] cuda back-end {R._res_tables(W, H)['ntiles']} super-tiles, {int(ok.sum())} splats")
