"""CPU self-tests of the float64 restatements the CUDA back-end tests lean on (tests/f64ref.py): the masked tile blend,
the SH polynomial and the fold over cameras."""
import math

import numpy as np
import torch

import edge_scenes as es
import f64ref as fr


def _records(sc, rs):
    """Projection records in the kernel's layout (csrc/s7_tiles.cu), from the float32 oracle's preprocess."""
    from oracle import gaussians as og, render_cuda as orc
    cov = og.build_covariance(sc["scales"], sc["rots"]).numpy()
    pre = orc.preprocess(sc["xyz"].numpy(), cov, rs)
    n = cov.shape[0]
    K = np.float32(fr.K_EXP2)
    rec = np.zeros((n, 12), dtype=np.float32)
    rec[:, 0], rec[:, 1] = pre["px"], pre["py"]
    rec[:, 2], rec[:, 3], rec[:, 4] = pre["conic"][:, 0] * K, 2 * pre["conic"][:, 1] * K, pre["conic"][:, 2] * K
    rec[:, 5] = np.log2(sc["opacities"].numpy())
    rec[:, 6:9] = sc["colours"].numpy()
    rec[:, 9], rec[:, 10] = pre["depth"], pre["radius"]
    bits = pre["rx0"] | ((pre["rx1"] - 1) << 8) | (pre["ry0"] << 16) | ((pre["ry1"] - 1) << 24)
    rec[:, 11] = np.where(pre["ok"], bits, 0).astype(np.uint32).view(np.float32)
    return rec, pre["ok"], pre


def test_tiles_blend_masks():
    """An all-ones mask equals no mask; an all-zeros mask writes nothing and records no surface distance; with the
    right and bottom partial tiles and an interior tile masked out the f64 blend agrees with the float32 oracle (image,
    depth, inverse depth, and surface distances defined on the same Gaussians): such tiles leave before round 0."""
    from oracle import render_cuda as orc
    W, H = 40, 23
    sc, cams, intr = es.huge(n_field=300, n_huge=1, res=(W, H))
    rs = orc.RasterSettings(cams[0], intr[0])
    rec, ok, pre = _records(sc, rs)
    bg = [1.0, 1.0, 1.0]
    f0 = fr.tiles_blend(rec, ok, W, H, bg)
    f1 = fr.tiles_blend(rec, ok, W, H, bg, mask=np.ones((H, W), np.int32))
    for key in ("image", "depth", "invdepth", "contrib", "pixel", "surface", "taint", "surf_taint"):
        assert np.array_equal(f0[key], f1[key], equal_nan=True), key
    assert f0["rounds_max"] >= 2
    fz = fr.tiles_blend(rec, ok, W, H, bg, mask=np.zeros(W * H, np.int32))
    assert not fz["image"].any() and not fz["depth"].any() and not fz["invdepth"].any() and not fz["contrib"].any()
    assert not np.isfinite(fz["surface"]).any() and fz["rounds_max"] == 0
    m = np.ones((H, W), np.int32)
    m[:, 32:] = 0
    m[16:, :] = 0
    m[0:16, 0:16] = 0  # only tile (1, 0) stays
    rsm = orc.RasterSettings(cams[0], intr[0], mask=m)
    fm = fr.tiles_blend(rec, ok, W, H, bg, mask=m)
    o = orc.render(pre, sc["opacities"].numpy(), sc["colours"].numpy().astype(np.float32), rsm, True)
    good = np.isfinite(fm["image"][0])
    assert np.abs(fm["image"] - o["image"])[:, good].max() < 1e-5
    assert np.abs(fm["depth"] - o["depth"])[good].max() < 1e-4
    assert np.abs(fm["invdepth"] - o["invdepth"])[good].max() < 1e-5
    assert not fm["image"][:, m == 0].any()
    assert np.array_equal(np.isfinite(fm["surface"]), o["surface"] < 3e38)
    assert np.isfinite(fm["surface"]).sum() < np.isfinite(f0["surface"]).sum()


def test_sh_polynomial():
    """Degree 0 is C0 s + 0.5 with C0 = 1 / (2 sqrt(pi)), clamped at 0; degree 1 is sqrt(3 / (4 pi)) (-y, z, -x); degrees
    0..3 agree with the float32 oracle within 8 u sum|term| in both layouts."""
    from oracle import render as orr
    rng = np.random.default_rng(1)
    d = rng.normal(size=(400, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    s = rng.normal(0, 1.5, size=(400, 3, 16))
    got, bound = fr.sh_colour(0, s, d)
    assert np.allclose(got, np.maximum(s[:, :, 0] / (2 * math.sqrt(math.pi)) + 0.5, 0), rtol=0, atol=1e-15)
    assert (got == 0).any() and (bound >= 0.5).all()
    c1 = math.sqrt(3 / (4 * math.pi))
    s1 = np.zeros_like(s[:, :, :4])
    s1[:, :, 1:] = rng.normal(size=(400, 3, 3))
    want = c1 * (-d[:, 1:2] * s1[:, :, 1] + d[:, 2:3] * s1[:, :, 2] - d[:, 0:1] * s1[:, :, 3]) + 0.5
    assert np.allclose(fr.sh_colour(1, s1, d)[0], np.maximum(want, 0), rtol=0, atol=1e-14)
    for deg in range(4):
        o = orr.sh_colour(deg, torch.as_tensor(s).float(), torch.as_tensor(d).float()).numpy()
        for layout, coef in ((0, s), (1, s.transpose(0, 2, 1))):
            g, b = fr.sh_colour(deg, coef.astype(np.float32), d.astype(np.float32), layout)
            assert (np.abs(g - o) <= 8 * fr.U32 * b).all(), (deg, layout)


def test_accumulate_strict_max_and_ties():
    """The fold keeps the first camera on an exact tie (and its image's colour), moves to a later camera only on a
    strictly larger maximum, sums the maxima, takes the minimum distance, carries taint and flags near-ties."""
    n, H, W = 4, 2, 3

    def cam(contrib, pixel, value, surface, taint=None):
        img = np.full((3, H, W), value, dtype=np.float64)
        return dict(image=img, contrib=np.asarray(contrib, float), pixel=np.asarray(pixel), second=np.zeros(n),
                    taint=np.zeros(n, bool) if taint is None else np.asarray(taint, bool),
                    surface=np.asarray(surface, float),
                    surf_taint=np.zeros(n, bool))

    a = cam([0.5, 0.5, 0.3, 0.0], [1, 2, 3, 0], 1.0, [1.0, np.inf, 2.0, np.inf])
    b = cam([0.5, 0.5 + 5e-7, 0.3 + 1e-3, 0.0], [4, 5, 0, 0], 0.25, [3.0, 0.5, np.inf, np.inf], [0, 0, 0, 1])
    acc = fr.accumulate([a, b])
    assert acc["winner"].tolist() == [0, 1, 1, -1]
    assert acc["colour"][0].tolist() == [1.0, 1.0, 1.0] and acc["colour"][2].tolist() == [0.25, 0.25, 0.25]
    assert acc["near_tie"].tolist() == [False, True, False, False]
    assert np.allclose(acc["total"], [1.0, 1.0 + 5e-7, 0.601, 0.0])
    assert acc["surface"].tolist() == [1.0, 0.5, 2.0, np.inf]
    assert acc["taint"].tolist() == [False, False, False, True]
