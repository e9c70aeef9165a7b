"""Seeded edge-case scenes for the kernel tests (CPU only, like g2pc.synth).

`synth.make_scene` draws every Gaussian from one benign distribution: small splats on a shell seen from 4.5 units away.
The families here reach the code paths that distribution never does.  Each returns the dict layout of
`synth.make_scene` (xyz f32, scales f64 log-space, rots f64, opacities f32, shs f64, colours f64) plus the cameras that
provoke the case, as (list of 4x4 c2w f32, list of [w, h, fx, fy]).

    inside    camera at the origin, looking down -z, inside a shell; probes at exact view depths around both near culls
              (python back-end: z_view <= -1e-6, CUDA back-end: z_view > 0.2) and behind the camera
    huge      a few splats larger than the frustum over a dense field: per-tile lists of well over 1000 entries
    ties      k exact copies (same xyz, covariance, opacity; different colours) and a splat centred between two pixels
    opacity   opacities at and above the 0.99 clamp and a sweep of f32 values around 1/255
    needle    scales spread over 1e-1 .. 1e-5, identity / axis-aligned / random non-normalised quaternions
    disc      as needle, with two large and one tiny axis
The image sizes and Gaussian counts of the `shapes` family are the constants below.
"""
import numpy as np
import torch

from g2pc import synth

# images whose 16x16 tiles, 32x32 super-tiles or quadtree leaves are partial or one pixel wide
SHAPES_WH = [(17, 9), (33, 31), (1, 40), (40, 1), (65, 17)]
# tail lanes that shadow the last Gaussian and partial 256-row tiles of the per-Gaussian kernels
SHAPES_N = [1, 31, 257, 1023, 1025]

# exact view depths of the `inside` probes (python back-end view z = -d, CUDA back-end view z = +d)
F32 = np.float32
_E6, _P2 = F32(1e-6), F32(0.2)
INSIDE_DEPTHS = [F32(1e-3), np.nextafter(_E6, F32(0)), _E6, np.nextafter(_E6, F32(1)), F32(0.15), F32(0.19),
                 F32(0.195), np.nextafter(_P2, F32(0)), _P2, np.nextafter(_P2, F32(1)), F32(0.205), F32(0.25),
                 F32(0.5), F32(1.0)]


def _finish(xyz, log_scales, rots, opac, seed, sh_degree=0):
    g = torch.Generator().manual_seed(seed + 7)
    n = xyz.shape[0]
    ncoef = (sh_degree + 1) ** 2
    shs = 0.05 * torch.randn(n, 3, ncoef, generator=g)
    shs[:, :, 0] = 0.8 * torch.randn(n, 3, generator=g)
    colours = (synth.SH_C0 * shs[:, :, 0].double() + 0.5).clip(0, 1)
    return {"xyz": torch.as_tensor(np.asarray(xyz, dtype=np.float32)).contiguous(),
            "scales": torch.as_tensor(np.asarray(log_scales, dtype=np.float64)),
            "rots": torch.as_tensor(np.asarray(rots, dtype=np.float64)),
            "opacities": torch.as_tensor(np.asarray(opac, dtype=np.float32)).contiguous(),
            "shs": shs.double(), "colours": colours}


def origin_camera(w, h, f):
    """Camera at the origin looking down -z (identity c2w): view-space z equals world z exactly in both back-ends."""
    return torch.eye(4, dtype=torch.float32), [w, h, float(f), float(f)]


def inside(n_shell=1500, seed=11, res=(96, 64)):
    """Camera inside a shell of radius 1.5, probes at exact depths INSIDE_DEPTHS (lateral offsets inside the view)
    and a few Gaussians behind the camera.  Returns (scene, cams, intr, probe_index, probe_depth)."""
    sc = synth.make_scene(n_shell, seed=seed, sh_degree=0)
    rng = np.random.default_rng(seed)
    xyz = [sc["xyz"].numpy()]
    ls = [sc["scales"].numpy()]
    rq = [sc["rots"].numpy()]
    op = [sc["opacities"].numpy()]
    probes = []
    for d in INSIDE_DEPTHS:
        for lat in (0.0, 0.25):
            probes.append((lat * d, -0.5 * lat * d, -d))
    for k in range(6):  # behind the camera
        probes.append((rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(0.05, 1.0)))
    probes = np.asarray(probes, dtype=np.float32)
    m = probes.shape[0]
    xyz.append(probes)
    ls.append(np.log(np.full((m, 3), 0.01)) + rng.normal(0, 0.3, (m, 3)))
    rq.append(rng.normal(size=(m, 4)))
    op.append(np.full(m, 0.8))
    scene = _finish(np.concatenate(xyz), np.concatenate(ls), np.concatenate(rq), np.concatenate(op), seed)
    c2w, k = origin_camera(res[0], res[1], 0.9 * res[0])
    idx = np.arange(n_shell, n_shell + m)
    return scene, [c2w], [k], idx, -probes[:, 2]


def huge(n_field=3000, n_huge=4, seed=12, res=(96, 64)):
    """A dense field in front of the camera plus n_huge splats whose sigma exceeds the frustum: every tile's list holds
    all of them plus a share of the field (> 1000 entries per tile at these sizes)."""
    rng = np.random.default_rng(seed)
    c2w, k = origin_camera(res[0], res[1], 0.9 * res[0])
    z = rng.uniform(2.0, 6.0, n_field)
    xy = rng.uniform(-0.6, 0.6, (n_field, 2)) * z[:, None]
    field = np.stack([xy[:, 0], xy[:, 1], -z], 1)
    ls = np.log(rng.uniform(0.05, 0.4, (n_field, 3)))
    op = rng.uniform(0.003, 0.02, n_field)  # faint: T stays above the 1e-4 stop for several 256-entry rounds
    hz = np.linspace(2.5, 5.5, n_huge)
    hxyz = np.stack([rng.uniform(-0.2, 0.2, n_huge), rng.uniform(-0.2, 0.2, n_huge), -hz], 1)
    hls = np.log(np.stack([np.full(n_huge, 8.0), np.full(n_huge, 6.0), np.full(n_huge, 0.5)], 1))
    hop = np.full(n_huge, 0.3)
    xyz = np.concatenate([field, hxyz])
    scene = _finish(xyz, np.concatenate([ls, hls]), rng.normal(size=(n_field + n_huge, 4)),
                    np.concatenate([op, hop]), seed)
    return scene, [c2w], [k]


def ties(k=6, seed=13, res=(64, 48)):
    """k exact copies of one Gaussian (different colours) at several places, plus, in front of everything, a splat
    centred exactly between two pixels (even image width, on the optical axis): its two central pixels tie exactly.
    A background splat on one side makes the colours of the tied pixels differ."""
    rng = np.random.default_rng(seed)
    c2w, kk = origin_camera(res[0], res[1], 0.8 * res[0])
    xyz, ls, rq, op = [], [], [], []
    for p in range(4):
        base = np.array([rng.uniform(-0.4, 0.4), rng.uniform(-0.3, 0.3), -rng.uniform(2.0, 4.0)])
        s = np.log(rng.uniform(0.05, 0.2, 3))
        q = rng.normal(size=4)
        o = rng.uniform(0.2, 0.9)
        for _ in range(k):
            xyz.append(base); ls.append(s); rq.append(q); op.append(o)
    xyz.append([0.0, 0.0, -1.0]); ls.append(np.log([0.02, 0.02, 0.02])); rq.append([1.0, 0, 0, 0]); op.append(0.6)
    xyz.append([0.3, 0.0, -3.0]); ls.append(np.log([0.3, 0.3, 0.3])); rq.append([1.0, 0, 0, 0]); op.append(0.9)
    scene = _finish(np.asarray(xyz), np.asarray(ls), np.asarray(rq), np.asarray(op), seed)
    scene["colours"] = torch.as_tensor(rng.uniform(0, 1, (len(op), 3)))
    return scene, [c2w], [kk]


def alpha_sweep(half_width=160):
    """f32 opacities: every value within +-half_width ulps of 1/255."""
    c = F32(1.0 / 255.0)
    bits = c.view(np.uint32).astype(np.int64) + np.arange(-half_width, half_width + 1)
    return bits.astype(np.uint32).view(np.float32)


CLAMP_OPACITIES = np.array([1.0, 0.999, 0.995, np.nextafter(F32(0.99), F32(1)), 0.99, np.nextafter(F32(0.99), F32(0)),
                            0.98], dtype=np.float32)


def opacity(res=(33, 31), spacing=10.0):
    """Gaussian i sits at (spacing * i, 0, -3) and camera i at (spacing * i, 0, 0) looking down -z, so Gaussian i is
    on the optical axis of camera i (view x = y = 0 exactly, odd image size: centred on a pixel centre, power 0 there)
    and outside every other camera's view: its alpha at that pixel is min(0.99, exp2(log2(opacity))) with T = 1, so its
    max contribution IS its alpha.  Opacities: CLAMP_OPACITIES, then alpha_sweep()."""
    ops = np.concatenate([CLAMP_OPACITIES, alpha_sweep()])
    n = ops.shape[0]
    x = spacing * np.arange(n)
    xyz = np.stack([x, np.zeros(n), np.full(n, -3.0)], 1)
    scene = _finish(xyz, np.log(np.full((n, 3), 0.05)), np.tile([1.0, 0, 0, 0], (n, 1)), ops, 14)
    cams, intr = [], []
    for i in range(n):
        c2w = torch.eye(4, dtype=torch.float32)
        c2w[0, 3] = float(x[i])
        cams.append(c2w)
        intr.append([res[0], res[1], 0.9 * res[0], 0.9 * res[0]])
    return scene, cams, intr


def _spread_scales(rng, n, kind):
    if kind == "needle":
        big = rng.uniform(-2.3, -1.0, n)                 # 1e-1 .. 3.7e-1
        small = np.log(10.0) * rng.uniform(-5.0, -3.0, n)  # 1e-5 .. 1e-3
        s = np.stack([big, small, small + rng.normal(0, 0.01, n)], 1)
    else:
        big = rng.uniform(-2.3, -1.0, n)
        small = np.log(10.0) * rng.uniform(-5.0, -3.0, n)
        s = np.stack([big, big + rng.normal(0, 0.1, n), small], 1)
    for i in range(n):  # the large axis is not always the first one
        s[i] = s[i, rng.permutation(3)]
    return s


def badly_conditioned(kind, n=1025, seed=15):
    """needle / disc family: cond(Sigma) from 1e6 to 1e10.  A quarter identity quaternions (the eigen-solver's
    diagonal branch), a quarter axis-aligned (quaternions with one non-zero entry, some not normalised: R is exactly
    diagonal), the rest random non-normalised quaternions (norm 0.3 .. 3)."""
    rng = np.random.default_rng(seed + (0 if kind == "needle" else 1))
    s = _spread_scales(rng, n, kind)
    q = rng.normal(size=(n, 4))
    q *= rng.uniform(0.3, 3.0, (n, 1)) / np.linalg.norm(q, axis=1, keepdims=True)
    a = n // 4
    q[:a] = [1.0, 0.0, 0.0, 0.0]
    exact = np.array([[0, 1, 0, 0], [0, 0, 1, 0], [0, 0, 0, 1], [2, 0, 0, 0], [0, 0.5, 0, 0]], dtype=np.float64)
    q[a:2 * a] = exact[np.arange(a) % exact.shape[0]]
    xyz = rng.uniform(-1, 1, (n, 3))
    return _finish(xyz, s, q, rng.uniform(0.05, 0.99, n), seed)


def diagonal_covariances():
    """Symmetric 3x3 inputs of the eigen-solver whose off-diagonals are exactly zero: every permutation of a diagonal
    with distinct, repeated and equal entries."""
    import itertools
    out = []
    for d in ([3.0, 1.0, 2.0], [1e-2, 1e-7, 1e-4], [2.0, 2.0, 1.0], [5.0, 5.0, 5.0], [1e-10, 1.0, 1e-5]):
        for p in itertools.permutations(d):
            out.append(np.diag(p))
    return np.asarray(out, dtype=np.float32)


def golden_scenes():
    """The edge scenes the reference's outputs are stored for (tests/golden/colour_edge.npz, tiles_edge.npz), small
    enough for the reference's dense CPU blend: name -> (scene, cams, intr).  The opacity family keeps its clamp cameras
    and every 16th camera of the 1/255 sweep."""
    sc_op, cams_op, intr_op = opacity()
    nc = CLAMP_OPACITIES.shape[0]
    pick = list(range(nc)) + list(range(nc, len(cams_op), 16))
    # the reference orders exact depth ties by its unstable torch.sort: the inside probes keep one Gaussian per depth,
    # and the copies of the ties family share one colour, so that its image and the multiset of the copies' maxima do
    # not depend on that order
    sc_in, cams_in, intr_in, pidx, _ = inside(n_shell=600)
    keep = np.ones(sc_in["xyz"].shape[0], dtype=bool)
    keep[pidx[0:2 * len(INSIDE_DEPTHS):2]] = False  # the on-axis probe of each (on-axis, lateral) pair
    sc_in = {k: v[torch.as_tensor(keep)] for k, v in sc_in.items()}
    sc_t, cams_t, intr_t = ties()
    sc_t["colours"] = sc_t["colours"].clone()
    for g0 in range(0, sc_t["colours"].shape[0] - 2, 6):
        sc_t["colours"][g0:g0 + 6] = sc_t["colours"][g0]
    return {
        "inside": (sc_in, cams_in, intr_in),
        "huge": huge(n_field=500, n_huge=3),
        "ties": (sc_t, cams_t, intr_t),
        "opacity": (sc_op, [cams_op[i] for i in pick], [intr_op[i] for i in pick]),
    }
