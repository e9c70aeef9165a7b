"""Plain float64 evaluations of the operations the kernels perform (numpy, no rounding mimicry).

The oracles under oracle/ restate the reference's float32 arithmetic, which is the right pin on benign inputs.  On
badly conditioned inputs both the kernel and the f32 oracle carry errors of cond * u, and only an exact-arithmetic
yardstick says which side is wrong and by how much.  Inputs are the f32 values the kernels see (upcast), so the
references measure the kernels' arithmetic, not the rounding of their inputs.
"""
import math

import numpy as np

U32 = 2.0 ** -24  # unit roundoff of float32
K_EXP2 = -0.72134752044448170368  # -0.5 * log2(e): the kernels store the conic pre-scaled by it


def rotation(q):
    """R(q) of gauss_handler.py:26-47, q = (r, x, y, z) NOT normalised."""
    q = np.asarray(q, dtype=np.float64)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = np.empty((q.shape[0], 3, 3))
    R[:, 0, 0] = 1 - 2 * (y * y + z * z); R[:, 0, 1] = 2 * (x * y - r * z); R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z); R[:, 1, 1] = 1 - 2 * (x * x + z * z); R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y); R[:, 2, 1] = 2 * (y * z + r * x); R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def covariance(log_scales, rots, modifier=1.0):
    """Sigma = (R diag(exp(mod * s))) (R diag(exp(mod * s)))^T."""
    L = rotation(rots) * np.exp(modifier * np.asarray(log_scales, dtype=np.float64))[:, None, :]
    return L @ L.transpose(0, 2, 1)


def normals(log_scales, rots):
    """Column argmin(scale) of R (first minimum on ties)."""
    a = np.argmin(np.asarray(log_scales, dtype=np.float64), axis=1)
    return rotation(rots)[np.arange(a.shape[0]), :, a]


def eigvalsh(cov):
    """Ascending eigenvalues of the symmetric part of each (f32) matrix."""
    c = np.asarray(cov, dtype=np.float64)
    return np.linalg.eigvalsh(0.5 * (c + c.transpose(0, 2, 1)))


def magnitudes(cov, contrib):
    """sqrt(ellipsoid surface area, Knud Thomsen p = 1.6075) * contribution."""
    return magnitudes_from_eig(eigvalsh(cov), contrib)


def cholesky_ladder(cov, step=1e-6, levels=3):
    """Level of the regularise-and-retry ladder (Sigma + level * step * I) at which the exact Cholesky exists, 3 if none,
    the factor L (n,3,3) of that level (zeros if none) and the margin: the smallest eigenvalue of the matrix the
    decision was taken on, relative to its largest (how far the decision is from a tie)."""
    c = 0.5 * (np.asarray(cov, dtype=np.float64) + np.asarray(cov, dtype=np.float64).transpose(0, 2, 1))
    n = c.shape[0]
    lvl = np.full(n, levels, dtype=np.int64)
    L = np.zeros((n, 3, 3))
    margin = np.full(n, np.inf)
    for i in range(n):
        for k in range(levels):
            m = c[i] + k * step * np.eye(3)
            ev = np.linalg.eigvalsh(m)
            margin[i] = min(margin[i], abs(ev[0]) / max(abs(ev[-1]), 1e-300))
            if ev[0] > 0:
                lvl[i] = k
                L[i] = np.linalg.cholesky(m)
                break
    return lvl, L, margin


def ewa(means, cov, view, focal_x, focal_y, tan_fovx, tan_fovy, z_sign):
    """EWA splat covariance J W Sigma W^T J^T + 0.3 I of both back-ends (row-vector view matrix; z_sign = -1 for the
    python back-end's -z forward view, +1 for the CUDA back-end's).  Returns (t (n,3) view position, cov2d (n,2,2))."""
    V = np.asarray(view, dtype=np.float64)
    m = np.asarray(means, dtype=np.float64)
    S = np.asarray(cov, dtype=np.float64)
    t = m @ V[:3, :3] + V[3, :3]
    tz = t[:, 2]
    limx, limy = 1.3 * tan_fovx, 1.3 * tan_fovy
    with np.errstate(divide="ignore", invalid="ignore"):
        tx = np.clip(t[:, 0] / tz, -limx, limx) * tz
        ty = np.clip(t[:, 1] / tz, -limy, limy) * tz
        J = np.zeros((m.shape[0], 2, 3))
        J[:, 0, 0] = focal_x / tz
        J[:, 0, 2] = -focal_x * tx / (tz * tz)
        J[:, 1, 1] = focal_y / tz
        J[:, 1, 2] = -focal_y * ty / (tz * tz)
        Wm = V[:3, :3].T
        T = J @ Wm[None]
        c2 = T @ S @ T.transpose(0, 2, 1) + 0.3 * np.eye(2)
    return t, c2


def radius_lambda(c2):
    """The larger root both back-ends take the radius from: mid + sqrt(max(mid^2 - det, 0.1)) (the 0.1 floor is the
    reference's, gauss_render.py:171-183 / forward.cu:222-224)."""
    a, b, c, d = c2[:, 0, 0], c2[:, 0, 1], c2[:, 1, 0], c2[:, 1, 1]
    det = a * d - b * c
    mid = 0.5 * (a + d)
    root = np.sqrt(np.maximum(mid * mid - det, 0.1))
    return np.maximum(mid + root, mid - root)


def magnitudes_from_eig(ev, contrib):
    a, b, c = (np.sqrt(np.clip(ev[:, k], 0.0, None)) for k in range(3))
    p = 1.6075
    rad = ((a * b) ** p + (a * c) ** p + (b * c) ** p) / 3.0
    return np.sqrt(4.0 * math.pi * rad ** (1.0 / p)) * np.asarray(contrib, dtype=np.float64)


def conic(c2):
    """Inverse of each 2x2."""
    a, b, c, d = c2[:, 0, 0], c2[:, 0, 1], c2[:, 1, 0], c2[:, 1, 1]
    det = a * d - b * c
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack([d / det, -b / det, -c / det, a / det], 1).reshape(-1, 2, 2)


def project_python(means, cov, cam):
    """gauss_render.py:101-193 in f64 on the f32 camera of oracle.render.Camera: in-front decision, mean in pixels,
    conic, and the argument sqrt(lambda_max) whose ceil (times 3) is the radius."""
    V = cam.world_view_transform.numpy().astype(np.float64)
    P = cam.projection_matrix.numpy().astype(np.float64)
    W, H = cam.image_width, cam.image_height
    t, c2 = ewa(means, cov, V, cam.focal_x, cam.focal_y, math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5), -1)
    po = np.concatenate([np.asarray(means, dtype=np.float64), np.ones((t.shape[0], 1))], 1)
    ph = po @ V @ P
    with np.errstate(divide="ignore", invalid="ignore"):
        pw = 1.0 / (ph[:, 3] + 1e-6)
        mx = ((ph[:, 0] * pw + 1) * W - 1.0) * 0.5
        my = ((ph[:, 1] * pw + 1) * H - 1.0) * 0.5
    return dict(z=t[:, 2], mx=mx, my=my, cov2d=c2, conic=conic(c2), sqrt_lmax=np.sqrt(radius_lambda(c2)))


def preprocess_cuda(means, cov, rs):
    """forward.cu:153-271 in f64 on the f32 matrices of oracle.render_cuda.RasterSettings: view depth, pixel mean,
    conic and the argument 3 sqrt(lambda_max) whose ceil is the radius."""
    V = rs.viewmatrix.numpy().astype(np.float64)
    M = rs.projmatrix.numpy().astype(np.float64)
    W, H = rs.image_width, rs.image_height
    fx, fy = W / (2.0 * rs.tanfovx), H / (2.0 * rs.tanfovy)
    t, c2 = ewa(means, cov, V, fx, fy, rs.tanfovx, rs.tanfovy, 1)
    m = np.asarray(means, dtype=np.float64)
    h = m @ M[:3] + M[3]
    with np.errstate(divide="ignore", invalid="ignore"):
        pw = 1.0 / (h[:, 3] + 1e-7)
        px = ((h[:, 0] * pw + 1.0) * W - 1.0) * 0.5
        py = ((h[:, 1] * pw + 1.0) * H - 1.0) * 0.5
    return dict(z=t[:, 2], px=px, py=py, cov2d=c2, conic=conic(c2), three_sigma=3.0 * np.sqrt(radius_lambda(c2)))


def unpack_rect(bits):
    """Tile rect [x0, x1] x [y0, y1] (inclusive) of g2pc_pack_range (s7_tiles.cu q2.w)."""
    b = np.asarray(bits).view(np.uint32).astype(np.int64)
    return b & 0xFF, (b >> 8) & 0xFF, (b >> 16) & 0xFF, (b >> 24) & 0xFF


def tiles_blend(rec, ok, W, H, bg, band_alpha=2e-5, band_T=1e-4, surface=True, mask=None):
    """renderCUDA (forward.cu:303-497) in f64, stage-wise: fed the kernel's own projection records `rec` ((n,12): {px,py,
    K kx, 2K ky} {K kz, log2 o, r, g} {b, depth, radius, tile rect}) and its `ok` mask, with the kernel's list order
    (stable by the depth's float bits).  Per tile in rounds of 256 list entries: alpha = min(0.99, o exp(power)),
    skip power > 0 or alpha < 1/255, stop before T (1 - alpha) < 1e-4, deterministic surface distance after each round.

    `mask` ((H*W) or (H,W), 0 = ignore): a masked pixel is never live, takes no part in the surface distances and is not
    written (image, depth and inverse depth stay 0).  A tile with no live pixel at the start of a round — round 0
    included — leaves before that round.

    A skip / stop decision whose f64 operand lies within a relative band of its threshold may go either way in f32:
    the pixel is marked `tainted` from that entry on.  Returns image (3,H,W), depth, invdepth (sum of c / depth),
    contrib (n) max over untainted pairs, pixel (n, lowest id among exact equals), second (n, the runner-up at another
    pixel), any_taint (n: a pair of that Gaussian was tainted or followed a taint), surface (n), surf_taint (n), and the
    decision counts."""
    n = rec.shape[0]
    mflat = None if mask is None else np.asarray(mask).reshape(-1) != 0
    px, py = rec[:, 0].astype(np.float64), rec[:, 1].astype(np.float64)
    kx, ky, kz = rec[:, 2] / K_EXP2, rec[:, 3] / (2 * K_EXP2), rec[:, 4] / K_EXP2
    op = np.exp2(rec[:, 5].astype(np.float64))
    col = rec[:, [6, 7, 8]].astype(np.float64)
    depth = rec[:, 9].astype(np.float64)
    x0, x1, y0, y1 = unpack_rect(rec[:, 11])
    idx = np.nonzero(ok)[0]
    order = idx[np.argsort(rec[idx, 9].view(np.uint32), kind="stable")]
    gx, gy = (W + 15) // 16, (H + 15) // 16
    img = np.zeros((3, H, W))
    dimg = np.zeros((H, W))
    iimg = np.zeros((H, W))
    contrib = np.zeros(n)
    pixel = np.full(n, -1, dtype=np.int64)
    second = np.zeros(n)  # runner-up: the largest untainted contribution at any other pixel
    taint = np.zeros(n, dtype=bool)
    surf = np.full(n, np.inf)
    staint = np.zeros(n, dtype=bool)
    counts = dict(skip_band=0, stop_band=0, rounds_max=0, list_max=0)
    for ty in range(gy):
        for tx in range(gx):
            sel = order[(x0[order] <= tx) & (tx <= x1[order]) & (y0[order] <= ty) & (ty <= y1[order])]
            counts["list_max"] = max(counts["list_max"], sel.shape[0])
            ys, xs = np.meshgrid(np.arange(ty * 16, ty * 16 + 16), np.arange(tx * 16, tx * 16 + 16), indexing="ij")
            ys, xs = ys.reshape(-1), xs.reshape(-1)
            inside = (xs < W) & (ys < H)
            pid = ys * W + xs
            live0 = inside.copy()
            if mflat is not None:
                live0[inside] = mflat[pid[inside]]
            # surface distances: unmasked pixels hold their expected depth, threads outside the image hold 0
            part = live0 | ~inside
            T = np.ones(256)
            done = ~live0
            tainted = np.zeros(256, dtype=bool)
            band_done = np.zeros(256, dtype=bool)  # stopped by a decision in the band: may still be live in f32
            slack = np.zeros(256)  # bound on how far a tainted pixel's expected depth may lie from the f32 one
            dmax = float(depth[sel].max()) if sel.shape[0] else 0.0
            C = np.zeros((256, 3))
            E = np.zeros(256)
            IE = np.zeros(256)
            rounds = 0
            for r0 in range(0, sel.shape[0], 256):
                # whether the tile leaves here is undetermined when a tainted pixel could be live in f32 and no
                # untainted one is
                if tainted.any() and not (~done & ~tainted).any() and (band_done.any() or not done.all()):
                    staint[sel[r0:]] = True
                    taint[sel[r0:]] = True
                if bool(done.all()):
                    break  # the tile leaves at the start of a round
                rounds += 1
                rnd = sel[r0:r0 + 256]
                for g in rnd:
                    dx = px[g] - xs
                    dy = py[g] - ys
                    power = -0.5 * (kx[g] * dx * dx + kz[g] * dy * dy) - ky[g] * dx * dy
                    alpha = np.minimum(0.99, op[g] * np.exp(power))
                    act = ~done
                    near_skip = act & (power <= 0) & (np.abs(alpha * 255.0 - 1.0) < band_alpha)
                    keep = act & ~(power > 0) & ~(alpha < 1.0 / 255.0)
                    testT = T * (1.0 - alpha)
                    near_stop = keep & (np.abs(testT / 1e-4 - 1.0) < band_T)
                    counts["skip_band"] += int(near_skip.sum())
                    counts["stop_band"] += int(near_stop.sum())
                    tainted |= near_skip | near_stop
                    # a flipped skip moves E by at most alpha (its own share and the attenuation of the rest) times the
                    # deepest entry, twice over; a flipped stop by at most T times it, twice over
                    slack += 2.0 * dmax * (np.where(near_skip, alpha, 0.0) + np.where(near_stop, T, 0.0))
                    stop = keep & (testT < 1e-4)
                    band_done |= stop & near_stop
                    done |= stop
                    take = keep & ~stop
                    c = np.where(take, alpha * T, 0.0)
                    C += c[:, None] * col[g][None, :]
                    E += depth[g] * c
                    IE += c / depth[g]
                    T = np.where(take, testT, T)
                    cu = np.where(tainted, 0.0, c)
                    if tainted[act | band_done].any():
                        taint[g] = True
                    at_max = np.flatnonzero(cu == cu.max())
                    k1 = int(at_max[np.argmin(pid[at_max])])  # lowest pixel id among the maxima
                    v1, p1 = cu[k1], pid[k1]
                    v2 = np.delete(cu, k1).max()
                    if v1 > contrib[g] or (v1 == contrib[g] and v1 > 0 and p1 < pixel[g]):
                        loser = contrib[g]
                        contrib[g], pixel[g] = v1, p1
                    else:
                        loser = v1
                    second[g] = max(second[g], v2, loser)
                if surface and part.any():
                    Ep = np.where(inside, E, 0.0)
                    dist = np.abs(depth[rnd][:, None] - Ep[None, :])
                    d = dist[:, part].min(axis=1)
                    surf[rnd] = np.minimum(surf[rnd], d)
                    # tainted: a tainted pixel, moved by its slack (plus a stop one entry early or late), could come
                    # at least as close as the others
                    tp = part & tainted
                    if tp.any():
                        d_clean = dist[:, part & ~tainted].min(axis=1, initial=np.inf)
                        d_low = (dist[:, tp] - (slack[tp] + 2e-4 * dmax)[None, :]).min(axis=1)
                        staint[rnd[d_low <= d_clean]] = True
            counts["rounds_max"] = max(counts["rounds_max"], rounds)
            w = live0
            img[:, ys[w], xs[w]] = (C[w] + T[w][:, None] * np.asarray(bg, dtype=np.float64)[None, :]).T
            dimg[ys[w], xs[w]] = E[w]
            iimg[ys[w], xs[w]] = IE[w]
            if tainted.any():
                img[:, ys[w & tainted], xs[w & tainted]] = np.nan
                dimg[ys[w & tainted], xs[w & tainted]] = np.nan
                iimg[ys[w & tainted], xs[w & tainted]] = np.nan
    return dict(image=img, depth=dimg, invdepth=iimg, contrib=contrib, pixel=pixel, second=second, taint=taint,
                surface=surf, surf_taint=staint, **counts)


def _sh_basis(deg):
    """Real spherical harmonics Y_lm (l <= deg, m = -l..l at index l^2 + l + m, Condon-Shortley phase) as polynomials
    in the unit direction: a list of {(a, b, c): coefficient of x^a y^b z^c}.  From the definitions:
    Y_l0 = K_l0 P_l(z), Y_lm = sqrt(2) K_lm P_l^|m|(z) {cos m phi (m > 0), sin |m| phi (m < 0)},
    K_lm = sqrt((2l + 1) / (4 pi) (l - |m|)! / (l + |m|)!), P_l^m(z) = (-1)^m (1 - z^2)^(m/2) d^m P_l / dz^m, and
    (1 - z^2)^(m/2) (cos m phi + i sin m phi) = (x + i y)^m on the unit sphere."""
    from numpy.polynomial import legendre as L
    out = []
    for l in range(deg + 1):
        for m in range(-l, l + 1):
            a = abs(m)
            K = math.sqrt((2 * l + 1) / (4.0 * math.pi) * math.factorial(l - a) / math.factorial(l + a))
            dz = L.leg2poly(L.legder(np.eye(l + 1)[l], a))  # d^a P_l / dz^a in the power basis
            # (x + i y)^a = sum_k C(a, k) x^(a-k) (i y)^k: real part (cos) even k, imaginary part (sin) odd k
            xy = {}
            for k in range(a + 1):
                if (m >= 0 and k % 2 == 0) or (m < 0 and k % 2 == 1):
                    xy[(a - k, k)] = math.comb(a, k) * (-1.0) ** (k // 2)
            scale = K * (1.0 if m == 0 else math.sqrt(2.0) * (-1.0) ** a)
            poly = {}
            for (px_, py_), cxy in xy.items():
                for pz, cz in enumerate(dz):
                    if cz != 0.0:
                        key = (px_, py_, pz)
                        poly[key] = poly.get(key, 0.0) + scale * cxy * cz
            out.append(poly)
    return out


def sh_colour(deg, shs, dirs, layout=0):
    """Colour of real SH degree `deg` in f64: max(sum_k Y_k(d) s_k + 0.5, 0) per channel.  shs: (n,3,stride) for layout 0
    (channel-major), (n,stride,3) for layout 1; dirs (n,3) unit directions.  Returns (rgb (n,3), bound (n,3)): bound is
    0.5 + sum over every monomial term of |coefficient x^a y^b z^c s_k|, the scale of the float32 rounding."""
    s = np.asarray(shs, dtype=np.float64)
    if layout == 1:
        s = s.transpose(0, 2, 1)
    d = np.asarray(dirs, dtype=np.float64)
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    r = np.zeros((d.shape[0], 3))
    bound = np.full((d.shape[0], 3), 0.5)
    for k, poly in enumerate(_sh_basis(deg)):
        for (a, b, c), coef in poly.items():
            t = (coef * x ** a * y ** b * z ** c)[:, None] * s[:, :, k]
            r += t
            bound += np.abs(t)
    return np.maximum(r + 0.5, 0.0), bound


def accumulate(per_camera, near=1e-6):
    """Fold per-camera f64 results in camera order, as the per-Gaussian accumulators do: maximum by strict > (the first
    camera keeps an exact tie), colour = the winning camera's f64 image at its arg-max pixel, total = f64 sum of the
    per-camera maxima, surface distance = minimum.  per_camera: dicts of tiles_blend (image, contrib, pixel, second,
    taint, surface, surf_taint).  A Gaussian tainted in any camera stays tainted.  `near_tie` marks a Gaussian whose
    maxima in two cameras lie within `near` of each other without being equal (which camera wins is undetermined in
    f32); `pixel_tie` one whose winning camera's arg-max pixel is a near-tie within that camera."""
    n = per_camera[0]["contrib"].shape[0]
    mx = np.zeros(n)
    winner = np.full(n, -1, dtype=np.int64)
    colour = np.zeros((n, 3))
    total = np.zeros(n)
    surf = np.full(n, np.inf)
    taint = np.zeros(n, dtype=bool)
    staint = np.zeros(n, dtype=bool)
    near_tie = np.zeros(n, dtype=bool)
    pixel_tie = np.zeros(n, dtype=bool)
    seen = []  # maxima of the earlier cameras
    for ci, f in enumerate(per_camera):
        v = f["contrib"]
        for prev in seen:
            near_tie |= (v > 0) & (prev > 0) & (v != prev) & (np.abs(v - prev) <= near)
        seen.append(v)
        upd = v > mx
        flat = f["image"].reshape(3, -1)
        pix = np.where(f["pixel"] >= 0, f["pixel"], 0)
        mx = np.where(upd, v, mx)
        winner = np.where(upd, ci, winner)
        colour = np.where(upd[:, None], flat[:, pix].T, colour)
        pixel_tie = np.where(upd, (v - f["second"]) < near, pixel_tie)
        total += v
        surf = np.minimum(surf, f["surface"])
        taint |= f["taint"]
        staint |= f["surf_taint"]
    return dict(max=mx, winner=winner, colour=colour, total=total, surface=surf, taint=taint, surf_taint=staint,
                near_tie=near_tie, pixel_tie=pixel_tie)


def leaf_blend(r0, c0, w, h, ids, proj, bg=1.0, transmittance=False):
    """gauss_render.py:337-369 for one quadtree leaf in f64, fed the kernel's records (python back-end layout:
    {mx, my, K c00, K (c01 + c10)} {K c11, log2 o, r, g} {b, depth, radius, valid}) and its depth-ordered list `ids`:
    alpha = min(0.99, o exp(power)), contribution T alpha, T *= 1 - alpha, background `bg` (white by default).
    Returns (colour (h*w, 3), contribution (h*w, len(ids))) with pixels row-major over the leaf, and the final
    transmittance (h*w,) as a third value when `transmittance` is set."""
    ys, xs = np.meshgrid(np.arange(r0, r0 + h), np.arange(c0, c0 + w), indexing="ij")
    px, py = xs.reshape(-1).astype(np.float64), ys.reshape(-1).astype(np.float64)
    P = proj[ids].astype(np.float64)
    T = np.ones(px.shape[0])
    col = np.zeros((px.shape[0], 3))
    contrib = np.zeros((px.shape[0], len(ids)))
    for j in range(len(ids)):
        dx, dy = px - P[j, 0], py - P[j, 1]
        e = (dx * dx * P[j, 2] + dy * dy * P[j, 4] + dx * dy * P[j, 3]) + P[j, 5]  # log2 of o * weight
        alpha = np.minimum(np.exp2(e), 0.99)
        c = T * alpha
        contrib[:, j] = c
        col += c[:, None] * P[j, 6:9][None, :]
        T = T * (1.0 - alpha)
    if transmittance:
        return col + bg * T[:, None], contrib, T
    return col + bg * T[:, None], contrib
