"""Oracle restatement of the colour stage, renderer_type=cuda (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows the reference's CUDA back-end on the CPU in numpy float32:
    camera_handler.py:72-108                                 get_camera("cuda"): z-forward view matrix, full projection
    cuda_rasterizer/forward.cu:153-271 + auxiliary.h:40-176  preprocessCUDA (near cull 0.2, EWA + 0.3, conic, radius, rect)
    cuda_rasterizer/rasterizer_impl.cu:69-137,285-326        per-tile lists ordered by (depth bits, emission order)
    cuda_rasterizer/forward.cu:303-497                       renderCUDA (rounds of 256, power > 0 / alpha < 1/255 skips,
                                                             stop before T < 1e-4, depth / inverse depth, mask)
    gaussian_pointcloud_rasterization/__init__.py:126-158    accumulator updates
with the racy parts replaced by what they aim at (SURVEY.md §2.1, §8a): per-Gaussian contribution = max over pixels,
arg-max = lowest pixel id among equals, surface distance = min over the tile's threads after every round of 256 entries
(threads outside the image hold expected depth 0, masked pixels have left the loop).
PARITY PIN: the reference extension needs a GPU; tests/test_tiles_gpu.py compares the kernels with this oracle and with
stored outputs of the unmodified extension (golden tiles_ref, written on an H100 by tests/golden/make_golden.py --gpu).
"""
import math

import numpy as np
import torch

F = np.float32


class RasterSettings:
    """get_camera("cuda") of the reference (camera_handler.py:53-108), host float32."""

    def __init__(self, c2w, intrinsic, colour_resolution=None, white_bkgd=True, mask=None, znear=10, zfar=100):
        c2w = torch.as_tensor(c2w, dtype=torch.float32).clone()
        diff = 1 if (colour_resolution is None or mask is not None) else colour_resolution / int(intrinsic[0])
        W = int(int(intrinsic[0]) * diff)
        H = int(int(intrinsic[1]) * diff)
        fx, fy = float(intrinsic[2]) * diff, float(intrinsic[3]) * diff
        c2w[:, 1:3] = -c2w[:, 1:3]
        fovX, fovY = 2 * math.atan(W / (2 * fx)), 2 * math.atan(H / (2 * fy))
        self.tanfovx, self.tanfovy = math.tan(fovX * 0.5), math.tan(fovY * 0.5)
        ty, tx = math.tan(fovY / 2), math.tan(fovX / 2)
        P = torch.zeros(4, 4)
        P[0, 0] = 2.0 * znear / (2 * tx * znear)
        P[1, 1] = 2.0 * znear / (2 * ty * znear)
        P[3, 2] = 1.0
        P[2, 2] = zfar / (zfar - znear)
        P[2, 3] = -(zfar * znear) / (zfar - znear)
        self.viewmatrix = torch.linalg.inv(c2w).permute(1, 0).contiguous()
        self.projmatrix = (self.viewmatrix @ P.transpose(0, 1)).contiguous()
        self.campos = self.viewmatrix.inverse()[3, :3]
        self.image_width, self.image_height = W, H
        self.bg = np.array([1, 1, 1] if white_bkgd else [0, 0, 0], dtype=F)
        self.mask = None if mask is None else np.asarray(mask).reshape(-1).astype(np.int32)


def preprocess(means, cov, rs):
    """Per Gaussian (forward.cu:153-271).  cov: (N,3,3) float32.  Returns a dict of arrays over all N (ok mask)."""
    m = np.asarray(means, dtype=F)
    S = np.asarray(cov, dtype=F)
    V = rs.viewmatrix.numpy().astype(F).reshape(-1)
    M = rs.projmatrix.numpy().astype(F).reshape(-1)
    W, H = rs.image_width, rs.image_height
    x, y, z = m[:, 0], m[:, 1], m[:, 2]
    vx = V[0] * x + V[4] * y + V[8] * z + V[12]
    vy = V[1] * x + V[5] * y + V[9] * z + V[13]
    vz = V[2] * x + V[6] * y + V[10] * z + V[14]
    ok = vz > F(0.2)
    vzs = np.where(ok, vz, F(1.0))
    hx = M[0] * x + M[4] * y + M[8] * z + M[12]
    hy = M[1] * x + M[5] * y + M[9] * z + M[13]
    hw = M[3] * x + M[7] * y + M[11] * z + M[15]
    pw = F(1.0) / (hw + F(0.0000001))
    ndx, ndy = hx * pw, hy * pw
    fx = F(W / (2.0 * rs.tanfovx))
    fy = F(H / (2.0 * rs.tanfovy))
    limx, limy = F(1.3 * rs.tanfovx), F(1.3 * rs.tanfovy)
    tx = np.minimum(limx, np.maximum(-limx, vx / vzs)) * vzs
    ty = np.minimum(limy, np.maximum(-limy, vy / vzs)) * vzs
    ja, jb = fx / vzs, -(fx * tx) / (vzs * vzs)
    jc, jd = fy / vzs, -(fy * ty) / (vzs * vzs)
    Mr = np.zeros((m.shape[0], 2, 3), dtype=F)
    for c in range(3):
        Mr[:, 0, c] = ja * V[4 * c + 0] + jb * V[4 * c + 2]
        Mr[:, 1, c] = jc * V[4 * c + 1] + jd * V[4 * c + 2]
    A = np.einsum("nrk,nkc->nrc", Mr, S).astype(F)
    c2 = np.einsum("nrk,nsk->nrs", A, Mr).astype(F)
    ca, cb, cc = c2[:, 0, 0] + F(0.3), c2[:, 0, 1], c2[:, 1, 1] + F(0.3)
    det = ca * cc - cb * cb
    ok &= det != 0
    dets = np.where(det != 0, det, F(1.0))
    kx, ky, kz = cc / dets, -cb / dets, ca / dets
    mid = F(0.5) * (ca + cc)
    root = np.sqrt(np.maximum(F(0.1), mid * mid - det))
    radius = np.ceil(F(3.0) * np.sqrt(np.maximum(mid + root, mid - root)))
    px = (((ndx.astype(np.float64) + 1.0) * W - 1.0) * 0.5).astype(F)
    py = (((ndy.astype(np.float64) + 1.0) * H - 1.0) * 0.5).astype(F)
    gx, gy = (W + 15) // 16, (H + 15) // 16
    ir = np.where(np.isfinite(radius), radius, 0).astype(np.int64)
    trunc = lambda a: np.trunc(np.where(np.isfinite(a), a, 0)).astype(np.int64)
    rx0 = np.clip(trunc((px - ir.astype(F)) / F(16)), 0, gx)
    ry0 = np.clip(trunc((py - ir.astype(F)) / F(16)), 0, gy)
    rx1 = np.clip(trunc((px + ir.astype(F) + F(16) - F(1)) / F(16)), 0, gx)
    ry1 = np.clip(trunc((py + ir.astype(F) + F(16) - F(1)) / F(16)), 0, gy)
    ok &= ((rx1 - rx0) * (ry1 - ry0)) != 0
    return dict(ok=ok, px=px, py=py, conic=np.stack([kx, ky, kz], 1), radius=ir, depth=vz, rx0=rx0, rx1=rx1, ry0=ry0,
                ry1=ry1, gx=gx, gy=gy)


def render(pre, opacity, colour, rs, calculate_surface_distance=False):
    """renderCUDA over all tiles.  colour (N,3) float32.  Returns dict(image (3,H,W), depth (H,W), invdepth (H,W),
    contrib (N), pixel (N), surface (N))."""
    W, H = rs.image_width, rs.image_height
    N = opacity.shape[0]
    op = np.asarray(opacity, dtype=F).reshape(-1)
    col = np.asarray(colour, dtype=F)
    img = np.zeros((3, H, W), dtype=F)
    depth_img = np.zeros((H, W), dtype=F)
    inv_img = np.zeros((H, W), dtype=F)
    contrib = np.zeros(N, dtype=F)
    pixel = np.zeros(N, dtype=np.int64)
    surface = np.full(N, np.finfo(F).max, dtype=F)
    ok = np.nonzero(pre["ok"])[0]
    order = ok[np.argsort(pre["depth"][ok].view(np.uint32), kind="stable")]  # radix sort on the float bits, stable
    gx, gy = pre["gx"], pre["gy"]
    mask = rs.mask
    for ty in range(gy):
        for tx in range(gx):
            sel = order[(pre["rx0"][order] <= tx) & (tx < pre["rx1"][order]) & (pre["ry0"][order] <= ty) & (ty < pre["ry1"][order])]
            ys, xs = np.meshgrid(np.arange(ty * 16, ty * 16 + 16), np.arange(tx * 16, tx * 16 + 16), indexing="ij")
            ys, xs = ys.reshape(-1), xs.reshape(-1)
            inside = (xs < W) & (ys < H)
            pid = ys * W + xs
            mpix = inside.copy()
            if mask is not None:
                mpix[inside] = mask[pid[inside]] != 0
            T = np.ones(256, dtype=F)
            done = ~mpix  # threads outside the image / of masked pixels never rasterise
            C = np.zeros((256, 3), dtype=F)
            E = np.zeros(256, dtype=F)
            IE = np.zeros(256, dtype=F)
            pxf, pyf = xs.astype(F), ys.astype(F)
            all_left = False
            for r0 in range(0, sel.shape[0], 256):
                if bool(done.all()):
                    break
                rnd = sel[r0:r0 + 256]
                for g in rnd:
                    act = ~done & mpix
                    dx = pre["px"][g] - pxf
                    dy = pre["py"][g] - pyf
                    kx, ky, kz = pre["conic"][g]
                    power = F(-0.5) * (kx * dx * dx + kz * dy * dy) - ky * dx * dy
                    alpha = np.minimum(F(0.99), op[g] * np.exp(power, dtype=F))
                    keep = act & ~(power > 0) & ~(alpha < F(1.0 / 255.0))
                    testT = T * (F(1.0) - alpha)
                    stop = keep & (testT < F(0.0001))
                    done = done | stop
                    take = keep & ~stop
                    c = np.where(take, alpha * T, F(0)).astype(F)
                    C += c[:, None] * col[g][None, :]
                    IE += (F(1.0) / pre["depth"][g]) * c
                    E += pre["depth"][g] * c
                    T = np.where(take, testT, T)
                    v = c.max()
                    if v > contrib[g]:
                        contrib[g] = v
                        pixel[g] = pid[np.nonzero(c == v)[0]].min()
                    elif v == contrib[g] and v > 0:
                        pixel[g] = min(pixel[g], pid[np.nonzero(c == v)[0]].min())
                if calculate_surface_distance:
                    # threads of masked pixels have left the loop (forward.cu:389-390); all others — including finished
                    # pixels and threads outside the image (expected depth 0) — take part (:460-477)
                    part = mpix | ~inside
                    if part.any():
                        d = np.abs(pre["depth"][rnd][:, None] - E[part][None, :]).min(axis=1).astype(F)
                        surface[rnd] = np.minimum(surface[rnd], d)
            w = inside & mpix
            img[:, ys[w], xs[w]] = (C[w] + T[w][:, None] * rs.bg[None, :]).T
            depth_img[ys[w], xs[w]] = E[w]
            inv_img[ys[w], xs[w]] = IE[w]
    return dict(image=img, depth=depth_img, invdepth=inv_img, contrib=contrib, pixel=pixel, surface=surface)


class CudaRasterizerOracle:
    """GaussianRasterizer (gaussian_pointcloud_rasterization/__init__.py:37-220) restated on the CPU."""

    def __init__(self, means3D, opacity, colour, cov3d, visible_gaussian_threshold=0.0, calculate_surface_distance=False):
        self.means = np.asarray(means3D, dtype=F)
        self.opacity = np.asarray(opacity, dtype=F).reshape(-1)
        self.colour = np.asarray(colour, dtype=F)
        self.cov = np.asarray(cov3d, dtype=F)
        n = self.means.shape[0]
        self.gaussian_max_contribution = np.zeros(n, dtype=F)
        self.gaussian_total_contribution = np.zeros(n, dtype=F)
        self.gaussian_min_surface_distance = np.full(n, np.finfo(F).max, dtype=F)
        self.gaussian_colours = np.zeros((n, 3), dtype=F)
        self.calculate_surface_distance = calculate_surface_distance
        self.visible_gaussian_threshold = visible_gaussian_threshold
        self.last = None

    def __call__(self, rs):
        pre = preprocess(self.means, self.cov, rs)
        out = render(pre, self.opacity, self.colour, rs, self.calculate_surface_distance)
        flat = out["image"].reshape(3, -1).T
        cur = flat[out["pixel"]]
        upd = out["contrib"] > self.gaussian_max_contribution
        self.gaussian_max_contribution[upd] = out["contrib"][upd]
        self.gaussian_colours[upd] = cur[upd]
        self.gaussian_total_contribution += out["contrib"]
        self.gaussian_min_surface_distance = np.minimum(self.gaussian_min_surface_distance, out["surface"])
        self.last = dict(pre=pre, **out)
        return out["image"], pre["radius"] * pre["ok"], out["invdepth"][None], out["depth"][None]

    def low_surface_distance_mask(self, std):
        d = self.gaussian_min_surface_distance
        finite = d < np.finfo(F).max
        return d < d[finite].mean() * std
