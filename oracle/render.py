"""Oracle restatement of the colour stage, renderer_type=python (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows gauss_render.py:101-193 (EWA covariance, projection, radius, rect), :266-402 (quadtree tiling,
front-to-back blend, per-Gaussian max contribution + colour) and camera_handler.py:14-50.  Written as an explicit
BFS over tiles and a *sequential* per-pixel blend (running transmittance), i.e. the way a kernel does it, rather than
with the reference's dense cumprod tensors.  torch-CPU float32 ops are used for the per-Gaussian geometry so that the
arithmetic matches the reference's CPU run.
"""
import math
from collections import deque

import numpy as np
import torch

C0 = 0.28209479177387814
C1 = 0.4886025119029199
C2 = [1.0925484305920792, -1.0925484305920792, 0.31539156525252005, -1.0925484305920792, 0.5462742152960396]
C3 = [-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154, -0.4570457994644658,
      1.445305721320277, -0.5900435899266435]


def sh_colour(deg, sh, dirs):
    """gauss_render.py:43-99 eval_sh (deg <= 3) + 0.5 and clamp >= 0 (forward.cu:65-72).  sh: (N,3,K) channel-major
    (gauss_dataloader.py:42-44), dirs: (N,3) unit vectors.  Returns (N,3)."""
    sh = torch.as_tensor(sh)
    dirs = torch.as_tensor(dirs)
    res = C0 * sh[..., 0]
    if deg > 0:
        x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
        res = res - C1 * y * sh[..., 1] + C1 * z * sh[..., 2] - C1 * x * sh[..., 3]
        if deg > 1:
            xx, yy, zz = x * x, y * y, z * z
            xy, yz, xz = x * y, y * z, x * z
            res = (res + C2[0] * xy * sh[..., 4] + C2[1] * yz * sh[..., 5] + C2[2] * (2.0 * zz - xx - yy) * sh[..., 6]
                   + C2[3] * xz * sh[..., 7] + C2[4] * (xx - yy) * sh[..., 8])
            if deg > 2:
                res = (res + C3[0] * y * (3 * xx - yy) * sh[..., 9] + C3[1] * xy * z * sh[..., 10]
                       + C3[2] * y * (4 * zz - xx - yy) * sh[..., 11] + C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * sh[..., 12]
                       + C3[4] * x * (4 * zz - xx - yy) * sh[..., 13] + C3[5] * z * (xx - yy) * sh[..., 14]
                       + C3[6] * x * (xx - 3 * yy) * sh[..., 15])
    return torch.clamp(res + 0.5, min=0.0)


class Camera:
    """camera_handler.py:36-50 + get_camera :53-70 (python branch)."""

    def __init__(self, c2w, intrinsic, colour_resolution=None, znear=10, zfar=100):
        c2w = torch.as_tensor(c2w, dtype=torch.float32)
        diff = 1 if colour_resolution is None else colour_resolution / int(intrinsic[0])
        self.image_width = int(int(intrinsic[0]) * diff)
        self.image_height = int(int(intrinsic[1]) * diff)
        self.focal_x = float(intrinsic[2]) * diff
        self.focal_y = float(intrinsic[3]) * diff
        self.FoVx = 2 * math.atan(self.image_width / (2 * self.focal_x))
        self.FoVy = 2 * math.atan(self.image_height / (2 * self.focal_y))
        self.world_view_transform = torch.linalg.inv(c2w).permute(1, 0)
        ty, tx = math.tan(self.FoVy / 2), math.tan(self.FoVx / 2)
        top, right = ty * znear, tx * znear
        P = torch.zeros(4, 4)
        P[0, 0] = 2.0 * znear / (2 * right)
        P[1, 1] = 2.0 * znear / (2 * top)
        P[3, 2] = 1.0
        P[2, 2] = zfar / (zfar - znear)
        P[2, 3] = -(zfar * znear) / (zfar - znear)
        self.projection_matrix = P.transpose(0, 1)
        self.camera_center = self.world_view_transform.inverse()[3, :3]


def project(means3D, cov3d, cam):
    """gauss_render.py:101-193,414-437: returns a dict of per-Gaussian f32 tensors (all N Gaussians, with in_mask)."""
    V, P = cam.world_view_transform, cam.projection_matrix
    W_, H_ = cam.image_width, cam.image_height
    tan_fovx, tan_fovy = math.tan(cam.FoVx * 0.5), math.tan(cam.FoVy * 0.5)
    t = (means3D @ V[:3, :3]) + V[-1:, :3]
    tx = (t[..., 0] / t[..., 2]).clip(min=-tan_fovx * 1.3, max=tan_fovx * 1.3) * t[..., 2]
    ty = (t[..., 1] / t[..., 2]).clip(min=-tan_fovy * 1.3, max=tan_fovy * 1.3) * t[..., 2]
    tz = t[..., 2]
    J = torch.zeros(means3D.shape[0], 3, 3)
    J[..., 0, 0] = 1 / tz * cam.focal_x
    J[..., 0, 2] = -tx / (tz * tz) * cam.focal_x
    J[..., 1, 1] = 1 / tz * cam.focal_y
    J[..., 1, 2] = -ty / (tz * tz) * cam.focal_y
    Wm = V[:3, :3].T
    cov2d = (J @ Wm @ cov3d @ Wm.T @ J.permute(0, 2, 1))[:, :2, :2] + torch.eye(2) * 0.3
    po = torch.cat([means3D, torch.ones_like(means3D[..., :1])], dim=-1)
    ph = po @ V @ P
    pw = 1.0 / (ph[..., -1:] + 0.000001)
    ndc = ph * pw
    pview = po @ V
    in_mask = pview[..., 2] <= -0.000001
    mx = ((ndc[..., 0] + 1) * W_ - 1.0) * 0.5
    my = ((ndc[..., 1] + 1) * H_ - 1.0) * 0.5
    det = cov2d[:, 0, 0] * cov2d[:, 1, 1] - cov2d[:, 0, 1] * cov2d[:, 1, 0]
    mid = 0.5 * (cov2d[:, 0, 0] + cov2d[:, 1, 1])
    root = torch.sqrt((mid ** 2 - det).clip(min=0.1))
    radii = 3.0 * torch.sqrt(torch.max(mid + root, mid - root)).ceil()
    rmin_x = (mx - radii).clip(0, W_ - 1.0)
    rmin_y = (my - radii).clip(0, H_ - 1.0)
    rmax_x = (mx + radii).clip(0, W_ - 1.0)
    rmax_y = (my + radii).clip(0, H_ - 1.0)
    return dict(mx=mx, my=my, depth=pview[..., 2], cov2d=cov2d, radii=radii, in_mask=in_mask,
                rmin_x=rmin_x, rmin_y=rmin_y, rmax_x=rmax_x, rmax_y=rmax_y)


def quadtree_leaves(W_, H_, rmin_x, rmin_y, rmax_x, rmax_y, max_tile_size=60, max_gaussians_per_tile=60000):
    """gauss_render.py:290-335 as an explicit BFS.  rect arrays are float32 numpy over the in-frustum Gaussians.
    Returns (leaves, background_tiles): leaves = list of (r0, c0, w, h, member_index_array) in BFS order."""
    q = deque([(0, 0, W_, H_)])
    leaves, background = [], []
    f = np.float32
    while q:
        r0, c0, w, h = q.popleft()
        if w <= 1 or h <= 1:
            continue
        w = min(w, W_ - c0)
        h = min(h, H_ - r0)
        tl_x = np.maximum(rmin_x, f(c0))
        tl_y = np.maximum(rmin_y, f(r0))
        br_x = np.minimum(rmax_x, f(c0 + w - 1))
        br_y = np.minimum(rmax_y, f(r0 + h - 1))
        member = (br_x > tl_x) & (br_y > tl_y)
        cnt = int(member.sum())
        if cnt <= 0:
            background.append((r0, c0, w, h))
            continue
        if cnt > max_gaussians_per_tile or w > max_tile_size or h > max_tile_size:
            w2, h2 = math.ceil(w / 2), math.ceil(h / 2)
            q.append((r0, c0, w2, h2))
            q.append((r0 + h2, c0, w2, h2))
            q.append((r0, c0 + w2, w2, h2))
            q.append((r0 + h2, c0 + w2, w2, h2))
            continue
        leaves.append((r0, c0, w, h, np.nonzero(member)[0]))
    return leaves, background


def blend_leaf(r0, c0, w, h, mx, my, conic, opacity, colour, white_bkgd=True):
    """gauss_render.py:337-369 for one leaf whose Gaussians are already depth-ordered (nearest first), as a
    sequential front-to-back loop per pixel: weight -> alpha = min(0.99, w*o) -> contribution T*alpha -> T *= 1-alpha.
    float32 geometry, float64 colour accumulation (the reference's colour tensor is f64).
    Returns (tile_colour (h*w,3) f64, contribution (h*w, G) f32)."""
    ys, xs = np.meshgrid(np.arange(r0, r0 + h), np.arange(c0, c0 + w), indexing="ij")
    px = xs.reshape(-1).astype(np.float32)
    py = ys.reshape(-1).astype(np.float32)
    npx = px.shape[0]
    G = mx.shape[0]
    T = np.ones(npx, dtype=np.float32)
    acc = np.zeros(npx, dtype=np.float32)
    col = np.zeros((npx, 3), dtype=np.float64)
    contrib = np.zeros((npx, G), dtype=np.float32)
    for j in range(G):
        dx = px - mx[j]
        dy = py - my[j]
        power = np.float32(-0.5) * (dx * dx * conic[j, 0, 0] + dy * dy * conic[j, 1, 1] + dx * dy * conic[j, 0, 1]
                                    + dx * dy * conic[j, 1, 0])
        wgt = np.exp(power, dtype=np.float32)
        alpha = np.minimum(wgt * opacity[j], np.float32(0.99))
        c = T * alpha
        contrib[:, j] = c
        acc += c
        col += c[:, None].astype(np.float64) * colour[j][None, :]
        T = T * (np.float32(1.0) - alpha)
    bg = 1.0 if white_bkgd else 0.0
    col = col + (1.0 - acc.astype(np.float64))[:, None] * bg
    return col, contrib


def blend_leaf_dense(r0, c0, w, h, mx, my, conic, opacity, colour, white_bkgd=True):
    """Same leaf blend as blend_leaf but with the reference's dense (pixels x Gaussians) tensor formulation
    (gauss_render.py:353-385: broadcast dx, exp, clip, exclusive cumprod, reductions) on torch-CPU, multi-threaded —
    the form the reference's own CPU run takes; used as the CPU baseline.  Returns (tile_colour, best, argbest)."""
    ys, xs = torch.meshgrid(torch.arange(r0, r0 + h), torch.arange(c0, c0 + w), indexing="ij")
    coord = torch.stack([xs.reshape(-1), ys.reshape(-1)], dim=-1)  # int64 (x, y) per pixel, row-major
    m2 = torch.as_tensor(np.stack([mx, my], axis=-1))
    con = torch.as_tensor(conic)
    op = torch.as_tensor(opacity).reshape(-1, 1)
    colr = torch.as_tensor(colour)
    dx = coord[:, None, :] - m2[None, :]
    wgt = torch.exp(-0.5 * (dx[:, :, 0] ** 2 * con[:, 0, 0] + dx[:, :, 1] ** 2 * con[:, 1, 1]
                            + dx[:, :, 0] * dx[:, :, 1] * con[:, 0, 1] + dx[:, :, 0] * dx[:, :, 1] * con[:, 1, 0]))
    alpha = (wgt[..., None] * op[None]).clip(max=0.99)
    T = torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha[:, :-1]], dim=1).cumprod(dim=1)
    acc = (alpha * T).sum(dim=1)
    bg = 1 if white_bkgd else 0
    col = (T * alpha * colr[None]).sum(dim=1) + (1 - acc) * bg
    best = torch.max((T * alpha).squeeze(2), 0)
    return col.numpy(), best[0].numpy(), best[1].numpy()


class PythonRendererOracle:
    """Restatement of GaussPythonRenderer (gauss_render.py:210-465) with pinned tile parameters."""

    def __init__(self, means3D, opacity, colour, cov3d, max_tile_size=60, max_gaussians_per_tile=60000, shs=None,
                 sh_degree=0, dense=False):
        self.dense = dense
        self.means3D = torch.as_tensor(means3D, dtype=torch.float32)
        self.opacity = torch.as_tensor(opacity, dtype=torch.float32).reshape(-1)
        self.colour = None if colour is None else torch.as_tensor(colour, dtype=torch.float64)
        self.cov3d = torch.as_tensor(cov3d, dtype=torch.float32)
        self.shs = None if shs is None else torch.as_tensor(shs, dtype=torch.float32)
        self.sh_degree = sh_degree
        n = self.means3D.shape[0]
        self.gaussian_max_contribution = np.zeros(n, dtype=np.float32)
        self.gaussian_colours = np.zeros((n, 3), dtype=np.float64)
        self.max_tile_size = max_tile_size
        self.max_gaussians_per_tile = max_gaussians_per_tile
        self.last = None

    def camera_colour(self, cam):
        if self.shs is None:
            return self.colour
        d = self.means3D - cam.camera_center[None, :]
        d = d / d.norm(dim=1, keepdim=True)
        return sh_colour(self.sh_degree, self.shs, d).to(torch.float64)

    def __call__(self, cam):
        pr = project(self.means3D, self.cov3d, cam)
        vis = np.nonzero(pr["in_mask"].numpy())[0]
        g = lambda k: pr[k][pr["in_mask"]].numpy()
        mx, my, depth = g("mx"), g("my"), g("depth")
        cov2d = pr["cov2d"][pr["in_mask"]]
        opacity = self.opacity[pr["in_mask"]].numpy()
        colour = self.camera_colour(cam)[pr["in_mask"]].numpy()
        W_, H_ = cam.image_width, cam.image_height
        leaves, background = quadtree_leaves(W_, H_, g("rmin_x"), g("rmin_y"), g("rmax_x"), g("rmax_y"),
                                             self.max_tile_size, self.max_gaussians_per_tile)
        image = np.ones((H_, W_, 3), dtype=np.float32)
        leaf_info = []
        for (r0, c0, w, h, members) in leaves:
            # nearest first: view-space z is negative in front of the camera; descending z (gauss_render.py:340-344).
            # ties are broken by Gaussian index (the reference's sort is unstable there).
            order = np.lexsort((members, -depth[members]))
            ids = members[order]
            conic = torch.inverse(cov2d[ids]).numpy()
            if self.dense:
                col, best, arg = blend_leaf_dense(r0, c0, w, h, mx[ids], my[ids], conic, opacity[ids], colour[ids])
            else:
                col, contrib = blend_leaf(r0, c0, w, h, mx[ids], my[ids], conic, opacity[ids], colour[ids])
                best = contrib.max(axis=0)
                arg = contrib.argmax(axis=0)
            image[r0:r0 + h, c0:c0 + w] = col.reshape(h, w, 3).astype(np.float32)
            gl = vis[ids]
            upd = best > self.gaussian_max_contribution[gl]
            self.gaussian_max_contribution[gl[upd]] = best[upd]
            self.gaussian_colours[gl[upd]] = col[arg[upd]]
            leaf_info.append((r0, c0, w, h, gl))
        self.last = dict(proj=pr, leaves=leaf_info, background=background)
        return image[:, ::-1].copy()

    def get_gaussian_colours(self):
        return self.gaussian_colours * 255
