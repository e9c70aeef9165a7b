"""Restatement of the TSDF fusion mesher's rules (N10, DESIGN.md §2, csrc/s14_tsdf.cu) in numpy: the grid frame, the
per-camera integration, the gather that keeps the surface of observed voxels and its compaction.  The float64 steps are
plain numpy float64 operations in the kernel's order (numpy never contracts to FMA) and the float32 steps numpy float32
operations, each correctly rounded like the kernel's _rn intrinsics: fed the kernel's images, the grid must agree bit
for bit.  Also synthetic depth maps of a sphere, for checks without a GPU."""
import numpy as np

import f64ref as fr
import f64ref_mesh as fm

F32 = np.float32


def frame(points, depth):
    """N6's frame rule: dict(origin, h, L, extent, R)."""
    return fm.frame(points, depth)


def new_grid(R):
    cells = R ** 3
    return dict(tsdf=np.ones(cells, F32), weight=np.zeros(cells, F32), colour=np.zeros((3, cells), F32))


def voxel_centres(fr):
    R = fr["R"]
    idx = np.arange(R ** 3, dtype=np.int64)
    i, j, k = idx % R, (idx // R) % R, idx // (R * R)
    o, h = fr["origin"], fr["h"]
    return [o[a] + (c.astype(np.float64) + 0.5) * h for a, c in enumerate((i, j, k))]


def _affine(M, c, x, y, z):
    return ((M[c] * x + M[4 + c] * y) + M[8 + c] * z) + M[12 + c]


def project(fr, view, proj, W, H):
    """Per voxel: view depth z, nearest pixel (ix, iy) as float64 (floor(pix + 1/2)), the float64 pixel coordinates."""
    x, y, z = voxel_centres(fr)
    V = np.asarray(view, np.float32).astype(np.float64).reshape(-1)
    P = np.asarray(proj, np.float32).astype(np.float64).reshape(-1)
    zv = _affine(V, 2, x, y, z)
    hx, hy, hw = _affine(P, 0, x, y, z), _affine(P, 1, x, y, z), _affine(P, 3, x, y, z)
    with np.errstate(divide="ignore", invalid="ignore"):
        pw = 1.0 / (hw + 1e-7)
        px = ((hx * pw + 1.0) * W - 1.0) * 0.5
        py = ((hy * pw + 1.0) * H - 1.0) * 0.5
    return zv, np.floor(px + 0.5), np.floor(py + 0.5), px, py


def integrate(grid, fr, trunc, zmed, T, image, mask, view, proj, bg):
    """One camera into grid (in place).  zmed, T (H,W) f32, image (3,H,W) f32, mask (H*W) or None, view / proj the 16
    float32 matrix entries (row-major, row-vector convention), bg (3,).  Returns the boolean mask of updated voxels."""
    H, W = zmed.shape
    zv, fx, fy, _, _ = project(fr, view, proj, W, H)
    with np.errstate(invalid="ignore"):
        ok = (zv > 0.2) & (fx >= 0) & (fx < W) & (fy >= 0) & (fy < H)
    idx = np.nonzero(ok)[0]
    pix = fy[idx].astype(np.int64) * W + fx[idx].astype(np.int64)
    if mask is not None:
        sel = np.asarray(mask).reshape(-1)[pix] != 0
        idx, pix = idx[sel], pix[sel]
    zm = zmed.reshape(-1)[pix]
    idx, pix, zm = idx[zm != 0], pix[zm != 0], zm[zm != 0]
    mu = F32(trunc * fr["h"])
    sdf = zm.astype(F32) - zv[idx].astype(F32)
    keep = ~(sdf < -mu)
    idx, pix, sdf = idx[keep], pix[keep], sdf[keep]
    tv = np.minimum(F32(1), sdf / mu)
    Tp = T.reshape(-1)[pix].astype(F32)
    w = grid["weight"][idx]
    w1 = w + F32(1)
    grid["tsdf"][idx] = (grid["tsdf"][idx] * w + tv) / w1
    img = image.reshape(3, -1)
    for c in range(3):
        raw = (img[c][pix] - Tp * F32(bg[c])) / (F32(1) - Tp)
        cc = np.minimum(np.maximum(raw, F32(0)), F32(1))
        grid["colour"][c][idx] = (grid["colour"][c][idx] * w + cc) / w1
    grid["weight"][idx] = w1
    out = np.zeros(zv.shape[0], bool)
    out[idx] = True
    return out


def gather(weight, colour, R, vkey, vt):
    """(keep (m,) bool, density (m,) float64, colours (m,3) uint8) of the extraction's vertices."""
    vkey = np.asarray(vkey, np.int64)
    a, d = vkey >> 3, vkey & 7
    b = a + (d & 1) + ((d >> 1) & 1) * R + (d >> 2) * R * R
    wa, wb = weight[a].astype(np.float64), weight[b].astype(np.float64)
    t = np.asarray(vt, np.float64)
    s = 1.0 - t
    col = np.empty((vkey.size, 3), np.uint8)
    for c in range(3):
        x = s * colour[c][a].astype(np.float64) + t * colour[c][b].astype(np.float64)
        col[:, c] = np.clip(np.floor(255.0 * x + 0.5), 0, 255).astype(np.uint8)
    return (wa > 0) & (wb > 0), s * wa + t * wb, col


def compact(keep, vpos, faces, *per_vertex):
    """The kept vertices in order and the triangles whose three vertices are kept, re-indexed."""
    keep = np.asarray(keep, bool)
    faces = np.asarray(faces, np.int64).reshape(-1, 3)
    tk = keep[faces].all(1)
    vmap = np.cumsum(keep) - 1
    return (np.asarray(vpos)[keep], vmap[faces[tk]]) + tuple(np.asarray(x)[keep] for x in per_vertex)


def mesh(grid, fr):
    """Marching tetrahedra of the tsdf at iso 0, then gather and compaction: (vpos, faces, colours, density, keep)."""
    R = fr["R"]
    vkey, vt, vpos, faces = fm.marching_tetrahedra(grid["tsdf"], R, 0.0, fr["origin"], fr["h"])
    keep, dens, col = gather(grid["weight"], grid["colour"], R, vkey, vt)
    v, f, c, d = compact(keep, vpos, faces, col, dens)
    return v, f, c, d, keep


# ---- the fusion blend's median depth -----------------------------------------------------------------------------
def median_depth(rec, ok, W, H, mask=None, band_alpha=2e-5, band_T=1e-4, band_half=2e-5):
    """T and z_med of g2pc_tiles_blend_fusion in float64, fed the kernel's projection records `rec` and `ok` mask, in the
    kernel's list order (stable by the depth's float bits) with its per-pixel rules: skip power > 0 or alpha < 1/255,
    stop before T (1 - alpha) < 1e-4; z_med = depth of the first taken entry whose step leaves T < 0.5 from T >= 0.5, 0
    when none.  Independent of f64ref.tiles_blend except for the record layout.

    A pixel is `tainted` when a decision that can set z_med may go the other way in float32: a skip or stop within the
    bands of f64ref.tiles_blend up to its crossing (or anywhere, when it has none), or a taken step whose T after it lies
    within band_half of 0.5.  Returns T (H,W), z_med (H,W) and tainted (H,W); masked pixels hold 0 and are not tainted."""
    mflat = None if mask is None else np.asarray(mask).reshape(-1) != 0
    px, py = rec[:, 0].astype(np.float64), rec[:, 1].astype(np.float64)
    kx, ky, kz = rec[:, 2] / fr.K_EXP2, rec[:, 3] / (2 * fr.K_EXP2), rec[:, 4] / fr.K_EXP2
    op = np.exp2(rec[:, 5].astype(np.float64))
    depth = rec[:, 9]
    x0, x1, y0, y1 = fr.unpack_rect(rec[:, 11])
    idx = np.nonzero(ok)[0]
    order = idx[np.argsort(rec[idx, 9].view(np.uint32), kind="stable")]
    Timg, zimg, timg = np.zeros((H, W)), np.zeros((H, W)), np.zeros((H, W), bool)
    for ty in range((H + 15) // 16):
        for tx in range((W + 15) // 16):
            sel = order[(x0[order] <= tx) & (tx <= x1[order]) & (y0[order] <= ty) & (ty <= y1[order])]
            ys, xs = np.meshgrid(np.arange(ty * 16, ty * 16 + 16), np.arange(tx * 16, tx * 16 + 16), indexing="ij")
            ys, xs = ys.reshape(-1), xs.reshape(-1)
            live = (xs < W) & (ys < H)
            if mflat is not None:
                live[live] = mflat[(ys * W + xs)[live]]
            T, z = np.ones(256), np.zeros(256)
            done, crossed, tainted = ~live, np.zeros(256, bool), np.zeros(256, bool)
            for g in sel:
                if done.all():
                    break
                dx, dy = px[g] - xs, py[g] - ys
                power = -0.5 * (kx[g] * dx * dx + kz[g] * dy * dy) - ky[g] * dx * dy
                alpha = np.minimum(0.99, op[g] * np.exp(power))
                act = ~done
                keep = act & ~(power > 0) & ~(alpha < 1.0 / 255.0)
                testT = T * (1.0 - alpha)
                near = (act & (power <= 0) & (np.abs(alpha * 255.0 - 1.0) < band_alpha)) | \
                       (keep & (np.abs(testT / 1e-4 - 1.0) < band_T))
                stop = keep & (testT < 1e-4)
                take = keep & ~stop
                tainted |= near & ~crossed
                tainted |= take & ~crossed & (np.abs(testT - 0.5) < band_half)
                cross = take & (testT < 0.5) & (T >= 0.5)
                z = np.where(cross, float(depth[g]), z)
                crossed |= cross
                done |= stop
                T = np.where(take, testT, T)
            w = (xs < W) & (ys < H)
            lv = live[w]
            Timg[ys[w], xs[w]] = np.where(lv, T[w], 0.0)
            zimg[ys[w], xs[w]] = np.where(lv, z[w], 0.0)
            timg[ys[w], xs[w]] = lv & tainted[w]
    return Timg, zimg, timg


# ---- synthetic depth maps -------------------------------------------------------------------------------------------
def sphere_images(rs, radius=1.0, colour=(0.2, 0.6, 0.9)):
    """Exact renders of an opaque sphere at the origin for the CUDA back-end's raster settings rs (host matrices):
    z_med = view depth of the first hit of each pixel centre's ray (0 on a miss), T = 0 on a hit and 1 on a miss,
    image = colour on a hit and the background on a miss."""
    W, H = int(rs.image_width), int(rs.image_height)
    V = np.asarray(rs._viewmatrix_host, np.float64).reshape(4, 4)
    tx, ty = float(rs.tanfovx), float(rs.tanfovy)
    u, v = np.meshgrid(np.arange(W), np.arange(H))
    d_view = np.stack([((2 * u + 1) / W - 1) * tx, ((2 * v + 1) / H - 1) * ty, np.ones_like(u, float)], -1)
    Rm = V[:3, :3]  # p_view = p_world Rm + t
    d = d_view @ Rm.T
    c = np.asarray(rs._campos_host, np.float64)
    a = (d * d).sum(-1)
    b = 2 * (d @ c)
    cc = c @ c - radius ** 2
    disc = b * b - 4 * a * cc
    hit = disc >= 0
    s = np.where(hit, (-b - np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
    if cc < 0:  # inside: the far root
        s = np.where(hit, (-b + np.sqrt(np.maximum(disc, 0))) / (2 * a), 0.0)
    hit &= s > 0.2
    zmed = np.where(hit, s, 0.0).astype(F32)
    T = np.where(hit, 0.0, 1.0).astype(F32)
    bg = np.asarray(rs._bg_host, F32)
    image = np.stack([np.where(hit, F32(colour[k]), bg[k]) for k in range(3)]).astype(F32)
    return zmed, T, image
