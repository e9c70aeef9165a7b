"""Feeding the CUDA back-end's own per-camera outputs to the float64 blend (tests/f64ref.py): one renderer over a scene,
and one camera rendered with the per-camera records (maximum, arg-max pixel, surface distance) switched on."""
import numpy as np
import torch

from util import scene_to

DEV = "cuda:0"


def cuda_setup(sc, surf=True):
    """GaussianRasterizer over scene `sc` with precomputed colours and the oracle's covariances."""
    from g2pc.rasterizer import GaussianRasterizer
    from oracle import gaussians as og
    cov = og.build_covariance(sc["scales"], sc["rots"])
    d = scene_to(sc, DEV)
    R = GaussianRasterizer(d["xyz"], None, d["opacities"], colors_precomp=d["colours"].float(),
                           cov3D_precomp=cov.to(DEV), calculate_surface_distance=surf)
    return R, d, cov


def tiles_camera(R, rs):
    """Render camera `rs` on R (its accumulators are updated as by any call) and return this camera's outputs as numpy:
    image (3,H,W), depth (H,W), invdepth (H,W), radii, the projection records rec (n,12) and their ok mask, and the
    per-camera maximum contrib, arg-max pixel and surface distance (FLT_MAX where none)."""
    n = R._n
    contrib = torch.zeros((n,), dtype=torch.float32, device=DEV)
    pixels = torch.zeros((n,), dtype=torch.int32, device=DEV)
    surf = torch.full((n,), torch.finfo(torch.float).max, dtype=torch.float32, device=DEV)
    R._per_camera = (contrib, pixels, surf)
    img, radii, invd, dep = R(rs)
    R._per_camera = None
    sl = R._slots[R._last_slot]
    ok = sl["depth_key"].cpu().numpy().view(np.uint32) != 0xFFFFFFFF
    return dict(image=img.cpu().numpy(), depth=dep.cpu().numpy()[0], invdepth=invd.cpu().numpy()[0],
                radii=radii.cpu().numpy(), rec=sl["proj"].cpu().numpy(), ok=ok, contrib=contrib.cpu().numpy(),
                pixel=pixels.cpu().numpy(), surface=surf.cpu().numpy())
