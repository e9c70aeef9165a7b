"""Deterministic synthetic 3DGS scenes and camera rigs (BASELINE.md §3.2) for tests and bench.py.

Everything is generated on the CPU with a seeded torch.Generator and moved to the device by the caller, so the
same scene is seen by the GPU path and by the CPU oracle; sampled_cloud is the exception, a point cloud sampled on the
device from such a scene.
"""
import math

import torch

SH_C0 = 0.28209479177387814


def make_scene(n, seed=1234, sh_degree=3, dtype_like_ply=True):
    """n synthetic Gaussians.  Returns a dict of CPU tensors with the dtypes the reference's .ply loader yields
    (gauss_dataloader.py:16-82): xyz f32, scales f64 (log-space), rots f64 (normalised), opacities f32 in (0,1),
    shs (n,3,(deg+1)^2) f64 channel-major, colours f64 = clip(C0*DC + 0.5, 0, 1)."""
    g = torch.Generator(device="cpu")
    g.manual_seed(seed)
    d = torch.randn(n, 3, generator=g)
    d = d / d.norm(dim=1, keepdim=True).clamp_min(1e-12)
    r = 1.5 + 0.15 * torch.randn(n, 1, generator=g)
    xyz = d * r
    floaters = torch.rand(n, generator=g) < 0.10
    xyz[floaters] = (torch.rand(int(floaters.sum()), 3, generator=g) * 6.0 - 3.0)
    scales = -4.2 + 0.8 * torch.randn(n, 3, generator=g)
    amin = scales.argmin(dim=1)
    scales[torch.arange(n), amin] -= 1.0
    rots = torch.randn(n, 4, generator=g)
    rots = rots / rots.norm(dim=1, keepdim=True).clamp_min(1e-12)
    opac = torch.sigmoid(0.5 + 2.0 * torch.randn(n, generator=g))
    ncoef = (sh_degree + 1) ** 2
    shs = 0.05 * torch.randn(n, 3, ncoef, generator=g)
    shs[:, :, 0] = 0.8 * torch.randn(n, 3, generator=g)
    colours = (SH_C0 * shs[:, :, 0].double() + 0.5).clip(0, 1)
    out = {
        "xyz": xyz.float().contiguous(),
        "scales": scales.double() if dtype_like_ply else scales.float(),
        "rots": rots.double() if dtype_like_ply else rots.float(),
        "opacities": opac.float().contiguous(),
        "shs": shs.double() if dtype_like_ply else shs.float(),
        "colours": colours,
    }
    return out


def sampled_cloud(n_gaussians, num_points, seed, device):
    """PointCloudData of make_scene(n_gaussians, seed) sampled on `device` the way the CLI samples with
    --no_render_colours; with 3 M Gaussians and 10 M points, the C3-like cloud of the point-cloud benchmarks."""
    import gauss_to_pc as g2p
    from . import sampler
    sc = {k: v.to(device) for k, v in make_scene(n_gaussians, seed=seed).items()}
    st = g2p.GaussPointCloudSettings(
        renderer_type="python", num_points=num_points, prioritise_visible_gaussians=True, mahalanobis_distance_std=2.0,
        camera_skip_rate=0, render_colours=False, min_opacity=0.0, bounding_box_min=None, bounding_box_max=None,
        calculate_normals=True, cull_large_percentage=0.0, remove_unrendered_gaussians=True, colour_resolution=None,
        max_sh_degree=3, exact_num_points=False, visibility_threshold=0.05, surface_distance_std=None,
        generate_mesh=False, quiet=True, device=device)
    sampler.reset_call_counter(0)
    pc, _ = g2p.convert_gaussians_to_pc(sc["xyz"], sc["scales"], sc["rots"], sc["colours"].clone() * 255,
                                        sc["opacities"], sc["shs"], None, None, None, st)
    return pc


def look_at_c2w(eye, target=(0.0, 0.0, 0.0), up=(0.0, 0.0, 1.0)):
    """OpenGL camera-to-world (x right, y up, camera looks down -z), 4x4 f32."""
    eye = torch.tensor(eye, dtype=torch.float64)
    target = torch.tensor(target, dtype=torch.float64)
    up = torch.tensor(up, dtype=torch.float64)
    f = target - eye
    f = f / f.norm()
    s = torch.linalg.cross(f, up)
    s = s / s.norm()
    u = torch.linalg.cross(s, f)
    c2w = torch.eye(4, dtype=torch.float64)
    c2w[:3, 0] = s
    c2w[:3, 1] = u
    c2w[:3, 2] = -f
    c2w[:3, 3] = eye
    return c2w.float()


def make_cameras(m, radius=4.5, height=1.5, turns=2.0, intrinsics=(1920, 1080, 1600.0, 1600.0)):
    """m poses on a `turns`-turn spiral of `radius` around the origin, height from -height to +height, looking at
    the origin.  Returns (list of 4x4 c2w f32 tensors, list of [w, h, fx, fy])."""
    cams, intr = [], []
    for i in range(m):
        t = (i + 0.5) / m
        ang = 2.0 * math.pi * turns * t
        z = -height + 2.0 * height * t
        eye = (radius * math.cos(ang), radius * math.sin(ang), z)
        cams.append(look_at_c2w(eye))
        intr.append(list(intrinsics))
    return cams, intr
