"""Oracle restatement of the per-Gaussian scene model on the hot path (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows gauss_handler.py; torch-CPU ops are used where the reference's arithmetic is a torch
library routine (bmm, eigvals, eigh) so that the CPU result has the same rounding behaviour.
"""
import math

import torch


def build_rotation(q):
    """gauss_handler.py:26-47 — R(q), q = (r,x,y,z) NOT normalised; elements formed in q's dtype, stored f32."""
    q = torch.as_tensor(q)
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.empty((q.shape[0], 3, 3), dtype=torch.float32)
    R[:, 0, 0] = 1 - 2 * (y * y + z * z)
    R[:, 0, 1] = 2 * (x * y - r * z)
    R[:, 0, 2] = 2 * (x * z + r * y)
    R[:, 1, 0] = 2 * (x * y + r * z)
    R[:, 1, 1] = 1 - 2 * (x * x + z * z)
    R[:, 1, 2] = 2 * (y * z - r * x)
    R[:, 2, 0] = 2 * (x * z - r * y)
    R[:, 2, 1] = 2 * (y * z + r * x)
    R[:, 2, 2] = 1 - 2 * (x * x + y * y)
    return R


def build_covariance(scales, rots, scaling_modifier=1.0):
    """gauss_handler.py:49-63 — L = R diag(exp(mod*s)) (exp in the input dtype, stored f32), Sigma = L L^T (f32)."""
    scales = torch.as_tensor(scales)
    R = build_rotation(rots)
    e = torch.exp(scaling_modifier * scales).to(torch.float32)  # rounded to f32 on assignment (:53-55)
    L = R * e[:, None, :]  # R @ diag(e): exact per element
    return L @ L.transpose(1, 2)


def calculate_normals(scales, rots):
    """gauss_handler.py:89-106 — normal = column argmin(scale) of R(q)."""
    scales = torch.as_tensor(scales)
    idx = torch.min(scales, 1)[1]
    R = build_rotation(rots)
    return R[torch.arange(R.shape[0]), :, idx]


def sqrt_surface_area(cov):
    """gauss_handler.py:259-270 — eigvals (general solver, f32) -> ellipsoid surface area (p=1.6075) -> sqrt."""
    ev = torch.linalg.eigvals(torch.as_tensor(cov)).real
    p = 1.6075
    a, b, c = torch.sqrt(ev[:, 0]), torch.sqrt(ev[:, 1]), torch.sqrt(ev[:, 2])
    radicand = (torch.pow(a * b, p) + torch.pow(a * c, p) + torch.pow(b * c, p)) / 3.0
    return torch.sqrt(4.0 * math.pi * torch.pow(radicand, 1.0 / p))


def gaussian_magnitudes(cov, contributions):
    """gauss_handler.py:252-279 — sqrt(area) * contribution, cast to f64."""
    return (sqrt_surface_area(cov) * torch.as_tensor(contributions)).to(torch.float64)


def validate_covariances(cov, epsilon=1e-7, min_ps_epsilon=1e-8, num_clamp_iters=3, reg=5e-7):
    """gauss_handler.py:108-166 — +5e-7*I, up to 3 eigen-clamp rounds on Gaussians with an eigenvalue <= 1e-7,
    then flag (for removal) those that still have an eigenvalue <= 1e-8.  Returns (cov, keep_mask)."""
    cov = torch.as_tensor(cov).clone()
    cov += reg * torch.eye(3)

    def bad(c, eps):
        return torch.any(torch.linalg.eigvals(c).real <= eps, 1)

    for _ in range(num_clamp_iters):
        m = bad(cov, epsilon)
        if m.sum() > 0:
            w, v = torch.linalg.eigh(cov[m])
            w = torch.clamp(w, min=epsilon)
            cov[m] = v @ torch.diag_embed(w) @ v.transpose(-1, -2)
    keep = ~bad(cov, min_ps_epsilon)
    return cov, keep
