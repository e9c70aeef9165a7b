"""Scene model of the hot path — drop-in for the reference's gauss_handler.py (same names, arguments, attributes).

Reference: gauss_handler.py (Gaussians :65-279, covariance helpers :12-63).  The arithmetic-heavy
members run as hand-written sm_90a kernels behind the C ABI (include/g2pc.h):
    build_covariance_from_scaling_rotation -> g2pc_cov_build        (csrc/s1_cov.cu)
    Gaussians.calculate_normals            -> g2pc_normals
    torch.linalg.eigvals(...).real         -> g2pc_eigvals_sym3     (used by validate_covariances / magnitudes)
Tensors must live on a CUDA device; there is no CPU fallback.
"""
from math import floor

import torch

from g2pc import capi


def _as_kernel_input(t):
    """f32 / f64 tensors go to the kernels as they are; anything else is promoted to f32."""
    if t.dtype not in (torch.float32, torch.float64):
        t = t.to(torch.float32)
    return t.contiguous()


def strip_lowerdiag(L):
    """(N,3,3) -> (N,6) [00,01,02,11,12,22]  (gauss_handler.py:12-21)."""
    idx = torch.tensor([0, 1, 2, 4, 5, 8], device=L.device)
    return L.reshape(L.shape[0], 9).index_select(1, idx).to(torch.float)


def strip_symmetric(sym):
    return strip_lowerdiag(sym)


def build_rotation(q):
    """R(q) for q = (r, x, y, z), not re-normalised (gauss_handler.py:26-47).  (N,3,3) f32."""
    q = _as_kernel_input(q)
    capi.require_cuda(q)
    # R is the covariance of unit scales' "L" factor: reuse the normals kernel column by column would cost 3
    # launches; the rotation itself is only needed by callers outside the hot path, so form it with torch ops.
    r, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    R = torch.stack([
        1 - 2 * (y * y + z * z), 2 * (x * y - r * z), 2 * (x * z + r * y),
        2 * (x * y + r * z), 1 - 2 * (x * x + z * z), 2 * (y * z - r * x),
        2 * (x * z - r * y), 2 * (y * z + r * x), 1 - 2 * (x * x + y * y)], dim=1)
    return R.to(torch.float32).reshape(-1, 3, 3)


def build_scaling_rotation(s, r):
    """L = R(r) @ diag(exp(s))  (gauss_handler.py:49-58).  (N,3,3) f32."""
    R = build_rotation(r)
    return R * torch.exp(s).to(torch.float32)[:, None, :]


def build_covariance_from_scaling_rotation(scaling, scaling_modifier, rotation):
    """Sigma = L L^T, L = R diag(exp(mod * s))  (gauss_handler.py:60-63) — one fused kernel.  (N,3,3) f32."""
    lib = capi.load()
    scaling = _as_kernel_input(scaling)
    rotation = _as_kernel_input(rotation)
    capi.require_cuda(scaling, rotation)
    if scaling.dtype != rotation.dtype:
        scaling, rotation = scaling.to(torch.float64), rotation.to(torch.float64)
    n = scaling.shape[0]
    if scaling.shape[1] != 3 or rotation.shape != (n, 4):
        raise ValueError("scaling must be (N,3) and rotation (N,4)")
    cov = torch.empty((n, 3, 3), dtype=torch.float32, device=scaling.device)
    capi.call("g2pc_cov_build", capi.ptr(scaling), capi.ptr(rotation), capi.dtype_code(scaling),
                                  float(scaling_modifier), n, capi.ptr(cov), capi.stream_ptr(scaling.device))
    return cov


def eigvals_sym3(covariances):
    """Eigenvalues (ascending, f32) of a batch of symmetric 3x3 — stands in for torch.linalg.eigvals(...).real."""
    lib = capi.load()
    capi.require_cuda(covariances)
    c = covariances.to(torch.float32).contiguous()
    ev = torch.empty((c.shape[0], 3), dtype=torch.float32, device=c.device)
    capi.call("g2pc_eigvals_sym3", capi.ptr(c), c.shape[0], capi.ptr(ev), capi.stream_ptr(c.device))
    return ev


class Gaussians():
    """
    Manages all loaded gaussians in the renderer  (reference: gauss_handler.py:65-279)

    `scales`, `rots` and `shs` are not read by anything after the colour stage; filters applied through fused_cull() keep
    them lazily (original tensor + pending row index) and materialise them on first access, so the 576 MB SH gather of a
    3 M-Gaussian scene is only paid by a caller that actually looks at them.
    """
    _LAZY = ("scales", "rots", "shs")

    def __init__(self, xyz, scales, rots, colours, opacities, shs=None):
        capi.require_cuda(xyz, scales, rots, colours, opacities, shs)
        self._lazy = {}
        self.xyz = xyz
        self.scales = scales
        self.rots = rots
        self.opacities = opacities
        self.colours = colours
        self.shs = shs
        self.normals = None
        # original row of every Gaussian: follows the culls, keys the sampler's RNG (so that the drawn points do not
        # depend on how the array is culled or sharded)
        self.ids = torch.arange(xyz.shape[0], dtype=torch.int32, device=xyz.device)

        self.scaling_modifier = 1.0

        # 3D covariance matrices (S1 kernel)
        self.covariances = build_covariance_from_scaling_rotation(scales, self.scaling_modifier, rots)

        self.set_default_filter()

    # ---- lazily filtered attributes ---------------------------------------------------------------------------------
    def __setattr__(self, name, value):
        if name in Gaussians._LAZY:
            self.__dict__["_lazy"][name] = (value, None)
        else:
            object.__setattr__(self, name, value)

    def __getattr__(self, name):  # only reached for names without a regular attribute
        if name in Gaussians._LAZY:
            tensor, idx = self.__dict__["_lazy"][name]
            if idx is not None and tensor is not None:
                tensor = tensor.index_select(0, idx)
                self.__dict__["_lazy"][name] = (tensor, None)
            return tensor
        raise AttributeError(name)

    def _lazy_filter(self, index64):
        for name, (tensor, idx) in list(self._lazy.items()):
            if tensor is not None:
                self._lazy[name] = (tensor, index64 if idx is None else idx.index_select(0, index64))

    def fused_cull(self, max_contribution=None, visibility_threshold=0.0, min_opacity=0.0, bounding_box_min=None,
                   bounding_box_max=None, surface_distance=None, surface_threshold=None, extra_mask=None,
                   index_range=None):
        """All culls of gauss_to_pc.py:483-496 + filter_gaussians (gauss_handler.py:171-193) as ONE mask / compaction:
        g2pc_cull_select builds the ascending list of kept rows, g2pc_gather_rows compacts xyz, colours, opacities,
        covariances, normals and ids in one call; scales / rots / shs follow lazily.  Also honours the pending
        filter_indices.  Returns the int64 row index of the kept Gaussians (use it like the reference's boolean mask)."""
        import ctypes
        n = self.xyz.shape[0]
        dev = self.xyz.device
        st = capi.stream_ptr(dev)
        f32 = lambda t: None if t is None else t.to(torch.float32).contiguous()
        mc, op, xyz, sd = f32(max_contribution), f32(self.opacities) if min_opacity > 0.0 else None, f32(self.xyz), f32(surface_distance)
        extra = self.filter_indices if not bool(getattr(self, "_filter_is_default", False)) else None
        if extra_mask is not None:
            extra = extra_mask if extra is None else (extra & extra_mask)
        extra_u8 = None if extra is None else extra.to(torch.uint8).contiguous()
        thr = None
        if sd is not None:
            thr = torch.as_tensor(surface_threshold, dtype=torch.float32, device=dev).reshape(1).contiguous()
        bmin = (ctypes.c_float * 3)(*[float(v) for v in bounding_box_min]) if bounding_box_min is not None else None
        bmax = (ctypes.c_float * 3)(*[float(v) for v in bounding_box_max]) if bounding_box_max is not None else None
        lo, hi = (0, n) if index_range is None else index_range
        index = torch.empty((max(n, 1),), dtype=torch.int32, device=dev)
        count = torch.zeros((1,), dtype=torch.int64, device=dev)
        ws = capi.workspace(capi.load().g2pc_cull_workspace_bytes(n), dev)
        capi.call("g2pc_cull_select", capi.ptr(mc), float(visibility_threshold), capi.ptr(op), float(min_opacity),
                  capi.ptr(xyz), bmin, bmax, capi.ptr(sd), capi.ptr(thr), capi.ptr(extra_u8), int(lo), int(hi), n,
                  capi.ptr(index), capi.ptr(count), capi.ptr(ws), ws.numel(), st)
        m = int(count.item())  # the one host read: output sizes
        index = index[:m]
        names = [k for k in ("xyz", "colours", "opacities", "covariances", "normals", "ids") if getattr(self, k) is not None]
        for name, d in zip(names, capi.gather_rows(index, m, [getattr(self, k) for k in names])):
            setattr(self, name, d)
        index64 = index.to(torch.int64)
        self._lazy_filter(index64)
        self.set_default_filter()
        return index64

    def points_per_gaussian(self, num_points, contributions=None):
        """get_gaussian_magnitudes (gauss_handler.py:252-279) + distribute_points (gauss_to_pc.py:73-90) as one
        entry point without a host round trip.  Returns (points_per_gaussian int32, magnitudes float64)."""
        n = self.xyz.shape[0]
        dev = self.xyz.device
        contrib = (self.opacities if contributions is None else contributions).to(torch.float32).reshape(-1).contiguous()
        cov = self.covariances.to(torch.float32).contiguous()
        mag = torch.empty((max(n, 1),), dtype=torch.float64, device=dev)
        ppg = torch.zeros((max(n, 1),), dtype=torch.int32, device=dev)
        ws = capi.workspace(capi.load().g2pc_ppg_workspace_bytes(n), dev)
        capi.call("g2pc_points_per_gaussian", capi.ptr(cov), capi.ptr(contrib), n, float(num_points), capi.ptr(mag),
                  capi.ptr(ppg), capi.ptr(ws), ws.numel(), capi.stream_ptr(dev))
        return ppg[:n], mag[:n]

    def set_default_filter(self):
        self.filter_indices = torch.ones((self.xyz.shape[0],), dtype=torch.bool, device=self.xyz.device)
        self._filter_is_default = True

    def calculate_normals(self):
        """Normal of each Gaussian = rotated axis of its smallest scale (gauss_handler.py:89-106)."""
        lib = capi.load()
        s = _as_kernel_input(self.scales)
        r = _as_kernel_input(self.rots)
        if s.dtype != r.dtype:
            s, r = s.to(torch.float64), r.to(torch.float64)
        n = s.shape[0]
        normals = torch.empty((n, 3), dtype=torch.float32, device=s.device)
        capi.call("g2pc_normals", capi.ptr(s), capi.ptr(r), capi.dtype_code(s), n, capi.ptr(normals),
                                    capi.stream_ptr(s.device))
        self.normals = normals

    def non_posdef_covariances(self, covariances, epsilon: float = 1e-10):
        """Mask of covariances with an eigenvalue <= epsilon (gauss_handler.py:108-112)."""
        return torch.any(eigvals_sym3(covariances) <= epsilon, 1)

    def clamp_covariances(self, covariances, mask=None, epsilon=1e-6):
        """Clip eigenvalues to >= epsilon (gauss_handler.py:114-127).  Only the (rare) flagged subset goes through
        torch.linalg.eigh."""
        if mask is None:
            mask = torch.ones(covariances.shape[0], dtype=torch.bool, device=covariances.device)
        eigvals, eigvecs = torch.linalg.eigh(covariances[mask])
        eigvals = torch.clamp(eigvals, min=epsilon)
        covariances[mask] = eigvecs @ torch.diag_embed(eigvals) @ eigvecs.transpose(-1, -2)
        return covariances

    def regularise_covariances(self, covariances, mask=None, epsilon=5e-7):
        """covariances (+)= epsilon * I (gauss_handler.py:129-140)."""
        eye = epsilon * torch.eye(3, device=covariances.device, dtype=covariances.dtype)
        if mask is None:
            covariances += eye
        else:
            covariances[mask] += eye
        return covariances

    def validate_covariances(self, regularise=True, epsilon=1e-7, min_ps_epsilon=1e-8, num_clamp_iters=3):
        """Regularise, eigen-clamp up to num_clamp_iters times, then drop Gaussians that still are not
        positive-definite (gauss_handler.py:142-166).  Returns the keep-mask over the Gaussians held on entry."""
        validated = self.regularise_covariances(self.covariances) if regularise else self.covariances

        for _ in range(num_clamp_iters):
            bad = self.non_posdef_covariances(validated, epsilon=epsilon)
            if bool(bad.any()):
                validated = self.clamp_covariances(validated, mask=bad, epsilon=epsilon)
            else:
                break  # nothing changes in further rounds

        self.covariances = validated

        bad = self.non_posdef_covariances(self.covariances, epsilon=min_ps_epsilon)
        if bool(bad.any()):
            self.add_gaussians_to_cull(~bad)
            self.filter_gaussians()

        return ~bad

    def add_gaussians_to_cull(self, indices_to_cull):
        self.filter_indices = self.filter_indices & indices_to_cull
        self._filter_is_default = False

    def filter_gaussians(self):
        """Keep the Gaussians selected by filter_indices (gauss_handler.py:171-193); returns the mask used."""
        keep = torch.clone(self.filter_indices)

        self.xyz = self.xyz[keep]
        self.scales = self.scales[keep]
        self.rots = self.rots[keep]
        self.colours = self.colours[keep]
        self.opacities = self.opacities[keep]
        self.covariances = self.covariances[keep]

        if self.shs is not None:
            self.shs = self.shs[keep]

        if self.normals is not None:
            self.normals = self.normals[keep]

        self.ids = self.ids[keep]

        self.set_default_filter()

        return keep

    def apply_min_opacity(self, min_opacity):
        """Drop Gaussians with opacity <= min_opacity (gauss_handler.py:195-203)."""
        if min_opacity > 0.0:
            self.filter_indices = self.filter_indices & (self.opacities > min_opacity)
            self._filter_is_default = False

    def apply_bounding_box(self, bounding_box_min, bounding_box_max):
        """Drop Gaussians outside the open box (gauss_handler.py:205-224)."""
        valid = torch.ones(self.xyz.shape[0], dtype=torch.bool, device=self.xyz.device)
        if bounding_box_min is not None:
            lo = torch.as_tensor(bounding_box_min, dtype=self.xyz.dtype, device=self.xyz.device)
            valid &= (self.xyz > lo).all(dim=1)
        if bounding_box_max is not None:
            hi = torch.as_tensor(bounding_box_max, dtype=self.xyz.dtype, device=self.xyz.device)
            valid &= (self.xyz < hi).all(dim=1)
        self.filter_indices = self.filter_indices & valid
        self._filter_is_default = False

    def cull_large_gaussians(self, cull_gauss_size_percent):
        """Remove the largest `cull_gauss_size_percent` fraction of Gaussians by magnitude.

        The reference (gauss_handler.py:235-250) ANDs the boolean filter with an int64 *index* tensor of a
        different length, which raises for any percentage > 0; the intended behaviour is implemented instead:
        keep the floor(N * (1 - p)) smallest."""
        if cull_gauss_size_percent > 0.0:
            sizes = self.get_gaussian_magnitudes()
            cull_index = floor(sizes.shape[0] * (1 - cull_gauss_size_percent))
            order = torch.sort(sizes).indices
            keep = torch.zeros(sizes.shape[0], dtype=torch.bool, device=sizes.device)
            keep[order[:cull_index]] = True
            self.filter_indices = self.filter_indices & keep
            self._filter_is_default = False

    def get_gaussian_magnitudes(self, contributions=None):
        """sqrt(ellipsoid surface area) * contribution, f64 (gauss_handler.py:252-279)."""
        eigvals = eigvals_sym3(self.covariances)

        p = 1.6075
        a, b, c = torch.sqrt(eigvals[:, 0]), torch.sqrt(eigvals[:, 1]), torch.sqrt(eigvals[:, 2])
        radicand = (torch.pow(a * b, p) + torch.pow(a * c, p) + torch.pow(b * c, p)) / 3.0
        surface_area = torch.sqrt(4.0 * torch.pi * torch.pow(radicand, 1.0 / p))

        if contributions is None:
            contributions = self.opacities

        return (surface_area * contributions).to(torch.float64)
