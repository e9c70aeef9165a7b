"""Oracle restatement of the sampling stage (TEST INFRASTRUCTURE, see oracle/__init__.py).

Follows gauss_to_pc.py:73-371 and torch.distributions.MultivariateNormal
(torch 2.11 multivariate_normal.py:194 Cholesky, :251-254 rsample = loc + L @ eps).  torch-CPU routines are used
for Cholesky / inverse / bmm so the arithmetic matches the reference's CPU run; the random draw is injected
(`eps_fn`) because the product defines its own counter-based stream (oracle/philox.py).
"""
import math

import numpy as np
import torch

from . import philox


# ---------------------------------------------------------------------------------------------------------
def distribute_points(sizes, num_points):
    """gauss_to_pc.py:73-90 — round(size * P / sum), then the first min(deficit, #zeros) zero entries become 1."""
    sizes = torch.as_tensor(sizes)
    ratio = num_points / torch.sum(sizes)
    ppg = torch.round(sizes * ratio)
    zeros = (ppg == 0).nonzero()
    deficit = (num_points - ppg.sum()).item()
    take = int(min(deficit, zeros.shape[0]))
    zeros = zeros[:take] if take >= 0 else zeros[:take]  # negative deficit slices from the end, like the reference
    ppg[zeros] = 1
    return ppg


def calculate_bin_sizes(hist_nonzero):
    """gauss_to_pc.py:105-138 — second-difference heuristic on the histogram of points-per-Gaussian.
    `hist_nonzero`: counts of each occurring ppg value, ascending by value.  Returns (start_bin, bin_size)."""
    dist = np.asarray(hist_nonzero)
    grad = np.absolute(np.gradient(np.gradient(dist)))
    bin_size = max(len(dist) // 100, 1)
    length = len(grad) - len(grad) % bin_size
    summed = grad[:length].reshape(-1, bin_size).sum(axis=1)
    cut_off = np.max(summed) // 50
    peak = np.argmax(summed)
    below = np.nonzero(summed[peak:] < cut_off)[0]
    start_bin = 1
    if below.shape[0] != 0:
        start_bin = below[0]
    return int(start_bin), int(bin_size)


def make_bins(ppg, exact_num_points):
    """gauss_to_pc.py:308-343 — list of (start, end, n) with n = floor(start + (end-start)/2), in loop order.
    Bins with n <= 0 are dropped here; empty bins are dropped by the caller (it needs the members)."""
    ppg = torch.as_tensor(ppg).to(torch.int32)
    pd = torch.unique(ppg)
    if not exact_num_points:
        hist = torch.bincount(ppg)
        hist = hist[hist.nonzero()].squeeze(1).numpy()
        start_bin, bin_size = calculate_bin_sizes(hist)
        pd = torch.cat((pd[:start_bin], torch.mul(torch.unique(torch.ceil(pd[start_bin:] / bin_size)), bin_size)), 0)
    bins = []
    for i in range(pd.shape[0]):
        start = pd[i].item()
        end = pd[i + 1].item() if i != pd.shape[0] - 1 else start + 1
        n = math.floor(start + (end - start) / 2)
        if n <= 0:
            continue
        bins.append((start, end, n))
    return bins


# ---------------------------------------------------------------------------------------------------------
def mahalanobis(means, samples, covs):
    """gauss_to_pc.py:92-103 — sqrt(d^T Sigma^-1 d), d = mu - x, fp32 inverse + two bmm."""
    delta = (means - samples).unsqueeze(2)
    inv = torch.inverse(covs)
    m = torch.bmm(delta.transpose(1, 2), torch.bmm(inv, delta))
    return torch.sqrt(m).squeeze(1).squeeze(1)


def mvn_sample(means, covs, eps, max_tries=3, epsilon=1e-6):
    """gauss_to_pc.py:140-155 + MultivariateNormal: Cholesky of every covariance of the batch; on any failure the
    WHOLE batch gets +1e-6*I (cumulative) and is retried, at most 3 tries, else None.  x = mu + L @ eps.
    eps: (k, n', 3).  Returns ((k, n', 3) samples or None, covs as modified)."""
    covs = covs.clone()
    for _ in range(max_tries):
        L, info = torch.linalg.cholesky_ex(covs)
        if bool((info == 0).all()) and bool(torch.isfinite(covs).all()):
            x = means.unsqueeze(0) + torch.matmul(L.unsqueeze(0), eps.unsqueeze(-1)).squeeze(-1)
            return x, covs
        covs = covs + epsilon * torch.eye(3)
    return None, covs


def create_new_gaussian_points(k, means, covs, colours, std, num_attempts, normals, gids, eps_fn):
    """gauss_to_pc.py:157-275.  Returns (points (P,3) f32, colours (P,3), normals (P,3) or None,
    per_attempt list of (todo_indices, counts, m)).  The accept test only decides HOW MANY of the first samples
    of each Gaussian's block are emitted (:242-258) — restated as such."""
    n = means.shape[0]
    added = torch.zeros(n, dtype=torch.int64)
    pts, cols, nrms, trace = [], [], [], []
    emitted = 0
    a = 0
    while emitted < k * n and a < num_attempts:
        todo = (added != k).nonzero().squeeze(1)
        mu, cv = means[todo], covs[todo]
        eps = torch.as_tensor(eps_fn(gids[todo.numpy()], k, a))  # (k, n', 3)
        x, cv = mvn_sample(mu, cv, eps)
        if x is None:
            a += 1
            continue
        samples = x.transpose(0, 1).contiguous().view(-1, 3)  # Gaussian-major (n'*k, 3)
        d = mahalanobis(torch.repeat_interleave(mu, k, dim=0), samples, torch.repeat_interleave(cv, k, dim=0))
        ok = (d <= std).view(-1, k)
        counts = ok.sum(1)
        m = torch.minimum(k - added[todo], counts)
        take = (torch.arange(k).unsqueeze(0) < m.unsqueeze(1)).flatten()
        pts.append(samples[take])
        cols.append(colours[todo].repeat_interleave(m, dim=0))
        if normals is not None:
            nrms.append(normals[todo].repeat_interleave(m, dim=0))
        added[todo] = torch.minimum(torch.full_like(counts, k), added[todo] + counts)
        emitted += int(m.sum())
        trace.append((todo.numpy().copy(), counts.numpy().copy(), m.numpy().copy(), d.numpy().copy()))
        a += 1
    cat = lambda xs, w: torch.cat(xs, 0) if xs else torch.zeros((0, w))
    return cat(pts, 3), cat(cols, 3), (cat(nrms, 3) if normals is not None else None), trace


def generate_pointcloud(xyz, cov, colours, normals, magnitudes, num_points, std=2.0, exact_num_points=False,
                        num_sample_attempts=5, seed=0, call_id=0, eps_fn=None, gid_offset=0, ppg=None):
    """gauss_to_pc.py:277-371.  `magnitudes`: output of get_gaussian_magnitudes (f64).  Returns a dict with
    points/colours/normals in the reference's output order plus the intermediate integer data."""
    xyz, cov = torch.as_tensor(xyz), torch.as_tensor(cov)
    colours = torch.as_tensor(colours)
    normals = None if normals is None else torch.as_tensor(normals)
    if eps_fn is None:
        eps_fn = lambda g, k, a: philox.draw_eps(g, k, a, seed, call_id)
    if ppg is None:
        ppg = distribute_points(magnitudes, num_points).to(torch.int32)
    else:
        ppg = torch.as_tensor(ppg).to(torch.int32)
    bins = make_bins(ppg, exact_num_points)
    P, C, Nn = [], [], []
    bin_trace = []
    for (start, end, n) in bins:
        idx = torch.where((ppg >= start) & (ppg < end))[0]
        if idx.shape[0] < 1:
            continue
        P.append(xyz[idx])
        C.append(colours[idx])
        if normals is not None:
            Nn.append(normals[idx])
        tr = None
        if n > 1:
            p, c, nn, tr = create_new_gaussian_points(n - 1, xyz[idx], cov[idx], colours[idx], std,
                                                      num_sample_attempts, None if normals is None else normals[idx],
                                                      idx.numpy() + gid_offset, eps_fn)
            P.append(p)
            C.append(c)
            if normals is not None:
                Nn.append(nn)
        bin_trace.append((start, end, n, idx.numpy(), tr))
    cat = lambda xs, w, dt: torch.cat(xs, 0) if xs else torch.zeros((0, w), dtype=dt)
    return {
        "points": cat(P, 3, torch.float32),
        "colours": cat(C, 3, colours.dtype),
        "normals": cat(Nn, 3, torch.float32) if normals is not None else None,
        "ppg": ppg,
        "bins": bins,
        "bin_trace": bin_trace,
    }
