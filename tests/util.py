"""Shared helpers for the parity tests."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


def gpu(a, dtype=None):
    """A numpy array (cast to dtype when given) as a contiguous tensor on cuda:0."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(a if dtype is None else a.astype(dtype))).to("cuda:0")


def same(a, b):
    """Bit-for-bit equality of two arrays as a plain bool (keeps pytest from diffing megabytes of bytes on a failure)."""
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def scene_to(sc, device):
    return {k: v.to(device) for k, v in sc.items()}


def counts_from_buffers(plan, xl, tile_totals):
    """Reconstruct m[a, j] (points Gaussian j emitted in attempt a, bin order) from the count pass' buffers."""
    A = plan.attempts_stored
    xl = xl.cpu().numpy().astype(np.int64)
    tt = tile_totals.cpu().numpy().astype(np.int64)
    M = np.zeros((A, plan.n), dtype=np.int64)
    for t, (j0, cnt, k, lpg) in enumerate(plan.tiles):
        if k <= 0:
            continue
        for a in range(A):
            tot = tt[t * A + a]
            if tot == 0:
                continue
            x = xl[a, j0:j0 + cnt]
            M[a, j0:j0 + cnt] = np.diff(np.concatenate([x, [tot]]))
    return M


def oracle_counts(bin_trace, attempts):
    """Per bin: m[a, local Gaussian] and the distances d from the oracle's trace."""
    out = []
    for (start, end, n, idx, tr) in bin_trace:
        m = np.zeros((attempts, idx.shape[0]), dtype=np.int64)
        dists = []
        if tr is not None:
            for a, (todo, counts, mm, d) in enumerate(tr):
                m[a, todo] = mm
                dists.append((todo, d.reshape(todo.shape[0], -1)))
        out.append((n, idx, m, dists))
    return out
