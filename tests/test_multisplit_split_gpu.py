"""The base-level lists of the multisplit (csrc/s4_tree.cu: the row split, then the column split) called directly on
synthetic depth-ordered streams over flat grids, against the lists restated on the host: for every cell, the ids of the
entries whose rectangle contains it, in stream order.

Covers the grid widths around the 32-bucket groups of the warp ballots (1, 31, 32, 33, 64, 65 and 256 cells per axis),
entries that span every row and every column, empty ranges, streams shorter than a warp and not a multiple of the warp
tile, and a row-list capacity too small for the frame: the frame then fails through the header and the failure word
without writing a list, and succeeds once the capacity the header reports is given.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
EMPTY = 1  # G2PC_RANGE_EMPTY


def _stream(n, gw, gh, seed):
    rng = np.random.default_rng(seed)
    x0 = rng.integers(0, gw, n); y0 = rng.integers(0, gh, n)
    x1 = np.minimum(gw - 1, x0 + rng.geometric(0.4, n) - 1)
    y1 = np.minimum(gh - 1, y0 + rng.geometric(0.4, n) - 1)
    wide = rng.random(n) < 0.02  # splats over every row / column
    y0[wide], y1[wide] = 0, gh - 1
    x0[wide[::-1]], x1[wide[::-1]] = 0, gw - 1
    rng_u = (x0 | (x1 << 8) | (y0 << 16) | (y1 << 24)).astype(np.uint64)
    rng_u[rng.random(n) < 0.05] = EMPTY
    gid = rng.permutation(n).astype(np.uint64)
    return (rng_u << np.uint64(32)) | gid


def _want(val, gw, gh):
    lists = [[] for _ in range(gw * gh)]
    for v in val.tolist():
        r, g = v >> 32, v & 0xFFFFFFFF
        x0, x1, y0, y1 = r & 255, (r >> 8) & 255, (r >> 16) & 255, r >> 24
        for y in range(y0, y1 + 1):
            for x in range(x0, x1 + 1):
                lists[y * gw + x].append(g)
    return lists


def _run(lib, val, gw, gh, row_cap):
    from g2pc import capi
    n = len(val)
    want = _want(val, gw, gh)
    cnt = np.array([len(w) for w in want], np.int64)
    padded = (cnt + 3) & ~3
    beg = np.concatenate([[0], np.cumsum(padded)[:-1]])
    leaves = np.zeros((gw * gh, capi.LEAF_WORDS), np.int32)
    leaves[:, 4], leaves[:, 5] = beg, cnt
    leaves_d = torch.from_numpy(leaves).to(DEV)
    val_d = torch.from_numpy(val.view(np.int64)).to(DEV)
    hdr = torch.zeros(capi.HDR_WORDS, dtype=torch.int32, device=DEV)
    fail = torch.full((1,), -1, dtype=torch.int32, device=DEV)
    ids = torch.full((int(padded.sum()) + 4,), -1, dtype=torch.int32, device=DEV)
    ws = capi.workspace(lib.g2pc_multisplit_workspace_bytes(n, row_cap, gw, gh), DEV)
    capi.call("g2pc_multisplit_grid", capi.ptr(val_d), n, gw, gh, capi.ptr(leaves_d), capi.ptr(hdr), capi.ptr(fail), 0,
              row_cap, capi.ptr(ws), ws.numel(), capi.ptr(ids), capi.stream_ptr(DEV))
    torch.cuda.synchronize()
    return want, beg, ids.cpu().numpy(), hdr.cpu().tolist(), int(fail.item())


def _row_entries(val, gh):
    r = val >> np.uint64(32)
    x0, x1 = r & np.uint64(255), (r >> np.uint64(8)) & np.uint64(255)
    y0, y1 = (r >> np.uint64(16)) & np.uint64(255), r >> np.uint64(24)
    ok = (x0 <= x1) & (y0 <= y1)
    return int((y1[ok] - y0[ok] + np.uint64(1)).sum())


@pytest.mark.parametrize("g", [1, 31, 32, 33, 64, 65, 256])
@pytest.mark.parametrize("n", [7, 32, 5000, 3 * 8192 + 517])
def test_grid_lists_are_the_host_lists(lib, g, n):
    from g2pc import capi
    for gw, gh in ((g, g), (g, max(1, g // 3)), (max(1, g // 2), g)):
        val = _stream(n, gw, gh, seed=g * 1000 + n + gw)
        want, beg, ids, hdr, fail = _run(lib, val, gw, gh, row_cap=_row_entries(val, gh))
        assert fail == -1 and hdr[capi.HDR_CAP_OVERFLOW] == 0, (gw, gh, hdr)
        assert hdr[capi.HDR_ROW_INST] == _row_entries(val, gh)
        for c, w in enumerate(want):
            got = ids[beg[c]:beg[c] + len(w)].tolist()
            assert got == w, (gw, gh, c, got[:8], w[:8])


def test_row_capacity_too_small_fails_the_frame_then_fits(lib):
    from g2pc import capi
    gw, gh, n = 40, 23, 20000
    val = _stream(n, gw, gh, seed=77)
    need = _row_entries(val, gh)
    want, beg, ids, hdr, fail = _run(lib, val, gw, gh, row_cap=need // 2)
    assert fail == 1 and hdr[capi.HDR_CAP_OVERFLOW] == 1 and hdr[capi.HDR_POISON] == 1
    assert hdr[capi.HDR_ROW_INST] == need
    assert (ids == -1).all(), "a failed frame wrote list slots"
    want, beg, ids, hdr, fail = _run(lib, val, gw, gh, row_cap=hdr[capi.HDR_ROW_INST])
    assert fail == -1 and hdr[capi.HDR_CAP_OVERFLOW] == 0
    for c, w in enumerate(want):
        assert ids[beg[c]:beg[c] + len(w)].tolist() == w, c
