"""The per-leaf lists of the multisplit (csrc/s4_tree.cu) at full scale: 3 M Gaussians, one camera (1280x720, and
2560x1440 for the tile grid), both colour back-ends.  The parity tests stop at 40 k Gaussians, a few dozen multisplit
chunks; here the stream spans thousands of chunks of several sub-steps each, with leaf tables that select C = 256, 128
and 64 entries per sub-step, and Gaussian counts that are not a multiple of the chunk size.

Checked on the device against the depth-sorted stream of the same frame:
  * every list holds as many ids as the leaf has overlapping Gaussians, counted independently from the packed ranges;
  * every id overlaps its leaf according to its packed range;
  * the ids' positions in the sorted stream strictly increase along every list.
Together these pin every list: the Gaussians overlapping the leaf, each once, nearest first.
"""
import pytest
import torch

from util import scene_to

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N = 3_000_000


@pytest.fixture(scope="module")
def scene():
    from g2pc import synth
    from oracle import gaussians as og
    sc = synth.make_scene(N, seed=1260, sh_degree=0)
    d = scene_to({k: sc[k] for k in ("xyz", "opacities", "colours")}, DEV)
    d["cov"] = og.build_covariance(sc["scales"], sc["rots"]).contiguous().to(DEV)
    return d


def _unpack(q):
    return q & 255, (q >> 8) & 255, (q >> 16) & 255, (q >> 24) & 255


def _check_lists(leaves, nl, inst_gid, val_sorted, n, bx, by, exact, gw, gh):
    """leaves (nl, 8) int32 of the frame; (bx, by): each leaf's cell in the grid of the packed ranges (gw x gh); exact:
    the leaf is that cell (False: a deeper leaf inside it, checked against its cell with the one-node overhang of
    child tiles and left out of the independent count)."""
    lv = leaves[:nl].long()
    beg, cnt = lv[:, 4], lv[:, 5]
    assert bool((cnt >= 0).all())
    assert bool((beg[1:] >= beg[:-1] + cnt[:-1]).all()), "lists overlap"
    total = int(cnt.sum())
    leaf_of = torch.repeat_interleave(torch.arange(nl, device=DEV), cnt)
    first = torch.cumsum(cnt, 0) - cnt
    ids = inst_gid[beg[leaf_of] + torch.arange(total, device=DEV) - first[leaf_of]].long()
    assert bool(((ids >= 0) & (ids < n)).all()), "list slot not written"

    vs = val_sorted[:n]
    gid = vs & 0xFFFFFFFF
    q_sorted = (vs >> 32) & 0xFFFFFFFF
    rank = torch.empty(n, dtype=torch.long, device=DEV)
    rank[gid] = torch.arange(n, device=DEV)
    rng = torch.empty(n, dtype=torch.long, device=DEV)
    rng[gid] = q_sorted

    # stream order along every list
    r = rank[ids]
    same = leaf_of[1:] == leaf_of[:-1]
    assert bool((r[1:] > r[:-1])[same].all()), "ids out of depth order (or repeated) in a list"

    # every id overlaps its leaf
    xlo, xhi, ylo, yhi = _unpack(rng[ids])
    X, Y = bx[leaf_of], by[leaf_of]
    inside = (xlo <= X) & (X <= xhi) & (ylo <= Y) & (Y <= yhi)
    near = (xlo - 1 <= X) & (X <= xhi) & (ylo - 1 <= Y) & (Y <= yhi)
    assert bool(torch.where(exact[leaf_of], inside, near).all()), "id does not overlap its leaf"

    # list lengths against an independent count: 2-D difference array of the ranges over the cells
    xlo, xhi, ylo, yhi = _unpack(q_sorted)
    ok = (xlo <= xhi) & (ylo <= yhi)
    xlo, xhi, ylo, yhi = xlo[ok], xhi[ok], ylo[ok], yhi[ok]
    assert bool((xhi < gw).all() and (yhi < gh).all())
    D = torch.zeros((gh + 1) * (gw + 1), dtype=torch.long, device=DEV)
    for yy, xx, s in ((ylo, xlo, 1), (ylo, xhi + 1, -1), (yhi + 1, xlo, -1), (yhi + 1, xhi + 1, 1)):
        D.index_add_(0, yy * (gw + 1) + xx, torch.full_like(yy, s))
    per_cell = D.view(gh + 1, gw + 1).cumsum(0).cumsum(1)
    want = per_cell[by[exact], bx[exact]]
    assert torch.equal(cnt[exact], want), "list length != Gaussians overlapping the leaf"
    return total, int(exact.sum())


def _run_twice(R, cam):
    # the first frame sizes the buffers; the lists of the second are checked on id slots pre-filled with -1
    R(cam)
    R.flush()
    for sl in R._slots:
        if sl["inst_gid"] is not None:
            sl["inst_gid"].fill_(-1)
    R(cam)
    R.flush()


@pytest.mark.parametrize("n,leaf_cap,max_tile,chunk", [
    (N, None, None, 256),           # C3's leaf table
    (N - 777, None, 32, 64),        # 20 px base tiles, 8192-leaf table: 64 entries per sub-step; n not a multiple of E
])
def test_quadtree_lists_at_scale(lib, scene, n, leaf_cap, max_tile, chunk):
    import camera_handler as ch
    import gauss_render as gr
    from g2pc import synth
    d = scene
    R = gr.get_renderer("python", d["xyz"][:n], d["opacities"][:n].unsqueeze(1), d["colours"][:n], d["cov"][:n],
                        visible_gaussian_threshold=0.05)
    if max_tile is not None:
        R.max_tile_size = max_tile
    cams, intr = synth.make_cameras(1)
    cam = ch.get_camera("python", cams[0].to(DEV), intr[0], colour_resolution=1280)
    W, H = int(cam.image_width), int(cam.image_height)
    if leaf_cap is not None:
        R._set_leaf_cap(R._get_tables(W, H), leaf_cap)
    _run_twice(R, cam)
    t, slot = R._last_tables, R._last_slot
    assert int(lib.g2pc_multisplit_chunk(t["leaf_cap"])) == chunk
    nl = R.last_stats["num_leaves"]
    leaves = t["slots"][slot]["leaves"]
    lb = t["base_level"]
    node = leaves[:nl, 7].long()
    level = torch.zeros_like(node)
    for lv in range(1, t["qt"].num_levels):
        level += (node >= ((1 << (2 * lv)) - 1) // 3).long()
    one = torch.ones_like(level)
    rem = node - (torch.bitwise_left_shift(one, 2 * level) - 1) // 3
    iy, ix = rem >> level, rem & (torch.bitwise_left_shift(one, level) - 1)
    assert bool((level >= lb).all())
    sl = R._slots[slot]
    total, n_exact = _check_lists(leaves, nl, sl["inst_gid"], sl["val_sorted"], n, ix >> (level - lb),
                                  iy >> (level - lb), level == lb, 1 << lb, 1 << lb)
    assert total > n
    print(f"[multisplit at scale] python n={n} C={chunk}: {nl} leaves ({n_exact} at the base level), {total} ids")


@pytest.mark.parametrize("n,res,chunk", [
    (N, 1280, 256), (N - 777, 1280, 256),
    (N - 777, 2560, 128),           # 80 x 45 super-tiles: 128 entries per sub-step
])
def test_tile_grid_lists_at_scale(lib, scene, n, res, chunk):
    import camera_handler as ch
    import gauss_render as gr
    from g2pc import synth
    d = scene
    R = gr.get_renderer("cuda", d["xyz"][:n], d["opacities"][:n].unsqueeze(1), d["colours"][:n], d["cov"][:n],
                        visible_gaussian_threshold=0.05)
    cams, intr = synth.make_cameras(1)
    rs = ch.get_camera("cuda", cams[0].to(DEV), intr[0], colour_resolution=res)
    _run_twice(R, rs)
    t, slot = R._last, R._last_slot
    assert int(lib.g2pc_multisplit_chunk(t["ntiles"])) == chunk
    nl, gx, gy = t["ntiles"], t["gx"], t["gy"]
    cell = torch.arange(nl, device=DEV)
    sl = R._slots[slot]
    total, _ = _check_lists(t["slots"][slot]["leaves"], nl, sl["inst_gid"], sl["val_sorted"], n, cell % gx, cell // gx,
                            torch.ones(nl, dtype=torch.bool, device=DEV), gx, gy)
    assert total > n // 2
    print(f"[multisplit at scale] cuda n={n} {res} px C={chunk}: {nl} super-tiles, {total} ids")
