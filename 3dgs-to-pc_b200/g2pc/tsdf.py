"""Mesh of a Gaussian scene by truncated signed-distance (TSDF) fusion of its rendered depth on the device (N10,
`gauss_to_mesh.py --mesh_method tsdf`).  The rules are written down in DESIGN.md §2 and restated by tests/f64ref_tsdf.py.

Steps: statistical outlier removal of the Gaussian means (k = 20, std_ratio 3; only to place the grid) -> g2pc_tsdf_frame
-> memory check -> per camera, in order, on the CUDA back-end's frame queue: g2pc_tiles_blend_fusion (colour, final
transmittance T, median depth z_med) then g2pc_tsdf_integrate into the 2^depth grid -> g2pc_mesh_extract_count / _emit
(the Poisson mesher's marching tetrahedra, unchanged, iso 0) -> g2pc_tsdf_gather_compact (keep the surface of the
observed voxels, vertex colours and weights) -> remove_components (with min_component_triangles or
keep_largest_components) -> fill_holes (with max_hole_edges) -> g2pc_mesh_smooth -> decimate (with target_triangles) ->
g2pc_mesh_normals.  Host reads: the frame after the outlier removal, the extraction counts, the kept counts.
"""
import collections
import ctypes

import torch

from . import capi, mesh, outliers
from .rasterizer import GaussianRasterizer, _host_list, _raster_struct

DEPTH_MIN, DEPTH_MAX = 2, 10
DEFAULT_DEPTH = 9
DEFAULT_TRUNC = 4.0  # voxels
BYTES_PER_VOXEL = 20  # tsdf, weight, 3 colour planes (f32)
EXTRACT_BYTES_PER_VOXEL = 5  # the extraction's node scratch
NB_NEIGHBORS, STD_RATIO = 20, 3.0

# the inputs of fuse_mesh that gauss_to_pc.convert_gaussians_to_pc(mesh_method="tsdf") hands over
Scene = collections.namedtuple("Scene", ["xyz", "opacities", "covariances", "colours", "shs", "cameras"])


def check_depth(depth):
    if isinstance(depth, bool) or int(depth) != depth or not DEPTH_MIN <= depth <= DEPTH_MAX:
        raise capi.G2pcError(f"tsdf depth must be an integer in {DEPTH_MIN}..{DEPTH_MAX}, got {depth}")


def check_trunc(trunc):
    if not float(trunc) > 0.0:
        raise capi.G2pcError(f"the tsdf truncation must be > 0 voxels, got {trunc}")


def grid_bytes(depth):
    """Device bytes of the grid, the extraction's node scratch and its workspace at `depth`: what the first memory check
    of fuse_mesh counts.  Not counted there: the fusion renderer's per-camera buffers (sized by the Gaussians and the
    image sizes) and the extraction's outputs, whose size is known only after its count pass; the gather's buffers are
    checked once it is known."""
    cells = 1 << (3 * int(depth))
    return cells * (BYTES_PER_VOXEL + EXTRACT_BYTES_PER_VOXEL) + int(capi.load().g2pc_mesh_extract_workspace_bytes(depth))


class FusionRasterizer(GaussianRasterizer):
    """The CUDA back-end whose every camera is blended by g2pc_tiles_blend_fusion and integrated into `grid` right after,
    on the frame's stream: a camera skipped by a failed frame is skipped by its integration too and integrated when it is
    replayed, so each camera is integrated exactly once and in order.  grid: dict of frame, depth, trunc, tsdf, weight,
    colour.  images: None, or a dict that receives copies of (colour, T, z_med) per camera index."""

    def __init__(self, grid, *args, images=None, **kw):
        super().__init__(*args, **kw)
        self.grid = grid
        self.images = images

    def _res_tables(self, W, H):
        t = super()._res_tables(W, H)
        if "T" not in t:
            t["T"] = torch.zeros((H, W), dtype=torch.float32, device=self.device)
            t["zmed"] = torch.zeros((H, W), dtype=torch.float32, device=self.device)
        return t

    def _enqueue_back(self, rs, frame, camera_index, slot):
        st = capi.stream_ptr(self.device)
        W, H = int(rs.image_width), int(rs.image_height)
        t = self._res_tables(W, H)
        sl, ts = self._slots[slot], t["slots"][slot]
        mask = sl.get("mask")
        if mask is not None:
            t["colour"].zero_(); t["depth"].zero_(); t["invdepth"].zero_()
        bg = (ctypes.c_float * 3)(*(getattr(rs, "_bg_host", None) or _host_list(rs.bg, 3)))
        # (the per-Gaussian maxima the blend writes into cam_best are never read here)
        capi.call("g2pc_tiles_blend_fusion", capi.ptr(ts["leaves"]), capi.ptr(ts["leaf_order"]), capi.ptr(sl["hdr"]),
                  capi.ptr(self._fail), frame, capi.ptr(sl["inst_gid"]), capi.ptr(sl["proj"]), capi.ptr(self._cam_best),
                  None, capi.ptr(mask), capi.ptr(t["colour"]), capi.ptr(t["depth"]), capi.ptr(t["invdepth"]), W, H, bg,
                  capi.ptr(sl["work"]), capi.ptr(self._stats), capi.ptr(t["T"]), capi.ptr(t["zmed"]), st)
        g = self.grid
        capi.call("g2pc_tsdf_integrate", capi.ptr(g["frame"]), g["depth"], float(g["trunc"]), capi.ptr(t["zmed"]),
                  capi.ptr(t["T"]), capi.ptr(t["colour"]), capi.ptr(mask), W, H, ctypes.byref(_raster_struct(rs)), bg,
                  capi.ptr(self._fail), frame, capi.ptr(g["tsdf"]), capi.ptr(g["weight"]), capi.ptr(g["colour"]), st)
        if self.images is not None:
            self.images[camera_index] = (t["colour"].clone(), t["T"].clone(), t["zmed"].clone())


def frame_of(xyz, depth):
    """Frame words (8,) float64 on the device of the grid over the points xyz (n,3) float32."""
    dev, n = xyz.device, xyz.shape[0]
    frame = torch.empty((mesh.FRAME_WORDS,), dtype=torch.float64, device=dev)
    ws = capi.workspace(capi.load().g2pc_tsdf_frame_workspace_bytes(n), dev)
    capi.call("g2pc_tsdf_frame", capi.ptr(xyz), n, int(depth), capi.ptr(frame), capi.ptr(ws), ws.numel(),
              capi.stream_ptr(dev))
    return frame


def gather_compact(weight, colour, depth, vkey, vt, vpos, faces):
    """(keep (m,) uint8, dens (mk,) float64, vpos (mk,3) float64, vcol (mk,3) uint8, faces (tk,3) int32) of the surface
    whose vertices lie on edges between observed voxels (weight > 0)."""
    dev, m, t = vpos.device, vpos.shape[0], faces.shape[0]
    keep = torch.empty((m,), dtype=torch.uint8, device=dev)
    dens = torch.empty((m,), dtype=torch.float64, device=dev)
    vcol = torch.empty((m, 3), dtype=torch.uint8, device=dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    outs = [torch.empty_like(dens), torch.empty_like(vpos), torch.empty_like(vcol), torch.empty_like(faces)]
    ws = capi.workspace(capi.load().g2pc_tsdf_compact_workspace_bytes(m, t), dev)
    capi.call("g2pc_tsdf_gather_compact", capi.ptr(weight), capi.ptr(colour), int(depth), capi.ptr(vkey), capi.ptr(vt),
              capi.ptr(vpos), m, capi.ptr(faces), t, capi.ptr(keep), capi.ptr(dens), capi.ptr(vcol), capi.ptr(counts),
              *[capi.ptr(o) for o in outs], capi.ptr(ws), ws.numel(), capi.stream_ptr(dev))
    mk, tk = counts.tolist()
    d, p, c, f = outs
    return keep, d[:mk], p[:mk], c[:mk], f[:tk]


def fuse_mesh(xyz, opacities, covariances, cameras, colours=None, shs=None, depth=DEFAULT_DEPTH, trunc=DEFAULT_TRUNC,
              laplacian_iters=10, target_triangles=None, timings=None, return_debug=False, async_mode=True,
              min_component_triangles=None, keep_largest_components=None, component_stats=None, max_hole_edges=None,
              hole_stats=None):
    """Mesh of the Gaussians (xyz (n,3), opacities (n,) or (n,1), covariances (n,3,3) or (n,6), and exactly one of
    colours (n,3) in 0..1 or shs (n,3,K) channel-major, all CUDA) seen by `cameras` (the CUDA back-end's raster settings,
    camera_handler.get_camera("cuda", ...)), in order.  Returns mesh.Mesh(vertices (m,3) float32, faces (t,3) int32,
    colours (m,3) uint8, normals (m,3) float32, densities (m,) float64 = the interpolated camera counts); faces run
    counter-clockwise seen from free space.

    Memory: before the grid is allocated, the grid, the extraction's node scratch and its workspace are checked against
    the free device memory (grid_bytes), and before the gather its buffers; a shortfall raises G2pcError with both
    numbers.  The fusion renderer's buffers and the extraction's outputs are not part of these checks.

    depth: the grid has 2^depth voxels per axis (2..10) over 1.1 x the extent of the means left by a statistical outlier
    removal (k = 20, std_ratio 3).  trunc: the truncation mu in voxels (> 0).  laplacian_iters, target_triangles: as
    mesh.poisson_mesh.  timings: a dict that receives CUDA event pairs per phase (frame, fusion, extract, gather,
    smooth, decimate, normals).  return_debug: also a dict with frame, tsdf, weight, colour (the grid), vkey, vt, vpos,
    faces (the extraction), keep (the vertex mask of the gather), images ({camera index: (colour, T, z_med)}) and
    replays.

    min_component_triangles, keep_largest_components, component_stats: as mesh.poisson_mesh; the component filter runs
    on the gathered mesh before the smoothing, timings add "components" and the debug dict component_labels.

    max_hole_edges, hole_stats: as mesh.poisson_mesh; the hole filling runs after the component filter and before the
    smoothing, timings add "holes" and the debug dict hole_labels."""
    check_depth(depth)
    check_trunc(trunc)
    if int(laplacian_iters) != laplacian_iters or laplacian_iters < 0:
        raise capi.G2pcError(f"laplacian_iters must be an integer >= 0, got {laplacian_iters}")
    if target_triangles is not None:
        mesh.check_target(target_triangles)
    mesh.check_component_params(min_component_triangles, keep_largest_components, need_one=False)
    if max_hole_edges is not None:
        mesh.check_max_hole_edges(max_hole_edges)
    if (colours is None) == (shs is None):
        raise capi.G2pcError("give exactly one of colours and shs")
    capi.check_cloud(xyz.to(torch.float32).contiguous() if torch.is_tensor(xyz) else xyz)
    if xyz.shape[0] == 0:
        raise capi.G2pcError("there is no Gaussian to render")
    if len(cameras) == 0:
        raise capi.G2pcError("TSDF fusion needs at least one camera")
    depth, dev = int(depth), xyz.device
    with capi.phase(timings, "frame"):
        means = xyz.to(torch.float32).contiguous()
        pts, _, _ = outliers.remove_statistical_outliers(means, None, None, NB_NEIGHBORS, STD_RATIO)
        if pts.shape[0] == 0:
            raise capi.G2pcError("no Gaussian mean is left after the outlier removal")
        frame = frame_of(pts.contiguous(), depth)
        host = frame.tolist()
    if not host[6] > 0.0:
        raise capi.G2pcError("the Gaussian means have zero extent: every mean is at the same place")
    cells = 1 << (3 * depth)
    mesh.check_memory(grid_bytes(depth), dev, f"the tsdf grid at depth {depth} ({cells} voxels, "
                      f"{BYTES_PER_VOXEL + EXTRACT_BYTES_PER_VOXEL} bytes each, extraction scratch included)",
                      remedy="use a smaller tsdf depth")
    grid = dict(frame=frame, depth=depth, trunc=float(trunc),
                tsdf=torch.ones((cells,), dtype=torch.float32, device=dev),
                weight=torch.zeros((cells,), dtype=torch.float32, device=dev),
                colour=torch.zeros((3, cells), dtype=torch.float32, device=dev))
    images = {} if return_debug else None
    with capi.phase(timings, "fusion"):
        common = dict(cov3D_precomp=covariances.to(torch.float32), images=images)
        op = opacities.to(torch.float32).reshape(-1, 1)
        if shs is None:
            r = FusionRasterizer(grid, means, None, op, colors_precomp=colours.to(torch.float32), **common)
        else:
            r = FusionRasterizer(grid, means, None, op, shs=shs.to(torch.float32), sh_layout=0, **common)
        r.async_mode = async_mode
        for cam in cameras:
            r(cam)
        r.flush()
        replays = r.replays
        del r
    tsdf, weight, colour = grid["tsdf"], grid["weight"], grid["colour"]
    iso = torch.zeros((3,), dtype=torch.float64, device=dev)
    with capi.phase(timings, "extract"):
        scratch = torch.empty((EXTRACT_BYTES_PER_VOXEL * cells,), dtype=torch.uint8, device=dev)
        vkey, vt, vpos, faces = mesh.extract(tsdf, depth, frame, iso, scratch)
        del scratch
    if vkey.shape[0] == 0:
        raise capi.G2pcError("no surface: the fused signed distance does not change sign anywhere")
    m_, t_ = vkey.shape[0], faces.shape[0]
    # keep, density, colours, the compacted copies (density, position, colours, faces) and the scan workspace
    mesh.check_memory((1 + 8 + 3) * m_ + (8 + 24 + 3) * m_ + 12 * t_ +
                      int(capi.load().g2pc_tsdf_compact_workspace_bytes(m_, t_)), dev,
                      f"the gather of the tsdf surface ({m_} vertices, {t_} triangles)", remedy="use a smaller tsdf depth")
    with capi.phase(timings, "gather"):
        keep, dens, vkept, vcol, fkept = gather_compact(weight, colour, depth, vkey, vt, vpos, faces)
    debug = None
    if return_debug:
        debug = dict(frame=frame, tsdf=tsdf, weight=weight, colour=colour, vkey=vkey, vt=vt, vpos=vpos, faces=faces,
                     keep=keep, images=images, replays=replays, points=pts)
    del grid, tsdf, weight, colour
    if fkept.shape[0] == 0:
        raise capi.G2pcError("no surface between observed voxels")
    vkept, fkept, vcol, dens = mesh.filter_components(vkept, fkept, vcol, dens, min_component_triangles,
                                                       keep_largest_components, component_stats, timings, debug)
    vkept, fkept, vcol, dens = mesh.close_holes(vkept, fkept, vcol, dens, max_hole_edges, hole_stats, timings, debug,
                                                smoothing=False)  # the one-ring check follows
    if laplacian_iters and 6 * fkept.shape[0] >= 2 ** 31 - 1:
        raise capi.G2pcError(f"the surface has {fkept.shape[0]} triangles: the Laplacian smoothing's one-ring lists "
                             f"(6 per triangle) exceed int32; use a smaller tsdf depth or laplacian_iters=0")
    with capi.phase(timings, "smooth"):
        mesh.smooth(vkept, fkept, laplacian_iters)
    if target_triangles is not None:
        with capi.phase(timings, "decimate"):
            vkept, fkept, vcol, dens = mesh.decimate(vkept, fkept, target_triangles, vcol, dens)
    with capi.phase(timings, "normals"):
        v, vn = mesh.vertex_normals(vkept, fkept)
    out = mesh.Mesh(v, fkept, vcol, vn, dens)
    return (out, debug) if return_debug else out
