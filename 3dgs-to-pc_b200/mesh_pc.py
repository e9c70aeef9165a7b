"""Mesh an existing point cloud on the GPU: Poisson reconstruction with a multigrid solve, marching tetrahedra, density
trim and Laplacian smoothing (g2pc/mesh.py).

    python mesh_pc.py --input_path cloud.ply [--mesh_output_path mesh.ply] [--poisson_depth 10] [--band_depth 12]
                      [--laplacian_iterations 10] [--orient_normals] [--target_triangles N]
                      [--min_component_triangles N] [--keep_largest_components K] [--max_hole_edges H] [--quiet]

The cloud must carry normals (nx ny nz), as gauss_to_pc.py writes them by default; its colours (red green blue) are
carried over to the mesh's vertices.  A mesh faces the way its normals point.  By default the normals are used as they
are; --orient_normals first gives them a consistent sign (g2pc/orient.py, k = 10), which the normals of a cloud sampled
from Gaussians lack: each takes its sign from its Gaussian's rotation.  --band_depth adds finer levels stored only in a narrow band around the points:
--poisson_depth 10 --band_depth 12 is the reference's Poisson depth 12.  --target_triangles decimates the smoothed mesh
to N or N - 1 triangles on the GPU (quadric edge collapse, g2pc.mesh.decimate) before its normals are computed.
--min_component_triangles and --keep_largest_components remove the small disconnected pieces of the trimmed mesh before
it is smoothed (g2pc.mesh.remove_components): those with fewer than N triangles, and all but the K largest.
--max_hole_edges then closes the holes whose boundary loop has at most H edges (3..1024), also before the smoothing
(g2pc.mesh.fill_holes)."""
import argparse
import time

import numpy as np
import torch

import gauss_dataloader
from g2pc import build, mesh, orient


def _depth(s):
    d = int(s)
    if not mesh.DEPTH_MIN <= d <= mesh.DEPTH_MAX:
        raise argparse.ArgumentTypeError(f"must be in {mesh.DEPTH_MIN}..{mesh.DEPTH_MAX}")
    return d


def _iterations(s):
    i = int(s)
    if i < 0:
        raise argparse.ArgumentTypeError("must be >= 0")
    return i


def target(s):
    n = int(s)
    if n < 1:
        raise argparse.ArgumentTypeError("must be >= 1")
    return n


def add_component_flags(p):
    p.add_argument("--min_component_triangles", type=target, default=None,
                   help="remove the connected pieces of the mesh with fewer triangles than this; default: keep them all")
    p.add_argument("--keep_largest_components", type=target, default=None,
                   help="keep only this many of the largest connected pieces; default: keep them all")


def hole_edges(s):
    n = int(s)
    if not 3 <= n <= mesh.MAX_HOLE_EDGES:
        raise argparse.ArgumentTypeError(f"must be in 3..{mesh.MAX_HOLE_EDGES}")
    return n


def add_hole_flag(p):
    p.add_argument("--max_hole_edges", type=hole_edges, default=None,
                   help=f"close the holes of the mesh whose boundary loop has at most this many edges "
                        f"(3..{mesh.MAX_HOLE_EDGES}); default: leave them open")


def hole_line(stats):
    """The one line the commands print about the hole filling."""
    return (f"Closed holes: {stats['holes']} hole(s) found, {stats['filled']} filled, {stats['too_long']} too long, "
            f"{stats['pinched']} pinched, {stats['added_triangles']} triangle(s) added")


def component_line(stats):
    """The one line the commands print about the component filter."""
    return (f"Removed small pieces: {stats['components']} component(s) found, {stats['kept']} kept, "
            f"{stats['removed_triangles']} triangle(s) removed")


def config_parser(argv=None):
    p = argparse.ArgumentParser(description="Mesh a point cloud with oriented normals (Poisson reconstruction)")
    p.add_argument("--input_path", required=True, help="point-cloud PLY with x y z and nx ny nz (red green blue optional)")
    p.add_argument("--mesh_output_path", default="mesh.ply", help="output mesh PLY")
    p.add_argument("--poisson_depth", type=_depth, default=10,
                   help=f"grid of 2^depth nodes per axis, {mesh.DEPTH_MIN}..{mesh.DEPTH_MAX}")
    p.add_argument("--band_depth", type=int, default=None,
                   help=f"mesh at this depth, poisson_depth + 1 .. {mesh.BAND_DEPTH_MAX}, solving the levels above "
                        f"poisson_depth only in a narrow band around the points (--poisson_depth 10 --band_depth 12 is "
                        f"the reference's depth 12); default: mesh at poisson_depth")
    p.add_argument("--laplacian_iterations", type=_iterations, default=10, help="Laplacian smoothing steps (0: none)")
    p.add_argument("--orient_normals", action="store_true",
                   help=f"orient the normals consistently (k = {orient.K_DEFAULT} nearest neighbours) before meshing")
    p.add_argument("--target_triangles", type=target, default=None,
                   help="decimate the mesh to this many triangles (or one fewer); default: keep every triangle")
    add_component_flags(p)
    add_hole_flag(p)
    p.add_argument("--quiet", action="store_true", help="print nothing")
    args = p.parse_args(argv)
    if args.band_depth is not None and not args.poisson_depth < args.band_depth <= mesh.BAND_DEPTH_MAX:
        p.error(f"--band_depth must be in {args.poisson_depth + 1}..{mesh.BAND_DEPTH_MAX}")
    return args


def load_cloud(path, device="cuda:0"):
    """(points (n,3) f32, normals (n,3) f32, colours (n,3) f32 or None) of a point-cloud PLY."""
    v = gauss_dataloader.read_ply_vertices(path)
    names = v.dtype.names
    if not all(k in names for k in ("nx", "ny", "nz")):
        raise ValueError(f"{path} has no normals (nx ny nz): Poisson meshing needs them")
    col = lambda *k: torch.from_numpy(np.ascontiguousarray(np.stack([v[c] for c in k], 1), dtype=np.float32))
    colours = col("red", "green", "blue").to(device) if "red" in names else None
    return col("x", "y", "z").to(device), col("nx", "ny", "nz").to(device), colours


def main(argv=None):
    args = config_parser(argv)
    build.build()
    t0 = time.perf_counter()
    points, normals, colours = load_cloud(args.input_path)
    if not args.quiet:
        band = f" with a band to depth {args.band_depth}" if args.band_depth is not None else ""
        print(f"Meshing {points.shape[0]} points at depth {args.poisson_depth}{band}")
    if args.orient_normals:
        normals, st = orient.orient_normals(points, normals, k=orient.K_DEFAULT)
        if not args.quiet:
            print(f"Oriented the normals: {st.flipped} flipped, {st.components} component(s), {st.skipped} skipped")
    cstats, hstats = {}, {}
    m = mesh.poisson_mesh(points, normals, colours, depth=args.poisson_depth, laplacian_iters=args.laplacian_iterations,
                          band_depth=args.band_depth, target_triangles=args.target_triangles,
                          min_component_triangles=args.min_component_triangles,
                          keep_largest_components=args.keep_largest_components, component_stats=cstats,
                          max_hole_edges=args.max_hole_edges, hole_stats=hstats)
    mesh.write_mesh_ply(args.mesh_output_path, m)
    if not args.quiet:
        if cstats:
            print(component_line(cstats))
        if hstats:
            print(hole_line(hstats))
        print(f"Wrote {m.vertices.shape[0]} vertices and {m.faces.shape[0]} triangles to {args.mesh_output_path} "
              f"in {time.perf_counter() - t0:.2f} s")
    return m


if __name__ == "__main__":
    main()
