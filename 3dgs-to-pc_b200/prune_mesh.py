"""Remove the small disconnected pieces of a mesh and close its small holes on the GPU (g2pc.mesh.remove_components and
g2pc.mesh.fill_holes, rules in DESIGN.md §2, N11 and N12).

    python prune_mesh.py --input_path mesh.ply [--min_component_triangles N] [--keep_largest_components K]
                         [--max_hole_edges H] [--mesh_output_path pruned_mesh.ply] [--quiet]

The input is a binary PLY as mesh_pc.py and gauss_to_mesh.py write it (g2pc.mesh.write_mesh_ply).  Two vertices are
connected when a face uses both; the pieces with fewer than N triangles, and all but the K largest, are removed, with
every vertex no face uses.  Positions, normals and colours of what stays are copied unchanged.  A mesh that takes long
to make can so be cleaned at several thresholds without meshing it again.

With --max_hole_edges H, the holes whose boundary loop has at most H edges (3..1024) are then closed: a hole of 3 edges
gets one triangle, a longer one a fan around a new vertex at the mean of its loop.  The pieces are removed first, so
small islands are dropped rather than capped.  Vertices on no filled loop keep their normals; the filled loops and the
new vertices get area-weighted normals of the filled mesh.  Nothing is smoothed here: the meshers smooth the patch
together with the rest of the surface, but smoothing a finished mesh would move every vertex of it.  At least one of
the three flags is needed."""
import argparse
import time

import torch

from g2pc import build, mesh
from mesh_pc import add_component_flags, add_hole_flag, component_line, hole_line


def config_parser(argv=None):
    p = argparse.ArgumentParser(description="Remove the small connected pieces of a triangle mesh and close its small "
                                            "holes")
    p.add_argument("--input_path", required=True, help="mesh PLY written by mesh_pc.py or gauss_to_mesh.py")
    add_component_flags(p)
    add_hole_flag(p)
    p.add_argument("--mesh_output_path", default="pruned_mesh.ply", help="output mesh PLY")
    p.add_argument("--quiet", action="store_true", help="print nothing")
    args = p.parse_args(argv)
    if args.min_component_triangles is None and args.keep_largest_components is None and args.max_hole_edges is None:
        p.error("give at least one of --min_component_triangles, --keep_largest_components and --max_hole_edges")
    return args


def main(argv=None):
    args = config_parser(argv)
    build.build()
    t0 = time.perf_counter()
    v, n, c, f = mesh.read_mesh_ply(args.input_path)
    dev = "cuda:0"
    m = mesh.Mesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), torch.from_numpy(c).to(dev),
                  torch.from_numpy(n).to(dev), None)
    stats, hstats, out = {}, {}, m
    if args.min_component_triangles is not None or args.keep_largest_components is not None:
        out = mesh.remove_components_mesh(out, args.min_component_triangles, args.keep_largest_components, stats=stats)
    if args.max_hole_edges is not None:
        out = mesh.fill_holes_mesh(out, args.max_hole_edges, stats=hstats)
    mesh.write_mesh_ply(args.mesh_output_path, out)
    if not args.quiet:
        if stats:
            print(component_line(stats))
        if hstats:
            print(hole_line(hstats))
        print(f"Wrote {out.vertices.shape[0]} vertices and {out.faces.shape[0]} triangles to {args.mesh_output_path} "
              f"in {time.perf_counter() - t0:.2f} s")
    return out


if __name__ == "__main__":
    main()
