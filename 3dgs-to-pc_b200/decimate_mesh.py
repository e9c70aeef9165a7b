"""Decimate a mesh on the GPU to a target triangle count by parallel quadric edge collapse (g2pc.mesh.decimate, rules in
DESIGN.md §2, N9).

    python decimate_mesh.py --input_path mesh.ply --target_triangles N [--mesh_output_path decimated_mesh.ply] [--quiet]

The input is a binary PLY as mesh_pc.py and gauss_to_mesh.py write it (g2pc.mesh.write_mesh_ply).  Boundary and
non-manifold vertices stay where they are; merged vertices take the rounded mean colour of the vertices merged into
them, and the normals are recomputed.  A mesh that takes long to make can so be decimated to several sizes without
meshing it again."""
import argparse
import time

import torch

from g2pc import build, mesh
from mesh_pc import target


def config_parser(argv=None):
    p = argparse.ArgumentParser(description="Decimate a triangle mesh by quadric edge collapse")
    p.add_argument("--input_path", required=True, help="mesh PLY written by mesh_pc.py or gauss_to_mesh.py")
    p.add_argument("--target_triangles", type=target, required=True, help="triangles to keep (the result has this many "
                                                                          "or one fewer)")
    p.add_argument("--mesh_output_path", default="decimated_mesh.ply", help="output mesh PLY")
    p.add_argument("--quiet", action="store_true", help="print nothing")
    return p.parse_args(argv)


def main(argv=None):
    args = config_parser(argv)
    build.build()
    t0 = time.perf_counter()
    v, n, c, f = mesh.read_mesh_ply(args.input_path)
    dev = "cuda:0"
    m = mesh.Mesh(torch.from_numpy(v).to(dev), torch.from_numpy(f).to(dev), torch.from_numpy(c).to(dev),
                  torch.from_numpy(n).to(dev), None)
    stats = {}
    out = mesh.decimate_mesh(m, args.target_triangles, stats=stats)
    mesh.write_mesh_ply(args.mesh_output_path, out)
    if not args.quiet:
        print(f"Decimated {f.shape[0]} to {out.faces.shape[0]} triangles in {stats['rounds']} round(s); wrote "
              f"{out.vertices.shape[0]} vertices to {args.mesh_output_path} in {time.perf_counter() - t0:.2f} s")
    return out


if __name__ == "__main__":
    main()
