"""3DGS -> point cloud + mesh in one command: the reference's `gauss_to_pc.py --generate_mesh`, meshed on the GPU.

    python gauss_to_mesh.py --input_path scene.ply --transform_path transforms.json [gauss_to_pc.py's flags]
                            [--mesh_output_path 3dgs_mesh.ply] [--poisson_depth 10] [--laplacian_iterations 10]
                            [--band_depth D] [--target_triangles N]
                            [--min_component_triangles N] [--keep_largest_components K] [--max_hole_edges H]
                            [--mesh_method {poisson,tsdf}] [--tsdf_depth 9] [--tsdf_trunc 4]

Same flags and validation as gauss_to_pc.py; it writes the same point cloud to --output_path.  Then, as the reference's
mesh recipe does: the Gaussians on a predicted surface (surface distance below its mean) are sampled into a second cloud
of min(num_points // 2, 25 * n_surface) points, whose normals are first turned toward the camera that saw each Gaussian
best (g2pc.orient.face_cameras), and that cloud is meshed by g2pc/mesh.py (outlier removal k = 20, std_ratio 3, Poisson,
10 % density trim, Laplacian smoothing, and with --target_triangles a decimation to that many triangles) and written
to --mesh_output_path.  Needs --renderer_type cuda and a depth in
2..10 (DESIGN.md §2).  With --min_component_triangles N and --keep_largest_components K, the connected pieces of the
trimmed mesh with fewer than N triangles, and all but the K largest, are removed before the smoothing
(g2pc.mesh.remove_components, DESIGN.md §2, N11); both methods take them.  With --max_hole_edges H the holes
whose boundary loop has at most H edges (3..1024) are then closed, also before the smoothing (g2pc.mesh.fill_holes,
DESIGN.md §2, N12); both methods take it.

With --mesh_method tsdf no surface cloud is sampled: the Gaussians the point cloud is sampled from are rendered again
from the same cameras with a median depth per pixel, every depth map is fused in order into a 2^tsdf_depth voxel grid
of truncated signed distances (truncation tsdf_trunc voxels), and the zero crossing between observed voxels is meshed,
smoothed, decimated with --target_triangles and written (g2pc/tsdf.py, DESIGN.md §2, N10).  --band_depth is refused
with it and --poisson_depth is unused."""
import gauss_to_pc


def config_parser(argv=None):
    return gauss_to_pc.config_parser(argv, mesh=True)


def main(argv=None):
    return gauss_to_pc.main(argv, mesh=True)


if __name__ == "__main__":
    main()
