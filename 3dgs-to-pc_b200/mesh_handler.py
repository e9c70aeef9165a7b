"""Point-cloud post-processing hooks (reference: mesh_handler.py).

clean_point_cloud is the reference's statistical outlier removal (Open3D remove_statistical_outlier, nb_neighbors=20)
built on the g2pc kernels: exact k-nearest-neighbour mean distances on the GPU, no Open3D (g2pc/outliers.py).
generate_mesh (Poisson reconstruction, Open3D) is OUT OF SCOPE of this build (SURVEY.md §2 row 15: third-party CPU
library); the name exists so that `--generate_mesh` fails with a clear message."""


def _need_open3d():
    try:
        import open3d  # noqa: F401
    except ImportError as e:
        raise ImportError("Open3D is required for meshing and is not part of g2pc") from e
    raise NotImplementedError("Open3D meshing is outside the scope of the g2pc hot path")


def clean_point_cloud(points, colours, normals, std_ratio=10, device="cuda:0"):
    """Remove statistical outliers: keep the points whose mean distance to their 20 nearest points (themselves
    included) is > 0 and < mean + std_ratio * std over the cloud.  Returns (points, colours clamped to 0..255 as int32,
    normals) of the kept points in their original order; normals=None stays None.  The tensors must already be on the
    CUDA device; `device` is accepted for the reference's signature."""
    from g2pc import outliers
    return outliers.remove_statistical_outliers(points, colours, normals, nb_neighbors=20, std_ratio=std_ratio)


def generate_mesh(points, colours, normals, output_path, depth=10, laplacian_iters=10):
    _need_open3d()
