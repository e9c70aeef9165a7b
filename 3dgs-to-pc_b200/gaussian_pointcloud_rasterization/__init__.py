"""Import-name compatibility with the reference's CUDA extension package
(gaussian-pointcloud-rasterization/gaussian_pointcloud_rasterization/__init__.py): the same public names, backed by the
sm_90a kernels behind the C ABI (g2pc/rasterizer.py).  `_C` stands in for the pybind11 module (ext.cpp:15-17)."""
import types

from g2pc.rasterizer import (GaussianRasterizationSettings, GaussianRasterizer, mark_visible,  # noqa: F401
                             rasterize_gaussians)

_C = types.SimpleNamespace(rasterize_gaussians=rasterize_gaussians, mark_visible=mark_visible)
