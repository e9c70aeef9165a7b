"""ctypes binding of libg2pc.so (the C-ABI CUDA library declared in include/g2pc.h).

This is the stub a maintainer of the reference would add in place of
`from gaussian_pointcloud_rasterization import _C` (gaussian_pointcloud_rasterization/__init__.py:14) and of
the torch call chains in gauss_to_pc.py:140-275.  There is NO fallback: if the library is missing or a call
fails, an exception is raised.
"""
import contextlib
import ctypes
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libg2pc.so")

F32, F64 = 0, 1
CULL_EPS_NORM, CULL_EXPLICIT = 0, 1
ST_OVERFLOW, ST_CHOLFAIL, ST_CHOLREG, ST_WORDS = 0, 1, 2, 4

_c_void_p = ctypes.c_void_p
_i32, _i64, _u32, _u64, _f32 = ctypes.c_int32, ctypes.c_int64, ctypes.c_uint32, ctypes.c_uint64, ctypes.c_float

# name -> argtypes, exactly as declared in include/g2pc.h
SIGNATURES = {
    "g2pc_version": ([], ctypes.c_int),
    "g2pc_last_error": ([], ctypes.c_char_p),
    "g2pc_cov_build": ([_c_void_p, _c_void_p, ctypes.c_int, _f32, _i64, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_normals": ([_c_void_p, _c_void_p, ctypes.c_int, _i64, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_eigvals_sym3": ([_c_void_p, _i64, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_sample_count": ([_c_void_p, _c_void_p, _c_void_p, ctypes.c_int, _c_void_p, _c_void_p, _c_void_p, _i64, _i64,
                           _c_void_p, _i32, _i32, _i32, _f32, _i32, _u64, _u32, _c_void_p, _c_void_p, _c_void_p,
                           _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_sample_emit_chunk_points": ([], ctypes.c_int),
    "g2pc_sample_emit": ([_c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i32, _u64, _u32, _c_void_p,
                          _c_void_p, _c_void_p, ctypes.c_int, _i64, _c_void_p], ctypes.c_int),
    "g2pc_dump_eps": ([_c_void_p, _i64, _i32, _i32, _u64, _u32, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_cull_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_cull_select": ([_c_void_p, _f32, _c_void_p, _f32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                          _c_void_p, _i64, _i64, _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_gather_rows": ([_c_void_p, _i64, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_ppg_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_knn_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_knn_mean_dist": ([_c_void_p, _i64, _i32, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_knn_ids": ([_c_void_p, _i64, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_sor_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_sor_mask": ([_c_void_p, _i64, ctypes.c_double, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_splat_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_splat": ([_c_void_p, _c_void_p, ctypes.c_int, _i64, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                         _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_solve_workspace_bytes": ([_i32], ctypes.c_int64),
    "g2pc_mesh_vcycle": ([_c_void_p, _c_void_p, _i32, _c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p],
                         ctypes.c_int),
    "g2pc_mesh_iso_workspace_bytes": ([], ctypes.c_int64),
    "g2pc_mesh_iso": ([_c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p],
                      ctypes.c_int),
    "g2pc_mesh_extract_workspace_bytes": ([_i32], ctypes.c_int64),
    "g2pc_mesh_extract_count": ([_c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_extract_emit": ([_c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i64, _c_void_p,
                                _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_mesh_gather_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_gather": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p,
                          _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_trim_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_trim": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                        _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_smooth_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_smooth": ([_c_void_p, _i64, _c_void_p, _i64, _i32, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_normals_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_normals": ([_c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p],
                          ctypes.c_int),
    "g2pc_mesh_band_bricks_workspace_bytes": ([_i32], ctypes.c_int64),
    "g2pc_mesh_band_bricks": ([_c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                               _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_list": ([_c_void_p, _i32, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_splat": ([_c_void_p, _c_void_p, ctypes.c_int, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _i64,
                              _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_ghosts": ([_c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                               _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_cg_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_band_cg_start": ([_c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i64,
                                 _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_cg_step": ([_c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p,
                                _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_iso_workspace_bytes": ([], ctypes.c_int64),
    "g2pc_mesh_band_iso": ([_c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                            _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_extract_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_band_extract_count": ([_c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                                      _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_band_extract_emit": ([_c_void_p, _i32, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i64,
                                     _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p],
                                    ctypes.c_int),
    "g2pc_mesh_band_gather_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_band_gather": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i32, _c_void_p, _c_void_p, _i64,
                               _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_decimate_prepare_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_decimate_prepare": ([_c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p],
                                   ctypes.c_int),
    "g2pc_mesh_decimate_round_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_decimate_select": ([_c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64,
                                   _c_void_p], ctypes.c_int),
    "g2pc_mesh_decimate_apply": ([_c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                  _c_void_p, _i64, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64,
                                  _c_void_p], ctypes.c_int),
    "g2pc_mesh_decimate_finish_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_mesh_decimate_finish": ([_c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                   _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p],
                                  ctypes.c_int),
    "g2pc_mesh_components_label": ([_c_void_p, _i64, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_mesh_components_select_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_components_select": ([_c_void_p, _i64, _i64, _c_void_p, _c_void_p, _i64, _i64, _i64, _c_void_p,
                                     _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_components_compact": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p,
                                      _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_holes_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_mesh_holes_find": ([_c_void_p, _i64, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64,
                              _c_void_p], ctypes.c_int),
    "g2pc_mesh_holes_plan": ([_i64, _i64, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                              _i64, _c_void_p], ctypes.c_int),
    "g2pc_mesh_holes_fill": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p,
                              _i64, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p],
                             ctypes.c_int),
    "g2pc_tsdf_frame_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_tsdf_frame": ([_c_void_p, _i64, _i32, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_tsdf_integrate": ([_c_void_p, _i32, ctypes.c_double, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _i32,
                             _c_void_p, _c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p],
                            ctypes.c_int),
    "g2pc_tsdf_compact_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_tsdf_gather_compact": ([_c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _i64,
                                  _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                                  _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_orient_prepare_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_orient_prepare": ([_c_void_p, _c_void_p, ctypes.c_int, _i64, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                             _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_orient_edges_workspace_bytes": ([_i64, _i32], ctypes.c_int64),
    "g2pc_orient_edges": ([_c_void_p, _i64, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                           _i64, _c_void_p], ctypes.c_int),
    "g2pc_orient_round_workspace_bytes": ([_i64, _i64], ctypes.c_int64),
    "g2pc_orient_round": ([_c_void_p, _c_void_p, _c_void_p, _i64, _i64, _i32, _i64, _c_void_p, _c_void_p, _c_void_p,
                           _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_orient_finish_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_orient_finish": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, ctypes.c_int, _i64, _c_void_p, _c_void_p,
                            _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_face_cameras": ([_c_void_p, _c_void_p, ctypes.c_int, _c_void_p, _i64, _c_void_p, _i64, _c_void_p, _i64,
                           _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_points_per_gaussian": ([_c_void_p, _c_void_p, _i64, ctypes.c_double, _c_void_p, _c_void_p, _c_void_p, _i64,
                                  _c_void_p], ctypes.c_int),
    "g2pc_pack_geometry": ([_c_void_p, _c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_preprocess": ([_c_void_p, _c_void_p, _c_void_p, _i32, _i32, _i64, _c_void_p, _c_void_p, _c_void_p, _i32, _u32,
                         _u32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_preprocess_cameras": ([_c_void_p, _c_void_p, _c_void_p, _i32, _i32, _i64, _c_void_p, _i32, _c_void_p,
                                 _c_void_p, _i32, _u32, _u32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p],
                                ctypes.c_int),
    "g2pc_depth_sort_workspace_bytes": ([_i64], ctypes.c_int64),
    "g2pc_depth_sort": ([_c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _i64, _c_void_p], ctypes.c_int),
    "g2pc_build_tree": ([_c_void_p, _i32, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _i64, _i64,
                         _i64, _i32, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_multisplit_chunk": ([_i32], ctypes.c_int32),
    "g2pc_multisplit_rows": ([_i64, _i32], ctypes.c_int32),
    "g2pc_multisplit_workspace_bytes": ([_i64, _i64, _i32, _i32], ctypes.c_int64),
    "g2pc_multisplit": ([_c_void_p, _i64, _c_void_p, _i32, _i32, _c_void_p, _i32, _u32, _u32, _c_void_p, _c_void_p,
                         _c_void_p, _c_void_p, _i32, _i32, _c_void_p, _i64, _c_void_p, _i64, _c_void_p, _c_void_p],
                        ctypes.c_int),
    "g2pc_blend": ([_c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _i32, _i32, _c_void_p, _c_void_p, _c_void_p,
                    _c_void_p, _c_void_p, _c_void_p, _i32, _i32, _f32, _f32, _c_void_p, _c_void_p, _c_void_p],
                   ctypes.c_int),
    "g2pc_blend_set_compact": ([ctypes.c_int], None),
    "g2pc_blend_set_cull": ([ctypes.c_int], None),
    "g2pc_accumulate": ([_c_void_p, _c_void_p, _i64, _c_void_p, _c_void_p, _c_void_p, _i32, _c_void_p], ctypes.c_int),
    "g2pc_tiles_preprocess": ([_c_void_p, _c_void_p, _c_void_p, _i32, _i32, _i32, _i64, _c_void_p, _c_void_p, _c_void_p,
                               _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_tiles_build": ([_c_void_p, _i32, _i32, _c_void_p, _c_void_p, _i32, _i64, _i64, _i32, _i32, _c_void_p,
                          _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_multisplit_grid": ([_c_void_p, _i64, _i32, _i32, _c_void_p, _c_void_p, _c_void_p, _i32, _i64, _c_void_p, _i64,
                              _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_tiles_blend": ([_c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p,
                          _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _i32, _c_void_p, _c_void_p, _c_void_p,
                          _c_void_p], ctypes.c_int),
    "g2pc_tiles_blend_fusion": ([_c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p,
                                 _c_void_p, _c_void_p, _c_void_p, _c_void_p, _c_void_p, _i32, _i32, _c_void_p, _c_void_p,
                                 _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_tiles_accumulate": ([_c_void_p, _c_void_p, _c_void_p, _i32, _i32, _i64, _c_void_p, _c_void_p, _c_void_p,
                               _c_void_p, _c_void_p, _i32, _c_void_p, _c_void_p, _c_void_p, _c_void_p], ctypes.c_int),
    "g2pc_fill_u32": ([_c_void_p, _u32, _i64, _c_void_p], ctypes.c_int),
    "g2pc_compose_image": ([_c_void_p, _c_void_p, _i32, _i32, _f32, _c_void_p, _c_void_p], ctypes.c_int),
}


class Raster(ctypes.Structure):
    """g2pc_raster_t"""
    _fields_ = [("viewmatrix", _f32 * 16), ("projmatrix", _f32 * 16), ("campos", _f32 * 3), ("tan_fovx", _f32),
                ("tan_fovy", _f32), ("width", _i32), ("height", _i32)]


class Camera(ctypes.Structure):
    """g2pc_camera_t"""
    _fields_ = [("view", _f32 * 16), ("proj", _f32 * 16), ("campos", _f32 * 3), ("tan_fovx", _f32),
                ("tan_fovy", _f32), ("focal_x", _f32), ("focal_y", _f32), ("width", _i32), ("height", _i32)]


(HDR_NUM_LEAVES, HDR_TOTAL_INST, HDR_TOTAL_PIX, HDR_NEED_DEEPER, HDR_LEAF_OVERFLOW, HDR_CAP_OVERFLOW, HDR_POISON,
 HDR_FRAME, HDR_TOTAL_INST_HI, HDR_ROW_INST) = range(10)
HDR_WORDS = 16
WORK_COUNTERS = 4
STAT_WARP_GAUSSIANS, STAT_WORDS = 0, 4
LEAF_WORDS = 8  # g2pc_leaf_t = 8 x int32
PREPROCESS_MAX_CAMERAS = 8  # G2PC_PREPROCESS_MAX_CAMERAS

_lib = None


class G2pcError(RuntimeError):
    pass


def load(path=None):
    """Load libg2pc.so and attach the argument types.  Raises if the library is absent (no fallback)."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise G2pcError(
            f"{path} not found: build it with `python -m g2pc.build` (or __graft_entry__.build()). "
            "There is no CPU fallback for the g2pc kernels.")
    lib = ctypes.CDLL(path)
    for name, (argtypes, restype) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.argtypes = argtypes
        fn.restype = restype
    _lib = lib
    return lib


# ---- launch accounting (bench.py reads these) -------------------------------------------------------------------
LAUNCHES = 0      # number of hand-written g2pc kernels launched since the last reset
TIMING = None     # None, or a dict filled as {entry point name: [(start_event, end_event), ...]}: every launch is
                  # bracketed with CUDA events on the current stream (bench.py)
# hand-written kernels launched per entry point (default 1); the radix sorts and selections inside g2pc_depth_sort,
# the k-NN and the orientation entry points are cub's (library); g2pc_multisplit launches 3 more on a table with levels
# below the base level
_OWN_KERNELS = {"g2pc_multisplit": 6, "g2pc_multisplit_grid": 6, "g2pc_depth_sort": 0, "g2pc_cull_select": 3,
                "g2pc_points_per_gaussian": 5, "g2pc_knn_mean_dist": 6, "g2pc_knn_ids": 6, "g2pc_sor_mask": 5, "g2pc_mesh_splat": 5,
                "g2pc_mesh_iso": 7, "g2pc_mesh_extract_count": 2, "g2pc_mesh_extract_emit": 2, "g2pc_mesh_gather": 3,
                "g2pc_mesh_trim": 6, "g2pc_mesh_normals": 3, "g2pc_mesh_band_bricks": 4, "g2pc_mesh_band_cg_start": 4,
                "g2pc_mesh_band_cg_step": 6,
                "g2pc_mesh_band_iso": 4, "g2pc_mesh_band_extract_count": 2, "g2pc_mesh_band_extract_emit": 2,
                "g2pc_mesh_band_gather": 2, "g2pc_mesh_decimate_prepare": 4, "g2pc_mesh_decimate_select": 8,
                "g2pc_mesh_decimate_apply": 5, "g2pc_mesh_decimate_finish": 4, "g2pc_mesh_components_label": 5,
                "g2pc_mesh_components_select": 4, "g2pc_mesh_components_compact": 2,"g2pc_mesh_holes_find": 7,
                "g2pc_mesh_holes_plan": 2, "g2pc_mesh_holes_fill": 1, "g2pc_orient_prepare": 2, "g2pc_orient_edges": 2,
                "g2pc_orient_round": 5, "g2pc_orient_finish": 3, "g2pc_tsdf_frame": 2, "g2pc_tsdf_gather_compact": 4}
# host-only entry points, besides every *_workspace_bytes size query
_NOT_KERNELS = {"g2pc_version", "g2pc_last_error", "g2pc_sample_emit_chunk_points", "g2pc_multisplit_chunk",
                "g2pc_multisplit_rows", "g2pc_blend_set_compact", "g2pc_blend_set_cull"}


def call(name, *args):
    """Invoke entry point `name` (must be declared in SIGNATURES), check its status, count it, and — when TIMING is a
    dict — bracket it with CUDA events on the current stream."""
    global LAUNCHES
    fn = getattr(load(), name)
    if TIMING is None or name in _NOT_KERNELS or name.endswith("_workspace_bytes"):
        status = fn(*args)
    else:
        with phase(TIMING, name):
            status = fn(*args)
    LAUNCHES += _OWN_KERNELS.get(name, 1)
    check(status, name)


@contextlib.contextmanager
def phase(timings, name):
    """Brackets the block with CUDA events on the current stream and appends the pair to timings[name] when `timings` is
    a dict; does nothing when it is None."""
    if timings is None:
        yield
        return
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    yield
    b.record()
    timings.setdefault(name, []).append((a, b))


def check(status, what):
    if status != 0:
        msg = load().g2pc_last_error()
        raise G2pcError(f"{what} failed (status {status}): {msg.decode() if msg else ''}")


def ptr(t):
    """Device pointer of a tensor (None -> NULL)."""
    if t is None:
        return None
    return t.data_ptr()


def workspace(nbytes, device):
    """Scratch for an entry point's workspace argument: a uint8 tensor of at least nbytes, and of at least 256 bytes, so
    that it is never empty (an empty tensor's NULL pointer is refused).  Pass its numel() as the size."""
    return torch.empty((max(int(nbytes), 256),), dtype=torch.uint8, device=device)


def stream_ptr(device=None):
    return torch.cuda.current_stream(device).cuda_stream


def dtype_code(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.float64:
        return F64
    raise G2pcError(f"unsupported dtype {t.dtype} (need float32 or float64)")


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise G2pcError("g2pc kernels need CUDA tensors; there is no CPU fallback "
                            f"(got a tensor on {t.device})")


def check_cloud(points, normals=None, colours=None, what=None):
    """Refuses a point cloud the point-cloud kernels cannot take: points (n, 3) float32; normals, when given, (n, 3)
    float32 or float64; colours, when given, (n, 3); all CUDA tensors on one device.  `what` names an operation that
    needs the normals (e.g. "Poisson meshing"): with it, missing normals are refused too."""
    if what is not None and normals is None:
        raise G2pcError(f"{what} needs normals (the cloud has none)")
    if points is None:
        raise G2pcError(f"{what or 'the point-cloud kernels'} needs the points")
    require_cuda(points, normals, colours)
    if points.dim() != 2 or points.shape[1] != 3 or points.dtype != torch.float32:
        raise G2pcError(f"points must be (n, 3) float32, got {tuple(points.shape)} {points.dtype}")
    if normals is not None and (normals.shape != points.shape or normals.dtype not in (torch.float32, torch.float64)):
        raise G2pcError(f"normals must be (n, 3) float32 or float64 like the points, got {tuple(normals.shape)} "
                        f"{normals.dtype}")
    if colours is not None and colours.shape != points.shape:
        raise G2pcError(f"colours must be (n, 3) like the points, got {tuple(colours.shape)}")
    devices = [str(t.device) for t in (points, normals, colours) if t is not None]
    if len(set(devices)) > 1:
        raise G2pcError(f"the points, normals and colours are on different devices ({', '.join(devices)})")


def gather_rows(index, m, tensors):
    """Rows index[:m] (int32 CUDA) of every tensor in `tensors`, compacted by one g2pc_gather_rows call: a list of new
    (m, ...) tensors with the sources' dtypes, in the order of `tensors`."""
    dev = index.device
    srcs = [t.contiguous() for t in tensors]
    dsts = [torch.empty((m,) + tuple(s.shape[1:]), dtype=s.dtype, device=dev) for s in srcs]
    if m > 0:
        k = len(srcs)
        call("g2pc_gather_rows", ptr(index), m, k, (ctypes.c_void_p * k)(*[s.data_ptr() for s in srcs]),
             (ctypes.c_void_p * k)(*[d.data_ptr() for d in dsts]),
             (ctypes.c_int32 * k)(*[s[0].numel() * s.element_size() for s in srcs]), stream_ptr(dev))
    return dsts
