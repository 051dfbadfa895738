"""Python host-side mirror of the reference's public interface, over the C ABI.

The product is libpopsift_b200.so (C ABI in include/popsift_b200.h, C++ drop-in API in
include/popsift/*.h).  This module binds the C ABI with ctypes and offers the same vocabulary as
the reference (popsift::Config setters, PopSift.enqueue -> SiftJob.get -> Features) so that the
parity tests read like the reference's own usage (reference src/application/main.cpp:172-264).

There is no CPU fallback here: if the shared library is missing, or no CUDA device is usable,
construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import namedtuple
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("POPSIFT_B200_LIB") or os.path.join(_HERE, "lib", "libpopsift_b200.so")

PS_MAX_OCTAVES = 20
MODE = {"popsift": 0, "opencv": 1, "vlfeat": 2}
NORM = {"rootsift": 0, "RootSift": 0, "classic": 1}
GAUSS = {"vlfeat": 0, "vlfeat-hw-interpolated": 1, "relative": 1, "vlfeat-direct": 2, "opencv": 3, "fixed9": 4, "fixed15": 5}
DESC = {"loop": 0, "iloop": 1, "grid": 2, "igrid": 3, "notile": 4}
FILTER_SORT = {"random": 0, "down": 1, "up": 2}
STAGES = ("h2d", "pyramid", "extrema", "orientation", "descriptors", "total")


class PsConfig(C.Structure):
    _fields_ = [("octaves", C.c_int32), ("levels", C.c_int32), ("sigma", C.c_float), ("edge_limit", C.c_float),
                ("threshold", C.c_float), ("upscale", C.c_float), ("initial_blur", C.c_float),
                ("has_initial_blur", C.c_int32), ("sift_mode", C.c_int32), ("gauss_mode", C.c_int32),
                ("desc_mode", C.c_int32), ("norm_mode", C.c_int32), ("norm_multi", C.c_int32),
                ("max_extrema", C.c_int32), ("scaling_mode", C.c_int32), ("filter_max_extrema", C.c_int32),
                ("filter_grid_size", C.c_int32), ("filter_sort", C.c_int32)]


class PsGaussTables(C.Structure):
    _fields_ = [("inc_filter", C.c_float * (12 * 32)), ("inc_sigma", C.c_float * 12), ("inc_span", C.c_int32 * 12),
                ("dd_filter0", C.c_float * 32), ("dd_sigma0", C.c_float), ("dd_span0", C.c_int32),
                ("peak_threshold", C.c_float), ("sigma_k", C.c_float),
                ("dd_filter", C.c_float * (20 * 32)), ("dd_sigma", C.c_float * 20), ("dd_span", C.c_int32 * 20),
                ("abs_filter", C.c_float * (12 * 32)), ("abs_sigma", C.c_float * 12), ("abs_span", C.c_int32 * 12),
                ("inc_ifilter", C.c_float * (12 * 32)), ("inc_ispan", C.c_int32 * 12),
                ("absn_filter", C.c_float * (12 * 32)), ("absn_sigma", C.c_float * 12), ("absn_span", C.c_int32 * 12)]


FEATURE_DTYPE = np.dtype([("octave", "<i4"), ("x", "<f4"), ("y", "<f4"), ("sigma", "<f4"), ("num_ori", "<i4"),
                          ("ori", "<f4", (4,)), ("pad", "<i4"), ("desc_ptr", "<u8", (4,))])
EXTREMUM_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("lpos", "<i4"), ("sigma", "<f4"), ("octave", "<i4"),
                           ("num_ori", "<i4"), ("idx_ori", "<i4"), ("ori", "<f4", (4,))])
# ps_keypoint: a keypoint for PopSift.describe, in input-image units; octave / level -1 = derived from sigma
KEYPOINT_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("sigma", "<f4"), ("ori", "<f4"), ("octave", "<i4"), ("level", "<i4")])
assert FEATURE_DTYPE.itemsize == 72 and EXTREMUM_DTYPE.itemsize == 44 and KEYPOINT_DTYPE.itemsize == 24
DESCRIBE_GIVEN, DESCRIBE_ORIENT = 0, 1
GEOM = {"homography": 0, "fundamental": 1}


class PsVerifyParams(C.Structure):
    """ps_verify_params (24 bytes)"""
    _fields_ = [("model", C.c_int32), ("n_samples", C.c_int32), ("threshold", C.c_float), ("refine", C.c_int32),
                ("seed", C.c_uint64)]


class PsVerifyTaps(C.Structure):
    _fields_ = [("d_counts", C.c_void_p), ("d_models", C.c_void_p)]


class PsTrackCounts(C.Structure):
    """ps_track_counts (20 bytes)"""
    _fields_ = [("n_tracks", C.c_int32), ("n_members", C.c_int32), ("n_components", C.c_int32), ("n_conflicting", C.c_int32),
                ("n_short", C.c_int32)]


class PsCamera(C.Structure):
    """ps_camera (16 bytes): pinhole intrinsics in pixels"""
    _fields_ = [("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float)]


class PsPoseParams(C.Structure):
    """ps_pose_params (24 bytes)"""
    _fields_ = [("n_samples", C.c_int32), ("threshold", C.c_float), ("refine", C.c_int32), ("pad_", C.c_int32),
                ("seed", C.c_uint64)]


# ps_two_view (128 bytes): the per-pair output of ps_relative_pose_batch
TWO_VIEW_DTYPE = np.dtype([("E", "<f4", (3, 3)), ("F", "<f4", (3, 3)), ("R", "<f4", (3, 3)), ("t", "<f4", 3),
                           ("n_inliers", "<i4"), ("n_front", "<i4")])

assert C.sizeof(PsVerifyParams) == 24 and C.sizeof(PsTrackCounts) == 20
assert C.sizeof(PsCamera) == 16 and C.sizeof(PsPoseParams) == 24 and TWO_VIEW_DTYPE.itemsize == 128


class PsRigid(C.Structure):
    """ps_rigid (96 bytes): X_cam = R X_world + t, R row-major"""
    _fields_ = [("R", C.c_double * 9), ("t", C.c_double * 3)]


class PsTriangulateParams(C.Structure):
    """ps_triangulate_params (32 bytes)"""
    _fields_ = [("max_error", C.c_float), ("min_angle", C.c_float), ("min_views", C.c_int32), ("n_samples", C.c_int32),
                ("refine_iters", C.c_int32), ("pad_", C.c_int32), ("seed", C.c_uint64)]


class PsTriangulateCounts(C.Structure):
    """ps_triangulate_counts (24 bytes)"""
    _fields_ = [("n_status", C.c_int32 * 5), ("n_inlier_obs", C.c_int32)]


# ps_track_point (40 bytes): the per-track output of ps_triangulate_tracks; status codes PS_TRI_*
TRACK_POINT_DTYPE = np.dtype([("X", "<f8", 3), ("error", "<f4"), ("angle", "<f4"), ("n_inliers", "<i4"), ("status", "<i4")])
TRI_STATUS = ("ok", "too_few_obs", "no_hypothesis", "too_few_inliers", "small_angle")
assert C.sizeof(PsRigid) == 96 and C.sizeof(PsTriangulateParams) == 32 and C.sizeof(PsTriangulateCounts) == 24
assert TRACK_POINT_DTYPE.itemsize == 40


class PsBundleParams(C.Structure):
    """ps_bundle_params (56 bytes)"""
    _fields_ = [("loss", C.c_int32), ("max_iters", C.c_int32), ("cg_max_iters", C.c_int32), ("scale_set", C.c_int32),
                ("scale_axis", C.c_int32), ("pad_", C.c_int32), ("loss_scale", C.c_double), ("function_tol", C.c_double),
                ("cg_tol", C.c_double), ("initial_lambda", C.c_double)]


class PsBundleReport(C.Structure):
    """ps_bundle_report (48 bytes)"""
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32), ("accepted", C.c_int32),
                ("cg_iterations", C.c_int32), ("termination", C.c_int32), ("n_obs", C.c_int32), ("n_points", C.c_int32),
                ("n_free_cams", C.c_int32), ("pad_", C.c_int32)]


BA_LOSS = ("squared", "huber", "cauchy")
BA_TERMINATION = ("max_iters", "function_tol", "lambda", "no_observations", "nonfinite_start")
assert C.sizeof(PsBundleParams) == 56 and C.sizeof(PsBundleReport) == 48


class PsRotationParams(C.Structure):
    """ps_rotation_params (40 bytes)"""
    _fields_ = [("loss", C.c_int32), ("max_iters", C.c_int32), ("cg_max_iters", C.c_int32), ("min_inliers", C.c_int32),
                ("loss_scale", C.c_double), ("step_tol", C.c_double), ("cg_tol", C.c_double)]


class PsRotationReport(C.Structure):
    """ps_rotation_report (40 bytes)"""
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32), ("cg_iterations", C.c_int32),
                ("n_pairs", C.c_int32), ("n_registered", C.c_int32), ("termination", C.c_int32), ("pad_", C.c_int32)]


class PsPositionParams(C.Structure):
    """ps_position_params (40 bytes)"""
    _fields_ = [("loss", C.c_int32), ("max_iters", C.c_int32), ("cg_max_iters", C.c_int32), ("pad_", C.c_int32),
                ("loss_scale", C.c_double), ("function_tol", C.c_double), ("cg_tol", C.c_double)]


class PsPositionReport(C.Structure):
    """ps_position_report (40 bytes)"""
    _fields_ = [("initial_cost", C.c_double), ("final_cost", C.c_double), ("iterations", C.c_int32), ("cg_iterations", C.c_int32),
                ("n_obs", C.c_int32), ("n_points", C.c_int32), ("n_cams", C.c_int32), ("termination", C.c_int32)]


class PsViewGraphParams(C.Structure):
    """ps_view_graph_params (32 bytes)"""
    _fields_ = [("min_inliers", C.c_int32), ("min_consistent", C.c_int32), ("keep_untested", C.c_int32), ("pad_", C.c_int32),
                ("max_cycle_error", C.c_double), ("min_fraction", C.c_double)]


class PsCycleStats(C.Structure):
    """ps_cycle_stats (12 bytes)"""
    _fields_ = [("n_triangles", C.c_int32), ("n_consistent", C.c_int32), ("min_error", C.c_float)]


class PsViewGraphReport(C.Structure):
    """ps_view_graph_report (32 bytes)"""
    _fields_ = [("n_triangles", C.c_int64), ("n_consistent_triangles", C.c_int64), ("n_used", C.c_int32), ("n_kept", C.c_int32),
                ("n_untested", C.c_int32), ("pad_", C.c_int32)]


# ps_cycle_stats as a numpy record
CYCLE_STATS_DTYPE = np.dtype([("n_triangles", "<i4"), ("n_consistent", "<i4"), ("min_error", "<f4")])
assert C.sizeof(PsViewGraphParams) == 32 and C.sizeof(PsCycleStats) == 12 and C.sizeof(PsViewGraphReport) == 32
assert CYCLE_STATS_DTYPE.itemsize == 12

class PsTwoViewConfigParams(C.Structure):
    """ps_two_view_config_params (32 bytes)"""
    _fields_ = [("min_inliers", C.c_int32), ("threshold", C.c_float), ("min_ef_ratio", C.c_double), ("max_h_ratio", C.c_double),
                ("min_rotation_ratio", C.c_double)]


class PsTwoViewInfo(C.Structure):
    """ps_two_view_info (40 bytes)"""
    _fields_ = [("config", C.c_int32), ("n_e", C.c_int32), ("n_f", C.c_int32), ("n_h", C.c_int32), ("n_rotation", C.c_int32),
                ("tri_angle", C.c_float), ("normal", C.c_float * 3), ("pad_", C.c_int32)]


# ps_two_view_info as a numpy record; TV_CONFIG names its config codes (PS_TV_*)
TWO_VIEW_INFO_DTYPE = np.dtype([("config", "<i4"), ("n_e", "<i4"), ("n_f", "<i4"), ("n_h", "<i4"), ("n_rotation", "<i4"),
                                ("tri_angle", "<f4"), ("normal", "<f4", 3), ("pad_", "<i4")])
TV_CONFIG = ("degenerate", "general", "planar", "panoramic", "uncalibrated")
assert C.sizeof(PsTwoViewConfigParams) == 32 and C.sizeof(PsTwoViewInfo) == 40 and TWO_VIEW_INFO_DTYPE.itemsize == 40

class PsImage(C.Structure):
    """ps_image (24 bytes): device grey levels, row-major"""
    _fields_ = [("data", C.c_void_p), ("pitch", C.c_int64), ("width", C.c_int32), ("height", C.c_int32)]


class PsDepthParams(C.Structure):
    """ps_depth_params (24 bytes)"""
    _fields_ = [("n_depths", C.c_int32), ("radius", C.c_int32), ("top_k", C.c_int32), ("min_sources", C.c_int32),
                ("max_cost", C.c_float), ("min_var", C.c_float)]


class PsDepthReport(C.Structure):
    """ps_depth_report (16 bytes)"""
    _fields_ = [("n_candidates", C.c_int64), ("n_depths", C.c_int64)]


class PsDepthFilterParams(C.Structure):
    """ps_depth_filter_params (16 bytes)"""
    _fields_ = [("max_reproj_error", C.c_float), ("max_depth_diff", C.c_float), ("min_consistent", C.c_int32), ("pad_", C.c_int32)]


class PsDepthFilterReport(C.Structure):
    """ps_depth_filter_report (16 bytes)"""
    _fields_ = [("n_tested", C.c_int64), ("n_points", C.c_int64)]


# ps_dense_point (24 bytes): one consistent pixel of ps_depth_filter
DENSE_POINT_DTYPE = np.dtype([("X", "<f4", 3), ("ref", "<i4"), ("x", "<u2"), ("y", "<u2"), ("n_consistent", "u1"), ("grey", "u1"),
                              ("pad_", "<u2")])
assert C.sizeof(PsImage) == 24 and C.sizeof(PsDepthParams) == 24 and C.sizeof(PsDepthReport) == 16
assert C.sizeof(PsDepthFilterParams) == 16 and C.sizeof(PsDepthFilterReport) == 16 and DENSE_POINT_DTYPE.itemsize == 24

class PsVolume(C.Structure):
    """ps_volume (72 bytes): a dense volume's geometry and its three device arrays"""
    _fields_ = [("origin", C.c_double * 3), ("voxel", C.c_double), ("nx", C.c_int32), ("ny", C.c_int32), ("nz", C.c_int32),
                ("pad_", C.c_int32), ("tsdf", C.c_void_p), ("weight", C.c_void_p), ("grey", C.c_void_p)]


class PsTsdfParams(C.Structure):
    """ps_tsdf_params (8 bytes)"""
    _fields_ = [("trunc", C.c_float), ("min_consistent", C.c_int32)]


class PsMeshParams(C.Structure):
    """ps_mesh_params (8 bytes)"""
    _fields_ = [("min_weight", C.c_float), ("pad_", C.c_int32)]


class PsTsdfReport(C.Structure):
    """ps_tsdf_report (16 bytes)"""
    _fields_ = [("n_updates", C.c_int64), ("n_voxels_touched", C.c_int64)]


class PsMeshReport(C.Structure):
    """ps_mesh_report (24 bytes)"""
    _fields_ = [("n_cells", C.c_int64), ("n_vertices", C.c_int64), ("n_triangles", C.c_int64)]


# ps_mesh_vertex (16 bytes): world position and grey level of one mesh vertex
MESH_VERTEX_DTYPE = np.dtype([("X", "<f4", 3), ("grey", "<f4")])
assert C.sizeof(PsVolume) == 72 and C.sizeof(PsTsdfParams) == 8 and C.sizeof(PsMeshParams) == 8
assert C.sizeof(PsTsdfReport) == 16 and C.sizeof(PsMeshReport) == 24 and MESH_VERTEX_DTYPE.itemsize == 16


class PsRenderParams(C.Structure):
    """ps_render_params (8 bytes)"""
    _fields_ = [("z_near", C.c_float), ("pad_", C.c_int32)]


class PsRenderReport(C.Structure):
    """ps_render_report (24 bytes)"""
    _fields_ = [("n_drawn", C.c_int64), ("n_big", C.c_int64), ("n_covered", C.c_int64)]


class PsTextureParams(C.Structure):
    """ps_texture_params (24 bytes)"""
    _fields_ = [("cell", C.c_int32), ("cells_per_row", C.c_int32), ("depth_tol", C.c_float), ("min_cos", C.c_float),
                ("z_near", C.c_float), ("pad_", C.c_int32)]


class PsTextureReport(C.Structure):
    """ps_texture_report (16 bytes)"""
    _fields_ = [("n_viewed", C.c_int64), ("n_fallback", C.c_int64)]


assert C.sizeof(PsRenderParams) == 8 and C.sizeof(PsRenderReport) == 24
assert C.sizeof(PsTextureParams) == 24 and C.sizeof(PsTextureReport) == 16

RA_TERMINATION = ("max_iters", "step_tol", "no_pairs")
GP_TERMINATION = ("max_iters", "function_tol", "no_observations")
assert C.sizeof(PsRotationParams) == 40 and C.sizeof(PsRotationReport) == 40
assert C.sizeof(PsPositionParams) == 40 and C.sizeof(PsPositionReport) == 40

EXPORTS = ["ps_abi_version", "ps_config_default", "ps_gauss_tables_compute", "ps_geometry", "ps_create", "ps_destroy",
           "ps_last_error", "ps_submit_u8", "ps_submit_f32", "ps_submit_dev_u8", "ps_counts", "ps_download",
           "ps_sync", "ps_debug_plane", "ps_debug_extrema", "ps_slot_geometry", "ps_set_timing", "ps_stage_ms",
           "ps_launch_count", "ps_slot_stream", "ps_run_pyramid_only", "ps_run_level_only", "ps_host_alloc", "ps_host_free",
           "ps_download_dev", "ps_dev_alloc", "ps_dev_free", "ps_dev_to_host", "ps_wait_input", "ps_match", "ps_match_batch", "ps_pointer_device", "ps_host_to_dev",
           "ps_descriptors_to_u8", "ps_match_u8_batch", "ps_describe_u8", "ps_describe_f32",
           "ps_debug_level0_plan", "ps_format_gauss_tables", "ps_match_correspondences", "ps_verify_batch"]
# guided matching, declared in popsift_b200_guided.h (same library)
GUIDED_EXPORTS = ["ps_match_guided_batch", "ps_match_u8_guided_batch"]
# image retrieval, declared in popsift_b200_retrieval.h (same library)
RETRIEVAL_EXPORTS = ["ps_vlad_train", "ps_vlad_encode", "ps_retrieve_pairs"]
# feature tracks, declared in popsift_b200_tracks.h (same library)
TRACKS_EXPORTS = ["ps_tracks_from_edges", "ps_tracks_from_matches"]
# calibrated two-view geometry, declared in popsift_b200_pose.h (same library)
POSE_EXPORTS = ["ps_relative_pose_batch"]
# multi-view triangulation, declared in popsift_b200_triangulate.h (same library)
TRIANGULATE_EXPORTS = ["ps_triangulate_tracks"]
# bundle adjustment, declared in popsift_b200_bundle.h (same library)
BUNDLE_EXPORTS = ["ps_bundle_adjust"]
# global poses, declared in popsift_b200_global.h (same library)
GLOBAL_EXPORTS = ["ps_rotation_averaging", "ps_global_positioning"]
# view-graph cleaning, declared in popsift_b200_viewgraph.h (same library)
VIEWGRAPH_EXPORTS = ["ps_view_graph_filter"]
# two-view configuration, declared in popsift_b200_twoview.h (same library)
TWOVIEW_EXPORTS = ["ps_two_view_config_batch"]
# dense depth maps, declared in popsift_b200_depth.h (same library)
DEPTH_EXPORTS = ["ps_depth_maps", "ps_depth_filter"]
# surface meshes, declared in popsift_b200_mesh.h (same library)
MESH_EXPORTS = ["ps_volume_clear", "ps_tsdf_integrate", "ps_tsdf_mesh"]
# mesh rendering and texturing, declared in popsift_b200_render.h (same library)
RENDER_EXPORTS = ["ps_mesh_render", "ps_mesh_texture"]

_lib = None


def load_library():
    """dlopen the product library; raises if it has not been built (python -m popsift_b200.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("popsift_b200: %s is missing - build it with `python -m popsift_b200.build` "
                           "(there is no fallback path)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    L.ps_abi_version.restype = C.c_int
    L.ps_config_default.argtypes = [C.POINTER(PsConfig)]
    L.ps_gauss_tables_compute.argtypes = [C.POINTER(PsConfig), C.POINTER(PsGaussTables)]
    L.ps_geometry.argtypes = [C.POINTER(PsConfig), C.c_int, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.ps_create.restype = C.c_void_p
    L.ps_create.argtypes = [C.c_int, C.POINTER(PsConfig), C.c_int, C.c_int, C.c_int]
    L.ps_destroy.argtypes = [C.c_void_p]
    L.ps_last_error.restype = C.c_char_p
    L.ps_last_error.argtypes = [C.c_void_p]
    L.ps_submit_u8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.ps_submit_f32.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.ps_submit_dev_u8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    L.ps_counts.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.ps_download.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.ps_sync.argtypes = [C.c_void_p, C.c_int]
    L.ps_wait_input.argtypes = [C.c_void_p, C.c_int]
    L.ps_match.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    if hasattr(L, "ps_match_batch"):    # absent from builds that predate it (POPSIFT_B200_LIB A/B runs)
        L.ps_match_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    if hasattr(L, "ps_match_u8_batch"):
        L.ps_descriptors_to_u8.argtypes = [C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.ps_match_u8_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    if hasattr(L, "ps_describe_u8"):
        L.ps_describe_u8.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
        L.ps_describe_f32.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    if hasattr(L, "ps_verify_batch"):
        L.ps_match_correspondences.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ps_verify_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsVerifyParams),
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsVerifyTaps)]
    if hasattr(L, "ps_match_guided_batch"):
        for name in GUIDED_EXPORTS:
            getattr(L, name).argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                         C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_int]
    if hasattr(L, "ps_vlad_train"):
        L.ps_vlad_train.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_uint64, C.c_void_p, C.c_int]
        L.ps_vlad_encode.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
        L.ps_retrieve_pairs.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    if hasattr(L, "ps_tracks_from_edges"):
        L.ps_tracks_from_edges.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.POINTER(PsTrackCounts)]
        L.ps_tracks_from_matches.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.POINTER(PsTrackCounts)]
    if hasattr(L, "ps_relative_pose_batch"):
        L.ps_relative_pose_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.POINTER(PsPoseParams), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsVerifyTaps)]
    if hasattr(L, "ps_triangulate_tracks"):
        L.ps_triangulate_tracks.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_int, C.POINTER(PsTriangulateParams), C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.POINTER(PsTriangulateCounts)]
    if hasattr(L, "ps_bundle_adjust"):
        L.ps_bundle_adjust.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                       C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsBundleParams), C.c_void_p, C.c_void_p,
                                       C.POINTER(PsBundleReport)]
    if hasattr(L, "ps_rotation_averaging"):
        L.ps_rotation_averaging.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(PsRotationParams), C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.POINTER(PsRotationReport)]
        L.ps_global_positioning.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                            C.c_void_p, C.c_void_p, C.c_int, C.POINTER(PsPositionParams), C.c_void_p, C.c_void_p,
                                            C.c_void_p, C.POINTER(PsPositionReport)]
    if hasattr(L, "ps_view_graph_filter"):
        L.ps_view_graph_filter.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(PsViewGraphParams), C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.POINTER(PsViewGraphReport)]
    if hasattr(L, "ps_two_view_config_batch"):
        L.ps_two_view_config_batch.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsTwoViewConfigParams), C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]
    if hasattr(L, "ps_depth_maps"):
        L.ps_depth_maps.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                    C.c_void_p, C.POINTER(PsDepthParams), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(PsDepthReport)]
        L.ps_depth_filter.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.POINTER(PsDepthFilterParams), C.c_void_p, C.c_void_p, C.POINTER(PsDepthFilterReport)]
    if hasattr(L, "ps_tsdf_integrate"):
        L.ps_volume_clear.argtypes = [C.c_int, C.POINTER(PsVolume)]
        L.ps_tsdf_integrate.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.POINTER(PsTsdfParams), C.POINTER(PsVolume), C.POINTER(PsTsdfReport)]
        L.ps_tsdf_mesh.argtypes = [C.c_int, C.POINTER(PsVolume), C.POINTER(PsMeshParams), C.c_int64, C.c_int64, C.c_void_p, C.c_void_p,
                                   C.POINTER(PsMeshReport)]
    if hasattr(L, "ps_mesh_render"):
        L.ps_mesh_render.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                     C.POINTER(PsRenderParams), C.c_void_p, C.c_void_p, C.POINTER(PsRenderReport)]
        L.ps_mesh_texture.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p,
                                      C.c_int64, C.POINTER(PsTextureParams), C.c_void_p, C.c_void_p, C.POINTER(PsTextureReport)]
    L.ps_pointer_device.argtypes = [C.c_void_p]
    L.ps_host_to_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.ps_debug_plane.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]
    L.ps_debug_extrema.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int]
    L.ps_debug_level0_plan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int]
    L.ps_format_gauss_tables.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.ps_slot_geometry.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.ps_set_timing.argtypes = [C.c_void_p, C.c_int]
    L.ps_stage_ms.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_float)]
    L.ps_launch_count.restype = C.c_int64
    L.ps_launch_count.argtypes = [C.c_void_p]
    L.ps_slot_stream.restype = C.c_void_p
    L.ps_slot_stream.argtypes = [C.c_void_p, C.c_int]
    L.ps_run_pyramid_only.argtypes = [C.c_void_p, C.c_int]
    L.ps_run_level_only.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.ps_host_alloc.restype = C.c_void_p
    L.ps_host_alloc.argtypes = [C.c_size_t]
    L.ps_host_free.argtypes = [C.c_void_p]
    L.ps_download_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.ps_dev_alloc.restype = C.c_void_p
    L.ps_dev_alloc.argtypes = [C.c_size_t]
    L.ps_dev_free.argtypes = [C.c_void_p]
    L.ps_dev_to_host.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    _lib = L
    return L


class PopSiftError(RuntimeError):
    pass


class Config:
    """popsift::Config (reference src/popsift/sift_conf.h:29-409): same setters, same defaults."""

    # enums, reference sift_conf.h:33-107
    PopSift, OpenCV, VLFeat = 0, 1, 2
    RootSift, Classic = 0, 1
    ExtractingMode, MatchingMode = 0, 1

    def __init__(self):
        self._c = PsConfig()
        load_library().ps_config_default(C.byref(self._c))
        self.verbose = False
        self._log_mode = 0
        self._print_gauss_tables = False

    # public fields of the reference struct
    octaves = property(lambda s: s._c.octaves, lambda s, v: setattr(s._c, "octaves", int(v)))
    levels = property(lambda s: s._c.levels, lambda s, v: setattr(s._c, "levels", int(v)))
    sigma = property(lambda s: s._c.sigma, lambda s, v: setattr(s._c, "sigma", float(v)))
    _edge_limit = property(lambda s: s._c.edge_limit, lambda s, v: setattr(s._c, "edge_limit", float(v)))

    def setMode(self, m):
        self._c.sift_mode = MODE[m] if isinstance(m, str) else int(m)

    def setGaussMode(self, m):
        if isinstance(m, str):
            if m not in GAUSS:
                raise PopSiftError("Bad Gauss mode.")          # reference sift_conf.cu:101
            m = GAUSS[m]
        self._c.gauss_mode = int(m)

    def setDescMode(self, m="loop"):
        if isinstance(m, str):
            if m not in DESC:
                raise PopSiftError("specified descriptor extraction mode must be one of loop, grid or igrid")
            m = DESC[m]
        self._c.desc_mode = int(m)

    def setNormMode(self, m):
        if isinstance(m, str):
            if m not in ("RootSift", "classic"):
                raise PopSiftError("Bad Normalization mode.")   # reference sift_conf.cu:202
            m = NORM[m]
        self._c.norm_mode = int(m)

    def setUseRootSift(self, on):
        self._c.norm_mode = 0 if on else 1

    def getUseRootSift(self):
        return self._c.norm_mode == 0

    def setNormalizationMultiplier(self, m):
        self._c.norm_multi = int(m)

    def getNormalizationMultiplier(self):
        return self._c.norm_multi

    def setDownsampling(self, v):
        self._c.upscale = -float(v)

    def getUpscaleFactor(self):
        return self._c.upscale

    def setOctaves(self, v): self._c.octaves = int(v)
    def setLevels(self, v): self._c.levels = int(v)
    def setSigma(self, v): self._c.sigma = float(v)
    def setEdgeLimit(self, v): self._c.edge_limit = float(v)
    def setThreshold(self, v): self._c.threshold = float(v)
    def setVerbose(self, on=True): self.verbose = bool(on)
    def setLogMode(self, mode=1): self._log_mode = int(mode)
    def setFilterMaxExtrema(self, n): self._c.filter_max_extrema = int(n)
    def setFilterGridSize(self, n): self._c.filter_grid_size = int(n)
    def getFilterMaxExtrema(self): return self._c.filter_max_extrema
    def getFilterGridSize(self): return self._c.filter_grid_size

    def setFilterSorting(self, m):
        if isinstance(m, str):
            if m not in FILTER_SORT:
                raise PopSiftError("filter sorting mode must be one of up, down or random")   # reference sift_conf.cu:141
            m = FILTER_SORT[m]
        self._c.filter_sort = int(m)

    def setScalingMode(self, m=1):
        """Config::ScaleDirect = 0, Config::ScaleDefault = 1 (reference sift_conf.h:75-80)"""
        self._c.scaling_mode = int(m)
    def setPrintGaussTables(self): self._print_gauss_tables = True

    def gauss_tables_text(self) -> str:
        """what the reference prints under setPrintGaussTables() (gauss_filter.cu:24-121,146-161)"""
        L = load_library()
        n = L.ps_format_gauss_tables(C.byref(self._c), None, 0)
        if n < 0:
            raise PopSiftError("unsupported configuration (sigma > 2.0 or levels > 12)")
        buf = C.create_string_buffer(n + 1)
        L.ps_format_gauss_tables(C.byref(self._c), buf, n + 1)
        return buf.value.decode()

    def setInitialBlur(self, blur):
        self._c.has_initial_blur = 0 if blur == 0.0 else 1      # reference sift_conf.cu:246-255
        self._c.initial_blur = float(blur)

    def hasInitialBlur(self): return bool(self._c.has_initial_blur)
    def getInitialBlur(self): return self._c.initial_blur
    def getSiftMode(self): return self._c.sift_mode
    def getMaxExtrema(self): return self._c.max_extrema

    def getPeakThreshold(self):
        return float(np.float32(self._c.threshold) * np.float32(0.5) * np.float32(255.0) / np.float32(self._c.levels))

    def equal(self, other: "Config") -> bool:
        """reference sift_conf.cu:286-304 (desc mode, filter settings, log mode, verbose not compared)"""
        a, b = self._c, other._c
        return all(getattr(a, f) == getattr(b, f) for f in
                   ("octaves", "levels", "sigma", "edge_limit", "threshold", "upscale", "max_extrema", "gauss_mode",
                    "sift_mode", "has_initial_blur", "initial_blur", "norm_mode", "norm_multi"))

    __eq__ = equal

    def gauss_tables(self) -> PsGaussTables:
        t = PsGaussTables()
        rc = load_library().ps_gauss_tables_compute(C.byref(self._c), C.byref(t))
        if rc != 0:
            raise PopSiftError("unsupported configuration (sigma > 2.0, levels > 12, gauss mode)")
        return t

    def geometry(self, w: int, h: int):
        W = (C.c_int32 * PS_MAX_OCTAVES)()
        H = (C.c_int32 * PS_MAX_OCTAVES)()
        n = load_library().ps_geometry(C.byref(self._c), w, h, W, H)
        if n < 1:
            raise PopSiftError("bad geometry")
        return [(W[i], H[i]) for i in range(n)]


class _PinnedBlock:
    """One page-locked result buffer (features + descriptors); returned to its pool when released."""

    def __init__(self, lib, n_feat: int, n_desc: int):
        self.lib, self.n_feat, self.n_desc = lib, n_feat, n_desc
        self.pf = lib.ps_host_alloc(max(n_feat, 1) * 72)
        self.pd = lib.ps_host_alloc(max(n_desc, 1) * 512)
        if not self.pf or not self.pd:
            raise PopSiftError("ps_host_alloc failed")
        self.feat = np.ctypeslib.as_array(C.cast(self.pf, C.POINTER(C.c_uint8)), shape=(max(n_feat, 1) * 72,)).view(FEATURE_DTYPE)
        self.desc = np.ctypeslib.as_array(C.cast(self.pd, C.POINTER(C.c_float)), shape=(max(n_desc, 1), 128))

    def free(self):
        if self.pf:
            self.lib.ps_host_free(self.pf); self.lib.ps_host_free(self.pd)
            self.pf = self.pd = None


class _Pool:
    """Page-locked result buffers of one PopSift, recycled between images."""

    def __init__(self):
        self.blocks, self.closed = [], False

    def close(self):
        self.closed = True
        while self.blocks:
            self.blocks.pop().free()


class _Lease:
    """Ties a page-locked block to the numpy arrays that view it: every array handed out has a ctypes
    buffer as its base, the buffers hold this object, and only when the LAST array is gone does the block
    go back to its pool (or is freed, if the PopSift it came from has been shut down meanwhile).  So
    `d = ps.enqueue(...).get().desc` stays valid for as long as `d` lives."""

    def __init__(self, pool: _Pool, block: _PinnedBlock):
        self._pool, self._block = pool, block

    def __del__(self):
        blk, self._block = self._block, None
        if blk is None:
            return
        if self._pool.closed:
            blk.free()
        else:
            self._pool.blocks.append(blk)


def _leased_views(pool: _Pool, blk: _PinnedBlock, nf: int, nd: int):
    lease = _Lease(pool, blk)
    fbuf = (C.c_uint8 * (nf * 72)).from_address(blk.pf)
    dbuf = (C.c_float * (nd * 128)).from_address(blk.pd)
    fbuf._lease = dbuf._lease = lease
    feat = np.frombuffer(fbuf, dtype=FEATURE_DTYPE, count=nf) if nf else np.zeros(0, FEATURE_DTYPE)
    desc = np.frombuffer(dbuf, dtype=np.float32, count=nd * 128).reshape(nd, 128) if nd else np.zeros((0, 128), np.float32)
    return feat, desc


class Features:
    """popsift::FeaturesHost (reference src/popsift/features.h:71-102).  `feat` / `desc` view a page-locked
    buffer that stays alive as long as any array that views it (see _Lease)."""

    def __init__(self, feat: np.ndarray, desc: np.ndarray):
        self.feat = feat
        self.desc = desc
        base = desc.ctypes.data if len(desc) else 0
        idx = np.full((len(feat), 4), -1, dtype=np.int64)
        for k in range(4):
            m = feat["num_ori"] > k
            idx[m, k] = (feat["desc_ptr"][m, k].astype(np.int64) - base) // 512
        self.desc_idx = idx

    def getFeatureCount(self): return len(self.feat)
    def getDescriptorCount(self): return len(self.desc)
    size = getFeatureCount

    def keypoints(self):
        """rows (x, y, sigma, theta) per (feature, orientation) and the matching descriptors"""
        rows, idx = [], []
        for i, f in enumerate(self.feat):
            for k in range(int(f["num_ori"])):
                rows.append((f["x"], f["y"], f["sigma"], f["ori"][k]))
                idx.append(int(self.desc_idx[i, k]))
        kp = np.array(rows, dtype=np.float64).reshape(-1, 4)
        return kp, (self.desc[np.array(idx, dtype=np.int64)] if idx else self.desc[:0])

    def print(self, fh, write_as_uchar=False):
        """reference Feature::print (features.cu:310-330): x y 1/s^2 0 1/s^2 d0..d127"""
        for i, f in enumerate(self.feat):
            sigval = np.float32(1.0) / (np.float32(f["sigma"]) * np.float32(f["sigma"]))
            for k in range(int(f["num_ori"])):
                d = self.desc[self.desc_idx[i, k]]
                if write_as_uchar:
                    ds = " ".join("%g" % np.round(v) for v in d)
                else:
                    ds = " ".join("%.3g" % v for v in d)
                fh.write("%g %g %g 0 %g %s \n" % (f["x"], f["y"], sigval, sigval, ds))


class FeaturesDev:
    """FeaturesDev (reference src/popsift/features.h:104-122): Feature records, descriptors and the
    descriptor -> feature reverse map in DEVICE memory owned by this object (Config.MatchingMode).
    getFeatures / getDescriptors / getReverseMap return raw device addresses."""

    def __init__(self, lib, n_feat: int, n_desc: int):
        self._lib, self._nf, self._nd = lib, n_feat, n_desc
        self._pf = lib.ps_dev_alloc(max(n_feat, 1) * 72)
        self._pd = lib.ps_dev_alloc(max(n_desc, 1) * 512)
        self._pr = lib.ps_dev_alloc(max(n_desc, 1) * 4)
        if not (self._pf and self._pd and self._pr):
            raise PopSiftError("Failed to allocate device memory for features")

    def getFeatureCount(self): return self._nf
    def getDescriptorCount(self): return self._nd
    size = getFeatureCount
    def getFeatures(self): return self._pf
    def getDescriptors(self): return self._pd
    def getReverseMap(self): return self._pr

    MATCH_AUTO, MATCH_EXACT, MATCH_TENSOR = 0, 1, 2

    def match(self, other: "FeaturesDev", flags: int = 0) -> np.ndarray:
        """FeaturesDev::match (reference features.cu:282-304) without the printing: (n_desc, 3) int32 rows
        (best index, second index, accept) of every descriptor of self among other's (C ABI ps_match)."""
        return match_descriptors_dev(self._lib, self._pd, self._nd, other._pd, other._nd, flags)

    def to_host(self):
        """(features, descriptors, reverse map) copied to numpy arrays; desc_ptr still holds DEVICE addresses"""
        feat = np.zeros(self._nf, FEATURE_DTYPE)
        desc = np.zeros((self._nd, 128), np.float32)
        rev = np.zeros(self._nd, np.int32)
        for arr, ptr in ((feat, self._pf), (desc, self._pd), (rev, self._pr)):
            if arr.nbytes and self._lib.ps_dev_to_host(arr.ctypes.data, ptr, arr.nbytes) != 0:
                raise PopSiftError("device -> host copy failed")
        return feat, desc, rev

    def __del__(self):
        lib = getattr(self, "_lib", None)
        if lib is not None:
            for p in (self._pf, self._pd, self._pr):
                if p:
                    lib.ps_dev_free(p)
            self._pf = self._pd = self._pr = None


def _last_error(lib) -> str:
    return lib.ps_last_error(None).decode()


def _check(lib, rc, name):
    if rc != 0:
        raise PopSiftError("%s error %d: %s" % (name, rc, _last_error(lib)))


def _c_pairs(pairs):
    """the (left, right) pairs as the C ABI's flat int32 array"""
    flat = [int(v) for pq in pairs for v in pq]
    return (C.c_int32 * max(len(flat), 1))(*flat)


def _pair_rows(counts, pairs) -> list:
    """each pair's result rows: its left set's count (none for an index out of range, which the C ABI refuses)"""
    return [counts[l] if 0 <= l < len(counts) else 0 for l, _ in pairs]


def _split_rows(out, rows) -> list:
    """out's rows split by pair, rows[p] of them for pair p"""
    ends = np.cumsum(rows, dtype=np.int64)
    return [out[e - n:e] for n, e in zip(rows, ends)]


def _model_code(model) -> int:
    """GEOM's code of a model name; a code is returned as it is"""
    if isinstance(model, str):
        if model not in GEOM:
            raise PopSiftError("model must be one of %s" % ", ".join(GEOM))
        model = GEOM[model]
    return int(model)


def match_descriptors_dev(lib, d_left, n_left, d_right, n_right, flags=0, device=None) -> np.ndarray:
    if n_left <= 0:
        return np.zeros((0, 3), np.int32)
    bufs = _DevBuffers(lib)
    try:
        d_out = bufs.alloc(n_left * 12)
        dev = device if device is not None else max(0, lib.ps_pointer_device(d_left))
        _check(lib, lib.ps_match(dev, d_left, n_left, d_right, n_right, d_out, flags), "ps_match")
        return bufs.download(d_out, (n_left, 3), np.int32)
    finally:
        bufs.free()


def match_descriptors(left: np.ndarray, right: np.ndarray, flags=0, device=0) -> np.ndarray:
    """host arrays (n, 128) float32 -> (n_left, 3) int32 (best, second, accept); copies through device memory"""
    lib = load_library()
    left = np.ascontiguousarray(left, np.float32); right = np.ascontiguousarray(right, np.float32)
    bufs = _DevBuffers(lib)
    try:
        return match_descriptors_dev(lib, bufs.upload(left), len(left), bufs.upload(right), len(right), flags, device)
    finally:
        bufs.free()


def _match_pairs(sets, pairs, flags, device, u8) -> list:
    """match_pairs (ps_match_batch) or match_pairs_u8 (ps_match_u8_batch)"""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    name = "ps_match_u8_batch" if u8 else "ps_match_batch"
    bufs = _DevBuffers(lib)
    try:
        c_sets, c_n, counts, device = _desc_sets(lib, bufs, sets, device, u8)
        rows = _pair_rows(counts, pairs)
        d_out = bufs.alloc(sum(rows) * 12)
        _check(lib, getattr(lib, name)(device, len(sets), c_sets, c_n, len(pairs), _c_pairs(pairs), d_out, flags), name)
        out = bufs.download(d_out, (sum(rows), 3), np.int32)
    finally:
        bufs.free()
    return _split_rows(out, rows)


def match_pairs(sets, pairs, flags=0, device=None) -> list:
    """2-NN matching of many pairs in one call (C ABI ps_match_batch; an addition to the reference's interface).
    `sets` holds FeaturesDev objects or host (n, 128) float32 arrays (copied through device memory); `pairs` is a list of
    (left, right) indices into `sets`.  Entry p is the (n_left, 3) int32 array (best, second, accept) that
    match_descriptors(sets[l], sets[r], flags) gives."""
    return _match_pairs(sets, pairs, flags, device, False)


def _to_u8_dev(lib, d_in, n, device) -> int:
    """device copy of n float descriptors at d_in quantised to 8 bits (ps_descriptors_to_u8); the caller frees it"""
    q = lib.ps_dev_alloc(max(n * 128, 16))
    if not q:
        raise PopSiftError("ps_dev_alloc failed")
    rc = lib.ps_descriptors_to_u8(device, d_in, n, q) if n else 0
    if rc != 0:
        lib.ps_dev_free(q)
        _check(lib, rc, "ps_descriptors_to_u8")
    return q


def descriptors_to_u8(x, device=None) -> np.ndarray:
    """8-bit descriptors computed on the device (C ABI ps_descriptors_to_u8): roundf(min(max(v, 0), 255)) per component,
    NaN -> 0 -- what the reference prints under --write-as-uchar, saturated.  `x` is a FeaturesDev or a host (n, 128)
    float32 array; returns a host (n, 128) uint8 array."""
    lib = load_library()
    bufs = _DevBuffers(lib)
    try:
        c_sets, _, (n,), device = _desc_sets(lib, bufs, [x], device)
        q = _to_u8_dev(lib, c_sets[0], n, device)
        bufs.ptrs.append(q)
        return bufs.download(q, (n, 128), np.uint8)
    finally:
        bufs.free()


def match_pairs_u8(sets, pairs, flags=0, device=None) -> list:
    """match_pairs for 8-bit descriptors with exact integer distances (C ABI ps_match_u8_batch).  `sets` holds host (n, 128)
    uint8 arrays (copied through device memory) or FeaturesDev objects (quantised on the device by ps_descriptors_to_u8;
    the descriptors never leave it).  Entry p is the (n_left, 3) int32 array (best, second, accept), row for row what
    match_pairs gives on float32 copies of the 8-bit sets under FeaturesDev.MATCH_EXACT."""
    return _match_pairs(sets, pairs, flags, device, True)


class _DevBuffers:
    """device allocations of one call, freed together"""

    def __init__(self, lib):
        self.lib, self.ptrs = lib, []

    def alloc(self, nbytes: int) -> int:
        p = self.lib.ps_dev_alloc(max(int(nbytes), 16))
        if not p:
            raise PopSiftError("ps_dev_alloc failed")
        self.ptrs.append(p)
        return p

    def upload(self, a: np.ndarray) -> int:
        a = np.ascontiguousarray(a)
        p = self.alloc(a.nbytes)
        if a.nbytes and self.lib.ps_host_to_dev(p, a.ctypes.data, a.nbytes) != 0:
            raise PopSiftError("host -> device copy failed")
        return p

    def download(self, ptr: int, shape, dtype) -> np.ndarray:
        out = np.zeros(shape, dtype)
        if out.nbytes and self.lib.ps_dev_to_host(out.ctypes.data, ptr, out.nbytes) != 0:
            raise PopSiftError("device -> host copy failed")
        return out

    def free(self):
        while self.ptrs:
            self.lib.ps_dev_free(self.ptrs.pop())


def _desc_sets(lib, bufs, sets, device=None, u8=False):
    """The C ABI arrays of descriptor sets: FeaturesDev objects, or host (n, 128) arrays uploaded into bufs (float32, or
    uint8 with u8=True).  With u8=True FeaturesDev sets are quantised on the device into bufs.  Returns (c_sets, c_n,
    counts, device); a device of None becomes that of the first non-empty set, else 0."""
    ptrs, counts = [], []
    for s in sets:
        if isinstance(s, FeaturesDev):
            ptrs.append(s.getDescriptors()); counts.append(s.getDescriptorCount())
            continue
        a = np.ascontiguousarray(s, np.uint8 if u8 else np.float32).reshape(-1, 128)
        ptrs.append(bufs.upload(a)); counts.append(len(a))
    if device is None:
        device = next((max(0, lib.ps_pointer_device(p)) for p, n in zip(ptrs, counts) if n > 0), 0)
    if u8:
        for i, s in enumerate(sets):
            if isinstance(s, FeaturesDev):
                ptrs[i] = _to_u8_dev(lib, ptrs[i], counts[i], device)
                bufs.ptrs.append(ptrs[i])
    n = max(len(sets), 1)
    return (C.c_void_p * n)(*ptrs), (C.c_int32 * n)(*counts), counts, device


def _verify_params(model="homography", threshold=4.0, n_samples=1024, seed=0, refine=True) -> PsVerifyParams:
    return PsVerifyParams(_model_code(model), int(n_samples), float(threshold), 1 if refine else 0, int(seed) & ((1 << 64) - 1))


def _correspondences_dev(lib, bufs, sets, pairs, d_match, device):
    """ps_match_correspondences on device-resident match rows: (d_corr, d_src, start, n_corr)"""
    for s in sets:
        if not isinstance(s, FeaturesDev):
            raise PopSiftError("correspondences need FeaturesDev sets (Config.MatchingMode)")
    counts = [s.getDescriptorCount() for s in sets]
    start = np.concatenate([[0], np.cumsum([counts[l] for l, _ in pairs])]).astype(np.int32)
    rows = int(start[-1])
    d_corr, d_src = bufs.alloc(rows * 16), bufs.alloc(rows * 4)
    n_corr = np.zeros(max(len(pairs), 1), np.int32)
    c_feat = (C.c_void_p * max(len(sets), 1))(*[s.getFeatures() for s in sets])
    c_rev = (C.c_void_p * max(len(sets), 1))(*[s.getReverseMap() for s in sets])
    c_n = (C.c_int32 * max(len(sets), 1))(*counts)
    rc = lib.ps_match_correspondences(device, len(sets), c_feat, c_rev, c_n, len(pairs), _c_pairs(pairs), d_match, d_corr, d_src,
                                      n_corr.ctypes.data)
    _check(lib, rc, "ps_match_correspondences")
    return d_corr, d_src, start[:len(pairs)].copy(), n_corr[:len(pairs)].copy()


def _verify_dev(lib, bufs, device, d_corr, start, n_corr, prm: PsVerifyParams, taps=False, d_models=None, d_mask=None):
    """ps_verify_batch: host (models (P, 3, 3), counts (P,), mask (rows,) bool[, tap counts, tap models]); the models are
    written to d_models (P x 9 floats of device memory) and the mask to d_mask (a byte per row) when given"""
    P = len(start)
    rows = int(max((int(a) + int(b) for a, b in zip(start, n_corr)), default=0))
    d_models = bufs.alloc(P * 36) if d_models is None else d_models
    d_n = bufs.alloc(P * 4)
    d_mask = bufs.alloc(rows) if d_mask is None else d_mask
    k = 1 if prm.model == 0 else 3
    tp = None
    if taps:
        nh = P * k * prm.n_samples
        tp = PsVerifyTaps(bufs.alloc(nh * 4), bufs.alloc(nh * 36))
    c_start = np.ascontiguousarray(start, np.int32)
    c_n = np.ascontiguousarray(n_corr, np.int32)
    rc = lib.ps_verify_batch(device, P, d_corr, c_start.ctypes.data, c_n.ctypes.data, C.byref(prm), d_models, d_n, d_mask,
                             C.byref(tp) if tp is not None else None)
    _check(lib, rc, "ps_verify_batch")
    out = [bufs.download(d_models, (P, 3, 3), np.float32), bufs.download(d_n, P, np.int32),
           bufs.download(d_mask, rows, np.uint8).astype(bool)]
    if taps:
        nh = k * prm.n_samples
        out += [bufs.download(tp.d_counts, (P, nh), np.int32), bufs.download(tp.d_models, (P, nh, 3, 3), np.float32)]
    return out


def match_correspondences(sets, pairs, matches, device=None):
    """Point correspondences of matched pairs (C ABI ps_match_correspondences; an addition to the reference's interface).
    `sets` are FeaturesDev objects (Config.MatchingMode), `pairs` the (left, right) list and `matches` the per-pair (n_left, 3)
    rows that match_pairs / match_pairs_u8 gave for them.  Returns (corrs, src): per pair an (n, 4) float32 array of
    x_l, y_l, x_r, y_r in pixels and the (n,) int32 left descriptor rows they came from."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    if len(matches) != len(pairs):
        raise PopSiftError("one match array per pair expected")
    bufs = _DevBuffers(lib)
    try:
        device = _desc_sets(lib, bufs, sets, device)[3]
        m = np.concatenate([np.asarray(r, np.int32).reshape(-1, 3) for r in matches]) if matches else np.zeros((0, 3), np.int32)
        d_corr, d_src, start, n_corr = _correspondences_dev(lib, bufs, sets, pairs, bufs.upload(m), device)
        rows = len(m)
        corr = bufs.download(d_corr, (rows, 4), np.float32)
        src = bufs.download(d_src, rows, np.int32)
    finally:
        bufs.free()
    return ([corr[a:a + n].copy() for a, n in zip(start, n_corr)], [src[a:a + n].copy() for a, n in zip(start, n_corr)])


def verify_correspondences(corrs, model="homography", threshold=4.0, n_samples=1024, seed=0, refine=True, taps=False, device=0):
    """Batched RANSAC on host correspondences (C ABI ps_verify_batch): `corrs` is a list of (n, 4) arrays x_l, y_l, x_r, y_r in
    pixels.  Returns per pair (model (3, 3) float32 mapping left to right, inlier count, (n,) bool inlier mask); with
    taps=True also (counts, models): every hypothesis's inlier count (P, k * n_samples; -1 invalid) and pixel model
    (P, k * n_samples, 3, 3), k = 1 for a homography and 3 for a fundamental matrix."""
    lib = load_library()
    prm = _verify_params(model, threshold, n_samples, seed, refine)
    arrs = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in corrs]
    n_corr = np.array([len(a) for a in arrs], np.int32)
    start = np.concatenate([[0], np.cumsum(n_corr)])[:len(arrs)].astype(np.int32)
    bufs = _DevBuffers(lib)
    try:
        allc = np.concatenate(arrs) if arrs else np.zeros((0, 4), np.float32)
        out = _verify_dev(lib, bufs, device, bufs.upload(allc), start, n_corr, prm, taps)
    finally:
        bufs.free()
    models, counts, mask = out[:3]
    res = [(models[p], int(counts[p]), mask[start[p]:start[p] + n_corr[p]]) for p in range(len(arrs))]
    return (res, (out[3], out[4])) if taps else res


def verify_pairs(sets, pairs, matches=None, flags=0, u8=False, device=None, guided=False, **params):
    """Verified matches and a two-view model per pair without leaving the device: match_pairs (or match_pairs_u8 with
    u8=True) when `matches` is None, then ps_match_correspondences and ps_verify_batch.  `sets` are FeaturesDev objects;
    params are verify_correspondences' (model, threshold, n_samples, seed, refine).  Returns per pair (model (3, 3) float32
    in pixels, inlier count, int32 array of the inliers' left descriptor rows).
    guided=True adds guided matching on the device-resident models at the same threshold (ps_match_guided_batch, or
    ps_match_u8_guided_batch with u8=True) and gathers the correspondences again: per pair (model, number of guided
    correspondences, int32 array of their left descriptor rows)."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    prm = _verify_params(**params)
    bufs = _DevBuffers(lib)
    try:
        ch = _verify_chain(lib, bufs, sets, pairs, matches, flags, u8, device, guided, prm)
        src = bufs.download(ch.d_src, ch.rows, np.int32)
    finally:
        bufs.free()
    out = []
    for p in range(len(pairs)):
        a, n = int(ch.start[p]), int(ch.n_corr[p])
        if guided:
            out.append((ch.models[p], n, src[a:a + n].copy()))
        else:
            out.append((ch.models[p], int(ch.n_in[p]), src[a:a + n][ch.mask[a:a + n]].copy()))
    return out


_Chain = namedtuple("_Chain", "device rows d_match d_src start n_corr d_mask models n_in mask")


def _matched_rows(lib, bufs, sets, pairs, matches, flags, u8, device, u8_copies):
    """The front of the device chains: match_pairs (match_pairs_u8) unless `matches` is given, then
    ps_match_correspondences.  Returns (descs, device, rows, d_match, d_corr, d_src, start, n_corr): descs as _desc_sets
    gave them (8-bit copies only with u8_copies), the device match rows and the correspondences."""
    counts = [s.getDescriptorCount() for s in sets]
    for l, r in pairs:
        if not (0 <= l < len(sets) and 0 <= r < len(sets)):
            raise PopSiftError("set index out of range")
    if matches is not None and len(matches) != len(pairs):
        raise PopSiftError("one match array per pair expected")
    rows = sum(counts[l] for l, _ in pairs)
    descs = _desc_sets(lib, bufs, sets, device, u8_copies)
    c_sets, c_n, _, device = descs
    if matches is not None:
        m = np.concatenate([np.asarray(r, np.int32).reshape(-1, 3) for r in matches]) if matches else np.zeros((0, 3), np.int32)
        d_match = bufs.upload(m)
    else:
        d_match = bufs.alloc(rows * 12)
        fn = lib.ps_match_u8_batch if u8 else lib.ps_match_batch
        _check(lib, fn(device, len(sets), c_sets, c_n, len(pairs), _c_pairs(pairs), d_match, flags), "matching")
    d_corr, d_src, start, n_corr = _correspondences_dev(lib, bufs, sets, pairs, d_match, device)
    return descs, device, rows, d_match, d_corr, d_src, start, n_corr


def _verify_chain(lib, bufs, sets, pairs, matches, flags, u8, device, guided, prm) -> _Chain:
    """verify_pairs' device chain: _matched_rows, ps_verify_batch, and with guided=True guided matching and the
    correspondences again.  Device arrays in bufs: d_match, the rows the final correspondences came from; d_src, start,
    n_corr, those correspondences; d_mask, the verification's inlier mask, or None after guided matching (every guided
    correspondence passed the model).  Host: models, n_in, mask."""
    # the 8-bit copies are made only when matching uses them
    descs, device, rows, d_match, d_corr, d_src, start, n_corr = _matched_rows(
        lib, bufs, sets, pairs, matches, flags, u8, device, u8 and (matches is None or guided))
    d_models, d_mask = bufs.alloc(len(pairs) * 36), bufs.alloc(rows)
    models, n_in, mask = _verify_dev(lib, bufs, device, d_corr, start, n_corr, prm, d_models=d_models, d_mask=d_mask)
    if guided:
        d_match = _match_guided_dev(lib, bufs, sets, descs, pairs, d_models, prm.model, prm.threshold, flags, u8)
        _, d_src, start, n_corr = _correspondences_dev(lib, bufs, sets, pairs, d_match, device)
        d_mask = mask = None
    return _Chain(device, rows, d_match, d_src, start, n_corr, d_mask, models, n_in, mask)


TwoView = namedtuple("TwoView", "E F R t n_inliers n_front mask points")
TwoView.__doc__ = """One pair's calibrated two-view geometry (ps_relative_pose_batch, popsift_b200_pose.h): E (3, 3) in calibrated
coordinates, F (3, 3) in pixels, R (3, 3) and unit t with X_r = R X_l + t, the two counts, the (n,) uint8 mask (bit 0
inlier, bit 1 also in front of both cameras) and the (n, 4) float32 points (X, Y, Z, 1) in the left frame with unit baseline,
zero for rows without bit 1 (None unless asked for)."""


def _pose_params(threshold=4.0, n_samples=1024, seed=0, refine=True) -> PsPoseParams:
    return PsPoseParams(int(n_samples), float(threshold), 1 if refine else 0, 0, int(seed) & ((1 << 64) - 1))


def _c_cameras(cams) -> np.ndarray:
    """(fx, fy, cx, cy) rows as a contiguous float32 array of ps_camera"""
    return np.ascontiguousarray(np.asarray(cams, np.float32).reshape(-1, 4))


def _pose_dev(lib, bufs, device, d_corr, start, n_corr, cams, prm: PsPoseParams, points=False, taps=False):
    """ps_relative_pose_batch: (d_out, d_mask, host two-view records, mask (rows,) uint8, points or None[, tap counts,
    tap models])"""
    P = len(start)
    rows = int(max((int(a) + int(b) for a, b in zip(start, n_corr)), default=0))
    d_out, d_mask = bufs.alloc(P * 128), bufs.alloc(rows)
    d_pts = bufs.alloc(rows * 16) if points else None
    tp = None
    if taps:
        nh = P * 10 * prm.n_samples
        tp = PsVerifyTaps(bufs.alloc(nh * 4), bufs.alloc(nh * 36))
    c_start = np.ascontiguousarray(start, np.int32)
    c_n = np.ascontiguousarray(n_corr, np.int32)
    rc = lib.ps_relative_pose_batch(device, P, d_corr, c_start.ctypes.data, c_n.ctypes.data, cams.ctypes.data, C.byref(prm), d_out,
                                    d_mask, d_pts, C.byref(tp) if tp is not None else None)
    _check(lib, rc, "ps_relative_pose_batch")
    out = [d_out, d_mask, bufs.download(d_out, P, TWO_VIEW_DTYPE), bufs.download(d_mask, rows, np.uint8),
           bufs.download(d_pts, (rows, 4), np.float32) if points else None]
    if taps:
        nh = 10 * prm.n_samples
        out += [bufs.download(tp.d_counts, (P, nh), np.int32), bufs.download(tp.d_models, (P, nh, 3, 3), np.float32)]
    return out


def relative_pose_correspondences(corrs, cameras, threshold=4.0, n_samples=1024, seed=0, refine=True, points=False, taps=False,
                                  device=0):
    """Batched five-point RANSAC, relative pose and triangulation on host correspondences (C ABI ps_relative_pose_batch in
    popsift_b200_pose.h; an addition to the reference's interface).  `corrs` is a list of (n, 4) arrays x_l, y_l, x_r, y_r
    in undistorted pixels and `cameras` one (left, right) pair of (fx, fy, cx, cy) per array.  Returns a TwoView per pair;
    with taps=True also (counts, models): every hypothesis's inlier count (P, 10 * n_samples; -1 invalid) and calibrated
    E (P, 10 * n_samples, 3, 3)."""
    lib = load_library()
    prm = _pose_params(threshold, n_samples, seed, refine)
    arrs = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in corrs]
    cams = np.asarray(cameras, np.float32)
    if cams.shape != (len(arrs), 2, 4):
        raise PopSiftError("one (left, right) pair of (fx, fy, cx, cy) per correspondence array expected")
    cams = _c_cameras(cams)
    n_corr = np.array([len(a) for a in arrs], np.int32)
    start = np.concatenate([[0], np.cumsum(n_corr)])[:len(arrs)].astype(np.int32)
    bufs = _DevBuffers(lib)
    try:
        allc = np.concatenate(arrs) if arrs else np.zeros((0, 4), np.float32)
        out = _pose_dev(lib, bufs, device, bufs.upload(allc), start, n_corr, cams, prm, points, taps)
    finally:
        bufs.free()
    tv, mask, pts = out[2:5]
    res = []
    for p in range(len(arrs)):
        a, n = int(start[p]), int(n_corr[p])
        r = tv[p]
        res.append(TwoView(r["E"].copy(), r["F"].copy(), r["R"].copy(), r["t"].copy(), int(r["n_inliers"]), int(r["n_front"]),
                           mask[a:a + n].copy(), pts[a:a + n].copy() if points else None))
    return (res, (out[5], out[6])) if taps else res


def relative_poses(sets, pairs, cameras, matches=None, flags=0, u8=False, device=None, points=False, **params):
    """Calibrated two-view geometry of matched pairs without leaving the device: match_pairs (match_pairs_u8 with u8=True)
    unless `matches` is given, ps_match_correspondences, then ps_relative_pose_batch.  `sets` are FeaturesDev objects,
    `cameras` one (fx, fy, cx, cy) per set, params relative_pose_correspondences' (threshold, n_samples, seed, refine).
    Returns per pair (TwoView, int32 left descriptor rows of the inliers (bit 0), int32 left descriptor rows of the rows
    in front (bit 1))."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    prm = _pose_params(**params)
    cam = np.asarray(cameras, np.float32).reshape(-1, 4)
    if len(cam) != len(sets):
        raise PopSiftError("one camera per set expected")
    bufs = _DevBuffers(lib)
    try:
        _, device, rows, _, d_corr, d_src, start, n_corr = _matched_rows(lib, bufs, sets, pairs, matches, flags, u8, device,
                                                                        u8 and matches is None)
        cams = _c_cameras([cam[i] for lr in pairs for i in lr])
        out = _pose_dev(lib, bufs, device, d_corr, start, n_corr, cams, prm, points)
        src = bufs.download(d_src, rows, np.int32)
    finally:
        bufs.free()
    tv, mask, pts = out[2:5]
    res = []
    for p in range(len(pairs)):
        a, n = int(start[p]), int(n_corr[p])
        r, m, sr = tv[p], mask[a:a + n], src[a:a + n]
        two = TwoView(r["E"].copy(), r["F"].copy(), r["R"].copy(), r["t"].copy(), int(r["n_inliers"]), int(r["n_front"]), m.copy(),
                      pts[a:a + n].copy() if points else None)
        res.append((two, sr[(m & 1) != 0].copy(), sr[(m & 2) != 0].copy()))
    return res


TwoViewGeometry = namedtuple("TwoViewGeometry", "config pose normal tri_angle n_e n_f n_h n_rotation inlier_rows front_rows")
TwoViewGeometry.__doc__ = """One pair's two-view configuration (ps_two_view_config_batch, popsift_b200_twoview.h): config, a name of
TV_CONFIG; pose, the TwoView that replaces ps_relative_pose_batch's (the essential pose for "general", the homography's
for "planar", the rotation alone with t = 0 for "panoramic", zero otherwise); the unit plane normal (3,) in the left frame
("planar", else zero); tri_angle, the median triangulation angle of the bit-1 rows in degrees; the inlier counts of E, F
and H and the H inliers the pure rotation explains; the rows with bit 0 and with bit 1 (left descriptor rows from
two_view_geometries, correspondence indices from two_view_config_correspondences)."""


def _two_view_config_params(threshold=4.0, min_inliers=15, min_ef_ratio=0.95, max_h_ratio=0.8, min_rotation_ratio=0.9):
    return PsTwoViewConfigParams(int(min_inliers), float(threshold), float(min_ef_ratio), float(max_h_ratio), float(min_rotation_ratio))


def _two_view_config_dev(lib, bufs, device, d_corr, start, n_corr, cams, pprm: PsPoseParams, cprm: PsTwoViewConfigParams, points=False):
    """The three RANSACs and ps_two_view_config_batch on device correspondences: ps_verify_batch with the homography and the
    fundamental matrix and ps_relative_pose_batch, all with pprm's threshold, samples, seed and refit.  Returns (d_out,
    d_mask, host two-view records, mask (rows,) uint8, points or None, info (P,) TWO_VIEW_INFO_DTYPE)."""
    P = len(start)
    rows = int(max((int(a) + int(b) for a, b in zip(start, n_corr)), default=0))
    c_start = np.ascontiguousarray(start, np.int32)
    c_n = np.ascontiguousarray(n_corr, np.int32)
    d_h, d_hn, d_hmask = bufs.alloc(P * 36), bufs.alloc(P * 4), bufs.alloc(rows)
    d_f, d_fn, d_fmask = bufs.alloc(P * 36), bufs.alloc(P * 4), bufs.alloc(rows)
    for model, dm, dn, dk in ((0, d_h, d_hn, d_hmask), (1, d_f, d_fn, d_fmask)):
        vp = PsVerifyParams(model, pprm.n_samples, pprm.threshold, pprm.refine, pprm.seed)
        _check(lib, lib.ps_verify_batch(device, P, d_corr, c_start.ctypes.data, c_n.ctypes.data, C.byref(vp), dm, dn, dk, None),
               "ps_verify_batch")
    d_e, d_emask = _pose_dev(lib, bufs, device, d_corr, start, n_corr, cams, pprm)[:2]
    d_out, d_mask = bufs.alloc(P * 128), bufs.alloc(rows)
    d_pts = bufs.alloc(rows * 16) if points else None
    info = np.zeros(max(P, 1), TWO_VIEW_INFO_DTYPE)
    rc = lib.ps_two_view_config_batch(device, P, d_corr, c_start.ctypes.data, c_n.ctypes.data, cams.ctypes.data, d_e, d_emask, d_fn,
                                      d_h, d_hmask, C.byref(cprm), d_out, d_mask, d_pts, info.ctypes.data)
    _check(lib, rc, "ps_two_view_config_batch")
    return (d_out, d_mask, bufs.download(d_out, P, TWO_VIEW_DTYPE), bufs.download(d_mask, rows, np.uint8),
            bufs.download(d_pts, (rows, 4), np.float32) if points else None, info[:P].copy())


def _two_view_geometry(rec, info, mask, pts, rows) -> "TwoViewGeometry":
    two = TwoView(rec["E"].copy(), rec["F"].copy(), rec["R"].copy(), rec["t"].copy(), int(rec["n_inliers"]), int(rec["n_front"]),
                  mask.copy(), pts)
    return TwoViewGeometry(TV_CONFIG[int(info["config"])], two, info["normal"].copy(), float(info["tri_angle"]), int(info["n_e"]),
                           int(info["n_f"]), int(info["n_h"]), int(info["n_rotation"]), rows[(mask & 1) != 0].copy(),
                           rows[(mask & 2) != 0].copy())


def two_view_config_correspondences(corrs, cameras, threshold=4.0, n_samples=1024, seed=0, refine=True, points=False, device=0,
                                    **config):
    """Two-view configuration on host correspondences (C ABI ps_two_view_config_batch in popsift_b200_twoview.h, after
    ps_verify_batch's homography and fundamental matrix and ps_relative_pose_batch, all with the given threshold, n_samples,
    seed and refine; an addition to the reference's interface).  `corrs` and `cameras` as for relative_pose_correspondences;
    config: min_inliers (15), min_ef_ratio (0.95), max_h_ratio (0.8), min_rotation_ratio (0.9); the pure-rotation test uses
    `threshold`.  Returns a TwoViewGeometry per pair, its rows the correspondence indices."""
    lib = load_library()
    pprm = _pose_params(threshold, n_samples, seed, refine)
    cprm = _two_view_config_params(threshold, **config)
    arrs = [np.ascontiguousarray(c, np.float32).reshape(-1, 4) for c in corrs]
    cams = np.asarray(cameras, np.float32)
    if cams.shape != (len(arrs), 2, 4):
        raise PopSiftError("one (left, right) pair of (fx, fy, cx, cy) per correspondence array expected")
    cams = _c_cameras(cams)
    n_corr = np.array([len(a) for a in arrs], np.int32)
    start = np.concatenate([[0], np.cumsum(n_corr)])[:len(arrs)].astype(np.int32)
    bufs = _DevBuffers(lib)
    try:
        allc = np.concatenate(arrs) if arrs else np.zeros((0, 4), np.float32)
        _, _, tv, mask, pts, info = _two_view_config_dev(lib, bufs, device, bufs.upload(allc), start, n_corr, cams, pprm, cprm, points)
    finally:
        bufs.free()
    out = []
    for p in range(len(arrs)):
        a, n = int(start[p]), int(n_corr[p])
        out.append(_two_view_geometry(tv[p], info[p], mask[a:a + n], pts[a:a + n].copy() if points else None, np.arange(n, dtype=np.int32)))
    return out


def two_view_geometries(sets, pairs, cameras, matches=None, flags=0, u8=False, device=None, points=False, threshold=4.0, n_samples=1024,
                        seed=0, refine=True, **config):
    """Two-view configuration of matched pairs without leaving the device: relative_poses' chain (matching unless `matches`
    is given, ps_match_correspondences), ps_verify_batch with the homography and the fundamental matrix and
    ps_relative_pose_batch on the same rows (threshold, n_samples, seed and refine for all three), then
    ps_two_view_config_batch.  `sets` are FeaturesDev objects, `cameras` one (fx, fy, cx, cy) per set, config
    two_view_config_correspondences'.  Returns a TwoViewGeometry per pair, its rows the left descriptor rows; its pose feeds
    rotation_averaging and filter_view_graph unchanged."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    pprm = _pose_params(threshold, n_samples, seed, refine)
    cprm = _two_view_config_params(threshold, **config)
    cam = np.asarray(cameras, np.float32).reshape(-1, 4)
    if len(cam) != len(sets):
        raise PopSiftError("one camera per set expected")
    bufs = _DevBuffers(lib)
    try:
        _, device, rows, _, d_corr, d_src, start, n_corr = _matched_rows(lib, bufs, sets, pairs, matches, flags, u8, device,
                                                                        u8 and matches is None)
        cams = _c_cameras([cam[i] for lr in pairs for i in lr])
        _, _, tv, mask, pts, info = _two_view_config_dev(lib, bufs, device, d_corr, start, n_corr, cams, pprm, cprm, points)
        src = bufs.download(d_src, rows, np.int32)
    finally:
        bufs.free()
    out = []
    for p in range(len(pairs)):
        a, n = int(start[p]), int(n_corr[p])
        out.append(_two_view_geometry(tv[p], info[p], mask[a:a + n], pts[a:a + n].copy() if points else None, src[a:a + n]))
    return out


Tracks = namedtuple("Tracks", "start set feature track_of n_components n_conflicting n_short")
Tracks.__doc__ = """Feature tracks: track t's members are set[start[t]:start[t + 1]] / feature[start[t]:start[t + 1]]
(ascending by set); track_of[i][f] is feature f of set i's track, or -1; the counts of dropped components."""


def _tracks_dev(lib, bufs, n_feat, min_length, call) -> Tracks:
    """the outputs of a track entry point: `call(d_track_of, d_track_start, d_members, counts)` returns its code"""
    return _tracks_run(lib, bufs, n_feat, min_length, call)[0]


def _tracks_run(lib, bufs, n_feat, min_length, call):
    """_tracks_dev's Tracks with the device arrays d_track_start and d_members they were read from (they stay in bufs)"""
    n_feat = [int(n) for n in n_feat]
    off = np.concatenate([[0], np.cumsum(n_feat, dtype=np.int64)]).astype(np.int64)
    N = int(off[-1])
    cap = N // max(int(min_length), 2) + 1
    d_of, d_start, d_mem = bufs.alloc(N * 4), bufs.alloc(cap * 4), bufs.alloc(N * 4)
    cnt = PsTrackCounts()
    _check(lib, call(d_of, d_start, d_mem, cnt), "tracks")
    start = bufs.download(d_start, cnt.n_tracks + 1, np.int32)
    mem = bufs.download(d_mem, cnt.n_members, np.int32)
    of = bufs.download(d_of, N, np.int32)
    s = (np.searchsorted(off, mem, side="right") - 1).astype(np.int32)
    return Tracks(start, s, (mem - off[s]).astype(np.int32), [of[off[i]:off[i + 1]] for i in range(len(n_feat))],
                  cnt.n_components, cnt.n_conflicting, cnt.n_short), d_start, d_mem


def build_tracks(n_feat, edges, min_length=2, device=0) -> Tracks:
    """Feature tracks of an explicit edge list (C ABI ps_tracks_from_edges in popsift_b200_tracks.h; an addition to the
    reference's interface): the connected components of the edges over all features, without those holding two features
    of one set and those shorter than min_length (>= 2).  `n_feat` is each set's feature count, `edges` an (E, 4) int32
    array of (set_a, feature_a, set_b, feature_b)."""
    lib = load_library()
    n_feat = [int(n) for n in n_feat]
    e = np.ascontiguousarray(edges, np.int64).reshape(-1, 4)
    nf = np.asarray(n_feat + [0], np.int64)
    for s, f in ((e[:, 0], e[:, 1]), (e[:, 2], e[:, 3])):
        if ((s < 0) | (s >= len(n_feat))).any() or ((f < 0) | (f >= nf[np.clip(s, 0, len(n_feat))])).any():
            raise PopSiftError("edge endpoint out of range")
    off = np.concatenate([[0], np.cumsum(n_feat, dtype=np.int64)])
    g = np.stack([off[e[:, 0]] + e[:, 1], off[e[:, 2]] + e[:, 3]], axis=1).astype(np.int32)
    c_n = (C.c_int32 * max(len(n_feat), 1))(*n_feat)
    bufs = _DevBuffers(lib)
    try:
        d_e = bufs.upload(g)
        return _tracks_dev(lib, bufs, n_feat, min_length, lambda of, st, mem, cnt: lib.ps_tracks_from_edges(
            device, len(n_feat), c_n, len(g), d_e, int(min_length), of, st, mem, C.byref(cnt)))
    finally:
        bufs.free()


def tracks(sets, pairs, matches=None, min_length=2, guided=False, u8=False, flags=0, device=None, **verify_params) -> Tracks:
    """Feature tracks of a whole SfM front end on the device (C ABI ps_tracks_from_matches in popsift_b200_tracks.h):
    verify_pairs' chain on FeaturesDev `sets` and `pairs` (match, correspond, verify with verify_params; guided matching with
    guided=True), then the tracks of its verified inliers (of every guided correspondence with guided=True).  Only the
    tracks come back."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    prm = _verify_params(**verify_params)
    bufs = _DevBuffers(lib)
    try:
        return _tracks_chain(lib, bufs, sets, pairs, matches, min_length, guided, u8, flags, device, prm)[0]
    finally:
        bufs.free()


def _tracks_chain(lib, bufs, sets, pairs, matches, min_length, guided, u8, flags, device, prm):
    """tracks()' device chain: _verify_chain, then ps_tracks_from_matches on its arrays.  Returns (Tracks, device,
    d_track_start, d_members), the device arrays in bufs"""
    ch = _verify_chain(lib, bufs, sets, pairs, matches, flags, u8, device, guided, prm)
    n = max(len(sets), 1)
    n_feat = [s.getFeatureCount() for s in sets]
    c_nf = (C.c_int32 * n)(*n_feat)
    c_rev = (C.c_void_p * n)(*[s.getReverseMap() for s in sets])
    c_nd = (C.c_int32 * n)(*[s.getDescriptorCount() for s in sets])
    c_corr = np.ascontiguousarray(ch.n_corr, np.int32)
    tr, d_start, d_mem = _tracks_run(lib, bufs, n_feat, min_length, lambda of, st, mem, cnt: lib.ps_tracks_from_matches(
        ch.device, len(sets), c_nf, c_rev, c_nd, len(pairs), _c_pairs(pairs), ch.d_match, ch.d_src, c_corr.ctypes.data,
        ch.d_mask, int(min_length), of, st, mem, C.byref(cnt)))
    return tr, ch.device, d_start, d_mem


TrackPoints = namedtuple("TrackPoints", "X error angle n_inliers status mask obs_error counts")
TrackPoints.__doc__ = """Multi-view triangulation of tracks (ps_triangulate_tracks, popsift_b200_triangulate.h): per track X (T, 3)
float64 in world coordinates, the mean pixel reprojection error over the inliers, the triangulation angle in degrees, the
inlier count and the status (an index into TRI_STATUS, 0 = ok); per member (aligned with Tracks.set / Tracks.feature) the
uint8 inlier mask and the float32 pixel error (+inf behind the camera or without a point); counts: tracks per status name
and 'inlier_obs'."""


def _tri_params(max_error=4.0, min_angle=1.5, min_views=2, n_samples=256, refine_iters=10, seed=0) -> PsTriangulateParams:
    return PsTriangulateParams(float(max_error), float(min_angle), int(min_views), int(n_samples), int(refine_iters), 0,
                               int(seed) & ((1 << 64) - 1))


def _c_rigids(poses):
    """ps_rigid array of poses given as (R (3, 3), t (3,)) or as [R | t] (3, 4), world to camera"""
    out = (PsRigid * max(len(poses), 1))()
    for i, p in enumerate(poses):
        if isinstance(p, (tuple, list)) and len(p) == 2:
            R, t = np.asarray(p[0], np.float64).reshape(3, 3), np.asarray(p[1], np.float64).reshape(3)
        else:
            m = np.asarray(p, np.float64).reshape(3, 4)
            R, t = m[:, :3], m[:, 3]
        out[i].R[:] = [float(v) for v in R.ravel()]
        out[i].t[:] = [float(v) for v in t]
    return out


def _triangulate_dev(lib, bufs, device, n_feat, c_feat, cameras, poses, n_tracks, d_start, d_mem, n_members, prm) -> TrackPoints:
    """ps_triangulate_tracks on device track arrays; Feature records at c_feat (a C array of device pointers)"""
    cam = _c_cameras(cameras)
    if len(cam) != len(n_feat) or len(poses) != len(n_feat):
        raise PopSiftError("one camera and one pose per set expected")
    n = max(len(n_feat), 1)
    d_pts, d_mask, d_err = bufs.alloc(n_tracks * 40), bufs.alloc(n_members), bufs.alloc(n_members * 4)
    cnt = PsTriangulateCounts()
    rc = lib.ps_triangulate_tracks(device, len(n_feat), (C.c_int32 * n)(*n_feat), c_feat, cam.ctypes.data, _c_rigids(poses), n_tracks,
                                   d_start, d_mem, n_members, C.byref(prm), d_pts, d_mask, d_err, C.byref(cnt))
    _check(lib, rc, "ps_triangulate_tracks")
    pts = bufs.download(d_pts, n_tracks, TRACK_POINT_DTYPE)
    counts = dict(zip(TRI_STATUS, [int(v) for v in cnt.n_status]))
    counts["inlier_obs"] = int(cnt.n_inlier_obs)
    return TrackPoints(pts["X"].copy(), pts["error"].copy(), pts["angle"].copy(), pts["n_inliers"].copy(), pts["status"].copy(),
                       bufs.download(d_mask, n_members, np.uint8), bufs.download(d_err, n_members, np.float32), counts)


def triangulate(sets, tracks, cameras, poses, device=None, **params) -> TrackPoints:
    """Multi-view triangulation of feature tracks from known poses (C ABI ps_triangulate_tracks in
    popsift_b200_triangulate.h; an addition to the reference's interface): a RANSAC over pairs of each track's
    observations, then a Gauss-Newton refinement, for every track in one call.  `sets` are FeaturesDev objects or host
    Features (their records are uploaded), `tracks` a Tracks over them (tracks() / build_tracks()), `cameras` one (fx, fy,
    cx, cy) per set and `poses` one world-to-camera pose per set, (R, t) or [R | t].  params: max_error (px, 4.0),
    min_angle (degrees, 1.5), min_views (2), n_samples (256), refine_iters (10), seed (0)."""
    lib = load_library()
    prm = _tri_params(**params)
    bufs = _DevBuffers(lib)
    try:
        ptrs, n_feat = [], []
        for s in sets:
            if isinstance(s, FeaturesDev):
                ptrs.append(s.getFeatures()); n_feat.append(s.getFeatureCount())
            else:
                f = np.ascontiguousarray(s.feat if isinstance(s, Features) else s, FEATURE_DTYPE)
                ptrs.append(bufs.upload(f)); n_feat.append(len(f))
        if device is None:
            device = next((max(0, lib.ps_pointer_device(p)) for p, k in zip(ptrs, n_feat) if k > 0), 0)
        off = np.concatenate([[0], np.cumsum(n_feat, dtype=np.int64)])
        st = np.ascontiguousarray(tracks.start, np.int32)
        mem = (off[np.asarray(tracks.set, np.int64)] + np.asarray(tracks.feature, np.int64)).astype(np.int32)
        c_feat = (C.c_void_p * max(len(sets), 1))(*ptrs)
        return _triangulate_dev(lib, bufs, device, n_feat, c_feat, cameras, poses, len(st) - 1, bufs.upload(st), bufs.upload(mem),
                                len(mem), prm)
    finally:
        bufs.free()


def triangulated_tracks(sets, pairs, cameras, poses, matches=None, min_length=2, guided=False, u8=False, flags=0, device=None,
                        verify=None, **params):
    """tracks() and triangulate() in one device chain: verify_pairs' chain on FeaturesDev `sets` and `pairs` with the
    verify_pairs parameters in the dict `verify`, ps_tracks_from_matches, then ps_triangulate_tracks on the same device
    arrays.  cameras, poses and params are triangulate()'s.  Returns (Tracks, TrackPoints)."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    vprm = _verify_params(**(verify or {}))
    prm = _tri_params(**params)
    bufs = _DevBuffers(lib)
    try:
        tr, device, d_start, d_mem = _tracks_chain(lib, bufs, sets, pairs, matches, min_length, guided, u8, flags, device, vprm)
        c_feat = (C.c_void_p * max(len(sets), 1))(*[s.getFeatures() for s in sets])
        pts = _triangulate_dev(lib, bufs, device, [s.getFeatureCount() for s in sets], c_feat, cameras, poses, len(tr.start) - 1,
                               d_start, d_mem, len(tr.set), prm)
    finally:
        bufs.free()
    return tr, pts


BundleReport = namedtuple("BundleReport", "initial_cost final_cost iterations accepted cg_iterations termination n_obs n_points "
                                          "n_free_cams")
BundleReport.__doc__ = """ps_bundle_report of ps_bundle_adjust (popsift_b200_bundle.h); termination is a name of BA_TERMINATION."""


def _bundle_params(loss="squared", loss_scale=1.0, max_iters=50, function_tol=1e-6, cg_max_iters=100, cg_tol=1e-6,
                   initial_lambda=1e-4, scale_set=-1, scale_axis=0) -> PsBundleParams:
    if loss not in BA_LOSS:
        raise PopSiftError("loss must be one of %s" % (BA_LOSS,))
    return PsBundleParams(BA_LOSS.index(loss), int(max_iters), int(cg_max_iters), int(scale_set), int(scale_axis), 0,
                          float(loss_scale), float(function_tol), float(cg_tol), float(initial_lambda))


def _bundle_report(r) -> BundleReport:
    return BundleReport(float(r.initial_cost), float(r.final_cost), int(r.iterations), int(r.accepted), int(r.cg_iterations),
                        BA_TERMINATION[r.termination], int(r.n_obs), int(r.n_points), int(r.n_free_cams))


def bundle_adjust(sets, tracks, points, cameras, poses, fixed, loss="squared", loss_scale=1.0, max_iters=50, function_tol=1e-6,
                  cg_max_iters=100, cg_tol=1e-6, initial_lambda=1e-4, scale_set=-1, scale_axis=0, device=None):
    """Bundle adjustment on the device (C ABI ps_bundle_adjust in popsift_b200_bundle.h; an addition to the reference's
    interface): Levenberg-Marquardt on the poses of the free sets and the points of the OK tracks, with a Schur-complement
    PCG solve.  `sets`, `tracks`, `cameras` and `poses` are triangulate()'s; `points` the TrackPoints triangulate() gave
    (the OK tracks' members with mask 1 are the observations); `fixed` one bool per set (at least one True).  loss is
    "squared", "huber" or "cauchy" at loss_scale pixels; scale_set / scale_axis hold one translation component of a free
    set.  Returns (poses as a list of (R, t), TrackPoints with the refined X, error and angle and the final per-member
    pixel errors, BundleReport)."""
    lib = load_library()
    prm = _bundle_params(loss, loss_scale, max_iters, function_tol, cg_max_iters, cg_tol, initial_lambda, scale_set, scale_axis)
    bufs = _DevBuffers(lib)
    try:
        ptrs, n_feat = [], []
        for s in sets:
            if isinstance(s, FeaturesDev):
                ptrs.append(s.getFeatures()); n_feat.append(s.getFeatureCount())
            else:
                f = np.ascontiguousarray(s.feat if isinstance(s, Features) else s, FEATURE_DTYPE)
                ptrs.append(bufs.upload(f)); n_feat.append(len(f))
        if device is None:
            device = next((max(0, lib.ps_pointer_device(p)) for p, k in zip(ptrs, n_feat) if k > 0), 0)
        cam = _c_cameras(cameras)
        if len(cam) != len(n_feat) or len(poses) != len(n_feat) or len(fixed) != len(n_feat):
            raise PopSiftError("one camera, one pose and one fixed flag per set expected")
        off = np.concatenate([[0], np.cumsum(n_feat, dtype=np.int64)])
        st = np.ascontiguousarray(tracks.start, np.int32)
        mem = (off[np.asarray(tracks.set, np.int64)] + np.asarray(tracks.feature, np.int64)).astype(np.int32)
        T, M = len(st) - 1, len(mem)
        rec = np.zeros(T, TRACK_POINT_DTYPE)
        for f in ("X", "error", "angle", "n_inliers", "status"):
            rec[f] = getattr(points, f)
        d_pts = bufs.upload(rec) if T else None
        d_mask = bufs.upload(np.ascontiguousarray(points.mask, np.uint8)) if M else None
        d_err = bufs.alloc(M * 4) if M else None
        n = max(len(n_feat), 1)
        c_fix = (C.c_uint8 * n)(*[1 if f else 0 for f in fixed])
        rig_in = _c_rigids(poses)
        rig_out = (PsRigid * n)()
        rep = PsBundleReport()
        rc = lib.ps_bundle_adjust(device, len(n_feat), (C.c_int32 * n)(*n_feat), (C.c_void_p * n)(*ptrs), cam.ctypes.data, rig_in, T,
                                  bufs.upload(st) if T else None, bufs.upload(mem) if M else None, M, d_pts, d_mask, c_fix,
                                  C.byref(prm), rig_out, d_err, C.byref(rep))
        _check(lib, rc, "ps_bundle_adjust")
        out = bufs.download(d_pts, T, TRACK_POINT_DTYPE) if T else rec
        err = bufs.download(d_err, M, np.float32) if M else np.zeros(0, np.float32)
    finally:
        bufs.free()
    new_poses = [(np.array(rig_out[i].R[:], np.float64).reshape(3, 3), np.array(rig_out[i].t[:], np.float64)) for i in range(len(n_feat))]
    tp = TrackPoints(out["X"].copy(), out["error"].copy(), out["angle"].copy(), out["n_inliers"].copy(), out["status"].copy(),
                     np.asarray(points.mask, np.uint8).copy(), err, dict(points.counts) if points.counts is not None else None)
    return new_poses, tp, _bundle_report(rep)


RotationReport = namedtuple("RotationReport", "initial_cost final_cost iterations cg_iterations n_pairs n_registered termination")
RotationReport.__doc__ = """ps_rotation_report of ps_rotation_averaging (popsift_b200_global.h); termination is a name of
RA_TERMINATION."""
PositionReport = namedtuple("PositionReport", "initial_cost final_cost iterations cg_iterations n_obs n_points n_cams termination")
PositionReport.__doc__ = """ps_position_report of ps_global_positioning (popsift_b200_global.h); termination is a name of
GP_TERMINATION."""
GlobalPoses = namedtuple("GlobalPoses", "tracks poses registered positioned rotation_report position_report pair_error")
GlobalPoses.__doc__ = """global_poses' result: the Tracks of the pairs kept, one world-to-camera (R, t) per set, the bool
registered (rotation averaging) and positioned (global positioning) flags per set, both reports and the pairs' final
rotation errors in degrees (+inf for pairs not used)."""


def _loss_code(loss) -> int:
    if loss not in BA_LOSS:
        raise PopSiftError("loss must be one of %s" % (BA_LOSS,))
    return BA_LOSS.index(loss)


def _rotation_params(loss="cauchy", loss_scale=5.0, max_iters=100, step_tol=1e-4, cg_max_iters=100, cg_tol=1e-8,
                     min_inliers=15) -> PsRotationParams:
    return PsRotationParams(_loss_code(loss), int(max_iters), int(cg_max_iters), int(min_inliers), float(loss_scale), float(step_tol),
                            float(cg_tol))


def _position_params(loss="huber", loss_scale=0.1, max_iters=100, function_tol=1e-8, cg_max_iters=300, cg_tol=1e-8) -> PsPositionParams:
    return PsPositionParams(_loss_code(loss), int(max_iters), int(cg_max_iters), 0, float(loss_scale), float(function_tol), float(cg_tol))


def _rotation_dev(lib, device, n_sets, pairs, d_two_view, prm: PsRotationParams):
    """ps_rotation_averaging on device two-view records: (R (S, 3, 3), registered bool (S,), pair_error (P,), RotationReport)"""
    n, P = max(int(n_sets), 1), len(pairs)
    R = np.zeros((n, 9), np.float64)
    reg = np.zeros(n, np.uint8)
    err = np.zeros(max(P, 1), np.float32)
    rep = PsRotationReport()
    rc = lib.ps_rotation_averaging(device, int(n_sets), P, _c_pairs(pairs), d_two_view if P else None, C.byref(prm), R.ctypes.data,
                                   reg.ctypes.data, err.ctypes.data, C.byref(rep))
    _check(lib, rc, "ps_rotation_averaging")
    out = RotationReport(float(rep.initial_cost), float(rep.final_cost), int(rep.iterations), int(rep.cg_iterations), int(rep.n_pairs),
                         int(rep.n_registered), RA_TERMINATION[rep.termination])
    return R[:n_sets].reshape(-1, 3, 3), reg[:n_sets].astype(bool), err[:P].copy(), out


def _two_view_records(two_view, n_pairs) -> np.ndarray:
    """ps_two_view records (TWO_VIEW_DTYPE) from TwoView tuples, such records or (R, n_front) tuples, one per pair"""
    if isinstance(two_view, np.ndarray) and two_view.dtype == TWO_VIEW_DTYPE:
        rec = np.ascontiguousarray(two_view)
    else:
        rec = np.zeros(len(two_view), TWO_VIEW_DTYPE)
        for p, tv in enumerate(two_view):
            if isinstance(tv, TwoView):
                rec[p]["R"], rec[p]["t"], rec[p]["n_inliers"], rec[p]["n_front"] = tv.R, tv.t, tv.n_inliers, tv.n_front
            else:
                rec[p]["R"], rec[p]["n_front"] = np.asarray(tv[0], np.float32).reshape(3, 3), int(tv[1])
    if len(rec) != n_pairs:
        raise PopSiftError("one two-view record per pair expected")
    return rec


def rotation_averaging(n_sets, pairs, two_view, device=0, **params):
    """Robust rotation averaging over a view graph (C ABI ps_rotation_averaging in popsift_b200_global.h; an addition to the
    reference's interface): a maximum-spanning-tree start, then IRLS on the device.  `pairs` is the (l, r) list and
    `two_view` one relative pose per pair (X_r = R X_l + t) as TwoView tuples, ps_two_view records (TWO_VIEW_DTYPE) or
    (R, n_front) tuples.  params: loss ("cauchy"), loss_scale (degrees, 5.0), max_iters (100), step_tol (degrees, 1e-4),
    cg_max_iters (100), cg_tol (1e-8), min_inliers (n_front threshold, 15).  Returns (R (n_sets, 3, 3) world to camera,
    registered bool (n_sets,), pair_error degrees (P,), RotationReport)."""
    lib = load_library()
    prm = _rotation_params(**params)
    pairs = [(int(a), int(b)) for a, b in pairs]
    rec = _two_view_records(two_view, len(pairs))
    bufs = _DevBuffers(lib)
    try:
        return _rotation_dev(lib, device, n_sets, pairs, bufs.upload(rec) if len(rec) else None, prm)
    finally:
        bufs.free()


ViewGraphReport = namedtuple("ViewGraphReport", "n_triangles n_consistent_triangles n_used n_kept n_untested")
ViewGraphReport.__doc__ = """ps_view_graph_report of ps_view_graph_filter (popsift_b200_viewgraph.h)."""
ViewGraph = namedtuple("ViewGraph", "keep n_triangles n_consistent min_error report")
ViewGraph.__doc__ = """filter_view_graph's result: keep bool (P,), per pair the triangles it lies in, the consistent ones and
the smallest cycle error in degrees (+inf: none), and the ViewGraphReport."""


def _view_graph_params(max_cycle_error=3.0, min_consistent=1, min_fraction=0.0, keep_untested=False, min_inliers=15) -> PsViewGraphParams:
    return PsViewGraphParams(int(min_inliers), int(min_consistent), 1 if keep_untested else 0, 0, float(max_cycle_error), float(min_fraction))


def _view_graph_dev(lib, device, n_sets, pairs, d_two_view, prm: PsViewGraphParams, d_kept=None) -> ViewGraph:
    """ps_view_graph_filter on device two-view records; the kept records go to d_kept when it is given"""
    P = len(pairs)
    keep = np.zeros(max(P, 1), np.uint8)
    st = np.zeros(max(P, 1), CYCLE_STATS_DTYPE)
    rep = PsViewGraphReport()
    rc = lib.ps_view_graph_filter(device, int(n_sets), P, _c_pairs(pairs), d_two_view if P else None, C.byref(prm), keep.ctypes.data,
                                  st.ctypes.data, d_kept, C.byref(rep))
    _check(lib, rc, "ps_view_graph_filter")
    r = ViewGraphReport(int(rep.n_triangles), int(rep.n_consistent_triangles), int(rep.n_used), int(rep.n_kept), int(rep.n_untested))
    return ViewGraph(keep[:P].astype(bool), st["n_triangles"][:P].copy(), st["n_consistent"][:P].copy(), st["min_error"][:P].copy(), r)


def filter_view_graph(n_sets, pairs, two_view, device=0, **params) -> ViewGraph:
    """View-graph cleaning by rotation loop consistency (C ABI ps_view_graph_filter in popsift_b200_viewgraph.h; an addition
    to the reference's interface): every triangle of the used pairs is tested, R(c->a) R(b->c) R(a->b) against the identity,
    and a pair is kept when enough of its triangles close.  `pairs` and `two_view` as for rotation_averaging (pairs must be
    distinct, in either order).  params: max_cycle_error (degrees, 3.0), min_consistent (1), min_fraction (0.0),
    keep_untested (False: a used pair in no triangle is dropped), min_inliers (n_front threshold, 15; use rotation
    averaging's).  Returns a ViewGraph."""
    lib = load_library()
    prm = _view_graph_params(**params)
    pairs = [(int(a), int(b)) for a, b in pairs]
    rec = _two_view_records(two_view, len(pairs))
    bufs = _DevBuffers(lib)
    try:
        return _view_graph_dev(lib, device, n_sets, pairs, bufs.upload(rec) if len(rec) else None, prm)
    finally:
        bufs.free()


def _positioning_dev(lib, bufs, device, n_feat, c_feat, cameras, R, registered, n_tracks, d_start, d_mem, n_members, prm):
    """ps_global_positioning on device track arrays: (poses [(R, t)], positioned bool (S,), X (T, 3), PositionReport)"""
    cam = _c_cameras(cameras)
    S = len(n_feat)
    Rs = np.ascontiguousarray(np.asarray(R, np.float64).reshape(-1, 9))
    reg = np.ascontiguousarray(np.asarray(registered).astype(np.uint8).reshape(-1))
    if len(cam) != S or len(Rs) != S or len(reg) != S:
        raise PopSiftError("one camera, one rotation and one registered flag per set expected")
    n = max(S, 1)
    out = (PsRigid * n)()
    pos = np.zeros(n, np.uint8)
    d_X = bufs.alloc(n_tracks * 24) if n_tracks else None
    rep = PsPositionReport()
    rc = lib.ps_global_positioning(device, S, (C.c_int32 * n)(*n_feat), c_feat, cam.ctypes.data, Rs.ctypes.data if S else None,
                                   reg.ctypes.data if S else None, n_tracks, d_start, d_mem, n_members, C.byref(prm), out,
                                   pos.ctypes.data, d_X, C.byref(rep))
    _check(lib, rc, "ps_global_positioning")
    X = bufs.download(d_X, (n_tracks, 3), np.float64) if n_tracks else np.zeros((0, 3))
    poses = [(np.array(out[i].R[:], np.float64).reshape(3, 3), np.array(out[i].t[:], np.float64)) for i in range(S)]
    r = PositionReport(float(rep.initial_cost), float(rep.final_cost), int(rep.iterations), int(rep.cg_iterations), int(rep.n_obs),
                       int(rep.n_points), int(rep.n_cams), GP_TERMINATION[rep.termination])
    return poses, pos[:S].astype(bool), X, r


def global_positioning(sets, tracks, cameras, rotations, registered, device=None, **params):
    """Global positioning of camera centres and track points from the tracks' viewing rays, rotations held (C ABI
    ps_global_positioning in popsift_b200_global.h; an addition to the reference's interface).  `sets` are FeaturesDev
    objects or host Features, `tracks` a Tracks over them, `cameras` one (fx, fy, cx, cy) per set, `rotations` one
    world-to-camera R per set and `registered` one bool per set (rotation_averaging's).  params: loss ("huber"),
    loss_scale (0.1), max_iters (100), function_tol (1e-8), cg_max_iters (300), cg_tol (1e-8).  Returns (poses as a list of
    (R, t), positioned bool (n_sets,), X (T, 3) points (0 for tracks that took no part), PositionReport); the positioned
    centres have an RMS distance of 1 from the root's."""
    lib = load_library()
    prm = _position_params(**params)
    bufs = _DevBuffers(lib)
    try:
        ptrs, n_feat = [], []
        for s in sets:
            if isinstance(s, FeaturesDev):
                ptrs.append(s.getFeatures()); n_feat.append(s.getFeatureCount())
            else:
                f = np.ascontiguousarray(s.feat if isinstance(s, Features) else s, FEATURE_DTYPE)
                ptrs.append(bufs.upload(f)); n_feat.append(len(f))
        if device is None:
            device = next((max(0, lib.ps_pointer_device(p)) for p, k in zip(ptrs, n_feat) if k > 0), 0)
        off = np.concatenate([[0], np.cumsum(n_feat, dtype=np.int64)])
        st = np.ascontiguousarray(tracks.start, np.int32)
        mem = (off[np.asarray(tracks.set, np.int64)] + np.asarray(tracks.feature, np.int64)).astype(np.int32)
        c_feat = (C.c_void_p * max(len(sets), 1))(*ptrs)
        return _positioning_dev(lib, bufs, device, n_feat, c_feat, cameras, rotations, registered, len(st) - 1, bufs.upload(st),
                                bufs.upload(mem) if len(mem) else None, len(mem), prm)
    finally:
        bufs.free()


def global_poses(sets, pairs, cameras, matches=None, flags=0, u8=False, device=None, min_length=2, max_pair_error=5.0, pose=None,
                 rotation=None, position=None, view_graph=None, two_view=None) -> GlobalPoses:
    """Poses for every image from images and intrinsics alone, without leaving the device: relative_poses' chain
    (matching unless `matches` is given, correspondences, ps_relative_pose_batch with the parameters in the dict `pose`),
    ps_rotation_averaging on its records (dict `rotation`: rotation_averaging's params), ps_tracks_from_matches on the
    pose masks of the pairs that were used, are registered and have a final rotation error <= max_pair_error degrees
    (the other pairs contribute no correspondence), then ps_global_positioning on those tracks (dict `position`:
    global_positioning's params).  A dict `view_graph` (filter_view_graph's params but min_inliers, which is the
    rotation's) cleans the view graph first: ps_view_graph_filter on the relative poses, rotation averaging on the kept
    pairs only, and the dropped pairs get pair_error +inf (so they contribute no correspondence).  A dict `two_view`
    (two_view_config_correspondences' config) classifies the pairs first: ps_verify_batch's homography and fundamental
    matrix with the pose parameters, then ps_two_view_config_batch, whose records and masks replace ps_relative_pose_batch's
    for everything after it (planar pairs posed from the homography, panoramic pairs by their rotation alone with the
    rotation-test rows as tracks, the other non-general pairs dropped).  `sets` are FeaturesDev
    objects and `cameras` one (fx, fy, cx, cy) per set.  The result feeds triangulate() and then bundle_adjust()."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    pprm = _pose_params(**(pose or {}))
    rprm = _rotation_params(**(rotation or {}))
    gprm = _position_params(**(position or {}))
    if view_graph is not None:
        if "min_inliers" in view_graph:
            raise PopSiftError("view_graph takes min_inliers from the rotation parameters")
        vgprm = _view_graph_params(min_inliers=rprm.min_inliers, **view_graph)
    if two_view is not None:
        cprm = _two_view_config_params(pprm.threshold, **two_view)
    cam = np.asarray(cameras, np.float32).reshape(-1, 4)
    if len(cam) != len(sets):
        raise PopSiftError("one camera per set expected")
    bufs = _DevBuffers(lib)
    try:
        _, device, rows, d_match, d_corr, d_src, start, n_corr = _matched_rows(lib, bufs, sets, pairs, matches, flags, u8, device,
                                                                              u8 and matches is None)
        pcams = _c_cameras([cam[i] for lr in pairs for i in lr])
        if two_view is None:
            d_out, d_mask = _pose_dev(lib, bufs, device, d_corr, start, n_corr, pcams, pprm)[:2]
        else:
            d_out, d_mask = _two_view_config_dev(lib, bufs, device, d_corr, start, n_corr, pcams, pprm, cprm)[:2]
        if view_graph is None:
            R, reg, perr, rrep = _rotation_dev(lib, device, len(sets), pairs, d_out, rprm)
        else:
            # rotation averaging on the kept pairs' records, its errors scattered back to the full pair list
            d_kept = bufs.alloc(max(len(pairs), 1) * TWO_VIEW_DTYPE.itemsize)
            vg = _view_graph_dev(lib, device, len(sets), pairs, d_out, vgprm, d_kept)
            kept = np.flatnonzero(vg.keep)
            R, reg, perr_k, rrep = _rotation_dev(lib, device, len(sets), [pairs[p] for p in kept], d_kept, rprm)
            perr = np.full(len(pairs), np.inf, np.float32)
            perr[kept] = perr_k
        keep = np.ascontiguousarray(np.where(perr <= float(max_pair_error), n_corr, 0), np.int32)
        n = max(len(sets), 1)
        n_feat = [s.getFeatureCount() for s in sets]
        c_nf = (C.c_int32 * n)(*n_feat)
        c_rev = (C.c_void_p * n)(*[s.getReverseMap() for s in sets])
        c_nd = (C.c_int32 * n)(*[s.getDescriptorCount() for s in sets])
        tr, d_start, d_mem = _tracks_run(lib, bufs, n_feat, min_length, lambda of, st, mem, cnt: lib.ps_tracks_from_matches(
            device, len(sets), c_nf, c_rev, c_nd, len(pairs), _c_pairs(pairs), d_match, d_src, keep.ctypes.data, d_mask,
            int(min_length), of, st, mem, C.byref(cnt)))
        c_feat = (C.c_void_p * n)(*[s.getFeatures() for s in sets])
        poses, positioned, _, grep = _positioning_dev(lib, bufs, device, n_feat, c_feat, cam, R, reg, len(tr.start) - 1, d_start,
                                                      d_mem, len(tr.set), gprm)
    finally:
        bufs.free()
    return GlobalPoses(tr, poses, reg, positioned, rrep, grep, perr)


DepthMaps = namedtuple("DepthMaps", "depth cost n_src report n_consistent points filter_report")
DepthMaps.__doc__ = """depth_maps' result, one entry per reference: depth (h, w) float32 (0 where there is none), cost (h, w) float32 (+inf
without a winner), n_src (h, w) uint8 and the report {"candidates", "depths"}.  With a filter: n_consistent (h, w) uint8
per reference, points (a DENSE_POINT_DTYPE array in (ref, y, x) order) and filter_report {"tested", "points"}; None
otherwise."""


def _depth_params(n_depths=128, radius=3, top_k=3, min_sources=1, max_cost=0.5, min_var=1.0) -> PsDepthParams:
    return PsDepthParams(int(n_depths), int(radius), int(top_k), int(min_sources), float(max_cost), float(min_var))


def _depth_filter_params(max_reproj_error=1.0, max_depth_diff=0.01, min_consistent=2) -> PsDepthFilterParams:
    return PsDepthFilterParams(float(max_reproj_error), float(max_depth_diff), int(min_consistent), 0)


def _c_images(lib, bufs, images, dtype=np.uint8):
    """ps_image array of 2-D images of element type dtype (pitch in bytes): numpy arrays are uploaded, objects with
    __cuda_array_interface__ (torch CUDA tensors, for example) are used in place.  Returns (the array, the device of the
    first device image or None)."""
    dtype = np.dtype(dtype)
    out = (PsImage * max(len(images), 1))()
    device = None
    for i, im in enumerate(images):
        cai = getattr(im, "__cuda_array_interface__", None)
        if cai is not None:
            if len(cai["shape"]) != 2 or np.dtype(cai["typestr"]) != dtype:
                raise PopSiftError("image %d: a 2-D %s device array expected" % (i, dtype))
            h, w = (int(v) for v in cai["shape"])
            st = cai.get("strides")
            if st is not None and int(st[1]) != dtype.itemsize:
                raise PopSiftError("image %d: rows must be contiguous" % i)
            ptr = int(cai["data"][0])
            out[i] = PsImage(ptr, int(st[0]) if st is not None else w * dtype.itemsize, w, h)
            if device is None:
                device = max(0, lib.ps_pointer_device(ptr))
        else:
            a = np.ascontiguousarray(im, dtype)
            if a.ndim != 2:
                raise PopSiftError("image %d: a 2-D %s array expected" % (i, dtype))
            out[i] = PsImage(bufs.upload(a), a.shape[1] * dtype.itemsize, a.shape[1], a.shape[0])
    return out, device


def _depth_csr(refs, sources):
    refs = [int(r) for r in refs]
    if len(sources) != len(refs):
        raise PopSiftError("one source list per reference expected")
    start = np.concatenate([[0], np.cumsum([len(s) for s in sources])]).astype(np.int32)
    flat = np.asarray([int(v) for s in sources for v in s] or [0], np.int32)
    return np.asarray(refs or [0], np.int32), start, flat


def depth_maps(images, cameras, poses, refs, sources, ranges, device=None, filter=None, **params) -> DepthMaps:
    """Dense depth maps by plane sweep (C ABI ps_depth_maps in popsift_b200_depth.h; an addition to the reference's
    interface): for each reference set refs[j], a fronto-parallel sweep of params["n_depths"] planes in inverse depth over
    ranges[j] = (d_min, d_max), a zero-mean NCC window of radius params["radius"] against the sets sources[j], the mean of
    the top_k best source costs per plane, the winning plane refined by a parabola.  `images` holds one 2-D uint8 image
    per set: numpy arrays (uploaded) or objects with __cuda_array_interface__ such as torch CUDA tensors (used in place,
    any row pitch); `cameras` one (fx, fy, cx, cy) and `poses` one world-to-camera (R, t) per set.  params: n_depths (128),
    radius (3), top_k (3), min_sources (1), max_cost (0.5), min_var (1.0 grey levels^2).  A dict `filter`
    (max_reproj_error 1.0 px, max_depth_diff 0.01, min_consistent 2) also runs ps_depth_filter on the device maps:
    the geometric consistency between the references and the consistent pixels as world points."""
    lib = load_library()
    prm = _depth_params(**params)
    fprm = _depth_filter_params(**filter) if filter is not None else None
    n_sets = len(images)
    cam = _c_cameras(cameras)
    if len(cam) != n_sets or len(poses) != n_sets:
        raise PopSiftError("one camera and one pose per image expected")
    c_refs, start, flat = _depth_csr(refs, sources)
    nr = len(refs)
    rng = np.ascontiguousarray(np.asarray(ranges, np.float32).reshape(-1, 2) if nr else np.zeros((1, 2)), np.float32)
    bufs = _DevBuffers(lib)
    try:
        c_img, dev0 = _c_images(lib, bufs, images)
        if device is None:
            device = dev0 if dev0 is not None else 0
        shapes = [(int(c_img[r].height), int(c_img[r].width)) if 0 <= r < n_sets else (0, 0) for r in c_refs[:nr]]
        d_depth = [bufs.alloc(h * w * 4) for h, w in shapes]
        d_cost = [bufs.alloc(h * w * 4) for h, w in shapes]
        d_nsrc = [bufs.alloc(h * w) for h, w in shapes]
        n = max(nr, 1)
        c_depth, c_cost, c_nsrc = (C.c_void_p * n)(*d_depth), (C.c_void_p * n)(*d_cost), (C.c_void_p * n)(*d_nsrc)
        rig = _c_rigids(poses)
        rep = PsDepthReport()
        _check(lib, lib.ps_depth_maps(device, n_sets, c_img, cam.ctypes.data, rig, nr, c_refs.ctypes.data, rng.ctypes.data,
                                      start.ctypes.data, flat.ctypes.data, C.byref(prm), c_depth, c_cost, c_nsrc, C.byref(rep)),
               "ps_depth_maps")
        depth = [bufs.download(d, s, np.float32) for d, s in zip(d_depth, shapes)]
        cost = [bufs.download(d, s, np.float32) for d, s in zip(d_cost, shapes)]
        nsrc = [bufs.download(d, s, np.uint8) for d, s in zip(d_nsrc, shapes)]
        report = {"candidates": int(rep.n_candidates), "depths": int(rep.n_depths)}
        ncons = points = frep = None
        if fprm is not None:
            d_ncons = [bufs.alloc(h * w) for h, w in shapes]
            cap = sum(h * w for h, w in shapes)
            d_pts = bufs.alloc(cap * DENSE_POINT_DTYPE.itemsize)
            fr = PsDepthFilterReport()
            _check(lib, lib.ps_depth_filter(device, n_sets, c_img, cam.ctypes.data, rig, nr, c_refs.ctypes.data, start.ctypes.data,
                                            flat.ctypes.data, c_depth, C.byref(fprm), (C.c_void_p * n)(*d_ncons), d_pts, C.byref(fr)),
                   "ps_depth_filter")
            ncons = [bufs.download(d, s, np.uint8) for d, s in zip(d_ncons, shapes)]
            points = bufs.download(d_pts, int(fr.n_points), DENSE_POINT_DTYPE)
            frep = {"tested": int(fr.n_tested), "points": int(fr.n_points)}
    finally:
        bufs.free()
    return DepthMaps(depth, cost, nsrc, report, ncons, points, frep)


Mesh = namedtuple("Mesh", "vertices triangles report")
Mesh.__doc__ = """TsdfVolume.mesh's result: vertices (a MESH_VERTEX_DTYPE array in edge-key order), triangles (m, 3) int32 with
normals (v1 - v0) x (v2 - v0) towards the cameras, and the report {"cells", "vertices", "triangles"}."""


class TsdfVolume:
    """A dense truncated signed distance volume on the device (C ABI ps_volume in popsift_b200_mesh.h; an addition to the
    reference's interface): shape = (nx, ny, nz) grid points from `origin` at spacing `voxel`, grid point (i, j, k) at
    index i + nx (j + ny k).  Owns its three float32 arrays (tsdf, weight, grey) and clears them at construction."""

    def __init__(self, origin, voxel, shape, device=0):
        self._lib = load_library()
        self.origin = tuple(float(v) for v in origin)
        self.voxel = float(voxel)
        self.shape = tuple(int(v) for v in shape)
        self.device = int(device)
        if len(self.origin) != 3 or len(self.shape) != 3:
            raise PopSiftError("origin and shape have three components")
        n = self.shape[0] * self.shape[1] * self.shape[2]
        self._ptrs = [self._lib.ps_dev_alloc(max(n, 1) * 4) for _ in range(3)]
        if not all(self._ptrs):
            self.free()
            raise PopSiftError("ps_dev_alloc failed")
        self.clear()

    def c_volume(self) -> PsVolume:
        if not self._ptrs:
            raise PopSiftError("the volume has been freed")
        return PsVolume((C.c_double * 3)(*self.origin), self.voxel, *self.shape, 0, *self._ptrs)

    def clear(self):
        """every grid point's tsdf, weight and grey to 0 (ps_volume_clear)"""
        _check(self._lib, self._lib.ps_volume_clear(self.device, C.byref(self.c_volume())), "ps_volume_clear")

    def integrate(self, images, cameras, poses, depths, masks=None, trunc=None, min_consistent=0) -> dict:
        """Folds depth maps into the volume (ps_tsdf_integrate): view v is images[v] (2-D uint8), cameras[v] (fx, fy, cx,
        cy), poses[v] (world-to-camera R, t) and depths[v], a float32 map of the image's size (depth_maps' output);
        masks[v] is the n_consistent map of depth_maps' filter, used when min_consistent > 0.  Images, depths and masks
        may be numpy arrays (uploaded) or __cuda_array_interface__ arrays such as torch CUDA tensors (used in place;
        depths and masks with contiguous rows).  trunc is the truncation distance in world units (default 3 voxels).
        Returns the report {"updates", "touched"}."""
        lib = self._lib
        n = len(images)
        if len(cameras) != n or len(poses) != n or len(depths) != n or (masks is not None and len(masks) != n):
            raise PopSiftError("one camera, pose, depth map (and mask) per image expected")
        if min_consistent > 0 and masks is None:
            raise PopSiftError("min_consistent > 0 needs masks")
        prm = PsTsdfParams(float(3.0 * self.voxel if trunc is None else trunc), int(min_consistent))
        cam = _c_cameras(cameras)
        bufs = _DevBuffers(lib)
        try:
            c_img, _ = _c_images(lib, bufs, images)
            c_dep, _ = _c_images(lib, bufs, depths, np.float32)
            c_msk = _c_images(lib, bufs, masks)[0] if masks is not None else None
            for v in range(n):
                for arr, size in ((c_dep, 4), (c_msk, 1)):
                    if arr is not None and (arr[v].width, arr[v].height, arr[v].pitch) != (c_img[v].width, c_img[v].height,
                                                                                            c_img[v].width * size):
                        raise PopSiftError("view %d: a depth map or mask must have its image's size and contiguous rows" % v)
            k = max(n, 1)
            d_dep = (C.c_void_p * k)(*[c_dep[v].data for v in range(n)])
            d_msk = (C.c_void_p * k)(*[c_msk[v].data for v in range(n)]) if c_msk is not None else None
            rep = PsTsdfReport()
            _check(lib, lib.ps_tsdf_integrate(self.device, n, c_img, cam.ctypes.data, _c_rigids(poses), d_dep, d_msk, C.byref(prm),
                                              C.byref(self.c_volume()), C.byref(rep)), "ps_tsdf_integrate")
        finally:
            bufs.free()
        return {"updates": int(rep.n_updates), "touched": int(rep.n_voxels_touched)}

    def mesh(self, min_weight=1.0) -> Mesh:
        """The surface T = 0 by marching tetrahedra over the cells whose 8 corners have weight >= min_weight
        (ps_tsdf_mesh): a count call, then the call that fills outputs of that size."""
        lib = self._lib
        prm = PsMeshParams(float(min_weight), 0)
        vol = self.c_volume()
        rep = PsMeshReport()
        rc = lib.ps_tsdf_mesh(self.device, C.byref(vol), C.byref(prm), 0, 0, None, None, C.byref(rep))
        if rc not in (0, -5):
            _check(lib, rc, "ps_tsdf_mesh")
        report = {"cells": int(rep.n_cells), "vertices": int(rep.n_vertices), "triangles": int(rep.n_triangles)}
        if rc == 0:
            return Mesh(np.zeros(0, MESH_VERTEX_DTYPE), np.zeros((0, 3), np.int32), report)
        if rep.n_vertices < 0:
            raise PopSiftError("ps_tsdf_mesh: the mesh has 2^31 vertices or more")
        bufs = _DevBuffers(lib)
        try:
            nv, nt = int(rep.n_vertices), int(rep.n_triangles)
            d_v, d_t = bufs.alloc(nv * MESH_VERTEX_DTYPE.itemsize), bufs.alloc(nt * 12)
            _check(lib, lib.ps_tsdf_mesh(self.device, C.byref(vol), C.byref(prm), nv, nt, d_v, d_t, C.byref(rep)), "ps_tsdf_mesh")
            return Mesh(bufs.download(d_v, nv, MESH_VERTEX_DTYPE), bufs.download(d_t, (nt, 3), np.int32), report)
        finally:
            bufs.free()

    def download(self):
        """(tsdf, weight, grey) as float32 numpy arrays of shape (nz, ny, nx)"""
        nx, ny, nz = self.shape
        bufs = _DevBuffers(self._lib)
        self.c_volume()
        return tuple(bufs.download(p, (nz, ny, nx), np.float32) for p in self._ptrs)

    def free(self):
        """releases the device arrays now (otherwise when the object is collected)"""
        lib = getattr(self, "_lib", None)
        for p in getattr(self, "_ptrs", None) or []:
            if p and lib is not None:
                lib.ps_dev_free(p)
        self._ptrs = []

    def __del__(self):
        self.free()


Rendered = namedtuple("Rendered", "depth triangle report")
Rendered.__doc__ = """render_mesh's result: per view the camera-frame depth (float32 (h, w), 0 where no triangle covers the pixel)
and the nearest triangle (int32 (h, w), -1 where none), and the report {"drawn", "big", "covered"}."""

TexturedMesh = namedtuple("TexturedMesh", "atlas view uv report")
TexturedMesh.__doc__ = """texture_mesh's result: the uint8 atlas (H, W), the view each triangle was textured from (int32, -1 for
the vertex-grey fallback), the corners' texture coordinates uv (m, 3, 2) in atlas texel units (atlas_uv) and the report
{"viewed", "fallback"}."""


def _mesh_arrays(lib, bufs, mesh):
    """device pointers and counts of a Mesh's vertices and triangles: numpy arrays are uploaded, __cuda_array_interface__
    arrays (a float32 (n, 4) vertex array and an int32 (m, 3) triangle array, contiguous) are used in place"""
    out = []
    for a, dtype, cols in ((mesh.vertices, np.float32, 4), (mesh.triangles, np.int32, 3)):
        cai = getattr(a, "__cuda_array_interface__", None)
        if cai is not None:
            shape = tuple(int(v) for v in cai["shape"])
            if len(shape) != 2 or shape[1] != cols or np.dtype(cai["typestr"]) != np.dtype(dtype) or cai.get("strides") not in (None, (cols * 4, 4)):
                raise PopSiftError("a contiguous %s (n, %d) device array expected" % (np.dtype(dtype), cols))
            out += [int(cai["data"][0]), shape[0]]
        else:
            h = np.ascontiguousarray(a)
            if h.dtype == MESH_VERTEX_DTYPE:
                h = h.view(np.float32).reshape(-1, 4)
            h = np.ascontiguousarray(h, dtype).reshape(-1, cols)
            out += [bufs.upload(h), h.shape[0]]
    return out


def _render_dev(lib, device, mesh_dev, cameras, poses, sizes, z_near, d_depth, d_tri) -> dict:
    d_v, nv, d_t, nt = mesh_dev
    n = len(sizes)
    cam = _c_cameras(cameras)
    if len(cam) != n or len(poses) != n:
        raise PopSiftError("one camera, one pose and one size per view expected")
    sz = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2) if n else np.zeros((1, 2), np.int32))
    k = max(n, 1)
    rep = PsRenderReport()
    _check(lib, lib.ps_mesh_render(device, n, sz.ctypes.data, cam.ctypes.data, _c_rigids(poses), d_v, nv, d_t, nt,
                                   C.byref(PsRenderParams(float(z_near), 0)), (C.c_void_p * k)(*d_depth), (C.c_void_p * k)(*d_tri),
                                   C.byref(rep)), "ps_mesh_render")
    return {"drawn": int(rep.n_drawn), "big": int(rep.n_big), "covered": int(rep.n_covered)}


def render_mesh(mesh, cameras, poses, sizes, z_near=1e-3, device=0) -> Rendered:
    """Renders a triangle mesh into posed views with a z-buffer (C ABI ps_mesh_render in popsift_b200_render.h; an addition
    to the reference's interface).  `mesh` is TsdfVolume.mesh's Mesh (or any object with vertices, a MESH_VERTEX_DTYPE or
    float32 (n, 4) array, and triangles, int32 (m, 3)); numpy arrays are uploaded, torch CUDA tensors used in place.
    View v is cameras[v] (fx, fy, cx, cy), poses[v] (world-to-camera R, t) and sizes[v] = (width, height).  Triangles with a
    vertex closer than z_near are not drawn (no near-plane clipping).  The maps are in depth_maps' layout and convention."""
    lib = load_library()
    bufs = _DevBuffers(lib)
    try:
        mesh_dev = _mesh_arrays(lib, bufs, mesh)
        shapes = [(int(h), int(w)) for w, h in sizes]
        d_depth = [bufs.alloc(h * w * 4) for h, w in shapes]
        d_tri = [bufs.alloc(h * w * 4) for h, w in shapes]
        report = _render_dev(lib, device, mesh_dev, cameras, poses, sizes, z_near, d_depth, d_tri)
        depth = [bufs.download(d, s, np.float32) for d, s in zip(d_depth, shapes)]
        tri = [bufs.download(d, s, np.int32) for d, s in zip(d_tri, shapes)]
    finally:
        bufs.free()
    return Rendered(depth, tri, report)


def atlas_cells_per_row(n_triangles, cell) -> int:
    """texture_mesh's default: the atlas close to square, at most 65535 texels wide"""
    return max(1, min(int(np.ceil(np.sqrt(max(int(n_triangles), 1)))), 65535 // int(cell)))


def atlas_uv(n_triangles, cell, cells_per_row):
    """the corners' positions (m, 3, 2) in atlas texel units (x right, y down) and the atlas size (W, H): triangle m owns
    cell (m mod cells_per_row, m div cells_per_row), its corners at (b, b), (cell - b, b), (b, cell - b) of the cell, b = 1"""
    m = np.arange(int(n_triangles))
    ox, oy = (m % cells_per_row) * cell, (m // cells_per_row) * cell
    corner = np.array([[1, 1], [cell - 1, 1], [1, cell - 1]], np.float64)
    uv = np.stack([ox, oy], 1)[:, None, :].astype(np.float64) + corner[None]
    W, H = int(cells_per_row * cell), int(-(-int(n_triangles) // cells_per_row) * cell)
    return uv, W, H


def texture_mesh(mesh, images, cameras, poses, cell=8, cells_per_row=None, depth_tol=0.01, min_cos=0.1, z_near=1e-3,
                 device=None) -> TexturedMesh:
    """A texture atlas of a mesh from posed grey images (C ABI ps_mesh_render, then ps_mesh_texture on the device maps, no
    host copy between them; popsift_b200_render.h).  Each triangle takes the view that sees it (facing it by at least
    min_cos, its corners and centroid not occluded beyond depth_tol relative depth) with the largest projected area, and
    gets a cell x cell cell of the atlas sampled bilinearly from that image; a triangle no view sees falls back to its
    vertices' grey.  `images` are 2-D uint8 numpy arrays (uploaded) or torch CUDA tensors (used in place, any row pitch),
    with cameras and poses as render_mesh; `mesh` as render_mesh.  cells_per_row defaults to atlas_cells_per_row."""
    lib = load_library()
    n_views = len(images)
    bufs = _DevBuffers(lib)
    try:
        c_img, dev0 = _c_images(lib, bufs, images)
        if device is None:
            device = dev0 if dev0 is not None else 0
        mesh_dev = _mesh_arrays(lib, bufs, mesh)
        nt = mesh_dev[3]
        cpr = atlas_cells_per_row(nt, cell) if cells_per_row is None else int(cells_per_row)
        uv, W, H = atlas_uv(nt, int(cell), max(cpr, 1))
        sizes = [(int(c_img[v].width), int(c_img[v].height)) for v in range(n_views)]
        d_depth = [bufs.alloc(w * h * 4) for w, h in sizes]
        d_tri = [bufs.alloc(w * h * 4) for w, h in sizes]
        _render_dev(lib, device, mesh_dev, cameras, poses, sizes, z_near, d_depth, d_tri)
        d_atlas, d_view = bufs.alloc(W * H), bufs.alloc(nt * 4)
        prm = PsTextureParams(int(cell), cpr, float(depth_tol), float(min_cos), float(z_near), 0)
        rep = PsTextureReport()
        k = max(n_views, 1)
        d_v, nv, d_t, _ = mesh_dev
        cam = _c_cameras(cameras)
        _check(lib, lib.ps_mesh_texture(device, n_views, c_img, cam.ctypes.data, _c_rigids(poses), (C.c_void_p * k)(*d_depth),
                                        d_v, nv, d_t, nt, C.byref(prm), d_atlas, d_view, C.byref(rep)), "ps_mesh_texture")
        atlas = bufs.download(d_atlas, (H, W), np.uint8)
        view = bufs.download(d_view, nt, np.int32)
    finally:
        bufs.free()
    return TexturedMesh(atlas, view, uv, {"viewed": int(rep.n_viewed), "fallback": int(rep.n_fallback)})


def _png_grey(path, img):
    """an 8-bit grey PNG (colour type 0, no interlace) with the standard library only"""
    import struct
    import zlib
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    raw = np.concatenate([np.zeros((h, 1), np.uint8), img], 1).tobytes()   # filter type 0 on every row
    with open(path, "wb") as f:
        f.write(b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 0, 0, 0, 0)) +
                chunk(b"IDAT", zlib.compress(raw, 6)) + chunk(b"IEND", b""))


def write_obj(path, mesh, textured=None):
    """Writes `mesh` as a Wavefront OBJ.  With `textured` (texture_mesh's result for this mesh) it also writes, next to it,
    an MTL and an 8-bit grey PNG of the atlas, and every face corner gets its texture coordinate (vt, v flipped to OBJ's
    bottom-left origin).  Returns the paths written."""
    base = os.path.splitext(path)[0]
    V = np.asarray(mesh.vertices)
    X = V["X"] if V.dtype == MESH_VERTEX_DTYPE else np.asarray(V, np.float32).reshape(-1, 4)[:, :3]
    T = np.asarray(mesh.triangles, np.int64).reshape(-1, 3)
    lines = []
    written = [path]
    if textured is not None:
        H, W = textured.atlas.shape
        if len(textured.uv) != len(T):
            raise PopSiftError("the texture is not this mesh's")
        name = os.path.basename(base)
        lines.append("mtllib %s.mtl" % name)
        with open(base + ".mtl", "w") as f:
            f.write("newmtl atlas\nKa 1 1 1\nKd 1 1 1\nKs 0 0 0\nillum 1\nmap_Kd %s.png\n" % name)
        _png_grey(base + ".png", textured.atlas)
        written += [base + ".mtl", base + ".png"]
    lines += ["v %.9g %.9g %.9g" % tuple(x) for x in X.astype(np.float64)]
    if textured is not None:
        uv = textured.uv.reshape(-1, 2)
        lines += ["vt %.9g %.9g" % (u / W, 1.0 - v / H) for u, v in uv]
        lines.append("usemtl atlas")
        lines += ["f %d/%d %d/%d %d/%d" % (a + 1, 3 * m + 1, b + 1, 3 * m + 2, c + 1, 3 * m + 3) for m, (a, b, c) in enumerate(T)]
    else:
        lines += ["f %d %d %d" % (a + 1, b + 1, c + 1) for a, b, c in T]
    with open(path, "w") as f:
        f.write("\n".join(lines) + "\n")
    return written


def _track_observations(tracks, points, poses):
    """(track, set, camera-frame depth) of the OK tracks' members with mask 1"""
    ok = np.asarray(points.status) == 0
    start = np.asarray(tracks.start, np.int64)
    tid = np.repeat(np.arange(len(start) - 1), np.diff(start))
    sel = ok[tid] & (np.asarray(points.mask) == 1)
    t, s = tid[sel], np.asarray(tracks.set, np.int64)[sel]
    X = np.asarray(points.X, np.float64)[t]
    R = np.stack([np.asarray(p[0], np.float64).reshape(3, 3) for p in poses]) if len(poses) else np.zeros((0, 3, 3))
    tv = np.stack([np.asarray(p[1], np.float64).reshape(3) for p in poses]) if len(poses) else np.zeros((0, 3))
    z = np.einsum("nj,nj->n", R[s, 2], X) + tv[s, 2]
    return t, s, z


def depth_ranges(tracks, points, poses, n_sets, lo=1.0, hi=99.0, margin=0.25) -> np.ndarray:
    """Per set, the depth range for depth_maps from a sparse reconstruction: the percentiles lo and hi (numpy's linear
    rule) of the camera-frame depths of the OK tracks' members with mask 1 in that set, divided and multiplied by
    1 + margin.  `tracks`, `points` and `poses` are what bundle_adjust / triangulate give.  A set without such depths gets
    (0, 0), which depth_maps refuses as a reference.  Returns (n_sets, 2) float64."""
    _, s, z = _track_observations(tracks, points, poses)
    out = np.zeros((int(n_sets), 2), np.float64)
    for i in range(int(n_sets)):
        zi = z[s == i]
        if len(zi):
            out[i] = (np.percentile(zi, lo) / (1.0 + margin), np.percentile(zi, hi) * (1.0 + margin))
    return out


def select_sources(tracks, points, poses, n_sources=5, min_angle=1.0) -> list:
    """Per set, the source sets for depth_maps, as COLMAP chooses them: the other sets ranked by the number of OK tracks
    both see (members with mask 1) whose viewing rays from the two camera centres meet at the track's point at an angle of
    at least min_angle degrees; ties to the lower set id, only counts > 0, at most n_sources."""
    t, s, _ = _track_observations(tracks, points, poses)
    n_sets = len(poses)
    Cs = np.stack([-np.asarray(p[0], np.float64).reshape(3, 3).T @ np.asarray(p[1], np.float64).reshape(3) for p in poses])
    X = np.asarray(points.X, np.float64)
    cos_min = np.cos(np.radians(float(min_angle)))
    count = np.zeros((n_sets, n_sets), np.int64)
    order = np.argsort(t, kind="stable")
    t, s = t[order], s[order]
    bounds = np.flatnonzero(np.r_[True, t[1:] != t[:-1], True])
    for a, b in zip(bounds[:-1], bounds[1:]):
        ss = s[a:b]
        if len(ss) < 2:
            continue
        u = Cs[ss] - X[t[a]]
        u /= np.linalg.norm(u, axis=1, keepdims=True)
        ok = (u @ u.T) <= cos_min
        np.fill_diagonal(ok, False)
        count[np.ix_(ss, ss)] += ok
    out = []
    for i in range(n_sets):
        c = count[i].copy()
        c[i] = 0
        rank = sorted((j for j in range(n_sets) if c[j] > 0), key=lambda j: (-c[j], j))
        out.append(rank[:int(n_sources)])
    return out


def _match_guided_dev(lib, bufs, sets, descs, pairs, d_models, model, threshold, flags, u8) -> int:
    """ps_match_guided_batch / ps_match_u8_guided_batch on FeaturesDev sets, their descriptors as _desc_sets gave them
    (`descs`, 8-bit with u8=True) and device-resident models: the device rows"""
    for s in sets:
        if not isinstance(s, FeaturesDev):
            raise PopSiftError("guided matching needs FeaturesDev sets (Config.MatchingMode)")
    c_sets, c_n, counts, device = descs
    d_out = bufs.alloc(sum(_pair_rows(counts, pairs)) * 12)
    name = "ps_match_u8_guided_batch" if u8 else "ps_match_guided_batch"
    n = max(len(sets), 1)
    c_feat = (C.c_void_p * n)(*[s.getFeatures() for s in sets])
    c_rev = (C.c_void_p * n)(*[s.getReverseMap() for s in sets])
    rc = getattr(lib, name)(device, len(sets), c_sets, c_feat, c_rev, c_n, len(pairs), _c_pairs(pairs), d_models, int(model),
                            float(threshold), d_out, flags)
    _check(lib, rc, name)
    return d_out


def match_pairs_guided(sets, pairs, models, model="homography", threshold=4.0, flags=0, u8=False, device=None) -> list:
    """Guided matching (C ABI ps_match_guided_batch / ps_match_u8_guided_batch in popsift_b200_guided.h; an addition to the
    reference's interface): match_pairs (match_pairs_u8 with u8=True) where the candidates of a left descriptor are only the
    right descriptors whose keypoints pass the pair's model at `threshold` pixels.  `sets` are FeaturesDev objects
    (Config.MatchingMode), `models` the (P, 3, 3) left-to-right pixel models (e.g. from verify_pairs), `model` "homography"
    or "fundamental".  Entry p is the (n_left, 3) int32 array (best, second, accept); no eligible descriptor gives (0, 0, 0)."""
    lib = load_library()
    pairs = [(int(a), int(b)) for a, b in pairs]
    model = _model_code(model)
    m = np.ascontiguousarray(models, np.float32).reshape(-1, 9)
    if len(m) != len(pairs):
        raise PopSiftError("one model per pair expected")
    bufs = _DevBuffers(lib)
    try:
        descs = _desc_sets(lib, bufs, sets, device, u8)
        rows = _pair_rows(descs[2], pairs)
        d_out = _match_guided_dev(lib, bufs, sets, descs, pairs, bufs.upload(m), model, threshold, flags, u8)
        out = bufs.download(d_out, (sum(rows), 3), np.int32)
    finally:
        bufs.free()
    return _split_rows(out, rows)


def vlad_codebook(sets, k=64, iters=10, seed=0, flags=0, device=None) -> np.ndarray:
    """k-means codebook of the pooled descriptors of `sets` (C ABI ps_vlad_train in popsift_b200_retrieval.h; an addition
    to the reference's interface): FeaturesDev objects or host (n, 128) float32 arrays.  Returns (k, 128) float32."""
    lib = load_library()
    bufs = _DevBuffers(lib)
    try:
        c_sets, c_n, _, device = _desc_sets(lib, bufs, sets, device)
        d_c = bufs.alloc(k * 512)
        _check(lib, lib.ps_vlad_train(device, len(sets), c_sets, c_n, int(k), int(iters), int(seed) & ((1 << 64) - 1), d_c, flags),
               "ps_vlad_train")
        return bufs.download(d_c, (k, 128), np.float32)
    finally:
        bufs.free()


def vlad_encode(sets, codebook, flags=0, assign=False, device=None):
    """VLAD vectors of `sets` under `codebook` ((k, 128) float32) (C ABI ps_vlad_encode): (n_sets, 128 k) float32, rows
    intra-normalised, signed-square-rooted and L2-normalised.  assign=True also returns the (N,) int32 centroid of every
    pooled descriptor (its visual word)."""
    lib = load_library()
    cb = np.ascontiguousarray(codebook, np.float32).reshape(-1, 128)
    k = len(cb)
    bufs = _DevBuffers(lib)
    try:
        c_sets, c_n, counts, device = _desc_sets(lib, bufs, sets, device)
        N = sum(counts)
        d_v = bufs.alloc(len(sets) * k * 512)
        d_a = bufs.alloc(N * 4) if assign else None
        _check(lib, lib.ps_vlad_encode(device, len(sets), c_sets, c_n, k, bufs.upload(cb), d_v, d_a, flags), "ps_vlad_encode")
        v = bufs.download(d_v, (len(sets), k * 128), np.float32)
        return (v, bufs.download(d_a, N, np.int32)) if assign else v
    finally:
        bufs.free()


def retrieve(vectors, m, device=0):
    """Each row's m nearest rows under the inner product (C ABI ps_retrieve_pairs): `vectors` is (n, dim) float32 with dim
    a multiple of 4.  Returns (nbr (n, m) int32, score (n, m) float32), best first; empty slots hold -1 and -inf."""
    lib = load_library()
    v = np.ascontiguousarray(vectors, np.float32)
    n, dim = v.shape
    bufs = _DevBuffers(lib)
    try:
        d_n, d_s = bufs.alloc(n * m * 4), bufs.alloc(n * m * 4)
        _check(lib, lib.ps_retrieve_pairs(device, n, bufs.upload(v), dim, int(m), d_n, d_s), "ps_retrieve_pairs")
        return bufs.download(d_n, (n, m), np.int32), bufs.download(d_s, (n, m), np.float32)
    finally:
        bufs.free()


def select_pairs(nbr) -> list:
    """The unordered pairs (i, j), i < j, of the union of every row's neighbours in `nbr` (retrieve's first output),
    sorted; -1 slots are dropped.  The pair list for match_pairs / verify_pairs."""
    nbr = np.asarray(nbr)
    out = set()
    for i, row in enumerate(nbr):
        for j in row:
            j = int(j)
            if j >= 0 and j != i:
                out.add((min(i, j), max(i, j)))
    return sorted(out)


def keypoints_array(keypoints) -> np.ndarray:
    """a contiguous KEYPOINT_DTYPE array from a KEYPOINT_DTYPE array or an (n, 4) array of x, y, sigma, angle (octave and
    level -1)"""
    if isinstance(keypoints, np.ndarray) and keypoints.dtype == KEYPOINT_DTYPE:
        return np.ascontiguousarray(keypoints)
    a = np.asarray(keypoints, dtype=np.float32).reshape(-1, 4)
    out = np.zeros(len(a), KEYPOINT_DTYPE)
    out["x"], out["y"], out["sigma"], out["ori"] = a[:, 0], a[:, 1], a[:, 2], a[:, 3]
    out["octave"] = out["level"] = -1
    return out


class SiftJob:
    """SiftJob (reference src/popsift/popsift.h:44-100): get() blocks until the features are there."""

    def __init__(self, owner: "PopSift", slot: int):
        self._owner, self._slot, self._result = owner, slot, None

    def getBase(self):
        if self._result is None:
            self._result = self._owner._collect(self._slot)
        return self._result

    def get(self) -> Features:
        """host features (None under Config.MatchingMode, like the reference's dynamic_cast)"""
        r = self.getBase()
        return r if isinstance(r, Features) else None

    getHost = get

    def getDev(self) -> "FeaturesDev":
        r = self.getBase()
        return r if isinstance(r, FeaturesDev) else None


class PopSift:
    """PopSift (reference src/popsift/popsift.h:105-317) over the C ABI: one context per device,
    `slots` images in flight (the reference has one)."""

    ByteImages, FloatImages = 0, 1

    def __init__(self, config: Optional[Config] = None, mode=Config.ExtractingMode, imode=0, device: int = 0,
                 max_width: int = 0, max_height: int = 0, slots: int = 2):
        self._lib = load_library()
        self._config = config or Config()
        self._imode, self._device, self._nslots = imode, device, slots
        self._mode = mode
        self._ctx = None
        self._max = (max_width, max_height)
        self._next = 0
        self._busy = [None] * slots
        self._keep = [None] * slots      # the image each slot's DMA may still be reading (page-locked inputs)
        self._pool = _Pool()     # page-locked result buffers, recycled when the arrays that view them die
        if max_width and max_height:
            self._create(max_width, max_height)

    def _create(self, w, h):
        ctx = self._lib.ps_create(self._device, C.byref(self._config._c), w, h, self._nslots)
        if not ctx:
            raise PopSiftError(_last_error(self._lib))
        self._ctx = ctx
        self._max = (w, h)

    def _check(self, rc):
        if rc != 0:
            raise PopSiftError("popsift_b200 error %d: %s" % (rc, self._lib.ps_last_error(self._ctx).decode()))

    def enqueue(self, w: int, h: int, image) -> SiftJob:
        img = np.ascontiguousarray(image)
        want = np.uint8 if self._imode == self.ByteImages else np.float32
        if img.dtype != want:
            raise PopSiftError("Image mode error")    # reference popsift.cpp:247-253
        assert img.size == w * h
        if self._ctx is None:
            self._create(w, h)
        if w > self._max[0] or h > self._max[1]:
            raise PopSiftError("image larger than the context was created for")
        slot = self._next
        self._next = (self._next + 1) % self._nslots
        if self._busy[slot] is not None:
            self._busy[slot].getBase()   # FIFO: the slot's previous job completes first
        fn = self._lib.ps_submit_u8 if self._imode == self.ByteImages else self._lib.ps_submit_f32
        self._keep[slot] = img           # released when the slot's next image is submitted (its job has completed by then)
        self._check(fn(self._ctx, slot, img.ctypes.data, w, h))
        job = SiftJob(self, slot)
        self._busy[slot] = job
        return job

    def describe(self, w: int, h: int, image, keypoints, orientations: bool = False) -> SiftJob:
        """Orientations (orientations=True) and descriptors at the caller's keypoints instead of detected ones (C ABI
        ps_describe_u8 / ps_describe_f32).  `keypoints` is a KEYPOINT_DTYPE array, or an (n, 4) float array of x, y, sigma,
        angle (radians) in input-image units with octave = level = -1 (derived from sigma).  The job's Features hold one
        record per keypoint, in input order; a rejected keypoint has num_ori 0.  Same FIFO of slots as enqueue."""
        img = np.ascontiguousarray(image)
        want = np.uint8 if self._imode == self.ByteImages else np.float32
        if img.dtype != want:
            raise PopSiftError("Image mode error")
        assert img.size == w * h
        kps = keypoints_array(keypoints)
        if self._ctx is None:
            self._create(w, h)
        if w > self._max[0] or h > self._max[1]:
            raise PopSiftError("image larger than the context was created for")
        slot = self._next
        self._next = (self._next + 1) % self._nslots
        if self._busy[slot] is not None:
            self._busy[slot].getBase()
        fn = self._lib.ps_describe_u8 if self._imode == self.ByteImages else self._lib.ps_describe_f32
        self._keep[slot] = img
        self._check(fn(self._ctx, slot, img.ctypes.data, w, h, kps.ctypes.data, len(kps),
                       DESCRIBE_ORIENT if orientations else DESCRIBE_GIVEN))
        job = SiftJob(self, slot)
        self._busy[slot] = job
        return job

    def _collect(self, slot: int) -> Features:
        nf, nd = C.c_int32(), C.c_int32()
        self._check(self._lib.ps_counts(self._ctx, slot, C.byref(nf), C.byref(nd)))
        if self._mode == Config.MatchingMode:
            fd = FeaturesDev(self._lib, nf.value, nd.value)
            self._check(self._lib.ps_download_dev(self._ctx, slot, fd.getFeatures(), fd.getDescriptors(), fd.getReverseMap()))
            self._busy[slot] = None
            return fd
        blk = None
        for i, b in enumerate(self._pool.blocks):
            if b.n_feat >= nf.value and b.n_desc >= nd.value:
                blk = self._pool.blocks.pop(i)
                break
        if blk is None:
            blk = _PinnedBlock(self._lib, int(nf.value * 1.25) + 1024, int(nd.value * 1.25) + 1024)
        rc = self._lib.ps_download(self._ctx, slot, blk.pf, blk.pd)
        feat, desc = _leased_views(self._pool, blk, nf.value, nd.value)     # from here on the lease owns the block
        self._check(rc)
        self._busy[slot] = None
        return Features(feat, desc)

    # --- test / benchmark taps ------------------------------------------------------------
    def plane(self, slot, octave, level, dog=False) -> np.ndarray:
        n = C.c_int32()
        W = (C.c_int32 * PS_MAX_OCTAVES)()
        H = (C.c_int32 * PS_MAX_OCTAVES)()
        self._check(self._lib.ps_slot_geometry(self._ctx, slot, C.byref(n), W, H))
        out = np.zeros((H[octave], W[octave]), dtype=np.float32)
        self._check(self._lib.ps_debug_plane(self._ctx, slot, octave, level, 1 if dog else 0, out.ctypes.data))
        return out

    def slot_geometry(self, slot):
        n = C.c_int32()
        W = (C.c_int32 * PS_MAX_OCTAVES)()
        H = (C.c_int32 * PS_MAX_OCTAVES)()
        self._check(self._lib.ps_slot_geometry(self._ctx, slot, C.byref(n), W, H))
        return [(W[i], H[i]) for i in range(n.value)]

    def extrema(self, slot) -> np.ndarray:
        n = self._lib.ps_debug_extrema(self._ctx, slot, None, 0)
        out = np.zeros(max(n, 0), dtype=EXTREMUM_DTYPE)
        if n > 0:
            self._lib.ps_debug_extrema(self._ctx, slot, out.ctypes.data, n)
        return out

    def set_timing(self, on=True):
        self._check(self._lib.ps_set_timing(self._ctx, 1 if on else 0))

    def stage_ms(self, slot):
        ms = (C.c_float * 6)()
        self._check(self._lib.ps_stage_ms(self._ctx, slot, ms))
        return dict(zip(STAGES, [float(v) for v in ms]))

    def launch_count(self) -> int:
        return int(self._lib.ps_launch_count(self._ctx))

    def uninit(self):
        if self._ctx:
            self._lib.ps_destroy(self._ctx)
            self._ctx = None
        self._pool.close()        # frees the idle blocks; blocks still viewed by arrays are freed when those die

    def __del__(self):
        try:
            self.uninit()
        except Exception:
            pass
