"""ctypes binding of liblocus_b200.so + host-side mirror of the reference interface.

GicpB200 mirrors the surface of pcl::MultithreadedGeneralizedIterativeClosestPoint
that LOCUS's callers use (multithreaded_gicp/include/multithreaded_gicp/gicp.h:134-298,
PointCloudOdometry.cc:147-155,265-269, PointCloudLocalization.cc:234-245,306-336):
same method names (setInputSource, setInputTarget, align, getFinalTransformation,
hasConverged, getFitnessScore, setMaximumIterations, ...), same argument meaning, same
error behaviour (empty source -> error + state untouched; failure -> last pose kept).
VoxelGridB200 mirrors point_cloud_filter::CustomVoxelGrid::filter and the setters its
config_callback drives (custom_voxel_grid.cc:62-149).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("LOCUS_B200_LIB") or os.path.join(_HERE, "liblocus_b200.so")   # env: experiments with variant builds

LB_MEM_HOST, LB_MEM_DEVICE = 0, 1
LB_OPT_BFGS, LB_OPT_GAUSS_NEWTON = 0, 1
LB_EXEC_PERSISTENT, LB_EXEC_HOST_DRIVEN, LB_EXEC_PERSISTENT_CLUSTER, LB_EXEC_STREAM_ORDERED = 0, 1, 2, 3
LB_FLOAT32 = 7


class LocusB200Error(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("locus_b200 status %d: %s" % (status, msg))
        self.status = status


class GicpParams(C.Structure):
    _fields_ = [
        ("k_correspondences", C.c_int), ("gicp_epsilon", C.c_double), ("rotation_epsilon", C.c_double),
        ("transformation_epsilon", C.c_double), ("max_correspondence_distance", C.c_double),
        ("max_iterations", C.c_int), ("max_optimizer_iterations", C.c_int),
        ("recompute_source_covariance", C.c_int), ("recompute_target_covariance", C.c_int),
        ("optimizer", C.c_int), ("execution", C.c_int), ("euclidean_fitness_epsilon", C.c_double),
        ("ransac_iterations", C.c_int), ("num_threads", C.c_int), ("enable_timing_output", C.c_int),
        ("index_cell_size", C.c_float), ("align_points_per_cta", C.c_int),
    ]


class GicpResult(C.Structure):
    _fields_ = [
        ("final_transformation", C.c_float * 16), ("converged", C.c_int), ("iterations", C.c_int),
        ("n_correspondences", C.c_int), ("delta", C.c_double), ("n_objective_evals", C.c_int),
        ("n_inner_iterations", C.c_int), ("t_covariances_ms", C.c_float), ("t_iterations_ms", C.c_float),
        ("t_total_ms", C.c_float), ("status", C.c_int), ("transformation", C.c_float * 16),
    ]


class NdtParams(C.Structure):
    _fields_ = [
        ("resolution", C.c_float), ("step_size", C.c_double), ("outlier_ratio", C.c_double),
        ("transformation_epsilon", C.c_double), ("max_iterations", C.c_int), ("min_points_per_voxel", C.c_int),
        ("min_covar_eigvalue_mult", C.c_double), ("search_method", C.c_int),
        ("max_correspondence_distance", C.c_double), ("ransac_iterations", C.c_int), ("num_threads", C.c_int),
        ("enable_timing_output", C.c_int),
    ]


class NdtResult(C.Structure):
    _fields_ = [
        ("final_transformation", C.c_float * 16), ("converged", C.c_int), ("nr_iterations", C.c_int),
        ("n_evaluations", C.c_int), ("n_target_voxels", C.c_int), ("trans_probability", C.c_double),
        ("pose", C.c_double * 6), ("t_total_s", C.c_double),
    ]


class OdometryResult(C.Structure):
    _fields_ = [("ticket", C.c_uint64), ("status", C.c_int), ("has_pose", C.c_int), ("n_filtered", C.c_size_t),
                ("gicp", GicpResult), ("error", C.c_char * 160), ("ndt", NdtResult)]


# lb_registration: a pipeline's registration method (registration_method: gicp | ndt)
LB_REG_GICP, LB_REG_NDT = 0, 1
_REG = {"gicp": LB_REG_GICP, "ndt": LB_REG_NDT}


def _reg_method(m):
    return _REG[m] if isinstance(m, str) else int(m)


class LocusThresholds(C.Structure):
    _fields_ = [("enabled", C.c_int), ("max_translation", C.c_double), ("max_rotation", C.c_double)]


class LocusFrontEnd(C.Structure):
    _fields_ = [("normals_k", C.c_int), ("viewpoint", C.c_float * 3), ("adaptive_voxelization", C.c_int),
                ("points_to_process", C.c_int)]


class LocusIcpCovariance(C.Structure):
    _fields_ = [("enabled", C.c_int), ("max_covariance", C.c_double)]


class LocusParams(C.Structure):
    _fields_ = [("odometry", GicpParams), ("localization", GicpParams), ("odometry_thresholds", LocusThresholds),
                ("localization_thresholds", LocusThresholds), ("translation_threshold_kf", C.c_double),
                ("rotation_threshold_kf", C.c_double), ("add_keyframes", C.c_int), ("refresh_every", C.c_int),
                ("msw", C.c_int), ("window_half_size", C.c_float), ("prior_map", C.c_int), ("initial_pose", C.c_double * 16),
                ("front_end", LocusFrontEnd), ("icp_covariance", LocusIcpCovariance), ("odometry_method", C.c_int),
                ("localization_method", C.c_int), ("odometry_ndt", NdtParams), ("localization_ndt", NdtParams)]


class LocusResult(C.Structure):
    _fields_ = [("ticket", C.c_uint64), ("status", C.c_int), ("error", C.c_char * 160), ("n_filtered", C.c_size_t),
                ("has_odometry", C.c_int), ("odometry", GicpResult), ("odometry_accepted", C.c_int),
                ("has_localization", C.c_int), ("localization", GicpResult), ("correction_accepted", C.c_int),
                ("odometry_pose", C.c_double * 16), ("incremental", C.c_double * 16), ("pose", C.c_double * 16),
                ("keyframe", C.c_int), ("n_inserted", C.c_size_t), ("n_removed", C.c_size_t), ("map_size", C.c_size_t),
                ("leaf_size", C.c_float), ("has_icp_covariance", C.c_int), ("icp_covariance", C.c_double * 36),
                ("condition_number", C.c_double), ("icp_covariance_flags", C.c_int), ("odometry_ndt", NdtResult),
                ("localization_ndt", NdtResult)]


# lb_icp_covariance.flags
LB_ICPCOV_CLAMPED, LB_ICPCOV_D_NAN, LB_ICPCOV_COV_NAN = 1, 2, 4


class IcpCovariance(C.Structure):
    _fields_ = [("Ap", C.c_double * 36), ("covariance", C.c_double * 36), ("condition_number", C.c_double),
                ("flags", C.c_int), ("n_query", C.c_size_t), ("n_used", C.c_size_t)]


class VoxelInput(C.Structure):
    _fields_ = [("data", C.c_void_p), ("n_pts", C.c_size_t), ("transform", C.c_void_p)]


class FeaturesParams(C.Structure):
    _fields_ = [("n_rings", C.c_int), ("lower_deg", C.c_float), ("upper_deg", C.c_float), ("scan_period", C.c_float),
                ("curvature_region", C.c_int), ("n_feature_regions", C.c_int), ("max_corner_sharp", C.c_int),
                ("max_corner_less_sharp", C.c_int), ("max_surface_flat", C.c_int), ("curvature_threshold", C.c_float),
                ("less_flat_leaf", C.c_float)]


class FeaturesResult(C.Structure):
    _fields_ = [("n_arranged", C.c_size_t), ("n_sharp", C.c_size_t), ("n_less_sharp", C.c_size_t), ("n_flat", C.c_size_t),
                ("n_less_flat", C.c_size_t), ("n_out", C.c_size_t)]


class Field(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("offset", C.c_uint32), ("datatype", C.c_uint8), ("count", C.c_uint32)]


# every symbol include/locus_b200.h declares (tests check the library exports all of them)
SYMBOLS = [
    "lb_version", "lb_last_error_string", "lb_status_string", "lb_device_count",
    "lb_gicp_default_params", "lb_gicp_create", "lb_gicp_create_on_stream", "lb_gicp_destroy",
    "lb_gicp_set_params", "lb_gicp_get_params", "lb_gicp_set_source", "lb_gicp_set_target",
    "lb_gicp_promote_source_to_target", "lb_gicp_reserve", "lb_gicp_prepare_source", "lb_gicp_share_source", "lb_gicp_set_target_cloud",
    "lb_gicp_set_source_cloud",
    "lb_cloud_release", "lb_gicp_align", "lb_gicp_transform_source", "lb_gicp_nn_target",
    "lb_gicp_fitness", "lb_gicp_point2plane_information", "lb_gicp_icp_covariance", "lb_gicp_compute_normals", "lb_gicp_compute_normals_radius",
    "lb_gicp_estimate_normals",
    "lb_gicp_statistical_outlier_removal", "lb_gicp_radius_outlier_removal", "lb_gicp_get_covariances", "lb_gicp_cloud_size", "lb_gicp_launch_count",
    "lb_gicp_kernel_time", "lb_gicp_reset_kernel_times",
    "lb_voxel_create", "lb_voxel_create_on_stream", "lb_voxel_destroy", "lb_voxel_set_leaf_size",
    "lb_voxel_get_leaf_size", "lb_voxel_set_filter_limits", "lb_voxel_set_min_points_per_voxel",
    "lb_voxel_set_downsample_all_data", "lb_voxel_set_body_filter", "lb_voxel_filter", "lb_voxel_launch_count", "lb_voxel_kernel_time",
    "lb_voxel_kernel_time_avg", "lb_voxel_set_input_passthrough", "lb_voxel_filter_merged",
    "lb_features_default_params", "lb_voxel_extract_features",
    "lb_submap_create", "lb_submap_destroy", "lb_submap_clear", "lb_submap_insert", "lb_submap_crop_box", "lb_submap_size",
    "lb_submap_generation", "lb_submap_points", "lb_submap_insert_with_normals", "lb_submap_normals", "lb_submap_neighbors", "lb_submap_launch_count", "lb_gicp_set_target_submap",
    "lb_odometry_create", "lb_odometry_destroy", "lb_odometry_voxel", "lb_odometry_gicp", "lb_odometry_depth",
    "lb_odometry_set_gicp_params", "lb_odometry_set_cloud_sharing", "lb_odometry_set_normals", "lb_odometry_set_registration", "lb_odometry_submit", "lb_odometry_next", "lb_odometry_pending",
    "lb_odometry_launch_count", "lb_odometry_stage_times", "lb_odometry_submit_merged",
    "lb_locus_default_params", "lb_locus_create", "lb_locus_destroy", "lb_locus_voxel", "lb_locus_set_params", "lb_locus_submit",
    "lb_locus_next", "lb_locus_pending", "lb_locus_stage_times", "lb_locus_submit_merged",
    "lb_ndt_default_params", "lb_ndt_create", "lb_ndt_create_on_stream", "lb_ndt_destroy", "lb_ndt_set_params", "lb_ndt_set_source",
    "lb_ndt_set_target", "lb_ndt_align", "lb_ndt_target_voxels", "lb_ndt_derivatives", "lb_ndt_launch_count",
    "lb_ndt_set_target_submap",
]


def lib_path():
    return _SO


def build(force=False, verbose=False):
    """Compile liblocus_b200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    cmd = ["make", "-C", os.path.join(_HERE, "csrc"), "-j4"] + (["-B"] if force else [])
    out = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or out.returncode:
        print(out.stdout)
    if out.returncode:
        raise RuntimeError("building liblocus_b200.so failed")
    return _SO


_lib = None


def lib():
    """Load the CUDA library.  Fails loudly when it is missing: there is no CPU path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        raise LocusB200Error(-3, "liblocus_b200.so not built (run __graft_entry__.build()); "
                                 "locus_b200 has no CPU fallback")
    L = C.CDLL(_SO)
    vp, sz, i32, u64p = C.c_void_p, C.c_size_t, C.c_int, C.POINTER(C.c_uint64)
    L.lb_last_error_string.restype = C.c_char_p
    L.lb_status_string.restype = C.c_char_p
    L.lb_status_string.argtypes = [i32]
    L.lb_device_count.argtypes = [C.POINTER(C.c_int)]
    L.lb_gicp_default_params.argtypes = [C.POINTER(GicpParams)]
    L.lb_gicp_create.argtypes = [i32, C.POINTER(vp)]
    L.lb_gicp_create_on_stream.argtypes = [i32, vp, C.POINTER(vp)]
    L.lb_gicp_destroy.argtypes = [vp]
    L.lb_gicp_set_params.argtypes = [vp, C.POINTER(GicpParams)]
    L.lb_gicp_get_params.argtypes = [vp, C.POINTER(GicpParams)]
    L.lb_gicp_set_source.argtypes = [vp, vp, sz, sz, sz, C.c_ssize_t, i32]
    L.lb_gicp_set_target.argtypes = [vp, vp, sz, sz, sz, C.c_ssize_t, i32, u64p]
    L.lb_gicp_promote_source_to_target.argtypes = [vp]
    if hasattr(L, "lb_gicp_reserve"):
        L.lb_gicp_reserve.argtypes = [vp, sz, i32]
    if hasattr(L, "lb_gicp_prepare_source"):
        L.lb_gicp_prepare_source.argtypes = [vp]
        L.lb_gicp_share_source.argtypes = [vp, C.POINTER(vp)]
        L.lb_gicp_set_target_cloud.argtypes = [vp, vp]
        if hasattr(L, "lb_gicp_set_source_cloud"):
            L.lb_gicp_set_source_cloud.argtypes = [vp, vp]
        L.lb_cloud_release.argtypes = [vp]
    L.lb_gicp_align.argtypes = [vp, vp, C.POINTER(GicpResult)]
    L.lb_gicp_transform_source.argtypes = [vp, vp, vp, sz, sz, C.c_ssize_t, i32]
    L.lb_gicp_nn_target.argtypes = [vp, vp, sz, sz, vp, vp, i32]
    L.lb_gicp_fitness.argtypes = [vp, vp, C.c_double, C.POINTER(C.c_double)]
    L.lb_gicp_point2plane_information.argtypes = [vp, vp, sz, sz, sz, vp, sz, sz, sz, vp, vp, i32, vp, i32]
    if hasattr(L, "lb_gicp_icp_covariance"):
        L.lb_gicp_icp_covariance.argtypes = [vp, vp, vp, i32, vp, C.c_double, C.POINTER(IcpCovariance)]
    L.lb_gicp_get_covariances.argtypes = [vp, i32, vp, sz]
    if hasattr(L, "lb_gicp_compute_normals"):
        L.lb_gicp_compute_normals.argtypes = [vp, i32, i32, vp, vp, i32]
    if hasattr(L, "lb_gicp_estimate_normals"):
        L.lb_gicp_estimate_normals.argtypes = [vp, i32, i32, vp]
    if hasattr(L, "lb_gicp_compute_normals_radius"):
        L.lb_gicp_compute_normals_radius.argtypes = [vp, i32, C.c_double, vp, vp, vp, C.POINTER(sz), i32]
    if hasattr(L, "lb_gicp_statistical_outlier_removal"):
        L.lb_gicp_statistical_outlier_removal.argtypes = [vp, i32, i32, C.c_double, i32, vp, C.POINTER(sz), vp, vp, i32]
        L.lb_gicp_radius_outlier_removal.argtypes = [vp, i32, C.c_double, i32, i32, i32, vp, C.POINTER(sz), i32]
    L.lb_gicp_cloud_size.argtypes = [vp, i32, C.POINTER(sz)]
    L.lb_gicp_launch_count.argtypes = [vp, u64p]
    L.lb_gicp_kernel_time.argtypes = [vp, C.c_char_p, C.POINTER(C.c_float), u64p]
    L.lb_gicp_reset_kernel_times.argtypes = [vp, i32]
    L.lb_voxel_create.argtypes = [i32, C.POINTER(vp)]
    L.lb_voxel_create_on_stream.argtypes = [i32, vp, C.POINTER(vp)]
    L.lb_voxel_destroy.argtypes = [vp]
    L.lb_voxel_set_leaf_size.argtypes = [vp, C.c_float, C.c_float, C.c_float]
    L.lb_voxel_get_leaf_size.argtypes = [vp, vp]
    L.lb_voxel_set_filter_limits.argtypes = [vp, C.c_char_p, C.c_double, C.c_double, i32]
    L.lb_voxel_set_min_points_per_voxel.argtypes = [vp, i32]
    L.lb_voxel_set_downsample_all_data.argtypes = [vp, i32]
    if hasattr(L, "lb_voxel_set_body_filter"):
        L.lb_voxel_set_body_filter.argtypes = [vp, i32, vp, vp, C.c_float]
    L.lb_voxel_filter.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(Field), i32, vp, sz, vp, sz,
                                  C.POINTER(sz), vp, i32, i32]
    if hasattr(L, "lb_voxel_filter_merged"):
        L.lb_voxel_set_input_passthrough.argtypes = [vp, C.c_char_p, C.c_double, C.c_double, i32]
        L.lb_voxel_filter_merged.argtypes = [vp, C.POINTER(VoxelInput), i32, C.c_uint32, C.POINTER(Field), i32, vp, sz,
                                             C.POINTER(sz), vp, i32, i32]
    if hasattr(L, "lb_voxel_extract_features"):
        L.lb_features_default_params.argtypes = [C.POINTER(FeaturesParams)]
        L.lb_voxel_extract_features.argtypes = [vp, vp, sz, sz, sz, i32, C.POINTER(FeaturesParams), vp, sz,
                                                C.POINTER(FeaturesResult), i32]
    L.lb_voxel_launch_count.argtypes = [vp, u64p]
    L.lb_voxel_kernel_time.argtypes = [vp, C.POINTER(C.c_float)]
    L.lb_voxel_kernel_time_avg.argtypes = [vp, C.POINTER(C.c_float), u64p, i32]
    if hasattr(L, "lb_submap_create"):
        L.lb_submap_create.argtypes = [i32, C.c_float, C.POINTER(vp)]
        L.lb_submap_destroy.argtypes = [vp]
        L.lb_submap_clear.argtypes = [vp]
        L.lb_submap_insert.argtypes = [vp, vp, sz, sz, sz, i32, C.POINTER(sz), vp]
        L.lb_submap_crop_box.argtypes = [vp, vp, C.c_float, C.POINTER(sz)]
        L.lb_submap_size.argtypes = [vp, C.POINTER(sz)]
        L.lb_submap_generation.argtypes = [vp, u64p]
        L.lb_submap_points.argtypes = [vp, vp, sz, i32]
        if hasattr(L, "lb_submap_normals"):
            L.lb_submap_insert_with_normals.argtypes = [vp, vp, sz, sz, sz, sz, i32, C.POINTER(sz), vp]
            L.lb_submap_normals.argtypes = [vp, vp, sz, i32]
        L.lb_submap_neighbors.argtypes = [vp, vp, sz, sz, sz, vp, vp, vp, i32]
        L.lb_submap_launch_count.argtypes = [vp, u64p]
        L.lb_gicp_set_target_submap.argtypes = [vp, vp]
    if hasattr(L, "lb_odometry_create"):     # absent only in older builds loaded through LOCUS_B200_LIB for A/B runs
        L.lb_odometry_create.argtypes = [i32, i32, sz, C.c_uint32, C.POINTER(vp)]
        L.lb_odometry_destroy.argtypes = [vp]
        L.lb_odometry_voxel.argtypes = [vp]; L.lb_odometry_voxel.restype = vp
        L.lb_odometry_gicp.argtypes = [vp, i32]; L.lb_odometry_gicp.restype = vp
        L.lb_odometry_depth.argtypes = [vp]
        L.lb_odometry_set_gicp_params.argtypes = [vp, C.POINTER(GicpParams)]
        if hasattr(L, "lb_odometry_set_cloud_sharing"):
            L.lb_odometry_set_cloud_sharing.argtypes = [vp, i32]
        if hasattr(L, "lb_odometry_set_normals"):
            L.lb_odometry_set_normals.argtypes = [vp, i32, vp]
        if hasattr(L, "lb_odometry_set_registration"):
            L.lb_odometry_set_registration.argtypes = [vp, i32, C.POINTER(NdtParams)]
        L.lb_odometry_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(Field), i32, i32, vp, vp, i32, u64p]
        L.lb_odometry_next.argtypes = [vp, C.POINTER(OdometryResult), i32]
        L.lb_odometry_pending.argtypes = [vp, C.POINTER(sz)]
        L.lb_odometry_launch_count.argtypes = [vp, u64p]
        L.lb_odometry_stage_times.argtypes = [vp, C.POINTER(C.c_double)]
        if hasattr(L, "lb_odometry_submit_merged"):
            L.lb_odometry_submit_merged.argtypes = [vp, C.POINTER(VoxelInput), i32, C.c_uint32, C.POINTER(Field), i32, i32, vp, vp,
                                                    i32, u64p]
    if hasattr(L, "lb_locus_create"):
        L.lb_locus_default_params.argtypes = [C.POINTER(LocusParams)]
        L.lb_locus_create.argtypes = [i32, i32, sz, C.c_uint32, vp, C.POINTER(vp)]
        L.lb_locus_destroy.argtypes = [vp]
        L.lb_locus_voxel.argtypes = [vp]; L.lb_locus_voxel.restype = vp
        L.lb_locus_set_params.argtypes = [vp, C.POINTER(LocusParams)]
        L.lb_locus_submit.argtypes = [vp, vp, sz, C.c_uint32, C.POINTER(Field), i32, i32, vp, vp, i32, u64p]
        L.lb_locus_next.argtypes = [vp, C.POINTER(LocusResult), i32]
        L.lb_locus_pending.argtypes = [vp, C.POINTER(sz)]
        L.lb_locus_stage_times.argtypes = [vp, C.POINTER(C.c_double)]
        if hasattr(L, "lb_locus_submit_merged"):
            L.lb_locus_submit_merged.argtypes = [vp, C.POINTER(VoxelInput), i32, C.c_uint32, C.POINTER(Field), i32, i32, vp, vp,
                                                 i32, u64p]
    if hasattr(L, "lb_ndt_create"):
        L.lb_ndt_default_params.argtypes = [C.POINTER(NdtParams)]
        L.lb_ndt_default_params.restype = None
        L.lb_ndt_create.argtypes = [i32, C.POINTER(vp)]
        L.lb_ndt_create_on_stream.argtypes = [i32, vp, C.POINTER(vp)]
        L.lb_ndt_destroy.argtypes = [vp]
        L.lb_ndt_set_params.argtypes = [vp, C.POINTER(NdtParams)]
        L.lb_ndt_set_source.argtypes = [vp, vp, sz, sz, sz, i32]
        L.lb_ndt_set_target.argtypes = [vp, vp, sz, sz, sz, i32]
        L.lb_ndt_align.argtypes = [vp, vp, C.POINTER(NdtResult)]
        L.lb_ndt_target_voxels.argtypes = [vp, sz, C.POINTER(sz), vp, vp, vp, vp, vp]
        L.lb_ndt_derivatives.argtypes = [vp, vp, vp, i32, C.POINTER(C.c_double), vp, vp]
        L.lb_ndt_launch_count.argtypes = [vp, u64p]
        if hasattr(L, "lb_ndt_set_target_submap"):
            L.lb_ndt_set_target_submap.argtypes = [vp, vp]
    _lib = L
    return L


def _check(status):
    if status != 0:
        raise LocusB200Error(status, lib().lb_last_error_string().decode(errors="replace"))


def device_count():
    n = C.c_int(0)
    lib().lb_device_count(C.byref(n))
    return n.value


def _ptr(a):
    """host numpy array -> (void*, LB_MEM_HOST); int -> raw device pointer."""
    if a is None:
        return None
    if isinstance(a, np.ndarray):
        return a.ctypes.data_as(C.c_void_p)
    return C.c_void_p(int(a))


def xyzi_fields():
    """PointField list of pcl::PointXYZI as it leaves BodyFilter (body_filter.cc:36-39)."""
    return [("x", 0, LB_FLOAT32, 1), ("y", 4, LB_FLOAT32, 1), ("z", 8, LB_FLOAT32, 1), ("intensity", 16, LB_FLOAT32, 1)]


def _merged_inputs(blobs, point_step, transforms):
    """lb_voxel_input[] for 1..3 clouds: each a host uint8 numpy array (n = size // point_step) or a (pointer, n_pts)
    pair (a device cloud); transforms: None or one 4x4 (or None) per cloud.  Returns (array, what must stay alive)."""
    transforms = [None] * len(blobs) if transforms is None else list(transforms)
    if len(transforms) != len(blobs):
        raise ValueError("one transform (or None) per cloud")
    arr = (VoxelInput * max(len(blobs), 1))()
    keep = []
    for i, (b, T) in enumerate(zip(blobs, transforms)):
        if isinstance(b, tuple):
            arr[i].data = int(b[0]) or None
            arr[i].n_pts = int(b[1])
        else:
            b = np.ascontiguousarray(b, dtype=np.uint8).reshape(-1)
            arr[i].data = b.ctypes.data_as(C.c_void_p).value
            arr[i].n_pts = b.size // point_step
        keep.append(b)
        if T is not None:
            T = np.ascontiguousarray(T, dtype=np.float32).reshape(16)      # the library copies it at submit
            arr[i].transform = T.ctypes.data_as(C.c_void_p).value
            keep.append(T)
    return arr, keep


class GicpB200:
    """Mirror of the pcl::Registration surface LOCUS calls (see module docstring)."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        L = lib()
        if stream is None:
            _check(L.lb_gicp_create(device, C.byref(self._h)))
        else:
            _check(L.lb_gicp_create_on_stream(device, C.c_void_p(int(stream)), C.byref(self._h)))
        self._p = GicpParams()
        L.lb_gicp_default_params(C.byref(self._p))
        self._res = None
        self._keep = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_borrowed", False):
            return
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_gicp_destroy(self._h)
            self._h = C.c_void_p()

    # ---- configuration (gicp.h:134-143,264-298 + pcl::Registration setters)
    def _apply(self):
        _check(lib().lb_gicp_set_params(self._h, C.byref(self._p)))

    def setTransformationEpsilon(self, v): self._p.transformation_epsilon = v; self._apply()
    def setMaxCorrespondenceDistance(self, v): self._p.max_correspondence_distance = v; self._apply()
    def setMaximumIterations(self, v): self._p.max_iterations = int(v); self._apply()
    def setRANSACIterations(self, v): self._p.ransac_iterations = int(v); self._apply()
    def setMaximumOptimizerIterations(self, v): self._p.max_optimizer_iterations = int(v); self._apply()
    def setNumThreads(self, v): self._p.num_threads = int(v); self._apply()
    def enableTimingOutput(self, v): self._p.enable_timing_output = int(bool(v)); self._apply()
    def RecomputeTargetCovariance(self, v): self._p.recompute_target_covariance = int(bool(v)); self._apply()
    def RecomputeSourceCovariance(self, v): self._p.recompute_source_covariance = int(bool(v)); self._apply()
    def setEuclideanFitnessEpsilon(self, v): self._p.euclidean_fitness_epsilon = v; self._apply()
    def setRotationEpsilon(self, v): self._p.rotation_epsilon = v; self._apply()
    def setCorrespondenceRandomness(self, k): self._p.k_correspondences = int(k); self._apply()
    def setOptimizer(self, v): self._p.optimizer = int(v); self._apply()
    def setExecution(self, v): self._p.execution = int(v); self._apply()
    def setIndexCellSize(self, v): self._p.index_cell_size = float(v); self._apply()
    def setAlignPointsPerCta(self, v): self._p.align_points_per_cta = int(v); self._apply()
    def getMaximumIterations(self): return self._p.max_iterations
    def getMaxCorrespondenceDistance(self): return self._p.max_correspondence_distance
    def getTransformationEpsilon(self): return self._p.transformation_epsilon
    def getRotationEpsilon(self): return self._p.rotation_epsilon
    def getCorrespondenceRandomness(self): return self._p.k_correspondences
    def getMaximumOptimizerIterations(self): return self._p.max_optimizer_iterations

    # ---- clouds.  cloud: (n, stride/4) float32 host array (xyz in columns xyz_col..+2), or
    # a raw device pointer with n/stride given explicitly.
    def _cloud_args(self, cloud, n, stride, xyz_off, normal_off):
        if isinstance(cloud, np.ndarray):
            a = np.ascontiguousarray(cloud, dtype=np.float32)
            assert a.ndim == 2 and a.shape[1] >= 3
            return a, a.ctypes.data_as(C.c_void_p), a.shape[0], a.shape[1] * 4, xyz_off, normal_off, LB_MEM_HOST
        return None, C.c_void_p(int(cloud)), int(n), int(stride), xyz_off, normal_off, LB_MEM_DEVICE

    def setInputSource(self, cloud, n=None, stride=None, xyz_off=0, normal_off=-1):
        keep, p, n_, st, xo, no, mem = self._cloud_args(cloud, n, stride, xyz_off, normal_off)
        _check(lib().lb_gicp_set_source(self._h, p, n_, st, xo, no, mem))
        self._keep["src"] = keep

    def setInputTarget(self, cloud, n=None, stride=None, xyz_off=0, normal_off=-1):
        keep, p, n_, st, xo, no, mem = self._cloud_args(cloud, n, stride, xyz_off, normal_off)
        gen = C.c_uint64(0)
        _check(lib().lb_gicp_set_target(self._h, p, n_, st, xo, no, mem, C.byref(gen)))
        self._keep["tgt"] = keep
        return gen.value

    def setTargetSubmap(self, submap):
        """the resident rolling submap as registration target (index + cached covariances live with the map)"""
        _check(lib().lb_gicp_set_target_submap(self._h, submap._h))
        self._keep["tgt"] = submap

    def reserve(self, max_points, spare_clouds=2):
        _check(lib().lb_gicp_reserve(self._h, int(max_points), int(spare_clouds)))

    def promoteSourceToTarget(self):
        _check(lib().lb_gicp_promote_source_to_target(self._h))

    # ---- prepared clouds shared between handles
    def prepareSource(self):
        _check(lib().lb_gicp_prepare_source(self._h))

    def shareSource(self):
        """opaque reference to the prepared source cloud (pass to another handle's setTargetCloud, then releaseCloud)"""
        c = C.c_void_p()
        _check(lib().lb_gicp_share_source(self._h, C.byref(c)))
        return c

    def setTargetCloud(self, cloud):
        _check(lib().lb_gicp_set_target_cloud(self._h, cloud))

    def setSourceCloud(self, cloud):
        """adopt a shared prepared cloud as source (no copy; the handle keeps its own reference)"""
        _check(lib().lb_gicp_set_source_cloud(self._h, cloud))

    @staticmethod
    def releaseCloud(cloud):
        lib().lb_cloud_release(cloud)

    def align(self, guess=None):
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        res = GicpResult()
        st = lib().lb_gicp_align(self._h, _ptr(g), C.byref(res))
        self._res = res
        _check(st)
        return res

    def getFinalTransformation(self):
        if self._res is None:
            return np.eye(4, dtype=np.float32)
        return np.array(self._res.final_transformation, dtype=np.float32).reshape(4, 4)

    def getLastIncrementalTransformation(self):
        """pcl::Registration::getLastIncrementalTransformation(): transformation_, the guess-free increment"""
        if self._res is None:
            return np.eye(4, dtype=np.float32)
        return np.array(self._res.transformation, dtype=np.float32).reshape(4, 4)

    def hasConverged(self):
        return bool(self._res.converged) if self._res is not None else False

    def getFitnessScore(self, max_range=1.7976931348623157e308):
        s = C.c_double(0)
        _check(lib().lb_gicp_fitness(self._h, None, max_range, C.byref(s)))
        return s.value

    def transformSource(self, T=None, with_normals=False):
        """The `output` cloud of align(): (n,3) float32 [, (n,3) normals]."""
        n = self.cloudSize(0)
        cols = 6 if with_normals else 3
        out = np.zeros((n, cols), dtype=np.float32)
        t = None if T is None else np.ascontiguousarray(T, dtype=np.float32).reshape(16)
        _check(lib().lb_gicp_transform_source(self._h, _ptr(t), _ptr(out), cols * 4, 0, 12 if with_normals else -1, LB_MEM_HOST))
        return out

    def nearestTarget(self, xyz):
        """getSearchMethodTarget()->nearestKSearch(pt, 1) for a batch: (idx int32, d2 float32)."""
        q = np.ascontiguousarray(xyz, dtype=np.float32)
        idx = np.zeros(q.shape[0], dtype=np.int32); d2 = np.zeros(q.shape[0], dtype=np.float32)
        _check(lib().lb_gicp_nn_target(self._h, _ptr(q), q.shape[0], q.shape[1] * 4, _ptr(idx), _ptr(d2), LB_MEM_HOST))
        return idx, d2

    def point2planeInformation(self, query_xyz, ref_normals, correspondences, T=None, normalize=True):
        """normalizePCloud + ComputeAp_ForPoint2PlaneICP (PointCloudLocalization.cc:694-750): 6x6 Ap."""
        q = np.ascontiguousarray(query_xyz, dtype=np.float32).reshape(-1, 3)
        r = np.ascontiguousarray(ref_normals, dtype=np.float32).reshape(-1, 3)
        co = np.ascontiguousarray(correspondences, dtype=np.int32)
        t = None if T is None else np.ascontiguousarray(T, dtype=np.float32).reshape(16)
        Ap = np.zeros(36)
        _check(lib().lb_gicp_point2plane_information(self._h, _ptr(q), q.shape[0], 12, 0, _ptr(r), r.shape[0], 12, 0,
                                                     _ptr(co), _ptr(t), int(normalize), _ptr(Ap), LB_MEM_HOST))
        return Ap.reshape(6, 6)

    def icpCovariance(self, T=None, correspondences=None, normal_rotation=None, max_covariance=0.01, device=False):
        """The ICP covariance after align (PointCloudLocalization.cc:325-336 + ComputePoint2PlaneICPCovariance): the
        source against the target's normals.  T: 4x4 (None = the final transformation); correspondences: int32 target
        index per source point (None = the exact 1-NN of T * source), a numpy array or, with device=True, a torch CUDA
        tensor; normal_rotation: 3x3 applied to the target normals (None = none).  Returns a dict: Ap, covariance (6x6),
        condition_number (NaN after the D-NaN fallback), flags (LB_ICPCOV_*), n_query, n_used."""
        t = None if T is None else np.ascontiguousarray(T, dtype=np.float32).reshape(16)
        r = None if normal_rotation is None else np.ascontiguousarray(normal_rotation, dtype=np.float32).reshape(9)
        mem, cp = LB_MEM_HOST, None
        if correspondences is not None:
            if device:
                mem, cp = LB_MEM_DEVICE, C.c_void_p(correspondences.data_ptr())
            else:
                co = np.ascontiguousarray(correspondences, dtype=np.int32)
                cp = _ptr(co)
        out = IcpCovariance()
        _check(lib().lb_gicp_icp_covariance(self._h, _ptr(t), cp, mem, _ptr(r), float(max_covariance), C.byref(out)))
        return {"Ap": np.array(out.Ap).reshape(6, 6), "covariance": np.array(out.covariance).reshape(6, 6),
                "condition_number": out.condition_number, "flags": out.flags, "n_query": out.n_query,
                "n_used": out.n_used}

    def covariances(self, which):
        n = self.cloudSize(which)
        out = np.zeros((n, 9))
        _check(lib().lb_gicp_get_covariances(self._h, which, _ptr(out), n))
        return out.reshape(n, 3, 3)

    def cloudSize(self, which):
        n = C.c_size_t(0)
        _check(lib().lb_gicp_cloud_size(self._h, which, C.byref(n)))
        return n.value

    def computeNormals(self, which=0, k=20, viewpoint=None):
        """NormalComputation nodelet, k-NN mode: (n, 4) float32 = normal_x, normal_y, normal_z, curvature of the cloud
        currently set as source (which=0) or target (which=1), in the caller's point order."""
        n = C.c_size_t(0)
        _check(lib().lb_gicp_cloud_size(self._h, which, C.byref(n)))
        out = np.zeros((n.value, 4), dtype=np.float32)
        vp_ = None if viewpoint is None else np.ascontiguousarray(viewpoint, dtype=np.float32)
        _check(lib().lb_gicp_compute_normals(self._h, which, int(k), _ptr(vp_), _ptr(out), LB_MEM_HOST))
        return out

    def estimateNormals(self, which=0, k=20, viewpoint=None):
        """the same normals written into the source (which=0) or target (which=1) cloud itself: it now has normals, and
        with recompute_*_covariance = 0 its covariances come from them"""
        vp_ = None if viewpoint is None else np.ascontiguousarray(viewpoint, dtype=np.float32)
        _check(lib().lb_gicp_estimate_normals(self._h, which, int(k), _ptr(vp_)))

    def computeNormalsRadius(self, which=0, radius=0.3, viewpoint=None):
        """NormalComputation nodelet, radius mode + NaN-normal removal: ((n, 4) float32 normals with NaN rows where a
        point has fewer than 3 neighbours, int32 indices of the points the nodelet keeps)"""
        n = self.cloudSize(which)
        out = np.zeros((n, 4), dtype=np.float32)
        vi = np.zeros(max(n, 1), dtype=np.int32)
        m = C.c_size_t(0)
        vp_ = None if viewpoint is None else np.ascontiguousarray(viewpoint, dtype=np.float32)
        _check(lib().lb_gicp_compute_normals_radius(self._h, which, float(radius), _ptr(vp_), _ptr(out), _ptr(vi), C.byref(m), LB_MEM_HOST))
        return out, vi[: m.value]

    def statisticalOutlierRemoval(self, which=0, mean_k=10, std_mul=1.0, negative=False):
        """pcl::StatisticalOutlierRemoval on the source (which=0) or target (which=1) cloud: (kept indices int32
        ascending, per-point mean distance (n,) float32, [mean, stddev, threshold] float64)"""
        n = self.cloudSize(which)
        kept = np.zeros(max(n, 1), dtype=np.int32); md = np.zeros(n, dtype=np.float32); st = np.zeros(3)
        m = C.c_size_t(0)
        _check(lib().lb_gicp_statistical_outlier_removal(self._h, which, int(mean_k), float(std_mul), int(bool(negative)),
                                                         _ptr(kept), C.byref(m), _ptr(md), _ptr(st), LB_MEM_HOST))
        return kept[: m.value], md, st

    def radiusOutlierRemoval(self, which=0, radius=0.15, min_neighbors=3, dense=True, negative=False):
        """pcl::RadiusOutlierRemoval on the source (which=0) or target (which=1) cloud; dense = the input's is_dense
        (PCL's k-NN branch) or not (its radius-search branch).  Returns the kept indices, int32 ascending."""
        n = self.cloudSize(which)
        kept = np.zeros(max(n, 1), dtype=np.int32)
        m = C.c_size_t(0)
        _check(lib().lb_gicp_radius_outlier_removal(self._h, which, float(radius), int(min_neighbors), int(bool(dense)),
                                                    int(bool(negative)), _ptr(kept), C.byref(m), LB_MEM_HOST))
        return kept[: m.value]

    def launchCount(self):
        n = C.c_uint64(0)
        lib().lb_gicp_launch_count(self._h, C.byref(n))
        return n.value

    def resetKernelTimes(self, enable=True):
        """False/0: off; True/1: all kernel classes + cycle counters; 2: only the align kernel's event pair"""
        _check(lib().lb_gicp_reset_kernel_times(self._h, int(enable)))

    def kernelTime(self, name):
        ms = C.c_float(0); n = C.c_uint64(0)
        lib().lb_gicp_kernel_time(self._h, name.encode(), C.byref(ms), C.byref(n))
        return ms.value, n.value


class VoxelGridB200:
    """Mirror of point_cloud_filter::CustomVoxelGrid's impl_ (pcl::VoxelGrid<PCLPointCloud2>)."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        if stream is None:
            _check(lib().lb_voxel_create(device, C.byref(self._h)))
        else:
            _check(lib().lb_voxel_create_on_stream(device, C.c_void_p(int(stream)), C.byref(self._h)))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_borrowed", False):
            return
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_voxel_destroy(self._h)
            self._h = C.c_void_p()

    def setLeafSize(self, lx, ly=None, lz=None):
        ly = lx if ly is None else ly
        lz = lx if lz is None else lz
        _check(lib().lb_voxel_set_leaf_size(self._h, np.float32(lx), np.float32(ly), np.float32(lz)))

    def getLeafSize(self):
        a = np.zeros(3, dtype=np.float32)
        _check(lib().lb_voxel_get_leaf_size(self._h, _ptr(a)))
        return a

    def setFilterFieldName(self, name): self._ff = name; self._push_limits()
    def setFilterLimits(self, lo, hi): self._lo, self._hi = lo, hi; self._push_limits()
    def setFilterLimitsNegative(self, neg): self._neg = bool(neg); self._push_limits()

    def _push_limits(self):
        name = getattr(self, "_ff", "")
        lo = getattr(self, "_lo", -3.4028234663852886e38); hi = getattr(self, "_hi", 3.4028234663852886e38)
        _check(lib().lb_voxel_set_filter_limits(self._h, name.encode() if name else None, lo, hi, int(getattr(self, "_neg", False))))

    def setMinimumPointsNumberPerVoxel(self, m): _check(lib().lb_voxel_set_min_points_per_voxel(self._h, int(m)))
    def setDownsampleAllData(self, a): _check(lib().lb_voxel_set_downsample_all_data(self._h, int(bool(a))))

    def setBodyFilter(self, min3=None, max3=None, rotation_z=0.0, enabled=True):
        """BodyFilter nodelet (pcl::CropBox, negative) folded into the filter: drop the points inside the rotated box"""
        if not enabled or min3 is None:
            _check(lib().lb_voxel_set_body_filter(self._h, 0, None, None, 0.0))
            return
        mn = np.ascontiguousarray(min3, dtype=np.float32); mx = np.ascontiguousarray(max3, dtype=np.float32)
        _check(lib().lb_voxel_set_body_filter(self._h, 1, _ptr(mn), _ptr(mx), np.float32(rotation_z)))

    @staticmethod
    def _fields(fields):
        arr = (Field * len(fields))()
        for i, (name, off, dt, cnt) in enumerate(fields):
            arr[i].name = name.encode(); arr[i].offset = off; arr[i].datatype = dt; arr[i].count = cnt
        return arr

    def filter(self, blob, point_step, fields, want_voxel_idx=False):
        """blob: uint8 host array (n*point_step).  returns (out (m, point_step) uint8[, voxel_idx int32])."""
        blob = np.ascontiguousarray(blob, dtype=np.uint8).reshape(-1)
        n = blob.size // point_step
        out = np.zeros(max(n, 1) * point_step, dtype=np.uint8)
        vidx = np.zeros(max(n, 1), dtype=np.int32) if want_voxel_idx else None
        n_out = C.c_size_t(0)
        fa = self._fields(fields)
        _check(lib().lb_voxel_filter(self._h, _ptr(blob), n, point_step, fa, len(fields), None, 0, _ptr(out), n,
                                     C.byref(n_out), _ptr(vidx), LB_MEM_HOST, LB_MEM_HOST))
        m = n_out.value
        o = out[: m * point_step].reshape(m, point_step)
        return (o, vidx[:m]) if want_voxel_idx else o

    def setInputPassThrough(self, field_name, lo, hi, negative=False):
        """the per-lidar pcl/PassThrough nodelet (raw field limits in the sensor frame + NaN removal) folded into the loads"""
        _check(lib().lb_voxel_set_input_passthrough(self._h, field_name.encode() if field_name else None, lo, hi, int(bool(negative))))

    def filterMerged(self, blobs, point_step, fields, transforms=None, want_voxel_idx=False):
        """1..3 clouds (uint8 host arrays) taken as one in the order given (point_cloud_merger), each optionally
        transformed by a 4x4 sensor -> base_link matrix; returns like filter()"""
        blobs = [np.ascontiguousarray(b, dtype=np.uint8).reshape(-1) for b in blobs]
        transforms = transforms or [None] * len(blobs)
        Ts = [None if T is None else np.ascontiguousarray(T, dtype=np.float32).reshape(16) for T in transforms]
        arr = (VoxelInput * len(blobs))()
        n = 0
        for i, b in enumerate(blobs):
            arr[i].data = b.ctypes.data_as(C.c_void_p).value
            arr[i].n_pts = b.size // point_step
            arr[i].transform = None if Ts[i] is None else Ts[i].ctypes.data_as(C.c_void_p).value
            n += b.size // point_step
        out = np.zeros(max(n, 1) * point_step, dtype=np.uint8)
        vidx = np.zeros(max(n, 1), dtype=np.int32) if want_voxel_idx else None
        n_out = C.c_size_t(0)
        fa = self._fields(fields)
        _check(lib().lb_voxel_filter_merged(self._h, arr, len(blobs), point_step, fa, len(fields), _ptr(out), n, C.byref(n_out),
                                            _ptr(vidx), LB_MEM_HOST, LB_MEM_HOST))
        m = n_out.value
        o = out[: m * point_step].reshape(m, point_step)
        return (o, vidx[:m]) if want_voxel_idx else o

    def filter_device(self, d_in, n, point_step, fields, d_out, capacity, d_vidx=None):
        """device pointers in/out; returns number of voxels."""
        n_out = C.c_size_t(0)
        fa = self._fields(fields)
        _check(lib().lb_voxel_filter(self._h, C.c_void_p(int(d_in)), n, point_step, fa, len(fields), None, 0,
                                     C.c_void_p(int(d_out)), capacity, C.byref(n_out),
                                     C.c_void_p(int(d_vidx)) if d_vidx else None, LB_MEM_DEVICE, LB_MEM_DEVICE))
        return n_out.value

    @staticmethod
    def featureParams(**params):
        """lb_features_params: the reference's defaults (PointCloudFilter.h:79-96) with `params` overriding fields"""
        p = FeaturesParams()
        _check(lib().lb_features_default_params(C.byref(p)))
        for k, v in params.items():
            if k not in dict(FeaturesParams._fields_):
                raise TypeError("unknown feature parameter %r" % k)
            setattr(p, k, v)
        return p

    def extractFeatures(self, xyz_or_blob, stride=None, xyz_off=0, out=None, **params):
        """The `filtering/extract_features` branch of PointCloudFilter::Filter (SURVEY 8f row f6).
        xyz_or_blob: an (n, >=3) float32 array (numpy on the host, or a contiguous CUDA tensor on the device), or a uint8
        host blob of `stride`-byte points with x, y, z at xyz_off.  out: None (a host array is returned) or a float32
        CUDA tensor of shape (capacity, 4) that receives the points on the device.  Returns (out (m, 4) float32
        x, y, z, intensity -- a view of `out` when given --, counts dict)."""
        p = self.featureParams(**params)
        if hasattr(xyz_or_blob, "data_ptr"):                    # CUDA tensor: device input
            t = xyz_or_blob
            assert t.is_cuda and t.dim() == 2 and t.shape[1] >= 3 and t.is_contiguous() and t.element_size() == 4
            src, n, mem_in = C.c_void_p(t.data_ptr()), t.shape[0], LB_MEM_DEVICE
            stride = t.shape[1] * 4
        else:
            a = np.ascontiguousarray(xyz_or_blob)
            if a.dtype == np.uint8:
                if stride is None:
                    raise ValueError("a byte blob needs its stride")
                a = a.reshape(-1)
                n = a.size // stride
            else:
                a = np.ascontiguousarray(a, dtype=np.float32)
                assert a.ndim == 2 and a.shape[1] >= 3
                n, stride = a.shape[0], a.shape[1] * 4
            src, mem_in = _ptr(a), LB_MEM_HOST
        r = FeaturesResult()
        if out is None:
            host = np.zeros((max(2 * n, 1), 4), np.float32)
            _check(lib().lb_voxel_extract_features(self._h, src, n, stride, xyz_off, mem_in, C.byref(p), _ptr(host),
                                                   host.shape[0], C.byref(r), LB_MEM_HOST))
            res = host[: r.n_out].copy()
        else:
            assert out.is_cuda and out.dim() == 2 and out.shape[1] == 4 and out.is_contiguous() and out.element_size() == 4
            _check(lib().lb_voxel_extract_features(self._h, src, n, stride, xyz_off, mem_in, C.byref(p),
                                                   C.c_void_p(out.data_ptr()), out.shape[0], C.byref(r), LB_MEM_DEVICE))
            res = out[: r.n_out]
        return res, {k: int(getattr(r, k)) for k, _ in FeaturesResult._fields_}

    def launchCount(self):
        n = C.c_uint64(0)
        lib().lb_voxel_launch_count(self._h, C.byref(n))
        return n.value

    def lastCallMs(self):
        ms = C.c_float(0)
        lib().lb_voxel_kernel_time(self._h, C.byref(ms))
        return ms.value

    def avgCallMs(self, reset=True):
        """mean CUDA-event duration of the filter calls since the last reset"""
        ms = C.c_float(0); n = C.c_uint64(0)
        lib().lb_voxel_kernel_time_avg(self._h, C.byref(ms), C.byref(n), int(reset))
        return ms.value


class SubmapB200:
    """Mirror of the mapper object LOCUS drives (locus/src/Locus.cc:464-465,479-486,522-543): InsertPoints,
    ApproxNearestNeighbors, Refresh -- resident on the GPU, and usable as a GICP target (GicpB200.setTargetSubmap)."""

    def __init__(self, device=0, resolution=0.05):
        self._h = C.c_void_p()
        _check(lib().lb_submap_create(device, np.float32(resolution), C.byref(self._h)))

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_submap_destroy(self._h)
            self._h = C.c_void_p()

    def Clear(self):
        _check(lib().lb_submap_clear(self._h))

    def InsertPoints(self, cloud, want_incremental=False):
        """cloud: (n, >=3) float32, fixed frame.  returns the number of points added [, the added points (m, 3)]"""
        a = np.ascontiguousarray(cloud, dtype=np.float32)
        n_ins = C.c_size_t(0)
        inc = np.zeros((max(len(a), 1), 3), dtype=np.float32) if want_incremental else None
        _check(lib().lb_submap_insert(self._h, _ptr(a), a.shape[0], a.shape[1] * 4, 0, LB_MEM_HOST, C.byref(n_ins), _ptr(inc)))
        return (n_ins.value, inc[: n_ins.value]) if want_incremental else n_ins.value

    def InsertPointsWithNormals(self, cloud, normals, want_incremental=False):
        """cloud, normals: (n, 3) float32, fixed frame; each voxel's winning point keeps its normal"""
        a = np.ascontiguousarray(np.hstack([np.asarray(cloud, np.float32)[:, :3], np.asarray(normals, np.float32)[:, :3]]))
        n_ins = C.c_size_t(0)
        inc = np.zeros((max(len(a), 1), 3), dtype=np.float32) if want_incremental else None
        _check(lib().lb_submap_insert_with_normals(self._h, _ptr(a), a.shape[0], 24, 0, 12, LB_MEM_HOST, C.byref(n_ins), _ptr(inc)))
        return (n_ins.value, inc[: n_ins.value]) if want_incremental else n_ins.value

    def insert_device(self, ptr, n, stride, xyz_off=0):
        n_ins = C.c_size_t(0)
        _check(lib().lb_submap_insert(self._h, C.c_void_p(int(ptr)), n, stride, xyz_off, LB_MEM_DEVICE, C.byref(n_ins), None))
        return n_ins.value

    def Refresh(self, center, half_size):
        """sliding window: keep the points inside the box centre +- half_size; returns the number removed"""
        c = np.ascontiguousarray(center, dtype=np.float32).reshape(3)
        n = C.c_size_t(0)
        _check(lib().lb_submap_crop_box(self._h, _ptr(c), np.float32(half_size), C.byref(n)))
        return n.value

    def size(self):
        n = C.c_size_t(0)
        _check(lib().lb_submap_size(self._h, C.byref(n)))
        return n.value

    def generation(self):
        g = C.c_uint64(0)
        _check(lib().lb_submap_generation(self._h, C.byref(g)))
        return g.value

    def points(self):
        out = np.zeros((self.size(), 3), dtype=np.float32)
        _check(lib().lb_submap_points(self._h, _ptr(out), out.shape[0], LB_MEM_HOST))
        return out

    def normals(self):
        """(n, 3) float32 in insertion order; NaN rows for points inserted without a normal"""
        out = np.zeros((self.size(), 3), dtype=np.float32)
        _check(lib().lb_submap_normals(self._h, _ptr(out), out.shape[0], LB_MEM_HOST))
        return out

    def ApproxNearestNeighbors(self, cloud):
        """(neighbors (n, 3), idx int32, d2 float32): the nearest map point of every point of `cloud`"""
        q = np.ascontiguousarray(cloud, dtype=np.float32)
        nb = np.zeros((q.shape[0], 3), dtype=np.float32)
        idx = np.zeros(q.shape[0], dtype=np.int32); d2 = np.zeros(q.shape[0], dtype=np.float32)
        _check(lib().lb_submap_neighbors(self._h, _ptr(q), q.shape[0], q.shape[1] * 4, 0, _ptr(nb), _ptr(idx), _ptr(d2), LB_MEM_HOST))
        return nb, idx, d2

    def launchCount(self):
        n = C.c_uint64(0)
        lib().lb_submap_launch_count(self._h, C.byref(n))
        return n.value


class OdometryB200:
    """Mirror of the per-scan chain of the reference's lidar callback (locus/src/Locus.cc:451-453:
    odometry_.SetLidar(filtered) + odometry_.UpdateEstimate(), PointCloudOdometry.cc:221-274) as the library's
    two-stage pipeline: VoxelGrid of scan k+1 overlaps the registration of scan k, `depth` registrations in flight."""

    def __init__(self, device=0, depth=3, max_points=1 << 18, max_point_step=32):
        self._h = C.c_void_p()
        _check(lib().lb_odometry_create(device, depth, max_points, max_point_step, C.byref(self._h)))
        self.depth = depth
        self.voxel = VoxelGridB200.__new__(VoxelGridB200)          # borrowed handles: never destroyed from here
        self.voxel._h = C.c_void_p(lib().lb_odometry_voxel(self._h)); self.voxel._borrowed = True
        self._g = []
        for i in range(depth):
            g = GicpB200.__new__(GicpB200)
            g._h = C.c_void_p(lib().lb_odometry_gicp(self._h, i)); g._borrowed = True
            g._p = GicpParams(); lib().lb_gicp_get_params(g._h, C.byref(g._p)); g._res = None; g._keep = {}
            self._g.append(g)
        self._keep = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_odometry_destroy(self._h)
            self._h = C.c_void_p()

    def gicp(self, i):
        return self._g[i]

    def setGicpParams(self, **kw):
        """keyword = lb_gicp_params field name; applied to every registration worker."""
        p = GicpParams()
        lib().lb_gicp_get_params(self._g[0]._h, C.byref(p))
        for k, v in kw.items():
            if not hasattr(p, k):
                raise AttributeError(k)
            setattr(p, k, v)
        _check(lib().lb_odometry_set_gicp_params(self._h, C.byref(p)))
        for g in self._g:
            lib().lb_gicp_get_params(g._h, C.byref(g._p))

    def setCloudSharing(self, on=True):
        """each scan's index + covariances computed once and adopted as the next registration's target (idle pipeline only)"""
        _check(lib().lb_odometry_set_cloud_sharing(self._h, int(bool(on))))

    def setNormals(self, k=20, viewpoint=None):
        """normals stage: every filtered scan gets its k-NN normals (k = 0: off); idle pipeline, before the first scan"""
        vp_ = None if viewpoint is None else np.ascontiguousarray(viewpoint, dtype=np.float32)
        _check(lib().lb_odometry_set_normals(self._h, int(k), _ptr(vp_)))

    def setRegistration(self, method="ndt", **ndt):
        """registration method of every worker: "gicp" (default) or "ndt"; keywords = lb_ndt_params fields over
        lb_ndt_default_params (idle pipeline; the method is fixed once the first scan is submitted)"""
        p = NdtParams()
        lib().lb_ndt_default_params(C.byref(p))
        for k, v in ndt.items():
            if not hasattr(p, k):
                raise AttributeError(k)
            setattr(p, k, v)
        _check(lib().lb_odometry_set_registration(self._h, _reg_method(method), C.byref(p)))

    def submit(self, scan, n_pts, point_step, fields, mem=LB_MEM_HOST, guess=None, filtered_out=None,
               mem_filtered=LB_MEM_HOST):
        """scan / filtered_out: host uint8 numpy arrays or raw pointers (int).  Returns the ticket."""
        fa = fields if not isinstance(fields, (list, tuple)) else VoxelGridB200._fields(fields)
        t = C.c_uint64(0)
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        _check(lib().lb_odometry_submit(self._h, _ptr(scan), n_pts, point_step, fa, len(fa), mem, _ptr(g),
                                        _ptr(filtered_out), mem_filtered, C.byref(t)))
        self._keep[t.value] = (scan, fa, g, filtered_out)        # buffers stay alive until the result is returned
        return t.value

    def submit_merged(self, blobs, point_step, fields, transforms=None, mem=LB_MEM_HOST, guess=None, filtered_out=None,
                      mem_filtered=LB_MEM_HOST):
        """one scan of 1..3 lidars merged in the VoxelGrid stage (lb_odometry_submit_merged), in the order given (the
        merger's alive_keys_ order); blobs: host uint8 numpy arrays or (pointer, n_pts) pairs; transforms: one 4x4
        sensor -> base_link (or None) per cloud.  filtered_out holds sum(n_pts) * point_step bytes.  Returns the ticket."""
        fa = fields if not isinstance(fields, (list, tuple)) else VoxelGridB200._fields(fields)
        arr, keep = _merged_inputs(blobs, point_step, transforms)
        t = C.c_uint64(0)
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        _check(lib().lb_odometry_submit_merged(self._h, arr, len(blobs), point_step, fa, len(fa), mem, _ptr(g),
                                               _ptr(filtered_out), mem_filtered, C.byref(t)))
        self._keep[t.value] = (keep, fa, g, filtered_out)         # the clouds stay alive until the result is returned
        return t.value

    def next(self, block=True):
        """next result in submission order, or None when block=False and it is not ready."""
        r = OdometryResult()
        s = lib().lb_odometry_next(self._h, C.byref(r), int(bool(block)))
        if s == 1:
            return None
        _check(s)
        self._keep.pop(r.ticket, None)
        return r

    def pending(self):
        n = C.c_size_t(0)
        _check(lib().lb_odometry_pending(self._h, C.byref(n)))
        return n.value

    def launchCount(self):
        n = C.c_uint64(0)
        lib().lb_odometry_launch_count(self._h, C.byref(n))
        return n.value

    def stageTimes(self):
        """host wall-clock accounting since creation (see lb_odometry_stage_times)"""
        a = (C.c_double * 6)()
        _check(lib().lb_odometry_stage_times(self._h, a))
        return {"filtered": int(a[0]), "voxel_busy_s": a[1], "voxel_wait_s": a[2], "registered": int(a[3]),
                "workers_busy_s": a[4], "workers_wait_s": a[5]}


def locus_params(**kw):
    """lb_locus_params with the reference's shipped values; keywords override top-level fields, and `odometry` /
    `localization` / `*_thresholds` / `front_end` / `icp_covariance` / `*_ndt` take dicts of their fields;
    `odometry_method` / `localization_method` take "gicp" or "ndt" (or LB_REG_*)"""
    p = LocusParams()
    _check(lib().lb_locus_default_params(C.byref(p)))
    for k, v in kw.items():
        if k not in dict(LocusParams._fields_):
            raise AttributeError(k)
        if isinstance(v, dict):
            sub = getattr(p, k)
            for kk, vv in v.items():
                if not hasattr(sub, kk):
                    raise AttributeError("%s.%s" % (k, kk))
                if kk == "viewpoint":
                    sub.viewpoint[:] = [float(x) for x in np.asarray(vv, dtype=np.float32).reshape(3)]
                else:
                    setattr(sub, kk, vv)
        elif k == "initial_pose":
            p.initial_pose[:] = [float(x) for x in np.asarray(v, dtype=np.float64).reshape(16)]
        elif k in ("odometry_method", "localization_method"):
            setattr(p, k, _reg_method(v))
        else:
            setattr(p, k, v)
    return p


class LocusB200:
    """Locus::LidarCallback (locus/src/Locus.cc:450-543) as one pipeline: VoxelGrid, scan-to-scan odometry,
    scan-to-submap localization and keyframe map updates of `submap` (a SubmapB200 on the same device, which the
    chain updates and the caller keeps).  Results come back in submission order with O_k, I_k and L_k as 4x4 doubles."""

    def __init__(self, submap, device=0, depth=3, max_points=1 << 18, max_point_step=32, **params):
        self._h = C.c_void_p()
        _check(lib().lb_locus_create(device, depth, max_points, max_point_step, submap._h, C.byref(self._h)))
        self.submap = submap
        self.voxel = VoxelGridB200.__new__(VoxelGridB200)          # borrowed handle: never destroyed from here
        self.voxel._h = C.c_void_p(lib().lb_locus_voxel(self._h)); self.voxel._borrowed = True
        self._keep = {}
        if params:
            self.setParams(**params)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_locus_destroy(self._h)
            self._h = C.c_void_p()

    def setParams(self, **kw):
        """keywords as locus_params(); only while no scan is in flight"""
        p = locus_params(**kw)
        _check(lib().lb_locus_set_params(self._h, C.byref(p)))
        self.params = p

    def submit(self, scan, n_pts, point_step, fields, mem=LB_MEM_HOST, guess=None, filtered_out=None,
               mem_filtered=LB_MEM_HOST):
        """as OdometryB200.submit; guess = the odometry prior.  Returns the ticket."""
        fa = fields if not isinstance(fields, (list, tuple)) else VoxelGridB200._fields(fields)
        t = C.c_uint64(0)
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        _check(lib().lb_locus_submit(self._h, _ptr(scan), n_pts, point_step, fa, len(fa), mem, _ptr(g),
                                     _ptr(filtered_out), mem_filtered, C.byref(t)))
        self._keep[t.value] = (scan, fa, g, filtered_out)
        return t.value

    def submit_merged(self, blobs, point_step, fields, transforms=None, mem=LB_MEM_HOST, guess=None, filtered_out=None,
                      mem_filtered=LB_MEM_HOST):
        """as OdometryB200.submit_merged (lb_locus_submit_merged): 1..3 lidars merged in the VoxelGrid stage; the
        keyframe the map receives is the merged filtered scan.  Returns the ticket."""
        fa = fields if not isinstance(fields, (list, tuple)) else VoxelGridB200._fields(fields)
        arr, keep = _merged_inputs(blobs, point_step, transforms)
        t = C.c_uint64(0)
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        _check(lib().lb_locus_submit_merged(self._h, arr, len(blobs), point_step, fa, len(fa), mem, _ptr(g),
                                            _ptr(filtered_out), mem_filtered, C.byref(t)))
        self._keep[t.value] = (keep, fa, g, filtered_out)
        return t.value

    def next(self, block=True):
        """next LocusResult in submission order, or None when block=False and it is not ready."""
        r = LocusResult()
        s = lib().lb_locus_next(self._h, C.byref(r), int(bool(block)))
        if s == 1:
            return None
        _check(s)
        self._keep.pop(r.ticket, None)
        return r

    def pending(self):
        n = C.c_size_t(0)
        _check(lib().lb_locus_pending(self._h, C.byref(n)))
        return n.value

    def stageTimes(self):
        a = (C.c_double * 9)()
        _check(lib().lb_locus_stage_times(self._h, a))
        return {"filtered": int(a[0]), "voxel_busy_s": a[1], "voxel_wait_s": a[2], "registered": int(a[3]),
                "workers_busy_s": a[4], "workers_wait_s": a[5], "localized": int(a[6]), "localization_busy_s": a[7],
                "localization_wait_s": a[8]}

    @staticmethod
    def poses(r):
        """(O_k, I_k, L_k) of a LocusResult as 4x4 float64 arrays"""
        return tuple(np.array(getattr(r, k), dtype=np.float64).reshape(4, 4) for k in ("odometry_pose", "incremental", "pose"))


NDT_KDTREE, NDT_DIRECT26, NDT_DIRECT7, NDT_DIRECT1 = 0, 1, 2, 3


class NdtB200:
    """Mirror of the pclomp::NormalDistributionsTransform surface LOCUS drives when `registration_method: ndt`
    (PointCloudOdometry.cc:182-195, PointCloudLocalization.cc:267-280; setters of ndt_omp.h:116-196)."""

    def __init__(self, device=0, stream=None):
        self._h = C.c_void_p()
        L = lib()
        if stream is None:
            _check(L.lb_ndt_create(device, C.byref(self._h)))
        else:
            _check(L.lb_ndt_create_on_stream(device, C.c_void_p(int(stream)), C.byref(self._h)))
        self._p = NdtParams()
        L.lb_ndt_default_params(C.byref(self._p))
        self._res = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            lib().lb_ndt_destroy(self._h)
            self._h = C.c_void_p()

    def _apply(self):
        _check(lib().lb_ndt_set_params(self._h, C.byref(self._p)))

    def setTransformationEpsilon(self, v): self._p.transformation_epsilon = v; self._apply()
    def setMaximumIterations(self, v): self._p.max_iterations = int(v); self._apply()
    def setMaxCorrespondenceDistance(self, v): self._p.max_correspondence_distance = v; self._apply()
    def setRANSACIterations(self, v): self._p.ransac_iterations = int(v); self._apply()
    def setNumThreads(self, v): self._p.num_threads = int(v); self._apply()
    def enableTimingOutput(self, v): self._p.enable_timing_output = int(bool(v)); self._apply()
    def setResolution(self, v): self._p.resolution = float(v); self._apply()
    def setStepSize(self, v): self._p.step_size = float(v); self._apply()
    def setOulierRatio(self, v): self._p.outlier_ratio = float(v); self._apply()           # the reference's spelling (ndt_omp.h:166)
    def setNeighborhoodSearchMethod(self, v): self._p.search_method = int(v); self._apply()
    def setMinPointPerVoxel(self, v): self._p.min_points_per_voxel = int(v); self._apply()
    def setCovEigValueInflationRatio(self, v): self._p.min_covar_eigvalue_mult = float(v); self._apply()
    def getResolution(self): return self._p.resolution
    def getStepSize(self): return self._p.step_size
    def getOulierRatio(self): return self._p.outlier_ratio

    @staticmethod
    def _cloud(cloud):
        a = np.ascontiguousarray(cloud, dtype=np.float32)
        assert a.ndim == 2 and a.shape[1] >= 3
        return a

    def setInputSource(self, cloud):
        a = self._cloud(cloud)
        _check(lib().lb_ndt_set_source(self._h, _ptr(a), a.shape[0], a.shape[1] * 4, 0, LB_MEM_HOST))

    def setInputTarget(self, cloud):
        a = self._cloud(cloud)
        _check(lib().lb_ndt_set_target(self._h, _ptr(a), a.shape[0], a.shape[1] * 4, 0, LB_MEM_HOST))

    def setTargetSubmap(self, submap):
        """the SubmapB200's current points as the target, gathered on the device (lb_ndt_set_target_submap); call again
        after the map changed -- while it is unchanged the call does nothing"""
        _check(lib().lb_ndt_set_target_submap(self._h, submap._h))

    def align(self, guess=None):
        g = None if guess is None else np.ascontiguousarray(guess, dtype=np.float32).reshape(16)
        r = NdtResult()
        _check(lib().lb_ndt_align(self._h, _ptr(g), C.byref(r)))
        self._res = r
        return r

    def _result(self):
        if self._res is None:
            raise LocusB200Error(-10, "no successful align() yet")
        return self._res

    def getFinalTransformation(self): return np.array(self._result().final_transformation, dtype=np.float32).reshape(4, 4)
    def hasConverged(self): return bool(self._result().converged)
    def getTransformationProbability(self): return self._result().trans_probability
    def getFinalNumIteration(self): return self._result().nr_iterations

    def targetVoxels(self):
        """The searchable voxels of the target (voxel_centroids_ order = ascending voxel index)."""
        n = C.c_size_t(0)
        _check(lib().lb_ndt_target_voxels(self._h, 0, C.byref(n), None, None, None, None, None))
        n = n.value
        out = {"leaf_idx": np.zeros(n, np.int32), "nr_points": np.zeros(n, np.int32), "mean": np.zeros((n, 3)),
               "icov": np.zeros((n, 9)), "centroid": np.zeros((n, 3), np.float32)}
        _check(lib().lb_ndt_target_voxels(self._h, n, C.byref(C.c_size_t(0)), _ptr(out["leaf_idx"]), _ptr(out["nr_points"]),
                                          _ptr(out["mean"]), _ptr(out["icov"]), _ptr(out["centroid"])))
        return out

    def derivatives(self, T, pose, compute_hessian=1):
        T = np.ascontiguousarray(T, dtype=np.float32).reshape(16)
        pose = np.ascontiguousarray(pose, dtype=np.float64)
        score = C.c_double(0); g = np.zeros(6); H = np.zeros((6, 6))
        _check(lib().lb_ndt_derivatives(self._h, _ptr(T), _ptr(pose), int(compute_hessian), C.byref(score), _ptr(g), _ptr(H)))
        return score.value, g, H

    def launchCount(self):
        n = C.c_uint64(0)
        _check(lib().lb_ndt_launch_count(self._h, C.byref(n)))
        return n.value
