"""ctypes binding of the C ABI declared in include/b2points.h (libb2points.so).

The library is hand-written CUDA for sm_90a and has no CPU fallback: if it cannot be loaded, or no CUDA device is
present, every entry point of this package raises -- nothing is silently computed elsewhere.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "lib", "libb2points.so")

B2_LINEARIZED_DOUBLES = 128
B2_CLOUD_DEFAULT = 0
B2_CLOUD_NO_REORDER = 1
B2_CLOUD_COMPACT_F32 = 2
B2_CLOUD_FORCE_F64 = 4

_STATUS = {0: "B2_OK", 1: "B2_ERR_INVALID_ARGUMENT", 2: "B2_ERR_CUDA", 3: "B2_ERR_OUT_OF_MEMORY", 4: "B2_ERR_INVALID_STATE", 5: "B2_ERR_NO_DEVICE"}


class B2Error(RuntimeError):
    def __init__(self, status, message):
        super().__init__(f"{_STATUS.get(status, status)}: {message}")
        self.status = status


class CloudInfo(C.Structure):
    _fields_ = [("num_points", C.c_uint64), ("point_bytes", C.c_int32), ("cov_bytes", C.c_int32), ("reordered", C.c_int32), ("normal_bytes", C.c_int32), ("device_bytes", C.c_uint64)]


class VoxelMapInfo(C.Structure):
    _fields_ = [("num_voxels", C.c_uint64), ("num_buckets", C.c_uint64), ("resolution", C.c_double), ("device_bytes", C.c_uint64)]


class Residency(C.Structure):
    _fields_ = [("loaded_on_gpu", C.c_int32), ("reserved", C.c_int32), ("last_access", C.c_uint64), ("device_bytes", C.c_uint64), ("host_bytes", C.c_uint64)]


class IvoxInfo(C.Structure):
    _fields_ = [("num_voxels", C.c_uint64), ("num_points", C.c_uint64), ("resolution", C.c_double), ("device_bytes", C.c_uint64)]


B2_IVOX_MAX_POINTS_IN_CELL = 32
B2_FEATURES_MAX_DIM = 128
B2_FPFH_DIM = 33
B2_PFH_DIM = 125


class MinCutParamsC(C.Structure):
    _fields_ = [("distance_sigma", C.c_double), ("angle_sigma", C.c_double), ("foreground_mask_radius", C.c_double), ("background_mask_radius", C.c_double),
                ("foreground_weight", C.c_double), ("background_weight", C.c_double), ("k_neighbors", C.c_int32), ("reserved", C.c_int32)]


class MinCutResultC(C.Structure):
    _fields_ = [("source_index", C.c_int64), ("sink_index", C.c_int64), ("max_flow", C.c_double), ("max_flow_q", C.c_int64), ("cluster_size", C.c_uint64),
                ("flags", C.c_int32), ("reserved", C.c_int32)]


B2_MIN_CUT_NO_SEED, B2_MIN_CUT_FEW_NEIGHBORS, B2_MIN_CUT_NO_SINK = 1, 2, 4


class OccGridInfo(C.Structure):
    _fields_ = [("resolution", C.c_double), ("num_occupied_cells", C.c_uint64), ("num_blocks", C.c_uint64), ("device_bytes", C.c_uint64)]


class FeaturesInfo(C.Structure):
    _fields_ = [("num_features", C.c_uint64), ("dim", C.c_int32), ("reserved", C.c_int32), ("device_bytes", C.c_uint64)]


class RansacParams(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("dof", C.c_int32), ("early_stop_inlier_rate", C.c_double), ("poly_error_thresh", C.c_double),
                ("inlier_voxel_resolution", C.c_double), ("seed", C.c_uint64), ("taboo_thresh_rot", C.c_double), ("taboo_thresh_trans", C.c_double),
                ("taboo_list", C.POINTER(C.c_double)), ("num_taboo", C.c_uint64)]


class GncParams(C.Structure):
    _fields_ = [("max_init_samples", C.c_int32), ("reciprocal_check", C.c_int32), ("tuple_check", C.c_int32), ("max_num_tuples", C.c_int32),
                ("tuple_thresh", C.c_double), ("div_factor", C.c_double), ("max_corr_dist", C.c_double), ("inner_iterations", C.c_int32),
                ("max_iterations", C.c_int32), ("dof", C.c_int32), ("reserved", C.c_int32), ("seed", C.c_uint64)]


class RegistrationResultC(C.Structure):
    _fields_ = [("T_target_source", C.c_double * 16), ("inlier_rate", C.c_double), ("num_inliers", C.c_int64), ("hypothesis", C.c_int64)]


class LmParamsC(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("reserved", C.c_int32), ("relative_error_tol", C.c_double), ("absolute_error_tol", C.c_double),
                ("error_tol", C.c_double), ("lambda_initial", C.c_double), ("lambda_factor", C.c_double), ("lambda_upper_bound", C.c_double),
                ("lambda_lower_bound", C.c_double), ("min_model_fidelity", C.c_double)]


class LmSummaryC(C.Structure):
    _fields_ = [("iterations", C.c_int64), ("outer_iterations", C.c_int64), ("inner_iterations", C.c_int64), ("linearizations", C.c_int64),
                ("error_evaluations", C.c_int64), ("error0", C.c_double), ("error", C.c_double), ("lambda_", C.c_double), ("termination", C.c_int32),
                ("reserved", C.c_int32)]


class PosePriorC(C.Structure):
    _fields_ = [("var", C.c_int32), ("reserved", C.c_int32), ("T_prior", C.c_double * 16), ("precision", C.c_double * 6)]


class LmGraphTraceEntryC(C.Structure):
    _fields_ = [("outer", C.c_int32), ("solved", C.c_int32), ("success", C.c_int32), ("stop", C.c_int32), ("lambda_", C.c_double),
                ("error", C.c_double), ("half_f", C.c_double), ("lin_change", C.c_double), ("error_trial", C.c_double), ("fidelity", C.c_double)]


B2_LM_MAX_POSES = 32
B2_LM_TERMINATION = {0: "none", 1: "max_iterations", 2: "non_finite", 3: "absolute_error_tol", 4: "relative_error_tol", 5: "error_tol", 6: "try_limit"}

_lib = None

# name -> (restype, argtypes); every symbol include/b2points.h declares
_vp, _dp, _ip, _lp = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int32), C.POINTER(C.c_int64)
_pp = C.POINTER(C.c_void_p)
SIGNATURES = {
    "b2_last_error": (C.c_char_p, []),
    "b2_version": (C.c_char_p, []),
    "b2_ctx_create": (C.c_int, [C.c_int, _vp, _pp]),
    "b2_ctx_destroy": (C.c_int, [_vp]),
    "b2_ctx_synchronize": (C.c_int, [_vp]),
    "b2_ctx_stream": (_vp, [_vp]),
    "b2_device_malloc": (C.c_int, [_vp, C.c_size_t, _pp]),
    "b2_device_free": (C.c_int, [_vp, _vp]),
    "b2_memcpy_d2h": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2_memcpy_h2d": (C.c_int, [_vp, _vp, _vp, C.c_size_t]),
    "b2_cloud_create": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_create_with_normals": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, _dp, C.c_int, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_download_normals": (C.c_int, [_vp, _dp]),
    "b2_cloud_create_with_intensities": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, _dp, C.c_int, _dp, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_intensity_bytes": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "b2_cloud_create_with_added_intensities": (C.c_int, [_vp, _dp, C.c_uint, _pp]),
    "b2_cloud_download_intensities": (C.c_int, [_vp, _dp]),
    "b2_cloud_create_voxelgrid_with_intensities": (C.c_int, [_vp, C.c_double, _dp, C.c_int, _dp, C.c_int, _dp, C.c_int, _dp, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_download": (C.c_int, [_vp, _dp, _dp, _dp]),
    "b2_cloud_create_voxelgrid": (C.c_int, [_vp, C.c_double, _dp, C.c_int, _dp, C.c_int, _dp, C.c_int, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_create_estimated": (C.c_int, [_vp, _vp, C.c_int, _dp, C.c_int, C.c_uint, _pp]),
    "b2_cloud_create_transformed": (C.c_int, [_vp, _dp, C.c_uint, _pp]),
    "b2_cloud_create_sampled": (C.c_int, [_vp, _lp, C.c_size_t, C.c_uint, _pp]),
    "b2_cloud_create_random_sampled": (C.c_int, [_vp, C.c_double, C.c_uint64, C.c_uint, _lp, _pp]),
    "b2_cloud_create_randomgrid": (C.c_int, [_vp, C.c_double, C.c_double, C.c_uint64, C.c_uint, _lp, _pp]),
    "b2_cloud_create_inliers": (C.c_int, [_vp, _vp, C.c_int, C.c_double, C.c_uint, _dp, _dp, _lp, _pp]),
    "b2_cloud_destroy": (C.c_int, [_vp]),
    "b2_cloud_get_info": (C.c_int, [_vp, C.POINTER(CloudInfo)]),
    "b2_voxelmap_create_from_points": (C.c_int, [_vp, C.c_double, _dp, C.c_int, _dp, C.c_int, C.c_size_t, _pp]),
    "b2_voxelmap_create": (C.c_int, [_vp, C.c_double, _pp]),
    "b2_voxelmap_set_lru": (C.c_int, [_vp, C.c_size_t, C.c_size_t]),
    "b2_voxelmap_insert": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, C.c_size_t]),
    "b2_voxelmap_insert_cloud": (C.c_int, [_vp, _vp, _dp]),
    "b2_voxelmap_insert_with_intensities": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, _dp, C.c_size_t]),
    "b2_voxelmap_create_from_voxels_with_intensities": (C.c_int, [_vp, C.c_double, _ip, _dp, _dp, _ip, _dp, C.c_size_t, _pp]),
    "b2_voxelmap_download_intensities": (C.c_int, [_vp, _dp]),
    "b2_voxelmap_create_from_voxels": (C.c_int, [_vp, C.c_double, _ip, _dp, _dp, _ip, C.c_size_t, _pp]),
    "b2_voxelmap_destroy": (C.c_int, [_vp]),
    "b2_voxelmap_get_info": (C.c_int, [_vp, C.POINTER(VoxelMapInfo)]),
    "b2_voxelmap_download": (C.c_int, [_vp, _ip, _dp, _dp, _ip]),
    "b2_voxelmap_save_compact": (C.c_int, [_vp, C.c_char_p]),
    "b2_voxelmap_load": (C.c_int, [_vp, C.c_char_p, _pp]),
    "b2_overlap": (C.c_int, [_pp, C.c_size_t, _vp, _dp, _dp]),
    "b2_merge_frames": (C.c_int, [_vp, _dp, C.POINTER(C.c_void_p), C.c_size_t, C.c_double, _dp, _dp, C.POINTER(C.c_size_t)]),
    "b2_merge_frames_to_cloud": (C.c_int, [_vp, _dp, C.POINTER(C.c_void_p), C.c_size_t, C.c_double, C.c_uint, _pp]),
    "b2_voxelmap_lookup": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, _ip]),
    "b2_cloud_offload": (C.c_int, [_vp, _ip]),
    "b2_cloud_reload": (C.c_int, [_vp, _ip]),
    "b2_cloud_touch": (C.c_int, [_vp, _ip]),
    "b2_cloud_residency": (C.c_int, [_vp, C.POINTER(Residency)]),
    "b2_voxelmap_offload": (C.c_int, [_vp, _ip]),
    "b2_voxelmap_reload": (C.c_int, [_vp, _ip]),
    "b2_voxelmap_touch": (C.c_int, [_vp, _ip]),
    "b2_voxelmap_residency": (C.c_int, [_vp, C.POINTER(Residency)]),
    "b2_access_time_current": (C.c_int, [C.POINTER(C.c_uint64)]),
    "b2_ivox_create": (C.c_int, [_vp, C.c_double, _pp]),
    "b2_ivox_destroy": (C.c_int, [_vp]),
    "b2_ivox_clear": (C.c_int, [_vp]),
    "b2_ivox_set_lru": (C.c_int, [_vp, C.c_size_t, C.c_size_t]),
    "b2_ivox_set_neighbor_voxel_mode": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_insertion_setting": (C.c_int, [_vp, C.c_double, C.c_int]),
    "b2_ivox_insert": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, C.c_size_t]),
    "b2_ivox_insert_cloud": (C.c_int, [_vp, _vp, _dp]),
    "b2_ivox_insert_with_intensities": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, _dp, C.c_size_t]),
    "b2_ivox_download_intensities": (C.c_int, [_vp, _dp]),
    "b2_ivox_get_info": (C.c_int, [_vp, C.POINTER(IvoxInfo)]),
    "b2_ivox_download": (C.c_int, [_vp, _ip, _ip, _dp, _dp]),
    "b2_ivox_knn": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_int, C.c_double, _lp, _dp]),
    "b2_ivox_create_covariance_estimation": (C.c_int, [_vp, C.c_double, _pp]),
    "b2_ivox_set_num_neighbors": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_min_num_neighbors": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_warmup_cycles": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_lowrate_cycles": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_remove_invalid_age_thresh": (C.c_int, [_vp, C.c_int]),
    "b2_ivox_set_eig_stddev_thresh_scale": (C.c_int, [_vp, C.c_double]),
    "b2_ivox_knn_force": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_int, C.c_double, _lp, _dp]),
    "b2_ivox_download_state": (C.c_int, [_vp, _ip, _ip, _dp, C.POINTER(C.c_uint64), _dp, _dp]),
    "b2_ivox_eig_stats": (C.c_int, [_vp, C.POINTER(C.c_uint64), _dp, _dp]),
    "b2_ivox_insert_timings": (C.c_int, [_vp, _dp]),
    "b2_kdtree_create": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, _pp]),
    "b2_kdtree_create_from_cloud": (C.c_int, [_vp, _pp]),
    "b2_kdtree_destroy": (C.c_int, [_vp]),
    "b2_kdtree_knn1": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_double, _lp, _dp]),
    "b2_kdtree_knn": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_int, C.c_double, _lp, _dp]),
    "b2_kdtree_radius_search": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_double, C.c_size_t, C.POINTER(C.c_uint64), C.c_size_t, _lp, _dp]),
    "b2_estimate_covariances": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_int, _dp, _dp]),
    "b2_kdtree_estimate_covariances": (C.c_int, [_vp, C.c_int, _dp, _dp]),
    "b2_estimate_normals_from_covs": (C.c_int, [_vp, _dp, C.c_int, _dp, C.c_int, C.c_size_t, _dp]),
    "b2_estimate_normals": (C.c_int, [_vp, _dp, C.c_int, C.c_size_t, C.c_int, _dp, _dp, _dp]),
    "b2_kdtree_estimate_normals": (C.c_int, [_vp, C.c_int, _dp, _dp, _dp]),
    "b2_features_create": (C.c_int, [_vp, _dp, C.c_size_t, C.c_int, _pp]),
    "b2_features_download": (C.c_int, [_vp, _dp]),
    "b2_features_get_info": (C.c_int, [_vp, C.POINTER(FeaturesInfo)]),
    "b2_features_destroy": (C.c_int, [_vp]),
    "b2_features_create_fpfh": (C.c_int, [_vp, _vp, C.c_double, C.c_size_t, _pp]),
    "b2_features_create_fpfh_at": (C.c_int, [_vp, _vp, C.c_double, C.c_size_t, _lp, C.c_size_t, _pp]),
    "b2_features_create_pfh": (C.c_int, [_vp, _vp, C.c_double, C.c_size_t, _lp, C.c_size_t, _pp]),
    "b2_features_nearest": (C.c_int, [_vp, _vp, _lp, _dp]),
    "b2_estimate_pose_ransac": (C.c_int, [_vp, _vp, _vp, _vp, C.POINTER(RansacParams), C.POINTER(RegistrationResultC), _ip]),
    "b2_estimate_pose_gnc": (C.c_int, [_vp, _vp, _vp, _vp, C.POINTER(GncParams), C.POINTER(RegistrationResultC), _lp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b2_region_growing_create": (C.c_int, [_vp, _vp, _dp, C.c_double, C.c_double, C.c_double, C.c_int, _pp]),
    "b2_region_growing_update": (C.c_int, [_vp, C.c_int, _ip]),
    "b2_region_growing_get": (C.c_int, [_vp, C.POINTER(C.c_uint64), _lp]),
    "b2_region_growing_destroy": (C.c_int, [_vp]),
    "b2_min_cut": (C.c_int, [_vp, _vp, C.c_int64, _dp, C.POINTER(MinCutParamsC), C.POINTER(MinCutResultC), _lp, _lp]),
    "b2_occgrid_create": (C.c_int, [_vp, C.c_double, _pp]),
    "b2_occgrid_destroy": (C.c_int, [_vp]),
    "b2_occgrid_get_info": (C.c_int, [_vp, C.POINTER(OccGridInfo)]),
    "b2_occgrid_insert": (C.c_int, [_vp, _vp, _dp]),
    "b2_occgrid_overlap": (C.c_int, [_vp, _vp, _dp, C.c_size_t, C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)]),
    "b2_occgrid_free_rays": (C.c_int, [_vp, _vp, _dp]),
    "b2_occgrid_download": (C.c_int, [_vp, _ip]),
    "b2_raycast": (C.c_int, [_vp, _dp, _dp, C.c_size_t, C.c_double, C.POINTER(C.c_uint64), C.c_size_t, _ip]),
    "b2_vgicp_factor_create": (C.c_int, [_vp, _vp, _vp, _pp]),
    "b2_gicp_factor_create": (C.c_int, [_vp, _vp, _vp, _vp, _pp]),
    "b2_icp_factor_create": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, _dp, _pp]),
    "b2_gicp_ivox_factor_create": (C.c_int, [_vp, _vp, _vp, _pp]),
    "b2_icp_ivox_factor_create": (C.c_int, [_vp, _vp, _vp, C.c_int, _pp]),
    "b2_factor_destroy": (C.c_int, [_vp]),
    "b2_factor_set_max_correspondence_distance": (C.c_int, [_vp, C.c_double]),
    "b2_factor_set_correspondence_update_tolerance": (C.c_int, [_vp, C.c_double, C.c_double]),
    "b2_factor_set_enable_surface_validation": (C.c_int, [_vp, C.c_int]),
    "b2_factor_num_points": (C.c_size_t, [_vp]),
    "b2_factor_set_enable_offloading": (C.c_int, [_vp, C.c_int]),
    "b2_factor_device_bytes": (C.c_int, [_vp, C.POINTER(C.c_uint64)]),
    "b2_factor_correspondences": (C.c_int, [_vp, _lp]),
    "b2_factor_linearize": (C.c_int, [_vp, _dp, _dp]),
    "b2_factor_error": (C.c_int, [_vp, _dp, _dp]),
    "b2_factor_issue_linearize": (C.c_int, [_vp, _dp, _vp]),
    "b2_factor_issue_error": (C.c_int, [_vp, _dp, _vp]),
    "b2_factor_sync": (C.c_int, [_vp]),
    "b2_factor_set_create": (C.c_int, [_vp, _pp, C.c_size_t, _pp]),
    "b2_factor_set_destroy": (C.c_int, [_vp]),
    "b2_factor_set_size": (C.c_size_t, [_vp]),
    "b2_factor_set_linearize": (C.c_int, [_vp, _dp, _dp]),
    "b2_factor_set_error": (C.c_int, [_vp, _dp, _dp]),
    "b2_factor_set_linearize_device": (C.c_int, [_vp, _vp, _vp]),
    "b2_factor_set_error_device": (C.c_int, [_vp, _vp, _vp]),
    "b2_factor_set_issue_linearize": (C.c_int, [_vp, _dp, _vp]),
    "b2_factor_set_issue_error": (C.c_int, [_vp, _dp, _vp]),
    "b2_factor_set_sync": (C.c_int, [_vp]),
    "b2_factor_set_store_linearized": (C.c_int, [_vp, _dp]),
    "b2_factor_set_store_errors": (C.c_int, [_vp, _dp]),
    "b2_exchange_create": (C.c_int, [_vp, C.c_int, C.c_int, C.c_size_t, _pp]),
    "b2_exchange_destroy": (C.c_int, [_vp]),
    "b2_exchange_export": (C.c_int, [_vp, C.POINTER(C.c_ubyte)]),
    "b2_exchange_import": (C.c_int, [_vp, C.c_int, C.POINTER(C.c_ubyte)]),
    "b2_exchange_enable_peer": (C.c_int, [_vp, C.c_int, _vp]),
    "b2_exchange_linearize": (C.c_int, [_vp, _vp, _dp, C.c_size_t, C.c_uint]),
    "b2_exchange_linearize_host": (C.c_int, [_vp, _vp, _dp, C.c_size_t, C.c_uint, _dp]),
    "b2_exchange_records": (_vp, [_vp, C.c_uint]),
    "b2_exchange_error": (C.c_int, [_vp, _vp, _dp, C.c_size_t, C.c_uint]),
    "b2_exchange_error_host": (C.c_int, [_vp, _vp, _dp, C.c_size_t, C.c_uint, _dp]),
    "b2_exchange_errors": (_vp, [_vp, C.c_uint]),
    "b2_exchange_barrier": (C.c_int, [_vp]),
    "b2_factor_set_launch_count": (C.c_uint64, [_vp]),
    "b2_lm_params_default": (None, [C.POINTER(LmParamsC)]),
    "b2_lm_graph_trace_doubles": (C.c_size_t, [C.c_size_t]),
    "b2_factor_set_optimize_poses": (C.c_int, [_vp, C.c_size_t, _ip, _dp, C.POINTER(PosePriorC), C.c_size_t, _dp, C.POINTER(LmParamsC), _dp, C.POINTER(LmSummaryC),
                                               C.POINTER(LmGraphTraceEntryC), _dp, C.c_size_t, C.POINTER(C.c_size_t)]),
    "b2_factor_set_lm_graph_builds": (C.c_uint64, [_vp]),
}


def lib():
    """Loads libb2points.so; raises if it has not been built (run `python -m gtsam_points_b200.build`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: the CUDA extension has not been built "
                "(python -m gtsam_points_b200.build).  There is no CPU fallback."
            )
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status):
    if status != 0:
        raise B2Error(status, lib().b2_last_error().decode("utf-8", "replace"))


def dptr(a: np.ndarray):
    return a.ctypes.data_as(_dp)


def as_f64(a, shape_tail=None):
    a = np.ascontiguousarray(a, dtype=np.float64)
    return a


def unpack_linearized(buf):
    """128-double record -> dict (same keys as the oracle's unpacker)."""
    buf = np.asarray(buf, dtype=np.float64)
    return dict(
        H_target=buf[0:36].reshape(6, 6).copy(),
        H_source=buf[36:72].reshape(6, 6).copy(),
        H_target_source=buf[72:108].reshape(6, 6).copy(),
        b_target=buf[108:114].copy(),
        b_source=buf[114:120].copy(),
        error=float(buf[120]),
        num_inliers=int(buf[121]),
    )
