"""ctypes binding of libmrcal_b200.so (include/mrcal_b200.h).

This plays the role of the reference's mrcal-pywrap.c for the calibration-solve
path: it converts Python arguments to the C structures and calls the C-ABI. The
library is REQUIRED: there is no Python/CPU fallback. If the .so is missing (or
was built for something else) importing this module raises immediately.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBPATH = os.path.join(_HERE, "libmrcal_b200.so")


class Lensmodel(C.Structure):
    """mrcal_lensmodel_t: int type @0, config union @8 (16 bytes)."""
    _fields_ = [("type", C.c_int), ("_pad", C.c_int), ("config", C.c_uint8 * 8)]


class Selections(C.Structure):
    """mrcal_problem_selections_t: one byte of bit flags, passed by value."""
    _fields_ = [("bits", C.c_uint8)]


class Metadata(C.Structure):
    _fields_ = [("bits", C.c_uint8)]


class Stats(C.Structure):
    _fields_ = [("rms_reproj_error__pixels", C.c_double),
                ("Noutliers_board", C.c_int),
                ("Noutliers_triangulated_point", C.c_int)]


class ObservationPointTriangulated(C.Structure):
    """mrcal_observation_point_triangulated_t (types.h:243-263): bit 0 of `bits` = last_in_set, bit 1 = outlier."""
    _fields_ = [("icam_intrinsics", C.c_int), ("icam_extrinsics", C.c_int),
                ("bits", C.c_uint8), ("px", C.c_double * 3)]


class Sparse(C.Structure):
    """mrcal_b200_sparse_t (== the public cholmod_sparse layout)."""
    _fields_ = [("nrow", C.c_size_t), ("ncol", C.c_size_t), ("nzmax", C.c_size_t),
                ("p", C.c_void_p), ("i", C.c_void_p), ("nz", C.c_void_p),
                ("x", C.c_void_p), ("z", C.c_void_p),
                ("stype", C.c_int), ("itype", C.c_int), ("xtype", C.c_int),
                ("dtype", C.c_int), ("sorted", C.c_int), ("packed", C.c_int)]


class ImageUint16(C.Structure):
    """mrcal_image_uint16_t (image.h:68-80): w, h in pixels, stride in bytes"""
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("stride", C.c_int), ("data", C.c_void_p)]


class ImageDouble(C.Structure):
    """mrcal_image_double_t (image.h:68-80)"""
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("stride", C.c_int), ("data", C.c_void_p)]


class SolverParameters(C.Structure):
    _fields_ = [("max_iterations", C.c_int),
                ("trustregion0", C.c_double),
                ("trustregion_decrease_factor", C.c_double),
                ("trustregion_decrease_threshold", C.c_double),
                ("trustregion_increase_factor", C.c_double),
                ("trustregion_increase_threshold", C.c_double),
                ("Jt_x_threshold", C.c_double),
                ("update_threshold", C.c_double),
                ("trustregion_threshold", C.c_double)]


class SolveInfo(C.Structure):
    _fields_ = [("Niterations", C.c_int), ("Nevaluations", C.c_int), ("Nfactorizations", C.c_int),
                ("Nouter", C.c_int), ("Nreduced", C.c_int), ("Nkernel_launches", C.c_int), ("Nsyncs", C.c_int), ("Ncollectives", C.c_int),
                ("norm2_x_initial", C.c_double), ("norm2_x_final", C.c_double),
                ("ms_total", C.c_double), ("ms_evaluate", C.c_double), ("ms_assemble", C.c_double),
                ("ms_factor", C.c_double), ("ms_solve", C.c_double), ("lambda_final", C.c_double)]

    def asdict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


SELECTION_BITS = ("do_optimize_intrinsics_core",
                  "do_optimize_intrinsics_distortions",
                  "do_optimize_extrinsics",
                  "do_optimize_frames",
                  "do_optimize_calobject_warp",
                  "do_apply_regularization",
                  "do_apply_outlier_rejection",
                  "do_apply_regularization_unity_cam01")

# every symbol include/mrcal_b200.h declares; tests check the .so exports each
EXPORTED_SYMBOLS = (
    "_mrcal_precompute_lensmodel_data", "mrcal_project", "mrcal_unproject", "mrcal_b200_problem_create_triangulated",
    "mrcal_b200_unproject_with_gradients", "mrcal_b200_model_resolution__deg_pixel", "mrcal_b200_stereo_pair_reproject",
    "mrcal_lensmodel_from_name", "mrcal_lensmodel_type_from_name", "mrcal_lensmodel_name",
    "mrcal_lensmodel_name_unconfigured", "mrcal_lensmodel_metadata", "mrcal_lensmodel_num_params",
    "mrcal_supported_lensmodel_names", "mrcal_knots_for_splined_models",
    "mrcal_num_intrinsics_optimization_params", "mrcal_num_states",
    "mrcal_num_states_intrinsics", "mrcal_num_states_extrinsics", "mrcal_num_states_frames",
    "mrcal_num_states_points", "mrcal_num_states_calobject_warp",
    "mrcal_state_index_intrinsics", "mrcal_state_index_extrinsics", "mrcal_state_index_frames",
    "mrcal_state_index_points", "mrcal_state_index_calobject_warp",
    "mrcal_measurement_index_boards", "mrcal_num_measurements_boards",
    "mrcal_measurement_index_points", "mrcal_num_measurements_points",
    "mrcal_measurement_index_points_triangulated",
    "mrcal_num_measurements_points_triangulated_initial_Npoints",
    "mrcal_num_measurements_points_triangulated",
    "mrcal_measurement_index_regularization", "mrcal_num_measurements_regularization",
    "mrcal_num_measurements", "_mrcal_num_j_nonzero",
    "mrcal_pack_solver_state_vector", "mrcal_unpack_solver_state_vector",
    "mrcal_corresponding_icam_extrinsics",
    "mrcal_optimizer_callback", "mrcal_optimize",
    "mrcal_b200_version", "mrcal_b200_device_count", "mrcal_b200_last_error",
    "mrcal_b200_default_solver_parameters",
    "mrcal_b200_problem_create", "mrcal_b200_problem_destroy",
    "mrcal_b200_problem_num_states", "mrcal_b200_problem_num_measurements",
    "mrcal_b200_problem_num_j_nonzero", "mrcal_b200_problem_reset", "mrcal_b200_problem_upload",
    "mrcal_b200_problem_callback", "mrcal_b200_problem_optimize", "mrcal_b200_problem_download",
    "mrcal_b200_problem_reduced_system", "mrcal_b200_problem_reduced_system_fused",
    "mrcal_b200_problem_time_callback",
    "mrcal_b200_problem_triangulated_outliers",
    "mrcal_b200_problem_drt_cross_reprojection__dbpacked",
    "mrcal_b200_problem_projection_uncertainty", "mrcal_b200_problem_projection_uncertainty_cameras",
    "mrcal_b200_problem_regional_statistics", "mrcal_b200_is_within_region",
    "mrcal_b200_implied_Rt10__from_unprojections", "mrcal_b200_projection_diff",
    "mrcal_rectified_resolution", "mrcal_rectified_system2", "mrcal_rectified_system", "mrcal_rectification_maps",
    "mrcal_stereo_range_sparse", "mrcal_stereo_range_dense", "mrcal_b200_stereo_unproject",
    "mrcal_b200_image_transformation_map", "mrcal_b200_transform_image", "mrcal_b200_transform_image_device",
    "mrcal_b200_match_feature", "mrcal_b200_match_feature_device",
    "mrcal_b200_poseutils", "mrcal_b200_poseutils_device",
    "mrcal_b200_nccl_get_unique_id", "mrcal_b200_nccl_comm_init", "mrcal_b200_nccl_comm_destroy",
    "mrcal_b200_problem_set_sharding",
    "mrcal_b200_factorization_create", "mrcal_b200_factorization_destroy",
    "mrcal_b200_factorization_solve_xt_JtJ_bt", "mrcal_b200_factorization_solve_sys", "mrcal_b200_factorization_rcond",
    "mrcal_b200_factorization_create_from_last_callback",
    "mrcal_b200_csr_create", "mrcal_b200_csr_destroy", "mrcal_b200_csr_Jt_x", "mrcal_b200_csr_A_Jt_J_At",
)

if not os.path.exists(LIBPATH):
    raise ImportError(
        f"{LIBPATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(or `make -C mrcal_b200/csrc`). mrcal_b200 has no fallback implementation.")

lib = C.CDLL(LIBPATH)

_int_fns = [s for s in EXPORTED_SYMBOLS
            if s.startswith(("mrcal_num_", "mrcal_state_index_", "mrcal_measurement_index_", "_mrcal_num_"))]
for _n in _int_fns + ["mrcal_lensmodel_num_params", "mrcal_lensmodel_type_from_name", "mrcal_b200_device_count",
                      "mrcal_b200_problem_num_states", "mrcal_b200_problem_num_measurements",
                      "mrcal_b200_problem_num_j_nonzero"]:
    getattr(lib, _n).restype = C.c_int
for _n in ["mrcal_lensmodel_from_name", "mrcal_lensmodel_name", "mrcal_knots_for_splined_models",
           "mrcal_corresponding_icam_extrinsics", "mrcal_optimizer_callback",
           "mrcal_b200_problem_reset", "mrcal_b200_problem_upload", "mrcal_b200_problem_callback",
           "mrcal_b200_problem_optimize", "mrcal_b200_problem_download", "mrcal_b200_problem_reduced_system",
           "mrcal_b200_problem_reduced_system_fused", "mrcal_b200_nccl_get_unique_id", "mrcal_b200_nccl_comm_init", "mrcal_b200_problem_set_sharding",
           "mrcal_b200_factorization_solve_xt_JtJ_bt", "mrcal_b200_factorization_solve_sys", "mrcal_project", "mrcal_unproject"]:
    getattr(lib, _n).restype = C.c_bool
lib.mrcal_lensmodel_metadata.restype = Metadata
lib.mrcal_lensmodel_name_unconfigured.restype = C.c_char_p
lib.mrcal_supported_lensmodel_names.restype = C.POINTER(C.c_char_p)
lib.mrcal_optimize.restype = Stats
lib.mrcal_b200_version.restype = C.c_char_p
lib.mrcal_b200_last_error.restype = C.c_char_p
lib.mrcal_b200_problem_create.restype = C.c_void_p
lib.mrcal_b200_problem_create_triangulated.restype = C.c_void_p
lib.mrcal_b200_problem_destroy.restype = None
lib.mrcal_b200_problem_time_callback.restype = C.c_double
lib.mrcal_b200_problem_triangulated_outliers.restype = C.c_int
lib.mrcal_b200_problem_drt_cross_reprojection__dbpacked.restype = C.c_bool
lib.mrcal_b200_problem_drt_cross_reprojection__dbpacked.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
lib.mrcal_b200_problem_projection_uncertainty.restype = C.c_bool
lib.mrcal_b200_problem_projection_uncertainty.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_bool, C.c_void_p, C.c_int,
                                                           C.c_double, C.c_void_p, C.c_void_p]
lib.mrcal_b200_problem_projection_uncertainty_cameras.restype = C.c_bool
lib.mrcal_b200_problem_projection_uncertainty_cameras.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                                   C.c_bool, C.c_void_p, C.c_double, C.c_void_p,
                                                                   C.c_void_p]
lib.mrcal_b200_problem_regional_statistics.restype = C.c_bool
lib.mrcal_b200_problem_regional_statistics.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                                       C.c_void_p, C.c_bool, C.c_void_p, C.c_void_p]
lib.mrcal_b200_is_within_region.restype = C.c_bool
lib.mrcal_b200_is_within_region.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int]
lib.mrcal_b200_implied_Rt10__from_unprojections.restype = C.c_bool
lib.mrcal_b200_implied_Rt10__from_unprojections.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                                             C.c_void_p, C.c_void_p, C.c_bool, C.c_void_p, C.c_double]
lib.mrcal_b200_projection_diff.restype = C.c_bool
lib.mrcal_b200_projection_diff.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int,
                                           C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_double, C.c_bool]
lib.mrcal_b200_unproject_with_gradients.restype = C.c_bool
lib.mrcal_b200_unproject_with_gradients.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_void_p, C.c_void_p, C.c_bool]
lib.mrcal_b200_model_resolution__deg_pixel.restype = C.c_bool
lib.mrcal_b200_model_resolution__deg_pixel.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
lib.mrcal_b200_stereo_pair_reproject.restype = C.c_bool
lib.mrcal_b200_stereo_pair_reproject.argtypes = [C.c_void_p] * 3 + [C.c_int] * 2 + [C.c_void_p] * 3 + [C.c_double]
for _n in ["mrcal_rectified_resolution", "mrcal_rectified_system2", "mrcal_rectified_system", "mrcal_rectification_maps",
           "mrcal_stereo_range_sparse", "mrcal_stereo_range_dense", "mrcal_b200_stereo_unproject"]:
    getattr(lib, _n).restype = C.c_bool
lib.mrcal_rectified_system2.argtypes = [C.c_void_p] * 8 + [C.c_double] + [C.c_void_p] * 4 + [C.c_int] + [C.c_bool] * 4
lib.mrcal_stereo_range_sparse.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p,
                                                               C.c_double]
lib.mrcal_stereo_range_dense.argtypes = [C.c_void_p, C.c_void_p, C.c_uint16, C.c_uint16, C.c_uint16, C.c_int,
                                         C.c_void_p, C.c_double]
lib.mrcal_b200_stereo_unproject.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint16, C.c_uint16, C.c_uint16,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_double,
                                            C.c_double, C.c_int, C.c_void_p, C.c_double]
for _n in ["mrcal_b200_image_transformation_map", "mrcal_b200_transform_image", "mrcal_b200_transform_image_device"]:
    getattr(lib, _n).restype = C.c_bool
lib.mrcal_b200_image_transformation_map.argtypes = [C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 7 + \
                                                   [C.c_double, C.c_void_p, C.c_int]
lib.mrcal_b200_transform_image.argtypes = [C.c_void_p, C.c_void_p] + [C.c_int] * 5 + [C.c_void_p] + [C.c_int] * 4 + \
                                          [C.c_void_p]
lib.mrcal_b200_transform_image_device.argtypes = lib.mrcal_b200_transform_image.argtypes + [C.c_void_p]
for _n in ["mrcal_b200_match_feature", "mrcal_b200_match_feature_device"]:
    getattr(lib, _n).restype = C.c_bool
lib.mrcal_b200_match_feature.argtypes = [C.c_void_p] * 3 + [C.c_int] * 3 + [C.c_void_p] + [C.c_int] * 4 + \
                                        [C.c_void_p] * 2 + [C.c_int] * 6
lib.mrcal_b200_match_feature_device.argtypes = lib.mrcal_b200_match_feature.argtypes + [C.c_void_p]
for _n in ["mrcal_b200_poseutils", "mrcal_b200_poseutils_device"]:
    getattr(lib, _n).restype = C.c_bool
lib.mrcal_b200_poseutils.argtypes = [C.c_int] * 3 + [C.c_void_p] * 8
lib.mrcal_b200_poseutils_device.argtypes = lib.mrcal_b200_poseutils.argtypes + [C.c_void_p]
lib.mrcal_b200_factorization_create_from_last_callback.restype = C.c_void_p
lib.mrcal_b200_csr_create.restype = C.c_void_p
lib.mrcal_b200_csr_destroy.restype = None
lib.mrcal_b200_csr_Jt_x.restype = C.c_bool
lib.mrcal_b200_csr_A_Jt_J_At.restype = C.c_bool
lib.mrcal_b200_factorization_create.restype = C.c_void_p
lib.mrcal_b200_factorization_destroy.restype = None
lib.mrcal_b200_factorization_rcond.restype = C.c_double
lib.mrcal_b200_default_solver_parameters.restype = None
lib.mrcal_b200_nccl_comm_destroy.restype = None
lib.mrcal_pack_solver_state_vector.restype = None
lib._mrcal_precompute_lensmodel_data.restype = None
lib.mrcal_unpack_solver_state_vector.restype = None


def last_error():
    return lib.mrcal_b200_last_error().decode(errors="replace")
