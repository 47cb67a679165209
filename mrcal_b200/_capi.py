"""ctypes binding of libmrcal_b200.so (include/mrcal_b200.h).

This plays the role of the reference's mrcal-pywrap.c for the calibration-solve
path: it converts Python arguments to the C structures and calls the C-ABI. The
library is REQUIRED: there is no Python/CPU fallback. If the .so is missing (or
was built for something else) importing this module raises immediately.

Every entry point is typed from one table, SIGNATURES, on two handles of the
library:
- `lib` is the C ABI as declared: a false or NULL return comes back as it is, for
  code that examines the ABI itself.
- `checked` is what the package calls: a function that reports failure by
  returning false or NULL raises RuntimeError with the library's message instead,
  so callers call checked.<name>(...) without checking the result.
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

if not os.path.exists(LIBPATH):
    raise ImportError(
        f"{LIBPATH} not found. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
        "(or `make -C mrcal_b200/csrc`). mrcal_b200 has no fallback implementation.")

lib = C.CDLL(LIBPATH)
checked = C.CDLL(LIBPATH)   # the same library; its own function objects carry the failure check


class _Raises:
    """A return type whose false (bool) or NULL (pointer) value means failure: a call through `checked` raises
    RuntimeError("<name>() failed: <mrcal_b200_last_error()>")"""

    def __init__(self, ctype):
        self.ctype = ctype


OK, HANDLE = _Raises(C.c_bool), _Raises(C.c_void_p)
# C types as ctypes sees them. Every pointer is a c_void_p, which takes None, an address, byref(), a ctypes array
# or bytes; mrcal_lensmodel_type_t is an int
P, I, D, B, U16, SIZE, SEL = C.c_void_p, C.c_int, C.c_double, C.c_bool, C.c_uint16, C.c_size_t, Selections
# (Ncameras_intrinsics, Ncameras_extrinsics, Nframes, Npoints, Npoints_fixed, Nobservations_board,
#  problem_selections, lensmodel): the layout functions' common tail
_COUNTS = [I] * 6 + [SEL, P]
# intrinsics .. problem_selections of mrcal_optimizer_callback(), mrcal_optimize() and
# mrcal_b200_problem_create_triangulated(): api._Inputs.c_problem() fills it
_PROBLEM = [P] * 5 + [I] * 5 + [P, P, I, I, P, I, P, P, P, P, SEL]

# name -> (return type, argument types) of every function include/mrcal_b200.h declares, in its order. A bool or
# pointer return that is not OK or HANDLE is a status the caller reads itself
SIGNATURES = {
    # part 1b: lens models
    "_mrcal_precompute_lensmodel_data": (None, [P, P]),
    # false leaves lensmodel->type saying why: api._lensmodel() words the reference's messages from it
    "mrcal_lensmodel_from_name": (B, [P, P]),
    "mrcal_lensmodel_type_from_name": (I, [P]),
    "mrcal_lensmodel_name": (OK, [P, I, P]),
    "mrcal_lensmodel_name_unconfigured": (C.c_char_p, [P]),
    "mrcal_lensmodel_metadata": (Metadata, [P]),
    "mrcal_lensmodel_num_params": (I, [P]),
    "mrcal_supported_lensmodel_names": (C.POINTER(C.c_char_p), []),
    "mrcal_knots_for_splined_models": (OK, [P, P, P]),
    # part 1c: state and measurement layout
    "mrcal_num_intrinsics_optimization_params": (I, [SEL, P]),
    "mrcal_num_states": (I, _COUNTS),
    "mrcal_num_states_intrinsics": (I, [I, SEL, P]),
    "mrcal_num_states_extrinsics": (I, [I, SEL]),
    "mrcal_num_states_frames": (I, [I, SEL]),
    "mrcal_num_states_points": (I, [I, I, SEL]),
    "mrcal_num_states_calobject_warp": (I, [SEL, I]),
    "mrcal_state_index_intrinsics": (I, [I] + _COUNTS),
    "mrcal_state_index_extrinsics": (I, [I] + _COUNTS),
    "mrcal_state_index_frames": (I, [I] + _COUNTS),
    "mrcal_state_index_points": (I, [I] + _COUNTS),
    "mrcal_state_index_calobject_warp": (I, _COUNTS),
    "mrcal_measurement_index_boards": (I, [I] * 5),
    "mrcal_num_measurements_boards": (I, [I] * 3),
    "mrcal_measurement_index_points": (I, [I] * 5),
    "mrcal_num_measurements_points": (I, [I]),
    "mrcal_measurement_index_points_triangulated": (I, [I, I, I, P, I, I, I]),
    "mrcal_num_measurements_points_triangulated_initial_Npoints": (I, [P, I, I]),
    "mrcal_num_measurements_points_triangulated": (I, [P, I]),
    "mrcal_measurement_index_regularization": (I, [P] + [I] * 10 + [SEL, P]),
    "mrcal_num_measurements_regularization": (I, _COUNTS),
    "mrcal_num_measurements": (I, [I, I, P] + [I] * 8 + [SEL, P]),
    "_mrcal_num_j_nonzero": (I, [I, I, P] + [I] * 8 + [P, P, SEL, P]),
    "mrcal_pack_solver_state_vector": (None, [P] + _COUNTS),
    "mrcal_unpack_solver_state_vector": (None, [P] + _COUNTS),
    "mrcal_corresponding_icam_extrinsics": (OK, [P, I, I, I, I, P, I, P]),
    # part 1d: projection, stereo, the hot path
    "mrcal_project": (OK, [P, P, P, P, I, P, P]),
    "mrcal_unproject": (OK, [P, P, I, P, P]),
    "mrcal_b200_unproject_with_gradients": (OK, [P] * 4 + [I, P, P, B]),
    "mrcal_b200_project": (OK, [P, I, I] + [P] * 8),
    "mrcal_b200_project_device": (OK, [P, I, I] + [P] * 9),
    "mrcal_b200_model_resolution__deg_pixel": (OK, [P, P, I, P, P, I]),
    "mrcal_rectified_resolution": (OK, [P] * 7 + [I]),
    "mrcal_rectified_system2": (OK, [P] * 8 + [D] + [P] * 4 + [I] + [B] * 4),
    "mrcal_rectified_system": (OK, [P] * 12 + [I] + [B] * 4),
    "mrcal_rectification_maps": (OK, [P] * 7 + [I, P, P, P]),
    "mrcal_stereo_range_sparse": (OK, [P, P, P, I, D, D, I, P, D]),
    "mrcal_stereo_range_dense": (OK, [P, P, U16, U16, U16, I, P, D]),
    "mrcal_optimizer_callback": (OK, [P, I, P, I, P] + _PROBLEM + [P, D, I, I, B]),
    # failure is a negative rms_reproj_error__pixels
    "mrcal_optimize": (Stats, [P, I, P, I] + _PROBLEM + [P, D, I, I, B, B]),
    # part 2: extensions
    "mrcal_b200_version": (C.c_char_p, []),
    "mrcal_b200_device_count": (I, []),
    "mrcal_b200_last_error": (C.c_char_p, []),
    "mrcal_b200_default_solver_parameters": (None, [P]),
    "mrcal_b200_problem_create": (HANDLE, [P] * 5 + [I] * 5 + [P, P, I, I, P, P, P, P, SEL, D, I, I]),
    "mrcal_b200_problem_create_triangulated": (HANDLE, _PROBLEM + [D, I, I]),
    "mrcal_b200_problem_destroy": (None, [P]),
    "mrcal_b200_problem_num_states": (I, [P]),
    "mrcal_b200_problem_num_measurements": (I, [P]),
    "mrcal_b200_problem_num_j_nonzero": (I, [P]),
    "mrcal_b200_problem_reset": (OK, [P, P]),
    "mrcal_b200_problem_upload": (OK, [P] * 8),
    "mrcal_b200_problem_callback": (OK, [P] * 6),
    "mrcal_b200_problem_optimize": (OK, [P] * 4),
    "mrcal_b200_problem_reduced_system": (OK, [P, D, P, P, P, P]),
    "mrcal_b200_problem_reduced_system_fused": (OK, [P, D, P, P, P, P]),
    "mrcal_b200_problem_cauchy_denominator": (OK, [P, B, P]),
    "mrcal_b200_problem_download": (OK, [P] * 9),
    "mrcal_b200_problem_triangulated_outliers": (I, [P, P, I]),
    "mrcal_b200_problem_drt_cross_reprojection__dbpacked": (OK, [P, I, P]),
    "mrcal_b200_problem_projection_uncertainty": (OK, [P, I, I, B, P, I, D, P, P]),
    "mrcal_b200_problem_projection_uncertainty_cameras": (OK, [P, P, P, I, I, B, P, D, P, P]),
    "mrcal_b200_problem_observed_pixel_uncertainty": (OK, [P, P]),
    "mrcal_b200_problem_regional_statistics": (OK, [P, P, I, I, I, P, P, B, P, P]),
    "mrcal_b200_implied_Rt10__from_unprojections": (OK, [P, P, I, P, I, P, P, B, P, D]),
    "mrcal_b200_projection_diff": (OK, [P, P, P, P, I, P, I, P, I, P, P, P, P, D, B]),
    "mrcal_b200_stereo_pair_reproject": (OK, [P, P, P, I, I, P, P, P, D]),
    "mrcal_b200_stereo_unproject": (OK, [P, P, P, U16, U16, U16, P, P, P, I, I, D, D, I, P, D]),
    "mrcal_b200_image_transformation_map": (OK, [P, I, I] + [P] * 7 + [D, P, I]),
    "mrcal_b200_is_within_region": (OK, [P, P, I, P, I]),
    "mrcal_b200_transform_image": (OK, [P, P] + [I] * 5 + [P] + [I] * 4 + [P]),
    "mrcal_b200_transform_image_device": (OK, [P, P] + [I] * 5 + [P] + [I] * 4 + [P, P]),
    "mrcal_b200_match_feature": (OK, [P, P, P, I, I, I, P] + [I] * 4 + [P, P] + [I] * 6),
    "mrcal_b200_match_feature_device": (OK, [P, P, P, I, I, I, P] + [I] * 4 + [P, P] + [I] * 6 + [P]),
    "mrcal_b200_poseutils": (OK, [I] * 3 + [P] * 8),
    "mrcal_b200_poseutils_device": (OK, [I] * 3 + [P] * 9),
    "mrcal_b200_triangulate": (OK, [I] * 3 + [P] * 11),
    "mrcal_b200_triangulate_device": (OK, [I] * 3 + [P] * 12),
    "mrcal_b200_synthesize_board_observations": (OK, [P, P, P, P, I, P, I, I, P, P, P, P]),
    "mrcal_b200_problem_corners": (OK, [P, P, P, P, I, P, I, P, I, P, I, P, I, P, I, P, P, I]),
    # failure is a negative time
    "mrcal_b200_problem_time_callback": (D, [P, I, B]),
    "mrcal_b200_nccl_get_unique_id": (OK, [P]),
    "mrcal_b200_nccl_comm_init": (OK, [P, I, I, I]),
    "mrcal_b200_nccl_comm_destroy": (None, []),
    "mrcal_b200_problem_set_sharding": (OK, [P, I, I, I, I]),
    "mrcal_b200_factorization_create": (HANDLE, [P, P, P, I, I]),
    "mrcal_b200_factorization_destroy": (None, [P]),
    "mrcal_b200_factorization_solve_xt_JtJ_bt": (OK, [P, P, P, I]),
    "mrcal_b200_factorization_solve_sys": (OK, [P, P, P, I, I]),
    "mrcal_b200_factorization_rcond": (D, [P]),
    # NULL also when J'J is not positive definite, which optimizer_callback() does not treat as an error
    "mrcal_b200_factorization_create_from_last_callback": (P, []),
    "mrcal_b200_csr_create": (HANDLE, [P, P, P, I, I]),
    "mrcal_b200_csr_destroy": (None, [P]),
    "mrcal_b200_csr_Jt_x": (OK, [P, P, P]),
    "mrcal_b200_csr_A_Jt_J_At": (OK, [P, P, P, I, I]),
}

# Not public: test and timing aids defined extern "C" in csrc/factorization.cu, nccl.cu and eval.cu, with no header.
# Their signatures may change with the code they probe
DEBUG_SIGNATURES = {
    "mrcal_b200_debug_cholesky": (OK, [P, I, I, I, P, P, P, P]),
    "mrcal_b200_debug_chol_solve": (OK, [P, P, I, I, P, I, I, I]),
    "mrcal_b200_debug_time_cholesky": (D, [I, I, I]),
    "mrcal_b200_debug_spine_stamps": (OK, [I, P, I]),
    "mrcal_b200_debug_potrf_stamps": (OK, [P]),
    "mrcal_b200_debug_time_allreduce": (D, [SIZE, I]),
    "mrcal_b200_debug_triangulated_error": (OK, [P, I, P]),
}

# every symbol include/mrcal_b200.h declares; tests check the .so exports each
EXPORTED_SYMBOLS = tuple(SIGNATURES)


def _raise_on_failure(result, func, args):
    if not result:
        raise RuntimeError(f"{func.__name__}() failed: {last_error()}")
    return result


for _name, (_ret, _args) in {**SIGNATURES, **DEBUG_SIGNATURES}.items():
    for _f in (getattr(lib, _name), getattr(checked, _name)):
        _f.argtypes = _args
        _f.restype = _ret.ctype if isinstance(_ret, _Raises) else _ret
    if isinstance(_ret, _Raises):
        getattr(checked, _name).errcheck = _raise_on_failure


def last_error():
    return lib.mrcal_b200_last_error().decode(errors="replace")
