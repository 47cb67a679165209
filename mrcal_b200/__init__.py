"""mrcal_b200: an H100-native (sm_90a CUDA) implementation of mrcal's
calibration solve -- the optimizer_callback residual/Jacobian evaluator and the
trust-region normal-equations solve -- behind mrcal's own Python API for that
path. See DESIGN.md and INTEGRATION.md at the repository root."""
from .api import (  # noqa: F401
    optimize, optimizer_callback, drt_cross_reprojection__dbpacked, Problem, CHOLMOD_factorization,
    lensmodel_num_params, supported_lensmodels, lensmodel_metadata_and_config, knots_for_splined_models,
    state_index_intrinsics, state_index_extrinsics, state_index_frames, state_index_points,
    state_index_calobject_warp,
    num_states, num_states_intrinsics, num_states_extrinsics, num_states_frames, num_states_points,
    num_states_calobject_warp, num_intrinsics_optimization_params,
    measurement_index_boards, measurement_index_points, measurement_index_points_triangulated,
    measurement_index_regularization,
    num_measurements, num_measurements_boards, num_measurements_points,
    num_measurements_points_triangulated, num_measurements_regularization,
    corresponding_icam_extrinsics, pack_state, unpack_state, project, unproject,
    _Jt_x, _A_Jt_J_At, _A_Jt_J_At__2,
)
from .seeding import (  # noqa: F401
    seed_stereographic, estimate_monocular_calobject_poses_Rt_tocam, estimate_joint_frame_poses,
)
from .cameramodel import cameramodel, CameramodelParseException  # noqa: F401
from ._capi import lib as _lib


def version():
    return _lib.mrcal_b200_version().decode()


def device_count():
    return _lib.mrcal_b200_device_count()
