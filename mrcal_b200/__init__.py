"""mrcal_b200: an H100-native (sm_90a CUDA) implementation of mrcal's
calibration solve -- the optimizer_callback residual/Jacobian evaluator and the
trust-region normal-equations solve -- behind mrcal's own Python API for that
path. See DESIGN.md and INTEGRATION.md at the repository root."""
from .api import (  # noqa: F401
    optimize, optimizer_callback, drt_cross_reprojection__dbpacked, projection_uncertainty, worst_direction_stdev,
    sample_imager, sample_imager_unproject, implied_Rt10__from_unprojections, projection_diff,
    Problem, CHOLMOD_factorization,
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
    project_pinhole, unproject_pinhole, project_stereographic, unproject_stereographic,
    project_lonlat, unproject_lonlat, project_latlon, unproject_latlon,
    model_resolution__deg_pixel, stereo_pair_diff,
    _Jt_x, _A_Jt_J_At, _A_Jt_J_At__2,
)
from .seeding import (  # noqa: F401
    seed_stereographic, estimate_monocular_calobject_poses_Rt_tocam, estimate_joint_frame_poses,
)
from .stereo import (  # noqa: F401
    rectified_resolution, rectified_system, rectification_maps, stereo_range, stereo_unproject,
    apply_homography, match_feature,
    TM_SQDIFF, TM_SQDIFF_NORMED, TM_CCORR, TM_CCORR_NORMED, TM_CCOEFF, TM_CCOEFF_NORMED,
    MATCH_OK, MATCH_EDGE_PEAK, MATCH_OUTSIDE_IMAGE1, MATCH_OUTSIDE_IMAGE0, MATCH_SEARCH_TOO_SMALL,
)
from .image_transforms import (  # noqa: F401
    scale_focal__best_pinhole_fit, pinhole_model_for_reprojection, image_transformation_map, transform_image,
    INTER_NEAREST, INTER_LINEAR, BORDER_CONSTANT, BORDER_TRANSPARENT,
)
from .poseutils import (  # noqa: F401
    R_from_r, r_from_R, Rt_from_rt, rt_from_Rt, invert_R, invert_Rt, invert_rt, compose_Rt, compose_r, compose_rt,
    compose_r_tinyr0_gradientr0, compose_r_tinyr1_gradientr1, compose_rt_tinyrt0_gradientrt0,
    compose_rt_tinyrt1_gradientrt1, rotate_point_r, rotate_point_R, transform_point_rt, transform_point_Rt,
    skew_symmetric, R_from_quat, quat_from_R, qt_from_Rt, Rt_from_qt, R_aligned_to_vector,
    identity_R, identity_r, identity_Rt, identity_rt,
)
from .triangulation import (  # noqa: F401
    triangulate_geometric, triangulate_leecivera_l1, triangulate_leecivera_linf, triangulate_leecivera_mid2,
    triangulate_leecivera_wmid2, triangulate_lindstrom, _triangulated_error,
)
from .synthetic_data import (  # noqa: F401
    ref_calibration_object, synthesize_board_observations, hypothesis_board_corner_positions, make_perfect_observations,
)
from .cameramodel import cameramodel, CameramodelParseException  # noqa: F401
from .regions import (  # noqa: F401
    measurements_board, measurements_point, residuals_board, residuals_chessboard, residuals_point,
    close_contour, imagergrid_using, is_within_valid_intrinsics_region, valid_intrinsics_regions,
    _report_regional_statistics, _compute_valid_intrinsics_region,
)
from ._capi import lib as _lib


def version():
    return _lib.mrcal_b200_version().decode()


def device_count():
    return _lib.mrcal_b200_device_count()
