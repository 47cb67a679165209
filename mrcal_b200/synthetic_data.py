"""Synthetic calibration data, with the reference's names, arguments, defaults, return values and refusals
(mrcal/synthetic_data.py and mrcal/utils.py):

    ref_calibration_object()               the board's geometry (host numpy: O(W H))
    synthesize_board_observations()        random board poses that the cameras see, and their projections
    hypothesis_board_corner_positions()    the corners the solver believes each camera saw
    make_perfect_observations()            a problem's observations replaced by exact projections, plus known noise

These are what the standard mrcal experiment uses: make perfect data, add noise of a known sigma, solve again and
compare against projection_uncertainty(). The per-corner work, transforming every board point and projecting it
through its camera's lens, runs on the device (csrc/synthetic_data.cu). The random draws and every operation whose
bits decide what the reference returns stay on the host in numpy, in the reference's order: the board poses
rt_ref_boardcenter + random * noiseradius (a device compiler would contract this into an FMA), the centered board,
the oblique-angle cull and the noise added to the observations. So with the same np.random seed these functions give
the reference's frames and noise, and leave the global RNG in the reference's state.

Inputs and outputs are numpy arrays and mrcal_b200.cameramodel objects."""
import ctypes as C

import numpy as np

from . import _capi
from ._capi import checked
from .api import Problem, _Inputs, _lensmodel, _ptr, _require_gpu
from .poseutils import compose_Rt

_WHICH = ('all-cameras-must-see-full-board',
          'some-cameras-must-see-full-board',
          'all-cameras-must-see-half-board',
          'some-cameras-must-see-half-board', )


def ref_calibration_object(W=None, H=None, object_spacing=None, *, optimization_inputs=None, calobject_warp=None,
                           x_corner0=0, x_corner1=None, Nx=None, y_corner0=0, y_corner1=None, Ny=None):
    """The geometry of the calibration object: an array (..., Ny, Nx, 3) of the board's points in its own coordinates,
    as mrcal.ref_calibration_object() returns it. Corner (0,0) is at the origin and the grid spans x and y; z is the
    deflection of the optional parabolic warp: calobject_warp (2,) adds calobject_warp[0] 4 xr (1 - xr) and then
    calobject_warp[1] 4 yr (1 - yr), with xr, yr the corner coordinates scaled to [0,1].

    Either W, H and object_spacing are all given, or optimization_inputs is, which then supplies them and the warp.
    object_spacing is a scalar or (..., 2), multiplying (x, y) in that order; object_spacing and calobject_warp
    broadcast over their leading dimensions. x_corner0, x_corner1, Nx select the np.linspace(x_corner0, x_corner1, Nx)
    points along x in corner units (by default the W corners), and the y_* arguments likewise along y."""
    options_base = ('W', 'H', 'object_spacing')
    Noptions_base = sum(v is not None for v in (W, H, object_spacing))
    if not (Noptions_base == 0 or Noptions_base == len(options_base)):
        raise Exception(f"Options '{options_base}': ALL must be given, or NONE must be given")
    if Noptions_base > 0 and optimization_inputs is not None:
        raise Exception(f"Options '{options_base}' and 'optimization_inputs' cannot both be given")
    if Noptions_base == 0 and optimization_inputs is None:
        raise Exception(f"One of options '{options_base}' and 'optimization_inputs' MUST be given")

    if optimization_inputs is not None:
        H, W = optimization_inputs['observations_board'].shape[-3:-1]
        object_spacing = optimization_inputs['calibration_object_spacing']
        calobject_warp = optimization_inputs['calobject_warp']

    if Nx is None: Nx = W
    if Ny is None: Ny = H
    if x_corner1 is None: x_corner1 = W - 1
    if y_corner1 is None: y_corner1 = H - 1

    # (Ny,Nx) each, then (Ny,Nx,3) with z = 0
    xx, yy = np.meshgrid(np.linspace(x_corner0, x_corner1, Nx), np.linspace(y_corner0, y_corner1, Ny))
    full_object = np.concatenate((xx[..., None], yy[..., None], np.zeros(xx.shape + (1,))), axis=-1)

    # (..., 2) -> (..., 1,1,2)
    object_spacing = np.array(object_spacing)
    if object_spacing.ndim == 0:
        object_spacing = np.array((1, 1)) * object_spacing
    object_spacing = object_spacing[..., None, None, :]
    if object_spacing.ndim > 3:
        full_object = full_object * np.ones(object_spacing.shape[:-3] + (1, 1, 1))
    full_object[..., :2] *= object_spacing

    if calobject_warp is not None:
        calobject_warp = np.asarray(calobject_warp)
        xr = xx / (W - 1)
        yr = yy / (H - 1)
        dx = 4. * xr * (1. - xr)
        dy = 4. * yr * (1. - yr)
        if calobject_warp.ndim > 1:
            # (..., 1,1,2)
            calobject_warp = calobject_warp[..., None, None, :]
            full_object = full_object * np.ones(calobject_warp.shape[:-3] + (1, 1, 1))
        full_object[..., 2] += calobject_warp[..., 0] * dx
        full_object[..., 2] += calobject_warp[..., 1] * dy

    return full_object


def _identity_Rt():
    return np.concatenate((np.eye(3), np.zeros((1, 3))), axis=0)


def synthesize_board_observations(models, *, object_width_n, object_height_n, object_spacing, calobject_warp,
                                  rt_ref_boardcenter, rt_ref_boardcenter__noiseradius, Nframes,
                                  max_oblique_angle_deg=None, pcamera_nominal_ref=np.array((0, 0, 0), dtype=float),
                                  which='all-cameras-must-see-full-board'):
    """Random board poses that the cameras see, and their perfect projections, as mrcal.synthesize_board_observations()
    makes them. Returns (q, Rt_ref_boardref): q (Nframes, Ncameras, object_height_n, object_width_n, 2), the pixels of
    every corner in every camera (some may be out of view, depending on `which`), and Rt_ref_boardref (Nframes, 4,3),
    the poses of the board of ref_calibration_object() in the reference frame.

    Each frame's pose is rt_ref_boardcenter + uniform(-1,1) * rt_ref_boardcenter__noiseradius, a pose of the board
    about its center. Frames are made in chunks of Nframes: each chunk draws np.random.uniform(-1, 1, (Nframes,6)), so
    the same seed gives the reference's frames, in its order, and leaves np.random in its state. A frame is kept if
    its board normal is within max_oblique_angle_deg of the direction to pcamera_nominal_ref (when given) and if the
    cameras see the board as `which` asks: 'all-' or 'some-cameras-must-see-' 'full-board' (every corner in
    0 <= q <= imagersize - 1) or 'half-board' (more than half of the corners). Chunks are made until Nframes frames are
    kept. As in the reference, nothing limits the number of chunks: if no pose can qualify this does not return (it
    can be interrupted with Ctrl-C). models: mrcal_b200.cameramodel objects, which may have different lens models."""
    if which not in _WHICH:
        raise Exception(f"'which' argument must be one of {_WHICH}")
    Ncameras = len(models)
    H, W = object_height_n, object_width_n

    # the board about its center (ignoring the warp), and the shift back to the corner-referenced board
    board_center = np.array(((object_width_n - 1) * object_spacing / 2., (object_height_n - 1) * object_spacing / 2., 0))
    board_reference = ref_calibration_object(object_width_n, object_height_n, object_spacing,
                                             calobject_warp=calobject_warp) - board_center
    Rt_boardref_origboardref = _identity_Rt()
    Rt_boardref_origboardref[3, :] = -board_center

    max_cos_oblique_angle = np.cos(max_oblique_angle_deg * np.pi / 180.) if max_oblique_angle_deg is not None else None

    _require_gpu()
    lensmodels = (_capi.Lensmodel * max(Ncameras, 1))()
    intrinsics, Rt_cam_ref, imagersizes = [], [], []
    for i, m in enumerate(models):
        name, intr = m.intrinsics()
        lensmodels[i] = _lensmodel(name)
        intrinsics.append(np.asarray(intr, np.float64).ravel())
        Rt_cam_ref.append(m.Rt_cam_ref())
        imagersizes.append(m.imagersize())
    intrinsics = np.ascontiguousarray(np.concatenate(intrinsics) if intrinsics else np.zeros(0))
    Rt_cam_ref = np.ascontiguousarray(np.array(Rt_cam_ref, np.float64).reshape(Ncameras, 4, 3))
    imagersizes = np.ascontiguousarray(np.array(imagersizes, np.int32).reshape(Ncameras, 2))
    board = np.ascontiguousarray(board_reference, np.float64).reshape(-1, 3)

    def get_observation_chunk():
        # the whole random block in one shot, of Nframes poses whatever is still needed, as the reference draws it
        randomblock = np.random.uniform(low=-1.0, high=1.0, size=(Nframes, 6))
        rt = np.ascontiguousarray(rt_ref_boardcenter + randomblock * rt_ref_boardcenter__noiseradius, np.float64)
        q = np.zeros((Nframes, Ncameras, H, W, 2))
        Nvisible = np.zeros((Nframes, Ncameras), np.int32)
        Rt = np.zeros((Nframes, 4, 3))
        checked.mrcal_b200_synthesize_board_observations(_ptr(q), _ptr(Nvisible), _ptr(Rt), _ptr(rt), Nframes,
                                                         _ptr(board), board.shape[0], Ncameras, lensmodels,
                                                         _ptr(intrinsics), _ptr(Rt_cam_ref), _ptr(imagersizes))
        return q, Rt, Nvisible

    def cull(q, Rt_ref_boardref, Nvisible):
        if max_cos_oblique_angle is not None:
            # the reference's expression: |<unit vector to the board, board normal>| > cos(max angle)
            nref_position = Rt_ref_boardref[..., 3, :] - pcamera_nominal_ref
            nref_position /= np.sqrt(np.einsum('...i,...i', nref_position, nref_position))[..., None]
            nref_orientation = Rt_ref_boardref[..., :3, 2]
            costh = np.abs(np.einsum('...i,...i', nref_position, nref_orientation))
            i = costh > max_cos_oblique_angle
            q, Rt_ref_boardref, Nvisible = q[i], Rt_ref_boardref[i], Nvisible[i]
        N = H * W
        if which == 'all-cameras-must-see-full-board':
            iframe = np.all(Nvisible == N, axis=-1)
        elif which == 'some-cameras-must-see-full-board':
            iframe = np.any(Nvisible == N, axis=-1)
        elif which == 'all-cameras-must-see-half-board':
            iframe = np.all(Nvisible > N // 2, axis=-1)
        else:
            iframe = np.any(Nvisible > N // 2, axis=-1)
        return q[iframe, ...], Rt_ref_boardref[iframe, ...]

    q = np.zeros((0, Ncameras, H, W, 2), dtype=float)
    Rt_ref_boardref = np.zeros((0, 4, 3), dtype=float)
    # one decision per chunk, until Nframes frames are in view
    while True:
        q_here, Rt_here = cull(*get_observation_chunk())
        q = np.concatenate((q, q_here), axis=0)
        Rt_ref_boardref = np.concatenate((Rt_ref_boardref, Rt_here), axis=0)
        if q.shape[0] >= Nframes:
            q = q[:Nframes, ...]
            Rt_ref_boardref = Rt_ref_boardref[:Nframes, ...]
            break

    return q, compose_Rt(Rt_ref_boardref, Rt_boardref_origboardref)


def _corners(optimization_inputs, *, pcam=False, project=False, boards=True, points=False):
    """(pcam_board, q_board, q_point) of the problem, from csrc/synthetic_data.cu: the corners of the board
    observations (if boards) in each observing camera's frame (if pcam), their projections (if project) and the
    projections of the point observations (if points). What is not asked for is None"""
    _require_gpu()
    g = optimization_inputs.get
    z = lambda n, dtype=np.float64: np.zeros((0, n), dtype)
    idx_b = np.ascontiguousarray(g('indices_frame_camintrinsics_camextrinsics'), np.int32) if boards else z(3, np.int32)
    idx_p = np.ascontiguousarray(g('indices_point_camintrinsics_camextrinsics'), np.int32) if points else z(3, np.int32)
    Nobs_b, Nobs_p = idx_b.shape[0], idx_p.shape[0]
    if Nobs_b:
        H, W = g('observations_board').shape[-3:-1]
        board = ref_calibration_object(W, H, g('calibration_object_spacing'), calobject_warp=g('calobject_warp'))
        rt_ref_frame = g('rt_ref_frame')
    else:
        H = W = 0
        board, rt_ref_frame = z(3), z(6)
    board = np.ascontiguousarray(board, np.float64).reshape(-1, 3)
    rt_ref_frame = np.ascontiguousarray(rt_ref_frame, np.float64).reshape(-1, 6)
    rt_cam_ref = np.ascontiguousarray(g('rt_cam_ref') if g('rt_cam_ref') is not None else z(6), np.float64).reshape(-1, 6)
    pts = np.ascontiguousarray(g('points') if Nobs_p else z(3), np.float64).reshape(-1, 3)
    pcam_board = np.zeros((Nobs_b, H, W, 3)) if pcam else None
    q_board = np.zeros((Nobs_b, H, W, 2)) if project and Nobs_b else None
    q_point = np.zeros((Nobs_p, 2)) if Nobs_p else None
    lm = intrinsics = None
    if project:
        lm = C.byref(_lensmodel(g('lensmodel')))
        intrinsics = np.ascontiguousarray(g('intrinsics'), np.float64)
    checked.mrcal_b200_problem_corners(_ptr(pcam_board), _ptr(q_board), _ptr(q_point), _ptr(idx_b), Nobs_b,
                                       _ptr(board), board.shape[0], _ptr(idx_p), Nobs_p, _ptr(pts), pts.shape[0],
                                       _ptr(rt_ref_frame), rt_ref_frame.shape[0], _ptr(rt_cam_ref), rt_cam_ref.shape[0],
                                       lm, _ptr(intrinsics), intrinsics.shape[0] if project else 0)
    return pcam_board, q_board, q_point


def hypothesis_board_corner_positions(icam_intrinsics=None, idx_inliers=None, **optimization_inputs):
    """The board corners the solver believes each camera saw, in the observing camera's frame, as
    mrcal.hypothesis_board_corner_positions() reports them: for each board observation,
    transform_point_Rt(compose_Rt(Rt_cam_ref, Rt_ref_frame), corner), Rt_cam_ref the identity for a camera at the
    reference. Returns four arrays:

    - (Nobservations, H, W, 3): every observation's corners
    - (Nobservations_thiscamera, H, W, 3): those of camera icam_intrinsics (all of them if it is None)
    - (N, 3): the corners of that camera that are inliers
    - (N, 3): the corners of that camera that are outliers

    idx_inliers: (Nobservations, H, W) booleans selecting the inliers; None takes observations_board[...,2] > 0. As
    in the reference, when icam_intrinsics is given the array given here is modified in place: the other cameras'
    entries are set to False."""
    observations_board = optimization_inputs.get('observations_board')
    if observations_board is None:
        raise Exception("No board observations available")
    indices_frame_camintrinsics_camextrinsics = optimization_inputs['indices_frame_camintrinsics_camextrinsics']
    p_cam_calobjects = _corners(optimization_inputs, pcam=True)[0]

    if idx_inliers is None:
        idx_inliers = observations_board[..., 2] > 0
    idx_outliers = ~idx_inliers

    if icam_intrinsics is None:
        return p_cam_calobjects, p_cam_calobjects, p_cam_calobjects[idx_inliers, ...], \
            p_cam_calobjects[idx_outliers, ...]

    idx_observations = indices_frame_camintrinsics_camextrinsics[:, 1] == icam_intrinsics
    idx_inliers[~idx_observations] = False
    idx_outliers[~idx_observations] = False
    return p_cam_calobjects, p_cam_calobjects[idx_observations, ...], p_cam_calobjects[idx_inliers, ...], \
        p_cam_calobjects[idx_outliers, ...]


def _observed_pixel_uncertainty_from_inputs(optimization_inputs):
    """The observed-pixel uncertainty estimated from the residuals at the given state: the estimate
    projection_uncertainty() makes (csrc/uncertainty.cu), bit for bit"""
    P = Problem(**optimization_inputs)
    try:
        sigma = C.c_double(0.)
        checked.mrcal_b200_problem_observed_pixel_uncertainty(P._h, C.byref(sigma))
        return sigma.value
    finally:
        P.close()


def _have(optimization_inputs, key):
    a = optimization_inputs.get(key)
    return a is not None and a.size > 0


def make_perfect_observations(optimization_inputs, *, observed_pixel_uncertainty=None):
    """Replace the observations of optimization_inputs with perfect ones, and add perfect noise, as
    mrcal.make_perfect_observations() does. THIS MODIFIES optimization_inputs IN PLACE, and returns None.

    observations_board[...,:2] become the projections of the hypothetical board corners
    (hypothesis_board_corner_positions()) and observations_point[...,:2] those of the points, through the solved
    geometry and intrinsics. Then, unless observed_pixel_uncertainty is 0, Gaussian noise of that standard deviation is
    added, drawn with np.random.randn, first for the boards and then for the points, and divided by the weight of each
    observation. observed_pixel_uncertainty=None estimates it from the residuals of the observations as given, before
    they are overwritten, with the estimate projection_uncertainty() uses. With 0 the RNG is not touched.

    Two behaviours of the reference are kept. A weight <= 0 (an outlier) counts as 1 when dividing the noise, and
    this is written through to the caller's array: when noise is added, an outlier's weight of -1 becomes 1.
    Triangulated-point observations are left untouched."""
    I = _Inputs(optimization_inputs)   # the refusals of the solver's own argument checks
    if observed_pixel_uncertainty is None:
        observed_pixel_uncertainty = _observed_pixel_uncertainty_from_inputs(optimization_inputs)

    boards = I.Nobs_board > 0 and _have(optimization_inputs, 'indices_frame_camintrinsics_camextrinsics')
    points = I.Nobs_point > 0 and _have(optimization_inputs, 'indices_point_camintrinsics_camextrinsics')
    if boards or points:
        _, q_board, q_point = _corners(optimization_inputs, project=True, boards=boards, points=points)
        if boards:
            optimization_inputs['observations_board'][..., :2] = q_board
        if points:
            optimization_inputs['observations_point'][..., :2] = q_point

    if observed_pixel_uncertainty == 0:
        return

    for what in ('observations_board', 'observations_point'):
        if _have(optimization_inputs, what):
            obs = optimization_inputs[what]
            noise_nominal = observed_pixel_uncertainty * np.random.randn(*obs[..., :2].shape)
            # a view of the weights: the fix-up below writes through to obs, as the reference's nps.dummy() view does
            weight = np.expand_dims(obs[..., 2], axis=-1)
            weight[weight <= 0] = 1.   # to avoid dividing by 0
            obs[..., :2] += noise_nominal / weight
