"""Valid-intrinsics regions: where a calibrated camera's intrinsics can be trusted, as mrcal-calibrate-cameras computes
it for every camera it writes (mrcal-calibrate-cameras:883-906; mrcal/calibration.py:1590-1866) and as
mrcal.is_within_valid_intrinsics_region() reads it (mrcal/model_analysis.py:2106-2149).

The heavy parts run on the device (csrc/regions.cu, csrc/uncertainty.cu): the residual statistics binned by imager
cell, the projection uncertainty of every camera's grid from one factorization of the problem, and the strict
point-in-region test. What stays here is a few hundred cells of host arithmetic: the thresholds, the mask, and the
mask's outer contour, which is cv2.findContours(RETR_EXTERNAL, CHAIN_APPROX_SIMPLE) restated so that the package
needs no OpenCV at run time."""
import re
import sys

import numpy as np

from . import api
from ._capi import checked
from .api import _ptr, _require_gpu


def close_contour(c):
    """The polyline c (N,2) closed: c if its first and last points coincide (within 1e-6), else c with its first point
    appended. None stays None; an empty array becomes (0,2) (mrcal/utils.py:941-1000)"""
    if c is None:
        return None
    c = np.asarray(c)
    if c.size == 0:
        return np.zeros((0, 2), dtype=float)
    if np.linalg.norm(c[0, :] - c[-1, :]) < 1e-6:
        return c
    return np.concatenate((c, c[:1, :]), axis=-2)


def imagergrid_using(imagersize, gridn_width, gridn_height=None):
    """The gnuplotlib 'using' expression that plots a (gridn_height, gridn_width) grid in imager pixels
    (mrcal/visualization.py:3160-3218)"""
    W, H = imagersize
    if gridn_height is None:
        gridn_height = int(round(H / W * gridn_width))
    return '($1*{}):($2*{}):3'.format(float(W - 1) / (gridn_width - 1), float(H - 1) / (gridn_height - 1))


####################################################################################################
# the contour of a mask: cv2.findContours(mask, RETR_EXTERNAL, CHAIN_APPROX_SIMPLE) and cv2.contourArea()
####################################################################################################
# the 8 neighbours by chain code: 0 east, then counterclockwise in image coordinates (y down): 2 north, 4 west, 6 south
_DX = (1, 1, 0, -1, -1, -1, 0, 1)
_DY = (0, -1, -1, -1, 0, 1, 1, 1)


def _follow_outer_border(img, x0, y0):
    """The outer border that starts at img[y0, x0] (its west neighbour is background), followed as Suzuki and Abe's
    border following does it, marking the border pixels: -1 where the search passed the east neighbour as background
    (a right edge), 2 elsewhere. Returns the vertices of the chain where its direction changes (CHAIN_APPROX_SIMPLE),
    in padded coordinates"""
    # the first neighbour clockwise from the north-west
    s = 4
    while True:
        s = (s - 1) & 7
        if img[y0 + _DY[s], x0 + _DX[s]] != 0 or s == 4:
            break
    if s == 4:   # a single pixel
        img[y0, x0] = -1
        return [(x0, y0)]
    x1, y1 = x0 + _DX[s], y0 + _DY[s]
    out = []
    x3, y3 = x0, y0
    prev_s = s ^ 4
    while True:
        # counterclockwise from the pixel we came from to the next border pixel
        s_end = s
        while s < 15:
            s += 1
            x4, y4 = x3 + _DX[s & 7], y3 + _DY[s & 7]
            if img[y4, x4] != 0:
                break
        s &= 7
        if 1 <= s <= s_end:
            img[y3, x3] = -1
        elif img[y3, x3] == 1:
            img[y3, x3] = 2
        if s != prev_s:
            out.append((x3, y3))
            prev_s = s
        if (x4, y4) == (x0, y0) and (x3, y3) == (x1, y1):
            return out
        x3, y3 = x4, y4
        s = (s + 4) & 7


def find_external_contours(mask):
    """The outer borders of the 8-connected blobs of mask (h, w) that lie in no other blob's hole, as lists of (x, y)
    vertices: what cv2.findContours(mask, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE) returns, in its order (the last
    border met in a raster scan first). Pixels on the border of the mask count: the mask is framed by background"""
    mask = np.asarray(mask)
    h, w = mask.shape
    img = np.zeros((h + 2, w + 2), np.int8)
    img[1:-1, 1:-1] = mask != 0
    found = []
    for y in range(1, h + 1):
        # lnbd: the last border pixel met in this row; a new outer border inside a blob (in a hole) starts after a
        # marked left edge (2), one outside every blob after a right edge (-1) or the row's start
        lnbd = 0
        prev = 0
        for x in range(1, w + 1):
            p = img[y, x]
            if p == prev:
                continue
            if prev == 0 and p == 1 and img[y, lnbd] <= 0:
                found.append([(px - 1, py - 1) for px, py in _follow_outer_border(img, x, y)])
                # the scan goes on from the marked start pixel, with lnbd where it was
                prev = img[y, x]
                continue
            prev = p
            if prev != 0 and prev != 1:
                lnbd = x
    return found[::-1]


def contour_area(c):
    """cv2.contourArea(c): the absolute shoelace area of the closed polygon c (N,2)"""
    c = np.asarray(c, np.float64).reshape(-1, 2)
    if c.shape[0] == 0:
        return 0.
    x, y = c[:, 0], c[:, 1]
    xp, yp = np.roll(x, 1), np.roll(y, 1)
    a = 0.
    for i in range(c.shape[0]):
        a += xp[i] * y[i] - yp[i] * x[i]
    return abs(a * 0.5)


def _region_from_mask(mask, imagersize):
    """The valid-intrinsics region of a (gridn_height, gridn_width) mask (mrcal/calibration.py:1686-1717): the
    largest outer contour, closed, scaled from cells to pixels and rounded; (0,2) if there is none or it has fewer
    than 4 points"""
    gh, gw = mask.shape
    contours = find_external_contours(mask)
    if not contours:
        return np.zeros((0, 2))
    areas = np.array([contour_area(c) for c in contours])
    contour = close_contour(np.array(contours[np.argmax(areas)], dtype=float))
    if contour.ndim != 2 or contour.shape[0] < 4:
        return np.zeros((0, 2))
    W, H = imagersize
    contour[:, 0] *= float(W - 1) / (gw - 1)
    contour[:, 1] *= float(H - 1) / (gh - 1)
    return contour.round().astype(np.int32)


def _region_mask(lensmodel, mean, stdev, count, uncertainty, threshold_uncertainty, threshold_mean, threshold_stdev,
                 threshold_count):
    """Which cells are valid (mrcal/calibration.py:1663-1684): a finite uncertainty below its threshold and, unless the
    model is splined, a signed mean, a stdev and a count (x and y counted apart) within theirs"""
    uncertainty = np.array(uncertainty, dtype=float)
    uncertainty[~np.isfinite(uncertainty)] = 1e9
    mask = uncertainty < threshold_uncertainty
    if not re.match('LENSMODEL_SPLINED_', lensmodel):
        mask = mask & (mean < threshold_mean) & (stdev < threshold_stdev) & (count > threshold_count)
    return mask


####################################################################################################
# the measurements of a solve (mrcal/utils.py:1286-1556)
####################################################################################################
def _measurements_x(optimization_inputs, x):
    if x is None:
        x = api.optimizer_callback(**optimization_inputs, no_jacobian=True, no_factorization=True)[1]
    return x


def measurements_board(optimization_inputs, *, icam_intrinsics=None, x=None, return_observations=False, i_cam=None):
    """The weighted reprojection errors (N,2) of the board observations that are not outliers, of camera
    icam_intrinsics (all cameras if None), as mrcal.measurements_board() selects them; with return_observations, also
    the observed pixels (N,2). x: the measurement vector; None evaluates it on the device. i_cam: an old name of
    icam_intrinsics"""
    observations_board = optimization_inputs.get('observations_board')
    if observations_board is None or observations_board.size == 0:
        return (np.zeros((0, 2)), np.zeros((0, 2))) if return_observations else np.zeros((0, 2))
    if i_cam is not None:
        icam_intrinsics = i_cam
    x = _measurements_x(optimization_inputs, x)
    imeas0 = api.measurement_index_boards(0, **optimization_inputs)
    Nmeas = api.num_measurements_boards(**optimization_inputs)
    x_board = x[imeas0:imeas0 + Nmeas].reshape(*observations_board.shape[:-1], 2)
    idx = np.ones(observations_board.shape[:-1], dtype=bool)
    if icam_intrinsics is not None:
        idx[optimization_inputs['indices_frame_camintrinsics_camextrinsics'][:, 1] != icam_intrinsics, ...] = False
    idx[observations_board[..., 2] <= 0.0] = False
    if return_observations:
        return x_board[idx, ...], observations_board[idx, ..., :2]
    return x_board[idx, ...]


def residuals_board(*args, residuals=None, **kwargs):
    """measurements_board() under its old name, with x called residuals"""
    return measurements_board(*args, x=residuals, **kwargs)


residuals_chessboard = residuals_board


def measurements_point(optimization_inputs, *, icam_intrinsics=None, x=None, return_observations=False):
    """The weighted reprojection errors (N,2) of the point observations that are not outliers, of camera
    icam_intrinsics (all cameras if None), as mrcal.measurements_point() selects them; with return_observations, also
    the observed pixels (N,2). x: the measurement vector; None evaluates it on the device"""
    observations_point = optimization_inputs.get('observations_point')
    if observations_point is None or observations_point.size == 0:
        return (np.zeros((0, 2)), np.zeros((0, 2))) if return_observations else np.zeros((0, 2))
    x = _measurements_x(optimization_inputs, x)
    Nobservations = len(observations_point)
    imeas0 = api.measurement_index_points(0, **optimization_inputs)
    Nmeas = api.num_measurements_points(**optimization_inputs)
    x_point = x[imeas0:imeas0 + Nmeas].reshape(Nobservations, 2)
    idx = np.ones((Nobservations,), dtype=bool)
    if icam_intrinsics is not None:
        idx[optimization_inputs['indices_point_camintrinsics_camextrinsics'][:, 1] != icam_intrinsics] = False
    idx[observations_point[..., 2] <= 0.0] = False
    if return_observations:
        return x_point[idx, ...], observations_point[idx, ..., :2]
    return x_point[idx, ...]


def residuals_point(*args, residuals=None, **kwargs):
    """measurements_point() under its old name, with x called residuals"""
    return measurements_point(*args, x=residuals, **kwargs)


####################################################################################################
# the regions
####################################################################################################
def _gridn_height(imagersize, gridn_width, gridn_height):
    W, H = imagersize
    return int(round(H / W * gridn_width)) if gridn_height is None else int(gridn_height)


def _cell_grid(imagersize, gridn_width, gridn_height):
    """(q_cell_center (gh, gw, 2), rcell (2,)) of a camera's grid (mrcal/calibration.py:1800-1808)"""
    W, H = imagersize
    q = api.sample_imager(gridn_width, gridn_height, W, H)
    rcell = np.array((float(W - 1) / (gridn_width - 1), float(H - 1) / (gridn_height - 1)), dtype=float) / 2.
    return q, rcell


def _statistics(P, icams, imagersizes, gridn_width, gridn_height, evaluate):
    """([(mean, stdev, count)] per camera, x) from the problem P: one device call per grid shape"""
    out = [None] * len(icams)
    x = None
    shapes = {}
    for k, size in enumerate(imagersizes):
        shapes.setdefault(_gridn_height(size, gridn_width, gridn_height), []).append(k)
    for gh, ks in shapes.items():
        grids = [_cell_grid(imagersizes[k], gridn_width, gh) for k in ks]
        stats, x = P.regional_statistics([icams[k] for k in ks], np.array([g[0] for g in grids]),
                                         np.array([g[1] for g in grids]), evaluate=evaluate and x is None)
        for j, k in enumerate(ks):
            out[k] = (stats[j, ..., 0], stats[j, ..., 1], stats[j, ..., 2])
    return out, x


def _model_inputs(model):
    optimization_inputs = model.optimization_inputs()
    if optimization_inputs is None:
        raise RuntimeError("optimization_inputs are unavailable in this model. The regional statistics and the "
                           "uncertainty cannot be computed")
    return optimization_inputs


def _report_regional_statistics(model, gridn_width=20, gridn_height=None):
    """(mean, stdev, count, using): the weighted board residuals of the model's camera binned by imager cell, each
    (gridn_height, gridn_width), as mrcal.calibration._report_regional_statistics() computes them; count counts x and
    y apart, and a cell with count <= 5 reports mean = stdev = 0. On the device (csrc/regions.cu)"""
    _require_gpu()
    optimization_inputs = _model_inputs(model)
    gridn_height = _gridn_height(model.imagersize(), gridn_width, gridn_height)
    P = api.Problem(**optimization_inputs)
    try:
        (stats,), _ = _statistics(P, [model.icam_intrinsics()], [model.imagersize()], gridn_width, gridn_height, True)
    finally:
        P.close()
    return stats + (imagergrid_using(model.imagersize(), gridn_width, gridn_height),)


def _regions(optimization_inputs, cameras, thresholds, distance, gridn_width, gridn_height):
    """The valid-intrinsics region of each camera (icam_intrinsics, lensmodel, intrinsics, imagersize) of one solve,
    or the exception that stopped it. One problem, one evaluation and one factorization serve every camera: the
    uncertainties of all the grids first, then the statistics on the residuals of that evaluation.
    thresholds(x) -> (uncertainty, mean, stdev, count) given the measurement vector"""
    results = [None] * len(cameras)
    queries = []   # (k, gh, pcam)
    for k, (icam, lensmodel, intrinsics, imagersize) in enumerate(cameras):
        try:
            gh = _gridn_height(imagersize, gridn_width, gridn_height)
            q, _ = _cell_grid(imagersize, gridn_width, gh)
            v = api.unproject(q, lensmodel, intrinsics)
            v = v / np.linalg.norm(v, axis=-1)[..., None]
            queries.append((k, gh, v if distance <= 0 else v * distance))
        except Exception as e:
            results[k] = e
    if not queries:
        return results
    try:
        P = api.Problem(**optimization_inputs)
        try:
            Var, _ = P.projection_uncertainty_cameras([p.reshape(-1, 3) for _, _, p in queries],
                                                      [cameras[k][0] for k, _, _ in queries], atinfinity=distance <= 0)
            stats, x = _statistics(P, [cameras[k][0] for k, _, _ in queries], [cameras[k][3] for k, _, _ in queries],
                                   gridn_width, gridn_height, evaluate=False)
        finally:
            P.close()
        threshold_uncertainty, threshold_mean, threshold_stdev, threshold_count = thresholds(x)
    except Exception as e:
        for k, _, _ in queries:
            results[k] = e
        return results
    for j, (k, gh, _) in enumerate(queries):
        try:
            mean, stdev, count = stats[j]
            uncertainty = api.worst_direction_stdev(Var[j]).reshape(gh, gridn_width)
            mask = _region_mask(cameras[k][1], mean, stdev, count, uncertainty, threshold_uncertainty, threshold_mean,
                                threshold_stdev, threshold_count)
            results[k] = _region_from_mask(mask, cameras[k][3])
        except Exception as e:
            results[k] = e
    return results


def _compute_valid_intrinsics_region(model, threshold_uncertainty, threshold_mean, threshold_stdev, threshold_count,
                                     distance, gridn_width=30, gridn_height=None):
    """The valid-intrinsics region of the model's camera, as mrcal.calibration._compute_valid_intrinsics_region()
    computes it: an (N,2) int32 closed contour in pixels, or (0,2) if the region is empty. A cell of the
    (gridn_height, gridn_width) grid is valid when the worst-direction stdev of its projection uncertainty (at
    infinity if distance <= 0, else at that distance) is below threshold_uncertainty and, unless the model is splined,
    its residuals' signed mean, stdev and count are below, below and above their thresholds. Raises on failure"""
    _require_gpu()
    optimization_inputs = _model_inputs(model)
    lensmodel, intrinsics = model.intrinsics()
    thresholds = (threshold_uncertainty, threshold_mean, threshold_stdev, threshold_count)
    (r,) = _regions(optimization_inputs, [(model.icam_intrinsics(), lensmodel, intrinsics, model.imagersize())],
                    lambda x: thresholds, distance, gridn_width, gridn_height)
    if isinstance(r, Exception):
        raise r
    return r


def valid_intrinsics_regions(optimization_inputs, parameters=(1, 0.5, 1.5, 3, 0), *, gridn_width=30,
                             gridn_height=None):
    """The valid-intrinsics region of every intrinsics camera of a solve, as mrcal-calibrate-cameras computes them
    (mrcal-calibrate-cameras:883-906): a list of (N,2) int32 arrays, (0,2) for an empty region and None for a camera
    whose region could not be computed (with a warning on stderr). parameters = (uncertainty, mean, stdev, count,
    distance), the tool's --valid-intrinsics-region-parameters: the uncertainty and stdev thresholds are multiples of
    the stdev of all the board measurements. Every camera comes from one evaluation and one factorization"""
    _require_gpu()
    p_u, p_mean, p_stdev, p_count, distance = parameters
    lensmodel = optimization_inputs['lensmodel']
    intrinsics = optimization_inputs['intrinsics']
    imagersizes = optimization_inputs['imagersizes']

    def thresholds(x):
        s = np.std(measurements_board(optimization_inputs, x=x).ravel())
        return p_u * s, p_mean, p_stdev * s, p_count
    cameras = [(i, lensmodel, intrinsics[i], imagersizes[i]) for i in range(len(intrinsics))]
    regions = _regions(optimization_inputs, cameras, thresholds, distance, gridn_width, gridn_height)
    for i, r in enumerate(regions):
        if isinstance(r, Exception):
            print(f"WARNING: Couldn't compute valid-intrinsics region for camera {i}. Will continue without. "
                  f"Error: {r}", file=sys.stderr)
            regions[i] = None
    return regions


def is_within_valid_intrinsics_region(q, model):
    """Which of the pixels q (..., 2) lie strictly inside the model's valid-intrinsics region, as
    mrcal.is_within_valid_intrinsics_region() decides it: a bool mask of shape q.shape[:-1], False on the region's
    edges and vertices and for NaN pixels, all False for an empty region; None if the model has no region. On the
    device (csrc/image_transforms.cu)"""
    r = model.valid_intrinsics_region()
    if r is None:
        return None
    _require_gpu()
    q = np.ascontiguousarray(q, np.float64)
    if q.ndim == 0 or q.shape[-1] != 2:
        raise RuntimeError(f"q must have shape (...,2); got {q.shape}")
    r = np.ascontiguousarray(r, np.float64).reshape(-1, 2)
    mask = np.zeros(q.shape[:-1], dtype=bool)
    if mask.size:
        checked.mrcal_b200_is_within_region(mask.ctypes.data, _ptr(q), mask.size, _ptr(r), r.shape[0])
    return mask
