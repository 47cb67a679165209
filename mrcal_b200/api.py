"""The Python surface of the calibration solve, with the reference's names,
keyword arguments, return values and error behaviour (mrcal-pywrap.c:890-937,
1557-2141, 2164-3595; optimize.docstring, optimizer_callback.docstring).

    mrcal_b200.optimize(**optimization_inputs)            -> dict
    mrcal_b200.optimizer_callback(**optimization_inputs)  -> (b_packed, x, J, factorization)
    mrcal_b200.state_index_*(), num_states*(), measurement_index_*(),
    num_measurements*(), num_intrinsics_optimization_params(),
    pack_state(), unpack_state(), corresponding_icam_extrinsics(),
    lensmodel_num_params(), lensmodel_metadata_and_config(),
    knots_for_splined_models(), supported_lensmodels(), CHOLMOD_factorization

Everything numeric happens in libmrcal_b200.so (CUDA, sm_90a). This module only
marshals arguments, the way mrcal-pywrap.c does for the reference.
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import scipy.sparse

from . import _capi
from ._capi import checked
from ._poses_host import compose_Rt, invert_Rt

_KNOWN_KWARGS = {
    "intrinsics", "lensmodel", "imagersizes",
    "extrinsics_rt_fromref", "frames_rt_toref", "rt_cam_ref", "rt_ref_frame", "points",
    "observations_board", "indices_frame_camintrinsics_camextrinsics",
    "observations_point", "indices_point_camintrinsics_camextrinsics",
    "observations_point_triangulated", "indices_point_triangulated_camintrinsics_camextrinsics",
    "observed_pixel_uncertainty", "calobject_warp", "Npoints_fixed",
    "do_optimize_intrinsics_core", "do_optimize_intrinsics_distortions", "do_optimize_extrinsics",
    "do_optimize_frames", "do_optimize_calobject_warp", "calibration_object_spacing", "verbose",
    "do_apply_regularization", "do_apply_regularization_unity_cam01", "do_apply_outlier_rejection",
    "imagepaths",
}


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None and a.size else None


def _lensmodel(name):
    if not isinstance(name, str):
        raise RuntimeError("The lens model must be given as a string")
    lm = _capi.Lensmodel()
    if not checked.mrcal_lensmodel_from_name(C.byref(lm), name.encode()):
        t = lm.type
        if t == -1:
            raise RuntimeError(f"Couldn't parse the configuration of the given lens model '{name}'")
        if t == -3:
            raise RuntimeError(f"The given lens model '{name}' needs a configuration, but none was given")
        raise RuntimeError(f"Invalid lens model '{name}'. Supported: {supported_lensmodels()}")
    return lm


def _check(name, a, dtype, shape, writable=False):
    """The reference's CHECK_LAYOUT (python-wrapping-utilities.h:67-114): exact
    dtype, C-contiguous, given trailing dims. No silent conversions: optimize()
    writes its results into the caller's arrays."""
    if not isinstance(a, np.ndarray):
        raise RuntimeError(f"'{name}' must be a numpy array")
    if a.dtype != dtype:
        raise RuntimeError(f"'{name}' must have dtype {np.dtype(dtype).name}; got {a.dtype.name}")
    if a.ndim != len(shape):
        raise RuntimeError(f"'{name}' must have exactly {len(shape)} dims; got {a.ndim}")
    for i, n in enumerate(shape):
        if n >= 0 and a.shape[i] != n:
            raise RuntimeError(f"'{name}' must have shape {shape} (-1: any); got {a.shape}")
    if not a.flags.c_contiguous:
        raise RuntimeError(f"'{name}' must be c-style contiguous")
    if writable and not a.flags.writeable:
        raise RuntimeError(f"'{name}' must be writeable")
    return a


class _Inputs:
    """Parsed, validated optimization_inputs (mrcal-pywrap.c:976-1244, 1589-1795)."""

    def __init__(self, kw, for_layout_only=False, explicit=None):
        kw = {k: v for k, v in kw.items() if v is not None}
        unknown = set(kw) - _KNOWN_KWARGS
        if unknown:
            raise RuntimeError(f"Unknown keyword argument(s): {sorted(unknown)}")
        for old, new in (("extrinsics_rt_fromref", "rt_cam_ref"), ("frames_rt_toref", "rt_ref_frame")):
            # optimization_inputs read from a .cameramodel carry the old names as a poison string, which the reference's
            # argument converter takes for "not given" (PyArray_Converter_checkrenamed_leaveNone, mrcal-pywrap.c:840-880)
            if isinstance(kw.get(old), str) and kw[old].startswith("ERROR:"):
                del kw[old]
            if old in kw:
                if new in kw:
                    raise RuntimeError(f"Both '{old}' and '{new}' were given; use '{new}' only")
                kw[new] = kw.pop(old)
        self.kw = kw
        z = np.zeros
        g = kw.get
        self.lensmodel_name = g("lensmodel")
        self.lensmodel = _lensmodel(self.lensmodel_name) if self.lensmodel_name is not None else None
        if self.lensmodel is None and not for_layout_only:
            raise RuntimeError("The 'lensmodel' argument is required")

        def arr(name, dtype, shape, empty):
            a = g(name)
            if a is None:
                return z(empty, dtype)
            return _check(name, a, dtype, shape)

        self.intrinsics = arr("intrinsics", np.float64, (-1, -1), (0, 0))
        self.imagersizes = arr("imagersizes", np.int32, (-1, 2), (0, 2))
        self.rt_cam_ref = arr("rt_cam_ref", np.float64, (-1, 6), (0, 6))
        self.rt_ref_frame = arr("rt_ref_frame", np.float64, (-1, 6), (0, 6))
        self.points = arr("points", np.float64, (-1, 3), (0, 3))
        self.observations_board = arr("observations_board", np.float64, (-1, -1, -1, 3), (0, 0, 0, 3))
        self.indices_board = arr("indices_frame_camintrinsics_camextrinsics", np.int32, (-1, 3), (0, 3))
        self.observations_point = arr("observations_point", np.float64, (-1, 3), (0, 3))
        self.indices_point = arr("indices_point_camintrinsics_camextrinsics", np.int32, (-1, 3), (0, 3))
        self.observations_tri = arr("observations_point_triangulated", np.float64, (-1, 3), (0, 3))
        self.indices_tri = arr("indices_point_triangulated_camintrinsics_camextrinsics", np.int32, (-1, 3), (0, 3))
        self.calobject_warp = g("calobject_warp")
        if self.calobject_warp is not None:
            _check("calobject_warp", self.calobject_warp, np.float64, (2,))
        self.Npoints_fixed = int(g("Npoints_fixed", 0))
        self.spacing = float(g("calibration_object_spacing", -1.0))
        self.verbose = bool(g("verbose", False))

        e = explicit or {}
        pick = lambda key, a: int(e[key]) if e.get(key) is not None and e[key] >= 0 else a.shape[0]
        self.Ncam_i = pick("Ncameras_intrinsics", self.intrinsics)
        self.Ncam_e = pick("Ncameras_extrinsics", self.rt_cam_ref)
        self.Nframes = pick("Nframes", self.rt_ref_frame)
        self.Npoints = pick("Npoints", self.points)
        self.Nobs_board = pick("Nobservations_board", self.observations_board)
        self.Nobs_point = pick("Nobservations_point", self.observations_point)
        self.Nobs_tri = self.observations_tri.shape[0]
        if self.observations_board.shape[0] > 0:
            self.H, self.W = self.observations_board.shape[1:3]
        else:
            self.H = self.W = -1

        # defaults: optimise whatever exists (mrcal-pywrap.c:1447-1457)
        d = dict(do_optimize_intrinsics_core=self.Ncam_i > 0,
                 do_optimize_intrinsics_distortions=self.Ncam_i > 0,
                 do_optimize_extrinsics=self.Ncam_e > 0,
                 do_optimize_frames=self.Nframes > 0,
                 do_optimize_calobject_warp=self.Nobs_board > 0,
                 do_apply_regularization=True,
                 do_apply_outlier_rejection=True,
                 do_apply_regularization_unity_cam01=False)
        bits = 0
        self.flags = {}
        for ib, name in enumerate(_capi.SELECTION_BITS):
            v = bool(kw[name]) if name in kw else d[name]
            self.flags[name] = v
            bits |= (1 << ib) if v else 0
        self.selections = _capi.Selections(bits)
        if not for_layout_only:
            self._validate()

    def _validate(self):
        if self.intrinsics.shape[0] != self.imagersizes.shape[0]:
            raise RuntimeError(f"Inconsistent Ncameras: 'intrinsics' says {self.intrinsics.shape[0]}, "
                               f"'imagersizes' says {self.imagersizes.shape[0]}")
        Nintr = checked.mrcal_lensmodel_num_params(C.byref(self.lensmodel))
        if self.intrinsics.shape[0] and self.intrinsics.shape[1] != Nintr:
            raise RuntimeError(f"intrinsics.shape[-1] MUST be {Nintr} for {self.lensmodel_name}. "
                               f"Instead got {self.intrinsics.shape[1]}")
        if self.indices_board.shape[0] != self.Nobs_board:
            raise RuntimeError(f"Inconsistent Nobservations_board: 'observations_board' says {self.Nobs_board}, "
                               f"'indices_frame_camintrinsics_camextrinsics' says {self.indices_board.shape[0]}")
        if self.Nobs_board > 0:
            if not self.spacing > 0.0:
                raise RuntimeError("We have board observations, so calibration_object_spacing MUST be a valid float > 0")
            if self.flags["do_optimize_calobject_warp"] and self.calobject_warp is None:
                raise RuntimeError("do_optimize_calobject_warp is True, so calobject_warp MUST be given as an array "
                                   "to seed the optimization and to receive the results")
        if self.indices_point.shape[0] != self.Nobs_point:
            raise RuntimeError(f"Inconsistent Nobservations_point: 'observations_point...' says {self.Nobs_point}, "
                               f"'indices_point_camintrinsics_camextrinsics' says {self.indices_point.shape[0]}")
        if self.indices_tri.shape[0] != self.Nobs_tri:
            raise RuntimeError("Inconsistent Nobservations_point_triangulated")
        if self.Nobs_tri > 0:
            it = self.indices_tri
            if (it[:, 1] < 0).any() or (it[:, 1] >= self.Ncam_i).any():
                raise RuntimeError(f"icam_intrinsics MUST be in [0,{self.Ncam_i - 1}] in indices_point_triangulated_camintrinsics_camextrinsics")
            if (it[:, 2] < -1).any() or (it[:, 2] >= self.Ncam_e).any():
                raise RuntimeError(f"icam_extrinsics MUST be in [-1,{self.Ncam_e - 1}] in indices_point_triangulated_camintrinsics_camextrinsics")
            # mrcal-pywrap.c:1406-1440: sets are runs of equal ipoint, consecutive, each seen at least twice
            if (it[:, 0] < 0).any():
                raise RuntimeError("Error in indices_point_triangulated_camintrinsics_camextrinsics. Each ipoint must be >=0")
            d = np.diff(it[:, 0])
            if ((d != 0) & (d != 1)).any() or it[0, 0] != 0:
                raise RuntimeError("Error in indices_point_triangulated_camintrinsics_camextrinsics. All ipoint must be consecutive and monotonic")
            if (np.bincount(it[:, 0]) < 2).any():
                raise RuntimeError("Error in indices_point_triangulated_camintrinsics_camextrinsics. Each point must be observed at least 2 times")

        ib = self.indices_board
        if self.Nobs_board:
            if (ib[:, 0] < 0).any() or (ib[:, 0] >= self.Nframes).any():
                raise RuntimeError(f"iframe MUST be in [0,{self.Nframes - 1}] in indices_frame_camintrinsics_camextrinsics")
            if (ib[:, 1] < 0).any() or (ib[:, 1] >= self.Ncam_i).any():
                raise RuntimeError(f"icam_intrinsics MUST be in [0,{self.Ncam_i - 1}] in indices_frame_camintrinsics_camextrinsics")
            if (ib[:, 2] < -1).any() or (ib[:, 2] >= self.Ncam_e).any():
                raise RuntimeError(f"icam_extrinsics MUST be in [-1,{self.Ncam_e - 1}] in indices_frame_camintrinsics_camextrinsics")
            dframe = np.diff(np.concatenate(([-1], ib[:, 0])))
            if (dframe < 0).any():
                raise RuntimeError("iframe MUST be monotonically increasing in indices_frame_camintrinsics_camextrinsics")
            if (dframe > 1).any():
                raise RuntimeError("iframe MUST be increasing sequentially in indices_frame_camintrinsics_camextrinsics")
            same = dframe[1:] == 0
            if (np.diff(ib[:, 1])[same] < 0).any():
                raise RuntimeError("icam_intrinsics MUST be monotonically increasing within a frame in "
                                   "indices_frame_camintrinsics_camextrinsics")
            if (np.diff(ib[:, 2])[same] < 0).any():
                raise RuntimeError("icam_extrinsics MUST be monotonically increasing within a frame in "
                                   "indices_frame_camintrinsics_camextrinsics")
            if ib[-1, 0] != self.Nframes - 1:
                raise RuntimeError("iframe in indices_frame_camintrinsics_camextrinsics must cover ALL frames. "
                                   f"Instead the last row has iframe={ib[-1, 0]}, but Nframes={self.Nframes}")
        if self.Npoints > 0:
            if self.Npoints_fixed > self.Npoints:
                raise RuntimeError(f"I have Npoints=len(points)={self.Npoints}, but Npoints_fixed={self.Npoints_fixed}. "
                                   "Npoints_fixed > Npoints makes no sense")
        elif self.Npoints_fixed:
            raise RuntimeError("No 'points' were given, so it's 'Npoints_fixed' doesn't do anything, and shouldn't be given")
        ip = self.indices_point
        if self.Nobs_point:
            if (ip[:, 0] < 0).any() or (ip[:, 0] >= self.Npoints).any():
                raise RuntimeError(f"i_point MUST be in [0,{self.Npoints - 1}] in indices_point_camintrinsics_camextrinsics")
            if (ip[:, 1] < 0).any() or (ip[:, 1] >= self.Ncam_i).any():
                raise RuntimeError(f"icam_intrinsics MUST be in [0,{self.Ncam_i - 1}] in indices_point_camintrinsics_camextrinsics")
            if (ip[:, 2] < -1).any() or (ip[:, 2] >= self.Ncam_e).any():
                raise RuntimeError(f"icam_extrinsics MUST be in [-1,{self.Ncam_e - 1}] in indices_point_camintrinsics_camextrinsics")
            running_max = np.maximum.accumulate(ip[:, 0])
            prev_max = np.concatenate(([-1], running_max[:-1]))
            if (ip[:, 0] > prev_max + 1).any():
                raise RuntimeError("indices_point_camintrinsics_camextrinsics should contain i_point that extend the "
                                   "existing set by one point at a time at most")
            biggest = running_max[-1]
        else:
            biggest = -1
        if biggest != self.Npoints - 1:
            raise RuntimeError(f"indices_point_camintrinsics_camextrinsics should cover all point indices in "
                               f"[0,{self.Npoints - 1}], but there are gaps. The biggest i_point={biggest}")

    # C-side observation structs: (icam_intrinsics, icam_extrinsics, iframe|i_point).
    # The Python arrays are (iframe|i_point, icam_intrinsics, icam_extrinsics): mrcal-pywrap.c:1246-1309
    def c_observations(self):
        ob = np.ascontiguousarray(self.indices_board[:, (1, 2, 0)]) if self.Nobs_board else np.zeros((0, 3), np.int32)
        op = np.ascontiguousarray(self.indices_point[:, (1, 2, 0)]) if self.Nobs_point else np.zeros((0, 3), np.int32)
        return ob, op

    def c_triangulated(self, rays=False):
        """(pointer, count) of the mrcal_observation_point_triangulated_t array: the pixel observations are
        unprojected to rays with the (fixed) intrinsics of their camera, weight <= 0 marks an outlier, the last
        observation of each point closes its set (mrcal-pywrap.c:1311-1440). The layout functions only look at
        the sets: rays=False leaves the rays zero (and needs no GPU)."""
        if self.Nobs_tri == 0:
            return None, 0
        if getattr(self, "_tri", None) is None or (rays and not self._tri_has_rays):
            it = self.indices_tri
            want = rays
            rays = np.zeros((self.Nobs_tri, 3))
            if want and self.observations_tri.shape[0] and self.intrinsics.shape[0]:
                _require_gpu()
                for icam in np.unique(it[:, 1]):
                    sel = np.flatnonzero(it[:, 1] == icam)
                    q = np.ascontiguousarray(self.observations_tri[sel, :2])
                    v = np.zeros((len(sel), 3))
                    intr = np.ascontiguousarray(self.intrinsics[icam])
                    checked.mrcal_unproject(_ptr(v), _ptr(q), len(sel), self.lm_ref(), _ptr(intr))
                    rays[sel] = v
            arr = (_capi.ObservationPointTriangulated * self.Nobs_tri)()
            last = np.concatenate((np.diff(it[:, 0]) != 0, [True]))
            for i in range(self.Nobs_tri):
                arr[i].icam_intrinsics = int(it[i, 1])
                arr[i].icam_extrinsics = int(it[i, 2])
                arr[i].bits = (1 if last[i] else 0) | (2 if self.observations_tri[i, 2] <= 0.0 else 0)
                arr[i].px[0], arr[i].px[1], arr[i].px[2] = rays[i]
            self._tri = arr
            self._tri_has_rays = bool(want)
        return self._tri, self.Nobs_tri

    def c_problem(self):
        """The arguments intrinsics .. problem_selections that mrcal_optimizer_callback(), mrcal_optimize() and
        mrcal_b200_problem_create_triangulated() share, with the triangulated observations as rays. The pointers keep
        their arrays alive"""
        ob, op = self.c_observations()
        tri, ntri = self.c_triangulated(rays=True)
        return (_ptr(self.intrinsics), _ptr(self.rt_cam_ref), _ptr(self.rt_ref_frame), _ptr(self.points),
                _ptr(self.calobject_warp), self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed,
                _ptr(ob), _ptr(op), self.Nobs_board, self.Nobs_point, tri, ntri,
                _ptr(self.observations_board), _ptr(self.observations_point), self.lm_ref(), _ptr(self.imagersizes),
                self.selections)

    def counts(self):
        return (self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed, self.Nobs_board)

    def lm_ref(self):
        if self.lensmodel is None:
            raise RuntimeError("The 'lensmodel' argument is required")
        return C.byref(self.lensmodel)

    def num_states(self):
        return checked.mrcal_num_states(*self.counts(), self.selections, self.lm_ref())

    def num_measurements(self):
        tri, ntri = self.c_triangulated()
        return checked.mrcal_num_measurements(self.Nobs_board, self.Nobs_point, tri, ntri, self.W, self.H,
                                              self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed,
                                              self.selections, self.lm_ref())

    def num_j_nonzero(self):
        ob, op = self.c_observations()
        tri, ntri = self.c_triangulated()
        return checked._mrcal_num_j_nonzero(self.Nobs_board, self.Nobs_point, tri, ntri, self.W, self.H,
                                            self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed,
                                            _ptr(ob), _ptr(op), self.selections, self.lm_ref())


def _require_gpu():
    if checked.mrcal_b200_device_count() <= 0:
        raise RuntimeError("mrcal_b200: no usable CUDA device. This backend has no CPU fallback")


####################################################################################################
# the hot path
####################################################################################################
def drt_cross_reprojection__dbpacked(icam_intrinsics=-1, **kwargs):
    """K = drt_ref_refperturbed/db_packed (icam_intrinsics < 0) or drt_cam_camperturbed/db_packed for that camera, as
    mrcal.drt_cross_reprojection__dbpacked(icam_intrinsics=..., **optimization_inputs) returns it (mrcal-pywrap.c:2016-2110;
    used by mrcal/model_analysis.py:1379,1441): shape (6, Nstate), zero outside the extrinsics, frames, points and
    calobject_warp columns. The Jacobian is evaluated at the given state and reduced on the device
    (csrc/cross_reprojection.cu; reference: _mrcal_drt_cross_reprojection__dbpacked, uncertainty.c:798)."""
    _require_gpu()
    P = Problem(**kwargs)
    try:
        return P.drt_cross_reprojection__dbpacked(icam_intrinsics)
    finally:
        P.close()


_UNCERTAINTY_METHODS = {"mean-pcam": 0, "cross-reprojection-rrp-Jfp": 1, "cross-reprojection-ccp": 2}   # mrcal_b200.h


def worst_direction_stdev(cov):
    """sqrt of the larger eigenvalue of each 2x2 covariance (..., 2, 2), in closed form"""
    cov = np.asarray(cov, np.float64)
    a, b, c = cov[..., 0, 0], cov[..., 0, 1], cov[..., 1, 1]
    return np.sqrt((a + c) / 2. + np.sqrt(((a - c) / 2.) ** 2 + b * b))


def projection_uncertainty(p_cam, model, *, method="cross-reprojection-ccp", atinfinity=False, what="covariance",
                           observed_pixel_uncertainty=None):
    """The uncertainty of the projection of the camera-frame points p_cam (..., 3) by the camera of `model`, propagated
    from the noise of the calibration's pixel observations, as mrcal.projection_uncertainty() computes it
    (mrcal/model_analysis.py:1192-1517). The model must carry optimization_inputs; its own (possibly edited)
    extrinsics are not used. what='covariance' returns (..., 2, 2); 'worstdirection-stdev' and 'rms-stdev' return
    (...). observed_pixel_uncertainty=None estimates it from the residuals at the solution."""
    known_methods = set(_UNCERTAINTY_METHODS)
    if method not in known_methods:
        raise RuntimeError(f"Unknown uncertainty method: '{method}'. I know about {known_methods}")
    what_known = {"covariance", "worstdirection-stdev", "rms-stdev"}
    if what not in what_known:
        raise RuntimeError(f"'what' kwarg must be in {what_known}, but got '{what}'")
    icam_intrinsics = model.icam_intrinsics()
    optimization_inputs = model.optimization_inputs()
    if optimization_inputs is None:
        raise RuntimeError("optimization_inputs are unavailable in this model. Uncertainty cannot be computed")
    _require_gpu()
    p = np.asarray(p_cam, np.float64)
    if p.shape[-1:] != (3,):
        raise RuntimeError(f"p_cam must have shape (...,3); got {p.shape}")
    P = Problem(**optimization_inputs)
    try:
        Var, _ = P.projection_uncertainty(p.reshape(-1, 3), icam_intrinsics, method=method, atinfinity=atinfinity,
                                          observed_pixel_uncertainty=observed_pixel_uncertainty)
    finally:
        P.close()
    Var = Var.reshape(p.shape[:-1] + (2, 2))
    if what == "covariance":
        return Var
    if what == "worstdirection-stdev":
        return worst_direction_stdev(Var)
    return np.sqrt((Var[..., 0, 0] + Var[..., 1, 1]) / 2.)


####################################################################################################
# comparing camera models (mrcal/utils.py:268-450, mrcal/model_analysis.py:27-395, 1520-1928)
####################################################################################################
def sample_imager(gridn_width, gridn_height, imager_width, imager_height):
    """A regular grid over the imager, shape (gridn_height, gridn_width, 2) of (x, y): [0,0] is (0,0), [-1,-1] is
    (W-1, H-1). gridn_height=None keeps the grid square-ish: int(round(H/W*gridn_width))"""
    if gridn_height is None:
        gridn_height = int(round(imager_height / imager_width * gridn_width))
    w = np.linspace(0, imager_width - 1, gridn_width)
    h = np.linspace(0, imager_height - 1, gridn_height)
    return np.ascontiguousarray(np.stack(np.meshgrid(w, h), axis=-1))


def sample_imager_unproject(gridn_width, gridn_height, imager_width, imager_height, lensmodel, intrinsics_data,
                            normalize=False):
    """(v, q): the grid of sample_imager() and its unprojection. One camera (lensmodel a string): v (Nh, Nw, 3). A
    list or tuple of lens models: v (Ncameras, Nh, Nw, 3), each camera unprojecting the same grid"""
    q = sample_imager(gridn_width, gridn_height, imager_width, imager_height)

    def unp(lm, intr):
        v = unproject(q, lm, intr)
        return v / np.linalg.norm(v, axis=-1)[..., None] if normalize else v
    if isinstance(lensmodel, (list, tuple)):
        return np.array([unp(lensmodel[i], intrinsics_data[i]) for i in range(len(lensmodel))]), q
    return unp(lensmodel, intrinsics_data), q


def _as_points(a, n, name):
    a = np.ascontiguousarray(a, np.float64)
    if a.ndim == 0 or a.shape[-1] != n:
        raise RuntimeError(f"{name} must have shape (...,{n}); got {a.shape}")
    return a


def implied_Rt10__from_unprojections(q0, p0, v1, *, weights=None, atinfinity=True, focus_center=(0., 0.),
                                     focus_radius=1.0e8):
    """The Rt transformation (4,3) from camera 0 to camera 1 that best lines up the unprojections p0 (..., Nh, Nw, 3)
    of camera 0 (unit vectors at infinity, else points) with the unit vectors v1 (Nh, Nw, 3) of camera 1 over the grid
    q0 (Nh, Nw, 2), as mrcal.implied_Rt10__from_unprojections() fits it. Leading dimensions of p0 and weights
    (..., Nh, Nw) are fitted together. atinfinity fits a rotation only (t = 0). Only grid points strictly within
    focus_radius of focus_center are used; non-finite rays and weights are ignored. The fit runs on the device
    (csrc/diff.cu)"""
    _require_gpu()
    q0 = _as_points(q0, 2, "q0").reshape(-1, 2)
    N = q0.shape[0]
    p0 = _as_points(p0, 3, "p0")
    v1 = _as_points(v1, 3, "v1").reshape(-1, 3)
    if v1.shape[0] != N or N == 0 or p0.size % (3 * N):
        raise RuntimeError(f"q0, p0, v1 must describe the same grid; got shapes {q0.shape}, {p0.shape}, {v1.shape}")
    p0 = p0.reshape(-1, N, 3)
    M = p0.shape[0]
    if weights is not None:
        weights = np.ascontiguousarray(weights, np.float64)
        if weights.size != M * N:
            raise RuntimeError(f"weights must have the shape of p0 without its last dimension; got {weights.shape}")
    fc = np.ascontiguousarray(focus_center, np.float64).reshape(2)
    Rt = np.zeros((4, 3))
    checked.mrcal_b200_implied_Rt10__from_unprojections(_ptr(Rt), _ptr(q0), N, _ptr(p0), M, _ptr(v1), _ptr(weights),
                                                        bool(atinfinity), _ptr(fc), float(focus_radius))
    return Rt


def _identity_Rt():
    return np.vstack((np.eye(3), np.zeros(3)))


def projection_diff(models, *, implied_Rt10=None, gridn_width=60, gridn_height=None, intrinsics_only=False,
                    distance=None, use_uncertainties=True, focus_center=None, focus_radius=-1.):
    """The difference in projection between camera models, as mrcal.projection_diff() computes it. Returns
    (difflen, diff, q0, Rt10): difflen (..., Nh, Nw) the length of the projection difference (2 models) or
    sqrt(mean_k |q_k - q0|^2) over models 1..N-1 (more); diff (..., Nh, Nw, 2) or None for more than 2 models; q0 the
    grid (Nh, Nw, 2); Rt10 (4,3), or (Nmodels-1, 4, 3), the transformations from camera 0 to each other camera. An
    iterable distance adds a leading dimension. Rt10 is implied_Rt10 if given, the identity if intrinsics_only, the
    models' relative extrinsics if focus_radius == 0, and otherwise fitted, weighted by the projection uncertainties
    if use_uncertainties and the models carry optimization_inputs. The fit and the reprojections run on the device
    (csrc/diff.cu), all pairs of models in one call"""
    if len(models) < 2:
        raise RuntimeError("At least 2 models are required to compute the diff")
    if len(models) > 2 and implied_Rt10 is not None:
        raise RuntimeError("A given implied_Rt10 is currently supported ONLY if exactly 2 models are being compared")
    try:
        len(distance)
        distance_is_iterable = True
    except TypeError:
        distance_is_iterable = False
    atinfinity = distance is None
    dist = np.ones(1) if atinfinity else np.ascontiguousarray(np.atleast_1d(np.array(distance, np.float64)).ravel())

    imagersizes = np.array([m.imagersize() for m in models])
    if np.linalg.norm(np.std(imagersizes, axis=-2)) != 0:
        raise RuntimeError(f"The diff function needs all the imager dimensions to match. Instead got {imagersizes}")
    W, H = imagersizes[0]
    lensmodels = [m.intrinsics()[0] for m in models]
    intrinsics_data = [m.intrinsics()[1] for m in models]
    # noncentral models (model_analysis.py:1759-1772)
    for i in range(len(models)):
        if lensmodel_metadata_and_config(lensmodels[i])["noncentral"] and not \
           (re.match("LENSMODEL_CAHVORE_", lensmodels[i]) and np.sum(intrinsics_data[i][-3:] ** 2) < 1e-12):
            if not atinfinity:
                raise RuntimeError(f"Model {i} is noncentral, so I can only evaluate the diff at infinity")
            if re.match("LENSMODEL_CAHVORE_", lensmodels[i]):
                if use_uncertainties:
                    raise RuntimeError("I have a noncentral model. No usable uncertainties for those yet")
                intrinsics_data[i][-3:] = 0   # a copy: centralize CAHVORE
            else:
                raise RuntimeError("I have a non-CAHVORE noncentral model. This isn't supported yet")

    v, q0 = sample_imager_unproject(gridn_width, gridn_height, W, H, lensmodels, intrinsics_data, normalize=True)
    Nmodels, Nd = len(models), dist.size

    uncertainties = None
    if use_uncertainties and not intrinsics_only and focus_radius != 0 and implied_Rt10 is None:
        try:
            uncertainties = np.array([projection_uncertainty(v[i] * dist[:, None, None, None], models[i],
                                                             atinfinity=atinfinity, what="worstdirection-stdev")
                                      for i in range(Nmodels)])
        except Exception as e:
            print("WARNING: projection_diff() was asked to use uncertainties, but they aren't available/couldn't be "
                  f"computed. Falling back on the region-based-only logic. Caught exception: {e}", file=sys.stderr)
    if focus_center is None:
        focus_center = ((W - 1.) / 2., (H - 1.) / 2.)
    if focus_radius < 0:
        focus_radius = float(max(W, H) * 100.) if uncertainties is not None else float(min(W, H) / 6.)

    fit = False
    if implied_Rt10 is not None:
        Rt10 = np.array(implied_Rt10, np.float64).reshape(1, 4, 3)
    elif intrinsics_only:
        Rt10 = np.array([_identity_Rt()] * (Nmodels - 1))
    elif focus_radius == 0:
        Rt10 = np.array([compose_Rt(models[k].Rt_cam_ref(), models[0].Rt_ref_cam()) for k in range(1, Nmodels)])
    else:
        Rt10 = np.zeros((Nmodels - 1, 4, 3))
        fit = True

    lms = (_capi.Lensmodel * Nmodels)(*[_lensmodel(lm) for lm in lensmodels])
    intr = np.ascontiguousarray(np.concatenate(intrinsics_data), np.float64)
    vv = np.ascontiguousarray(v.reshape(Nmodels, -1, 3))
    qq = q0.reshape(-1, 2)
    N = qq.shape[0]
    difflen = np.zeros((Nd, N))
    diff = np.zeros((Nd, N, 2)) if Nmodels == 2 else None
    fc = np.ascontiguousarray(focus_center, np.float64).reshape(2)
    U = np.ascontiguousarray(uncertainties.reshape(Nmodels, Nd, N)) if uncertainties is not None and fit else None
    checked.mrcal_b200_projection_diff(_ptr(Rt10), _ptr(difflen), _ptr(diff), _ptr(qq), N, _ptr(vv), Nmodels,
                                       None if atinfinity else _ptr(dist), Nd, lms, _ptr(intr), _ptr(U), _ptr(fc),
                                       float(focus_radius), fit)

    difflen = difflen.reshape((Nd,) + q0.shape[:2])
    if diff is not None:
        diff = diff.reshape((Nd,) + q0.shape)
    if not distance_is_iterable:
        difflen = difflen[0]
        if diff is not None:
            diff = diff[0]
    if implied_Rt10 is not None:
        return difflen, diff, q0, implied_Rt10
    return difflen, diff, q0, (Rt10[0] if Nmodels == 2 else Rt10)


_RESOLUTION_MODES = {"mean": 0, "min": 1, "max": 2, "eccentricity": 3}   # MB200_RESOLUTION_* in mrcal_b200.h


def model_resolution__deg_pixel(q, model, *, mode="mean"):
    """The angular resolution of the camera of `model` at pixels q (...,2), in degrees per pixel, as
    mrcal.model_resolution__deg_pixel() computes it (mrcal/model_analysis.py:2152-2246): from the sensitivity of the
    projection to motions perpendicular to each unit ray. mode 'min' and 'max' report the finest and the coarsest
    direction, 'mean' their average and 'eccentricity' max/min. One fused kernel on the device (csrc/project.cu)"""
    if mode not in _RESOLUTION_MODES:
        raise RuntimeError("Mode must be one of ('min','max','mean','eccentricity')")
    _require_gpu()
    q = np.ascontiguousarray(q, dtype=np.float64)
    if q.shape[-1:] != (2,):
        raise RuntimeError(f"q must have shape (...,2); got {q.shape}")
    lensmodel, intrinsics = model.intrinsics()
    lm = _lensmodel(lensmodel)
    intr = np.ascontiguousarray(intrinsics, dtype=np.float64)
    flat = q.reshape(-1, 2)
    out = np.zeros(flat.shape[0])
    checked.mrcal_b200_model_resolution__deg_pixel(_ptr(out), _ptr(flat), flat.shape[0], C.byref(lm), _ptr(intr),
                                                   _RESOLUTION_MODES[mode])
    return out.reshape(q.shape[:-1])


def _stereo_pair_reproject(q, models, Rts, distance):
    """out, |out|: the pixels q (...,2) of camera 0 of each (camera 0, camera 1) pair in models, reprojected into its
    camera 1 through Rt (4,3) from camera 0 to camera 1: q1 for one pair, q1[1] - q1[0] for two"""
    q = np.ascontiguousarray(q, dtype=np.float64)
    if q.shape[-1:] != (2,):
        raise RuntimeError(f"q must have shape (...,2); got {q.shape}")
    flat = q.reshape(-1, 2)
    lms = (_capi.Lensmodel * len(models))(*[_lensmodel(lm) for lm, _ in models])
    intr = np.ascontiguousarray(np.concatenate([i for _, i in models]), np.float64)
    Rt = np.ascontiguousarray(Rts, np.float64)
    out = np.zeros(flat.shape)
    outlen = np.zeros(flat.shape[0])
    checked.mrcal_b200_stereo_pair_reproject(_ptr(out), _ptr(outlen), _ptr(flat), flat.shape[0], len(models) // 2, lms,
                                             _ptr(intr), _ptr(Rt), float(distance))
    return out.reshape(q.shape), outlen.reshape(q.shape[:-1])


def stereo_pair_diff(model_pairs, *, gridn_width=60, gridn_height=None, distance=None):
    """The difference between two calibrations of a camera pair, intrinsics and extrinsics together, as
    mrcal.stereo_pair_diff() computes it (mrcal/model_analysis.py:1931-2103): a grid q0 over the imager of camera 0 is
    unprojected by each pair's camera 0 to the distance (infinity if None: distance 1 and no translation), mapped to
    camera 1 by that pair's Rt10 = Rt_cam_ref(m1) Rt_ref_cam(m0) and projected by its camera 1. Returns (difflen, diff,
    q0, reproject_pairp_from_cami): diff (Nh, Nw, 2) = q1[pair 1] - q1[pair 0], difflen its length, q0 the grid (Nh, Nw,
    2), and reproject_pairp_from_cami(q, p, i) mapping pixels q of camera i of pair p to the other camera of that pair.
    A noncentral CAHVORE model is centralized (E = 0) in a copy where that is exact (|E|^2 < 1e-12) or at infinity. The
    unprojections and reprojections run on the device (csrc/diff.cu)"""
    if len(model_pairs) != 2:
        raise RuntimeError("Exactly 2 model_pairs are expected")
    Rt10_pairs = np.array([compose_Rt(m1.Rt_cam_ref(), m0.Rt_ref_cam()) for m0, m1 in model_pairs])
    atinfinity = distance is None
    if atinfinity:
        distance = 1.
        Rt10_pairs[:, 3, :] = 0
    intrinsics = [[m.intrinsics() for m in pair] for pair in model_pairs]
    for pair in intrinsics:
        for i, (lm, intr) in enumerate(pair):
            if not lensmodel_metadata_and_config(lm)["noncentral"]:
                continue
            if not re.match("LENSMODEL_CAHVORE_", lm):
                raise RuntimeError("I have a noncentral model that I cannot centralize. unproject() isn't implemented "
                                   "yet in this case")
            if np.sum(intr[-3:] ** 2) < 1e-12 or atinfinity:
                intr = np.array(intr, np.float64)
                intr[-3:] = 0
                pair[i] = (lm, intr)
                continue
            raise RuntimeError("I have a noncentral model. I can centralize it, but that's only valid at infinity")
    imagersizes0 = np.array([pair[0].imagersize() for pair in model_pairs])
    if np.any(imagersizes0[1] - imagersizes0[0]):
        raise RuntimeError("The first camera in each given pair MUST have identical imager dimensions")
    imagersizes1 = np.array([pair[1].imagersize() for pair in model_pairs])
    if np.any(imagersizes1[1] - imagersizes1[0]):
        raise RuntimeError("The second camera in each given pair must have identical imager dimensions. I technically "
                           "don't NEED this, but it's extremely likely to be an unintentional mistake by the caller")
    Rt10_Rt01_pairs = (Rt10_pairs, invert_Rt(Rt10_pairs))
    d = float(distance)

    def reproject_pairp_from_cami(q, p, i):
        return _stereo_pair_reproject(q, (intrinsics[p][i], intrinsics[p][1 - i]), Rt10_Rt01_pairs[i][p][None], d)[0]

    q0 = sample_imager(gridn_width, gridn_height, *imagersizes0[0])
    diff, difflen = _stereo_pair_reproject(q0, intrinsics[0] + intrinsics[1], Rt10_pairs, d)
    return difflen, diff, q0, reproject_pairp_from_cami


def optimizer_callback(no_jacobian=False, no_factorization=False, **kwargs):
    """One evaluation of the cost function at the given seed.

    Returns (b_packed, x, J, factorization), as mrcal.optimizer_callback() does
    (mrcal-pywrap.c:2008-2012): b_packed (Nstate,), x (Nmeasurements,), J a
    scipy.sparse.csr_matrix of shape (Nmeasurements,Nstate) with int32 indices
    (None if no_jacobian), factorization a CHOLMOD_factorization-like object
    (None if no_jacobian or no_factorization, or if JtJ is not positive definite)."""
    _require_gpu()
    I = _Inputs(kwargs)
    if not no_factorization:
        no_jacobian = False   # mrcal-pywrap.c:1709-1710
    Nstate, Nmeas = I.num_states(), I.num_measurements()
    b = np.zeros(Nstate)
    x = np.zeros(Nmeas)
    Jt, keep = None, None
    if not no_jacobian:
        nnz = I.num_j_nonzero()
        P = np.zeros(Nmeas + 1, np.int32)
        Ii = np.zeros(nnz, np.int32)
        X = np.zeros(nnz, np.float64)
        Jt = _capi.Sparse(nrow=Nstate, ncol=Nmeas, nzmax=nnz, p=P.ctypes.data, i=Ii.ctypes.data, x=X.ctypes.data,
                          sorted=1, packed=1)
        keep = (P, Ii, X)
    checked.mrcal_optimizer_callback(_ptr(b), b.nbytes, _ptr(x), x.nbytes, C.byref(Jt) if Jt is not None else None,
                                     *I.c_problem(), None, I.spacing, max(I.W, 0), max(I.H, 0), I.verbose)
    J = None
    factorization = None
    if keep is not None:
        P, Ii, X = keep
        J = scipy.sparse.csr_matrix((X, Ii, P), shape=(Nmeas, Nstate))
        if not no_factorization:
            # the problem's own structure (frames/points eliminated, dense factor of the reduced system only); the dense
            # Nstate x Nstate object on request.
            # "JtJ is not positive definite" is not an error here: mrcal-pywrap.c:1981-1988 returns None. Anything else
            # (out of memory, a CUDA failure) is one
            if os.environ.get("MRCAL_B200_DENSE_FACTORIZATION"):
                try:
                    factorization = CHOLMOD_factorization(J)
                except RuntimeError as e:
                    if "not positive definite" not in str(e):
                        raise
                    factorization = None
            else:
                h = checked.mrcal_b200_factorization_create_from_last_callback()   # NULL comes back as None
                if h:
                    factorization = CHOLMOD_factorization._from_handle(h, J.shape)
                elif "not positive definite" not in _capi.last_error():
                    raise RuntimeError("mrcal_optimizer_callback(): factorization failed: " + _capi.last_error() +
                                       " (MRCAL_B200_DENSE_FACTORIZATION=1 gives the dense factorization of J'J instead)")
    return b, x, J, factorization


def optimize(**kwargs):
    """Solve the calibration problem. Returns the reference's stats dict
    (mrcal-pywrap.c:1851-1889) and writes the solution INTO the given intrinsics,
    rt_cam_ref, rt_ref_frame, points, calobject_warp arrays; outliers are marked
    by negating observations_board[...,2]."""
    _require_gpu()
    I = _Inputs(kwargs)
    for name, a in (("intrinsics", I.intrinsics), ("rt_cam_ref", I.rt_cam_ref), ("rt_ref_frame", I.rt_ref_frame),
                    ("points", I.points), ("observations_board", I.observations_board)):
        if a.size and not a.flags.writeable:
            raise RuntimeError(f"'{name}' must be writeable: optimize() stores its results there")
    Nstate, Nmeas = I.num_states(), I.num_measurements()
    b = np.zeros(Nstate)
    x = np.zeros(Nmeas)
    stats = checked.mrcal_optimize(_ptr(b), b.nbytes, _ptr(x), x.nbytes, *I.c_problem(), None, I.spacing, max(I.W, 0),
                                   max(I.H, 0), I.verbose, False)
    if stats.rms_reproj_error__pixels < 0.0:
        raise RuntimeError("mrcal.optimize() failed! " + _capi.last_error())
    return dict(rms_reproj_error__pixels=stats.rms_reproj_error__pixels,
                Noutliers_board=stats.Noutliers_board,
                Noutliers_triangulated_point=stats.Noutliers_triangulated_point,
                b_packed=b, x=x)


def check_gradient(**kwargs):
    """The reference's gradient self-check, mrcal_optimize(..., check_gradient=true) (mrcal.c:6601-6605; driven by
    test/test-gradients.c + test/test-gradients.py): every column of the Jacobian against a forward difference of
    the residuals. The C entry point prints libdogleg's vnlog to stdout; this helper captures and parses it.
    Returns an array of rows (ivar, imeasurement, gradient_reported, gradient_observed)."""
    import os
    import tempfile
    _require_gpu()
    I = _Inputs(kwargs)
    problem = I.c_problem()
    sys_stdout_fd = 1
    with tempfile.TemporaryFile(mode="w+b") as tmp:
        import sys as _sys
        _sys.stdout.flush()
        saved = os.dup(sys_stdout_fd)
        os.dup2(tmp.fileno(), sys_stdout_fd)
        try:
            checked.mrcal_optimize(None, 0, None, 0, *problem, None, I.spacing, max(I.W, 0), max(I.H, 0), False, True)
        finally:
            os.dup2(saved, sys_stdout_fd)
            os.close(saved)
        tmp.seek(0)
        rows = [l.split() for l in tmp.read().decode().splitlines() if l and not l.startswith("#")]
    if not rows:
        raise RuntimeError("check_gradient produced no output: " + _capi.last_error())
    return np.array([[float(v) for v in r[:4]] for r in rows])


class Problem:
    """Device-resident problem (extension; include/mrcal_b200.h part 2): upload
    once, then solve / evaluate repeatedly without touching the host inputs."""

    def __init__(self, **kwargs):
        _require_gpu()
        I = self._I = _Inputs(kwargs)
        self._h = C.c_void_p(checked.mrcal_b200_problem_create_triangulated(*I.c_problem(), I.spacing, max(I.W, 0),
                                                                            max(I.H, 0)))
        self.Nstate = checked.mrcal_b200_problem_num_states(self._h)
        self.Nmeasurements = checked.mrcal_b200_problem_num_measurements(self._h)
        self.N_j_nonzero = checked.mrcal_b200_problem_num_j_nonzero(self._h)

    def close(self):
        if getattr(self, "_h", None):
            checked.mrcal_b200_problem_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, b_packed=None):
        if b_packed is not None:
            b_packed = np.ascontiguousarray(b_packed, np.float64)
            assert b_packed.shape == (self.Nstate,)
        checked.mrcal_b200_problem_reset(self._h, _ptr(b_packed))

    def upload(self):
        """Re-send the seed and the observation pool from the host arrays given at construction."""
        I = self._I
        checked.mrcal_b200_problem_upload(self._h, _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame),
                                          _ptr(I.points), _ptr(I.calobject_warp), _ptr(I.observations_board),
                                          _ptr(I.observations_point))

    def drt_cross_reprojection__dbpacked(self, icam_intrinsics=-1):
        """K (6, Nstate) at the problem's current state: see the module-level function."""
        K = np.zeros((6, self.Nstate))
        checked.mrcal_b200_problem_drt_cross_reprojection__dbpacked(self._h, int(icam_intrinsics), _ptr(K))
        return K

    def projection_uncertainty(self, p_cam, icam_intrinsics, method="cross-reprojection-ccp", atinfinity=False,
                               observed_pixel_uncertainty=None):
        """(Var, sigma): the raw (N,2,2) covariances of the projections of the points p_cam (N,3) by camera
        icam_intrinsics at the problem's current state, and the observed-pixel uncertainty used (estimated from the
        residuals if None). Everything but the reshaping runs on the device (csrc/uncertainty.cu)"""
        if method not in _UNCERTAINTY_METHODS:
            raise RuntimeError(f"Unknown uncertainty method: '{method}'. I know about {set(_UNCERTAINTY_METHODS)}")
        p = np.ascontiguousarray(p_cam, np.float64)
        if p.ndim != 2 or p.shape[1] != 3:
            raise RuntimeError(f"p_cam must have shape (N,3); got {p.shape}")
        Var = np.zeros((p.shape[0], 2, 2))
        sigma = C.c_double(0.)
        s = -1.0 if observed_pixel_uncertainty is None else float(observed_pixel_uncertainty)
        if observed_pixel_uncertainty is not None and not s > 0:
            raise RuntimeError("observed_pixel_uncertainty must be > 0 (or None to estimate it)")
        checked.mrcal_b200_problem_projection_uncertainty(self._h, int(icam_intrinsics), _UNCERTAINTY_METHODS[method],
                                                         bool(atinfinity), _ptr(p), p.shape[0], s, _ptr(Var),
                                                         C.byref(sigma))
        return Var, sigma.value

    def projection_uncertainty_cameras(self, p_cams, icams_intrinsics, method="cross-reprojection-ccp", atinfinity=False,
                                       observed_pixel_uncertainty=None):
        """([Var], sigma): projection_uncertainty() of the points p_cams[k] (N_k,3) by camera icams_intrinsics[k], for
        every k from one evaluation and factorization of the problem. Each Var equals what projection_uncertainty()
        gives for that camera alone, bit for bit"""
        if method not in _UNCERTAINTY_METHODS:
            raise RuntimeError(f"Unknown uncertainty method: '{method}'. I know about {set(_UNCERTAINTY_METHODS)}")
        if len(p_cams) != len(icams_intrinsics):
            raise RuntimeError("p_cams and icams_intrinsics must have the same length")
        ps = [np.ascontiguousarray(p, np.float64) for p in p_cams]
        for p in ps:
            if p.ndim != 2 or p.shape[1] != 3:
                raise RuntimeError(f"each p_cam must have shape (N,3); got {p.shape}")
        N = np.array([p.shape[0] for p in ps], np.int32)
        icams = np.array(icams_intrinsics, np.int32).reshape(-1)
        p_all = np.ascontiguousarray(np.concatenate(ps) if ps else np.zeros((0, 3)))
        Var = np.zeros((p_all.shape[0], 2, 2))
        sigma = C.c_double(0.)
        s = -1.0 if observed_pixel_uncertainty is None else float(observed_pixel_uncertainty)
        if observed_pixel_uncertainty is not None and not s > 0:
            raise RuntimeError("observed_pixel_uncertainty must be > 0 (or None to estimate it)")
        checked.mrcal_b200_problem_projection_uncertainty_cameras(self._h, _ptr(icams), _ptr(N), len(ps),
                                                                 _UNCERTAINTY_METHODS[method], bool(atinfinity),
                                                                 _ptr(p_all), s, _ptr(Var), C.byref(sigma))
        return np.split(Var, np.cumsum(N)[:-1]), sigma.value

    def regional_statistics(self, icams_intrinsics, q_cell_center, rcell, evaluate=True):
        """(stats, x): the board residuals binned by imager cell for the cameras icams_intrinsics, one grid shape for
        all: stats (Ncameras, gridn_height, gridn_width, 3) of (mean, stdev, count), from the cell centres
        q_cell_center (Ncameras, gridn_height, gridn_width, 2) and half-sizes rcell (Ncameras, 2); x the residuals used.
        evaluate=False uses the residuals of the last evaluation (csrc/regions.cu)"""
        icams = np.array(icams_intrinsics, np.int32).reshape(-1)
        q = np.ascontiguousarray(q_cell_center, np.float64)
        r = np.ascontiguousarray(rcell, np.float64)
        if q.ndim != 4 or q.shape[0] != icams.size or q.shape[-1] != 2 or r.shape != (icams.size, 2):
            raise RuntimeError(f"q_cell_center must have shape (Ncameras,Nh,Nw,2) and rcell (Ncameras,2); got "
                               f"{q.shape} and {r.shape} for {icams.size} cameras")
        stats = np.zeros(q.shape[:-1] + (3,))
        x = np.zeros(self.Nmeasurements)
        checked.mrcal_b200_problem_regional_statistics(self._h, _ptr(icams), icams.size, q.shape[2], q.shape[1],
                                                       _ptr(q), _ptr(r), bool(evaluate), _ptr(stats), _ptr(x))
        return stats, x

    def callback(self, jacobian=True):
        b = np.zeros(self.Nstate)
        x = np.zeros(self.Nmeasurements)
        if jacobian:
            P = np.zeros(self.Nmeasurements + 1, np.int32)
            Ii = np.zeros(self.N_j_nonzero, np.int32)
            X = np.zeros(self.N_j_nonzero)
            checked.mrcal_b200_problem_callback(self._h, _ptr(b), _ptr(x), _ptr(P), _ptr(Ii), _ptr(X))
        else:
            checked.mrcal_b200_problem_callback(self._h, _ptr(b), _ptr(x), None, None, None)
        if not jacobian:
            return b, x, None
        return b, x, scipy.sparse.csr_matrix((X, Ii, P), shape=(self.Nmeasurements, self.Nstate))

    def optimize(self, **parameters):
        p = _capi.SolverParameters()
        checked.mrcal_b200_default_solver_parameters(C.byref(p))
        for k, v in parameters.items():
            if not hasattr(p, k):
                raise RuntimeError(f"unknown solver parameter '{k}'")
            setattr(p, k, v)
        stats = _capi.Stats()
        info = _capi.SolveInfo()
        checked.mrcal_b200_problem_optimize(self._h, C.byref(p), C.byref(stats), C.byref(info))
        out = dict(rms_reproj_error__pixels=stats.rms_reproj_error__pixels,
                   Noutliers_board=stats.Noutliers_board,
                   Noutliers_triangulated_point=stats.Noutliers_triangulated_point)
        out.update(info.asdict())
        return out

    def download(self, into_inputs=True):
        """Fetch b_packed, x and the unpacked solution; if into_inputs, store the
        solution in the arrays given at construction (like optimize())."""
        I = self._I
        b = np.zeros(self.Nstate)
        x = np.zeros(self.Nmeasurements)
        tgt = (I.intrinsics, I.rt_cam_ref, I.rt_ref_frame, I.points, I.calobject_warp, I.observations_board)
        if not into_inputs:
            tgt = tuple(None if a is None else a.copy() for a in tgt)
        intr, rtc, rtf, pts, warp, obs = tgt
        checked.mrcal_b200_problem_download(self._h, _ptr(b), _ptr(x), _ptr(intr), _ptr(rtc), _ptr(rtf), _ptr(pts),
                                            _ptr(warp), _ptr(obs))
        return dict(b_packed=b, x=x, intrinsics=intr, rt_cam_ref=rtc, rt_ref_frame=rtf, points=pts,
                    calobject_warp=warp, observations_board=obs)

    def reduced_system(self, lambda_=0.0, fused=False):
        """(S, g_reduced, g_full): the Schur-reduced normal equations at the current state (introspection).
        fused: the board observations' blocks come from the fused evaluation that optimize() uses for splined models
        with the core locked, not from the stored Jacobian (RuntimeError if this problem does not take that path)."""
        fn = checked.mrcal_b200_problem_reduced_system_fused if fused else checked.mrcal_b200_problem_reduced_system
        n = C.c_int(0)
        fn(self._h, lambda_, C.byref(n), None, None, None)
        S = np.zeros((n.value, n.value))
        g = np.zeros(n.value)
        gf = np.zeros(self.Nstate)
        fn(self._h, lambda_, C.byref(n), _ptr(S), _ptr(g), _ptr(gf))
        S = np.tril(S) + np.tril(S, -1).T
        return S, g, gf

    def cauchy_denominator(self, fused=False):
        """(|g|^2, |J g|^2), g = J'x at the current state, from the kernels an optimize() step runs (introspection).
        fused: the board rows from the fused evaluation's blocks, as in reduced_system(fused=True)."""
        out = np.zeros(2)
        checked.mrcal_b200_problem_cauchy_denominator(self._h, bool(fused), _ptr(out))
        return float(out[0]), float(out[1])

    def time_callback(self, N=10, jacobian=True):
        ms = checked.mrcal_b200_problem_time_callback(self._h, int(N), jacobian)
        if ms < 0:
            raise RuntimeError(_capi.last_error())
        return ms


class CHOLMOD_factorization:
    """Cholesky factorization of JtJ held on the GPU. Same surface as
    mrcal.CHOLMOD_factorization (mrcal-pywrap.c:110-649; known-answer test:
    test/test-CHOLMOD-factorization.py): construct from a scipy CSR matrix J;
    solve_xt_JtJ_bt(bt) solves JtJ x = b for each row of bt; rcond()."""

    def __init__(self, J):
        _require_gpu()
        if not scipy.sparse.issparse(J):
            raise RuntimeError("J must be a scipy.sparse matrix")
        J = scipy.sparse.csr_matrix(J)
        P = np.ascontiguousarray(J.indptr, np.int32)
        Ii = np.ascontiguousarray(J.indices, np.int32)
        X = np.ascontiguousarray(J.data, np.float64)
        self.shape = J.shape
        self._h = C.c_void_p(checked.mrcal_b200_factorization_create(_ptr(P) or P.ctypes.data_as(C.c_void_p), _ptr(Ii),
                                                                     _ptr(X), J.shape[0], J.shape[1]))

    @classmethod
    def _from_handle(cls, h, shape):
        self = cls.__new__(cls)
        self.shape = shape
        self._h = C.c_void_p(h)
        return self

    def __del__(self):
        if getattr(self, "_h", None):
            checked.mrcal_b200_factorization_destroy(self._h)
            self._h = None

    _SYS = ("A", "LDLt", "LD", "DLt", "L", "Lt", "D", "P", "Pt")   # mrcal-pywrap.c:467-476; codes of mrcal_b200.h

    def solve_xt_JtJ_bt(self, bt, sys="A"):
        """sys as in the reference (mrcal-pywrap.c:425-578, optionally spelled "CHOLMOD_..."). The factorization
        here is P JtJ Pt = L D Lt with P = I, D = I: "P","Pt","D" return bt, "L"/"LD" solve L x = b, "Lt"/"DLt"
        solve Lt x = b. CHOLMOD's own P and D differ; the identities between the systems hold."""
        name = sys[len("CHOLMOD_"):] if isinstance(sys, str) and sys.startswith("CHOLMOD_") else sys
        if name not in self._SYS:
            raise RuntimeError(f"Unknown sys '{sys}' given. Known values of sys: ({','.join(self._SYS)},)")
        code = self._SYS.index(name)
        bt = np.asarray(bt, dtype=np.float64)
        if bt.ndim < 1 or bt.shape[-1] != self.shape[1]:
            raise RuntimeError(f"bt must have shape (...,Nstate={self.shape[1]}); got {bt.shape}")
        flat = np.ascontiguousarray(bt.reshape(-1, self.shape[1]))
        out = np.empty_like(flat)
        if flat.shape[0]:
            checked.mrcal_b200_factorization_solve_sys(self._h, _ptr(out), _ptr(flat), flat.shape[0], code)
        return out.reshape(bt.shape)

    def rcond(self):
        return checked.mrcal_b200_factorization_rcond(self._h)


####################################################################################################
# consumers of the sparse Jacobian (the reference's _mrcal_npsp._Jt_x / _A_Jt_J_At, mrcal-genpywrap.py:477-731)
####################################################################################################
class _DeviceCSR:
    """A CSR matrix uploaded once; the last one is kept, keyed by the identity of the arrays, because the
    uncertainty code calls these functions over and over with the same J (mrcal/model_analysis.py:716-870)."""
    _last = None

    def __init__(self, Jp, Ji, Jx, Ncols):
        self.key = (Jp.ctypes.data, Ji.ctypes.data, Jx.ctypes.data, Jp.size, Ji.size, Ncols)
        self.Nrows, self.Ncols = Jp.size - 1, Ncols
        self._h = C.c_void_p(checked.mrcal_b200_csr_create(_ptr(Jp) or Jp.ctypes.data_as(C.c_void_p), _ptr(Ji),
                                                           _ptr(Jx), self.Nrows, Ncols))

    def __del__(self):
        if getattr(self, "_h", None):
            checked.mrcal_b200_csr_destroy(self._h)
            self._h = None

    @classmethod
    def get(cls, Jp, Ji, Jx, Ncols):
        _require_gpu()
        Jp = np.ascontiguousarray(Jp, np.int32)
        Ji = np.ascontiguousarray(Ji, np.int32)
        Jx = np.ascontiguousarray(Jx, np.float64)
        key = (Jp.ctypes.data, Ji.ctypes.data, Jx.ctypes.data, Jp.size, Ji.size, Ncols)
        if cls._last is None or cls._last.key != key:
            cls._last = cls(Jp, Ji, Jx, Ncols)
            cls._last._keep = (Jp, Ji, Jx)   # the key is only meaningful while the arrays live
        return cls._last


def _Jt_x(Jp, Ji, Jx, xt, out=None):
    """Jt*xt for a sparse J given as the indptr/indices/data of a scipy.sparse.csr_matrix; `out` (shape (Nstate,))
    must be given, as in the reference (mrcal-genpywrap.py:640-731: its length is the number of columns of J)."""
    if out is None:
        raise RuntimeError("_Jt_x(): the output array must be passed in: there is no other way to know the number of columns of J")
    xt = np.ascontiguousarray(xt, np.float64)
    if xt.ndim != 1 or xt.shape[0] != np.asarray(Jp).size - 1:
        raise RuntimeError("len(xt) must match the number of rows in J")
    if out.dtype != np.float64 or not out.flags.c_contiguous or out.ndim != 1:
        raise RuntimeError("out must be a contiguous 1-dimensional float64 array")
    J = _DeviceCSR.get(Jp, Ji, Jx, out.shape[0])
    checked.mrcal_b200_csr_Jt_x(J._h, _ptr(out), _ptr(xt))
    return out


def _A_Jt_J_At(A, Jp, Ji, Jx, Nleading_rows_J=-1, out=None):
    """matmult(A,Jt,J,At) over the Nleading_rows_J leading rows of a sparse J (mrcal-genpywrap.py:477-567).
    A: (...,Nx,Nstate), broadcast over the leading dimensions; returns (...,Nx,Nx)."""
    if Nleading_rows_J is None or Nleading_rows_J <= 0:
        raise RuntimeError("Nleading_rows_J must be passed, and must be > 0")
    A = np.asarray(A, np.float64)
    if A.ndim < 2:
        raise RuntimeError("A must have shape (...,Nx,Nstate)")
    Nx, Nstate = A.shape[-2:]
    J = _DeviceCSR.get(Jp, Ji, Jx, Nstate)
    flat = np.ascontiguousarray(A.reshape(-1, Nx, Nstate))
    res = np.zeros((flat.shape[0], Nx, Nx))
    for k in range(flat.shape[0]):
        checked.mrcal_b200_csr_A_Jt_J_At(J._h, _ptr(res[k]), _ptr(flat[k]), Nx, int(Nleading_rows_J))
    res = res.reshape(A.shape[:-2] + (Nx, Nx))
    if out is not None:
        out[...] = res
        return out
    return res


def _A_Jt_J_At__2(A, Jp, Ji, Jx, Nleading_rows_J=-1, out=None):
    """_A_Jt_J_At() for A.shape = (...,2,Nstate) (mrcal-genpywrap.py:569-638)."""
    if np.asarray(A).shape[-2] != 2:
        raise RuntimeError("_A_Jt_J_At__2(): A must have shape (...,2,Nstate)")
    return _A_Jt_J_At(A, Jp, Ji, Jx, Nleading_rows_J, out)


####################################################################################################
# lens models
####################################################################################################
def lensmodel_num_params(lensmodel):
    return checked.mrcal_lensmodel_num_params(C.byref(_lensmodel(lensmodel)))


def supported_lensmodels():
    names = checked.mrcal_supported_lensmodel_names()
    out, i = [], 0
    while names[i]:
        out.append(names[i].decode())
        i += 1
    return tuple(out)


def lensmodel_metadata_and_config(lensmodel):
    lm = _lensmodel(lensmodel)
    m = checked.mrcal_lensmodel_metadata(C.byref(lm)).bits
    out = dict(has_core=(m >> 0) & 1, can_project_behind_camera=(m >> 1) & 1,
               has_gradients=(m >> 2) & 1, noncentral=(m >> 3) & 1)
    if lm.type == 10:
        cfg = np.frombuffer(bytes(lm.config), np.uint16)
        out.update(order=int(cfg[0]), Nx=int(cfg[1]), Ny=int(cfg[2]), fov_x_deg=int(cfg[3]))
    elif lm.type == 9:
        out.update(linearity=float(np.frombuffer(bytes(lm.config), np.float64)[0]))
    return out


def knots_for_splined_models(lensmodel):
    lm = _lensmodel(lensmodel)
    if lm.type != 10:
        raise RuntimeError("This function works only with the LENSMODEL_SPLINED_STEREOGRAPHIC model. "
                           f"'{lensmodel}' passed in")
    cfg = np.frombuffer(bytes(lm.config), np.uint16)
    ux, uy = np.zeros(int(cfg[1])), np.zeros(int(cfg[2]))
    checked.mrcal_knots_for_splined_models(_ptr(ux), _ptr(uy), C.byref(lm))
    return ux, uy


####################################################################################################
# layout: either the full optimization_inputs, or explicit counts (mrcal-pywrap.c:2164-2380)
####################################################################################################
_EXPLICIT = ("Ncameras_intrinsics", "Ncameras_extrinsics", "Nframes", "Npoints",
             "Nobservations_board", "Nobservations_point")


def _layout_inputs(kwargs):
    explicit = {k: kwargs.pop(k) for k in _EXPLICIT if k in kwargs}
    return _Inputs(kwargs, for_layout_only=True, explicit=explicit)


def _none_if_negative(i):
    return i if i >= 0 else None


def state_index_intrinsics(icam_intrinsics, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_state_index_intrinsics(int(icam_intrinsics), *I.counts(), I.selections,
                                                                  I.lm_ref()))


def state_index_extrinsics(icam_extrinsics, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_state_index_extrinsics(int(icam_extrinsics), *I.counts(), I.selections,
                                                                  I.lm_ref()))


def state_index_frames(iframe, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_state_index_frames(int(iframe), *I.counts(), I.selections, I.lm_ref()))


def state_index_points(i_point, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_state_index_points(int(i_point), *I.counts(), I.selections, I.lm_ref()))


def state_index_calobject_warp(**kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_state_index_calobject_warp(*I.counts(), I.selections, I.lm_ref()))


def num_states_intrinsics(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_states_intrinsics(I.Ncam_i, I.selections, I.lm_ref())


def num_states_extrinsics(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_states_extrinsics(I.Ncam_e, I.selections)


def num_states_frames(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_states_frames(I.Nframes, I.selections)


def num_states_points(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_states_points(I.Npoints, I.Npoints_fixed, I.selections)


def num_states_calobject_warp(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_states_calobject_warp(I.selections, I.Nobs_board)


def num_states(**kwargs):
    return _layout_inputs(kwargs).num_states()


def num_intrinsics_optimization_params(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_intrinsics_optimization_params(I.selections, I.lm_ref())


def measurement_index_boards(i_observation_board, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_measurement_index_boards(int(i_observation_board), I.Nobs_board,
                                                                    I.Nobs_point, I.W, I.H))


def num_measurements_boards(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_measurements_boards(I.Nobs_board, I.W, I.H)


def measurement_index_points(i_observation_point, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(checked.mrcal_measurement_index_points(int(i_observation_point), I.Nobs_board,
                                                                    I.Nobs_point, I.W, I.H))


def num_measurements_points(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_measurements_points(I.Nobs_point)


def measurement_index_points_triangulated(i_point_triangulated, **kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    if ntri == 0:
        return None
    return _none_if_negative(checked.mrcal_measurement_index_points_triangulated(
            int(i_point_triangulated), I.Nobs_board, I.Nobs_point, tri, ntri, max(I.W, 0), max(I.H, 0)))


def num_measurements_points_triangulated(**kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    return checked.mrcal_num_measurements_points_triangulated(tri, ntri)


def measurement_index_regularization(**kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    return _none_if_negative(checked.mrcal_measurement_index_regularization(
            tri, ntri, I.W, I.H, I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed, I.Nobs_board, I.Nobs_point,
            I.selections, I.lm_ref()))


def num_measurements_regularization(**kwargs):
    I = _layout_inputs(kwargs)
    return checked.mrcal_num_measurements_regularization(*I.counts(), I.selections, I.lm_ref())


def num_measurements(**kwargs):
    return _layout_inputs(kwargs).num_measurements()


def corresponding_icam_extrinsics(icam_intrinsics, **kwargs):
    I = _layout_inputs(kwargs)
    ob, op = I.c_observations()
    out = C.c_int(-100)
    checked.mrcal_corresponding_icam_extrinsics(C.byref(out), int(icam_intrinsics), I.Ncam_i, I.Ncam_e, ob.shape[0],
                                                _ptr(ob), op.shape[0], _ptr(op))
    return out.value


def _pack_unpack(b, pack, kwargs):
    """In place, broadcasting over the leading dims (mrcal-pywrap.c:3423-3585)."""
    I = _layout_inputs(kwargs)
    if not isinstance(b, np.ndarray) or b.dtype != np.float64 or not b.flags.c_contiguous:
        raise RuntimeError("The given array MUST be a C-style contiguous numpy array of dtype float64")
    if b.ndim < 1:
        raise RuntimeError("The given array MUST have at least one dimension")
    Nstate = I.num_states()
    if b.shape[-1] != Nstate:
        raise RuntimeError(f"The given array MUST have last dimension of size Nstate={Nstate}; "
                           f"instead got {b.shape[-1]}")
    f = checked.mrcal_pack_solver_state_vector if pack else checked.mrcal_unpack_solver_state_vector
    flat = b.reshape(-1, Nstate)
    for i in range(flat.shape[0]):
        f(flat[i].ctypes.data, *I.counts(), I.selections, I.lm_ref())
    return None


def pack_state(b, **kwargs):
    return _pack_unpack(b, True, kwargs)


def unpack_state(b, **kwargs):
    return _pack_unpack(b, False, kwargs)


_PROJECT_UNPROJECT, _PROJECT_NORMALIZE = 2, 4   # MRCAL_B200_PROJECT_* of include/mrcal_b200.h


def _projection(fname, x, lensmodel, intrinsics_data, flags, get_gradients, out, names, dintrinsics=True):
    """The (un)projection of x through intrinsics_data in the pose utilities' call frame (poseutils._pose()):
    mrcal_b200_project[_device](). dintrinsics: whether the gradients include the one in the intrinsics"""
    from .poseutils import _pose
    lm = _lensmodel(lensmodel)
    Nintr = checked.mrcal_lensmodel_num_params(C.byref(lm))
    w_in, w_out = (2, 3) if flags & _PROJECT_UNPROJECT else (3, 2)
    grads = ((w_out, w_in),) + (((w_out, Nintr),) if dintrinsics else ()) if get_gradients else ()
    return _pose(fname, (x, intrinsics_data), ((w_in,), (Nintr,)), ((w_out,),) + grads, out, get_gradients,
                 entry="project", op=flags, lensmodel=lm, names=names)


def project(v, lensmodel, intrinsics_data, get_gradients=False, *, out=None):
    """q = project(v), as the reference's mrcal.project() (mrcal/projections.py, mrcal.h:165-191). v: (...,3) points
    in camera coordinates; intrinsics_data: (...,Nintrinsics), one lens model for all. The leading dimensions
    broadcast together (at most 8 of them); a broadcast operand is read in place, never expanded. Returns q
    (...,2); with get_gradients, as the reference, (q, dq_dv (...,2,3), dq_dintrinsics (...,2,Nintrinsics): dense,
    0 where the projection does not depend on an intrinsic). v and intrinsics_data (and out) are either numpy arrays
    (or lists), converted to float64, or all torch CUDA float64 tensors on one device: the results are then tensors on
    that device, and the kernel is enqueued on torch.cuda.current_stream() without waiting for it. out= writes the
    results into the given array (a tuple of three with get_gradients) and returns it."""
    return _projection("project", v, lensmodel, intrinsics_data, 0, get_gradients, out, ("v", "intrinsics_data"))


def unproject(q, lensmodel, intrinsics_data, *, normalize=False, get_gradients=False, out=None):
    """Observation rays of pixels q (...,2), as the reference's mrcal.unproject() returns them
    (mrcal/projections.py:112-397). Returns v (...,3); with get_gradients, (v, dv_dq (...,3,2), dv_dintrinsics
    (...,3,Nintrinsics), dense). The rays are not normalised unless normalize; then the gradients are those of the unit
    rays. As in the reference, the magnitude of an unnormalised ray may change with get_gradients: the gradients are
    those of the ray returned with them. A pixel that cannot be unprojected gives NaN (the zero vector with normalize
    and no gradients). intrinsics_data is (...,Nintrinsics); broadcasting, the torch CUDA tensors and out= are those of
    project(). CAHVORE with E != 0 in any intrinsics row is refused; with tensors that check brings one flag back to the
    host, so unprojecting through CAHVORE waits for the current stream."""
    flags = _PROJECT_UNPROJECT | (_PROJECT_NORMALIZE if normalize else 0)
    return _projection("unproject", q, lensmodel, intrinsics_data, flags, get_gradients, out, ("q", "intrinsics_data"))


_FXYCXY_IDENTITY = np.array((1.0, 1.0, 0.0, 0.0))


def _fxycxy(points, fxycxy):
    """fxycxy; the default core f = 1, c = 0 on the device of tensor points"""
    torch = sys.modules.get("torch")
    if fxycxy is _FXYCXY_IDENTITY and torch is not None and isinstance(points, torch.Tensor) and points.is_cuda:
        # filled on the device, in stream order: no upload from the host
        fxycxy = torch.zeros(4, dtype=torch.float64, device=points.device)
        fxycxy[:2] = 1.
    return fxycxy


def _project_closed_form(lensmodel, points, fxycxy, get_gradients, out):
    return _projection(f"project_{lensmodel[10:].lower()}", points, lensmodel, _fxycxy(points, fxycxy), 0,
                       get_gradients, out, ("points", "fxycxy"), dintrinsics=False)


def _unproject_closed_form(lensmodel, points, fxycxy, get_gradients, out):
    return _projection(f"unproject_{lensmodel[10:].lower()}", points, lensmodel, _fxycxy(points, fxycxy),
                       _PROJECT_UNPROJECT, get_gradients, out, ("points", "fxycxy"), dintrinsics=False)


def project_pinhole(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """q = (f x/z + c) of points (...,3), as mrcal.project_pinhole(); with get_gradients, (q, dq_dp (...,2,3)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _project_closed_form("LENSMODEL_PINHOLE", points, fxycxy, get_gradients, out)


def unproject_pinhole(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """v = ((q - c)/f, 1) of pixels (...,2), as mrcal.unproject_pinhole(); with get_gradients, (v, dv_dq (...,3,2)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _unproject_closed_form("LENSMODEL_PINHOLE", points, fxycxy, get_gradients, out)


def project_stereographic(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """The stereographic projection of points (...,3), as mrcal.project_stereographic(); with get_gradients,
    (q, dq_dp (...,2,3)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _project_closed_form("LENSMODEL_STEREOGRAPHIC", points, fxycxy, get_gradients, out)


def unproject_stereographic(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """The stereographic unprojection of pixels (...,2), as mrcal.unproject_stereographic(); with get_gradients,
    (v, dv_dq (...,3,2)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _unproject_closed_form("LENSMODEL_STEREOGRAPHIC", points, fxycxy, get_gradients, out)


def project_lonlat(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """The equirectangular (longitude, latitude) projection of points (...,3), as mrcal.project_lonlat(); with
    get_gradients, (q, dq_dp (...,2,3)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _project_closed_form("LENSMODEL_LONLAT", points, fxycxy, get_gradients, out)


def unproject_lonlat(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """Unit rays of equirectangular (longitude, latitude) pixels (...,2), as mrcal.unproject_lonlat(); with
    get_gradients, (v, dv_dq (...,3,2)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _unproject_closed_form("LENSMODEL_LONLAT", points, fxycxy, get_gradients, out)


def project_latlon(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """The transverse equirectangular (latitude, longitude) projection of points (...,3), as mrcal.project_latlon();
    with get_gradients, (q, dq_dp (...,2,3)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _project_closed_form("LENSMODEL_LATLON", points, fxycxy, get_gradients, out)


def unproject_latlon(points, fxycxy=_FXYCXY_IDENTITY, *, get_gradients=False, out=None):
    """Unit rays of transverse equirectangular (latitude, longitude) pixels (...,2), as mrcal.unproject_latlon(); with
    get_gradients, (v, dv_dq (...,3,2)).
    fxycxy (...,4) broadcasts with the points; torch CUDA tensors and out= as in project()"""
    return _unproject_closed_form("LENSMODEL_LATLON", points, fxycxy, get_gradients, out)
