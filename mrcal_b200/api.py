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

import numpy as np
import scipy.sparse

from . import _capi
from ._capi import lib

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
    if not lib.mrcal_lensmodel_from_name(C.byref(lm), name.encode()):
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
        Nintr = lib.mrcal_lensmodel_num_params(C.byref(self.lensmodel))
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
                    if not lib.mrcal_unproject(_ptr(v), _ptr(q), len(sel), self.lm_ref(), _ptr(intr)):
                        raise RuntimeError("mrcal_unproject() failed: " + _capi.last_error())
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

    def counts(self):
        return (self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed, self.Nobs_board)

    def lm_ref(self):
        if self.lensmodel is None:
            raise RuntimeError("The 'lensmodel' argument is required")
        return C.byref(self.lensmodel)

    def num_states(self):
        return lib.mrcal_num_states(*self.counts(), self.selections, self.lm_ref())

    def num_measurements(self):
        tri, ntri = self.c_triangulated()
        return lib.mrcal_num_measurements(self.Nobs_board, self.Nobs_point, tri, ntri, self.W, self.H,
                                          self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed,
                                          self.selections, self.lm_ref())

    def num_j_nonzero(self):
        ob, op = self.c_observations()
        tri, ntri = self.c_triangulated()
        return lib._mrcal_num_j_nonzero(self.Nobs_board, self.Nobs_point, tri, ntri, self.W, self.H,
                                        self.Ncam_i, self.Ncam_e, self.Nframes, self.Npoints, self.Npoints_fixed,
                                        _ptr(ob), _ptr(op), self.selections, self.lm_ref())


def _require_gpu():
    if lib.mrcal_b200_device_count() <= 0:
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
    ob, op = I.c_observations()
    tri, ntri = I.c_triangulated(rays=True)
    ok = lib.mrcal_optimizer_callback(
        _ptr(b), C.c_int(b.nbytes), _ptr(x), C.c_int(x.nbytes),
        C.byref(Jt) if Jt is not None else None,
        _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame), _ptr(I.points),
        _ptr(I.calobject_warp) if I.calobject_warp is not None else None,
        I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed,
        _ptr(ob), _ptr(op), I.Nobs_board, I.Nobs_point, tri, ntri,
        _ptr(I.observations_board), _ptr(I.observations_point),
        I.lm_ref(), _ptr(I.imagersizes), I.selections, None,
        C.c_double(I.spacing), max(I.W, 0), max(I.H, 0), C.c_bool(I.verbose))
    if not ok:
        raise RuntimeError("mrcal_optimizer_callback() failed: " + _capi.last_error())
    J = None
    factorization = None
    if keep is not None:
        P, Ii, X = keep
        J = scipy.sparse.csr_matrix((X, Ii, P), shape=(Nmeas, Nstate))
        if not no_factorization:
            # the problem's own structure first (frames/points eliminated, dense factor of the reduced system only);
            # the dense Nstate x Nstate object only where that does not apply
            if not os.environ.get("MRCAL_B200_DENSE_FACTORIZATION"):
                h = lib.mrcal_b200_factorization_create_from_last_callback()   # NULL comes back as None
                if h:
                    return b, x, J, CHOLMOD_factorization._from_handle(h, J.shape)
                if "not positive definite" in _capi.last_error():
                    return b, x, J, None   # not an error: mrcal-pywrap.c:1981-1988
            try:
                factorization = CHOLMOD_factorization(J)
            except RuntimeError as e:
                # "JtJ is not positive definite" is not an error here: mrcal-pywrap.c:1981-1988 returns None.
                # Anything else (out of memory, a CUDA failure) is one
                if "not positive definite" not in str(e):
                    raise
                factorization = None
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
    ob, op = I.c_observations()
    tri, ntri = I.c_triangulated(rays=True)
    stats = lib.mrcal_optimize(
        _ptr(b), C.c_int(b.nbytes), _ptr(x), C.c_int(x.nbytes),
        _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame), _ptr(I.points),
        _ptr(I.calobject_warp) if I.calobject_warp is not None else None,
        I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed,
        _ptr(ob), _ptr(op), I.Nobs_board, I.Nobs_point, tri, ntri,
        _ptr(I.observations_board), _ptr(I.observations_point),
        I.lm_ref(), _ptr(I.imagersizes), I.selections, None,
        C.c_double(I.spacing), max(I.W, 0), max(I.H, 0), C.c_bool(I.verbose), C.c_bool(False))
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
    ob, op = I.c_observations()
    tri, ntri = I.c_triangulated(rays=True)
    sys_stdout_fd = 1
    with tempfile.TemporaryFile(mode="w+b") as tmp:
        import sys as _sys
        _sys.stdout.flush()
        saved = os.dup(sys_stdout_fd)
        os.dup2(tmp.fileno(), sys_stdout_fd)
        try:
            lib.mrcal_optimize(
                None, C.c_int(0), None, C.c_int(0),
                _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame), _ptr(I.points),
                _ptr(I.calobject_warp) if I.calobject_warp is not None else None,
                I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed,
                _ptr(ob), _ptr(op), I.Nobs_board, I.Nobs_point, tri, ntri,
                _ptr(I.observations_board), _ptr(I.observations_point),
                I.lm_ref(), _ptr(I.imagersizes), I.selections, None,
                C.c_double(I.spacing), max(I.W, 0), max(I.H, 0), C.c_bool(False), C.c_bool(True))
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
        ob, op = I.c_observations()
        tri, ntri = I.c_triangulated(rays=True)
        self._h = lib.mrcal_b200_problem_create_triangulated(
            _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame), _ptr(I.points),
            _ptr(I.calobject_warp) if I.calobject_warp is not None else None,
            I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed,
            _ptr(ob), _ptr(op), I.Nobs_board, I.Nobs_point, tri, ntri,
            _ptr(I.observations_board), _ptr(I.observations_point),
            I.lm_ref(), _ptr(I.imagersizes), I.selections,
            C.c_double(I.spacing), max(I.W, 0), max(I.H, 0))
        if not self._h:
            raise RuntimeError("mrcal_b200_problem_create() failed: " + _capi.last_error())
        self._h = C.c_void_p(self._h)
        self.Nstate = lib.mrcal_b200_problem_num_states(self._h)
        self.Nmeasurements = lib.mrcal_b200_problem_num_measurements(self._h)
        self.N_j_nonzero = lib.mrcal_b200_problem_num_j_nonzero(self._h)

    def close(self):
        if getattr(self, "_h", None):
            lib.mrcal_b200_problem_destroy(self._h)
            self._h = None

    __del__ = close

    def reset(self, b_packed=None):
        if b_packed is not None:
            b_packed = np.ascontiguousarray(b_packed, np.float64)
            assert b_packed.shape == (self.Nstate,)
        if not lib.mrcal_b200_problem_reset(self._h, _ptr(b_packed) if b_packed is not None else None):
            raise RuntimeError(_capi.last_error())

    def upload(self):
        """Re-send the seed and the observation pool from the host arrays given at construction."""
        I = self._I
        if not lib.mrcal_b200_problem_upload(self._h, _ptr(I.intrinsics), _ptr(I.rt_cam_ref), _ptr(I.rt_ref_frame),
                                             _ptr(I.points),
                                             _ptr(I.calobject_warp) if I.calobject_warp is not None else None,
                                             _ptr(I.observations_board), _ptr(I.observations_point)):
            raise RuntimeError(_capi.last_error())

    def drt_cross_reprojection__dbpacked(self, icam_intrinsics=-1):
        """K (6, Nstate) at the problem's current state: see the module-level function."""
        K = np.zeros((6, self.Nstate))
        if not lib.mrcal_b200_problem_drt_cross_reprojection__dbpacked(self._h, int(icam_intrinsics), _ptr(K)):
            raise RuntimeError("_mrcal_drt_cross_reprojection__dbpacked() failed: " + _capi.last_error())
        return K

    def callback(self, jacobian=True):
        b = np.zeros(self.Nstate)
        x = np.zeros(self.Nmeasurements)
        if jacobian:
            P = np.zeros(self.Nmeasurements + 1, np.int32)
            Ii = np.zeros(self.N_j_nonzero, np.int32)
            X = np.zeros(self.N_j_nonzero)
            ok = lib.mrcal_b200_problem_callback(self._h, _ptr(b), _ptr(x), _ptr(P), _ptr(Ii), _ptr(X))
        else:
            ok = lib.mrcal_b200_problem_callback(self._h, _ptr(b), _ptr(x), None, None, None)
        if not ok:
            raise RuntimeError(_capi.last_error())
        if not jacobian:
            return b, x, None
        return b, x, scipy.sparse.csr_matrix((X, Ii, P), shape=(self.Nmeasurements, self.Nstate))

    def optimize(self, **parameters):
        p = _capi.SolverParameters()
        lib.mrcal_b200_default_solver_parameters(C.byref(p))
        for k, v in parameters.items():
            if not hasattr(p, k):
                raise RuntimeError(f"unknown solver parameter '{k}'")
            setattr(p, k, v)
        stats = _capi.Stats()
        info = _capi.SolveInfo()
        if not lib.mrcal_b200_problem_optimize(self._h, C.byref(p), C.byref(stats), C.byref(info)):
            raise RuntimeError("mrcal_b200_problem_optimize() failed: " + _capi.last_error())
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
        ok = lib.mrcal_b200_problem_download(self._h, _ptr(b), _ptr(x), _ptr(intr), _ptr(rtc), _ptr(rtf), _ptr(pts),
                                             _ptr(warp) if warp is not None else None, _ptr(obs))
        if not ok:
            raise RuntimeError(_capi.last_error())
        return dict(b_packed=b, x=x, intrinsics=intr, rt_cam_ref=rtc, rt_ref_frame=rtf, points=pts,
                    calobject_warp=warp, observations_board=obs)

    def reduced_system(self, lambda_=0.0):
        """(S, g_reduced, g_full): the Schur-reduced normal equations at the current state (introspection)."""
        n = C.c_int(0)
        if not lib.mrcal_b200_problem_reduced_system(self._h, C.c_double(lambda_), C.byref(n), None, None, None):
            raise RuntimeError(_capi.last_error())
        S = np.zeros((n.value, n.value))
        g = np.zeros(n.value)
        gf = np.zeros(self.Nstate)
        if not lib.mrcal_b200_problem_reduced_system(self._h, C.c_double(lambda_), C.byref(n), _ptr(S), _ptr(g), _ptr(gf)):
            raise RuntimeError(_capi.last_error())
        S = np.tril(S) + np.tril(S, -1).T
        return S, g, gf

    def time_callback(self, N=10, jacobian=True):
        ms = lib.mrcal_b200_problem_time_callback(self._h, int(N), C.c_bool(jacobian))
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
        self._h = lib.mrcal_b200_factorization_create(_ptr(P) or P.ctypes.data_as(C.c_void_p), _ptr(Ii), _ptr(X),
                                                      J.shape[0], J.shape[1])
        if not self._h:
            raise RuntimeError("CHOLMOD_factorization: " + _capi.last_error())
        self._h = C.c_void_p(self._h)

    @classmethod
    def _from_handle(cls, h, shape):
        self = cls.__new__(cls)
        self.shape = shape
        self._h = C.c_void_p(h)
        return self

    def __del__(self):
        if getattr(self, "_h", None):
            lib.mrcal_b200_factorization_destroy(self._h)
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
            if not lib.mrcal_b200_factorization_solve_sys(self._h, _ptr(out), _ptr(flat), flat.shape[0], code):
                raise RuntimeError("solve_xt_JtJ_bt: " + _capi.last_error())
        return out.reshape(bt.shape)

    def rcond(self):
        return lib.mrcal_b200_factorization_rcond(self._h)


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
        h = lib.mrcal_b200_csr_create(_ptr(Jp) or Jp.ctypes.data_as(C.c_void_p), _ptr(Ji), _ptr(Jx), self.Nrows, Ncols)
        if not h:
            raise RuntimeError(_capi.last_error())
        self._h = C.c_void_p(h)

    def __del__(self):
        if getattr(self, "_h", None):
            lib.mrcal_b200_csr_destroy(self._h)
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
    if not lib.mrcal_b200_csr_Jt_x(J._h, _ptr(out), _ptr(xt)):
        raise RuntimeError(_capi.last_error())
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
        if not lib.mrcal_b200_csr_A_Jt_J_At(J._h, _ptr(res[k]), _ptr(flat[k]), Nx, int(Nleading_rows_J)):
            raise RuntimeError(_capi.last_error())
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
    return lib.mrcal_lensmodel_num_params(C.byref(_lensmodel(lensmodel)))


def supported_lensmodels():
    names = lib.mrcal_supported_lensmodel_names()
    out, i = [], 0
    while names[i]:
        out.append(names[i].decode())
        i += 1
    return tuple(out)


def lensmodel_metadata_and_config(lensmodel):
    lm = _lensmodel(lensmodel)
    m = lib.mrcal_lensmodel_metadata(C.byref(lm)).bits
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
    if not lib.mrcal_knots_for_splined_models(_ptr(ux), _ptr(uy), C.byref(lm)):
        raise RuntimeError(_capi.last_error())
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
    return _none_if_negative(lib.mrcal_state_index_intrinsics(int(icam_intrinsics), *I.counts(), I.selections, I.lm_ref()))


def state_index_extrinsics(icam_extrinsics, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_state_index_extrinsics(int(icam_extrinsics), *I.counts(), I.selections, I.lm_ref()))


def state_index_frames(iframe, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_state_index_frames(int(iframe), *I.counts(), I.selections, I.lm_ref()))


def state_index_points(i_point, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_state_index_points(int(i_point), *I.counts(), I.selections, I.lm_ref()))


def state_index_calobject_warp(**kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_state_index_calobject_warp(*I.counts(), I.selections, I.lm_ref()))


def num_states_intrinsics(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_states_intrinsics(I.Ncam_i, I.selections, I.lm_ref())


def num_states_extrinsics(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_states_extrinsics(I.Ncam_e, I.selections)


def num_states_frames(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_states_frames(I.Nframes, I.selections)


def num_states_points(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_states_points(I.Npoints, I.Npoints_fixed, I.selections)


def num_states_calobject_warp(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_states_calobject_warp(I.selections, I.Nobs_board)


def num_states(**kwargs):
    return _layout_inputs(kwargs).num_states()


def num_intrinsics_optimization_params(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_intrinsics_optimization_params(I.selections, I.lm_ref())


def measurement_index_boards(i_observation_board, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_measurement_index_boards(int(i_observation_board), I.Nobs_board, I.Nobs_point,
                                                                I.W, I.H))


def num_measurements_boards(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_measurements_boards(I.Nobs_board, I.W, I.H)


def measurement_index_points(i_observation_point, **kwargs):
    I = _layout_inputs(kwargs)
    return _none_if_negative(lib.mrcal_measurement_index_points(int(i_observation_point), I.Nobs_board, I.Nobs_point,
                                                                I.W, I.H))


def num_measurements_points(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_measurements_points(I.Nobs_point)


def measurement_index_points_triangulated(i_point_triangulated, **kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    if ntri == 0:
        return None
    return _none_if_negative(lib.mrcal_measurement_index_points_triangulated(
        int(i_point_triangulated), I.Nobs_board, I.Nobs_point, tri, ntri, max(I.W, 0), max(I.H, 0)))


def num_measurements_points_triangulated(**kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    return lib.mrcal_num_measurements_points_triangulated(tri, ntri)


def measurement_index_regularization(**kwargs):
    I = _layout_inputs(kwargs)
    tri, ntri = I.c_triangulated()
    return _none_if_negative(lib.mrcal_measurement_index_regularization(
        tri, ntri, I.W, I.H, I.Ncam_i, I.Ncam_e, I.Nframes, I.Npoints, I.Npoints_fixed, I.Nobs_board, I.Nobs_point,
        I.selections, I.lm_ref()))


def num_measurements_regularization(**kwargs):
    I = _layout_inputs(kwargs)
    return lib.mrcal_num_measurements_regularization(*I.counts(), I.selections, I.lm_ref())


def num_measurements(**kwargs):
    return _layout_inputs(kwargs).num_measurements()


def corresponding_icam_extrinsics(icam_intrinsics, **kwargs):
    I = _layout_inputs(kwargs)
    ob, op = I.c_observations()
    out = C.c_int(-100)
    if not lib.mrcal_corresponding_icam_extrinsics(C.byref(out), int(icam_intrinsics), I.Ncam_i, I.Ncam_e,
                                                   ob.shape[0], _ptr(ob), op.shape[0], _ptr(op)):
        raise RuntimeError("Error calling mrcal_corresponding_icam_extrinsics(): " + _capi.last_error())
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
    f = lib.mrcal_pack_solver_state_vector if pack else lib.mrcal_unpack_solver_state_vector
    flat = b.reshape(-1, Nstate)
    for i in range(flat.shape[0]):
        f(C.c_void_p(flat[i].ctypes.data), *I.counts(), I.selections, I.lm_ref())
    return None


def pack_state(b, **kwargs):
    return _pack_unpack(b, True, kwargs)


def unpack_state(b, **kwargs):
    return _pack_unpack(b, False, kwargs)


def project(v, lensmodel, intrinsics_data, get_gradients=False):
    """q = project(v): the reference's mrcal.project() for one camera (mrcal-pywrap.c / mrcal.h:165-191).
    v: (...,3) points in camera coordinates. Returns q (...,2); with get_gradients, as the reference,
    (q, dq_dv (...,2,3), dq_dintrinsics (...,2,Nintrinsics))."""
    _require_gpu()
    v = np.ascontiguousarray(v, dtype=np.float64)
    if v.shape[-1] != 3:
        raise RuntimeError("project(): the last dimension of v must be 3")
    lm = _lensmodel(lensmodel)
    intr = np.ascontiguousarray(intrinsics_data, dtype=np.float64)
    if intr.shape != (lib.mrcal_lensmodel_num_params(C.byref(lm)),):
        raise RuntimeError(f"project(): intrinsics_data must have shape ({lib.mrcal_lensmodel_num_params(C.byref(lm))},)")
    flat = v.reshape(-1, 3)
    q = np.zeros((flat.shape[0], 2))
    g = np.zeros((flat.shape[0], 2, 3)) if get_gradients else None
    gi = np.zeros((flat.shape[0], 2, intr.shape[0])) if get_gradients else None
    if not lib.mrcal_project(_ptr(q), _ptr(g) if g is not None else None, _ptr(gi) if gi is not None else None,
                             _ptr(flat), flat.shape[0], C.byref(lm), _ptr(intr)):
        raise RuntimeError("mrcal_project() failed: " + _capi.last_error())
    q = q.reshape(v.shape[:-1] + (2,))
    if not get_gradients:
        return q
    return q, g.reshape(v.shape[:-1] + (2, 3)), gi.reshape(v.shape[:-1] + (2, intr.shape[0]))


def unproject(q, lensmodel, intrinsics_data):
    """Observation rays (not normalised) of pixels q (...,2): the reference's mrcal.unproject() without
    gradients (mrcal.h:193-224)."""
    _require_gpu()
    q = np.ascontiguousarray(q, dtype=np.float64)
    if q.shape[-1] != 2:
        raise RuntimeError("unproject(): the last dimension of q must be 2")
    lm = _lensmodel(lensmodel)
    intr = np.ascontiguousarray(intrinsics_data, dtype=np.float64)
    flat = q.reshape(-1, 2)
    v = np.zeros((flat.shape[0], 3))
    if not lib.mrcal_unproject(_ptr(v), _ptr(flat), flat.shape[0], C.byref(lm), _ptr(intr)):
        raise RuntimeError("mrcal_unproject() failed: " + _capi.last_error())
    return v.reshape(q.shape[:-1] + (3,))
