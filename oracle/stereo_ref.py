"""TEST INFRASTRUCTURE ONLY -- ctypes driver for oracle/_ref/libmrcal_stereo_ref.so.

libmrcal_stereo_ref.so is the reference's OWN stereo.c, compiled by oracle/stereo.mk from the source where it lies
under /root/reference and linked against oracle/_ref/libmrcal_ref.so (oracle/ref.py), which provides the projections
and pose utilities it calls. The ground truth for the stereo geometry, the rectification maps and the ranges.

stereo.c's pinhole rectification asks LAPACK's dgeev_ for the roots of a quartic. LAPACK is not in this image: the
stand-in in stubs/stereo_stubs.c calls a hook, set here to numpy.linalg.eigvals, which is LAPACK's own dgeev.

Only tests/ and scripts/ import this module. The product (mrcal_b200/) never does.
"""
import ctypes as C
import os

import numpy as np

from . import ref
from .ref import _dp, lensmodel_from_name

_HERE = os.path.dirname(os.path.abspath(__file__))
LIBPATH = os.path.join(_HERE, "_ref", "libmrcal_stereo_ref.so")

_DGEEV_HOOK_T = C.CFUNCTYPE(C.c_int, C.c_int, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double))


def available():
    return ref.available() and os.path.exists(LIBPATH)


def _dgeev_eigvals(n, a, lda, wr, wi):
    try:
        A = np.ctypeslib.as_array(a, shape=(n, lda))[:, :n].T   # column-major
        w = np.linalg.eigvals(A)
        for i in range(n):
            wr[i], wi[i] = w[i].real, w[i].imag
        return 0
    except Exception:
        return 1


_dgeev_hook = _DGEEV_HOOK_T(_dgeev_eigvals)
_lib = None


def _stereo_lib():
    global _lib
    if _lib is None:
        if not available():
            raise RuntimeError(f"{LIBPATH} is missing: run `make -C oracle -f stereo.mk` where /root/reference exists")
        ref.lib()   # libmrcal_ref.so first: the big stack its VLAs need, and the library this one links against
        L = C.CDLL(LIBPATH)
        C.c_void_p.in_dll(L, "oracle_dgeev_hook").value = C.cast(_dgeev_hook, C.c_void_p).value
        for n in ("mrcal_rectified_system2", "mrcal_rectification_maps", "mrcal_stereo_range_sparse",
                  "mrcal_stereo_range_dense"):
            getattr(L, n).restype = C.c_bool
        _lib = L
    return _lib


class _Image(C.Structure):
    """mrcal_image_*_t (image.h:68-80)"""
    _fields_ = [("w", C.c_int), ("h", C.c_int), ("stride", C.c_int), ("data", C.c_void_p)]


def rectified_system2(lensmodel0, intrinsics0, rt_cam0_ref, rt_cam1_ref, *, az_fov_deg, el_fov_deg, az0_deg=None,
                      el0_deg=0., az_edge_margin_deg=10., pixels_per_deg_az=-1., pixels_per_deg_el=-1.,
                      rectification_model="LENSMODEL_LATLON"):
    """The reference's mrcal_rectified_system2() (stereo.c:390-718); az0_deg None autodetects. A dict of its outputs,
    or None where it refuses"""
    L = _stereo_lib()
    lm = lensmodel_from_name(lensmodel0)
    size = (C.c_uint * 2)()
    fxycxy, rt = np.zeros(4), np.zeros(6)
    baseline = C.c_double()
    az, el = C.c_double(pixels_per_deg_az), C.c_double(pixels_per_deg_el)
    fov = (C.c_double * 2)(az_fov_deg, el_fov_deg)
    azel0 = (C.c_double * 2)(0. if az0_deg is None else az0_deg, el0_deg)
    intr = np.ascontiguousarray(intrinsics0, np.float64)
    r0 = np.ascontiguousarray(rt_cam0_ref, np.float64)
    r1 = np.ascontiguousarray(rt_cam1_ref, np.float64)
    ok = L.mrcal_rectified_system2(size, _dp(fxycxy), _dp(rt), C.byref(baseline), C.byref(az), C.byref(el), fov, azel0,
                                   C.c_double(az_edge_margin_deg), C.byref(lm), _dp(intr), _dp(r0), _dp(r1),
                                   C.c_int(lensmodel_from_name(rectification_model).type),
                                   C.c_bool(az0_deg is None), C.c_bool(False), C.c_bool(False), C.c_bool(False))
    if not ok:
        return None
    return dict(imagersize=(int(size[0]), int(size[1])), fxycxy=fxycxy, rt_rect0_ref=rt, baseline=baseline.value,
                pixels_per_deg_az=az.value, pixels_per_deg_el=el.value, az_fov_deg=fov[0], el_fov_deg=fov[1],
                az0_deg=azel0[0], el0_deg=azel0[1])


def rectification_maps(lensmodel0, intrinsics0, r_cam0_ref, lensmodel1, intrinsics1, r_cam1_ref,
                       rectification_model, fxycxy, imagersize, r_rect0_ref):
    """The reference's mrcal_rectification_maps() (stereo.c:824-972): float32 (2, Nel, Naz, 2)"""
    L = _stereo_lib()
    Naz, Nel = (int(x) for x in imagersize)
    maps = np.zeros((2, Nel, Naz, 2), np.float32)
    a = [np.ascontiguousarray(x, np.float64) for x in (intrinsics0, r_cam0_ref, intrinsics1, r_cam1_ref, fxycxy, r_rect0_ref)]
    if not L.mrcal_rectification_maps(maps.ctypes.data_as(C.c_void_p), C.byref(lensmodel_from_name(lensmodel0)),
                                      _dp(a[0]), _dp(a[1]), C.byref(lensmodel_from_name(lensmodel1)), _dp(a[2]),
                                      _dp(a[3]), C.c_int(lensmodel_from_name(rectification_model).type), _dp(a[4]),
                                      (C.c_uint * 2)(Naz, Nel), _dp(a[5])):
        raise RuntimeError("reference mrcal_rectification_maps() failed")
    return maps


def stereo_range_sparse(disparity, qrect0, disparity_min, disparity_max, rectification_model, fxycxy, baseline):
    """The reference's mrcal_stereo_range_sparse() (stereo.c:1310-1352): range (N,)"""
    L = _stereo_lib()
    d = np.ascontiguousarray(disparity, np.float64).ravel()
    q = np.ascontiguousarray(qrect0, np.float64).reshape(-1, 2)
    f = np.ascontiguousarray(fxycxy, np.float64)
    r = np.zeros(d.size)
    if not L.mrcal_stereo_range_sparse(_dp(r), _dp(d), _dp(q), C.c_int(d.size), C.c_double(disparity_min),
                                       C.c_double(disparity_max), C.c_int(lensmodel_from_name(rectification_model).type),
                                       _dp(f), C.c_double(baseline)):
        raise RuntimeError("reference mrcal_stereo_range_sparse() failed")
    return r


def stereo_range_dense(disparity_scaled, disparity_scale, disparity_scaled_min, disparity_scaled_max,
                       rectification_model, fxycxy, baseline):
    """The reference's mrcal_stereo_range_dense() (stereo.c:1354-1417) on a uint16 (H, W) array, which may be a
    strided view: range (H, W)"""
    L = _stereo_lib()
    d = disparity_scaled
    assert d.dtype == np.uint16 and d.strides[1] == 2
    H, W = d.shape
    r = np.zeros((H, W))
    f = np.ascontiguousarray(fxycxy, np.float64)
    din = _Image(W, H, d.strides[0], d.ctypes.data)
    rout = _Image(W, H, r.strides[0], r.ctypes.data)
    if not L.mrcal_stereo_range_dense(C.byref(rout), C.byref(din), C.c_uint16(disparity_scale),
                                      C.c_uint16(disparity_scaled_min), C.c_uint16(disparity_scaled_max),
                                      C.c_int(lensmodel_from_name(rectification_model).type), _dp(f),
                                      C.c_double(baseline)):
        raise RuntimeError("reference mrcal_stereo_range_dense() failed")
    return r
