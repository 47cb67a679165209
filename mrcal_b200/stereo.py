"""Stereo rectification and ranging, with the reference's names, keyword arguments, defaults, return values and
refusals (mrcal/stereo.py:23-484, 784-923, 978-1308, 1453-1607):

    mrcal_b200.rectified_resolution(model0, ...)        -> (pixels_per_deg_az, pixels_per_deg_el)
    mrcal_b200.rectified_system(models, ...)            -> (model_rect0, model_rect1) [, metadata]
    mrcal_b200.rectification_maps(models, models_rect)  -> float32 (2, Nel, Naz, 2)
    mrcal_b200.stereo_range(disparity, models_rect)     -> ranges
    mrcal_b200.stereo_unproject(disparity, models_rect) -> points in rectified camera-0 coordinates

The geometry is host code in libmrcal_b200.so (csrc/stereo.cu); the maps, the ranges and the points are computed on
the device, one thread per element. This module only marshals arguments.
"""
import ctypes as C
import re

import numpy as np

from . import _capi
from ._capi import lib
from .api import _compose_Rt, _lensmodel, _ptr, _require_gpu, lensmodel_metadata_and_config
from .cameramodel import cameramodel

# the reference's Python wrapper takes an az0_deg above this for "autodetect" (mrcal-pywrap.c:4029-4030)
_AZ0_AUTODETECT = 1e7


def _rectification_model_type(name):
    return _lensmodel(name).type


def _fail(what):
    raise RuntimeError(f"{what} failed: {_capi.last_error()}")


def rectified_resolution(model0, *, az_fov_deg, el_fov_deg, az0_deg, el0_deg, R_cam0_rect0,
                         pixels_per_deg_az=-1., pixels_per_deg_el=-1., rectification_model="LENSMODEL_LATLON"):
    """The resolution (pixels_per_deg_az, pixels_per_deg_el) of a rectified view centred at (az0_deg, el0_deg) in
    the rectified frame R_cam0_rect0 (3,3). A value > 0 is used as given; a value < 0 asks for that multiple of
    model0's resolution at the centre of the view (-1: full resolution, -0.5: half), which takes one projection on the
    device. LENSMODEL_LATLON and LENSMODEL_LONLAT then fit a whole number of pixels into the field of view;
    LENSMODEL_PINHOLE keeps the value."""
    lensmodel, intrinsics = model0.intrinsics()
    lm = _lensmodel(lensmodel)
    intr = np.ascontiguousarray(intrinsics, np.float64)
    R = np.ascontiguousarray(R_cam0_rect0, np.float64)
    if R.shape != (3, 3):
        raise RuntimeError(f"R_cam0_rect0 must have shape (3,3); got {R.shape}")
    az, el = C.c_double(pixels_per_deg_az), C.c_double(pixels_per_deg_el)
    azel_fov = (C.c_double * 2)(az_fov_deg, el_fov_deg)
    azel0 = (C.c_double * 2)(az0_deg, el0_deg)
    if not lib.mrcal_rectified_resolution(C.byref(az), C.byref(el), C.byref(lm), _ptr(intr), azel_fov, azel0, _ptr(R),
                                          _rectification_model_type(rectification_model)):
        _fail("mrcal_rectified_resolution()")
    return az.value, el.value


def rectified_system(models, *, az_fov_deg, el_fov_deg, az0_deg=None, el0_deg=0, az_edge_margin_deg=10.,
                     pixels_per_deg_az=-1., pixels_per_deg_el=-1., rectification_model="LENSMODEL_LATLON",
                     return_metadata=False):
    """The pair of rectified models of the stereo pair `models`: the same intrinsics (rectification_model:
    LENSMODEL_LATLON or LENSMODEL_PINHOLE) and orientation, camera 1's rectified origin `baseline` along the rectified
    x axis. x runs from camera 0 to camera 1, z is the cameras' mean forward direction without its component along x.
    az0_deg=None centres the view on the cameras' mean forward direction, kept az_edge_margin_deg away from the
    baseline. pixels_per_deg_* < 0 scales camera 0's resolution at the centre of the view. With return_metadata, also
    a dict of az_fov_deg, el_fov_deg, az0_deg, el0_deg, pixels_per_deg_az, pixels_per_deg_el and baseline."""
    for m in models:
        lensmodel, intrinsics = m.intrinsics()
        if lensmodel_metadata_and_config(lensmodel)["noncentral"]:
            if re.match("^LENSMODEL_CAHVORE", lensmodel):
                if np.sum(intrinsics[-3:] ** 2) > 0:
                    raise RuntimeError("Stereo rectification is only possible with a central projection. Please "
                                       "centralize your models. This is CAHVORE, so set E=0 to centralize. This will "
                                       "ignore all noncentral effects near the lens")
            else:
                raise RuntimeError("Stereo rectification is only possible with a central projection. Please centralize "
                                   "your models")
    lensmodel0, intrinsics0 = models[0].intrinsics()
    lm = _lensmodel(lensmodel0)
    intr = np.ascontiguousarray(intrinsics0, np.float64)
    rt0 = np.ascontiguousarray(models[0].rt_cam_ref(), np.float64)
    rt1 = np.ascontiguousarray(models[1].rt_cam_ref(), np.float64)
    if az0_deg is None:
        az0_deg = _AZ0_AUTODETECT
    imagersize = (C.c_uint * 2)()
    fxycxy = np.zeros(4)
    rt_rect0_ref = np.zeros(6)
    baseline = C.c_double()
    az, el = C.c_double(pixels_per_deg_az), C.c_double(pixels_per_deg_el)
    azel_fov = (C.c_double * 2)(az_fov_deg, el_fov_deg)
    azel0 = (C.c_double * 2)(az0_deg, el0_deg)
    if not lib.mrcal_rectified_system2(imagersize, _ptr(fxycxy), _ptr(rt_rect0_ref), C.byref(baseline), C.byref(az),
                                       C.byref(el), azel_fov, azel0, float(az_edge_margin_deg), C.byref(lm), _ptr(intr),
                                       _ptr(rt0), _ptr(rt1), _rectification_model_type(rectification_model),
                                       az0_deg > _AZ0_AUTODETECT / 10., False, False, False):
        _fail("mrcal_rectified_system()")
    # rect1 has rect0's orientation, its origin at camera 1: rt_rect1_ref = (0,0,0, -baseline,0,0) rt_rect0_ref
    rt_rect1_ref = rt_rect0_ref.copy()
    rt_rect1_ref[3] -= baseline.value
    Naz, Nel = int(imagersize[0]), int(imagersize[1])
    models_rectified = (cameramodel(intrinsics=(rectification_model, fxycxy), imagersize=(Naz, Nel), rt_cam_ref=rt_rect0_ref),
                        cameramodel(intrinsics=(rectification_model, fxycxy), imagersize=(Naz, Nel), rt_cam_ref=rt_rect1_ref))
    if not return_metadata:
        return models_rectified
    metadata = dict(az_fov_deg=azel_fov[0], el_fov_deg=azel_fov[1], az0_deg=azel0[0], el0_deg=azel0[1],
                    pixels_per_deg_az=az.value, pixels_per_deg_el=el.value, baseline=baseline.value)
    return models_rectified, metadata


def _validate_models_rectified(models_rectified):
    """Two LENSMODEL_LATLON or two LENSMODEL_PINHOLE models with the same intrinsics, imager and orientation, the
    second translated along the rectified x axis only: what rectified_system() returns (mrcal/stereo.py:784-819)"""
    if len(models_rectified) != 2:
        raise RuntimeError(f"Must have received exactly two models. Got {len(models_rectified)} instead")
    intrinsics = [m.intrinsics() for m in models_rectified]
    Rt01 = _compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
    if not ((intrinsics[0][0] == "LENSMODEL_LATLON" and intrinsics[1][0] == "LENSMODEL_LATLON") or
            (intrinsics[0][0] == "LENSMODEL_PINHOLE" and intrinsics[1][0] == "LENSMODEL_PINHOLE")):
        raise RuntimeError(f"Expected two models with the same  'LENSMODEL_LATLON' or 'LENSMODEL_PINHOLE' but got "
                           f"{intrinsics[0][0]} and {intrinsics[1][0]}")
    if np.sum((intrinsics[0][1] - intrinsics[1][1]) ** 2) > 1e-6:
        raise RuntimeError("The two rectified models MUST have the same intrinsics values")
    if np.any(np.array(models_rectified[0].imagersize()) - np.array(models_rectified[1].imagersize())):
        raise RuntimeError("The two rectified models MUST have the same imager size")
    costh = (np.trace(Rt01[:3, :]) - 1.) / 2.
    if costh < 0.999999:
        raise RuntimeError("The two rectified models MUST have the same relative rotation")
    if np.sum(Rt01[3, 1:] ** 2) > 1e-9:
        raise RuntimeError("The two rectified models MUST have a translation ONLY in the +x rectified direction")


def rectification_maps(models, models_rectified):
    """The maps that rectify images of the cameras `models` into `models_rectified`: float32 (2, Nel, Naz, 2), for
    each camera and rectified pixel the pixel of that camera that sees the same ray, as cv2.remap() consumes them.
    Computed on the device, one thread per rectified pixel per camera."""
    _validate_models_rectified(models_rectified)
    _require_gpu()
    Naz, Nel = (int(x) for x in models_rectified[0].imagersize())
    maps = np.zeros((2, Nel, Naz, 2), dtype=np.float32)
    lms, intr = [], []
    for m in models:
        lensmodel, intrinsics = m.intrinsics()
        lms.append(_lensmodel(lensmodel))
        intr.append(np.ascontiguousarray(intrinsics, np.float64))
    rect, fxycxy = models_rectified[0].intrinsics()
    fxycxy = np.ascontiguousarray(fxycxy, np.float64)
    r = [np.ascontiguousarray(m.rt_cam_ref()[:3]) for m in (models[0], models[1], models_rectified[0])]
    size = (C.c_uint * 2)(Naz, Nel)
    if not lib.mrcal_rectification_maps(_ptr(maps), C.byref(lms[0]), _ptr(intr[0]), _ptr(r[0]),
                                        C.byref(lms[1]), _ptr(intr[1]), _ptr(r[1]),
                                        _rectification_model_type(rect), _ptr(fxycxy), size, _ptr(r[2])):
        _fail("mrcal_rectification_maps()")
    return maps


def _range_arguments(disparity, models_rectified, disparity_scale, disparity_min, disparity_scaled_min,
                     disparity_max, disparity_scaled_max, qrect0):
    """stereo_range()'s argument handling (mrcal/stereo.py:1226-1277): the validation, the defaults of the bounds in
    the units of the path taken (scaled uint16 for a whole image, qrect0 is None; pixels otherwise), scalars"""
    _validate_models_rectified(models_rectified)
    if disparity_min is not None and disparity_scaled_min is not None and disparity_min != disparity_scaled_min:
        raise RuntimeError("disparity_min and disparity_scaled_min may not both be given")
    if disparity_max is not None and disparity_scaled_max is not None and disparity_max != disparity_scaled_max:
        raise RuntimeError("disparity_max and disparity_scaled_max may not both be given")
    # int16 disparities (OpenCV's) with no upper bound: the negative ones are invalid. They become large uint16 values
    if disparity_scaled_max is None and disparity_max is None and \
       (isinstance(disparity, np.ndarray) and disparity.dtype == np.int16):
        disparity_scaled_max = 0x7FFF
    if qrect0 is None:
        if disparity_scaled_min is None:
            disparity_scaled_min = 0 if disparity_min is None else disparity_min * disparity_scale
        if disparity_scaled_max is None:
            disparity_scaled_max = np.uint16(np.iinfo(np.uint16).max) if disparity_max is None else \
                disparity_max * disparity_scale
    else:
        if disparity_min is None:
            disparity_min = 0 if disparity_scaled_min is None else disparity_scaled_min / disparity_scale
        if disparity_max is None:
            disparity_max = np.finfo(float).max if disparity_scaled_max is None else disparity_scaled_max / disparity_scale
    is_scalar = np.ndim(disparity) == 0
    if is_scalar:
        disparity = np.array((disparity,))
    Rt01 = _compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
    rect, fxycxy = models_rectified[0].intrinsics()
    return dict(disparity=disparity, is_scalar=is_scalar, baseline=float(np.linalg.norm(Rt01[3, :])),
                rect=_rectification_model_type(rect), fxycxy=np.ascontiguousarray(fxycxy, np.float64),
                scaled_min=disparity_scaled_min, scaled_max=disparity_scaled_max,
                dmin=disparity_min, dmax=disparity_max)


def _dense_image(a, models_rectified, disparity_scale):
    """The uint16 disparity image of a whole rectified view, as the reference converts it (astype(np.uint16): -1
    becomes 65535)"""
    W, H = models_rectified[0].imagersize()
    if a["disparity"].shape != (H, W):
        raise RuntimeError(f"qrect0 is None, so the given disparity and full rectified images MUST have the same "
                           f"dimensions. I have disparity.shape={a['disparity'].shape} and "
                           f"models_rectified[0].imagersize()={models_rectified[0].imagersize()}")
    d16 = np.ascontiguousarray(a["disparity"].astype(np.uint16))
    img = _capi.ImageUint16(int(W), int(H), int(d16.strides[0]), d16.ctypes.data)
    return img, d16, (np.uint16(disparity_scale), np.uint16(a["scaled_min"]), np.uint16(a["scaled_max"]))


def _sparse_inputs(disparity, qrect0, disparity_scale):
    d = np.asarray(disparity, np.float64) / disparity_scale
    q = np.asarray(qrect0, np.float64)
    if q.ndim == 0 or q.shape[-1] != 2:
        raise RuntimeError(f"qrect0 must have shape (...,2); got {q.shape}")
    shape = np.broadcast_shapes(d.shape, q.shape[:-1])
    d = np.ascontiguousarray(np.broadcast_to(d, shape)).ravel()
    q = np.ascontiguousarray(np.broadcast_to(q, shape + (2,))).reshape(-1, 2)
    return d, q, shape


def stereo_range(disparity, models_rectified, *, disparity_scale=1, disparity_min=None, disparity_scaled_min=None,
                 disparity_max=None, disparity_scaled_max=None, qrect0=None):
    """Ranges from disparities, as mrcal.stereo_range() computes them. qrect0=None: disparity is a whole rectified
    image (Nel, Naz), read as scaled uint16 values; otherwise disparities (any shape, broadcast with qrect0 (...,2))
    at those rectified camera-0 pixels. Invalid disparities (<= 0, outside the bounds) and non-finite ranges give 0.
    A scalar disparity gives a scalar. Computed on the device, one thread per element."""
    a = _range_arguments(disparity, models_rectified, disparity_scale, disparity_min, disparity_scaled_min,
                         disparity_max, disparity_scaled_max, qrect0)
    if qrect0 is None:
        img, d16, (scale, smin, smax) = _dense_image(a, models_rectified, disparity_scale)
        _require_gpu()
        r = np.zeros(d16.shape)
        out = _capi.ImageDouble(img.w, img.h, int(r.strides[0]), r.ctypes.data)
        if not lib.mrcal_stereo_range_dense(C.byref(out), C.byref(img), int(scale), int(smin), int(smax), a["rect"],
                                            _ptr(a["fxycxy"]), a["baseline"]):
            _fail("mrcal_stereo_range_dense()")
    else:
        d, q, shape = _sparse_inputs(a["disparity"], qrect0, disparity_scale)
        _require_gpu()
        r = np.zeros(d.shape)
        if not lib.mrcal_stereo_range_sparse(_ptr(r), _ptr(d), _ptr(q), d.size, float(a["dmin"]), float(a["dmax"]),
                                             a["rect"], _ptr(a["fxycxy"]), a["baseline"]):
            _fail("mrcal_stereo_range_sparse()")
        r = r.reshape(shape)
    if a["is_scalar"]:
        r = r[0]
    return r


def stereo_unproject(disparity, models_rectified, *, ranges=None, disparity_scale=1, qrect0=None):
    """The point cloud, in rectified camera-0 coordinates, of disparities (as stereo_range() reads them) or of ranges
    (given instead: disparity=None): range times the unit ray of the rectified pixel, (0,0,0) where the range is 0.
    qrect0=None means the whole rectified image. The ranges and the points are computed on the device in one pass."""
    if (ranges is None and disparity is None) or (ranges is not None and disparity is not None):
        raise RuntimeError("Exactly one of (disparity,ranges) must be non-None")
    _validate_models_rectified(models_rectified)
    W, H = (int(x) for x in models_rectified[0].imagersize())
    rect, fxycxy = models_rectified[0].intrinsics()
    rect = _rectification_model_type(rect)
    fxycxy = np.ascontiguousarray(fxycxy, np.float64)
    if ranges is not None:
        _require_gpu()
        Rt01 = _compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
        baseline = float(np.linalg.norm(Rt01[3, :]))
        rg = np.asarray(ranges, np.float64)
        if qrect0 is None:
            shape = np.broadcast_shapes(rg.shape, (H, W))
            if shape != (H, W):
                raise RuntimeError(f"qrect0 is None, so ranges must broadcast to the rectified image ({H},{W}); "
                                   f"got {rg.shape}")
            rg, q = np.ascontiguousarray(np.broadcast_to(rg, shape)).ravel(), None
        else:
            rg, q, shape = _sparse_inputs(rg, qrect0, 1.)
        p = np.zeros((rg.size, 3))
        if not lib.mrcal_b200_stereo_unproject(_ptr(p), None, None, 0, 0, 0, None, _ptr(rg), _ptr(q) if q is not None else None,
                                               rg.size, W, 0., 0., rect, _ptr(fxycxy), baseline):
            _fail("mrcal_b200_stereo_unproject()")
        return p.reshape(shape + (3,))
    a = _range_arguments(disparity, models_rectified, disparity_scale, None, None, None, None, qrect0)
    _require_gpu()
    if qrect0 is None:
        img, d16, (scale, smin, smax) = _dense_image(a, models_rectified, disparity_scale)
        p = np.zeros((H, W, 3))
        if not lib.mrcal_b200_stereo_unproject(_ptr(p), None, C.byref(img), int(scale), int(smin), int(smax), None, None,
                                               None, 0, 0, 0., 0., rect, _ptr(fxycxy), a["baseline"]):
            _fail("mrcal_b200_stereo_unproject()")
        return p
    d, q, shape = _sparse_inputs(a["disparity"], qrect0, disparity_scale)
    p = np.zeros((d.size, 3))
    if not lib.mrcal_b200_stereo_unproject(_ptr(p), None, None, 0, 0, 0, _ptr(d), None, _ptr(q), d.size, 0,
                                           float(a["dmin"]), float(a["dmax"]), rect, _ptr(fxycxy), a["baseline"]):
        _fail("mrcal_b200_stereo_unproject()")
    p = p.reshape(shape + (3,))
    if a["is_scalar"] and np.ndim(qrect0) == 1:
        p = p[0]
    return p
