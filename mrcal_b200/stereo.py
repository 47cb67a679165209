"""Stereo rectification and ranging, with the reference's names, keyword arguments, defaults, return values and
refusals (mrcal/stereo.py:23-484, 784-923, 978-1308, 1453-1607):

    mrcal_b200.rectified_resolution(model0, ...)        -> (pixels_per_deg_az, pixels_per_deg_el)
    mrcal_b200.rectified_system(models, ...)            -> (model_rect0, model_rect1) [, metadata]
    mrcal_b200.rectification_maps(models, models_rect)  -> float32 (2, Nel, Naz, 2)
    mrcal_b200.stereo_range(disparity, models_rect)     -> ranges
    mrcal_b200.stereo_unproject(disparity, models_rect) -> points in rectified camera-0 coordinates
    mrcal_b200.apply_homography(H, q)                   -> q mapped through the homography H
    mrcal_b200.match_feature(image0, image1, q0, ...)   -> (q1, diagnostics)

The geometry is host code in libmrcal_b200.so (csrc/stereo.cu); the maps, the ranges and the points are computed on
the device, one thread per element. match_feature() decides on the host which features can be matched, and matches
all of them on the device in one call (csrc/match.cu). This module only marshals arguments.

TM_SQDIFF .. TM_CCOEFF_NORMED have OpenCV's values.
"""
import ctypes as C
import operator
import re
import sys

import numpy as np

from . import _capi
from ._capi import checked
from ._poses_host import compose_Rt
from .api import _lensmodel, _ptr, _require_gpu, lensmodel_metadata_and_config
from .cameramodel import cameramodel

# the reference's Python wrapper takes an az0_deg above this for "autodetect" (mrcal-pywrap.c:4029-4030)
_AZ0_AUTODETECT = 1e7

# cv2.TemplateMatchModes
TM_SQDIFF, TM_SQDIFF_NORMED, TM_CCORR, TM_CCORR_NORMED, TM_CCOEFF, TM_CCOEFF_NORMED = range(6)
# match_feature()'s per-feature status in a batched call (MRCAL_B200_MATCH_* of include/mrcal_b200.h)
MATCH_OK, MATCH_EDGE_PEAK, MATCH_OUTSIDE_IMAGE1, MATCH_OUTSIDE_IMAGE0, MATCH_SEARCH_TOO_SMALL = range(5)


def _rectification_model_type(name):
    return _lensmodel(name).type


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
    checked.mrcal_rectified_resolution(C.byref(az), C.byref(el), C.byref(lm), _ptr(intr), azel_fov, azel0, _ptr(R),
                                       _rectification_model_type(rectification_model))
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
    checked.mrcal_rectified_system2(imagersize, _ptr(fxycxy), _ptr(rt_rect0_ref), C.byref(baseline), C.byref(az),
                                    C.byref(el), azel_fov, azel0, float(az_edge_margin_deg), C.byref(lm), _ptr(intr),
                                    _ptr(rt0), _ptr(rt1), _rectification_model_type(rectification_model),
                                    az0_deg > _AZ0_AUTODETECT / 10., False, False, False)
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
    Rt01 = compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
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
    checked.mrcal_rectification_maps(_ptr(maps), C.byref(lms[0]), _ptr(intr[0]), _ptr(r[0]), C.byref(lms[1]),
                                     _ptr(intr[1]), _ptr(r[1]), _rectification_model_type(rect), _ptr(fxycxy), size,
                                     _ptr(r[2]))
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
    Rt01 = compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
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
        checked.mrcal_stereo_range_dense(C.byref(out), C.byref(img), int(scale), int(smin), int(smax), a["rect"],
                                         _ptr(a["fxycxy"]), a["baseline"])
    else:
        d, q, shape = _sparse_inputs(a["disparity"], qrect0, disparity_scale)
        _require_gpu()
        r = np.zeros(d.shape)
        checked.mrcal_stereo_range_sparse(_ptr(r), _ptr(d), _ptr(q), d.size, float(a["dmin"]), float(a["dmax"]),
                                          a["rect"], _ptr(a["fxycxy"]), a["baseline"])
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
        Rt01 = compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
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
        checked.mrcal_b200_stereo_unproject(_ptr(p), None, None, 0, 0, 0, None, _ptr(rg), _ptr(q), rg.size, W, 0., 0.,
                                            rect, _ptr(fxycxy), baseline)
        return p.reshape(shape + (3,))
    a = _range_arguments(disparity, models_rectified, disparity_scale, None, None, None, None, qrect0)
    _require_gpu()
    if qrect0 is None:
        img, d16, (scale, smin, smax) = _dense_image(a, models_rectified, disparity_scale)
        p = np.zeros((H, W, 3))
        checked.mrcal_b200_stereo_unproject(_ptr(p), None, C.byref(img), int(scale), int(smin), int(smax), None, None,
                                            None, 0, 0, 0., 0., rect, _ptr(fxycxy), a["baseline"])
        return p
    d, q, shape = _sparse_inputs(a["disparity"], qrect0, disparity_scale)
    p = np.zeros((d.size, 3))
    checked.mrcal_b200_stereo_unproject(_ptr(p), None, None, 0, 0, 0, _ptr(d), None, _ptr(q), d.size, 0,
                                        float(a["dmin"]), float(a["dmax"]), rect, _ptr(fxycxy), a["baseline"])
    p = p.reshape(shape + (3,))
    if a["is_scalar"] and np.ndim(qrect0) == 1:
        p = p[0]
    return p


####################################################################################################
# feature matching
####################################################################################################
def apply_homography(H, q):
    """q (..., 2) mapped through the homography H (..., 3, 3), broadcasting: ((H00 x + H01 y) + H02) / ((H20 x + H21 y)
    + H22), and likewise for y, as the reference computes it. In float32 if both are float32, else in float64; every
    operation is rounded on its own, so the bits are the reference's"""
    H, q = np.asarray(H), np.asarray(q)
    if H.ndim < 2 or H.shape[-2:] != (3, 3):
        raise RuntimeError(f"H must have shape (...,3,3); got {H.shape}")
    if q.ndim < 1 or q.shape[-1] != 2:
        raise RuntimeError(f"q must have shape (...,2); got {q.shape}")
    dtype = np.float32 if H.dtype == np.float32 and q.dtype == np.float32 else np.float64
    H, q = H.astype(dtype, copy=False), q.astype(dtype, copy=False)
    x, y = q[..., 0], q[..., 1]
    with np.errstate(all="ignore"):
        xyz = [(H[..., i, 0] * x + H[..., i, 1] * y) + H[..., i, 2] for i in range(3)]
        return np.stack((xyz[0] / xyz[2], xyz[1] / xyz[2]), axis=-1)


def _template_size(template_size1):
    """(width, height), refused as the reference refuses it (stereo.py:1853-1862)"""
    try:
        N = len(template_size1)
    except TypeError:
        N = 2
        template_size1 = (template_size1, template_size1)
    if N != 2:
        raise RuntimeError(f"template_size1 must be an interable of length 2 OR a scalar. Got an iterable of length {N}")
    for i in range(2):
        if not (isinstance(template_size1[i], int) and template_size1[i] > 0):
            raise RuntimeError(f"Each element of template_size1 must be an integer > 0. Got {template_size1[i]}")
    return np.array(template_size1, dtype=int)


def _edge_refusal(shape, what, *qall):
    """the reference's checkdims() message for the first of qall outside an image of this shape (H, W); None if all
    are inside. NaN coordinates are inside, as the reference's comparisons have it"""
    for q in qall:
        if q[0] < 0:
            return f"Too close to the left edge in {what}"
        if q[1] < 0:
            return f"Too close to the top edge in {what} "
        if q[0] >= shape[1]:
            return f"Too close to the right edge in {what} "
        if q[1] >= shape[0]:
            return f"Too close to the bottom edge in {what} "
    return None


def _images(image0, image1):
    """(torch or None, dtype code, (H0, W0), (H1, W1)) of two images that cv2.matchTemplate() would accept: 2-D, both
    uint8 or both float32; numpy arrays, or contiguous torch CUDA tensors on one device"""
    if image0.ndim != 2 or image1.ndim != 2:
        raise RuntimeError("match_feature() accepts ONLY grayscale images of shape (H,W)")
    torch = sys.modules.get("torch")
    is_tensor = [torch is not None and isinstance(x, torch.Tensor) for x in (image0, image1)]
    if any(is_tensor):
        if not all(is_tensor):
            raise RuntimeError("match_feature(): image0 and image1 must both be numpy arrays or both be torch CUDA "
                               "tensors")
        if not (image0.is_cuda and image1.is_cuda) or image0.device != image1.device:
            raise RuntimeError("match_feature(): torch images must be CUDA tensors on one device")
        if not (image0.is_contiguous() and image1.is_contiguous()):
            raise RuntimeError("match_feature(): torch images must be contiguous")
        types = {torch.uint8: 0, torch.float32: 2}
    else:
        if not (isinstance(image0, np.ndarray) and isinstance(image1, np.ndarray)):
            raise RuntimeError("match_feature(): image0 and image1 must be numpy arrays or torch CUDA tensors")
        torch = None
        types = {np.dtype(np.uint8): 0, np.dtype(np.float32): 2}
    if image0.dtype != image1.dtype:
        raise RuntimeError(f"match_feature(): image0 and image1 must have the same dtype, as cv2.matchTemplate() "
                           f"requires; got {image0.dtype} and {image1.dtype}")
    if image0.dtype not in types:
        raise RuntimeError(f"match_feature() supports uint8 and float32 images only, as cv2.matchTemplate() does; "
                           f"got {image0.dtype}")
    return torch, types[image0.dtype], tuple(image0.shape), tuple(image1.shape)


def _packed_rows(image):
    """image, or a copy of it, with packed pixels and a positive row stride"""
    if image.strides[1] != image.itemsize or image.strides[0] < image.shape[1] * image.itemsize:
        image = np.ascontiguousarray(image)
    return image


def _match_features(image0, image1, q0, search_radius1, template_size1, q1_estimate, H10, method, single,
                    return_templates=False):
    """match_feature()'s work for q0 (2,) (single) or (N,2). Returns a dict of per-feature arrays: status, q1,
    q1_estimate, q1_template_min, q1_min, at, value, qshift and matchoutput_image; the message of the refusal
    a single call raises (None if it does not); and, with return_templates, the (M, th, tw) templates of the features
    that were matched"""
    ts = _template_size(template_size1)
    if image0.ndim != 2 or image1.ndim != 2:
        raise RuntimeError("match_feature() accepts ONLY grayscale images of shape (H,W)")
    if (H10 is None) == (q1_estimate is None):
        raise RuntimeError("Exactly one of (q1_estimate,H10) must be given")
    torch, type_code, shape0, shape1 = _images(image0, image1)
    if method is None:
        method = TM_CCORR_NORMED
    if method not in range(6):
        raise RuntimeError(f"method must be one of the TM_* constants 0..5; got {method}")
    try:
        r = operator.index(search_radius1)
    except TypeError:
        raise RuntimeError(f"search_radius1 must be an integer; got {search_radius1!r}") from None

    # the reference's scalars, in its dtypes (stereo.py:1876-1901), for all features at once
    q0 = np.asarray(q0).astype(np.float32)
    if q0.shape[-1:] != (2,) or q0.ndim != (1 if single else 2):
        raise RuntimeError(f"q0 must have shape (2,) or (N,2); got {q0.shape}")
    q0 = q0.reshape(-1, 2)
    N = q0.shape[0]
    if H10 is None:
        q1e = np.asarray(q1_estimate)
        if q1e.shape not in ((2,), (N, 2)):
            raise RuntimeError(f"q1_estimate must have shape (2,) or (N,2); got {q1e.shape}")
        q1e = np.broadcast_to(q1e, (N, 2))
        H = np.zeros((N, 3, 3), np.float32)
        H[:, 0, 0] = H[:, 1, 1] = H[:, 2, 2] = 1.
        H[:, :2, 2] = q1e - q0
        q1e = q1e.astype(np.float32)
    else:
        H = np.asarray(H10).astype(np.float32)
        if H.shape not in ((3, 3), (N, 3, 3)):
            raise RuntimeError(f"H10 must have shape (3,3) or (N,3,3); got {H.shape}")
        H = np.ascontiguousarray(np.broadcast_to(H, (N, 3, 3)))
        q1e = apply_homography(H, q0)
    tmin_f = np.round(q1e - (ts - 1.) / 2.)

    status = np.full(N, MATCH_OK, np.int32)
    H1, W1 = shape1
    # a template whose corner is not a finite pixel of image 1 is outside it, as the reference's integer cast makes it
    finite = np.all(np.isfinite(tmin_f) & (np.abs(tmin_f) < 2. ** 40), axis=1)
    tmin = np.where(finite[:, None], tmin_f, 0.).astype(int)
    tmax = tmin + ts - 1
    out1 = ~finite | np.any((tmin < 0) | (tmax < 0), axis=1) | \
        (tmin[:, 0] >= W1) | (tmin[:, 1] >= H1) | (tmax[:, 0] >= W1) | (tmax[:, 1] >= H1)
    status[out1] = MATCH_OUTSIDE_IMAGE1
    refusal = None
    if single and out1[0]:
        # the corner as the reference's astype(int) makes it: NaN, +-inf and anything beyond int64 become INT64_MIN
        t = [int(v) if np.isfinite(v) and abs(v) < 2. ** 63 else -2 ** 63 for v in tmin_f[0]]
        refusal = _edge_refusal(shape1, "image1", t, [v + int(n) - 1 for v, n in zip(t, ts)])

    # the templates' maps: np.linalg.inv() in float32, the call the reference makes. A singular H10 raises in a single
    # call, as in the reference; in a batch, its feature has no template in image 0
    if single:
        Hinv = np.linalg.inv(H[0])[None] if refusal is None else np.eye(3, dtype=np.float32)[None]
    else:
        try:
            Hinv = np.linalg.inv(H)
        except np.linalg.LinAlgError:
            Hinv = np.empty_like(H)
            for i in range(N):
                try:
                    Hinv[i] = np.linalg.inv(H[i])
                except np.linalg.LinAlgError:
                    Hinv[i] = np.nan
                    if status[i] == MATCH_OK:
                        status[i] = MATCH_OUTSIDE_IMAGE0
    # the map's corners [0,0], [-1,0], [0,-1], [-1,-1], checked on image 0 (stereo.py:1927-1933)
    corners = np.stack((tmin, np.stack((tmin[:, 0], tmax[:, 1]), 1), np.stack((tmax[:, 0], tmin[:, 1]), 1), tmax),
                       axis=1).astype(np.float32)
    q0c = apply_homography(Hinv[:, None], corners)
    H0, W0 = shape0
    with np.errstate(invalid="ignore"):
        out0 = np.any((q0c[..., 0] < 0) | (q0c[..., 1] < 0) | (q0c[..., 0] >= W0) | (q0c[..., 1] >= H0), axis=1)
    status[(status == MATCH_OK) & out0] = MATCH_OUTSIDE_IMAGE0
    if single and refusal is None and out0[0]:
        refusal = _edge_refusal(shape0, "image0", *q0c[0])

    # the search cut, clipped to image 1 (stereo.py:1939-1950)
    qmin = np.maximum(tmin - r, 0)
    qmax = np.minimum(tmin + r + ts - 1, (W1 - 1, H1 - 1))
    cut = qmax - qmin + 1
    small = np.any(cut < ts, axis=1)
    status[(status == MATCH_OK) & small] = MATCH_SEARCH_TOO_SMALL
    if single and refusal is None and small[0]:
        refusal = f"match_feature(): the search region {cut[0][0]}x{cut[0][1]} of image1 is smaller than the " \
                  f"template {ts[0]}x{ts[1]}, which cv2.matchTemplate() refuses"

    run = np.flatnonzero(status == MATCH_OK)
    M = run.size
    slot_w, slot_h = (max(1, min(2 * r + 1, n - t + 1)) for n, t in ((W1, ts[0]), (H1, ts[1])))
    features = np.ascontiguousarray(np.concatenate((tmin[run], qmin[run], cut[run]), axis=1), np.int32)
    Hinv_run = np.ascontiguousarray(Hinv[run], np.float32).reshape(M, 9)
    # out: M rows of (x, y, value, status), then the M slots of float32 match output, in one buffer and one download
    buf = np.empty(4 * M + (M * slot_w * slot_h + 1) // 2, np.float64)
    dtype = np.uint8 if type_code == 0 else np.float32
    templates = np.empty((M, ts[1], ts[0]), dtype) if return_templates else None
    args = (features.ctypes.data, Hinv_run.ctypes.data, M, int(ts[0]), int(ts[1]), slot_w, slot_h, int(method))
    if M > 0:
        if torch is None:
            image0, image1 = _packed_rows(image0), _packed_rows(image1)
            _require_gpu()
            checked.mrcal_b200_match_feature(buf.ctypes.data, _ptr(templates), image0.ctypes.data, W0, H0,
                                             image0.strides[0], image1.ctypes.data, W1, H1, image1.strides[0],
                                             type_code, *args)
        else:
            es = image0.element_size()
            with torch.cuda.device(image0.device):
                stream = torch.cuda.current_stream(image0.device).cuda_stream
                checked.mrcal_b200_match_feature_device(buf.ctypes.data, _ptr(templates), image0.data_ptr(), W0, H0,
                                                        W0 * es, image1.data_ptr(), W1, H1, W1 * es, type_code, *args,
                                                        stream)
    res = buf[:4 * M].reshape(M, 4)
    slots = buf[4 * M:].view(np.float32)[:M * slot_w * slot_h].reshape(M, slot_w * slot_h)

    status[run] = res[:, 3].astype(np.int32)
    at = np.full((N, 2), np.nan)
    value = np.full(N, np.nan)
    at[run], value[run] = res[:, :2], res[:, 2]
    qshift = np.full((N, 2), np.nan)
    qshift[run] = qmin[run] + q1e[run] - tmin[run]
    ok = status == MATCH_OK
    at[~ok], value[~ok], qshift[~ok] = np.nan, np.nan, np.nan
    q1 = at + qshift
    matchoutput = [None] * N
    for k, i in enumerate(run):
        ow, oh = cut[i] - ts + 1
        matchoutput[i] = slots[k, :ow * oh].reshape(oh, ow)
    result = dict(status=status, q1=q1, at=at, value=value, qshift=qshift, matchoutput_image=matchoutput)
    return result, refusal, templates


def match_feature(image0, image1, q0, *, search_radius1, template_size1, q1_estimate=None, H10=None, method=None,
                  visualize=False, extratitle=None, return_plot_args=False, **kwargs):
    """The pixel of image1 that matches the pixel q0 of image0, as mrcal.match_feature() finds it: the template is
    image0 remapped through the homography H10 (or the translation to q1_estimate) around q1_estimate =
    apply_homography(H10, q0), template_size1 (width, height) pixels of image1; it is matched with method (OpenCV's
    TM_*; TM_CCORR_NORMED by default) over a window of image1 search_radius1 pixels around it in each direction, clipped
    to the image; the discrete optimum is refined by a quadratic fit to its 3x3 neighbourhood.

    q0 (2,): returns (q1, diagnostics) with the reference's keys; q1 is None if the optimum is on the edge of the match
    output. It raises where the reference or cv2.matchTemplate() would: a template too close to an edge of either image,
    bad arguments, mixed or unsupported dtypes, a search region smaller than the template.

    q0 (N,2): every feature in one call; H10 (3,3) or (N,3,3), q1_estimate (2,) or (N,2). Returns q1 (N,2), NaN where a
    feature failed, and diagnostics of stacked arrays (matchoutput_optimum_subpixel_at, matchoutput_optimum_subpixel,
    qshift_image1_matchoutput, NaN where a feature failed), a per-feature status (MATCH_OK, MATCH_EDGE_PEAK,
    MATCH_OUTSIDE_IMAGE1, MATCH_OUTSIDE_IMAGE0, MATCH_SEARCH_TOO_SMALL) and matchoutput_image, a list of each feature's
    match output (None where there is none). No feature's failure raises, and row i is bit for bit the single call's.

    Images: 2-D, both uint8 or both float32; numpy arrays (rows may be strided) or contiguous torch CUDA tensors on one
    device, in which case the work is enqueued on torch.cuda.current_stream() with nothing uploaded. The results are
    numpy arrays either way. visualize=True is refused: it needs gnuplotlib, which this package does not use."""
    if visualize:
        raise RuntimeError("match_feature(visualize=True) is not supported: it plots with gnuplotlib, which this "
                           "package does not use. The diagnostics hold what the plot shows")
    single = np.ndim(q0) == 1
    r, refusal, _ = _match_features(image0, image1, q0, search_radius1, template_size1, q1_estimate, H10, method,
                                    single)
    if not single:
        diagnostics = dict(matchoutput_image=r["matchoutput_image"], matchoutput_optimum_subpixel_at=r["at"],
                           matchoutput_optimum_subpixel=r["value"], qshift_image1_matchoutput=r["qshift"],
                           status=r["status"])
        return r["q1"], diagnostics
    if refusal is not None:
        raise RuntimeError(refusal)
    diagnostics = dict(matchoutput_image=r["matchoutput_image"][0])
    if r["status"][0] != MATCH_OK:
        return None, diagnostics
    diagnostics["matchoutput_optimum_subpixel_at"] = r["at"][0]
    diagnostics["matchoutput_optimum_subpixel"] = r["value"][0]
    diagnostics["qshift_image1_matchoutput"] = r["qshift"][0]
    return r["q1"][0], diagnostics
