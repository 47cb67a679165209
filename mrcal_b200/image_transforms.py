"""Image reprojection, with the reference's names, keyword arguments, defaults, return values and refusals
(mrcal/image_transforms.py):

    mrcal_b200.scale_focal__best_pinhole_fit(model, fit)          -> scale
    mrcal_b200.pinhole_model_for_reprojection(model_from, ...)    -> a LENSMODEL_PINHOLE cameramodel
    mrcal_b200.image_transformation_map(model_from, model_to)     -> float32 (H_to, W_to, 2)
    mrcal_b200.transform_image(image, mapxy)                      -> the remapped image

image_transformation_map() and transform_image() run on the device, one thread per target pixel
(csrc/image_transforms.cu). transform_image() restates cv2.remap()'s arithmetic, so it needs no OpenCV, and it also
takes torch CUDA tensors: maps uploaded once, each frame then costs one kernel on the current stream.

INTER_NEAREST, INTER_LINEAR, BORDER_CONSTANT and BORDER_TRANSPARENT have OpenCV's values.
"""
import ctypes as C
import re
import sys

import numpy as np

from ._capi import checked
from ._poses_host import compose_Rt
from .api import _lensmodel, _ptr, _require_gpu, lensmodel_metadata_and_config, unproject
from .cameramodel import cameramodel

INTER_NEAREST = 0
INTER_LINEAR = 1
BORDER_CONSTANT = 0
BORDER_TRANSPARENT = 5

_FITS = ("corners", "centers-horizontal", "centers-vertical")
# element type codes of include/mrcal_b200.h (MRCAL_B200_IMAGE_*)
_NUMPY_TYPES = {np.dtype(np.uint8): 0, np.dtype(np.uint16): 1, np.dtype(np.float32): 2}


def _require_core(lensmodel):
    if not lensmodel_metadata_and_config(lensmodel)["has_core"]:
        raise RuntimeError("This currently works only with models that have an fxfycxcy core")


def scale_focal__best_pinhole_fit(model, fit):
    """The largest scale k of model's focal lengths for which a pinhole (k fx, k fy, cx, cy) still sees every pixel of
    `fit`: an (N,2) array of pixels of model, or "corners", "centers-horizontal" or "centers-vertical" of its imager.
    fit=None gives 1. The pixels are unprojected on the device."""
    if fit is None:
        return 1.0
    W, H = WH = np.array(model.imagersize(), dtype=float)
    if type(fit) is np.ndarray:
        q_edges = fit
    elif type(fit) is str and fit in _FITS:
        q_edges = {"corners": np.array(((0., 0.), (0., H - 1.), (W - 1., H - 1.), (W - 1., 0.))),
                   "centers-horizontal": np.array(((0, (H - 1.) / 2.), (W - 1., (H - 1.) / 2.))),
                   "centers-vertical": np.array((((W - 1.) / 2., 0), ((W - 1.) / 2., H - 1.)))}[fit]
    else:
        raise RuntimeError("fit must be either None or a numpy array or one of "
                           "('corners','centers-horizontal','centers-vertical')")
    lensmodel, intrinsics_data = model.intrinsics()
    _require_core(lensmodel)
    v_edges = unproject(q_edges, lensmodel, intrinsics_data)
    fxy, cxy = intrinsics_data[:2], intrinsics_data[2:4]
    # each point's pinhole projection k fxy xy/z + cxy must stay in [0, WH-1]; the most conservative k wins
    normxy_edges = v_edges[:, :2] / v_edges[:, (2,)]
    normxy_min = (-cxy) / fxy
    normxy_max = (WH - 1. - cxy) / fxy
    scale = 1e6
    for p in normxy_edges:
        for ixy in range(2):
            if p[ixy] > 0:
                scale = np.min((scale, normxy_max[ixy] / p[ixy]))
            else:
                scale = np.min((scale, normxy_min[ixy] / p[ixy]))
    return float(scale)


def pinhole_model_for_reprojection(model_from, fit=None, *, scale_focal=None, scale_image=None):
    """A LENSMODEL_PINHOLE model with model_from's core and pose, for undistorting its images: the focal lengths
    scaled by scale_focal, or by scale_focal__best_pinhole_fit(model_from, fit); the imager scaled by scale_image
    (rounded as Python's round() does) with the centre pixel unprojecting to the same ray."""
    if scale_focal is None:
        if fit is not None:
            if isinstance(fit, np.ndarray):
                if fit.shape[-1] != 2:
                    raise RuntimeError("'fit' is an array, so it must have shape (...,2)")
                fit = fit.reshape(-1, 2)
            elif not (isinstance(fit, str) and re.match("^(corners|centers-horizontal|centers-vertical)$", fit)):
                raise RuntimeError("'fit' must be an array of shape (...,2) or one of "
                                   "('corners','centers-horizontal','centers-vertical')")
        scale_focal = scale_focal__best_pinhole_fit(model_from, fit)
    elif fit is not None:
        raise RuntimeError("At most one of 'scale_focal' and 'fit' may be non-None")

    lensmodel, intrinsics_data = model_from.intrinsics()
    imagersize = model_from.imagersize()
    _require_core(lensmodel)
    cx, cy = intrinsics_data[2:4]
    intrinsics_data[:2] *= scale_focal
    if scale_image is not None:
        # the centre of the imager keeps its ray: (WH-1)/2 - cxy)/fxy is unchanged with fxy scaled by ki = scale_image
        # and cxy by kc = (ki + 2 cxy ki - 1) / (2 cxy)
        imagersize[0] = round(imagersize[0] * scale_image)
        imagersize[1] = round(imagersize[1] * scale_image)
        kfxy = scale_image
        kcx = (kfxy + 2. * cx * kfxy - 1.) / (2. * cx)
        kcy = (kfxy + 2. * cy * kfxy - 1.) / (2. * cy)
        intrinsics_data[:2] *= kfxy
        intrinsics_data[2] *= kcx
        intrinsics_data[3] *= kcy
    return cameramodel(intrinsics=("LENSMODEL_PINHOLE", intrinsics_data[:4]), rt_cam_ref=model_from.rt_cam_ref(),
                       imagersize=imagersize)


def image_transformation_map(model_from, model_to, *, intrinsics_only=False, distance=None, plane_n=None, plane_d=None,
                             mask_valid_intrinsics_region_from=False):
    """The map (H_to, W_to, 2), float32, from each pixel of model_to's imager to the pixel of model_from that sees the
    same point, for transform_image(). By default the points are at infinity (only the relative rotation matters);
    `distance` puts them that far out along each ray; plane_n, plane_d (in model_from's frame: all p with
    inner(p, plane_n) = plane_d) map a plane; intrinsics_only ignores the poses. With
    mask_valid_intrinsics_region_from, map points outside model_from's valid-intrinsics region become (-1, -1).
    Every pixel is unprojected, transformed and projected on the device."""
    if (plane_n is None) != (plane_d is None):
        raise RuntimeError("plane_n and plane_d should both be None or neither should be None")
    if plane_n is not None and intrinsics_only:
        raise RuntimeError("We're looking at remapping a plane (plane_d, plane_n are not None), so intrinsics_only "
                           "should be False")
    if distance is not None and (plane_n is not None or intrinsics_only):
        raise RuntimeError("'distance' makes sense only without plane_n/plane_d and without intrinsics_only")

    lensmodel_from, intrinsics_from = model_from.intrinsics()
    lensmodel_to, intrinsics_to = model_to.intrinsics()
    lm_from, lm_to = _lensmodel(lensmodel_from), _lensmodel(lensmodel_to)
    if re.match("^LENSMODEL_CAHVORE", lensmodel_to) and np.any(intrinsics_to[-3:] != 0):
        raise RuntimeError("unproject() currently only works with a central projection. So I cannot "
                           "unproject(CAHVORE,E!=0)")
    region = None
    if mask_valid_intrinsics_region_from:
        region = model_from.valid_intrinsics_region()
        if region is None:
            raise RuntimeError("mask_valid_intrinsics_region_from is True, but model_from has no "
                               "valid_intrinsics_region")
        region = np.ascontiguousarray(region, np.float64)
    Rt_to_from = None if intrinsics_only else \
        np.ascontiguousarray(compose_Rt(model_to.Rt_cam_ref(), model_from.Rt_ref_cam()), np.float64)
    if plane_n is not None:
        plane_n = np.ascontiguousarray(plane_n, np.float64)
        if plane_n.shape != (3,):
            raise RuntimeError(f"plane_n must have shape (3,); got {plane_n.shape}")
    d = None if distance is None else np.array([float(distance)])
    _require_gpu()

    W, H = (int(x) for x in model_to.imagersize())
    mapxy = np.empty((H, W, 2), dtype=np.float32)
    checked.mrcal_b200_image_transformation_map(_ptr(mapxy), W, H, C.byref(lm_from),
                                                _ptr(np.ascontiguousarray(intrinsics_from, np.float64)), C.byref(lm_to),
                                                _ptr(np.ascontiguousarray(intrinsics_to, np.float64)), _ptr(Rt_to_from),
                                                _ptr(d), _ptr(plane_n), 0. if plane_d is None else float(plane_d),
                                                _ptr(region), 0 if region is None else region.shape[0])
    return mapxy


def _border_values(borderValue):
    """OpenCV's Scalar: a number v means (v, 0, 0); a sequence of up to 4 values is padded with zeros"""
    v = np.atleast_1d(np.asarray(borderValue, np.float64))
    if v.ndim != 1 or v.size > 4:
        raise RuntimeError(f"borderValue must be a number or up to 4 numbers; got {borderValue!r}")
    out = np.zeros(3)
    n = min(v.size, 3)
    out[:n] = v[:n]
    return out


def _image_layout(shape, what):
    """(H, W, channels) of an image of this shape; refuses what transform_image() does not support"""
    if len(shape) == 2:
        return shape[0], shape[1], 1
    if len(shape) == 3 and shape[2] == 3:
        return shape[0], shape[1], 3
    raise RuntimeError(f"transform_image() supports images of shape (H,W) and (H,W,3) only; {what} has shape "
                       f"{tuple(shape)}")


def _torch_if_tensors(*xs, what="transform_image(): image, mapxy and out"):
    """torch, if the given arrays are torch tensors; None if they are not. Mixing the two is refused: `what` names the
    caller and its arrays in the message. torch is only imported by a caller who already has tensors"""
    torch = sys.modules.get("torch")
    given = [x for x in xs if x is not None]
    is_tensor = [torch is not None and isinstance(x, torch.Tensor) for x in given]
    if not any(is_tensor):
        return None
    if not all(is_tensor):
        raise RuntimeError(f"{what} must all be numpy arrays or all be torch CUDA tensors; they may not be mixed")
    return torch


def transform_image(image, mapxy, *, out=None, borderMode=None, borderValue=0, interpolation=None):
    """image remapped through mapxy (Ho, Wo, 2), float32: out[y, x] = image sampled at mapxy[y, x], as cv2.remap()
    computes it, pixel for pixel. image: uint8, uint16 or float32, of shape (H, W) or (H, W, 3); its rows may be
    strided. interpolation: INTER_LINEAR (the default) or INTER_NEAREST. borderMode: BORDER_CONSTANT (the default;
    pixels from outside the image take borderValue) or BORDER_TRANSPARENT (they are left as out has them; 0 if no out
    is given). image, mapxy and out may instead all be torch CUDA tensors on one device, contiguous: the result is then
    a tensor and the kernel is enqueued on torch.cuda.current_stream() without waiting for it."""
    if borderMode is None:
        borderMode = BORDER_CONSTANT
    if interpolation is None:
        interpolation = INTER_LINEAR
    if interpolation not in (INTER_NEAREST, INTER_LINEAR):
        raise RuntimeError(f"transform_image() supports interpolation=INTER_NEAREST (0) and INTER_LINEAR (1) only; "
                           f"got {interpolation}")
    if borderMode not in (BORDER_CONSTANT, BORDER_TRANSPARENT):
        raise RuntimeError(f"transform_image() supports borderMode=BORDER_CONSTANT (0) and BORDER_TRANSPARENT (5) "
                           f"only; got {borderMode}")
    bv = _border_values(borderValue)
    torch = _torch_if_tensors(image, mapxy, out)
    if torch is not None:
        return _transform_image_device(torch, image, mapxy, out, borderMode, bv, interpolation)

    if not isinstance(image, np.ndarray):
        raise RuntimeError("'image' must be a numpy array")
    if not isinstance(mapxy, np.ndarray):
        raise RuntimeError("'mapxy' must be a numpy array")
    if image.dtype not in _NUMPY_TYPES:
        raise RuntimeError(f"transform_image() supports uint8, uint16 and float32 images only; got {image.dtype}")
    H, W, channels = _image_layout(image.shape, "image")
    if mapxy.dtype != np.float32 or mapxy.ndim != 3 or mapxy.shape[2] != 2:
        raise RuntimeError(f"mapxy must be a float32 array of shape (Nheight,Nwidth,2); got {mapxy.dtype} "
                           f"{mapxy.shape}")
    Ho, Wo = mapxy.shape[:2]
    out_shape = (Ho, Wo) if channels == 1 else (Ho, Wo, 3)
    if out is None:
        out = np.zeros(out_shape, image.dtype)
    elif not isinstance(out, np.ndarray) or out.shape != out_shape or out.dtype != image.dtype:
        raise RuntimeError(f"out must be a numpy array of shape {out_shape} and dtype {image.dtype}")
    elif not out.flags.c_contiguous or not out.flags.writeable:
        raise RuntimeError("out must be C-contiguous and writeable")
    # rows may be strided; the pixels of a row must be packed
    item = image.dtype.itemsize
    if image.strides[1] != channels * item or (channels == 3 and image.strides[2] != item) or image.strides[0] <= 0:
        image = np.ascontiguousarray(image)
    mapxy = np.ascontiguousarray(mapxy)
    _require_gpu()
    checked.mrcal_b200_transform_image(out.ctypes.data, image.ctypes.data, W, H, image.strides[0],
                                       _NUMPY_TYPES[image.dtype], channels, _ptr(mapxy), Wo, Ho, interpolation,
                                       borderMode, _ptr(bv))
    return out


def _transform_image_device(torch, image, mapxy, out, borderMode, bv, interpolation):
    types = {torch.uint8: 0, torch.uint16: 1, torch.float32: 2}
    tensors = [t for t in (image, mapxy, out) if t is not None]
    if not all(t.is_cuda for t in tensors):
        raise RuntimeError("transform_image(): torch tensors must be CUDA tensors")
    if any(t.device != image.device for t in tensors):
        raise RuntimeError("transform_image(): image, mapxy and out must be on the same device")
    if not all(t.is_contiguous() for t in tensors):
        raise RuntimeError("transform_image(): torch tensors must be contiguous")
    if image.dtype not in types:
        raise RuntimeError(f"transform_image() supports uint8, uint16 and float32 images only; got {image.dtype}")
    H, W, channels = _image_layout(tuple(image.shape), "image")
    if mapxy.dtype != torch.float32 or mapxy.dim() != 3 or mapxy.shape[2] != 2:
        raise RuntimeError(f"mapxy must be a float32 tensor of shape (Nheight,Nwidth,2); got {mapxy.dtype} "
                           f"{tuple(mapxy.shape)}")
    Ho, Wo = (int(x) for x in mapxy.shape[:2])
    out_shape = (Ho, Wo) if channels == 1 else (Ho, Wo, 3)
    if out is None:
        alloc = torch.zeros if borderMode == BORDER_TRANSPARENT else torch.empty
        out = alloc(out_shape, dtype=image.dtype, device=image.device)
    elif tuple(out.shape) != out_shape or out.dtype != image.dtype:
        raise RuntimeError(f"out must be a tensor of shape {out_shape} and dtype {image.dtype}")
    # the launch goes to the tensors' device, whichever device is current
    with torch.cuda.device(image.device):
        stream = torch.cuda.current_stream(image.device).cuda_stream
        checked.mrcal_b200_transform_image_device(out.data_ptr(), image.data_ptr(), W, H,
                                                  W * channels * image.element_size(), types[image.dtype], channels,
                                                  mapxy.data_ptr(), Wo, Ho, interpolation, borderMode, _ptr(bv), stream)
    return out
