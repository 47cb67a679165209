"""CPU: every one-shot C entry point, called with valid arguments and no device, refuses with the library's
no-device message instead of touching device memory."""
import ctypes as C

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import _capi
from mrcal_b200.api import _lensmodel, _ptr

pytestmark = pytest.mark.skipif(mrcal_b200.device_count() > 0, reason="checks the behaviour without a device")

LIB = _capi.lib
INTR = np.array((1000., 1000., 499.5, 399.5))
FXYCXY = np.array((800., 800., 320., 240.))


def _refused(ok):
    assert not ok
    assert "no usable CUDA device" in _capi.last_error()


def test_project_unproject():
    lm = _lensmodel("LENSMODEL_PINHOLE")
    p = np.array(((0., 0., 1.), (0.1, -0.2, 3.)))
    q = np.zeros((2, 2))
    _refused(LIB.mrcal_project(_ptr(q), None, None, _ptr(p), 2, C.byref(lm), _ptr(INTR)))
    v = np.zeros((2, 3))
    _refused(LIB.mrcal_unproject(_ptr(v), _ptr(q), 2, C.byref(lm), _ptr(INTR)))


def test_image_transforms():
    lm = _lensmodel("LENSMODEL_PINHOLE")
    mapxy = np.zeros((3, 4, 2), np.float32)
    _refused(LIB.mrcal_b200_image_transformation_map(_ptr(mapxy), 4, 3, C.byref(lm), _ptr(INTR), C.byref(lm), _ptr(INTR),
                                                     None, None, None, 0., None, 0))
    image = np.arange(12, dtype=np.uint8).reshape(3, 4)
    out = np.zeros((3, 4), np.uint8)
    bv = np.zeros(3)
    _refused(LIB.mrcal_b200_transform_image(out.ctypes.data, image.ctypes.data, 4, 3, image.strides[0], 0, 1,
                                            _ptr(mapxy), 4, 3, 1, 0, _ptr(bv)))
    region = np.array(((0., 0.), (10., 0.), (10., 10.), (0., 10.)))
    mask = np.zeros(2, bool)
    _refused(LIB.mrcal_b200_is_within_region(mask.ctypes.data_as(C.c_void_p), _ptr(np.array(((1., 1.), (20., 1.)))), 2,
                                             _ptr(region), 4))


def test_stereo():
    lm = _lensmodel("LENSMODEL_PINHOLE")
    latlon = _lensmodel("LENSMODEL_LATLON").type
    maps = np.zeros((2, 3, 4, 2), np.float32)
    r = np.zeros(3)
    size = (C.c_uint * 2)(4, 3)
    _refused(LIB.mrcal_rectification_maps(_ptr(maps), C.byref(lm), _ptr(INTR), _ptr(r), C.byref(lm), _ptr(INTR), _ptr(r),
                                          latlon, _ptr(FXYCXY), size, _ptr(r)))
    d = np.array((10., 20.))
    q = np.array(((100., 200.), (300., 100.)))
    ranges = np.zeros(2)
    _refused(LIB.mrcal_stereo_range_sparse(_ptr(ranges), _ptr(d), _ptr(q), 2, 0., 100., latlon, _ptr(FXYCXY), 0.5))
    p = np.zeros((2, 3))
    _refused(LIB.mrcal_b200_stereo_unproject(_ptr(p), None, None, 0, 0, 0, _ptr(d), None, _ptr(q), 2, 0, 0., 100.,
                                             latlon, _ptr(FXYCXY), 0.5))


def test_match_feature():
    image = np.zeros((40, 50), np.uint8)
    # x0, y0 of the template in image 0, then the search cut in image 1: x, y, w, h
    features = np.array(((10, 10, 5, 5, 20, 20),), np.int32)
    Hinv = np.eye(3, dtype=np.float32).reshape(1, 9)
    tw, th = 7, 7
    slot_w, slot_h = 20 - tw + 1, 20 - th + 1
    out = np.zeros(64 + slot_w * slot_h, np.float64)
    _refused(LIB.mrcal_b200_match_feature(out.ctypes.data, None, image.ctypes.data, 50, 40, image.strides[0],
                                          image.ctypes.data, 50, 40, image.strides[0], 0, _ptr(features), _ptr(Hinv), 1,
                                          tw, th, slot_w, slot_h, 5))


def test_projection_diff():
    lm = (_capi.Lensmodel * 2)(_lensmodel("LENSMODEL_PINHOLE"), _lensmodel("LENSMODEL_PINHOLE"))
    intr = np.concatenate((INTR, INTR))
    q0 = np.array(((100., 100.), (500., 400.), (900., 700.), (300., 600.)))
    v = np.tile(np.array(((0., 0., 1.), (0.1, 0., 1.), (0., 0.1, 1.), (-0.1, 0.1, 1.))), (2, 1))
    center = np.array((499.5, 399.5))
    Rt = np.zeros((4, 3))
    _refused(LIB.mrcal_b200_implied_Rt10__from_unprojections(_ptr(Rt), _ptr(q0), 4, _ptr(v[:4].copy()), 1,
                                                             _ptr(v[4:].copy()), None, True, _ptr(center), 1e6))
    difflen = np.zeros(4)
    diff = np.zeros((4, 2))
    _refused(LIB.mrcal_b200_projection_diff(_ptr(Rt), _ptr(difflen), _ptr(diff), _ptr(q0), 4, _ptr(v), 2, None, 1, lm,
                                            _ptr(intr), None, _ptr(center), 1e6, True))
