"""Image reprojection without a GPU: every refusal and its message, the numpy restatement of cv2.remap() on cases
worked by hand (and against OpenCV's fixture, or OpenCV itself, where they are present), and
pinhole_model_for_reprojection()'s host arithmetic."""
import os

import numpy as np
import pytest

import mrcal_b200

import remap_np

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")
FIXTURE = os.path.join(os.path.dirname(__file__), "golden", "transform_image.npz")


def _model(name):
    return mrcal_b200.cameramodel(os.path.join(MODELS, name))


def test_constants_have_opencv_values():
    assert (mrcal_b200.INTER_NEAREST, mrcal_b200.INTER_LINEAR) == (0, 1)
    assert (mrcal_b200.BORDER_CONSTANT, mrcal_b200.BORDER_TRANSPARENT) == (0, 5)


@pytest.mark.parametrize("kw, msg", [
    (dict(plane_n=np.array((0., 0., 1.))), "plane_n and plane_d should both be None or neither should be None"),
    (dict(plane_d=1.), "plane_n and plane_d should both be None or neither should be None"),
    (dict(plane_n=np.array((0., 0., 1.)), plane_d=1., intrinsics_only=True), "so intrinsics_only should be False"),
    (dict(distance=10., intrinsics_only=True), "'distance' makes sense only without plane_n/plane_d"),
    (dict(distance=10., plane_n=np.array((0., 0., 1.)), plane_d=1.), "'distance' makes sense only without"),
    (dict(mask_valid_intrinsics_region_from=True), "model_from has no valid_intrinsics_region"),
])
def test_image_transformation_map_refusals(kw, msg):
    m = _model("cam0.opencv8.cameramodel")
    with pytest.raises(Exception, match=msg):
        mrcal_b200.image_transformation_map(m, m, **kw)


def test_image_transformation_map_refuses_noncentral_cahvore_to():
    m_from = _model("cam0.opencv8.cameramodel")
    m_to = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_CAHVORE_linearity=0.00",
                                              np.array((1000., 1000., 500., 400., 0., 0., 0., 0., 0., 0.1, 0., 0.))),
                                  imagersize=(1000, 800))
    with pytest.raises(Exception, match=r"So I cannot unproject\(CAHVORE,E!=0\)"):
        mrcal_b200.image_transformation_map(m_from, m_to, intrinsics_only=True)


@pytest.mark.parametrize("kw, msg", [
    (dict(interpolation=2), "INTER_NEAREST \\(0\\) and INTER_LINEAR \\(1\\) only"),
    (dict(borderMode=1), "BORDER_CONSTANT \\(0\\) and BORDER_TRANSPARENT \\(5\\) only"),
    (dict(borderValue=(1, 2, 3, 4, 5)), "borderValue must be a number or up to 4 numbers"),
])
def test_transform_image_refuses_options(kw, msg):
    with pytest.raises(Exception, match=msg):
        mrcal_b200.transform_image(np.zeros((4, 4), np.uint8), np.zeros((2, 2, 2), np.float32), **kw)


@pytest.mark.parametrize("image, mapxy, kw, msg", [
    ([[0]], np.zeros((2, 2, 2), np.float32), {}, "'image' must be a numpy array"),
    (np.zeros((4, 4), np.uint8), [[0., 0.]], {}, "'mapxy' must be a numpy array"),
    (np.zeros((4, 4), np.float64), np.zeros((2, 2, 2), np.float32), {}, "uint8, uint16 and float32 images only"),
    (np.zeros((4, 4), np.int16), np.zeros((2, 2, 2), np.float32), {}, "uint8, uint16 and float32 images only"),
    (np.zeros((4, 4, 4), np.uint8), np.zeros((2, 2, 2), np.float32), {}, "shape \\(H,W\\) and \\(H,W,3\\) only"),
    (np.zeros((4, 4), np.uint8), np.zeros((2, 2, 2), np.float64), {}, "mapxy must be a float32 array"),
    (np.zeros((4, 4), np.uint8), np.zeros((2, 2), np.float32), {}, "mapxy must be a float32 array"),
    (np.zeros((4, 4), np.uint8), np.zeros((2, 2, 2), np.float32), dict(out=np.zeros((2, 3), np.uint8)),
     "out must be a numpy array of shape \\(2, 2\\) and dtype uint8"),
    (np.zeros((4, 4), np.uint8), np.zeros((2, 2, 2), np.float32), dict(out=np.zeros((2, 2), np.uint16)),
     "out must be a numpy array of shape"),
    (np.zeros((4, 4), np.uint8), np.zeros((2, 2, 2), np.float32), dict(out=np.zeros((2, 4), np.uint8)[:, ::2]),
     "out must be C-contiguous and writeable"),
])
def test_transform_image_refuses_arrays(image, mapxy, kw, msg):
    with pytest.raises(Exception, match=msg):
        mrcal_b200.transform_image(image, mapxy, **kw)


def test_transform_image_refuses_tensors_mixed_with_arrays():
    torch = pytest.importorskip("torch")
    with pytest.raises(Exception, match="may not be mixed"):
        mrcal_b200.transform_image(torch.zeros((4, 4), dtype=torch.uint8), np.zeros((2, 2, 2), np.float32))
    with pytest.raises(Exception, match="must be CUDA tensors"):
        mrcal_b200.transform_image(torch.zeros((4, 4), dtype=torch.uint8), torch.zeros((2, 2, 2)))


@pytest.mark.parametrize("kw, msg", [
    (dict(fit="everything"), "'fit' must be an array of shape \\(...,2\\) or one of"),
    (dict(fit=np.zeros((3, 3))), "'fit' is an array, so it must have shape \\(...,2\\)"),
    (dict(fit="corners", scale_focal=2.), "At most one of 'scale_focal' and 'fit' may be non-None"),
])
def test_pinhole_model_for_reprojection_refusals(kw, msg):
    with pytest.raises(Exception, match=msg):
        mrcal_b200.pinhole_model_for_reprojection(_model("cam0.opencv8.cameramodel"), **kw)


def test_scale_focal_without_fit_and_with_an_unknown_fit():
    m = _model("cam0.opencv8.cameramodel")
    assert mrcal_b200.scale_focal__best_pinhole_fit(m, None) == 1.0
    with pytest.raises(Exception, match="fit must be either None or a numpy array or one of"):
        mrcal_b200.scale_focal__best_pinhole_fit(m, "middle")
    with pytest.raises(Exception, match="fit must be either None or a numpy array or one of"):
        mrcal_b200.scale_focal__best_pinhole_fit(m, [(0., 0.)])


@pytest.mark.parametrize("scale_image", [None, 0.1, 0.5, 0.25, 1. / 3.])
def test_pinhole_model_for_reprojection_arithmetic(scale_image):
    m = _model("cam0.opencv8.cameramodel")
    lensmodel, intr = m.intrinsics()
    k = 0.731
    p = mrcal_b200.pinhole_model_for_reprojection(m, scale_focal=k, scale_image=scale_image)
    assert p.intrinsics()[0] == "LENSMODEL_PINHOLE"
    np.testing.assert_array_equal(p.rt_cam_ref(), m.rt_cam_ref())
    fxy, cxy = intr[:2] * k, intr[2:4].copy()
    WH = m.imagersize()
    if scale_image is None:
        np.testing.assert_array_equal(p.imagersize(), WH)
        np.testing.assert_array_equal(p.intrinsics()[1], np.r_[fxy, cxy])
        return
    WH1 = np.array([round(int(x) * scale_image) for x in WH])
    np.testing.assert_array_equal(p.imagersize(), WH1)
    f1, c1 = p.intrinsics()[1][:2], p.intrinsics()[1][2:]
    np.testing.assert_allclose(f1, fxy * scale_image, rtol=1e-15)
    # the centre of the original imager, scaled, unprojects to the same pinhole ray
    np.testing.assert_allclose(((WH * scale_image - 1.) / 2. - c1) / f1, ((WH - 1.) / 2. - cxy) / fxy, rtol=1e-12,
                               atol=1e-12)


def test_python_round_is_half_to_even():
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((100., 100., 12., 12.))), imagersize=(25, 15))
    p = mrcal_b200.pinhole_model_for_reprojection(m, scale_focal=1., scale_image=0.5)
    # 25 * 0.5 = 12.5 -> 12; 15 * 0.5 = 7.5 -> 8
    np.testing.assert_array_equal(p.imagersize(), (12, 8))


####################################################################################################
# the remap rule
####################################################################################################
def test_cv_round():
    v = np.array((0.5, 1.5, 2.5, -0.5, -1.5, 2.4999, np.nan, np.inf, -np.inf, 3e9, -3e9, 2147483520.), np.float32)
    np.testing.assert_array_equal(remap_np.cv_round(v),
                                  (0, 2, 2, 0, -2, 2, remap_np.INT_MIN, remap_np.INT_MIN, remap_np.INT_MIN,
                                   remap_np.INT_MIN, remap_np.INT_MIN, 2147483520))


def test_remap_rule_by_hand():
    img = np.array(((10, 20, 30), (40, 50, 60)), np.uint8)
    m = np.array(((
        (0., 0.),                 # a pixel
        (0.5, 0.),                # half-way: (10 + 20) / 2
        (1. / 64, 0.),            # x*32 = 0.5: the tie rounds to even, fraction 0 -> 10
        (3. / 64, 0.),            # x*32 = 1.5 -> 2: 10 + 10 * 2/32 = 10.625 -> 11
        (2., 1.),                 # the last pixel: its right and lower taps are outside, weight 0
        (2.5, 0.),                # half outside: (30 + border 7) / 2 = 18.5 -> 19 under constant
        (np.nan, 0.),             # outside
        (1e9, 0.),                # x*32 beyond int32: INT_MIN, outside
        (-1., -1.),               # the block's lower right tap is pixel (0,0), weight 0: the border value
        (-0.5, 0.),               # half outside on the left: (7 + 10) / 2 = 8.5 -> 9
    ),), np.float32)
    r = remap_np.remap(img, m, border=0, border_value=7, interpolation=1)
    np.testing.assert_array_equal(r, [[10, 15, 10, 11, 60, 19, 7, 7, 7, 9]])
    # transparent: outside (X, Y) leaves out alone; partly outside clamps the taps to the last column
    out = np.full((1, 10), 99, np.uint8)
    r = remap_np.remap(img, m, out=out, border=5, interpolation=1)
    np.testing.assert_array_equal(r, [[10, 15, 10, 11, 60, 30, 99, 99, 99, 99]])
    # nearest: cvRound half to even
    m2 = np.array((((0.5, 0.), (1.5, 0.), (2.5, 0.), (-0.5, 0.), (0.5, 1.5), (np.inf, 0.)),), np.float32)
    r = remap_np.remap(img, m2, border=0, border_value=3, interpolation=0)
    np.testing.assert_array_equal(r, [[10, 30, 30, 10, 3, 3]])


def test_remap_rule_float_and_uint16_sums():
    img = np.array(((1., 2.), (4., 8.)), np.float32)
    m = np.array((((0.25, 0.75),),), np.float32)
    # a = 8/32, b = 24/32: ((1*.1875 + 2*.0625) + 4*.5625) + 8*.1875
    np.testing.assert_array_equal(remap_np.remap(img, m), [[np.float32(4.0625)]])
    img16 = np.array(((1, 2), (4, 9)), np.uint16)
    # 1*.1875 + 2*.0625 + 4*.5625 + 9*.1875 = 4.25 -> 4
    np.testing.assert_array_equal(remap_np.remap(img16, m), [[4]])
    # ties round to even
    m = np.array((((0.5, 0.),),), np.float32)
    np.testing.assert_array_equal(remap_np.remap(np.array(((1, 2), (0, 0)), np.uint16), m), [[2]])   # 1.5 -> 2
    np.testing.assert_array_equal(remap_np.remap(np.array(((2, 3), (0, 0)), np.uint16), m), [[2]])   # 2.5 -> 2


def _fixture_cases():
    f = np.load(FIXTURE)
    keys = sorted({k[:k.rindex("_", 0, len(k) - len("result"))] for k in f.files if k.endswith("_result")})
    return f, keys


def test_remap_rule_against_opencv_fixture():
    f, keys = _fixture_cases()
    for key in keys:
        p = key + "_"
        border = int(key.split("_b")[-1])
        interpolation = int(key.split("_i")[-1].split("_")[0])
        r = remap_np.remap(f[p + "image"], f[p + "mapxy"], out=f[p + "out"], border=border,
                           border_value=f[p + "border_value"], interpolation=interpolation)
        remap_np.assert_matches_opencv(r, f[p + "result"], f[p + "image"], f[p + "mapxy"],
                                       key.startswith("float32") and interpolation == 1 and border == 5)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.float32])
@pytest.mark.parametrize("channels", [1, 3])
@pytest.mark.parametrize("interpolation", [0, 1])
@pytest.mark.parametrize("border", [0, 5])
def test_remap_rule_against_live_opencv(dtype, channels, interpolation, border):
    cv2 = pytest.importorskip("cv2")
    image = remap_np.seeded_image(29, 37, channels, dtype, 1)
    mapxy = remap_np.special_map(41, 47, 29, 37, 2)
    out = remap_np.seeded_image(41, 47, channels, dtype, 3)
    ref = cv2.remap(image, mapxy, None, interpolation=interpolation, borderMode=border, borderValue=5.,
                    dst=out.copy())
    r = remap_np.remap(image, mapxy, out=out, border=border, border_value=5., interpolation=interpolation)
    remap_np.assert_matches_opencv(r, ref, image, mapxy, dtype == np.float32 and interpolation == 1 and border == 5)
