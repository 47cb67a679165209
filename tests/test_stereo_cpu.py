"""CPU: the stereo geometry that needs no device (a positive resolution makes no projection): the refusals of the
rectified system and of the rectified models, stereo_range()'s argument handling, the roots of the pinhole quartic and
the rectified systems against the compiled reference."""
import ctypes as C
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import _capi, stereo
from mrcal_b200._poses_host import Rt_from_rt, compose_Rt, rt_from_Rt

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")


@pytest.fixture(scope="module")
def stereo_oracle():
    """The reference's own stereo.c (oracle/_ref/libmrcal_stereo_ref.so), built by build() where the reference tree is
    readable"""
    from oracle import stereo_ref
    if not stereo_ref.available():
        pytest.skip("oracle/_ref/libmrcal_stereo_ref.so not built (needs the reference tree: make -C oracle -f stereo.mk)")
    return stereo_ref


def _pair(rt01=(0., 0., 0., 3., 0., 0.), name="cam0.opencv8.cameramodel"):
    """camera 1 at rt01 from camera 0 (rt01 maps camera-1 coordinates to camera 0)"""
    m0 = mrcal_b200.cameramodel(os.path.join(MODELS, name))
    m1 = mrcal_b200.cameramodel(m0)
    m1.rt_ref_cam(rt_from_Rt(compose_Rt(m0.Rt_ref_cam(), Rt_from_rt(rt01))))
    return m0, m1


def _rectified(models, **kw):
    kw.setdefault("az_fov_deg", 90.)
    kw.setdefault("el_fov_deg", 50.)
    kw.setdefault("pixels_per_deg_az", 10.)
    kw.setdefault("pixels_per_deg_el", 12.)
    return mrcal_b200.rectified_system(models, **kw)


def _c_system(model0, rt0, rt1, *, fov=(90., 50.), azel0=(0., 0.), margin=10., ppd=(10., 10.), rect=3,
              autodetect=(False, False, False, False)):
    """mrcal_rectified_system2() directly: the autodetection flags the Python layer never sets"""
    lm = mrcal_b200.api._lensmodel(model0.intrinsics()[0])
    intr = np.ascontiguousarray(model0.intrinsics()[1])
    size = (C.c_uint * 2)()
    f, rt = np.zeros(4), np.zeros(6)
    b, az, el = C.c_double(), C.c_double(ppd[0]), C.c_double(ppd[1])
    ok = _capi.lib.mrcal_rectified_system2(size, f.ctypes.data, rt.ctypes.data, C.byref(b), C.byref(az), C.byref(el),
                                           (C.c_double * 2)(*fov), (C.c_double * 2)(*azel0), margin, C.byref(lm),
                                           intr.ctypes.data, np.ascontiguousarray(rt0).ctypes.data,
                                           np.ascontiguousarray(rt1).ctypes.data, rect, *autodetect)
    return ok, _capi.last_error()


def test_refusals_of_the_rectified_system():
    m0, m1 = _pair()
    rt0, rt1 = m0.rt_cam_ref(), m1.rt_cam_ref()
    for i, what in enumerate(("el0_deg", "az_fov_deg", "el_fov_deg")):
        flags = [False] * 4
        flags[i + 1] = True
        ok, err = _c_system(m0, rt0, rt1, autodetect=tuple(flags))
        assert not ok and err == f"{what}_autodetect is not yet supported"
    with pytest.raises(RuntimeError, match="Unsupported rectification model 'LENSMODEL_LONLAT'. Only LENSMODEL_LATLON "
                                           "and LENSMODEL_PINHOLE are supported"):
        _rectified((m0, m1), rectification_model="LENSMODEL_LONLAT")
    with pytest.raises(RuntimeError, match="pixels_per_deg_az == 0 is illegal"):
        _rectified((m0, m1), pixels_per_deg_az=0)
    with pytest.raises(RuntimeError, match="pixels_per_deg_el == 0 is illegal"):
        _rectified((m0, m1), pixels_per_deg_el=0)
    for fov in ((0., 50.), (90., -1.)):
        with pytest.raises(RuntimeError, match="az_fov_deg, el_fov_deg must be > 0"):
            _rectified((m0, m1), az_fov_deg=fov[0], el_fov_deg=fov[1])
    with pytest.raises(RuntimeError, match="unnaturally small baseline"):
        _rectified((m0, mrcal_b200.cameramodel(m0)))
    with pytest.raises(RuntimeError, match="rectified view looks along the baseline vector. Reduce az_fov_deg"):
        _rectified((m0, m1), az0_deg=60.)
    with pytest.raises(RuntimeError, match="cannot avoid looking along the baseline vector: az_fov_deg is too large"):
        _rectified((m0, m1), az_fov_deg=170.)
    with pytest.raises(RuntimeError, match="Resulting stereo geometry has Nel=0"):
        _rectified((m0, m1), el_fov_deg=0.1, pixels_per_deg_el=1.)


def test_central_models_only():
    m0, m1 = _pair()
    intr = np.array((1000., 1000., 499.5, 399.5, 0., 0., 0., 0., 0., 0., 0., 0.))
    cahvore = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_CAHVORE_linearity=0.00", intr), imagersize=(1000, 800),
                                     rt_cam_ref=m1.rt_cam_ref())
    # E = 0: central, accepted
    models = _rectified((m0, cahvore))
    assert models[0].intrinsics()[0] == "LENSMODEL_LATLON"
    intr[-2] = 0.01
    cahvore = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_CAHVORE_linearity=0.00", intr), imagersize=(1000, 800),
                                     rt_cam_ref=m1.rt_cam_ref())
    with pytest.raises(RuntimeError, match="This is CAHVORE, so set E=0 to centralize"):
        _rectified((m0, cahvore))
    # the C entry checks camera 0 itself
    ok, err = _c_system(cahvore, cahvore.rt_cam_ref(), m0.rt_cam_ref())
    assert not ok and "This is CAHVORE, so set E=0 to centralize" in err


def test_validate_models_rectified():
    m0, m1 = _pair()
    r0, r1 = _rectified((m0, m1))
    stereo._validate_models_rectified((r0, r1))
    with pytest.raises(RuntimeError, match="Must have received exactly two models. Got 1 instead"):
        stereo._validate_models_rectified((r0,))
    with pytest.raises(RuntimeError, match="Expected two models with the same"):
        stereo._validate_models_rectified((r0, m1))
    bad = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_LATLON", r1.intrinsics()[1] + 1.), imagersize=r1.imagersize(),
                                 rt_cam_ref=r1.rt_cam_ref())
    with pytest.raises(RuntimeError, match="MUST have the same intrinsics values"):
        stereo._validate_models_rectified((r0, bad))
    bad = mrcal_b200.cameramodel(intrinsics=r1.intrinsics(), imagersize=r1.imagersize() + 1, rt_cam_ref=r1.rt_cam_ref())
    with pytest.raises(RuntimeError, match="MUST have the same imager size"):
        stereo._validate_models_rectified((r0, bad))
    rt = r1.rt_cam_ref()
    rt[:3] += (0.01, 0., 0.)
    bad = mrcal_b200.cameramodel(intrinsics=r1.intrinsics(), imagersize=r1.imagersize(), rt_cam_ref=rt)
    with pytest.raises(RuntimeError, match="MUST have the same relative rotation"):
        stereo._validate_models_rectified((r0, bad))
    rt = r1.rt_cam_ref()
    rt[4] += 0.1
    bad = mrcal_b200.cameramodel(intrinsics=r1.intrinsics(), imagersize=r1.imagersize(), rt_cam_ref=rt)
    with pytest.raises(RuntimeError, match="translation ONLY in the \\+x rectified direction"):
        stereo._validate_models_rectified((r0, bad))


def test_stereo_range_argument_errors():
    m0, m1 = _pair()
    rect = _rectified((m0, m1))
    W, H = rect[0].imagersize()
    d = np.ones((H, W))
    with pytest.raises(RuntimeError, match="disparity_min and disparity_scaled_min may not both be given"):
        mrcal_b200.stereo_range(d, rect, disparity_min=1, disparity_scaled_min=2)
    with pytest.raises(RuntimeError, match="disparity_max and disparity_scaled_max may not both be given"):
        mrcal_b200.stereo_range(d, rect, disparity_max=1, disparity_scaled_max=2)
    with pytest.raises(RuntimeError, match="qrect0 is None, so the given disparity and full rectified images MUST"):
        mrcal_b200.stereo_range(np.ones((H, W + 1)), rect)
    with pytest.raises(RuntimeError, match="Exactly one of \\(disparity,ranges\\) must be non-None"):
        mrcal_b200.stereo_unproject(None, rect)
    with pytest.raises(RuntimeError, match="Exactly one of \\(disparity,ranges\\) must be non-None"):
        mrcal_b200.stereo_unproject(d, rect, ranges=d)
    with pytest.raises(RuntimeError, match="Must have received exactly two models"):
        mrcal_b200.stereo_range(d, rect[:1])


def test_int16_disparities_become_uint16():
    """int16 with no upper bound: scaled_max = 0x7FFF and the array is cast to uint16, so -1 is 65535: invalid"""
    m0, m1 = _pair()
    rect = _rectified((m0, m1))
    W, H = rect[0].imagersize()
    d = np.full((H, W), 100, np.int16)
    d[0, 0] = -1
    a = stereo._range_arguments(d, rect, 16, None, None, None, None, None)
    assert a["scaled_max"] == 0x7FFF and a["scaled_min"] == 0
    img, d16, (scale, smin, smax) = stereo._dense_image(a, rect, 16)
    assert d16.dtype == np.uint16 and d16[0, 0] == 65535 and d16[0, 1] == 100
    assert (scale, smin, smax) == (16, 0, 0x7FFF) and img.stride == 2 * W
    # given a max, or not int16: the uint16 range
    a = stereo._range_arguments(d.astype(np.float64), rect, 16, None, None, None, None, None)
    assert a["scaled_max"] == 65535
    a = stereo._range_arguments(d, rect, 16, None, None, 10., None, None)
    assert a["scaled_max"] == 160.
    # with qrect0, the bounds are in pixels
    a = stereo._range_arguments(np.array((-1,), np.int16), rect, 16, None, None, None, None, np.zeros(2))
    assert a["dmax"] == 0x7FFF / 16 and a["dmin"] == 0 and not a["is_scalar"]
    # a numpy scalar is not an array: no int16 rule, as in the reference
    a = stereo._range_arguments(np.int16(-1), rect, 16, None, None, None, None, np.zeros(2))
    assert a["dmax"] == np.finfo(float).max and a["is_scalar"]


def _np_pinhole_c(tanazel0, fov_deg, fxy):
    """stereo.c:299-385 over numpy's roots: the chosen C = c/f"""
    cosfov = np.cos(fov_deg * np.pi / 180.)
    c2 = cosfov * cosfov
    K = 2. * tanazel0
    poly = (1., 2. * K, K * K + 2 + 4. / (c2 - 1), 2. * K + K * 4. / (c2 - 1), K * K + 1. + K * K / (c2 - 1))
    r = np.roots(poly)
    C = [x.real for x in r if abs(x.imag) <= 1e-7]
    C = [c for c in C if cosfov * (1. - K * c - c * c) >= -1e-9]
    C = [c for c in C if (tanazel0 * fxy + c * fxy) * 2. + 1. > 0]
    return max(C, key=lambda c: cosfov * (1. - K * c - c * c))


def test_pinhole_quartic_roots(stereo_oracle):
    """cy of a rectified pinhole is the chosen root of the quartic times fy: a sweep of el0 (tan in [-1, 1]) and
    el_fov against numpy's roots, then the whole system against the reference's (its dgeev is LAPACK's)"""
    m0, m1 = _pair()
    for tan_el0 in np.linspace(-1., 1., 9):
        for fov in np.linspace(20., 170., 13):
            el0 = np.arctan(tan_el0) * 180. / np.pi
            r0, _ = _rectified((m0, m1), az_fov_deg=80., el0_deg=el0, el_fov_deg=fov,
                               rectification_model="LENSMODEL_PINHOLE")
            fx, fy, cx, cy = r0.intrinsics()[1]
            assert abs(cy / fy - _np_pinhole_c(tan_el0, fov, fy)) <= 1e-10, (tan_el0, fov)
            o = stereo_oracle.rectified_system2(m0.intrinsics()[0], m0.intrinsics()[1], m0.rt_cam_ref(), m1.rt_cam_ref(),
                                                az_fov_deg=80., el_fov_deg=fov, el0_deg=el0, pixels_per_deg_az=10.,
                                                pixels_per_deg_el=12., rectification_model="LENSMODEL_PINHOLE")
            assert np.abs(r0.intrinsics()[1] - o["fxycxy"]).max() <= 1e-12 * np.abs(o["fxycxy"]).max(), (tan_el0, fov)
            assert tuple(r0.imagersize()) == o["imagersize"]


@pytest.mark.parametrize("rect", ("LENSMODEL_LATLON", "LENSMODEL_PINHOLE"))
@pytest.mark.parametrize("geometry", ("vanilla", "complex", "margin40"))
def test_rectified_system_against_reference(stereo_oracle, rect, geometry):
    rt01 = (0., 0., 0., 3., 0., 0.) if geometry == "vanilla" else (0.1, 0.2, 0.05, 3.0, 0.2, 1.0)
    m0, m1 = _pair(rt01)
    kw = dict(az_fov_deg=90., el_fov_deg=50., el0_deg=0. if geometry == "vanilla" else 10., pixels_per_deg_az=8.3,
              pixels_per_deg_el=4.1, az_edge_margin_deg=40. if geometry == "margin40" else 10.)
    (r0, r1), meta = mrcal_b200.rectified_system((m0, m1), rectification_model=rect, return_metadata=True, **kw)
    o = stereo_oracle.rectified_system2(m0.intrinsics()[0], m0.intrinsics()[1], m0.rt_cam_ref(), m1.rt_cam_ref(),
                                        rectification_model=rect, **kw)
    assert tuple(r0.imagersize()) == o["imagersize"] == tuple(r1.imagersize())
    fxycxy = r0.intrinsics()[1]
    if rect == "LENSMODEL_PINHOLE":
        # az_fov = 90 deg: cos(fov) = 0 makes the quartic for cx a perfect square, (1 - K C - C^2)^2 = 0, so its roots
        # are double and any eigenvalue solver (LAPACK's included) resolves them only to ~sqrt(eps). Compare cx with
        # that accuracy, and with the closed-form root
        K = 2. * np.tan(meta["az0_deg"] * np.pi / 180.)
        C_exact = (-K + np.sqrt(K * K + 4.)) / 2.
        for cx in (fxycxy[2], o["fxycxy"][2]):
            assert abs(cx - C_exact * fxycxy[0]) <= 1e-7 * fxycxy[0]
        fxycxy = np.array(fxycxy)
        fxycxy[2] = o["fxycxy"][2]
    for a, b in ((fxycxy, o["fxycxy"]), (r0.rt_cam_ref(), o["rt_rect0_ref"]),
                 (meta["baseline"], o["baseline"])):
        assert np.abs(np.asarray(a) - b).max() <= 1e-12 * max(1., np.abs(b).max()), (a, b)
    for k in ("az0_deg", "el0_deg", "az_fov_deg", "el_fov_deg", "pixels_per_deg_az", "pixels_per_deg_el"):
        assert abs(meta[k] - o[k]) <= 1e-12 * max(1., abs(o[k])), k
    rt1 = o["rt_rect0_ref"].copy()
    rt1[3] -= o["baseline"]
    assert np.abs(r1.rt_cam_ref() - rt1).max() <= 1e-12 * max(1., np.abs(rt1).max())
    stereo._validate_models_rectified((r0, r1))
