"""Stereo on the device: the reference's own tests (test-stereo.py, test-rectification-maps.py) with their thresholds,
the maps and the ranges against the compiled reference's C functions, stereo_unproject() against numpy, and
determinism."""
import ctypes as C
import os

import numpy as np
import pytest
import scipy.interpolate

import mrcal_b200
from mrcal_b200 import _capi, stereo
from mrcal_b200._poses_host import R_from_r, Rt_from_rt, compose_Rt, invert_Rt, rt_from_Rt, transform_point_Rt

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")
RECTS = ("LENSMODEL_LATLON", "LENSMODEL_PINHOLE")


@pytest.fixture(scope="module")
def stereo_oracle():
    """The reference's own stereo.c (oracle/_ref/libmrcal_stereo_ref.so), built by build() where the reference tree is
    readable"""
    from oracle import stereo_ref
    if not stereo_ref.available():
        pytest.skip("oracle/_ref/libmrcal_stereo_ref.so not built (needs the reference tree: make -C oracle -f stereo.mk)")
    return stereo_ref


def _model(name):
    return mrcal_b200.cameramodel(os.path.join(MODELS, name))


def _place(m0, m1, rt01):
    """camera 1 at rt01 from camera 0 (rt01 maps camera-1 coordinates to camera-0 coordinates)"""
    m1.rt_ref_cam(rt_from_Rt(compose_Rt(m0.Rt_ref_cam(), Rt_from_rt(np.asarray(rt01, float)))))


def _unit(v):
    return v / np.linalg.norm(v, axis=-1)[..., None]


def _unproject_rect(q, rect, fxycxy):
    """the closed-form unprojection of the rectified models, in numpy"""
    fx, fy, cx, cy = fxycxy
    a, b = (q[..., 0] - cx) / fx, (q[..., 1] - cy) / fy
    if rect == "LENSMODEL_LATLON":
        return np.stack((np.sin(a), np.cos(a) * np.sin(b), np.cos(a) * np.cos(b)), axis=-1)
    return np.stack((a, b, np.ones_like(a)), axis=-1)


def _angle_deg(v0, v1):
    return np.arccos(np.dot(v0, v1) / (np.linalg.norm(v0) * np.linalg.norm(v1))) * 180. / np.pi


def _check_against_reference(models, models_rectified, meta, stereo_oracle, rect, **kw):
    o = stereo_oracle.rectified_system2(models[0].intrinsics()[0], models[0].intrinsics()[1], models[0].rt_cam_ref(),
                                        models[1].rt_cam_ref(), rectification_model=rect, **kw)
    assert tuple(models_rectified[0].imagersize()) == o["imagersize"]
    # the reference's own threshold for its C-vs-Python comparison (test-stereo.py:74-90)
    assert np.abs(models_rectified[0].intrinsics()[1] - o["fxycxy"]).max() <= 1e-5
    assert np.abs(models_rectified[0].rt_cam_ref() - o["rt_rect0_ref"]).max() <= 1e-5
    assert abs(meta["baseline"] - o["baseline"]) <= 1e-12 * o["baseline"]


# 1. test/test-stereo.py of the reference, with its thresholds
@pytest.mark.parametrize("rect", RECTS)
def test_reference_stereo(stereo_oracle, rect):
    model0 = _model("cam0.opencv8.cameramodel")
    model1 = mrcal_b200.cameramodel(model0)
    az_fov_deg, el_fov_deg = 90, 50
    kw = dict(az_fov_deg=az_fov_deg, el_fov_deg=el_fov_deg, pixels_per_deg_az=-1. / 8., pixels_per_deg_el=-1. / 4.)
    for geometry in ("vanilla", "complex"):
        rt01 = np.array((0, 0, 0, 3.0, 0, 0)) if geometry == "vanilla" else np.array((0.1, 0.2, 0.05, 3.0, 0.2, 1.0))
        _place(model0, model1, rt01)
        el0_deg = 0. if geometry == "vanilla" else 10.
        models_rectified, meta = mrcal_b200.rectified_system((model0, model1), el0_deg=el0_deg, rectification_model=rect,
                                                             return_metadata=True, **kw)
        _check_against_reference((model0, model1), models_rectified, meta, stereo_oracle, rect, el0_deg=el0_deg, **kw)
        stereo._validate_models_rectified(models_rectified)
        assert models_rectified[0].intrinsics()[0] == rect and models_rectified[1].intrinsics()[0] == rect
        Rt_cam0_rect = compose_Rt(model0.Rt_cam_ref(), models_rectified[0].Rt_ref_cam())
        Rt01_rectified = compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())
        if geometry == "vanilla":
            az0, el0 = 0., 0.
            assert np.abs(Rt_cam0_rect - np.vstack((np.eye(3), np.zeros(3)))).max() < 1e-6
        else:
            el0 = el0_deg * np.pi / 180.
            baseline = rt01[3:] / np.linalg.norm(rt01[3:])
            forward01 = np.array((0, 0, 1.)) + R_from_r(rt01[:3]) @ np.array((0, 0, 1.))
            az0 = np.arcsin(np.dot(forward01, baseline) / np.linalg.norm(forward01))
            # the geometry the reference pins (test-stereo.py:297-302)
            assert np.abs(Rt_cam0_rect - np.array([[0.9467916, -0.08500675, -0.31041828],
                                                   [0.06311944, 0.99480206, -0.07990489],
                                                   [0.3155972, 0.05605985, 0.94723582],
                                                   [0., -0., -0.]])).max() < 1e-6
        assert abs(Rt01_rectified[3, 0] - np.linalg.norm(rt01[3:])) < 1e-6

        lm_r, intr_r = models_rectified[0].intrinsics()
        Naz, Nel = models_rectified[0].imagersize()
        q0 = np.array(((Naz - 1.) / 2., (Nel - 1.) / 2.))
        v0 = _unit(mrcal_b200.unproject(q0, lm_r, intr_r))
        if rect == "LENSMODEL_LATLON":
            v0_rect = np.array((np.sin(az0), np.cos(az0) * np.sin(el0), np.cos(az0) * np.cos(el0)))
            assert np.abs(v0_rect - v0).max() < 1e-6
        else:
            v0_rect = _unit(np.array((np.tan(az0), np.tan(el0), 1.)))
            assert np.abs(v0_rect - v0).max() < 1e-3

        # pixel density: 1/8 and 1/4 of camera 0's
        dq0x, dq0y = np.array((1e-1, 0)), np.array((0, 1e-1))
        v0x = mrcal_b200.unproject(q0 + dq0x, lm_r, intr_r)
        v0y = mrcal_b200.unproject(q0 + dq0y, lm_r, intr_r)
        dthx = _angle_deg(v0x, v0) * np.pi / 180.
        dthy = _angle_deg(v0y, v0) * np.pi / 180.
        q_cam0 = lambda v: mrcal_b200.project(Rt_cam0_rect[:3] @ v, *model0.intrinsics())
        ppr_az_cam0 = np.linalg.norm(q_cam0(v0x) - q_cam0(v0)) / dthx
        ppr_el_cam0 = np.linalg.norm(q_cam0(v0y) - q_cam0(v0)) / dthy
        assert abs(np.linalg.norm(dq0x) / dthx * 8. - ppr_az_cam0) <= 1e-2 * abs(ppr_az_cam0)
        assert abs(np.linalg.norm(dq0y) / dthy * 4. - ppr_el_cam0) <= 1e-2 * abs(ppr_el_cam0)

        # the fields of view
        v0 = mrcal_b200.unproject(np.array((0, (Nel - 1.) / 2.)), lm_r, intr_r)
        v1 = mrcal_b200.unproject(np.array((Naz - 1, (Nel - 1.) / 2.)), lm_r, intr_r)
        assert abs(_angle_deg(v0, v1) - az_fov_deg) <= (0.5 if geometry == "vanilla" else 1.)
        v0 = mrcal_b200.unproject(np.array(((Naz - 1.) / 2., 0)), lm_r, intr_r)
        v1 = mrcal_b200.unproject(np.array(((Naz - 1.) / 2., Nel - 1)), lm_r, intr_r)
        v0[0] = v1[0] = 0   # el_fov applies at the stereo center only
        assert abs(_angle_deg(v0, v1) - el_fov_deg) <= 0.5
    # the rest on the complex geometry, as the reference: points seen by both cameras
    pcam0 = np.array(((1., 2., 12.), (-4., 3., 12.)))
    qcam0 = mrcal_b200.project(pcam0, *model0.intrinsics())
    pcam1 = transform_point_Rt(invert_Rt(Rt_from_rt(rt01)), pcam0)
    qcam1 = mrcal_b200.project(pcam1, *model1.intrinsics())
    prect0 = transform_point_Rt(invert_Rt(Rt_cam0_rect), pcam0)
    prect1 = prect0 - Rt01_rectified[3, :]
    qrect0 = mrcal_b200.project(prect0, *models_rectified[0].intrinsics())
    qrect1 = mrcal_b200.project(prect1, *models_rectified[1].intrinsics())

    maps = mrcal_b200.rectification_maps((model0, model1), models_rectified)
    assert maps.shape == (2, Nel, Naz, 2) and maps.dtype == np.float32
    row, col = np.arange(Naz, dtype=float), np.arange(Nel, dtype=float)
    for m, qrect, qcam in ((maps[0], qrect0, qcam0), (maps[1], qrect1, qcam1)):
        ix = scipy.interpolate.RectBivariateSpline(row, col, m[..., 0].T)
        iy = scipy.interpolate.RectBivariateSpline(row, col, m[..., 1].T)
        q_from_map = np.stack((ix(*qrect.T, grid=False), iy(*qrect.T, grid=False)), axis=-1)
        assert np.abs(q_from_map - qcam).max() <= 1e-1
    assert np.abs(qrect0[:, 1] - qrect1[:, 1]).max() < 1e-6   # same point, same elevation

    disparity = qrect0[:, 0] - qrect1[:, 0]
    r = mrcal_b200.stereo_range(disparity, models_rectified, qrect0=qrect0)
    assert np.abs(r - np.linalg.norm(pcam0, axis=-1)).max() < 1e-6
    r = mrcal_b200.stereo_range(disparity[:1], models_rectified, qrect0=qrect0[0])
    assert r.shape == (1,) and abs(r[0] - np.linalg.norm(pcam0[0])) <= 2e-6
    r = mrcal_b200.stereo_range(float(disparity[0]), models_rectified, qrect0=qrect0[0])
    assert np.ndim(r) == 0 and abs(r - np.linalg.norm(pcam0[0])) <= 2e-6
    r = mrcal_b200.stereo_range(np.int16(-1), models_rectified, qrect0=qrect0[0], disparity_min=0)
    assert r == 0

    # dense: made-up disparities give reasonable ranges; the invalid pixel gives 0
    disparity_scale = 16
    range_mean = np.mean(np.linalg.norm(pcam0, axis=-1))
    disparity_dense = np.int16(disparity_scale * np.mean(disparity)) * np.ones((Nel, Naz), dtype=np.int16)
    disparity_dense[0, 0] = -1
    mask_valid = disparity_dense > 0
    r = mrcal_b200.stereo_range(disparity_dense, models_rectified, disparity_scale=disparity_scale, disparity_min=0)
    assert np.all(r[mask_valid] > range_mean / 2) and np.all(r[mask_valid] < range_mean * 2.)
    assert r[0, 0] == 0

    p = mrcal_b200.stereo_unproject(disparity, models_rectified, qrect0=qrect0)
    assert np.abs(p - prect0).max() < 1e-6
    p = mrcal_b200.stereo_unproject(float(disparity[0]), models_rectified, qrect0=qrect0[0])
    assert p.shape == (3,) and np.abs(p - prect0[0]).max() < 1e-6
    p = mrcal_b200.stereo_unproject(disparity[:1], models_rectified, qrect0=qrect0[:1])
    assert p.shape == (1, 3) and np.abs(p - prect0[:1]).max() < 1e-6

    # a larger margin, against the reference (test-stereo.py:512-549)
    kw40 = dict(kw, el0_deg=el0_deg, az_edge_margin_deg=40.)
    models_rectified, meta = mrcal_b200.rectified_system((model0, model1), rectification_model=rect,
                                                         return_metadata=True, **kw40)
    _check_against_reference((model0, model1), models_rectified, meta, stereo_oracle, rect, **kw40)


# 2. test/test-rectification-maps.py of the reference: the maps against its mrcal_rectification_maps()
def _maps_case(stereo_oracle, models, rect, zoom=1., az_fov_deg=90., el_fov_deg=50.):
    """The rectified system of the models zoomed in by `zoom` (from the reference, so that only the maps are under
    test), then both maps of the unzoomed models"""
    zoomed = []
    for m in models:
        lm, intr = m.intrinsics()
        intr = intr.copy()
        intr[:2] *= zoom
        zoomed.append((lm, intr))
    o = stereo_oracle.rectified_system2(zoomed[0][0], zoomed[0][1], models[0].rt_cam_ref(), models[1].rt_cam_ref(),
                                        az_fov_deg=az_fov_deg / zoom, el_fov_deg=el_fov_deg / zoom, pixels_per_deg_az=-1. / 8.,
                                        pixels_per_deg_el=-1. / 4., rectification_model=rect)
    rt1 = o["rt_rect0_ref"].copy()
    rt1[3] -= o["baseline"]
    models_rectified = [mrcal_b200.cameramodel(intrinsics=(rect, o["fxycxy"]), imagersize=o["imagersize"], rt_cam_ref=rt)
                        for rt in (o["rt_rect0_ref"], rt1)]
    maps = mrcal_b200.rectification_maps(models, models_rectified)
    maps_ref = stereo_oracle.rectification_maps(*models[0].intrinsics(), models[0].rt_cam_ref()[:3],
                                                *models[1].intrinsics(), models[1].rt_cam_ref()[:3],
                                                rect, o["fxycxy"], o["imagersize"], o["rt_rect0_ref"][:3])
    # some pinhole maps are wild far out of view; the reference ignores those (test-rectification-maps.py:69-72)
    maps[maps > 1e6] = 0
    maps_ref[maps_ref > 1e6] = 0
    # every entry within one float32 ulp of the reference's (the two round different doubles), or 1e-6
    tol = np.maximum(np.spacing(np.abs(maps_ref)), 1e-6)
    err = np.abs(maps.astype(np.float64) - maps_ref.astype(np.float64))
    assert np.all(err <= tol), (np.max(err / tol), maps.shape)
    return maps, models_rectified


def _reference_pair():
    """cam0.opencv8 and the reference's tweak of it, at the reference's rt01 (test-rectification-maps.py:19-33)"""
    model0 = _model("cam0.opencv8.cameramodel")
    lm, intr = model0.intrinsics()
    intr[:2] *= np.array((1.01, -0.98))
    intr[2:4] += np.array((50, 80.))
    model1 = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=model0.imagersize(),
                                    rt_cam_ref=model0.rt_cam_ref())
    _place(model0, model1, (0.1, 0.2, 0.05, 3.0, 0.2, 1.0))
    return model0, model1


@pytest.mark.parametrize("rect", RECTS)
@pytest.mark.parametrize("zoom", (0.6, 1., 10.))
def test_rectification_maps_opencv8(stereo_oracle, rect, zoom):
    _maps_case(stereo_oracle, _reference_pair(), rect, zoom)


@pytest.mark.parametrize("rect", RECTS)
def test_rectification_maps_splined(stereo_oracle, rect):
    model0, model1 = _model("cam0.splined.cameramodel"), _model("cam1.splined.cameramodel")
    _place(model0, model1, (0.1, 0.2, 0.05, 3.0, 0.2, 1.0))
    _maps_case(stereo_oracle, (model0, model1), rect)


@pytest.mark.parametrize("lens", ("cahvore", "stereographic"))
def test_rectification_maps_other_lenses(stereo_oracle, lens):
    if lens == "cahvore":
        intr = np.array((1000., 1000., 499.5, 399.5, 0.01, -0.02, 0., 0.01, -0.001, 0., 0., 0.))
        lm = "LENSMODEL_CAHVORE_linearity=0.00"
    else:
        intr, lm = np.array((700., 710., 499.5, 399.5)), "LENSMODEL_STEREOGRAPHIC"
    model0 = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=(1000, 800))
    model1 = mrcal_b200.cameramodel(model0)
    _place(model0, model1, (0.01, 0.02, 0.005, 1.0, 0.05, 0.1))
    for rect in RECTS:
        _maps_case(stereo_oracle, (model0, model1), rect, az_fov_deg=60., el_fov_deg=40.)


def _rectified_pair(rect):
    model0, model1 = _reference_pair()
    return mrcal_b200.rectified_system((model0, model1), az_fov_deg=90., el_fov_deg=50., pixels_per_deg_az=-1. / 8.,
                                       pixels_per_deg_el=-1. / 4., rectification_model=rect)


def _disparity_image(rng, H, W, pad):
    """uint16 with zeros, values beyond the maximum and values in range, as a view into rows `pad` elements wider"""
    big = rng.integers(1, 3000, size=(H, W + pad)).astype(np.uint16)
    d = big[:, :W]
    d[rng.random((H, W)) < 0.1] = 0
    d[rng.random((H, W)) < 0.05] = 60000
    return d


def _baseline(models_rectified):
    return float(np.linalg.norm(compose_Rt(models_rectified[0].Rt_cam_ref(), models_rectified[1].Rt_ref_cam())[3]))


# 3. the ranges against the reference's C functions
@pytest.mark.parametrize("rect", RECTS)
def test_stereo_range_against_reference(stereo_oracle, rect):
    rng = np.random.default_rng(5)
    models_rectified = _rectified_pair(rect)
    W, H = (int(x) for x in models_rectified[0].imagersize())
    fxycxy = models_rectified[0].intrinsics()[1]
    baseline = _baseline(models_rectified)
    d = _disparity_image(rng, H, W, pad=3)
    assert d.strides[0] == 2 * (W + 3)
    scale, smin, smax = 16, 20, 50000
    r_ref = stereo_oracle.stereo_range_dense(d, scale, smin, smax, rect, fxycxy, baseline)

    # the C entry on the strided image, into a strided range image
    lm = mrcal_b200.api._lensmodel(rect).type
    r_big = np.full((H, W + 5), -7.)
    img = _capi.ImageUint16(W, H, d.strides[0], d.ctypes.data)
    out = _capi.ImageDouble(W, H, r_big.strides[0], r_big.ctypes.data)
    assert _capi.lib.mrcal_stereo_range_dense(C.byref(out), C.byref(img), scale, smin, smax, lm, fxycxy.ctypes.data,
                                              baseline), _capi.last_error()
    assert np.all(r_big[:, W:] == -7.)
    for r in (r_big[:, :W], mrcal_b200.stereo_range(d, models_rectified, disparity_scale=scale,
                                                    disparity_scaled_min=smin, disparity_scaled_max=smax)):
        assert np.array_equal(r == 0, r_ref == 0)
        assert np.count_nonzero(r) > H * W // 2
        nz = r_ref != 0
        assert np.all(np.abs(r[nz] - r_ref[nz]) <= 1e-12 * np.abs(r_ref[nz]))

    # sparse: pixels anywhere, disparities in pixels with invalid ones mixed in
    N = 5000
    q = np.stack((rng.uniform(0, W - 1, N), rng.uniform(0, H - 1, N)), axis=-1)
    disp = rng.uniform(-1., 200., N)
    disp[::17] = 0.
    dmin, dmax = 0.5, 150.
    r_ref = stereo_oracle.stereo_range_sparse(disp, q, dmin, dmax, rect, fxycxy, baseline)
    r = mrcal_b200.stereo_range(disp, models_rectified, qrect0=q, disparity_min=dmin, disparity_max=dmax)
    assert np.array_equal(r == 0, r_ref == 0) and np.count_nonzero(r) > N // 2
    nz = r_ref != 0
    assert np.all(np.abs(r[nz] - r_ref[nz]) <= 1e-12 * np.abs(r_ref[nz]))


# 4. stereo_unproject against numpy
@pytest.mark.parametrize("rect", RECTS)
def test_stereo_unproject_against_numpy(rect):
    rng = np.random.default_rng(7)
    models_rectified = _rectified_pair(rect)
    W, H = (int(x) for x in models_rectified[0].imagersize())
    fxycxy = models_rectified[0].intrinsics()[1]
    d = np.ascontiguousarray(_disparity_image(rng, H, W, pad=0))
    r = mrcal_b200.stereo_range(d, models_rectified, disparity_scale=16)
    p = mrcal_b200.stereo_unproject(d, models_rectified, disparity_scale=16)
    qgrid = np.stack(np.meshgrid(np.arange(W, dtype=float), np.arange(H, dtype=float)), axis=-1)
    p_np = _unit(_unproject_rect(qgrid, rect, fxycxy)) * r[..., None]
    assert p.shape == (H, W, 3)
    assert np.all(p[r == 0] == 0)
    assert np.abs(p - p_np).max() <= 1e-12 * max(1., np.abs(p_np).max())
    # from given ranges, on the grid and at given pixels
    p2 = mrcal_b200.stereo_unproject(None, models_rectified, ranges=r)
    assert np.abs(p2 - p_np).max() <= 1e-12 * max(1., np.abs(p_np).max())
    q = np.stack((rng.uniform(0, W - 1, 1000), rng.uniform(0, H - 1, 1000)), axis=-1)
    disp = rng.uniform(0.5, 100., 1000)
    rs = mrcal_b200.stereo_range(disp, models_rectified, qrect0=q)
    ps = mrcal_b200.stereo_unproject(disp, models_rectified, qrect0=q)
    ps_np = _unit(_unproject_rect(q, rect, fxycxy)) * rs[..., None]
    assert np.abs(ps - ps_np).max() <= 1e-12 * max(1., np.abs(ps_np).max())
    ps2 = mrcal_b200.stereo_unproject(None, models_rectified, ranges=rs, qrect0=q)
    assert np.abs(ps2 - ps_np).max() <= 1e-12 * max(1., np.abs(ps_np).max())


# 5. determinism
def test_two_calls_are_bit_identical():
    models = _reference_pair()
    models_rectified = mrcal_b200.rectified_system(models, az_fov_deg=90., el_fov_deg=50., pixels_per_deg_az=-1. / 8.,
                                                   pixels_per_deg_el=-1. / 4.)
    a, b = (mrcal_b200.rectification_maps(models, models_rectified) for _ in range(2))
    assert np.array_equal(a, b)
    W, H = (int(x) for x in models_rectified[0].imagersize())
    d = np.ascontiguousarray(_disparity_image(np.random.default_rng(3), H, W, pad=0))
    a, b = (mrcal_b200.stereo_range(d, models_rectified, disparity_scale=16) for _ in range(2))
    assert np.array_equal(a, b)
    a, b = (mrcal_b200.stereo_unproject(d, models_rectified, disparity_scale=16) for _ in range(2))
    assert np.array_equal(a, b)
