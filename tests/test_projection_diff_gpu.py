"""projection_diff() and implied_Rt10__from_unprojections() on the device: the reference's own test (its thresholds,
its models), the fit against the reference's scipy fit restated in numpy (diff_np), recovery of a known transform, the
reprojection against numpy, uncertainty weighting, determinism and the noncentral rules."""
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import synthetic
import diff_np

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")


def _model(name):
    return mrcal_b200.cameramodel(os.path.join(MODELS, name))


def _rotation_deg(Rt):
    return np.arccos(min(1., (np.trace(Rt[:3]) - 1) / 2.)) * 180. / np.pi


def _transform(Rt, p):
    return p @ Rt[:3].T + Rt[3]


def _check_cost(Rt_dev, Rt_ref, *args, **kwargs):
    """the device's fit is at least as good as scipy's, by the objective itself"""
    c_dev = diff_np.robust_cost(Rt_dev, *args, **kwargs)
    c_ref = diff_np.robust_cost(Rt_ref, *args, **kwargs)
    floor = diff_np.cost_floor(Rt_ref, *args, **kwargs)
    assert c_dev <= c_ref * (1 + 1e-6) + floor, (c_dev, c_ref, floor)


# 1. test/test-projection-diff.py of the reference, with its thresholds
def test_reference_projection_diff():
    opencv8, splined = _model("cam0.opencv8.cameramodel"), _model("cam0.splined.cameramodel")
    gridn_width = 50
    for distance in (None, 3.):
        difflen, diff, q0, Rt = mrcal_b200.projection_diff((splined, splined), gridn_width=gridn_width,
                                                           distance=distance, use_uncertainties=False)
        assert difflen.shape == (int(round(2200 / 4000 * gridn_width)), gridn_width) == q0.shape[:2]
        assert diff.shape == q0.shape
        assert np.nanmax(np.abs(difflen)) <= 0.08
        assert _rotation_deg(Rt) <= 0.01
        assert np.linalg.norm(Rt[3]) <= 0.01
        if distance is None:
            assert np.array_equal(Rt, np.vstack((np.eye(3), np.zeros(3))))   # a zero gradient: the exact identity

    icenter = np.array(difflen.shape) // 2
    for r in (800, 366):
        difflen, *_ = mrcal_b200.projection_diff((opencv8, splined), gridn_width=gridn_width, distance=5,
                                                 use_uncertainties=False, focus_radius=r)
        assert difflen[icenter[0], icenter[1]] <= 0.1

    lm, intr = opencv8.intrinsics()
    intr[0] *= 1.0001
    intr[1] *= 1.0002
    shifted = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=opencv8.imagersize())
    difflen, *_ = mrcal_b200.projection_diff((opencv8, shifted), gridn_width=gridn_width, distance=50000,
                                             use_uncertainties=False, focus_radius=1500)
    assert difflen[icenter[0], icenter[1]] <= 2e-2
    assert np.mean(difflen) <= 0.2


def _unprojections(gridn=30):
    opencv8, splined = _model("cam0.opencv8.cameramodel"), _model("cam0.splined.cameramodel")
    v, q0 = mrcal_b200.sample_imager_unproject(gridn, None, 4000, 2200, [opencv8.intrinsics()[0], splined.intrinsics()[0]],
                                               [opencv8.intrinsics()[1], splined.intrinsics()[1]], normalize=True)
    return q0, v[0], v[1]


# 2. the fit against the reference's scipy fit, fed the same unprojections
@pytest.mark.parametrize("atinfinity", [True, False])
@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("salted", [False, True])
def test_fit_against_scipy(atinfinity, weighted, salted):
    q0, v0, v1 = _unprojections()
    rng = np.random.default_rng(3)
    dist = np.array((1.,)) if atinfinity else np.array((2., 5., 20.))
    p0 = v0[None] * dist[:, None, None, None]
    w = rng.uniform(0.3, 3., size=p0.shape[:-1]) if weighted else None
    if salted:
        p0 = p0.copy()
        v1 = v1.copy()
        p0[0, 3, 4] = np.nan
        v1[5, 6] = np.nan
        v1[6, 7, 1] = np.inf
        if w is not None:
            w[-1, 8, 9] = np.inf
            w[0, 9, 10] = np.nan
    kw = dict(weights=w, atinfinity=atinfinity, focus_center=(1999.5, 1099.5), focus_radius=1200.)
    Rt_dev = mrcal_b200.implied_Rt10__from_unprojections(q0, p0, v1, **kw)
    Rt_ref = diff_np.fit(q0, p0, v1, **kw)
    assert Rt_dev.shape == (4, 3)
    if atinfinity:
        assert not Rt_dev[3].any()
    _check_cost(Rt_dev, Rt_ref, q0, p0, v1, **kw)


def test_fit_refuses_an_empty_focus_region():
    q0, v0, v1 = _unprojections(10)
    with pytest.raises(RuntimeError, match="Focus region contained too few points"):
        mrcal_b200.implied_Rt10__from_unprojections(q0, v0, v1, focus_center=(-1e4, -1e4), focus_radius=10.)


# 3. a known transform, without noise, comes back to the objective's resolution
@pytest.mark.parametrize("atinfinity", [True, False])
def test_known_transform(atinfinity):
    q0, v0, _ = _unprojections()
    r = np.array((0.01, -0.02, 0.005))
    Rt = np.vstack((diff_np.R_from_r(r), np.zeros(3) if atinfinity else (0.05, -0.02, 0.1)))
    d = 1. if atinfinity else 3.
    a = _transform(Rt, v0 * d)
    v1 = a / np.linalg.norm(a, axis=-1)[..., None]
    Rt_dev = mrcal_b200.implied_Rt10__from_unprojections(q0, v0 * d, v1, atinfinity=atinfinity)
    dR = Rt_dev[:3] @ Rt[:3].T
    assert np.arccos(min(1., (np.trace(dR) - 1) / 2.)) <= 1e-6
    assert np.linalg.norm(Rt_dev[3] - Rt[3]) <= 1e-6 * d


# 4. the reprojection against numpy
def _numpy_diff(models, Rt10, gridn, distance):
    lms = [m.intrinsics()[0] for m in models]
    intr = [m.intrinsics()[1] for m in models]
    v, q0 = mrcal_b200.sample_imager_unproject(gridn, None, *models[0].imagersize(), lms, intr, normalize=True)
    d = np.atleast_1d(1. if distance is None else np.array(distance, float))[:, None, None, None]
    Rt10 = np.reshape(Rt10, (-1, 4, 3))
    q = np.array([mrcal_b200.project(_transform(Rt10[k - 1], v[0] * d), lms[k], intr[k]) for k in range(1, len(models))])
    return q - q0, q0


@pytest.mark.parametrize("distance", [None, 4., [1., 10.]])
def test_reprojection(distance):
    opencv8, splined, cam1 = (_model(n) for n in ("cam0.opencv8.cameramodel", "cam0.splined.cameramodel",
                                                  "cam1.opencv8.cameramodel"))
    gridn = 24
    iterable = isinstance(distance, list)
    lead = (len(distance),) if iterable else ()
    H = int(round(2200 / 4000 * gridn))
    cases = [dict(use_uncertainties=False),
             dict(implied_Rt10=np.vstack((diff_np.R_from_r(np.array((0.001, 0.002, -0.003))), (0.01, 0.02, 0.03)))),
             dict(intrinsics_only=True),
             dict(focus_radius=0)]
    for kw in cases:
        models = (opencv8, cam1) if kw.get("focus_radius") == 0 else (opencv8, splined)
        difflen, diff, q0, Rt = mrcal_b200.projection_diff(models, gridn_width=gridn, distance=distance, **kw)
        assert difflen.shape == lead + (H, gridn) and diff.shape == lead + (H, gridn, 2) and Rt.shape == (4, 3)
        if kw.get("intrinsics_only"):
            assert np.array_equal(Rt, np.vstack((np.eye(3), np.zeros(3))))
        if kw.get("focus_radius") == 0:
            assert np.allclose(Rt, np.vstack((cam1.Rt_cam_ref()[:3] @ opencv8.Rt_ref_cam()[:3],
                                              cam1.Rt_cam_ref()[:3] @ opencv8.Rt_ref_cam()[3] + cam1.Rt_cam_ref()[3])),
                               atol=1e-15)
        ref, q0_ref = _numpy_diff(models, Rt, gridn, distance)
        assert np.array_equal(q0, q0_ref)
        ref = ref[0].reshape(diff.shape)
        ok = np.isfinite(ref)
        assert np.array_equal(ok, np.isfinite(diff))
        assert np.abs(diff[ok] - ref[ok]).max() <= 1e-9
        assert np.allclose(difflen, np.linalg.norm(diff, axis=-1), rtol=0, atol=1e-12, equal_nan=True)

    # 3 models: the rms over models 1..2
    shifted = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_OPENCV8", opencv8.intrinsics()[1] * 1.0001),
                                     imagersize=opencv8.imagersize())
    models = (opencv8, splined, shifted)
    difflen, diff, q0, Rt = mrcal_b200.projection_diff(models, gridn_width=gridn, distance=distance,
                                                       use_uncertainties=False)
    assert diff is None and Rt.shape == (2, 4, 3) and difflen.shape == lead + (H, gridn)
    ref, _ = _numpy_diff(models, Rt, gridn, distance)
    ref = np.sqrt(np.mean(np.sum(ref * ref, axis=-1), axis=0)).reshape(difflen.shape)
    ok = np.isfinite(ref)
    assert np.array_equal(ok, np.isfinite(difflen))
    assert np.abs(difflen[ok] - ref[ok]).max() <= 1e-9
    # each pair's fit is the 2-model fit
    for k in (1, 2):
        assert np.array_equal(Rt[k - 1], mrcal_b200.projection_diff((opencv8, models[k]), gridn_width=gridn,
                                                                    distance=distance, use_uncertainties=False)[3])


# 5. weighted by the projection uncertainties of two calibrations of one truth
def _two_calibrations():
    models = []
    for k in range(2):
        kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=1, Nframes=20, W=10, H=10, seed=31,
                                       pixel_noise=0.)
        rng = np.random.default_rng(100 + k)
        ob = kw["observations_board"]
        ob[..., :2] += rng.normal(0., 0.3, ob[..., :2].shape) / ob[..., 2:3]
        mrcal_b200.optimize(**kw)
        models.append(mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=0))
    return models


@pytest.mark.parametrize("distance", [None, [2., 8.]])
def test_uncertainty_weighted(distance, capsys):
    models = _two_calibrations()
    gridn = 20
    difflen, diff, q0, Rt = mrcal_b200.projection_diff(models, gridn_width=gridn, distance=distance)
    assert "WARNING" not in capsys.readouterr().err
    atinfinity = distance is None
    d = np.atleast_1d(1. if atinfinity else np.array(distance))[:, None, None, None]
    v, _ = mrcal_b200.sample_imager_unproject(gridn, None, *models[0].imagersize(), [m.intrinsics()[0] for m in models],
                                              [m.intrinsics()[1] for m in models], normalize=True)
    u = [mrcal_b200.projection_uncertainty(v[k] * d, models[k], atinfinity=atinfinity, what="worstdirection-stdev")
         for k in range(2)]
    w = (1. / (u[0] * u[1])) ** 2
    kw = dict(weights=w, atinfinity=atinfinity, focus_center=(1999.5, 1099.5), focus_radius=4000. * 100.)
    _check_cost(Rt, diff_np.fit(q0, v[0] * d, v[1], **kw), q0, v[0] * d, v[1], **kw)

    # without optimization_inputs: the warning, then the region-based fit
    bare = [mrcal_b200.cameramodel(intrinsics=m.intrinsics(), imagersize=m.imagersize()) for m in models]
    out = mrcal_b200.projection_diff(bare, gridn_width=gridn, distance=distance)
    assert "WARNING: projection_diff() was asked to use uncertainties, but they aren't available" in capsys.readouterr().err
    plain = mrcal_b200.projection_diff(models, gridn_width=gridn, distance=distance, use_uncertainties=False)
    for a, b in zip(out, plain):
        assert np.array_equal(a, b, equal_nan=True)


# 6. determinism
def test_bit_identical():
    opencv8, splined = _model("cam0.opencv8.cameramodel"), _model("cam0.splined.cameramodel")
    a = mrcal_b200.projection_diff((opencv8, splined), gridn_width=60, distance=[3., 10.], use_uncertainties=False,
                                   focus_radius=1000)
    b = mrcal_b200.projection_diff((opencv8, splined), gridn_width=60, distance=[3., 10.], use_uncertainties=False,
                                   focus_radius=1000)
    assert np.array_equal(a[3], b[3])
    assert np.array_equal(a[0], b[0], equal_nan=True)


# 7. noncentral: CAHVORE
def test_cahvore():
    def cahvore(E):
        return mrcal_b200.cameramodel(
            intrinsics=("LENSMODEL_CAHVORE_linearity=0.00",
                        np.array((1000., 1000., 499.5, 399.5, 0.001, -0.002, 0.01, -0.02, 0.005) + tuple(E))),
            imagersize=(1000, 800))
    central, noncentral = cahvore((0., 0., 0.)), cahvore((0.01, 0.02, 0.03))
    pinhole = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((1000., 1000., 499.5, 399.5))),
                                     imagersize=(1000, 800))
    # |E|^2 < 1e-12 counts as central: a finite distance is fine
    difflen, *_ = mrcal_b200.projection_diff((pinhole, central), gridn_width=20, distance=5., use_uncertainties=False)
    assert np.isfinite(difflen).any()
    # E != 0 at infinity without uncertainties: E is zeroed on a copy
    a = mrcal_b200.projection_diff((pinhole, noncentral), gridn_width=20, use_uncertainties=False)
    b = mrcal_b200.projection_diff((pinhole, central), gridn_width=20, use_uncertainties=False)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)
    assert noncentral.intrinsics()[1][-1] == 0.03
    with pytest.raises(RuntimeError, match="No usable uncertainties for those yet"):
        mrcal_b200.projection_diff((pinhole, noncentral), gridn_width=20)
    with pytest.raises(RuntimeError, match="Model 1 is noncentral, so I can only evaluate the diff at infinity"):
        mrcal_b200.projection_diff((pinhole, noncentral), gridn_width=20, distance=5., use_uncertainties=False)
