"""model_resolution__deg_pixel() (csrc/project.cu) and stereo_pair_diff() (csrc/diff.cu) against the reference's
algorithms restated in tests/unproject_np.py, through the fixture of test_unproject_gradients_gpu.py (the compiled
reference, or its answers stored in tests/golden/unproject_gradients.npz)."""
import os

import numpy as np
import pytest

import mrcal_b200
from test_unproject_gradients_gpu import behind_ok, reference  # noqa: F401  (reference: the fixture)

pytestmark = pytest.mark.gpu

CAMERAS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cameramodels")
MODES = ("mean", "min", "max", "eccentricity")


def camera(name):
    return mrcal_b200.cameramodel(os.path.join(CAMERAS, name + ".cameramodel"))


def resolution_pixels(m):
    W, H = m.imagersize()
    return mrcal_b200.sample_imager(9, 6, W, H)


def pairs(kind):
    return ((camera("cam0." + kind), camera("cam1." + kind)),)


def pair_args(pair):
    (lm0, i0), (lm1, i1) = pair[0].intrinsics(), pair[1].intrinsics()
    return lm0, i0, lm1, i1


def Rt10(pair, atinfinity):
    Rt = np.vstack((pair[1].Rt_cam_ref()[:3] @ pair[0].Rt_ref_cam()[:3],
                    pair[1].Rt_cam_ref()[:3] @ pair[0].Rt_ref_cam()[3] + pair[1].Rt_cam_ref()[3]))
    if atinfinity:
        Rt[3] = 0
    return Rt


def second_calibration(pair):
    """the same pair, calibrated again: the intrinsics and the extrinsics of camera 1 moved a little"""
    m0, m1 = pair
    lm, intr = m1.intrinsics()
    intr = intr.copy()
    intr[:4] *= (1.0004, 0.9997, 1.0002, 0.9999)
    m1b = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=m1.imagersize(),
                                 rt_cam_ref=m1.rt_cam_ref() + (1e-4, -2e-4, 1e-4, 1e-3, 0., -2e-3))
    return m0, m1b


def reference_calls():
    """(key, method, args) of every call these tests make of the restatement"""
    for kind in ("opencv8", "splined"):
        m = camera("cam0." + kind)
        lm, intr = m.intrinsics()
        for mode in MODES:
            yield f"resolution/{kind}/{mode}", "model_resolution", (resolution_pixels(m), lm, intr, mode, behind_ok(lm))
        pair0 = pairs(kind)[0]
        pair1 = second_calibration(pair0)
        W, H = pair0[0].imagersize()
        q0 = mrcal_b200.sample_imager(20, None, W, H)
        for distance in (None, 5.):
            for p, pair in enumerate((pair0, pair1)):
                yield (f"stereo_pair/{kind}/{distance}/{p}", "reproject",
                       (q0, *pair_args(pair), Rt10(pair, distance is None), 1. if distance is None else distance,
                        behind_ok(lm)))


@pytest.mark.parametrize("kind", ("opencv8", "splined"))
def test_model_resolution(reference, kind):  # noqa: F811
    m = camera("cam0." + kind)
    lm, intr = m.intrinsics()
    q = resolution_pixels(m)
    for mode in MODES:
        r_ref, = reference.call(f"resolution/{kind}/{mode}", "model_resolution", q, lm, intr, mode, behind_ok(lm))
        r = mrcal_b200.model_resolution__deg_pixel(q, m, mode=mode)
        assert r.shape == q.shape[:-1]
        assert np.abs(r - r_ref.reshape(r.shape)).max() <= 1e-9 * np.abs(r_ref).max()
    assert mrcal_b200.model_resolution__deg_pixel(q[0, 0], m).shape == ()


def test_model_resolution_pinhole_center():
    f = 1234.
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((f, f, 499.5, 399.5))), imagersize=(1000, 800))
    r = mrcal_b200.model_resolution__deg_pixel(np.array((499.5, 399.5)), m, mode="max")
    assert abs(r - np.degrees(np.arctan(1. / f))) < 1e-6 * r
    assert abs(mrcal_b200.model_resolution__deg_pixel(np.array((499.5, 399.5)), m, mode="eccentricity") - 1.) < 1e-12


@pytest.mark.parametrize("kind", ("opencv8", "splined"))
def test_stereo_pair_diff(reference, kind):  # noqa: F811
    pair0 = pairs(kind)[0]
    pair1 = second_calibration(pair0)
    lm = pair0[0].intrinsics()[0]
    W, H = pair0[0].imagersize()
    before = [(m.intrinsics()[1].copy(), m.rt_cam_ref()) for m in pair0 + pair1]
    for distance in (None, 5.):
        q1 = [reference.call(f"stereo_pair/{kind}/{distance}/{p}", "reproject",
                             mrcal_b200.sample_imager(20, None, W, H), *pair_args(pair),
                             Rt10(pair, distance is None), 1. if distance is None else distance, behind_ok(lm))[0]
              for p, pair in enumerate((pair0, pair1))]
        difflen, diff, q0, reproject = mrcal_b200.stereo_pair_diff((pair0, pair1), gridn_width=20, distance=distance)
        diff_ref = (q1[1] - q1[0]).reshape(diff.shape)
        assert q0.shape == diff.shape and difflen.shape == q0.shape[:-1]
        assert np.array_equal(q0, mrcal_b200.sample_imager(20, None, W, H))
        assert np.abs(diff - diff_ref).max() <= 1e-9 * (1. + np.abs(q1[0]).max())
        assert np.abs(difflen - np.linalg.norm(diff_ref, axis=-1)).max() <= 1e-9 * (1. + np.abs(q1[0]).max())
        # a pair diffed with itself
        difflen0, diff0, _, _ = mrcal_b200.stereo_pair_diff((pair0, pair0), gridn_width=20, distance=distance)
        assert not np.any(diff0) and not np.any(difflen0)
    # the callers' models are untouched
    for m, (intr, rt) in zip(pair0 + pair1, before):
        assert np.array_equal(m.intrinsics()[1], intr) and np.array_equal(m.rt_cam_ref(), rt)


def test_stereo_pair_reprojection_round_trip():
    pair = pairs("opencv8")[0]
    _, _, q0, reproject = mrcal_b200.stereo_pair_diff((pair, pair), gridn_width=30)
    q1 = reproject(q0, 0, 0)
    assert q1.shape == q0.shape
    # the pixels camera 1 sees: elsewhere a lens model need not be invertible
    W, H = pair[1].imagersize()
    inside = (q1[..., 0] > 100) & (q1[..., 0] < W - 100) & (q1[..., 1] > 100) & (q1[..., 1] < H - 100)
    assert inside.sum() > 100
    assert np.abs(reproject(q1[inside], 0, 1) - q0[inside]).max() < 1e-6


def test_stereo_pair_diff_cahvore():
    lm = "LENSMODEL_CAHVORE_linearity=0.37"
    intr = np.array((1000., 1000., 499.5, 399.5, 0., 0., 0., 0., 0., 0.01, 0.02, 0.03))
    m = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=(1000, 800))
    m1 = mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=(1000, 800), rt_cam_ref=(0., 0., 0., -0.1, 0., 0.))
    with pytest.raises(RuntimeError, match="only valid at infinity"):
        mrcal_b200.stereo_pair_diff(((m, m1), (m, m1)), distance=5.)
    # at infinity E is zeroed, in a copy
    difflen, diff, _, _ = mrcal_b200.stereo_pair_diff(((m, m1), (m, m1)), gridn_width=10)
    assert not np.any(diff) and np.array_equal(m.intrinsics()[1], intr)
