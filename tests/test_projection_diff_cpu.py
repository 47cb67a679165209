"""CPU: the parts of projection_diff() that need no device (the grid, the refusals before any device work, the C entry
points without a device), and the Jacobians of the numpy restatement the GPU tests compare against."""
import os

import numpy as np
import pytest

import mrcal_b200
import diff_np

MODELS = os.path.join(os.path.dirname(__file__), "golden", "cameramodels")


def _pinhole(W=1000, H=800):
    return mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((1000., 1000., (W - 1) / 2., (H - 1) / 2.))),
                                  imagersize=(W, H))


def test_sample_imager():
    q = mrcal_b200.sample_imager(60, 40, 1000, 800)
    assert q.shape == (40, 60, 2)
    assert np.array_equal(q[0, 0], (0., 0.)) and np.array_equal(q[-1, -1], (999., 799.))
    assert np.allclose(q[3, 7], (7 * 999. / 59, 3 * 799. / 39), rtol=0, atol=1e-12)
    assert np.all(q[:, :, 1] == q[:, :1, 1]) and np.all(q[:, :, 0] == q[:1, :, 0])
    # Python's round(): 2200/4000*50 = 27.5 rounds to the even 28
    assert mrcal_b200.sample_imager(50, None, 4000, 2200).shape == (28, 50, 2)
    assert mrcal_b200.sample_imager(50, None, 3000, 2000).shape == (33, 50, 2)


def test_refusals_before_device_work():
    m = _pinhole()
    with pytest.raises(RuntimeError, match="At least 2 models"):
        mrcal_b200.projection_diff((m,))
    with pytest.raises(RuntimeError, match="supported ONLY if exactly 2 models"):
        mrcal_b200.projection_diff((m, m, m), implied_Rt10=np.vstack((np.eye(3), np.zeros(3))))
    with pytest.raises(RuntimeError, match="imager dimensions to match"):
        mrcal_b200.projection_diff((m, _pinhole(1000, 700)))
    cahvore = mrcal_b200.cameramodel(
        intrinsics=("LENSMODEL_CAHVORE_linearity=0.00",
                    np.array((1000., 1000., 499.5, 399.5, 0., 0., 0., 0., 0., 0.01, 0.02, 0.03))),
        imagersize=(1000, 800))
    with pytest.raises(RuntimeError, match="Model 1 is noncentral, so I can only evaluate the diff at infinity"):
        mrcal_b200.projection_diff((m, cahvore), distance=5., use_uncertainties=False)


def test_model_pose_getters():
    m = mrcal_b200.cameramodel(os.path.join(MODELS, "cam1.opencv8.cameramodel"))
    rt = m.rt_cam_ref()
    Rt = m.Rt_cam_ref()
    assert Rt.shape == (4, 3)
    assert np.allclose(Rt[:3], diff_np.R_from_r(rt[:3]), atol=1e-14) and np.array_equal(Rt[3], rt[3:])
    p = np.array((0.3, -0.2, 4.))
    assert np.allclose(m.Rt_ref_cam()[:3] @ (Rt[:3] @ p + Rt[3]) + m.Rt_ref_cam()[3], p, atol=1e-12)


@pytest.mark.skipif(mrcal_b200.device_count() > 0, reason="checks the behaviour without a device")
def test_no_device():
    from mrcal_b200 import _capi
    Rt = np.zeros((4, 3))
    assert not _capi.lib.mrcal_b200_implied_Rt10__from_unprojections(Rt.ctypes.data, None, 0, None, 1, None, None,
                                                                     True, None, 1.)
    assert "no usable CUDA device" in _capi.last_error()
    assert not _capi.lib.mrcal_b200_projection_diff(None, None, None, None, 0, None, 2, None, 1, None, None, None, None,
                                                    1., True)
    assert "no usable CUDA device" in _capi.last_error()


@pytest.mark.parametrize("atinfinity", [True, False])
def test_restatement_jacobians(atinfinity):
    rng = np.random.default_rng(5)
    M, N = 2, 40
    v1 = rng.normal(size=(N, 3)) + (0., 0., 4.)
    v1 /= np.linalg.norm(v1, axis=-1)[..., None]
    p0 = v1 + rng.normal(scale=0.02, size=(M, N, 3))
    if atinfinity:
        p0 /= np.linalg.norm(p0, axis=-1)[..., None]
        x = np.array((0.01, -0.02, 0.015))
        f = diff_np.residual_jacobian_r
    else:
        p0 *= np.array((3., 7.))[:, None, None]
        x = np.array((0.01, -0.02, 0.015, 0.1, -0.05, 0.2))
        f = diff_np.residual_jacobian_rt
    w = rng.uniform(0.5, 2., size=(M, N))
    _, J = f(x, p0, v1, w)
    h = 1e-6
    for k in range(x.size):
        d = np.zeros_like(x)
        d[k] = h
        fd = (f(x + d, p0, v1, w)[0] - f(x - d, p0, v1, w)[0]) / (2 * h)
        assert np.allclose(J[:, k], fd, rtol=0, atol=1e-8 * (1 + np.abs(fd).max())), k
