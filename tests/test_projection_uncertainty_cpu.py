"""CPU: the parts of projection_uncertainty() that need no device, and the test oracle of
test_projection_uncertainty_gpu.py checked against finite differences of projection through the pose chain."""
import numpy as np
import pytest

import mrcal_b200
import uncertainty_np as unp


@pytest.mark.skipif(mrcal_b200.device_count() > 0, reason="checks the behaviour without a device")
def test_no_device():
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((1000., 1000., 500., 400.))),
                               imagersize=(1000, 800))
    m._optimization_inputs_string = None
    with pytest.raises(RuntimeError, match="optimization_inputs are unavailable"):
        mrcal_b200.projection_uncertainty(np.array((0., 0., 1.)), m)
    from mrcal_b200 import _capi
    assert not _capi.lib.mrcal_b200_problem_projection_uncertainty(None, 0, 2, False, None, 0, -1., None, None)
    assert "no usable CUDA device" in _capi.last_error()


def test_worst_direction_closed_form():
    rng = np.random.default_rng(1)
    A = rng.normal(size=(50, 2, 2))
    V = A @ np.swapaxes(A, -1, -2)
    assert np.allclose(mrcal_b200.worst_direction_stdev(V), np.sqrt(np.linalg.eigvalsh(V)[..., -1]), rtol=1e-12)


def _pinhole(p, f=800., c=(600., 400.)):
    return np.array((f * p[0] / p[2] + c[0], f * p[1] / p[2] + c[1]))


def _dpinhole(p, f=800.):
    return np.array(((f / p[2], 0., -f * p[0] / p[2] ** 2), (0., f / p[2], -f * p[1] / p[2] ** 2)))


@pytest.mark.parametrize("atinfinity", [False, True])
def test_restatement_against_finite_differences(atinfinity):
    """mean-pcam rows of the restatement: q(p_cam') with p_cam' = T_cam' (T_frame' (T_frame^-1 (T_cam^-1 p_cam))),
    perturbing one unknown of an extrinsics or frame pose at a time (rotation only at infinity)"""
    rng = np.random.default_rng(4)
    rt_cam = np.array([[0.02, -0.1, 0.05, -0.5, 0.1, 0.2]])
    rt_frames = rng.normal(scale=(0.3, 0.3, 0.3, 1., 1., 1.), size=(3, 6))
    p = np.array((0.4, -0.2, 5.))
    Nstate = 6 + 18

    def q_of(dcam, dframe, f):
        rc = rt_cam[0] + dcam
        R0 = unp.R_from_r(rt_cam[0, :3])
        t0 = np.zeros(3) if atinfinity else rt_cam[0, 3:]
        p_ref = R0.T @ (p - t0)
        Rf0 = unp.R_from_r(rt_frames[f, :3])
        tf0 = np.zeros(3) if atinfinity else rt_frames[f, 3:]
        p_frame = Rf0.T @ (p_ref - tf0)
        rf = rt_frames[f] + dframe
        p_ref2 = unp.R_from_r(rf[:3]) @ p_frame + (0. if atinfinity else rf[3:])
        return _pinhole(unp.R_from_r(rc[:3]) @ p_ref2 + (0. if atinfinity else rc[3:]))

    A, G = unp.dq_db_unpacked(p, _dpinhole(p), np.zeros((2, 4)), method="mean-pcam", atinfinity=atinfinity,
                              Nstate=Nstate, intr_cols=[], intr_arg0=0, rt_cam=rt_cam, extr_col0=0,
                              rt_frames=rt_frames, frame_col0=6)
    assert not G.any()
    h = 1e-6
    for k in range(6):
        d = np.zeros(6); d[k] = h
        fd = np.mean([(q_of(d, 0., f) - q_of(-d, 0., f)) / (2 * h) for f in range(3)], axis=0)
        expect = 0. * fd if (atinfinity and k >= 3) else fd
        assert np.allclose(A[:, k], expect, atol=1e-6 * (1 + np.abs(fd).max()))
        for f in range(3):
            fdf = (q_of(0., d, f) - q_of(0., -d, f)) / (2 * h) / 3.
            expect = 0. * fdf if (atinfinity and k >= 3) else fdf
            assert np.allclose(A[:, 6 + 6 * f + k], expect, atol=1e-6 * (1 + np.abs(fdf).max()))


def test_restatement_ccp_term():
    """ccp: q(p_cam*) with p_cam* = T(rt) p_cam for a tiny rt has  dq/drt = [dq/dpcam skew(p)... ] up to the sign
    convention of the reference (p_cam = p_cam* + r x p_cam + t): G = dq/dpcam [skew(p_cam) | -I]"""
    p = np.array((0.4, -0.2, 5.))
    _, G = unp.dq_db_unpacked(p, _dpinhole(p), np.zeros((2, 4)), method="cross-reprojection-ccp", atinfinity=False,
                              Nstate=1, intr_cols=[], intr_arg0=0)
    h = 1e-6
    for k in range(6):
        d = np.zeros(6); d[k] = h
        # p_cam* = p_cam - r x p_cam - t to first order
        fd = (_pinhole(p - np.cross(d[:3], p) - d[3:]) - _pinhole(p + np.cross(d[:3], p) + d[3:])) / (2 * h)
        assert np.allclose(G[:, k], fd, atol=1e-6 * (1 + np.abs(fd).max()))
