"""projection_uncertainty() against Monte Carlo, independent of any restated formula: a noiseless calibration is
perturbed 200 times with seeded pixel noise of standard deviation sigma/weight, each copy is re-solved on the device,
and about 10 query points are reprojected through each solution the way the method defines the perturbed projection
q*. The empirical covariance of q* must match the predicted one (sigma known): worst-direction stdev within 20 % at
every point. The sigma estimated from a noisy solution's residuals must be within 10 % of the true one. Seeds are
fixed: the outcome is fixed."""
import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import synthetic
import uncertainty_np as unp

pytestmark = pytest.mark.gpu

SIGMA = 0.3
NSAMPLES = 200


def _clone(kw):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}


def _query(kw, icam, n=10):
    W, H = kw["imagersizes"][icam]
    q = np.stack(np.meshgrid(np.linspace(0.15 * W, 0.85 * W, 5), np.linspace(0.25 * H, 0.75 * H, 2)), -1).reshape(-1, 2)[:n]
    v = mrcal_b200.unproject(q, kw["lensmodel"], kw["intrinsics"][icam])
    return 10. * v / np.linalg.norm(v, axis=-1)[..., None]


def _transform(rt, p):
    return p @ unp.R_from_r(rt[:3]).T + rt[3:]


def _transform_inv(rt, p):
    return (p - rt[3:]) @ unp.R_from_r(rt[:3])


def _run(kw0, icam, qstar):
    """kw0: a solved noiseless problem. qstar(kw_solved) -> (Npts, 2). Returns (empirical cov, predicted cov, sigma_est)"""
    pts = _query(kw0, icam)
    q0 = qstar(kw0, pts)
    rng = np.random.default_rng(11)
    dq = []
    sigma_est = None
    for k in range(NSAMPLES):
        kw = _clone(kw0)
        ob = kw["observations_board"]
        ob[..., :2] += rng.normal(0., SIGMA, ob[..., :2].shape) / ob[..., 2:3]
        mrcal_b200.optimize(**kw)
        dq.append(qstar(kw, pts) - q0)
        if k == 0:
            sigma_est = mrcal_b200.Problem(**kw).projection_uncertainty(pts[:1], icam, method="mean-pcam")[1]
    dq = np.array(dq)                                                   # (Nsamples, Npts, 2)
    dq -= dq.mean(axis=0)
    emp = np.einsum("spi,spj->pij", dq, dq) / (NSAMPLES - 1)
    Var, s = mrcal_b200.Problem(**_clone(kw0)).projection_uncertainty(pts, icam, method="mean-pcam",
                                                                      observed_pixel_uncertainty=SIGMA)
    assert s == SIGMA
    return emp, Var, sigma_est


def _check(emp, Var, sigma_est):
    w_emp = mrcal_b200.worst_direction_stdev(emp)
    w_pred = mrcal_b200.worst_direction_stdev(Var)
    assert np.all(np.abs(w_emp / w_pred - 1.) < 0.2), (w_emp, w_pred)
    assert abs(sigma_est / SIGMA - 1.) < 0.1, sigma_est


def test_surveyed_camera_at_reference():
    """(a) one camera at the reference, the board poses surveyed (not optimized): q* = project(p_cam, intrinsics*)"""
    kw, truth = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=1, Nframes=20, W=10, H=10, seed=21,
                                       pixel_noise=0.)
    kw["rt_ref_frame"] = np.ascontiguousarray(truth["rt_ref_frame"])
    kw["calobject_warp"] = np.array(truth["calobject_warp"], float)
    kw["do_optimize_frames"] = False
    kw["do_optimize_calobject_warp"] = False
    mrcal_b200.optimize(**kw)

    def qstar(k, pts):
        return mrcal_b200.project(pts, k["lensmodel"], k["intrinsics"][0])
    _check(*_run(kw, 0, qstar))


def test_two_cameras_frames_optimized():
    """(b) two cameras, frames optimized; camera 1 has extrinsics. q* projects the mean over the frames of the point
    carried through each frame: p_ref = T_ref,cam p_cam, p_frame_f = T_f,ref p_ref (solution without noise),
    p_cam* = mean_f T*_cam,ref T*_ref,f p_frame_f, q* = project(p_cam*, intrinsics*)"""
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=2, Nframes=20, W=10, H=10, seed=22,
                                   pixel_noise=0.)
    mrcal_b200.optimize(**kw)
    rt_cam0, rt_f0 = kw["rt_cam_ref"][0].copy(), kw["rt_ref_frame"].copy()

    def qstar(k, pts):
        p_ref = _transform_inv(rt_cam0, pts)
        p_cam = np.zeros_like(pts)
        for f in range(rt_f0.shape[0]):
            p_cam += _transform(k["rt_cam_ref"][0], _transform(k["rt_ref_frame"][f], _transform_inv(rt_f0[f], p_ref)))
        return mrcal_b200.project(p_cam / rt_f0.shape[0], k["lensmodel"], k["intrinsics"][1])
    _check(*_run(kw, 1, qstar))
