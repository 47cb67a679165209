"""The pose conversions the host-side plumbing needs (seeding, camera models, stereo and reprojection set-up), in
numpy, for arrays too small to be worth a device call. Layouts are the reference's: R is (...,3,3); Rt is (...,4,3),
R then t; rt is (...,6), r then t. Leading dimensions broadcast. The public, device-backed versions of these
functions, with gradients, are in poseutils.py."""
import numpy as np


def _skew(r):
    z = np.zeros(r.shape[:-1])
    return np.stack((np.stack((z, -r[..., 2], r[..., 1]), -1), np.stack((r[..., 2], z, -r[..., 0]), -1),
                     np.stack((-r[..., 1], r[..., 0], z), -1)), -2)


def R_from_r(r):
    """Rodrigues vectors (...,3) -> rotation matrices (...,3,3)"""
    r = np.asarray(r, float)
    th = np.linalg.norm(r, axis=-1)[..., None, None]
    K = _skew(r)
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(th < 1e-10, 1., np.sin(th) / th)
        c = np.where(th < 1e-10, 0., (1. - np.cos(th)) / (th * th))
    return np.eye(3) + s * K + c * (K @ K)


def _r_from_R(R):
    # the branches of mrcal_r_from_R_full (poseutils.c:1140-1437), as csrc/pose.cuh's r_from_R() takes them
    u = np.array((R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]))
    costh = (R[0, 0] + R[1, 1] + R[2, 2] - 1.) / 2.
    eps = 1e-8
    norm2u = u @ u
    if norm2u > 4. * eps * eps and 1. - abs(costh) > eps * eps / 2.:
        sinth = np.sqrt(norm2u) / 2.
        th = np.arccos(costh) if sinth > np.sqrt(2.) / 2. else (np.arcsin(sinth) if costh > 0 else
                                                                  np.pi - np.arcsin(sinth))
        return u / np.sqrt(norm2u) * th
    if costh > 0:
        return u / 2.
    # near a half-turn: |v_i| = sqrt((1 + R_ii)/2), the signs from the symmetric part
    v = np.sqrt(np.maximum((np.diag(R) + 1.) / 2., 0.))
    i = 0 if v[0] > 0.1 else (1 if v[1] > 0.1 else 2)
    for j in range(3):
        if j != i and R[i, j] + R[j, i] < 0:
            v[j] *= -1.
    return u / -2. + v * np.pi


def r_from_R(R):
    """Rotation matrices (...,3,3) -> Rodrigues vectors (...,3)"""
    R = np.asarray(R, float)
    return np.array([_r_from_R(M) for M in R.reshape(-1, 3, 3)]).reshape(R.shape[:-2] + (3,))


def Rt_from_rt(rt):
    rt = np.asarray(rt, float)
    return np.concatenate((R_from_r(rt[..., :3]), rt[..., None, 3:]), -2)


def rt_from_Rt(Rt):
    Rt = np.asarray(Rt, float)
    return np.concatenate((r_from_R(Rt[..., :3, :]), Rt[..., 3, :]), -1)


def invert_Rt(Rt):
    Rt = np.asarray(Rt, float)
    Ri = np.swapaxes(Rt[..., :3, :], -1, -2)
    return np.concatenate((Ri, -(Ri @ Rt[..., 3, :, None])[..., None, :, 0]), -2)


def invert_rt(rt):
    """(r,t) of the inverse transform: x = R y + t  <=>  y = R' x - R' t"""
    rt = np.asarray(rt, float)
    Ri = np.swapaxes(R_from_r(rt[..., :3]), -1, -2)
    return np.concatenate((-rt[..., :3], -(Ri @ rt[..., 3:, None])[..., 0]), -1)


def transform_point_Rt(Rt, p):
    """x -> R x + t"""
    Rt = np.asarray(Rt, float)
    return (Rt[..., :3, :] @ np.asarray(p, float)[..., None])[..., 0] + Rt[..., 3, :]


def compose_Rt(Rt0, Rt1):
    """x -> Rt0(Rt1(x))"""
    Rt0, Rt1 = np.asarray(Rt0, float), np.asarray(Rt1, float)
    return np.concatenate((Rt0[..., :3, :] @ Rt1[..., :3, :], transform_point_Rt(Rt0, Rt1[..., 3, :])[..., None, :]),
                          -2)
