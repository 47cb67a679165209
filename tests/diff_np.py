"""A plain numpy + scipy restatement of mrcal.implied_Rt10__from_unprojections() (mrcal/model_analysis.py:27-395):
the same data cleanup, focus region, residuals (rotation only, and rt) and scipy.optimize.least_squares call
(method='dogbox', loss='huber', f_scale=(5 deg)^2, gtol=eps). robust_cost() evaluates the objective at any Rt, so a
test can compare two fits by what they minimize rather than by their path."""
import numpy as np
import scipy.optimize

C = (5. * np.pi / 180.) ** 2


def skew(p):
    """[p]x for p (..., 3): (..., 3, 3)"""
    z = np.zeros(p.shape[:-1])
    return np.stack((np.stack((z, -p[..., 2], p[..., 1]), -1),
                     np.stack((p[..., 2], z, -p[..., 0]), -1),
                     np.stack((-p[..., 1], p[..., 0], z), -1)), -2)


def R_from_r(r):
    th2 = float(r @ r)
    K = skew(np.asarray(r, float))
    if th2 < 1e-20:
        return np.eye(3) + K
    th = np.sqrt(th2)
    return np.eye(3) + np.sin(th) / th * K + (1. - np.cos(th)) / th2 * (K @ K)


def rotate_point_r(r, p):
    """(R p, d(R p)/dr (..., 3, 3)): d(R p)/dr = -R [p]x J_r(r), J_r the right Jacobian of SO(3)"""
    R = R_from_r(r)
    th2 = float(r @ r)
    K = skew(np.asarray(r, float))
    if th2 < 1e-12:
        a, b = 0.5 - th2 / 24., 1. / 6. - th2 / 120.
    else:
        th = np.sqrt(th2)
        a, b = (1. - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    Jr = np.eye(3) - a * K + b * (K @ K)
    return p @ R.T, -np.einsum("ij,...jk,kl->...il", R, skew(p), Jr)


def residual_jacobian_r(r, p0, v1, w):
    """at infinity: x = w th2, th2 = 2 (1 - (R p0).v1), for p0 (M,N,3), v1 (N,3), w (M,N)"""
    rp, drp = rotate_point_r(r, p0)
    inner = np.sum(rp * v1, axis=-1)
    x = 2. * (1. - inner) * w
    J = -2. * np.einsum("...i,...ik->...k", np.broadcast_to(v1, rp.shape), drp) * w[..., None]
    return x.ravel(), J.reshape(-1, 3)


def residual_jacobian_rt(rt, p0, v1, w):
    """at a distance: x = w th2, th2 = 2 (1 - a.v1/|a|), a = R p0 + t"""
    rp, drp = rotate_point_r(rt[:3], p0)
    a = rp + rt[3:]
    da = np.concatenate((drp, np.broadcast_to(np.eye(3), drp.shape)), axis=-1)   # (M,N,3,6)
    mag = np.linalg.norm(a, axis=-1)
    inner = np.sum(a * v1, axis=-1)
    x = 2. * (1. - inner / mag) * w
    dmag = np.einsum("...i,...ik->...k", a, da) / mag[..., None]
    dinner = np.einsum("...i,...ik->...k", np.broadcast_to(v1, a.shape), da)
    J = 2. * (inner[..., None] * dmag - mag[..., None] * dinner) / (mag * mag)[..., None] * w[..., None]
    return x.ravel(), J.reshape(-1, 6)


def prepare(q0, p0, v1, weights=None, focus_center=(0., 0.), focus_radius=1e8):
    """The reference's cleanup: (p0 (M,n,3), v1 (n,3), w (M,n)) over the n points of the focus region, with the
    non-finite entries zeroed and their weights 0"""
    q0 = np.reshape(q0, (-1, 2))
    N = q0.shape[0]
    p0 = np.array(p0, float).reshape(-1, N, 3)
    v1 = np.array(v1, float).reshape(N, 3)
    w = np.ones(p0.shape[:-1]) if weights is None else np.array(weights, float).reshape(p0.shape[:-1])
    w[~np.isfinite(w)] = 0.
    bad = ~np.isfinite(p0)
    p0[bad] = 0.
    w[bad.any(axis=-1)] = 0.
    bad = ~np.isfinite(v1)
    v1[bad] = 0.
    w[:, bad.any(axis=-1)] = 0.
    d = q0 - np.asarray(focus_center, float)
    i = np.sum(d * d, axis=-1) < focus_radius * focus_radius
    if np.count_nonzero(i) < 3:
        raise Exception("Focus region contained too few points")
    return p0[:, i], v1[i], w[:, i]


def fit(q0, p0, v1, weights=None, atinfinity=True, focus_center=(0., 0.), focus_radius=1e8, seed=0):
    """The reference's scipy fit; Rt (4,3)"""
    p0, v1, w = prepare(q0, p0, v1, weights, focus_center, focus_radius)
    f = residual_jacobian_r if atinfinity else residual_jacobian_rt
    x0 = np.random.default_rng(seed).random(3 if atinfinity else 6) * 1e-5
    res = scipy.optimize.least_squares(lambda x: f(x, p0, v1, w)[0], x0, jac=lambda x: f(x, p0, v1, w)[1],
                                       method="dogbox", loss="huber", f_scale=C, gtol=np.finfo(float).eps)
    Rt = np.zeros((4, 3))
    Rt[:3] = R_from_r(res.x[:3])
    if not atinfinity:
        Rt[3] = res.x[3:]
    return Rt


def robust_terms(Rt, q0, p0, v1, weights=None, atinfinity=True, focus_center=(0., 0.), focus_radius=1e8):
    """(f, w) over the kept points: f = w th2 at Rt"""
    p0, v1, w = prepare(q0, p0, v1, weights, focus_center, focus_radius)
    a = p0 @ Rt[:3].T
    if atinfinity:
        th2 = 2. * (1. - np.sum(a * v1, axis=-1))
    else:
        a = a + Rt[3]
        th2 = 2. * (1. - np.sum(a * v1, axis=-1) / np.linalg.norm(a, axis=-1))
    return np.where(w != 0., w * th2, 0.), w


def robust_cost(Rt, *args, **kwargs):
    """sum of huber(f^2): f^2 below C^2, 2 C |f| - C^2 above"""
    f, _ = robust_terms(Rt, *args, **kwargs)
    af = np.abs(f)
    return float(np.sum(np.where(af <= C, f * f, 2. * C * af - C * C)))


def cost_floor(Rt, *args, **kwargs):
    """What rounding th2 (about 4 eps per point) can move the cost by"""
    f, w = robust_terms(Rt, *args, **kwargs)
    e = 4. * np.finfo(float).eps * w
    return float(np.sum(2. * np.abs(f) * e + e * e))
