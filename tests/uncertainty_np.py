"""A dense numpy restatement of projection uncertainty, written from the math, used as the test oracle.

Notation: b is the packed state, u = D b the unpacked one (D = diag of the pack scales), J = dx/db the packed
Jacobian, Jo its leading board/point rows, x the residuals. Pixel noise of standard deviation sigma on the
observations moves the optimum by  db = -inv(J'J) Jo' dx_o,  so

    Var(b) = sigma^2 inv(J'J) Jo'Jo inv(J'J)        (= sigma^2 inv(J'J) without regularization rows)

and a quantity F(b) has  Var(F) = dF/db Var(b) dF/db',  dF/db = dF/du D.

F is the projection q of a camera-frame point p_cam by camera icam. What q depends on is the method's choice:

    all methods:  q depends on the camera's intrinsics:             dq/dintrinsics
    mean-pcam:    p_cam is the mean over the camera's extrinsics j and the frames f of
                  T_cam_j,ref T_ref,f T_f,ref T_ref,cam_j p_cam with the frames' and extrinsics' perturbations:
                     dq/drt_cam_j   = dq/dpcam dpcam/drt_cam_j (at p_ref_j) / Ne
                     dq/drt_frame_f = mean_j dq/dpcam R_j dpref/drt_frame_f (at p_frame) / Nframes
    rrp-Jfp:      the extrinsics term above, plus the reference frame moving by rt(b) = K_rrp b:
                     p_ref* ~ p_ref + skew(p_ref) r - t  ->  dq/db += dq/dpref (skew(p_ref) K[:3] - K[3:])
    ccp:          the camera frame moving by rt(b) = K_ccp b:  dq/db += dq/dpcam (skew(p_cam) K[:3] - K[3:])

At infinity only rotations act: translations, and the terms in K[3:], drop out. K = drt/db (packed) is per packed
unknown already, so it is not multiplied by D.

sigma, when not given: sqrt(sum x_o^2 / No) / sqrt(1 - Nstate/No) over the No board/point residuals.
"""
import numpy as np


def skew(v):
    return np.array([[0., -v[2], v[1]], [v[2], 0., -v[0]], [-v[1], v[0], 0.]])


def R_from_r(r):
    """Rodrigues; works on complex input (for complex-step derivatives)"""
    r = np.asarray(r)
    th2 = np.sum(r * r)
    if abs(th2) < 1e-30:
        return np.eye(3) + skew(r)
    th = np.sqrt(th2)
    return np.cos(th) * np.eye(3) + np.sin(th) / th * skew(r) + (1 - np.cos(th)) / th2 * np.outer(r, r)


def dRp_dr(r, p):
    """d(R(r) p)/dr (3x3), by complex step: exact to roundoff"""
    h = 1e-30
    out = np.zeros((3, 3))
    for k in range(3):
        rc = np.array(r, complex)
        rc[k] += 1j * h
        out[:, k] = (R_from_r(rc) @ p).imag / h
    return out


def dq_db_unpacked(p_cam, dq_dp, dq_di, *, method, atinfinity, Nstate, intr_cols, intr_arg0,
                   rt_cam=None, extr_col0=None, rt_frames=None, frame_col0=None, K=None):
    """The two rows dq/du (unpacked, 2 x Nstate) of one point, without the K term (returned as G (2,6): the K term is
    G @ K, per packed unknown).  intr_cols: the state columns of the camera's optimized intrinsics, which are the
    model's parameters intr_arg0, intr_arg0+1, ... rt_cam: (Ne,6) the camera's extrinsics (None: at the reference),
    extr_col0: the state column of the first of them (None: not optimized). rt_frames (Nframes,6) and frame_col0:
    the frames, for mean-pcam (None: not optimized)."""
    A = np.zeros((2, Nstate))
    for j, c in enumerate(intr_cols):
        A[:, c] = dq_di[:, intr_arg0 + j]
    rts = np.zeros((1, 6)) if rt_cam is None else np.atleast_2d(rt_cam)
    Ne = rts.shape[0]
    G = np.zeros((2, 6))
    for j in range(Ne):
        R = R_from_r(rts[j, :3])
        t = np.zeros(3) if atinfinity else rts[j, 3:]
        p_ref = R.T @ (p_cam - t)
        dq_dpref = dq_dp @ R
        if method != "cross-reprojection-ccp" and rt_cam is not None and extr_col0 is not None:
            c0 = extr_col0 + 6 * j
            A[:, c0:c0 + 3] = dq_dp @ dRp_dr(rts[j, :3], p_ref) / Ne
            if not atinfinity:
                A[:, c0 + 3:c0 + 6] = dq_dp / Ne
        if method == "mean-pcam" and rt_frames is not None and frame_col0 is not None:
            Nf = rt_frames.shape[0]
            for f in range(Nf):
                Rf = R_from_r(rt_frames[f, :3])
                tf = np.zeros(3) if atinfinity else rt_frames[f, 3:]
                p_frame = Rf.T @ (p_ref - tf)
                c0 = frame_col0 + 6 * f
                A[:, c0:c0 + 3] += dq_dpref @ dRp_dr(rt_frames[f, :3], p_frame) / (Ne * Nf)
                if not atinfinity:
                    A[:, c0 + 3:c0 + 6] += dq_dpref / (Ne * Nf)
        if j == 0 and method != "mean-pcam":
            x, g = (p_cam, dq_dp) if method == "cross-reprojection-ccp" else (p_ref, dq_dpref)
            G[:, :3] = g @ skew(x)
            if not atinfinity:
                G[:, 3:] = -g
    return A, G


def sigma_estimate(x_obs, Nstate):
    n = x_obs.size
    return np.sqrt(np.sum(x_obs * x_obs) / n) / np.sqrt(1. - Nstate / n)


def propagate(dF_dbpacked, J, Nobs_rows, sigma):
    """Var(F) (..., 2, 2) for dF/db_packed (N, 2, Nstate), with a dense solve of J'J and Jo'Jo over the leading rows"""
    Jd = J.toarray() if hasattr(J, "toarray") else J
    JtJ = Jd.T @ Jd
    A = dF_dbpacked.reshape(-1, JtJ.shape[0])
    X = np.linalg.solve(JtJ, A.T)                  # inv(J'J) dF'
    if Nobs_rows < Jd.shape[0]:
        Y = Jd[:Nobs_rows] @ X
        V = Y.T @ Y
    else:
        V = A @ X
    N = dF_dbpacked.shape[0]
    out = np.zeros((N, 2, 2))
    for i in range(N):
        out[i] = V[2 * i:2 * i + 2, 2 * i:2 * i + 2]
    return sigma * sigma * out, np.linalg.cond(JtJ)
