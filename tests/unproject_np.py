"""A numpy restatement of mrcal.unproject(normalize=, get_gradients=) (mrcal/projections.py:112-397),
mrcal.model_resolution__deg_pixel() (mrcal/model_analysis.py:2152-2246) and the reprojection of mrcal.stereo_pair_diff()
(:1931-2103), built on the compiled reference (oracle/_ref): its mrcal_project() with both gradients, its iterative
unprojection (oracle/ref.py unproject()) and its closed-form mrcal_project_* / mrcal_unproject_* (mrcal.c:1436-1880)."""
import ctypes as C

import numpy as np

from oracle import ref

CLOSED_FORM = {"LENSMODEL_PINHOLE": "pinhole", "LENSMODEL_STEREOGRAPHIC": "stereographic",
               "LENSMODEL_LONLAT": "lonlat", "LENSMODEL_LATLON": "latlon"}
IDENTITY = np.array((1., 1., 0., 0.))


def closed_form(fn, kind, x, fxycxy=IDENTITY):
    """The reference's mrcal_<fn>_<kind>() with its gradient: fn 'project' (x (N,3) -> q (N,2), dq_dv (N,2,3)) or
    'unproject' (x (N,2) -> v (N,3), dv_dq (N,3,2))"""
    nin, nout = (3, 2) if fn == "project" else (2, 3)
    x = np.ascontiguousarray(x, np.float64).reshape(-1, nin)
    out, g = np.zeros((x.shape[0], nout)), np.zeros((x.shape[0], nout, nin))
    f = getattr(ref.lib(), f"mrcal_{fn}_{kind}")
    f.restype = None
    fxycxy = np.ascontiguousarray(fxycxy, np.float64)
    # one point per call: with N > 1 mrcal_project_pinhole() writes every q into the first slot (mrcal.c:1458-1459)
    for i in range(x.shape[0]):
        o, gi, xi = np.zeros(nout), np.zeros((nout, nin)), np.ascontiguousarray(x[i])
        f(ref._dp(o), ref._dp(gi), ref._dp(xi), C.c_int(1), ref._dp(fxycxy))
        out[i], g[i] = o, gi
    return out, g


def _normalize(v, dv_dq, dv_di):
    """mrcal/projections.py:220-247"""
    r = 1. / np.linalg.norm(v, axis=-1, keepdims=True)
    v = v * r

    def proj(d):
        d = d * r[..., None]
        return d - v[..., :, None] * np.einsum("ni,nij->nj", v, d)[:, None, :]
    return v, proj(dv_dq), proj(dv_di)


def unproject(q, lm, intr, normalize=False, get_gradients=False, behind_ok=False):
    """v (N,3) [, dv_dq (N,3,2), dv_dintrinsics (N,3,Nintrinsics)] of pixels q (N,2). behind_ok: the model can project
    behind the camera (otherwise a ray found behind it is flipped to the front, mrcal.c:3263-3270)"""
    q = np.ascontiguousarray(q, np.float64).reshape(-1, 2)
    intr = np.asarray(intr, np.float64)
    if lm in CLOSED_FORM:
        kind = CLOSED_FORM[lm]
        v, dv_dq = closed_form("unproject", kind, q, intr)
        unit = kind in ("lonlat", "latlon")
        if not get_gradients:
            return v / np.linalg.norm(v, axis=-1, keepdims=True) if normalize and not unit else v
        # q = f l(v) + c: dv/df = (c - q)/f dv/dq, dv/dc = -dv/dq
        dv_di = np.zeros((q.shape[0], 3, 4))
        dv_di[..., :2] = ((intr[2:4] - q) / intr[:2])[:, None, :] * dv_dq
        dv_di[..., 2:] = -dv_dq
        if normalize and not unit:
            return _normalize(v, dv_dq, dv_di)
        return v, dv_dq, dv_di
    vs = ref.unproject(q, lm, intr)
    if not behind_ok:
        vs[vs[:, 2] < 0] *= -1.
    if not get_gradients:
        if not normalize:
            return vs
        good = np.isfinite(vs).all(-1)
        out = np.zeros_like(vs)
        out[good] = vs[good] / np.linalg.norm(vs[good], axis=-1, keepdims=True)
        return out
    # q -> vs -> u -> v
    u, _ = closed_form("project", "stereographic", vs)
    v, dv_du = closed_form("unproject", "stereographic", u)
    _, dq_dv, dq_di = ref.project_with_intrinsics_gradient(v, lm, intr)
    dq_du = dq_dv @ dv_du
    dv_dq = dv_du @ np.linalg.inv(dq_du)
    dv_di = -dv_dq @ dq_di
    if normalize:
        return _normalize(v, dv_dq, dv_di)
    return v, dv_dq, dv_di


def perpendicular_basis(v):
    """(N,3,2): an orthonormal basis of the plane perpendicular to each unit vector v (N,3), from the SVD"""
    return np.linalg.svd(np.eye(3)[None] - v[:, :, None] * v[:, None, :])[0][..., :2]


def resolution_from_M(M, mode):
    """The reference's closed-form eigenvalues of M'M (model_analysis.py:2221-2246)"""
    a = (M[..., :, 0] * M[..., :, 0]).sum(-1)
    b = (M[..., :, 0] * M[..., :, 1]).sum(-1)
    c = (M[..., :, 1] * M[..., :, 1]).sum(-1)
    sd = np.sqrt((a - c) * (a - c) / 4 + b * b)
    lmax = (a + c) / 2 + sd
    lmin = (a + c) / 2 - sd
    lmin[lmin < 1e-6] = 1e-6
    rmax = 1. / np.sqrt(lmin) * 180. / np.pi
    rmin = 1. / np.sqrt(lmax) * 180. / np.pi
    return {"min": rmin, "max": rmax, "eccentricity": rmax / rmin, "mean": (rmin + rmax) / 2.}[mode]


def resolution_M(q, lm, intr, behind_ok=False):
    """M = dq/dv [u0 u1] (N,2,2) at the unit rays of pixels q (N,2)"""
    v = unproject(q, lm, intr, normalize=True, behind_ok=behind_ok)
    _, dq_dv, _ = ref.project_with_intrinsics_gradient(v, lm, intr)
    return dq_dv @ perpendicular_basis(v)


def model_resolution(q, lm, intr, mode, behind_ok=False):
    return resolution_from_M(resolution_M(q, lm, intr, behind_ok), mode)


def reproject(q, lm0, intr0, lm1, intr1, Rt10, distance, behind_ok0=False):
    """project_1(R (distance unproject_0(q, normalized)) + t)"""
    p = distance * unproject(q, lm0, intr0, normalize=True, behind_ok=behind_ok0)
    return ref.project(p @ Rt10[:3].T + Rt10[3], lm1, intr1)
