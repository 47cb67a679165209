"""projection_uncertainty() on the GPU (mrcal_b200/csrc/uncertainty.cu) against the numpy restatement of
tests/uncertainty_np.py: a dense solve of J'J and Jo'Jo over the leading observation rows, fed either the compiled
reference's own Jacobian, K and projection gradients (oracle/_ref) or this library's. Gate, as in
test_factorization_gpu.py:  |Var - Var_ref| <= max(1e-8, 64 eps cond(J'J)) max|Var_ref|."""
import os
import tempfile

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import synthetic
import uncertainty_np as unp

pytestmark = pytest.mark.gpu

SPL = "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=11_Ny=8_fov_x_deg=150"
METHODS = ("mean-pcam", "cross-reprojection-rrp-Jfp", "cross-reprojection-ccp")


def _clone(kw):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}


def _solved(**args):
    kw, _ = synthetic.make_problem(**args)
    mrcal_b200.optimize(**kw)
    return kw


def _query_points(kw, icam, n=12, dist=10., seed=0):
    rng = np.random.default_rng(seed)
    W, H = kw["imagersizes"][icam]
    q = np.stack((rng.uniform(0.1 * W, 0.9 * W, n), rng.uniform(0.1 * H, 0.9 * H, n)), -1)
    v = mrcal_b200.unproject(q, kw["lensmodel"], kw["intrinsics"][icam])
    v = v[np.isfinite(v).all(axis=-1)]   # (pixels outside the lens's field of view unproject to NaN)
    assert len(v) >= n // 2
    return dist * v / np.linalg.norm(v, axis=-1)[..., None]


def _camera_extrinsics(kw, icam):
    e = []
    for name in ("indices_frame_camintrinsics_camextrinsics", "indices_point_camintrinsics_camextrinsics"):
        a = kw.get(name)
        if a is not None and len(a):
            e += list(a[a[:, 1] == icam, 2])
    return np.unique(e)


def _expected(kw, icam, method, atinfinity, pts, sigma, source):
    """Var from the restatement; source = (J, x, K(icam), project(p, intr) -> (dq_dp, dq_di), D)"""
    rows, s, Nobs = _rows(kw, icam, method, atinfinity, pts, sigma, source)
    Var, cond = unp.propagate(rows, source[0], Nobs if Nobs < source[0].shape[0] else source[0].shape[0], s)
    return Var, s, cond


def _rows(kw, icam, method, atinfinity, pts, sigma, source):
    """dF/db_packed (N, 2, Nstate) of the restatement, the sigma, and the number of board/point measurements"""
    J, x, Kfun, proj, D = source
    Nstate = J.shape[1]
    Nobs = mrcal_b200.num_measurements_boards(**kw) + mrcal_b200.num_measurements_points(**kw)
    i_intr = mrcal_b200.state_index_intrinsics(icam, **kw)
    Nis = mrcal_b200.num_intrinsics_optimization_params(**kw)
    intr_cols = [] if i_intr is None else list(range(i_intr, i_intr + Nis))
    intr_arg0 = 0 if kw.get("do_optimize_intrinsics_core", True) else 4
    e = _camera_extrinsics(kw, icam)
    rt_cam = None if e[0] < 0 else kw["rt_cam_ref"][e]
    extr_col0 = None if e[0] < 0 else mrcal_b200.state_index_extrinsics(int(e[0]), **kw)
    frame_col0 = mrcal_b200.state_index_frames(0, **kw)
    rt_frames = kw.get("rt_ref_frame")
    K = None if method == "mean-pcam" else Kfun(icam if method == "cross-reprojection-ccp" else -1)
    dq_dp, dq_di = proj(pts, kw["intrinsics"][icam])
    rows = np.zeros((len(pts), 2, Nstate))
    for i, p in enumerate(pts):
        A, G = unp.dq_db_unpacked(p, dq_dp[i], dq_di[i], method=method, atinfinity=atinfinity, Nstate=Nstate,
                                  intr_cols=intr_cols, intr_arg0=intr_arg0, rt_cam=rt_cam, extr_col0=extr_col0,
                                  rt_frames=rt_frames, frame_col0=frame_col0)
        rows[i] = A * D + (G @ K if K is not None else 0.)
    s = unp.sigma_estimate(x[:Nobs], Nstate) if sigma is None else sigma
    return rows, s, Nobs


def _self_source(kw):
    P = mrcal_b200.Problem(**_clone(kw))
    b, x, J = P.callback()
    D = np.ones(J.shape[1])
    mrcal_b200.unpack_state(D, **kw)

    def proj(p, intr):
        _, g, gi = mrcal_b200.project(p, kw["lensmodel"], intr, get_gradients=True)
        return g, gi
    return (J, x, lambda icam: P.drt_cross_reprojection__dbpacked(icam), proj, D), P


def _ref_source(ref, kw):
    R = ref.Problem(_clone(kw))
    b, x, J = R.callback()
    D = R.unpack_vector(np.ones(J.shape[1]))

    def proj(p, intr):
        _, g, gi = ref.project_with_intrinsics_gradient(p, kw["lensmodel"], intr)
        return g, gi
    return (J, x, lambda icam: R.drt_cross_reprojection__dbpacked(icam)[0], proj, D)


def _gate(Var, Var_ref, cond):
    tol = max(1e-8, 64 * np.finfo(float).eps * cond) * np.abs(Var_ref).max()
    err = np.abs(Var - Var_ref).max()
    assert err <= tol, (err, tol)


def _cases():
    out = []
    # parametric: camera 1's observations touch all of its shared columns
    for reg in (True, False):
        for method in METHODS:
            for icam in ((0, 1) if reg else (1,)):
                for inf in ((False, True) if reg else (False,)):
                    out.append(("LENSMODEL_OPENCV4", 3, reg, method, icam, inf))
    for method in METHODS:
        for icam in (0, 1):
            for inf in (False, True):
                out.append((SPL, 3, True, method, icam, inf))
    for method in METHODS:
        out.append((SPL, 2, True, method, 1, False))
    return out


_PROBLEMS = {}


def _problem(lensmodel, Ncameras, reg):
    key = (lensmodel, Ncameras, reg)
    if key not in _PROBLEMS:
        _PROBLEMS[key] = _solved(lensmodel=lensmodel, Ncameras=Ncameras, Nframes=10, W=6, H=5, seed=3, pixel_noise=0.3)
        if not reg:
            _PROBLEMS[key]["do_apply_regularization"] = False
            mrcal_b200.optimize(**_PROBLEMS[key])
    return _PROBLEMS[key]


@pytest.mark.parametrize("lensmodel,Ncameras,reg,method,icam,atinfinity", _cases())
def test_against_restatement(ref, lensmodel, Ncameras, reg, method, icam, atinfinity):
    """the reference's J, K and projection gradients, composed by the dense restatement; camera 0 is at the reference,
    camera 1 has extrinsics; sigma estimated, and given"""
    kw = _problem(lensmodel, Ncameras, reg)
    pts = _query_points(kw, icam)
    src = _ref_source(ref, kw)
    P = mrcal_b200.Problem(**_clone(kw))
    for sigma in (None, 0.25):
        Var, s = P.projection_uncertainty(pts, icam, method=method, atinfinity=atinfinity, observed_pixel_uncertainty=sigma)
        Var_ref, s_ref, cond = _expected(kw, icam, method, atinfinity, pts, sigma, src)
        assert abs(s - s_ref) <= 1e-12 * s_ref
        _gate(Var, Var_ref, cond)
    P.close()


@pytest.mark.parametrize("method", ["cross-reprojection-rrp-Jfp", "cross-reprojection-ccp"])
def test_points_only(ref, method):
    # (the first of these seeds whose solution has a positive definite J'J: a point seen at grazing angles by two
    # cameras only can leave it singular, and then there is no uncertainty to compute, here as in the reference)
    for seed in (5, 6, 7, 8):
        kw, _ = synthetic.make_problem(lensmodel=SPL, Ncameras=3, Nframes=2, W=6, H=5, seed=seed,
                                       pixel_noise=0.2, Npoints=120, Npoints_fixed=3, which="all")
        for k in ("observations_board", "indices_frame_camintrinsics_camextrinsics", "rt_ref_frame", "calobject_warp"):
            kw.pop(k, None)
        kw["do_optimize_calobject_warp"] = False
        mrcal_b200.optimize(**kw)
        if mrcal_b200.optimizer_callback(**_clone(kw))[3] is not None:
            break
    # (sigma is given: the points alone leave too few measurements per unknown for the residual estimate)
    for icam in (0, 2):
        pts = _query_points(kw, icam)
        Var, _ = mrcal_b200.Problem(**_clone(kw)).projection_uncertainty(pts, icam, method=method, observed_pixel_uncertainty=0.3)
        Var_ref, _, cond = _expected(kw, icam, method, False, pts, 0.3, _ref_source(ref, kw))
        _gate(Var, Var_ref, cond)
    with pytest.raises(RuntimeError, match="only cross-reprojection uncertainty can work here"):
        mrcal_b200.Problem(**_clone(kw)).projection_uncertainty(pts, 0, method="mean-pcam")


def test_config3_grid():
    """config 3 size, the 60 x 33 grid: 20 points against the restatement fed this library's own primitives; every
    2x2 symmetric positive definite; two calls bit-identical"""
    kw, _ = synthetic.baseline_config(3, pixel_noise=0.3)
    mrcal_b200.optimize(**kw)
    icam = 1
    W, H = kw["imagersizes"][icam]
    qx, qy = np.meshgrid(np.linspace(0, W - 1, 60), np.linspace(0, H - 1, 33))
    v = mrcal_b200.unproject(np.stack((qx, qy), -1), kw["lensmodel"], kw["intrinsics"][icam])
    pts = (10. * v / np.linalg.norm(v, axis=-1)[..., None]).reshape(-1, 3)
    src, P = _self_source(kw)
    Var, s = P.projection_uncertainty(pts, icam)
    Var2, s2 = P.projection_uncertainty(pts, icam)
    assert np.array_equal(Var, Var2, equal_nan=True) and s == s2
    assert np.array_equal(Var[:, 0, 1], Var[:, 1, 0], equal_nan=True)
    # (grid corners outside the lens's field of view unproject to NaN)
    ok = np.isfinite(pts).all(axis=-1)
    assert ok.sum() > 0.9 * len(pts) and np.isfinite(Var[ok]).all()
    V = Var[ok]
    assert (V[:, 0, 0] > 0).all() and (V[:, 0, 0] * V[:, 1, 1] - V[:, 0, 1] ** 2 > 0).all()
    sel = np.flatnonzero(ok)[np.linspace(0, ok.sum() - 1, 20).astype(int)]
    # the reference's algorithm from this library's primitives: solve_xt_JtJ_bt, then _A_Jt_J_At over the leading rows
    rows, s_ref, Nobs = _rows(kw, icam, "cross-reprojection-ccp", False, pts[sel], None, src)
    _, _, J, F = mrcal_b200.optimizer_callback(**_clone(kw))
    X = F.solve_xt_JtJ_bt(rows)
    Var_ref = mrcal_b200._A_Jt_J_At__2(X, J.indptr, J.indices, J.data, Nleading_rows_J=Nobs) * s_ref ** 2
    assert abs(s - s_ref) <= 1e-12 * s_ref
    _gate(Var[sel], Var_ref, 1. / F.rcond())


def _model(kw, icam):
    return mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=icam)


def test_api_shapes_and_file_roundtrip():
    kw = _problem(SPL, 3, True)
    m = _model(kw, 1)
    pts = _query_points(kw, 1, n=6).reshape(2, 3, 3)
    V = mrcal_b200.projection_uncertainty(pts, m)
    assert V.shape == (2, 3, 2, 2)
    w = mrcal_b200.projection_uncertainty(pts, m, what="worstdirection-stdev")
    r = mrcal_b200.projection_uncertainty(pts, m, what="rms-stdev")
    assert w.shape == r.shape == (2, 3)
    ev = np.linalg.eigvalsh(V)
    assert np.allclose(w, np.sqrt(ev[..., -1]), rtol=1e-12)
    assert np.allclose(r, np.sqrt((V[..., 0, 0] + V[..., 1, 1]) / 2), rtol=1e-15)
    assert mrcal_b200.projection_uncertainty(pts[0, 0], m).shape == (2, 2)
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "cam1.cameramodel")
        m.write(f)
        V2 = mrcal_b200.projection_uncertainty(pts, mrcal_b200.cameramodel(f))
    assert np.allclose(V2, V, rtol=1e-9, atol=0)


def test_refusals():
    kw = _problem(SPL, 3, True)
    m = _model(kw, 1)
    p = np.array((0.1, 0.2, 5.))
    with pytest.raises(RuntimeError, match="Unknown uncertainty method"):
        mrcal_b200.projection_uncertainty(p, m, method="nope")
    with pytest.raises(RuntimeError, match="'what' kwarg must be in"):
        mrcal_b200.projection_uncertainty(p, m, what="nope")
    bare = mrcal_b200.cameramodel(intrinsics=m.intrinsics(), imagersize=m.imagersize())
    with pytest.raises(RuntimeError, match="optimization_inputs are unavailable"):
        mrcal_b200.projection_uncertainty(p, bare)
    # a moving camera: camera 1's observations split over extrinsics 0 and 1, or over the reference and extrinsics 0
    for e_new, msg in ((1, None), (-1, "some poses are at the reference")):
        kw2 = _clone(kw)
        idx = kw2["indices_frame_camintrinsics_camextrinsics"]
        sel = np.flatnonzero(idx[:, 1] == 1)
        idx[sel[::2], 2] = e_new
        P = mrcal_b200.Problem(**kw2)
        if msg:
            with pytest.raises(RuntimeError, match=msg):
                P.projection_uncertainty(p[None], 1, method="mean-pcam")
        else:
            with pytest.raises(RuntimeError, match="I only handle stationary cameras for now"):
                P.projection_uncertainty(p[None], 1, method="cross-reprojection-rrp-Jfp")

    # triangulated observations: measurements other than boards, points and regularization
    import problems
    kw2 = _clone(kw)
    kw2["do_optimize_intrinsics_core"] = kw2["do_optimize_intrinsics_distortions"] = False
    problems.add_triangulated_points(kw2, dict(rt_cam_ref=kw2["rt_cam_ref"]), 4, seed=1, outliers=0)
    with pytest.raises(RuntimeError, match="Some measurements other than boards, points and regularization"):
        mrcal_b200.Problem(**kw2).projection_uncertainty(p[None], 1, method="cross-reprojection-ccp")


def test_ccp_ignores_the_extrinsics_block():
    """ccp looks only at the camera frame (model_analysis.py:1347-1417): a camera seen from the reference and from an
    extrinsics pose is accepted by ccp, refused by mean-pcam"""
    kw = _clone(_problem(SPL, 3, True))
    idx = kw["indices_frame_camintrinsics_camextrinsics"]
    sel = np.flatnonzero(idx[:, 1] == 1)
    idx[sel[::2], 2] = -1
    P = mrcal_b200.Problem(**kw)
    p = np.array((0.1, 0.2, 5.))
    Var, _ = P.projection_uncertainty(p[None], 1, method="cross-reprojection-ccp")
    assert np.isfinite(Var).all() and Var[0, 0, 0] > 0
    with pytest.raises(RuntimeError, match="some poses are at the reference"):
        P.projection_uncertainty(p[None], 1, method="mean-pcam")
