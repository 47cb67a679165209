"""The Schur-reduced normal equations built on the GPU (normal.cu) against the same
quantities computed with numpy from the CUDA path's own Jacobian (which
test_callback_gpu.py ties to the reference)."""
import numpy as np
import pytest

import mrcal_b200
import problems
from mrcal_b200 import synthetic

pytestmark = pytest.mark.gpu


def reduced_reference(J, x, e0, e1, lam=0.0):
    Jd = J.toarray()
    H = Jd.T @ Jd + lam * np.eye(Jd.shape[1])
    g = Jd.T @ x
    n = H.shape[0]
    sh = np.r_[0:e0, e1:n]
    el = np.r_[e0:e1]
    if len(el) == 0:
        return H, g, g, np.abs(H).max()
    # eliminated unknowns nothing constrains (a point seen only by outlier observations, at lambda = 0) have zero rows
    # in J'J: they couple to nothing, so they drop out of the elimination -- the device leaves them out the same way
    # instead of inverting their zero block
    free = ~np.any(H[el] != 0, axis=1)
    el = el[~free]
    A, B, D = H[np.ix_(sh, sh)], H[np.ix_(sh, el)], H[np.ix_(el, el)]
    assert np.linalg.cond(D) < 1e12, "the constrained part of the eliminated block is singular"
    Dinv = np.linalg.inv(D)
    # S is a difference of two nearly equal terms: the achievable accuracy is relative to |A|
    return A - B @ Dinv @ B.T, g[sh] - B @ Dinv @ g[el], g, (np.abs(A).max() if A.size else 1.)


CASES = [c for c in problems.golden_cases() if c[0] in (
    "opencv8_2cam_all", "opencv8_frames_only", "opencv8_intrinsics_only", "opencv8_extrinsics_warp",
    "splined3_2cam_corelocked", "splined3_3cam_all", "splined2_2cam_corelocked", "opencv8_points",
    "opencv8_points_fixed", "splined3_points_core", "opencv4_unity", "pinhole_points_noframes", "opencv8_1cam")]


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("lam", [0.0, 1e-3])
def test_reduced_system(name, kw, lam):
    P = mrcal_b200.Problem(**kw)
    b, x, J = P.callback()
    S, g, gfull = P.reduced_system(lam)
    fr0 = mrcal_b200.state_index_frames(0, **kw)
    pt0 = mrcal_b200.state_index_points(0, **kw)
    e0 = fr0 if fr0 is not None else (pt0 if pt0 is not None else P.Nstate)
    e1 = e0 + mrcal_b200.num_states_frames(**kw) * (fr0 is not None) + mrcal_b200.num_states_points(**kw) * (pt0 is not None)
    S_ref, g_ref, gfull_ref, scale = reduced_reference(J, x, e0, e1, lam)
    assert np.abs(gfull - gfull_ref).max() <= 1e-10 * np.abs(gfull_ref).max(), "J'x"
    assert S.shape == S_ref.shape
    if S_ref.size:
        # the device system covers the ACTIVE shared unknowns (those some observation touches); the
        # rest appear only in their own regularization blocks and must be decoupled from the active ones
        act = np.diag(S) != 0
        assert act.sum() > 0
        assert np.abs(S_ref[np.ix_(~act, act)]).max(initial=0.) == 0.
        assert np.abs(S[np.ix_(act, act)] - S_ref[np.ix_(act, act)]).max() <= 1e-9 * scale, "S"
        assert np.abs(g[act] - g_ref[act]).max() <= 1e-9 * np.abs(gfull_ref).max(), "g'"
        if "splined" in name and "core" not in name and lam == 0.0:
            assert (~act).sum() > 0, "expected untouched knots in this case"
