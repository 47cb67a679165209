"""Without a GPU: the extended-precision reference of test_board_sizes_gpu.py against the float64 ones, and the coverage
each of that file's problems claims, from the compiled reference's Jacobian (oracle/_ref). A change to the synthetic
problems that loses a case fails here."""
import numpy as np
import pytest
import scipy.linalg

import board_sizes as bs
import problems

SMALL = ["opencv8_2cam_all", "splined3_2cam_corelocked", "splined2_2cam_corelocked", "opencv8_noreg_outliers",
         "opencv8_points", "opencv4_unity"]


def scipy_reduced(J, x, e0, e1, lam):
    """S and g' with the eliminated block solved through its float64 Cholesky factor (scipy)"""
    Jd = J.toarray()
    H = Jd.T @ Jd + lam * np.eye(Jd.shape[1])
    g = Jd.T @ x
    n = H.shape[0]
    sh, el = np.r_[0:e0, e1:n], np.r_[e0:e1]
    el = el[np.any(H[el] != 0, axis=1)]
    A, B, D = H[np.ix_(sh, sh)], H[np.ix_(sh, el)], H[np.ix_(el, el)]
    c = scipy.linalg.cho_factor(D, lower=True)
    return A - B @ scipy.linalg.cho_solve(c, B.T), g[sh] - B @ scipy.linalg.cho_solve(c, g[el])


@pytest.mark.parametrize("name", SMALL)
@pytest.mark.parametrize("lam", [0.0, 1e-3])
def test_longdouble_reference_matches_float64(ref, name, lam):
    kw = dict(problems.golden_cases())[name]
    P = ref.Problem(kw)
    b, x, J = P.callback()
    S, g, gfull, scale = bs.reduced_reference_ld(J, x, P, lam)
    e0, e1, sizes = bs.eliminated_groups(P)
    assert sum(sizes) == e1 - e0 > 0
    S2, g2, gfull2, scale2 = problems.reduced_reference(J, x, e0, e1, lam)
    S3, g3 = scipy_reduced(J, x, e0, e1, lam)
    assert abs(scale - scale2) <= 1e-14 * scale2
    gs = np.abs(gfull).max()
    assert np.abs(gfull - gfull2).max() <= 1e-13 * gs
    for Sx, gx in ((S2, g2), (S3, g3)):
        assert np.abs(S - Sx).max() <= 1e-12 * scale
        assert np.abs(g - gx).max() <= 1e-12 * gs


@pytest.mark.parametrize("name", SMALL)
def test_longdouble_cauchy_reference(ref, name):
    kw = dict(problems.golden_cases())[name]
    b, x, J = ref.Problem(kw).callback()
    g2, Jg2 = bs.cauchy_reference_ld(J, x)
    g = J.T @ x
    assert abs(g2 - g @ g) <= 1e-13 * g2
    assert abs(Jg2 - np.sum((J @ g) ** 2)) <= 1e-12 * Jg2


def test_eval_sizes_cover_every_kernel_path():
    """100 corners (today's largest), one full chunk of 128, 160 threads with a partial last warp, one full chunk of 256,
    two chunks with a second of 4 corners and of 144"""
    got = [(W * H, bs.eval_threads(W * H), bs.eval_chunks(W * H), W * H - (bs.eval_chunks(W * H) - 1) * bs.eval_threads(W * H))
           for W, H in bs.EVAL_SHAPES]
    assert got == [(100, 128, 1, 100), (128, 128, 1, 128), (132, 160, 1, 132), (256, 256, 1, 256), (260, 256, 2, 4),
                   (400, 256, 2, 144)]
    assert set(bs.EVAL_LENSES) == {"opencv8", "splined3_corelocked", "splined3_core"}


@pytest.mark.parametrize("name,W,H,kw", bs.eval_cases(), ids=[c[0] for c in bs.eval_cases()])
def test_eval_cases_have_their_shape(ref, name, W, H, kw):
    P = ref.Problem(kw)
    assert (P.W, P.H, P.Ncam_i, P.Nobs_board) == (W, H, 2, 6)
    lm, core = bs.EVAL_LENSES[name.rsplit("_", 1)[0]]
    assert kw["lensmodel"] == lm and kw["do_optimize_intrinsics_core"] == core


def test_fused_shared_memory():
    """the sizes of the fused kernel's shared memory: 112 corners fit in the 110 KB it was limited to, 113 to 128 do not,
    and every size fits in what one H100 block may have (227 KB)"""
    assert bs.fused_smem_bytes(bs.fused_K(112)) == 111776 <= 110 * 1024
    for nwh, need in ((113, 115104), (114, 115104), (121, 121760), (128, 125088)):
        assert bs.fused_smem_bytes(bs.fused_K(nwh)) == need > 110 * 1024
    assert bs.fused_smem_bytes(bs.fused_K(128)) <= 227 * 1024


@pytest.mark.parametrize("name", list(bs.FUSED))
def test_fused_cases_have_their_coverage(ref, name):
    c = bs.FUSED[name]
    kw = bs.fused_case(name)
    P = ref.Problem(kw)
    b, x, J = P.callback()
    nwh = P.W * P.H
    assert nwh <= 128 and (P.W, P.H) == (c["W"], c["H"])
    # the fused path's problem: splined, the core locked, the distortions and frames optimized
    assert kw["lensmodel"].startswith("LENSMODEL_SPLINED") and not kw["do_optimize_intrinsics_core"]
    assert kw["do_optimize_intrinsics_distortions"] and kw["do_optimize_frames"]
    claims = c["claims"]
    K = bs.fused_K(nwh)
    if "pad" in claims:
        assert K - nwh == claims["pad"]
    if "fits" in claims:
        assert (bs.fused_smem_bytes(K) <= 110 * 1024) == claims["fits"]
    nk = bs.observation_knots(P, kw, J)
    assert max(nk) <= 64, nk   # nothing here takes the fallback
    if "nk" in claims:
        lo, hi = claims["nk"]
        assert lo <= max(nk) <= hi, nk
        if hi < 64:
            assert max(nk) % 8 != 0, nk   # the last 8x8 tile partly filled
    extr = bs.observation_columns(P, J, "extrinsics")
    warp = bs.observation_columns(P, J, "calobject_warp")
    assert (max(extr) == 0) == claims.get("ncam0", False), extr
    assert (max(warp) == 0) == claims.get("nwarp0", False), warp
    free = bs.unconstrained_frames(P, J)
    if claims.get("outlier_frame", False):
        assert free == [P.Nframes - 1]
        last = np.flatnonzero(P.indices_board[:, 0] == P.Nframes - 1)
        assert len(last) == 1 and np.all(P.observations_board[last[0], ..., 2] < 0)
    else:
        assert free == []


def test_fallback_case_needs_the_fallback(ref):
    kw = bs.fallback_case()
    P = ref.Problem(kw)
    b, x, J = P.callback()
    assert P.W * P.H <= 128 and not kw["do_optimize_intrinsics_core"]
    assert max(bs.observation_knots(P, kw, J)) >= 65


def test_solve121_case_takes_the_fused_path(ref):
    kw = bs.solve121_case()
    P = ref.Problem(kw)
    b, x, J = P.callback()
    assert P.W * P.H == 121 and not kw["do_optimize_intrinsics_core"]
    assert max(bs.observation_knots(P, kw, J)) <= 64
