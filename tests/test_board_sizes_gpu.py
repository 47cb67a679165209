"""The board kernels at every board size where they change path, against the compiled reference (oracle/_ref):

- the cost function (eval.cu's eval_boards_kernel) at 100 to 400 corners: one chunk of 128, 160 or 256 threads, and two
  chunks that reuse the staging buffer;
- the reduced normal equations on the stored-Jacobian path at those sizes, and on the fused path (fused_eval.cu) at the
  padding, patch-width and column-set edges of its kernel, including the boards of 113 to 128 corners, each against an
  extended-precision reference built from the reference's J and x (tests/board_sizes.py);
- the fused kernel's give-up on patches of more than 64 knots, and the solve that then continues on the stored path;
- the sums of the Cauchy step, |g|^2 and |J g|^2, on both paths.

The cases and the coverage each claims are in tests/board_sizes.py; test_board_sizes_cpu.py checks the claims."""
import numpy as np
import pytest

import board_sizes as bs
import mrcal_b200

pytestmark = pytest.mark.gpu
TOL = 1e-9

EVAL = bs.eval_cases()
FUSED = list(bs.FUSED)


def assert_close(a, b, what, tol=TOL):
    err = np.abs(np.asarray(a) - np.asarray(b)) / (1. + np.abs(b))
    assert err.size == 0 or err.max() <= tol, f"{what}: worst relative-to-scale error {err.max():.3g} at {err.argmax()}"


@pytest.mark.parametrize("name,W,H,kw", EVAL, ids=[c[0] for c in EVAL])
def test_callback_matches_reference(ref, name, W, H, kw):
    """x, J and the CSR structure at test_callback_gpu.py's gate; the no_jacobian path gives the same x"""
    b_ref, x_ref, J_ref = ref.Problem(kw).callback()
    b, x, J, _ = mrcal_b200.optimizer_callback(**kw, no_factorization=True)
    assert np.array_equal(J.indptr, J_ref.indptr) and np.array_equal(J.indices, J_ref.indices)
    assert_close(b, b_ref, "b_packed")
    assert_close(x, x_ref, "x")
    assert_close(J.data, J_ref.data, "J values")
    _, x2, J2, _ = mrcal_b200.optimizer_callback(**kw, no_jacobian=True, no_factorization=True)
    assert J2 is None
    assert np.allclose(x, x2, rtol=1e-13, atol=1e-12)


def check_reduced(S, g, gfull, S_ref, g_ref, gfull_ref, scale):
    """test_normal_gpu.py's gates"""
    assert np.abs(gfull - gfull_ref).max() <= 1e-10 * np.abs(gfull_ref).max(), "J'x"
    assert S.shape == S_ref.shape
    # the device system covers the shared unknowns some observation touches; the others must be decoupled
    act = np.diag(S) != 0
    assert act.sum() > 0
    assert np.abs(S_ref[np.ix_(~act, act)]).max(initial=0.) == 0.
    assert np.abs(S[np.ix_(act, act)] - S_ref[np.ix_(act, act)]).max() <= 1e-9 * scale, "S"
    assert np.abs(g[act] - g_ref[act]).max() <= 1e-9 * np.abs(gfull_ref).max(), "g'"


def reference(ref, kw):
    P = ref.Problem(kw)
    b, x, J = P.callback()
    return P, x, J


@pytest.mark.parametrize("name,W,H,kw", EVAL, ids=[c[0] for c in EVAL])
def test_reduced_system_stored_path(ref, name, W, H, kw):
    Pr, x_ref, J_ref = reference(ref, kw)
    P = mrcal_b200.Problem(**kw)
    for lam in (0.0, 1e-3):
        check_reduced(*P.reduced_system(lam), *bs.reduced_reference_ld(J_ref, x_ref, Pr, lam))
    fused_path = "corelocked" in name
    if fused_path and W * H <= 128:
        for lam in (0.0, 1e-3):
            check_reduced(*P.reduced_system(lam, fused=True), *bs.reduced_reference_ld(J_ref, x_ref, Pr, lam))
    elif fused_path:
        with pytest.raises(RuntimeError, match="does not take the fused evaluation"):
            P.reduced_system(0.0, fused=True)
        with pytest.raises(RuntimeError, match="does not take the fused evaluation"):
            P.cauchy_denominator(fused=True)


@pytest.mark.parametrize("name", FUSED)
@pytest.mark.parametrize("lam", [0.0, 1e-3])
def test_reduced_system_fused_path(ref, name, lam):
    kw = bs.fused_case(name)
    Pr, x_ref, J_ref = reference(ref, kw)
    want = bs.reduced_reference_ld(J_ref, x_ref, Pr, lam)
    P = mrcal_b200.Problem(**kw)
    check_reduced(*P.reduced_system(lam, fused=True), *want)
    check_reduced(*P.reduced_system(lam), *want)


def check_cauchy(P, fused, J_ref, x_ref):
    g2_ref, Jg2_ref = bs.cauchy_reference_ld(J_ref, x_ref)
    g2, Jg2 = P.cauchy_denominator(fused=fused)
    assert abs(g2 - g2_ref) <= 1e-9 * g2_ref, (g2, g2_ref)
    assert abs(Jg2 - Jg2_ref) <= 1e-9 * Jg2_ref, (Jg2, Jg2_ref)


@pytest.mark.parametrize("name", FUSED)
def test_cauchy_denominator_fused_path(ref, name):
    """quadform_items_kernel over the board observations' blocks plus jv_kernel over the other rows, and jv_kernel alone"""
    kw = bs.fused_case(name)
    Pr, x_ref, J_ref = reference(ref, kw)
    P = mrcal_b200.Problem(**kw)
    check_cauchy(P, True, J_ref, x_ref)
    check_cauchy(P, False, J_ref, x_ref)


@pytest.mark.parametrize("name,W,H,kw", EVAL, ids=[c[0] for c in EVAL])
def test_cauchy_denominator_stored_path(ref, name, W, H, kw):
    Pr, x_ref, J_ref = reference(ref, kw)
    check_cauchy(mrcal_b200.Problem(**kw), False, J_ref, x_ref)


def _clone(kw):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}


def check_solve(ref, kw, capfd, fallback):
    """optimize() against the reference's mrcal_optimize() at test_solve_golden.py's gates for the splined solves"""
    rr = ref.Problem(_clone(kw)).optimize()
    capfd.readouterr()
    r = mrcal_b200.optimize(**_clone(kw))
    err = capfd.readouterr().err
    assert err.count("more control points") == (1 if fallback else 0), err
    norm2 = float(r["x"] @ r["x"])
    assert abs(norm2 - rr["norm2_x"]) <= 1e-9 * rr["norm2_x"], (norm2, rr["norm2_x"])
    assert abs(r["rms_reproj_error__pixels"] - rr["rms_reproj_error__pixels"]) <= 1e-7
    assert np.abs(r["b_packed"] - rr["b_packed"]).max() <= 2e-3


def test_fallback_when_a_patch_is_too_wide(ref, capfd):
    """An observation touching more than 64 knots: the fused evaluation gives up, reduced_system(fused=True) says so, and
    optimize() says so once and finishes on the stored-Jacobian path"""
    kw = bs.fallback_case()
    P = mrcal_b200.Problem(**kw)
    with pytest.raises(RuntimeError, match="do not fit this problem"):
        P.reduced_system(0.0, fused=True)
    with pytest.raises(RuntimeError, match="do not fit this problem"):
        P.cauchy_denominator(fused=True)
    check_solve(ref, kw, capfd, fallback=True)


def test_solve_at_121_corners(ref, capfd):
    """11x11 boards on the fused path, a whole solve"""
    check_solve(ref, bs.solve121_case(), capfd, fallback=False)
