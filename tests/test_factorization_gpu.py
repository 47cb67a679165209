"""The factorization object (stand-in for mrcal.CHOLMOD_factorization), end to end. The
known-answer case is the reference's test/test-CHOLMOD-factorization.py; the random
sparse cases solve with J'J of a random J (0.5 I stacked into it) at n = 50 .. 8300
(1, 2, 4, 11, 18 and 130 64-blocks: the spine kernel, and at 8300 the blocked
factorization) and gate the relative residual at 1e-10. The Cholesky kernels
themselves -- every block count where their code changes, the not-positive-definite
report, the solve kernels' selection, with sharp gates -- are tested one by one in
test_cholesky_gpu.py."""
import numpy as np
import scipy.linalg
import pytest
import scipy.sparse

import mrcal_b200

pytestmark = pytest.mark.gpu


def test_reference_known_answer():
    # test/test-CHOLMOD-factorization.py:20-50: a 4x3 J; solve_xt_JtJ_bt(bt) == solve(JtJ, bt')'
    indptr = np.array([0, 2, 3, 6, 8])
    indices = np.array([0, 2, 2, 0, 1, 2, 1, 2])
    data = np.array([1, 2, 3, 4, 5, 6, 7, 8], dtype=float)
    Jsparse = scipy.sparse.csr_matrix((data, indices, indptr))
    Jdense = Jsparse.toarray()
    Jdense_ref = np.array(((1, 0, 2), (0, 0, 3), (4, 5, 6), (0, 7, 8)), dtype=float)
    assert np.array_equal(Jdense, Jdense_ref)
    bt = np.array(((1., 5., 3.), (2., -2., -8)))
    F = mrcal_b200.CHOLMOD_factorization(Jsparse)
    xt = F.solve_xt_JtJ_bt(bt)
    JtJ = Jdense.T @ Jdense
    xt_ref = np.linalg.solve(JtJ, bt.T).T
    assert np.allclose(xt, xt_ref, rtol=1e-6, atol=0)       # the reference's bar
    assert np.allclose(xt, xt_ref, rtol=1e-12, atol=1e-14)  # ours
    # broadcasting over leading dims, and a single vector
    assert np.allclose(F.solve_xt_JtJ_bt(bt[0]), xt_ref[0], rtol=1e-12)
    assert np.allclose(F.solve_xt_JtJ_bt(bt[None, ...]), xt_ref[None, ...], rtol=1e-12)
    L = np.linalg.cholesky(JtJ)
    d = np.diag(L)
    assert np.isclose(F.rcond(), (d.min() / d.max()) ** 2, rtol=1e-10)
    assert np.allclose(F.solve_xt_JtJ_bt(bt, sys="L"), np.linalg.solve(L, bt.T).T, rtol=1e-12)


# n = 100: two 64-blocks; n = 8300: 130 of them. 3 right-hand sides take the per-block solve; 1100 the tiled one, which
# takes over at 8 right-hand sides per 64-block
_SPARSE = [(50, 200, 0.2), (64, 300, 0.1), (100, 400, 0.1), (200, 1500, 0.05), (700, 6000, 0.02), (1100, 9000, 0.01),
           (8300, 9000, 0.0005)]


@pytest.mark.parametrize("n,m,density,nrhs", [pytest.param(*c, 3, id="-".join(map(str, c))) for c in _SPARSE] +
                         [pytest.param(8300, 9000, 0.0005, 1100, id="8300-9000-0.0005-1100rhs")])
def test_random_sparse(n, m, density, nrhs):
    rng = np.random.default_rng(n)
    J = scipy.sparse.random(m, n, density=density, random_state=np.random.RandomState(n), format="csr")
    J = (J + scipy.sparse.vstack([scipy.sparse.eye(n) * 0.5, scipy.sparse.csr_matrix((m - n, n))])).tocsr()
    H = (J.T @ J).toarray()
    bt = rng.normal(size=(nrhs, n))
    F = mrcal_b200.CHOLMOD_factorization(J)
    xt = F.solve_xt_JtJ_bt(bt)
    r = (H @ xt.T).T - bt
    assert np.abs(r).max() / np.abs(bt).max() < 1e-10   # SURVEY.md 8d: ||JtJ d - Jtx|| / ||Jtx|| <= 1e-10
    assert np.allclose(xt, np.linalg.solve(H, bt.T).T, rtol=1e-7, atol=1e-9)


def test_not_positive_definite_gives_no_object():
    # a zero column makes JtJ singular; the reference returns None for the
    # factorization in that case (mrcal-pywrap.c:1981-1988)
    J = scipy.sparse.csr_matrix(np.array(((1., 0., 2.), (0., 0., 3.), (4., 0., 6.))))
    with pytest.raises(RuntimeError, match="positive definite"):
        mrcal_b200.CHOLMOD_factorization(J)


def test_optimizer_callback_returns_factorization():
    from mrcal_b200 import synthetic
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=2, Nframes=6, W=6, H=5)
    b, x, J, F = mrcal_b200.optimizer_callback(**kw)
    assert F is not None
    Jd = J.toarray()
    g = Jd.T @ x
    d = F.solve_xt_JtJ_bt(g)
    assert np.abs(Jd.T @ (Jd @ d) - g).max() / np.abs(g).max() < 1e-9


def test_solve_systems():
    """solve_xt_JtJ_bt(sys=...) (mrcal-pywrap.c:467-493). With P = I and D = I the factor L is THE Cholesky factor
    of JtJ (unique), so 'L' and 'Lt' are pinned by numpy; the identities the reference's callers rely on
    (mrcal/model_analysis.py:837-841: P, then L, then D, and A2 A3' = b' inv(JtJ) b) are checked as such.
    n = 150 is three 64-blocks: 7 right-hand sides take the per-block solve, 100 (three full tiles and a partial one)
    the tiled solve."""
    rng = np.random.default_rng(5)
    J = scipy.sparse.random(400, 150, density=0.08, random_state=7, format="csr") + \
        scipy.sparse.vstack((scipy.sparse.eye(150), scipy.sparse.csr_matrix((250, 150))))
    F = mrcal_b200.CHOLMOD_factorization(J)
    JtJ = (J.T @ J).toarray()
    L = np.linalg.cholesky(JtJ)
    for bt in (rng.normal(size=(7, 150)), rng.normal(size=(100, 150))):
        _check_solve_systems(F, JtJ, L, bt)


def _check_solve_systems(F, JtJ, L, bt):
    tol = dict(rtol=0, atol=1e-9 * np.abs(bt).max())
    xA = F.solve_xt_JtJ_bt(bt)
    assert np.allclose(xA, np.linalg.solve(JtJ, bt.T).T, **tol)
    assert np.allclose(F.solve_xt_JtJ_bt(bt, sys="LDLt"), xA, **tol)
    for name in ("L", "LD", "CHOLMOD_L"):
        assert np.allclose(F.solve_xt_JtJ_bt(bt, sys=name), np.linalg.solve(L, bt.T).T, **tol)
    for name in ("Lt", "DLt"):
        assert np.allclose(F.solve_xt_JtJ_bt(bt, sys=name), np.linalg.solve(L.T, bt.T).T, **tol)
    for name in ("D", "P", "Pt"):
        assert np.array_equal(F.solve_xt_JtJ_bt(bt, sys=name), bt)
    # the chain the reference's uncertainty code runs
    A1 = F.solve_xt_JtJ_bt(bt, sys="P")
    A2 = F.solve_xt_JtJ_bt(A1, sys="L")
    A3 = F.solve_xt_JtJ_bt(A2, sys="D")
    assert np.allclose(A2 @ A3.T, bt @ np.linalg.solve(JtJ, bt.T), rtol=1e-9, atol=1e-12)
    # and Lt after L is A (after undoing P)
    assert np.allclose(F.solve_xt_JtJ_bt(F.solve_xt_JtJ_bt(F.solve_xt_JtJ_bt(A2, sys="D"), sys="Lt"), sys="Pt"), xA, **tol)
    with pytest.raises(RuntimeError, match="Unknown sys"):
        F.solve_xt_JtJ_bt(bt, sys="LL")
    # a single right-hand side takes the graph path
    assert np.allclose(F.solve_xt_JtJ_bt(bt[0], sys="L"), np.linalg.solve(L, bt[0]), **tol)


@pytest.mark.parametrize("lensmodel,Ncameras,Npoints", [
    ("LENSMODEL_OPENCV4", 2, 0),
    ("LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=11_Ny=8_fov_x_deg=150", 3, 0),   # most knots uncoupled: the L_I part
    ("LENSMODEL_OPENCV8", 3, 9),                                                  # point groups next to frame groups
])
@pytest.mark.parametrize("nrhs", [5, 100])   # the per-block and the tiled solve of L_S (100: a partial tile)
def test_structured_factorization_of_a_problem(lensmodel, Ncameras, Npoints, nrhs):
    """optimizer_callback()'s factorization is built from the problem's structure (factorization_schur.cu); it must
    agree with the dense factorization of the same J for every system, up to its own (documented) permutation."""
    from mrcal_b200 import synthetic
    kw, _ = synthetic.make_problem(lensmodel=lensmodel, Ncameras=Ncameras, Nframes=8, W=6, H=5, seed=6, pixel_noise=0.2,
                                   Npoints=Npoints, which="some" if Npoints else "all")
    b, x, J, F = mrcal_b200.optimizer_callback(**kw)
    assert F is not None
    Fd = mrcal_b200.CHOLMOD_factorization(J)          # dense, P = I
    JtJ = (J.T @ J).toarray()
    rng = np.random.default_rng(0)
    bt = rng.normal(size=(nrhs, J.shape[1]))
    # Two correct factorizations of the same matrix agree to eps*cond(JtJ), not better -- and these problems are not
    # well conditioned (barely-observed knots held by the regularization alone): forward gates scale with the
    # condition number, and every solve also passes a backward (residual) gate that does not
    eps = np.finfo(float).eps
    cond = np.linalg.cond(JtJ)
    xref = np.linalg.solve(JtJ, bt.T).T
    tol = dict(rtol=0, atol=max(1e-8, 64 * eps * cond) * np.abs(xref).max())

    def backward_ok(M, X, B):
        """M X' = B' to working precision: |M X' - B'| <= 1e3 eps (|M| |X'| + |B'|)"""
        return np.all(np.abs(M @ X.T - B.T) <= 1e3 * eps * (np.abs(M) @ np.abs(X.T) + np.abs(B.T)).max())

    xA = F.solve_xt_JtJ_bt(bt)
    assert backward_ok(JtJ, xA, bt)
    assert np.allclose(xA, Fd.solve_xt_JtJ_bt(bt), **tol)
    assert np.allclose(xA, xref, **tol)
    assert np.allclose(F.solve_xt_JtJ_bt(bt[0]), xA[0], **tol)
    # P is a permutation, Pt undoes it
    Pb = F.solve_xt_JtJ_bt(bt, sys="P")
    assert np.allclose(np.sort(Pb, axis=-1), np.sort(bt, axis=-1))
    assert np.array_equal(F.solve_xt_JtJ_bt(Pb, sys="Pt"), bt)
    assert np.array_equal(F.solve_xt_JtJ_bt(bt, sys="D"), bt)
    # L is lower triangular with L L' = P JtJ P': recover it column by column from solves with unit vectors
    n = J.shape[1]
    I = np.eye(n)
    Linv = F.solve_xt_JtJ_bt(I, sys="L").T          # column j = inv(L) e_j
    assert np.abs(np.triu(Linv, 1)).max() == 0.
    L = scipy.linalg.solve_triangular(Linv, I, lower=True)
    Pm = F.solve_xt_JtJ_bt(I, sys="P").T             # P as a matrix: P e_j in column j
    PJP = Pm @ JtJ @ Pm.T
    # (L comes out of an explicit inverse: it carries cond(L) = sqrt(cond(JtJ)) of roundoff)
    assert np.allclose(L @ L.T, PJP, rtol=0, atol=max(1e-9, 64 * eps * np.sqrt(cond)) * np.abs(JtJ).max())
    assert backward_ok(L.T, F.solve_xt_JtJ_bt(bt, sys="Lt"), bt)
    assert backward_ok(L, F.solve_xt_JtJ_bt(bt, sys="L"), bt)
    assert backward_ok(PJP, F.solve_xt_JtJ_bt(Pb, sys="LDLt"), Pb)
    assert np.allclose(F.solve_xt_JtJ_bt(F.solve_xt_JtJ_bt(F.solve_xt_JtJ_bt(Pb, sys="L"), sys="Lt"), sys="Pt"), xA, **tol)
    assert np.allclose(F.solve_xt_JtJ_bt(Pb, sys="LDLt"), F.solve_xt_JtJ_bt(xA, sys="P"), **tol)
    # the chain the reference's uncertainty code runs (mrcal/model_analysis.py:837-841)
    A2 = F.solve_xt_JtJ_bt(Pb, sys="L")
    A3 = F.solve_xt_JtJ_bt(A2, sys="D")
    want = bt @ xref.T
    assert np.allclose(A2 @ A3.T, want, rtol=0, atol=max(1e-8, 64 * eps * cond) * np.abs(want).max())
    # rcond as cholmod_rcond defines it for LL': (min diag / max diag)^2 of THIS factor
    d = np.abs(np.diag(L))
    assert abs(F.rcond() - (d.min() / d.max()) ** 2) <= 1e-6 * (d.min() / d.max()) ** 2


def test_structured_factorization_at_config3():
    """BASELINE config 3 (Nstate 7220): the factorization optimizer_callback() returns by default, many right-hand sides."""
    from mrcal_b200 import synthetic
    kw, _ = synthetic.baseline_config(3, pixel_noise=0.3)
    b, x, J, F = mrcal_b200.optimizer_callback(**kw)
    assert F is not None
    rng = np.random.default_rng(1)
    bt = rng.normal(size=(64, J.shape[1]))
    X = F.solve_xt_JtJ_bt(bt)
    R = (J.T @ (J @ X.T)).T - bt
    # a backward gate: the residual against what roundoff in forming JtJ X alone amounts to
    Ja = abs(J)
    scale = (Ja.T @ (Ja @ np.abs(X.T))).max()
    assert np.abs(R).max() <= 1e3 * np.finfo(float).eps * scale, (np.abs(R).max(), scale)
