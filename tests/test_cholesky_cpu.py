"""The oracle of the dense Cholesky tests (chol_np.py) checked on its own, without a GPU: the longdouble factor and
solves against LAPACK, and each matrix generator against what it claims."""
import numpy as np
import pytest
import scipy.linalg

import chol_np

EPS = np.finfo(float).eps


@pytest.mark.parametrize("n", [1, 5, 64, 130])
def test_longdouble_factor_matches_lapack(n):
    rng = np.random.default_rng(n)
    A = chol_np.spd_cond(n, 1e3, rng)
    L = chol_np.cholesky_ld(A)
    assert L.dtype == np.longdouble and np.all(np.triu(L, 1) == 0)
    Lf = scipy.linalg.cholesky(A, lower=True)
    assert np.abs(L.astype(float) - Lf).max() <= 64 * n * EPS
    # and it is the better of the two: the residual of L L' - A in longdouble is far below fp64's
    R = L @ L.T - A.astype(np.longdouble)
    assert float(np.abs(R).max()) <= 16 * EPS * 2. ** -8


def test_longdouble_is_extended():
    """the oracle needs 11 more bits than fp64 (x87 80-bit long double)"""
    assert np.finfo(np.longdouble).nmant >= 63


def test_longdouble_solves_and_block_inverses():
    rng = np.random.default_rng(1)
    n = 150
    L = chol_np.cholesky_ld(chol_np.spd_cond(n, 1e2, rng))
    B = rng.normal(size=(n, 3))
    Y = chol_np.solve_lower_ld(L, B)
    X = chol_np.solve_upper_ld(L, B)
    Lf = L.astype(float)
    assert np.allclose(Y.astype(float), scipy.linalg.solve_triangular(Lf, B, lower=True), rtol=0, atol=1e-12)
    assert np.allclose(X.astype(float), scipy.linalg.solve_triangular(Lf, B, lower=True, trans="T"), rtol=0, atol=1e-12)
    assert float(np.abs(L @ Y - B).max()) < 1e-17 and float(np.abs(L.T @ X - B).max()) < 1e-17
    Lp = np.eye(192, dtype=np.longdouble)
    Lp[:n, :n] = L
    W = chol_np.block_inverses_ld(Lp)
    assert W.shape == (3, 64, 64)
    for k in range(3):
        assert float(np.abs(W[k] @ Lp[64 * k:64 * k + 64, 64 * k:64 * k + 64] - np.eye(64)).max()) < 1e-16
        assert np.all(np.triu(W[k], 1) == 0)
    assert np.array_equal(W[2][n - 128:, n - 128:], np.eye(192 - n))


@pytest.mark.parametrize("n,cond", [(40, 1e3), (300, 1e12), (1600, 1e3)])
def test_spd_cond(n, cond):
    A = chol_np.spd_cond(n, cond, np.random.default_rng(2))
    assert np.array_equal(A, A.T)
    w = np.linalg.eigvalsh(A)
    assert w.min() > 0
    assert abs(w.max() / w.min() / cond - 1) < (1e-6 if cond <= 1e3 else 1e-2)
    # dense, not diagonal
    assert np.abs(A - np.diag(np.diag(A))).max() > 1e-3 / np.sqrt(n)


def test_graded_is_exact_and_keeps_its_factor():
    rng = np.random.default_rng(3)
    n = 100
    M = chol_np.spd_cond(n, 1e2, rng)
    k = rng.integers(-200, 201, size=n)
    A = chol_np.graded(M, k)
    s = np.ldexp(1., k)
    assert np.array_equal(A / s[:, None] / s[None, :], M)
    # L(D M D) = D L(M): LAPACK's factor scales exactly too
    assert np.array_equal(scipy.linalg.cholesky(A, lower=True), scipy.linalg.cholesky(M, lower=True) * s[:, None])
    d = np.diag(scipy.linalg.cholesky(A, lower=True)) ** 2
    assert d.min() > 2. ** -450 and d.max() < 2. ** 450


@pytest.mark.parametrize("p", [0, 15, 16, 63, 64, 130, 199])
def test_minor_failure(p):
    rng = np.random.default_rng(p)
    S = chol_np.spd_cond(200, 1e2, rng)
    A = chol_np.minor_failure(S, p, 0.5)
    assert np.array_equal(A, A.T)
    assert np.array_equal(A[:p, :p], S[:p, :p])
    assert chol_np.first_bad_pivot(A) == p
    d = chol_np.ldl_pivots_ld(A)
    assert abs(float(d[p]) + 0.5) < 1e-12
    assert np.array_equal(d[:p], chol_np.ldl_pivots_ld(S)[:p])


def test_nan_and_first_bad_pivot():
    S = chol_np.spd_cond(100, 1e2, np.random.default_rng(4))
    assert chol_np.first_bad_pivot(S) is None
    A = chol_np.with_nan(S, 37, 37)
    assert np.isnan(A[37, 37]) and np.isnan(A).sum() == 1
    assert chol_np.first_bad_pivot(A) == 37
    with pytest.raises(ValueError, match="pivot 37"):
        chol_np.cholesky_ld(A)


def test_augmented_layout():
    rng = np.random.default_rng(5)
    nreal = 70
    S = chol_np.spd_cond(nreal, 1e2, rng)
    b = 3. * rng.normal(size=nreal)
    A = chol_np.augmented(S, b)
    assert A.shape == (nreal + 2, nreal + 2) and np.array_equal(A, A.T)
    assert np.array_equal(A[:nreal, :nreal], S)
    assert np.array_equal(A[nreal, :nreal], b) and A[nreal, nreal] == 1 and A[nreal, nreal + 1] == 0
    assert np.all(A[nreal + 1, :nreal] == 0) and A[nreal + 1, nreal + 1] == 1
    # row nreal of the factor is inv(L_S) b; its pivot 1 - |inv(L_S) b|^2 is negative here
    L = chol_np.cholesky_ld(S)
    y = chol_np.solve_lower_ld(L, b)
    assert float(y @ y) > 1
    assert chol_np.first_bad_pivot(A) == nreal
    assert chol_np.padded(nreal + 2) == 128
