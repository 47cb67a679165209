"""The dense Cholesky kernels one by one -- the persistent spine kernel (chol_dataflow.cu), the multi-kernel blocked
factorization and the triangular solves (chol.cu), and potrf_block (potrf_block.cuh) inside both factorizations --
through the test entry points mrcal_b200_debug_cholesky() and mrcal_b200_debug_chol_solve(), at the sizes where their
code paths change, against the extended-precision references of chol_np.py.

The gates follow one principle: a kernel may be no worse than 4x LAPACK, plus a floor of 8 eps.
  - Small sizes (n <= 1300, where the longdouble reference is cheap): the kernel's entrywise error against the
    longdouble reference is at most 4 times the error of LAPACK's fp64 result (scipy.linalg.cholesky,
    solve_triangular) against the same reference, plus 8 eps. Errors of L are measured relative to the row scale
    sqrt(A_ii) (which bounds |L_ij|), of a solve relative to the largest entry of each solution.
  - Large sizes: the probe backward error |A V - L L' V| / (|A| |V|) for a few random vectors V, evaluated in
    longdouble, against the same quantity for LAPACK's factor, with the same rule.
Forward comparisons use well-conditioned matrices (cond <= 1e3); cond up to 1e12 is used only with the backward
error. Each diagonal block of invL is held to the same rule against the inverse of the matching block of the kernel's
own L, and its strictly upper part must be exactly zero. The path and the cooperative grid each factorization ran with
are recorded (record_property, and in every failure message), so that a failure names the regime.
"""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse

import chol_np
import mrcal_b200
from mrcal_b200 import _capi

pytestmark = pytest.mark.gpu

EPS = np.finfo(float).eps
LD = np.longdouble
SMALL = 1300          # up to here the longdouble reference factor is computed

_fac = _capi.lib.mrcal_b200_debug_cholesky
_solve = _capi.lib.mrcal_b200_debug_chol_solve


class Factor:
    def __init__(self, L, invL, info, grid):
        self.L, self.invL, self.info = L, invL, info
        self.path, self.grid, self.sms, self.tasks = (int(g) for g in grid)

    def regime(self):
        return f"path {self.path} ({'spine' if self.path == 1 else 'blocked'}), grid {self.grid}, " \
               f"{self.tasks} helper tasks, {self.sms} SMs"


def factor(A, path=0, nreal=None, record=None):
    """the device factor of the symmetric A (lower triangle read), padded; path 0: chol_factor's choice, 1: the spine
    kernel, 2: the blocked factorization"""
    A = np.ascontiguousarray(A, dtype=float)
    n = A.shape[0]
    npad = chol_np.padded(n)
    L = np.empty((npad, npad))
    invL = np.empty((npad // 64, 64, 64))
    info = C.c_int(-1)
    grid = np.zeros(4, dtype=np.int32)
    assert _fac(A.ctypes.data, n, n if nreal is None else nreal, path, L.ctypes.data, invL.ctypes.data, C.byref(info),
                grid.ctypes.data), _capi.last_error()
    f = Factor(L, invL, info.value, grid)
    if record is not None:
        record("regime", f.regime())
    print(f"n={n} path={path}: {f.regime()}")
    return f


def solve(L, invL, nreal, B, parts, kernel):
    out = np.array(B, dtype=float, order="C")
    assert _solve(L.ctypes.data, invL.ctypes.data, L.shape[0], nreal, out.ctypes.data, out.shape[0], parts, kernel), \
        _capi.last_error()
    return out


@pytest.fixture(scope="module")
def sms():
    """the SM count, from the grid of a factorization with more helper tasks than SMs"""
    f = factor(np.eye(40 * 64) * 2.)
    assert f.path == 1 and f.tasks > f.grid and f.grid == f.sms, f.regime()
    return f.grid


def oversubscribed_nb(sms):
    """the smallest number of 64-blocks whose helper tasks, (nb-1) nb/2 - 1, exceed the helper CTAs (sms - 1)"""
    nb = 3
    while (nb - 1) * nb // 2 - 1 <= sms - 1:
        nb += 1
    return nb


def gate(e_dev, e_lapack):
    return e_dev <= 4. * e_lapack + 8. * EPS


def _mat_ld(M, V):
    """M V in longdouble, a block of rows at a time"""
    out = np.empty((M.shape[0], V.shape[1]), dtype=LD)
    Vl = V.astype(LD)
    for r in range(0, M.shape[0], 512):
        out[r:r + 512] = M[r:r + 512].astype(LD) @ Vl
    return out


def probe_backward_error(A, L, V):
    """max |A V - L (L' V)| / max (|A| |V|), the residual in longdouble"""
    R = _mat_ld(A, V) - _mat_ld(L, _mat_ld(L.T, V).astype(float))
    return float(np.abs(R).max() / (np.abs(A) @ np.abs(V)).max())


def check_invL(f, msg):
    """every diagonal block of invL against the longdouble inverse of the matching block of the kernel's own L"""
    I = np.eye(64)
    for k in range(f.invL.shape[0]):
        X = f.invL[k]
        assert np.all(np.triu(X, 1) == 0), f"block {k}: invL is not lower triangular; {msg}"
        Lk = f.L[64 * k:64 * k + 64, 64 * k:64 * k + 64]
        Xref = chol_np.solve_lower_ld(Lk, I)
        scale = float(np.abs(Xref).max())
        e_dev = float(np.abs(X - Xref).max()) / scale
        e_lap = float(np.abs(scipy.linalg.solve_triangular(Lk, I, lower=True) - Xref).max()) / scale
        assert gate(e_dev, e_lap), f"block {k}: invL error {e_dev / EPS:.1f} eps, LAPACK's {e_lap / EPS:.1f} eps; {msg}"


def check_factor(A, f, nreal=None, probe=False, msg=""):
    """L of the kernel against the reference (small: entrywise; large or probe=True: probe backward error), invL,
    the zeros above the diagonal, the padding (identity when there are no augmented rows), info == 0"""
    n = A.shape[0]
    nreal = n if nreal is None else nreal
    msg = f"n={n}: {f.regime()} {msg}"
    assert f.info == 0, f"info {f.info}; {msg}"
    assert np.all(np.triu(f.L, 1) == 0), msg
    Lr = f.L[:nreal, :nreal]
    Ar = A[:nreal, :nreal]
    Llap = scipy.linalg.cholesky(Ar, lower=True)
    if nreal <= SMALL and not probe:
        Lref = chol_np.cholesky_ld(Ar)
        scale = np.sqrt(np.diag(Ar))[:, None]
        e_dev = float((np.abs(Lr - Lref) / scale).max())
        e_lap = float((np.abs(Llap - Lref) / scale).max())
        kind = "entrywise"
    else:
        V = np.random.default_rng(nreal).normal(size=(nreal, 4))
        e_dev, e_lap = probe_backward_error(Ar, Lr, V), probe_backward_error(Ar, Llap, V)
        kind = "probe backward"
    print(f"  {kind} error {e_dev / EPS:.2f} eps (LAPACK {e_lap / EPS:.2f} eps)")
    assert gate(e_dev, e_lap), f"{kind} error {e_dev / EPS:.2f} eps, LAPACK's {e_lap / EPS:.2f} eps; {msg}"
    if nreal == n:
        npad = f.L.shape[0]
        pad = np.zeros((npad - n, npad))
        pad[:, n:] = np.eye(npad - n)
        assert np.array_equal(f.L[n:, :], pad), f"padding rows of L; {msg}"
    check_invL(f, msg)


def _spd(n, cond=1e3, seed=None):
    return chol_np.spd_cond(n, cond, np.random.default_rng(n if seed is None else seed))


############################################################ the spine kernel


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 257, "oversubscribed-1", "oversubscribed",
                               1268, 8191, 8192])
def test_spine(n, sms, record_property):
    """every structural edge of the spine kernel: one block (no helper), two (no pre task), three (the first helper CTA
    and pre task), partial blocks; the last nb whose helper tasks fit on the helper CTAs and the first that does not
    (each CTA then walks several tasks); config 3's reduced system (1268); the largest size the kernel takes"""
    nb_over = oversubscribed_nb(sms)
    if isinstance(n, str):
        n = 64 * (nb_over - (1 if n.endswith("-1") else 0)) - 5
    A = _spd(n)
    f = factor(A, 0, record=record_property)
    assert f.path == 1, f.regime()
    nb = chol_np.padded(n) // 64
    tasks = (nb - 1) * nb // 2 - 1 if nb >= 3 else 0
    assert f.tasks == tasks and f.grid == 1 + min(tasks, sms - 1), f.regime()
    if nb == nb_over:
        assert f.tasks > f.grid - 1, f.regime()
    if nb == nb_over - 1:
        assert f.tasks <= f.grid - 1, f.regime()
    check_factor(A, f)


def test_spine_ill_conditioned(sms, record_property):
    """cond 1e12, with the backward error only"""
    for n in (1100, 4000):
        A = _spd(n, 1e12)
        f = factor(A, 1, record=record_property)
        check_factor(A, f, probe=True)


############################################################ the blocked factorization


@pytest.mark.parametrize("n", [64, 65, 257, 320, 511, 513, 1100])
def test_blocked_forced(n, record_property):
    """the multi-kernel factorization below its natural sizes: an outer panel that is not a multiple of 256 columns,
    partial 128-tiles of the trailing update"""
    A = _spd(n)
    f = factor(A, 2, record=record_property)
    assert f.path == 2 and f.grid == 0, f.regime()
    check_factor(A, f)


_large = {}


def _large_factor(n):
    if n not in _large:
        A = _spd(n, 1e3)
        _large.clear()
        _large[n] = (A, factor(A, 0))
    return _large[n]


@pytest.mark.parametrize("n", [8193, "sms+3 blocks"])
def test_blocked_natural(n, sms, record_property):
    """above npad = 8192 chol_factor takes the blocked factorization"""
    if isinstance(n, str):
        n = 64 * (sms + 3) - 7
    A, f = _large_factor(n)
    record_property("regime", f.regime())
    assert f.path == 2 and f.grid == 0, f.regime()
    check_factor(A, f)


@pytest.mark.parametrize("n", [129, 1100])
def test_both_paths_same_matrix(n, record_property):
    A = _spd(n)
    for path in (1, 2):
        f = factor(A, path, record=record_property)
        assert f.path == path
        check_factor(A, f)


############################################################ graded matrices, pivot threshold


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("n", [130, 700])
def test_graded(n, path, record_property):
    """L(D M D) = D L(M) for D = diag(2^k), k in [-200, 200]: powers of two commute with rounding, so the kernel's
    own factor of M, scaled, must come back -- entrywise, which a normwise gate would not see in the tiny entries.
    invL scales by inv(D) on the right"""
    rng = np.random.default_rng(n + path)
    M = chol_np.spd_cond(n, 1e2, rng)
    k = rng.integers(-200, 201, size=n)
    f0 = factor(M, path)
    check_factor(M, f0)
    f1 = factor(chol_np.graded(M, k), path, record=record_property)
    assert f1.info == 0, f1.regime()
    npad = f0.L.shape[0]
    s = np.ones(npad)
    s[:n] = np.ldexp(1., k)
    want = f0.L * s[:, None]
    low = np.tril(np.ones((npad, npad), bool))
    assert np.all(np.abs(f1.L - want)[low] <= 4 * EPS * np.abs(want)[low]), f1.regime()
    assert np.all(f1.L[~low] == 0)
    wantX = f0.invL / s.reshape(-1, 64)[:, None, :]
    assert np.all(np.abs(f1.invL - wantX) <= 4 * EPS * np.abs(wantX)), f1.regime()
    identical = np.array_equal(f1.L, want) and np.array_equal(f1.invL, wantX)
    record_property("bit_identical", identical)
    print(f"  graded factor bit-identical to the scaled one: {identical}")


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("log2_pivot,accepted", [(-950, True), (-1000, False)])
def test_pivot_threshold(log2_pivot, accepted, path, record_property):
    """potrf_block accepts a pivot (of the square-root-free form, L_jj^2) when its high word says at least 2^-960: a
    pivot of 2^-950 is factored, one of 2^-1000 -- normal, but below that -- is reported as not positive definite"""
    n, p = 130, 70
    rng = np.random.default_rng(7)
    M = chol_np.spd_cond(n, 10., rng)
    d = float(chol_np.ldl_pivots_ld(M)[p])
    k = np.zeros(n, dtype=int)
    k[p] = int(np.round((log2_pivot - np.log2(d)) / 2))
    A = chol_np.graded(M, k)
    assert abs(np.log2(float(chol_np.ldl_pivots_ld(A)[p])) - log2_pivot) <= 1
    f = factor(A, path, record=record_property)
    if accepted:
        check_factor(M, factor(M, path))
        assert f.info == 0, f.regime()
        s = np.ones(f.L.shape[0])
        s[:n] = np.ldexp(1., k)
        want = factor(M, path).L * s[:, None]
        assert np.all(np.abs(f.L - want) <= 4 * EPS * np.abs(want)), f.regime()
    else:
        assert f.info == p + 1, f"info {f.info}; {f.regime()}"


############################################################ not positive definite


@pytest.mark.parametrize("path", [1, 2])
@pytest.mark.parametrize("p", [0, 15, 16, 63, 64, 130, 199])
def test_not_positive_definite(p, path, record_property):
    """info = 1 + the first bad pivot, exactly: a leading minor that fails at p (every earlier pivot unchanged), and a
    NaN on the diagonal at p"""
    n = 200
    S = _spd(n, 1e2, seed=p)
    A = chol_np.minor_failure(S, p, 0.5)
    assert chol_np.first_bad_pivot(A) == p
    f = factor(A, path, record=record_property)
    assert f.info == p + 1, f"info {f.info}; {f.regime()}"
    f = factor(chol_np.with_nan(S, p, p), path)
    assert f.info == p + 1, f"NaN at ({p}, {p}): info {f.info}; {f.regime()}"


@pytest.mark.parametrize("p", [16, 130])
def test_not_positive_definite_factorization_object(p):
    """CHOLMOD_factorization of a J whose column p is zero: J'J has a zero pivot at p, and the message names it"""
    n, m = 200, 600
    J = scipy.sparse.random(m, n, density=0.05, random_state=np.random.RandomState(p), format="lil")
    J = (J + scipy.sparse.vstack([scipy.sparse.eye(n) * 0.5, scipy.sparse.csr_matrix((m - n, n))])).tolil()
    J[:, p] = 0.
    with pytest.raises(RuntimeError, match=rf"positive definite \(pivot {p}\)"):
        mrcal_b200.CHOLMOD_factorization(J.tocsr())


############################################################ the augmented row


@pytest.mark.parametrize("n_c,path", [(62, 1), (63, 1), (64, 1), (127, 1), (1268, 1), (127, 2)])
def test_augmented_row(n_c, path, record_property):
    """The solver factors S with the right-hand side b' as an extra row n_c (normal_schur.cu) and reads its forward
    substitution from row n_c of L. That row must equal inv(L) b; its pivot, 1 - |inv(L) b|^2, is negative here and
    must stay unreported (only pivots < nreal count)"""
    rng = np.random.default_rng(n_c)
    S = chol_np.spd_cond(n_c, 1e2, rng)
    b = 3. * rng.normal(size=n_c)
    A = chol_np.augmented(S, b)
    f = factor(A, path, nreal=n_c, record=record_property)
    Ls = f.L[:n_c, :n_c]
    yref = chol_np.solve_lower_ld(Ls, b)
    assert float(yref @ yref) > 1.
    check_factor(A, f, nreal=n_c)
    scale = float(np.abs(yref).max())
    e_dev = float(np.abs(f.L[n_c, :n_c] - yref).max()) / scale
    e_lap = float(np.abs(scipy.linalg.solve_triangular(Ls, b, lower=True) - yref).max()) / scale
    assert gate(e_dev, e_lap), f"augmented row: {e_dev / EPS:.2f} eps, LAPACK's {e_lap / EPS:.2f} eps; {f.regime()}"


############################################################ repeatability


@pytest.mark.parametrize("n,path", [(1100, 1), (4000, 1), (1100, 2)])
def test_repeatable(n, path, record_property):
    """the same matrix factored twice on the same path is bit-identical: every tile sums its products in a fixed order"""
    A = _spd(n)
    f0 = factor(A, path, record=record_property)
    f1 = factor(A, path)
    assert f0.info == 0 and f1.info == 0
    assert np.array_equal(f0.L, f1.L) and np.array_equal(f0.invL, f1.invL), f0.regime()


############################################################ chol_solve


_solve_factors = {}


def _solve_factor(nb, nreal):
    key = (nb, nreal)
    if key not in _solve_factors:
        A = _spd(nreal, 1e2, seed=nb * 1000 + nreal)
        f = factor(A, 0)
        assert f.info == 0 and f.L.shape[0] == 64 * nb
        _solve_factors[key] = f
    return _solve_factors[key]


def _nrhs_cases():
    out = []
    for nb in (1, 3, 20):
        for nrhs in sorted({1, 2, 8 * nb - 1, 8 * nb, 8 * nb + 1, 31, 32, 33, 100}):
            for r in (0, 1, 63):
                out.append(pytest.param(nb, nrhs, r, id=f"nb{nb}-nrhs{nrhs}-nreal{r}mod64"))
    return out


@pytest.mark.parametrize("nb,nrhs,r", _nrhs_cases())
def test_chol_solve(nb, nrhs, r):
    """chol_solve() with each of its kernels (0: its own choice, 1: the per-block kernels, 2: the tiled kernel) and
    parts (1: L Y = B, 2: L' X = B, 3: both), around its selection edge nrhs = 8 nb and the 32-right-hand-side tiles,
    with nreal = 0, 1, 63 mod 64. The padding of B holds NaN: no kernel may let it reach a real unknown"""
    nreal = 64 * nb if r == 0 else 64 * (nb - 1) + r
    f = _solve_factor(nb, nreal)
    npad = 64 * nb
    rng = np.random.default_rng(nb * 100 + nrhs + r)
    B = np.full((nrhs, npad), np.nan)
    B[:, :nreal] = rng.normal(size=(nrhs, nreal))
    Ls = f.L[:nreal, :nreal]
    Bt = B[:, :nreal].T
    Y = chol_np.solve_lower_ld(Ls, Bt)
    ref = {1: Y, 2: chol_np.solve_upper_ld(Ls, Bt), 3: chol_np.solve_upper_ld(Ls, Y)}
    Ylap = scipy.linalg.solve_triangular(Ls, Bt, lower=True)
    lap = {1: Ylap, 2: scipy.linalg.solve_triangular(Ls, Bt, lower=True, trans="T"),
           3: scipy.linalg.solve_triangular(Ls, Ylap, lower=True, trans="T")}
    for parts in (1, 2, 3):
        scale = np.abs(ref[parts]).max(axis=0).astype(float)
        e_lap = float((np.abs(lap[parts] - ref[parts]) / scale).max())
        for kernel in (0, 1, 2):
            X = solve(f.L, f.invL, nreal, B, parts, kernel)[:, :nreal].T
            what = f"parts {parts}, kernel {kernel} (nrhs {nrhs}, nreal {nreal}, npad {npad})"
            assert np.all(np.isfinite(X)), f"the padding reached a real unknown: {what}"
            e_dev = float((np.abs(X - ref[parts]) / scale).max())
            assert gate(e_dev, e_lap), f"{e_dev / EPS:.2f} eps, LAPACK's {e_lap / EPS:.2f} eps: {what}"


@pytest.mark.parametrize("nb", [1, 2, 3, 20, "sms+3"])
def test_backward_substitution(nb, sms, record_property):
    """chol_solve_backward(), the solver's persistent backward substitution, one right-hand side over the whole
    padded system (zero in the padding, as the solver passes it). At nb = SMs + 3 each CTA loops over several blocks"""
    if nb == "sms+3":
        nb = sms + 3
        n = 64 * nb - 7
        A, f = _large_factor(n)
    else:
        n = 64 * nb - 7
        A = _spd(n)
        f = factor(A, 0)
    record_property("regime", f"{nb} blocks on {min(nb, sms)} CTAs")
    assert f.info == 0
    npad = 64 * nb
    b = np.zeros(npad)
    b[:n] = np.random.default_rng(nb).normal(size=n)
    x = solve(f.L, f.invL, n, b[None, :], 2, 3)[0]
    assert np.all(x[n:] == 0)
    Ls = f.L[:n, :n]
    xref = chol_np.solve_upper_ld(Ls, b[:n])
    scale = float(np.abs(xref).max())
    e_dev = float(np.abs(x[:n] - xref).max()) / scale
    e_lap = float(np.abs(scipy.linalg.solve_triangular(Ls, b[:n], lower=True, trans="T") - xref).max()) / scale
    print(f"  nb={nb}: {e_dev / EPS:.2f} eps (LAPACK {e_lap / EPS:.2f} eps)")
    assert gate(e_dev, e_lap), f"{e_dev / EPS:.2f} eps, LAPACK's {e_lap / EPS:.2f} eps; {nb} blocks, {sms} SMs"
