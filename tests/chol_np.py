"""A numpy restatement of the dense Cholesky and its triangular solves in extended precision, and the matrices that
exercise them, used as the test oracle of the device kernels (chol_dataflow.cu, potrf_block.cuh, chol.cu).

The references run in np.longdouble: the x87 80-bit format on x86-64, 64 bits of mantissa against fp64's 53, so its
own rounding error is 2^-11 of what is being measured. They are plain column algorithms, fine up to n ~ 1300.

Generators:
    spd_cond(n, cond)        Q diag(lambda) Q' with eigenvalues from 1 down to 1/cond
    graded(M, k)             D M D, D = diag(2^k_i): the Cholesky factor is D L(M), exactly, in any binary arithmetic
    minor_failure(S, p, d)   S with its trailing block [p:, p:] changed so that pivot p becomes -d: the leading p x p
                             block is S's, bit for bit, so every earlier pivot is unchanged
    with_nan(A, i, j)        one NaN (and its mirror)
    augmented(S, b)          the solver's augmented layout (normal_schur.cu): rows < nreal: S; row nreal: b' with 1 on
                             the diagonal; row nreal+1: g' (zero by default) with 1 on the diagonal
"""
import numpy as np

LD = np.longdouble
BLOCK = 64


def padded(n):
    return (n + BLOCK - 1) // BLOCK * BLOCK


def cholesky_ld(A):
    """Lower Cholesky factor of the symmetric A (its lower triangle is read) in longdouble, by columns. Raises
    ValueError naming the first pivot that is not positive"""
    A = np.tril(np.asarray(A, dtype=LD))
    n = A.shape[0]
    L = np.zeros((n, n), dtype=LD)
    for j in range(n):
        v = A[j:, j] - L[j:, :j] @ L[j, :j]
        if not v[0] > 0:
            raise ValueError(f"pivot {j} is not positive")
        d = np.sqrt(v[0])
        L[j, j] = d
        L[j + 1:, j] = v[1:] / d
    return L


def ldl_pivots_ld(A):
    """The pivots of A = L D L' (D) in longdouble, carried on past non-positive ones"""
    A = np.array(A, dtype=LD)
    n = A.shape[0]
    d = np.zeros(n, dtype=LD)
    for j in range(n):
        d[j] = A[j, j]
        if j + 1 < n and d[j] != 0:
            l = A[j + 1:, j] / d[j]
            A[j + 1:, j + 1:] -= np.outer(l, A[j + 1:, j])
    return d


def first_bad_pivot(A):
    """Index of the first pivot that is not positive (NaN included), or None"""
    d = ldl_pivots_ld(A)
    bad = np.nonzero(~(d > 0))[0]
    return int(bad[0]) if len(bad) else None


def solve_lower_ld(L, B):
    """L Y = B for a lower triangular L; B (n,) or (n, k). In longdouble"""
    L = np.asarray(L, dtype=LD)
    Y = np.array(B, dtype=LD)
    for i in range(L.shape[0]):
        Y[i] = (Y[i] - L[i, :i] @ Y[:i]) / L[i, i]
    return Y


def solve_upper_ld(L, B):
    """L' X = B for a lower triangular L; B (n,) or (n, k). In longdouble"""
    L = np.asarray(L, dtype=LD)
    X = np.array(B, dtype=LD)
    for i in range(L.shape[0] - 1, -1, -1):
        X[i] = (X[i] - L[i + 1:, i] @ X[i + 1:]) / L[i, i]
    return X


def block_inverses_ld(L, nb=BLOCK):
    """The inverse of each nb x nb diagonal block of L, (n/nb, nb, nb), in longdouble"""
    n = L.shape[0]
    return np.stack([solve_lower_ld(L[k:k + nb, k:k + nb], np.eye(nb, dtype=LD)) for k in range(0, n, nb)])


def spd_cond(n, cond, rng, reflectors=None):
    """A symmetric positive definite Q diag(lambda) Q' with lambda geometric from 1 down to 1/cond, in random order.
    Q: a random orthogonal matrix (QR of a Gaussian one), or above n = 1500 -- where that costs seconds -- a product
    of `reflectors` random Householder reflections (default 8)"""
    lam = np.geomspace(1., 1. / cond, n) if n > 1 else np.ones(1)
    lam = rng.permutation(lam)
    if reflectors is None and n <= 1500:
        Q, R = np.linalg.qr(rng.normal(size=(n, n)))
        Q *= np.sign(np.diag(R))
        A = (Q * lam) @ Q.T
    else:
        A = np.diag(lam)
        for _ in range(reflectors or 8):
            u = rng.normal(size=n)
            u /= np.linalg.norm(u)
            Au = A @ u
            w = 2. * (Au - (u @ Au) * u)   # (I - 2uu') A (I - 2uu') = A - u w' - w u'
            A -= np.outer(u, w)
            A -= np.outer(w, u)
    return (A + A.T) / 2.


def graded(M, k):
    """D M D with D = diag(2^k): exact (powers of two), for |k| small enough to stay inside the normal range"""
    s = np.ldexp(1., np.asarray(k))
    return M * s[:, None] * s[None, :]


def minor_failure(S, p, delta):
    """S - (d_p + delta) l_p l_p', d_p and l_p the pivot p and column p of S = L D L' (L unit lower triangular): pivot p
    becomes -delta, and since l_p is zero above row p, the leading p x p block is S's unchanged"""
    S = np.asarray(S, dtype=float)
    n = S.shape[0]
    Lc = np.linalg.cholesky(S)
    l = np.zeros(n)
    l[p:] = Lc[p:, p] / Lc[p, p]
    A = S.copy()
    A[p:, p:] -= (Lc[p, p] ** 2 + delta) * np.outer(l[p:], l[p:])
    A = (A + A.T) / 2.
    A[:p, :p] = S[:p, :p]
    return A


def with_nan(A, i, j):
    A = np.array(A, dtype=float)
    A[i, j] = A[j, i] = np.nan
    return A


def augmented(S, b, g=None):
    """(nreal + 2) x (nreal + 2): S, then the row b' with 1 on the diagonal, then the row g' (zero if None) with 1 on
    the diagonal (the entry (nreal+1, nreal) is zero). Symmetric"""
    nreal = S.shape[0]
    A = np.zeros((nreal + 2, nreal + 2))
    A[:nreal, :nreal] = S
    A[nreal, :nreal] = A[:nreal, nreal] = b
    if g is not None:
        A[nreal + 1, :nreal] = A[:nreal, nreal + 1] = g
    A[nreal, nreal] = A[nreal + 1, nreal + 1] = 1.
    return A
