"""Without a GPU: every case of structured_factor.py has the shape it claims, proved from the compiled reference's
Jacobian (oracle/_ref) and the layout functions, and the longdouble reference agrees with scipy. A change to the
synthetic problems that loses a case fails here."""
import numpy as np
import pytest
import scipy.linalg

import structured_factor as sf
from chol_np import LD


def shape_of(ref, name):
    kw = sf.case(name)
    b, x, J = ref.Problem(kw).callback()
    return kw, J, sf.Shape(kw, J)


@pytest.mark.parametrize("name", list(sf.CASES))
def test_case_has_its_shape(ref, name):
    claims = sf.CASES[name]["claims"]
    kw, J, S = shape_of(ref, name)
    # P: the eliminated unknowns, then the coupled ones, then the uncoupled ones; a permutation
    assert np.array_equal(np.sort(S.perm), np.arange(J.shape[1]))
    assert len(S.group_cols) * 6 >= S.nelim == 6 * S.Nframe_groups + 3 * (len(S.group_cols) - S.Nframe_groups)
    for key in ("n_c", "nelim", "nblk"):
        if key in claims:
            assert getattr(S, key) == claims[key], (key, getattr(S, key))
    if "groups" in claims:
        assert (S.Nframe_groups, len(S.group_cols) - S.Nframe_groups) == claims["groups"]
    if "reach" in claims:
        assert {b: len(S.reach[b]) for b in claims["reach"]} == claims["reach"]
    if "n_i" in claims:
        assert len(S.uncoupled) == claims["n_i"]
    if "kinds" in claims:
        assert set(S.kinds) == claims["kinds"]
        if claims["kinds"] == {1, 2}:
            # each knot whole: a first and a second column next to each other
            k = np.array(S.kinds)
            assert np.all(S.uncoupled[k == 2] - 1 == S.uncoupled[k == 1])
    stages = [st for b in S.reach for st in S.stages(b)]
    mixed = any(min(st) < S.Nframe_groups <= max(st) for st in stages)
    assert mixed == claims.get("mixed_stage", False)
    zero = np.flatnonzero(np.asarray(abs(J).sum(axis=0)).ravel() == 0)
    if claims.get("singular"):
        # a column of J that is zero makes J'J singular: the longdouble factorization must stop at it
        assert len(zero) > 0
        with pytest.raises(ValueError, match="not positive"):
            sf.Reference(J, S.perm)
        return
    assert len(zero) == 0
    R = sf.Reference(J, S.perm)
    d = R.pivots()
    i = int(np.argmin(d))
    where = "D" if i < S.nelim else "S" if i < S.nelim + S.n_c else "I"
    if "min_pivot" in claims:
        assert where == claims["min_pivot"], (where, d[:S.nelim].min() if S.nelim else None)
        # and not by a hair: the smallest pivot of each other piece is at least 1 % larger
        pieces = dict(D=d[:S.nelim], S=d[S.nelim:S.nelim + S.n_c], I=d[S.nelim + S.n_c:])
        for k, v in pieces.items():
            if k != where and len(v):
                assert v.min() > 1.01 * d[i]
    if "min_kind" in claims:
        assert S.kinds[i - S.nelim - S.n_c] == claims["min_kind"]


def test_cases_cover_every_path():
    """The claims together reach every path named in structured_factor.py's docstring"""
    cl = [c["claims"] for c in sf.CASES.values()]
    reach = {v for c in cl for v in c.get("reach", {}).values()}
    assert {1, 8, 9, 32, 33, 65} <= reach
    assert {0, 62, 63, 64, 65} <= {c["n_c"] for c in cl if "n_c" in c}
    assert max(c.get("nblk", 0) for c in cl) >= 4
    assert any(c.get("nelim") == 0 for c in cl)
    assert any(c.get("groups", (1, 0))[0] == 0 and c["groups"][1] > 0 for c in cl)   # points only
    assert any(c.get("mixed_stage") for c in cl)
    assert {1, 2, 3} <= set().union(*(c.get("kinds", set()) for c in cl))
    assert {"D", "S", "I"} == {c["min_pivot"] for c in cl if "min_pivot" in c}
    assert len(sf.REFUSED) == 2
    # the right-hand-side counts: the graph, both sides of chol_solve()'s crossover and of the 32-row tile
    for nblk in (1, 2, 4):
        n = sf.rhs_counts(nblk)
        assert {1, 8 * nblk - 1, 8 * nblk, 31, 32, 33} <= set(n) and max(n) >= 8 * nblk


def test_shape_from_layout_matches_reference(ref):
    """The package's layout functions, which Shape uses, say what the reference's do"""
    for name in ("stage_mixed", "points_only", "uncoupled_1x1", "nelim0_intrinsics_only"):
        kw = sf.case(name)
        P = ref.Problem(kw)
        b, x, J = P.callback()
        S = sf.Shape(kw, J)
        nf, npt = P.num_states_of("frames"), P.num_states_of("points")
        assert S.nelim == nf + npt
        if nf:
            assert S.e0 == P.state_index("frames", 0)
        elif npt:
            assert S.e0 == P.state_index("points", 0)


def test_longdouble_reference_matches_scipy(ref):
    """The longdouble factor and its solves against scipy's float64 ones, within what float64 can tell apart"""
    kw, J, S = shape_of(ref, "pivot_in_LD")
    R = sf.Reference(J, S.perm)
    eps = np.finfo(float).eps
    # L L' is P J'J P' to longdouble rounding
    E = R.L @ R.L.T - R.PHP
    assert float(np.abs(E).max()) <= 1e-16 * float(np.abs(R.PHP).max())
    L64 = scipy.linalg.cholesky(R.PHPf, lower=True)
    cond = np.linalg.cond(R.PHPf)
    assert np.abs(L64 - R.L.astype(float)).max() <= 64 * eps * cond * np.abs(L64).max()
    bt = np.random.default_rng(0).normal(size=(5, J.shape[1]))
    for sys in sf.SYSTEMS:
        X = R.solve(sys, bt).astype(float)
        X64 = R.solve(sys, bt, L=L64)
        assert np.abs(X - X64).max() <= 64 * eps * cond * np.abs(X).max(), sys
    assert np.allclose(R.solve("A", bt).astype(float), np.linalg.solve(R.Hf, bt.T).T, rtol=0,
                       atol=64 * eps * cond * np.abs(R.solve("A", bt).astype(float)).max())
    assert R.L.dtype == LD
