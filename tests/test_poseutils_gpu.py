"""GPU: the pose utilities (mrcal_b200/poseutils.py, csrc/poseutils.cu) against the reference's answers
(tests/poseutils_np.py: the compiled reference, or tests/golden/poseutils.npz without it), against central
differences of their own values, and through broadcasting, out=, torch tensors on a side stream, NaN and empty
inputs."""
import numpy as np
import pytest

import mrcal_b200
import poseutils_np as U

pytestmark = pytest.mark.gpu

_CASES = None
RODRIGUES_GRADIENT = ("R_from_r", "Rt_from_rt", "r_from_R", "rt_from_Rt")


def cases():
    global _CASES
    if _CASES is None:
        _CASES = U.load()
    return _CASES


def _keys():
    return [c[0] for c in U.cases(ref_available=False)]


@pytest.mark.parametrize("key", _keys())
def test_against_reference(key):
    _, fname, args, kw, _, want = next(c for c in cases() if c[0] == key)
    got = getattr(mrcal_b200, fname)(*args, **kw)
    got = got if isinstance(got, tuple) else (got,)
    assert len(got) == len(want)
    ok = U.check_value(key, fname, got[0], want[0], mrcal_b200.R_from_r)
    for k, (g, w) in enumerate(zip(got[1:], want[1:]), 1):
        assert g.shape == w.shape, key
        g, w = g[ok], w[ok]
        err = np.abs(g - w).reshape(len(g), -1)
        tol = np.full(len(g), 1e-12 * max(1., np.abs(w).max()))
        if fname in RODRIGUES_GRADIENT:
            # the reference's closed-form dR/dr at small |r| cancels: its error is ~eps/|r| (below |r|, since the
            # cancelling terms are themselves O(|r|)); rodrigues() uses a series there
            r = (args[0] if fname in ("R_from_r", "Rt_from_rt") else want[0])[ok][..., :3]
            m = np.linalg.norm(r, axis=-1)
            tol += 8 * np.minimum(U.EPS / np.maximum(m, 1e-300), m)
        if fname in ("compose_r", "compose_rt"):
            # a composition whose result is a small rotation |r| takes its half-angle C (or pi - C) from acos() of a
            # cosine within |r|^2/8 of +-1, and its gradient from sin(C) = sqrt(1 - cos(C)^2): that carries a
            # relative error of ~eps/sin(C)^2 = 4 eps/|r|^2, in the reference's gradient as in this one
            m = np.linalg.norm(want[0][ok][..., :3], axis=-1)
            tol += np.minimum(16 * U.EPS / np.maximum(m * m, 1e-300), 1e-6) * max(1., np.abs(w).max())
        bad = np.nonzero(err.max(-1) > tol)[0]
        assert len(bad) == 0, f"{key} output {k}: element {bad[:3]} error {err.max(-1)[bad[:3]]} > {tol[bad[:3]]}"


def _central(f, x, h=1e-6):
    x = np.array(x, float)
    cols = []
    for i in np.ndindex(x.shape):
        xp, xm = x.copy(), x.copy()
        xp[i] += h
        xm[i] -= h
        cols.append((f(xp) - f(xm)) / (2 * h))
    return np.stack(cols, -1).reshape(np.shape(f(x)) + x.shape)


def test_gradients_match_central_differences():
    rng = np.random.default_rng(5)
    r0, r1 = rng.normal(size=(2, 3))
    rt0, rt1 = rng.normal(size=(2, 6))
    x = rng.normal(size=3) * 3
    R = mrcal_b200.R_from_r(rng.normal(size=3))
    Rt = np.vstack((R, rng.normal(size=(1, 3))))
    check = lambda a, b: np.abs(a - b).max() <= 1e-6 * (1 + np.abs(b).max())   # noqa: E731
    assert check(mrcal_b200.R_from_r(r0, get_gradients=True)[1], _central(mrcal_b200.R_from_r, r0))
    assert check(mrcal_b200.invert_rt(rt0, get_gradients=True)[1], _central(mrcal_b200.invert_rt, rt0))
    for i0 in (False, True):
        for i1 in (False, True):
            kw = dict(inverted0=i0, inverted1=i1)
            _, d0, d1 = mrcal_b200.compose_r(r0, r1, get_gradients=True, **kw)
            assert check(d0, _central(lambda a: mrcal_b200.compose_r(a, r1, **kw), r0))
            assert check(d1, _central(lambda b: mrcal_b200.compose_r(r0, b, **kw), r1))
            _, d0, d1 = mrcal_b200.compose_rt(rt0, rt1, get_gradients=True, **kw)
            assert check(d0, _central(lambda a: mrcal_b200.compose_rt(a, rt1, **kw), rt0))
            assert check(d1, _central(lambda b: mrcal_b200.compose_rt(rt0, b, **kw), rt1))
    for inv in (False, True):
        for f, pose in ((mrcal_b200.rotate_point_r, r0), (mrcal_b200.transform_point_rt, rt0),
                        (mrcal_b200.rotate_point_R, R), (mrcal_b200.transform_point_Rt, Rt)):
            _, dp, dx = f(pose, x, get_gradients=True, inverted=inv)
            assert check(dp, _central(lambda p: f(p, x, inverted=inv), pose))
            assert check(dx, _central(lambda y: f(pose, y, inverted=inv), x))
    # the tiny-composition gradients are the composition's gradients at a zero operand
    z = np.zeros(6)
    assert check(mrcal_b200.compose_rt_tinyrt0_gradientrt0(rt1), _central(lambda a: mrcal_b200.compose_rt(a, rt1), z))
    assert check(mrcal_b200.compose_rt_tinyrt1_gradientrt1(rt0), _central(lambda b: mrcal_b200.compose_rt(rt0, b), z))
    # r_from_R: dr/dR dR/dr = I on the manifold
    r, drdR = mrcal_b200.r_from_R(R, get_gradients=True)
    _, dRdr = mrcal_b200.R_from_r(r, get_gradients=True)
    assert np.abs(np.einsum("kij,ijl->kl", drdR, dRdr) - np.eye(3)).max() < 1e-12


def test_broadcasting():
    rng = np.random.default_rng(6)
    rt = rng.normal(size=6)
    x = rng.normal(size=(1000, 3))
    y = mrcal_b200.transform_point_rt(rt, x)
    assert np.array_equal(y, mrcal_b200.transform_point_rt(np.tile(rt, (1000, 1)), x))
    y, drt, dx = mrcal_b200.transform_point_rt(rt, x, get_gradients=True)
    assert drt.shape == (1000, 3, 6) and dx.shape == (1000, 3, 3)
    A, B = 4, 7
    rts = rng.normal(size=(A, 1, 6))
    xs = rng.normal(size=(B, 3))
    y = mrcal_b200.transform_point_rt(rts, xs, inverted=True)
    assert y.shape == (A, B, 3)
    for a in range(A):
        for b in range(B):
            assert np.array_equal(y[a, b], mrcal_b200.transform_point_rt(rts[a, 0], xs[b], inverted=True))
    # non-contiguous inputs: every other row, a transposed leading pair, a Fortran-ordered array
    big = rng.normal(size=(20, 2, 6))
    nc = big[::2, 1]
    assert np.array_equal(mrcal_b200.compose_rt(nc, nc[::-1]), mrcal_b200.compose_rt(nc.copy(), nc[::-1].copy()))
    X = rng.normal(size=(3, 5, 3)).transpose(1, 0, 2)
    assert np.array_equal(mrcal_b200.rotate_point_r(rt[:3], X), mrcal_b200.rotate_point_r(rt[:3], X.copy()))
    R = np.asfortranarray(mrcal_b200.R_from_r(rng.normal(size=(5, 3))))
    assert np.array_equal(mrcal_b200.r_from_R(R), mrcal_b200.r_from_R(np.ascontiguousarray(R)))
    # chained compositions: compose(x0, compose(x1, x2))
    a, b, c = rng.normal(size=(3, 6))
    assert np.array_equal(mrcal_b200.compose_rt(a, b, c), mrcal_b200.compose_rt(a, mrcal_b200.compose_rt(b, c)))


def test_out_numpy():
    rng = np.random.default_rng(7)
    rt0, rt1 = rng.normal(size=(2, 10, 6))
    want = mrcal_b200.compose_rt(rt0, rt1, get_gradients=True)
    out = (np.zeros((10, 6)), np.zeros((10, 6, 6)), np.zeros((20, 6, 6))[::2])   # the last one strided
    got = mrcal_b200.compose_rt(rt0, rt1, get_gradients=True, out=out)
    assert all(g is o for g, o in zip(got, out))
    assert all(np.array_equal(g, w) for g, w in zip(got, want))
    o = np.zeros((10, 4, 3))
    assert mrcal_b200.Rt_from_rt(rt0, out=o) is o and np.array_equal(o, mrcal_b200.Rt_from_rt(rt0))


def test_torch_side_stream_out_and_inputs_unchanged():
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(8)
    rt = rng.normal(size=(3000, 6))
    x = rng.normal(size=(3000, 3))
    want = mrcal_b200.transform_point_rt(rt, x, get_gradients=True, inverted=True)
    trt = torch.tensor(rt, device="cuda")
    tx = torch.tensor(x, device="cuda")
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        got = mrcal_b200.transform_point_rt(trt, tx, get_gradients=True, inverted=True)
        out = torch.empty(3000, 6, dtype=torch.float64, device="cuda")
        out2 = torch.empty(6, 3000, dtype=torch.float64, device="cuda").T   # not contiguous
        r1 = mrcal_b200.compose_rt(trt, trt.flip(0), out=out)
        r2 = mrcal_b200.compose_rt(trt, trt.flip(0), out=out2)
    s.synchronize()
    assert all(isinstance(g, torch.Tensor) and g.device == trt.device for g in got)
    for g, w in zip(got, want):
        assert np.array_equal(g.cpu().numpy(), w)
    want_c = mrcal_b200.compose_rt(rt, rt[::-1])
    assert r1 is out and r2 is out2
    assert np.array_equal(out.cpu().numpy(), want_c) and np.array_equal(out2.cpu().numpy(), want_c)
    assert np.array_equal(trt.cpu().numpy(), rt) and np.array_equal(tx.cpu().numpy(), x)
    # a broadcast (expanded) tensor is read in place
    e = trt[:1].expand(3000, 6)
    assert np.array_equal(mrcal_b200.transform_point_rt(e, tx).cpu().numpy(), mrcal_b200.transform_point_rt(rt[0], x))
    with pytest.raises(ValueError, match="CUDA float64"):
        mrcal_b200.R_from_r(trt[:, :3].float())


def test_nan_gives_nan():
    rt = np.array([[np.nan, 0, 0, 1, 2, 3], [0.1, 0.2, 0.3, 1, 2, 3]])
    y, d0, d1 = mrcal_b200.compose_rt(rt, rt[::-1], get_gradients=True)
    assert np.isnan(y).any(axis=-1).all()
    R, dR = mrcal_b200.R_from_r(rt[:, :3], get_gradients=True)
    assert np.isnan(R[0]).all() and np.isfinite(R[1]).all()
    r = mrcal_b200.r_from_R(np.full((3, 3), np.nan))
    assert np.isnan(r).all()
    x = mrcal_b200.transform_point_rt(rt, np.zeros(3))
    assert np.isnan(x[0]).any() and np.isfinite(x[1]).all()


def test_empty():
    y = mrcal_b200.transform_point_rt(np.zeros(6), np.zeros((0, 3)))
    assert y.shape == (0, 3)
    y, d0, d1 = mrcal_b200.compose_rt(np.zeros((0, 6)), np.zeros(6), get_gradients=True)
    assert y.shape == (0, 6) and d0.shape == (0, 6, 6) and d1.shape == (0, 6, 6)
    torch = pytest.importorskip("torch")
    t = mrcal_b200.R_from_r(torch.zeros(0, 3, dtype=torch.float64, device="cuda"))
    assert tuple(t.shape) == (0, 3, 3)


def test_ten_million_points_through_tensors():
    torch = pytest.importorskip("torch")
    N = 10_000_000
    g = torch.Generator(device="cuda").manual_seed(9)
    x = torch.randn(N, 3, dtype=torch.float64, device="cuda", generator=g)
    rt = torch.tensor([0.3, -1.2, 2.0, 1., 2., 3.], dtype=torch.float64, device="cuda")
    y = mrcal_b200.transform_point_rt(rt, x)
    torch.cuda.synchronize()
    idx = np.concatenate((np.random.default_rng(10).integers(0, N, 2000), np.arange(N - 100, N)))
    xs = x[torch.as_tensor(idx, device="cuda")].cpu().numpy()
    want = mrcal_b200.transform_point_rt(rt.cpu().numpy(), xs)
    assert np.array_equal(y[torch.as_tensor(idx, device="cuda")].cpu().numpy(), want)
