"""project(), unproject() and the closed-form project_* / unproject_* broadcast over stacked intrinsics, on numpy arrays
and on torch CUDA tensors (csrc/project.cu, csrc/unproject.cuh). Every element of a stacked call must equal, bit for
bit, the call through its own intrinsics row; the tensor path must equal the numpy path bit for bit; both must match
the compiled reference where oracle/_ref is built."""
import numpy as np
import pytest

import mrcal_b200
from test_project_gpu import MODELS, _points, _unproject_intrinsics
from test_unproject_gradients_gpu import CLOSED_FORM, closed_form_points, pixels

pytestmark = pytest.mark.gpu

# (normalize, get_gradients)
UNPROJECT_FLAVOURS = ((False, False), (True, False), (False, True), (True, True))


def _rows(lm, n, seed=3):
    """n intrinsics rows of lm, each perturbed by about 1e-3 relative. CAHVORE keeps E = 0, so every row unprojects"""
    intr = _unproject_intrinsics(lm)
    rng = np.random.default_rng(seed)
    return intr * (1. + 1e-3 * rng.standard_normal((n, len(intr))))


def _tuple(r):
    return r if isinstance(r, tuple) else (r,)


def _assert_equal(a, b):
    a, b = _tuple(a), _tuple(b)
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert x.shape == y.shape and np.array_equal(x, y, equal_nan=True)


@pytest.fixture(scope="module")
def ref():
    from oracle import ref
    return ref if ref.available() else None


@pytest.mark.parametrize("lm", MODELS)
def test_stacked_intrinsics_project(lm, ref):
    rows = _rows(lm, 5)
    p = _points(21, 1).reshape(3, 7, 3)
    stacked = mrcal_b200.project(p, lm, rows[:3, None, :], get_gradients=True)
    assert [a.shape for a in stacked] == [(3, 7, 2), (3, 7, 2, 3), (3, 7, 2, rows.shape[1])]
    for k in range(3):
        single = mrcal_b200.project(p[k], lm, rows[k], get_gradients=True)
        _assert_equal(tuple(a[k] for a in stacked), single)
        if ref is not None:
            for a, b in zip(stacked, ref.project_with_intrinsics_gradient(p[k], lm, rows[k])):
                assert np.abs(a[k] - b).max() <= 1e-9 * (1. + np.abs(b).max())
    q = mrcal_b200.project(p, lm, rows[:3, None, :])
    for k in range(3):
        _assert_equal(q[k], mrcal_b200.project(p[k], lm, rows[k]))
    # one point against five rows
    one = mrcal_b200.project(p[0, 0], lm, rows, get_gradients=True)
    assert one[0].shape == (5, 2)
    for j in range(5):
        _assert_equal(tuple(a[j] for a in one), mrcal_b200.project(p[0, 0], lm, rows[j], get_gradients=True))


@pytest.mark.parametrize("lm", MODELS)
def test_stacked_intrinsics_unproject(lm, ref):
    rows = _rows(lm, 5)
    q = pixels(lm, rows[0], n=21).reshape(3, 7, 2)
    for normalize, grad in UNPROJECT_FLAVOURS:
        kw = dict(normalize=normalize, get_gradients=grad)
        stacked = _tuple(mrcal_b200.unproject(q, lm, rows[:3, None, :], **kw))
        assert stacked[0].shape == (3, 7, 3)
        for k in range(3):
            single = mrcal_b200.unproject(q[k], lm, rows[k], **kw)
            _assert_equal(tuple(a[k] for a in stacked), single)
            if ref is not None and not normalize and not grad:
                assert np.abs(stacked[0][k] - ref.unproject(q[k], lm, rows[k])).max() < 1e-9
        one = _tuple(mrcal_b200.unproject(q[0, 0], lm, rows, **kw))
        assert one[0].shape == (5, 3)
        for j in range(5):
            _assert_equal(tuple(a[j] for a in one), mrcal_b200.unproject(q[0, 0], lm, rows[j], **kw))


@pytest.mark.parametrize("lm", MODELS)
def test_strided_repeated_and_empty_operands(lm):
    rows = _rows(lm, 4)
    N = rows.shape[1]
    # points every other row of a bigger array; the intrinsics repeated through stride 0, never copied
    big = _points(40, 4).reshape(4, 10, 3)
    p = big[:, ::2]
    assert not p.flags.c_contiguous
    intr = np.broadcast_to(rows[:, None, :], (4, 5, N))
    assert intr.strides[1] == 0
    got = mrcal_b200.project(p, lm, intr, get_gradients=True)
    for k in range(4):
        _assert_equal(tuple(a[k] for a in got), mrcal_b200.project(np.ascontiguousarray(p[k]), lm, rows[k],
                                                                   get_gradients=True))
    q = pixels(lm, rows[0], n=40).reshape(4, 10, 2)[:, ::2]
    got = mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)
    for k in range(4):
        _assert_equal(tuple(a[k] for a in got), mrcal_b200.unproject(np.ascontiguousarray(q[k]), lm, rows[k],
                                                                     normalize=True, get_gradients=True))
    # a zero-size leading dimension
    empty = mrcal_b200.project(np.zeros((0, 3)), lm, rows[:, None, :], get_gradients=True)
    assert [a.shape for a in empty] == [(4, 0, 2), (4, 0, 2, 3), (4, 0, 2, N)]
    empty = mrcal_b200.unproject(np.zeros((0, 1, 2)), lm, rows, get_gradients=True)
    assert [a.shape for a in empty] == [(0, 4, 3), (0, 4, 3, 2), (0, 4, 3, N)]


@pytest.mark.parametrize("lm", MODELS)
def test_tensors_match_numpy_on_a_side_stream(lm):
    torch = pytest.importorskip("torch")
    rows = _rows(lm, 3)
    p = _points(21, 5).reshape(3, 7, 3)
    q = pixels(lm, rows[0], n=21).reshape(3, 7, 2)
    want_p = mrcal_b200.project(p, lm, rows[:, None, :], get_gradients=True)
    want_p0 = mrcal_b200.project(p, lm, rows[:, None, :])
    want_u = {f: _tuple(mrcal_b200.unproject(q, lm, rows[:, None, :], normalize=f[0], get_gradients=f[1]))
              for f in UNPROJECT_FLAVOURS}
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        # the inputs are made on the side stream, and the calls are enqueued there
        tp = torch.tensor(p, device="cuda") * 1.
        tq = torch.tensor(q, device="cuda") * 1.
        ti = torch.tensor(rows, device="cuda")[:, None, :] * 1.
        got_p = mrcal_b200.project(tp, lm, ti, get_gradients=True)
        got_p0 = mrcal_b200.project(tp, lm, ti)
        got_u = {f: _tuple(mrcal_b200.unproject(tq, lm, ti, normalize=f[0], get_gradients=f[1]))
                 for f in UNPROJECT_FLAVOURS}
    s.synchronize()
    assert all(a.is_cuda and a.dtype == torch.float64 for a in got_p)
    _assert_equal(tuple(a.cpu().numpy() for a in got_p), want_p)
    _assert_equal(got_p0.cpu().numpy(), want_p0)
    for f in UNPROJECT_FLAVOURS:
        _assert_equal(tuple(a.cpu().numpy() for a in got_u[f]), want_u[f])


@pytest.mark.parametrize("lm", ("LENSMODEL_OPENCV8", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100"))
def test_out(lm):
    torch = pytest.importorskip("torch")
    rows = _rows(lm, 3)
    N = rows.shape[1]
    p = _points(12, 6).reshape(3, 4, 3)
    q = pixels(lm, rows[0], n=12).reshape(3, 4, 2)
    want_p = mrcal_b200.project(p, lm, rows[:, None, :], get_gradients=True)
    want_u = mrcal_b200.unproject(q, lm, rows[:, None, :], normalize=True)
    shapes = ((3, 4, 2), (3, 4, 2, 3), (3, 4, 2, N))
    # numpy: contiguous targets, then strided ones (views of transposed arrays)
    out = tuple(np.full(s, 7.) for s in shapes)
    r = mrcal_b200.project(p, lm, rows[:, None, :], get_gradients=True, out=out)
    assert all(a is b for a, b in zip(r, out))
    _assert_equal(out, want_p)
    strided = tuple(np.full(s[::-1], 7.).T for s in shapes)
    assert not any(a.flags.c_contiguous for a in strided)
    r = mrcal_b200.project(p, lm, rows[:, None, :], get_gradients=True, out=strided)
    assert all(a is b for a, b in zip(r, strided))
    _assert_equal(strided, want_p)
    v = np.full((3, 3, 4), 7.).transpose(1, 2, 0)
    assert mrcal_b200.unproject(q, lm, rows[:, None, :], normalize=True, out=v) is v
    _assert_equal(v, want_u)
    # tensors
    tp, tq = torch.tensor(p, device="cuda"), torch.tensor(q, device="cuda")
    ti = torch.tensor(rows, device="cuda")[:, None, :]
    out = tuple(torch.full(s, 7., dtype=torch.float64, device="cuda") for s in shapes)
    strided = tuple(torch.full(s[::-1], 7., dtype=torch.float64, device="cuda").permute(*range(len(s) - 1, -1, -1))
                    for s in shapes)
    for o in (out, strided):
        r = mrcal_b200.project(tp, lm, ti, get_gradients=True, out=o)
        assert all(a is b for a, b in zip(r, o))
        _assert_equal(tuple(a.cpu().numpy() for a in o), want_p)
    v = torch.full((3, 3, 4), 7., dtype=torch.float64, device="cuda").permute(1, 2, 0)
    assert mrcal_b200.unproject(tq, lm, ti, normalize=True, out=v) is v
    _assert_equal(v.cpu().numpy(), want_u)
    # an out on the wrong device is refused before any work
    with pytest.raises(ValueError, match="out must be float64 on cuda"):
        mrcal_b200.project(tp, lm, ti, out=torch.empty(3, 4, 2, dtype=torch.float64))


def test_noncentral_cahvore_in_a_stack():
    torch = pytest.importorskip("torch")
    lm = "LENSMODEL_CAHVORE_linearity=0.37"
    rows = _rows(lm, 3)
    q = pixels(lm, rows[0], n=6)
    assert (rows[:, -3:] == 0.).all()
    ok = mrcal_b200.unproject(q[:, None, :], lm, rows, get_gradients=True)
    _assert_equal(tuple(a.cpu().numpy() for a in mrcal_b200.unproject(
        torch.tensor(q[:, None, :], device="cuda"), lm, torch.tensor(rows, device="cuda"), get_gradients=True)), ok)
    rows[1, -2] = 0.01
    for kw in ({}, {"normalize": True}, {"get_gradients": True}):
        with pytest.raises(RuntimeError, match=r"So I cannot unproject\(CAHVORE,E!=0\)"):
            mrcal_b200.unproject(q[:, None, :], lm, rows, **kw)
        with pytest.raises(RuntimeError, match=r"So I cannot unproject\(CAHVORE,E!=0\)"):
            mrcal_b200.unproject(torch.tensor(q[:, None, :], device="cuda"), lm, torch.tensor(rows, device="cuda"),
                                 **kw)
    # projecting is fine with any E
    mrcal_b200.project(_points(6, 2)[:, None, :], lm, rows)


def test_failed_pixel_inside_a_broadcast():
    # the pixel of test_project_gpu.py's test_unproject_reports_failure_as_nan that no ray projects to, in every row
    lm = "LENSMODEL_OPENCV8"
    intr = np.array((1000., 1000., 500., 500., 0., 0., 0., 0., 0., 1., 0., 0.))
    rows = np.stack((intr, intr * (1. + 1e-3 * np.arange(12))))
    q = np.array(((5500., 500.), (600., 520.)))
    for normalize in (False, True):
        v, dv_dq, dv_di = mrcal_b200.unproject(q, lm, rows[:, None, :], normalize=normalize, get_gradients=True)
        assert np.isnan(v[:, 0, :2]).all() and np.isnan(dv_dq[:, 0]).all() and np.isnan(dv_di[:, 0]).all()
        assert np.isfinite(v[:, 1]).all() and np.isfinite(dv_dq[:, 1]).all() and np.isfinite(dv_di[:, 1]).all()
    v = mrcal_b200.unproject(q, lm, rows[:, None, :], normalize=True)
    assert (v[:, 0] == 0.).all() and np.abs(np.linalg.norm(v[:, 1], axis=-1) - 1.).max() < 1e-14
    v = mrcal_b200.unproject(q, lm, rows[:, None, :])
    assert np.isnan(v[:, 0, :2]).all() and np.isfinite(v[:, 1]).all()


@pytest.mark.parametrize("kind", tuple(CLOSED_FORM.values()))
def test_closed_form_stacked_fxycxy(kind):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(9)
    fxycxy = np.array((1100., 1050., 1000., 700.)) * (1. + 1e-2 * rng.standard_normal((4, 4)))
    for fn in ("project", "unproject"):
        f = getattr(mrcal_b200, f"{fn}_{kind}")
        x = closed_form_points(fn).reshape(4, 5, -1)
        got = f(x, fxycxy[:, None, :], get_gradients=True)
        assert len(got) == 2
        for k in range(4):
            _assert_equal(tuple(a[k] for a in got), f(x[k], fxycxy[k], get_gradients=True))
            _assert_equal(f(x, fxycxy[:, None, :])[k], f(x[k], fxycxy[k]))
        out = (np.empty(got[0].shape), np.empty(got[1].shape[::-1]).T)
        r = f(x, fxycxy[:, None, :], get_gradients=True, out=out)
        assert all(a is b for a, b in zip(r, out))
        _assert_equal(out, got)
        # tensors, with the default core made on the points' device
        tx = torch.tensor(x, device="cuda")
        _assert_equal(tuple(a.cpu().numpy() for a in f(tx, torch.tensor(fxycxy, device="cuda")[:, None, :],
                                                       get_gradients=True)), got)
        _assert_equal(f(tx).cpu().numpy(), f(x))
