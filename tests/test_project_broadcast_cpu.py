"""The refusals of project(), unproject() and the closed-form project_* / unproject_* over stacked intrinsics and
torch tensors, and of the C entries mrcal_b200_project[_device](): each is raised before any device work, so these
run without a GPU."""
import ctypes as C

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import _capi

LM = "LENSMODEL_OPENCV8"
INTR = np.array((1000., 1000., 500., 500., 0.1, -0.05, 0., 0., 0., 0., 0., 0.))


def _calls():
    """(function, its operand's width, the intrinsics): every function that takes the stacked intrinsics"""
    yield (lambda x, i, **kw: mrcal_b200.project(x, LM, i, **kw)), 3, INTR
    yield (lambda x, i, **kw: mrcal_b200.unproject(x, LM, i, **kw)), 2, INTR
    for kind in ("pinhole", "stereographic", "lonlat", "latlon"):
        yield getattr(mrcal_b200, f"project_{kind}"), 3, INTR[:4]
        yield getattr(mrcal_b200, f"unproject_{kind}"), 2, INTR[:4]


def test_numpy_refusals():
    for f, w, intr in _calls():
        x = np.zeros((4, w))
        with pytest.raises(ValueError, match=r"must have shape \(\.\.\.,%d\); got \(4, %d\)" % (w, w + 1)):
            f(np.zeros((4, w + 1)), intr)
        with pytest.raises(ValueError, match=r"must have shape \(\.\.\.,%d\)" % len(intr)):
            f(x, intr[:-1])
        with pytest.raises(ValueError, match="do not broadcast"):
            f(x, np.tile(intr, (3, 1)))
        with pytest.raises(ValueError, match="at most 8 broadcast dimensions are supported; got 9"):
            f(np.zeros((1,) * 9 + (w,)), intr)
        # lists are arrays
        with pytest.raises(ValueError, match="do not broadcast"):
            f(x.tolist(), np.tile(intr, (3, 1)).tolist())
        with pytest.raises(ValueError, match=r"out must have shape \(4, %d\)" % (5 - w)):
            f(x, intr, out=np.zeros((4, w)))
        with pytest.raises(ValueError, match="out must be float64"):
            f(x, intr, out=np.zeros((4, 5 - w), np.float32))
        with pytest.raises(ValueError, match="out must be a tuple of"):
            f(x, intr, get_gradients=True, out=np.zeros((4, 5 - w)))


def test_tensor_refusals():
    torch = pytest.importorskip("torch")
    for f, w, intr in _calls():
        x = np.zeros((4, w))
        tx, ti = torch.zeros(4, w, dtype=torch.float64), torch.tensor(intr)
        with pytest.raises(RuntimeError, match="must all be numpy arrays or all be torch CUDA tensors"):
            f(x, ti)
        with pytest.raises(RuntimeError, match="must all be numpy arrays or all be torch CUDA tensors"):
            f(tx, intr)
        with pytest.raises(RuntimeError, match="must all be numpy arrays or all be torch CUDA tensors"):
            f(x, intr, out=torch.zeros(4, 5 - w, dtype=torch.float64))
        # CPU tensors, float32 tensors
        with pytest.raises(ValueError, match="must be CUDA float64 tensors"):
            f(tx, ti)
        with pytest.raises(ValueError, match="must be CUDA float64 tensors"):
            f(tx.float(), ti.float())


def _c_args(ndim, shape):
    shape = np.array(shape, np.int64)
    st = np.zeros(max(ndim, 1), np.int64)
    buf = np.zeros(64)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    return (ndim, p(shape), p(buf), p(st), p(buf), p(st), p(buf), None, None)


def test_c_entries_refuse_before_device_work():
    lm = mrcal_b200.api._lensmodel(LM)
    for name, extra in (("mrcal_b200_project", ()), ("mrcal_b200_project_device", (None,))):
        f = getattr(_capi.lib, name)
        assert not f(C.byref(lm), 0, 9, *_c_args(9, (1,) * 9)[1:], *extra)
        assert "at most 8 broadcast dimensions are supported; got 9" in _capi.last_error()
        assert not f(C.byref(lm), 8, 1, *_c_args(1, (4,))[1:], *extra)
        assert "invalid flags 0x8" in _capi.last_error()
        # normalize only unprojects
        assert not f(C.byref(lm), 4, 1, *_c_args(1, (4,))[1:], *extra)
        assert "invalid flags 0x4" in _capi.last_error()
        assert not f(C.byref(lm), 0, 1, *_c_args(1, (-1,))[1:], *extra)
        assert "negative size or stride" in _capi.last_error()
        # an empty call does nothing, and needs no device
        assert f(C.byref(lm), 3, 2, *_c_args(2, (5, 0))[1:], *extra)
