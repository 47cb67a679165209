"""mrcal_project() / mrcal_unproject() of the C-ABI library (mrcal_b200/csrc/project.cu) against the compiled
reference: values and dq/dp of every lens model, the closed-form unprojections directly, the iterative ones
through the reference's own project() (the reference's iterative unproject needs libdogleg, which the oracle
build stubs out: oracle/ref.py unproject()). Where oracle/_ref is not built, the reference's answers stored in
tests/golden/project_reference.npz (tests/golden/make_project_golden.py) stand in for it."""
import collections
import os

import numpy as np
import pytest

import mrcal_b200
import problems
from mrcal_b200 import synthetic

pytestmark = pytest.mark.gpu

MODELS = ("LENSMODEL_PINHOLE", "LENSMODEL_STEREOGRAPHIC", "LENSMODEL_LONLAT", "LENSMODEL_LATLON",
          "LENSMODEL_OPENCV4", "LENSMODEL_OPENCV5", "LENSMODEL_OPENCV8", "LENSMODEL_OPENCV12", "LENSMODEL_CAHVOR",
          "LENSMODEL_CAHVORE_linearity=0.37", "LENSMODEL_CAHVORE_linearity=-0.25",
          "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100",
          "LENSMODEL_SPLINED_STEREOGRAPHIC_order=2_Nx=8_Ny=6_fov_x_deg=100")


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "project_reference.npz")


def _points(n, seed):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1., 1., (n, 3))
    p[:, 2] += 3.
    return p


def _unproject_intrinsics(lm):
    intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
    if lm.startswith("LENSMODEL_CAHVORE"):
        intr[-3:] = 0.   # the reference only unprojects central models (mrcal.c:3203-3214)
    return intr


class StoredReference:
    """The compiled reference's stored answers to the calls one test makes, in the order it makes them. A call is
    answered only if its arguments have the stored fingerprints (sum, sum of squares) of those the answer was
    computed for."""

    def __init__(self, test):
        self.test = test
        self.d = np.load(GOLDEN)
        self.calls = collections.Counter()

    def _answer(self, fn, lm, *args):
        k = self.calls[fn]
        self.calls[fn] += 1
        key = f"{self.test}/{lm}/{fn}/{k}"
        for i, a in enumerate(args):
            a = np.asarray(a, np.float64)
            # (loose enough for an unprojection that agrees with the reference's to 1e-9 per entry)
            assert np.allclose((a.sum(), (a * a).sum()), self.d[f"{key}/in{i}"], rtol=1e-9, atol=1e-6), f"{key}: argument {i} differs"
        out = []
        while f"{key}/out{len(out)}" in self.d:
            out.append(self.d[f"{key}/out{len(out)}"])
        return out[0] if len(out) == 1 else tuple(out)

    def project(self, p, lm, intr, gradients=False):
        r = self._answer("project", lm, p, intr)
        assert gradients == isinstance(r, tuple), "stored with gradients" if gradients else "stored without gradients"
        return r

    def project_with_intrinsics_gradient(self, p, lm, intr):
        # (q and dq/dp: those of the project() call this test made first, with the same arguments)
        q, dq_dp = self.d[f"{self.test}/{lm}/project/0/out0"], self.d[f"{self.test}/{lm}/project/0/out1"]
        return q, dq_dp, self._answer("project_with_intrinsics_gradient", lm, p, intr)

    def unproject(self, q, lm, intr):
        return self._answer("unproject", lm, q, intr)


@pytest.fixture
def reference(request):
    from oracle import ref
    return ref if ref.available() else StoredReference(request.node.originalname)


@pytest.mark.parametrize("lm", MODELS)
def test_project_matches_reference(reference, lm):
    ref = reference
    intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
    p = _points(40, 1)
    q_ref, g_ref = ref.project(p, lm, intr, gradients=True)
    q, g, gi = mrcal_b200.project(p, lm, intr, get_gradients=True)
    assert np.abs(q - q_ref).max() <= 1e-9 * (1. + np.abs(q_ref).max())
    assert np.abs(g - g_ref).max() <= 1e-9 * (1. + np.abs(g_ref).max())
    # the gradient with respect to the intrinsics: dense (N,2,Nintrinsics), mrcal.c:2866-2992
    q3, g3, gi_ref = ref.project_with_intrinsics_gradient(p, lm, intr)
    assert gi.shape == gi_ref.shape == (40, 2, len(intr))
    assert np.abs(gi - gi_ref).max() <= 1e-9 * (1. + np.abs(gi_ref).max())
    assert np.abs(g - g3).max() <= 1e-9 * (1. + np.abs(g3).max())
    # broadcasting over leading dimensions, and the no-gradient flavour
    q2 = mrcal_b200.project(p.reshape(8, 5, 3), lm, intr)
    # (another instantiation of the kernel: the compiler contracts its multiply-adds differently, last-bit differences)
    assert q2.shape == (8, 5, 2) and np.abs(q2.reshape(-1, 2) - q).max() <= 1e-12 * (1. + np.abs(q).max())


@pytest.mark.parametrize("lm", MODELS)
def test_unproject(reference, lm):
    ref = reference
    intr = _unproject_intrinsics(lm)
    p = _points(40, 2)
    q = ref.project(p, lm, intr)
    v = mrcal_b200.unproject(q, lm, intr)
    v_ref = ref.unproject(q, lm, intr)
    n = lambda a: a / np.linalg.norm(a, axis=-1, keepdims=True)
    assert np.abs(n(v) - n(p)).max() < 1e-9           # it inverts the projection
    assert np.abs(v - v_ref).max() < 1e-9             # ... with the reference's scale convention
    assert np.abs(ref.project(v, lm, intr) - q).max() < 1e-8


def test_unproject_refuses_noncentral_cahvore():
    lm = "LENSMODEL_CAHVORE_linearity=0.37"
    intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
    with pytest.raises(RuntimeError, match="central"):
        mrcal_b200.unproject(np.array(((100., 200.),)), lm, intr)


def test_unproject_reports_failure_as_nan():
    # a pixel no ray projects to: with only k4 = 1 the radial map is r / (1 + r^2) <= 0.5, and this pixel sits
    # at 5. NaN x,y, as mrcal.c:3247-3262
    lm = "LENSMODEL_OPENCV8"
    intr = np.array((1000., 1000., 500., 500., 0., 0., 0., 0., 0., 1., 0., 0.))
    v = mrcal_b200.unproject(np.array(((5500., 500.), (600., 520.))), lm, intr)
    assert np.isnan(v[0, 0]) and np.isnan(v[0, 1])
    assert np.isfinite(v[1]).all()
