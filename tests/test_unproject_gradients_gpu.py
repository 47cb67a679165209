"""unproject(normalize=, get_gradients=) and the closed-form project_* / unproject_* functions (csrc/unproject.cuh,
csrc/project.cu) against the reference's algorithm restated in tests/unproject_np.py on the compiled reference, and
against the identities the gradients must satisfy. Where oracle/_ref is not built, the restatement's answers stored in
tests/golden/unproject_gradients.npz (tests/golden/make_unproject_golden.py) stand in for it."""
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import synthetic
from test_project_gpu import MODELS, _unproject_intrinsics

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "unproject_gradients.npz")
CLOSED_FORM = {"LENSMODEL_PINHOLE": "pinhole", "LENSMODEL_STEREOGRAPHIC": "stereographic",
               "LENSMODEL_LONLAT": "lonlat", "LENSMODEL_LATLON": "latlon"}


def fingerprint(args):
    out = []
    for a in args:
        if isinstance(a, np.ndarray) or isinstance(a, (float, int)) and not isinstance(a, bool):
            a = np.asarray(a, np.float64)
            out += [a.sum(), (a * a).sum()]
    return np.array(out)


class Restatement:
    """tests/unproject_np.py on the compiled reference. call(key, method, *args): the answer of unproject_np.<method>"""

    def call(self, key, method, *args):
        import unproject_np
        r = getattr(unproject_np, method)(*args)
        return r if isinstance(r, tuple) else (r,)


class StoredRestatement:
    """The restatement's answers stored by tests/golden/make_unproject_golden.py, each given only for arguments with
    the stored fingerprints (sums and sums of squares)"""

    def __init__(self):
        self.d = np.load(GOLDEN)

    def call(self, key, method, *args):
        assert np.allclose(fingerprint(args), self.d[f"{key}/in"], rtol=1e-12, atol=1e-12), f"{key}: arguments differ"
        out = []
        while f"{key}/out{len(out)}" in self.d:
            out.append(self.d[f"{key}/out{len(out)}"])
        return tuple(out)


@pytest.fixture(scope="module")
def reference():
    from oracle import ref
    return Restatement() if ref.available() else StoredRestatement()


def behind_ok(lm):
    return bool(mrcal_b200.lensmodel_metadata_and_config(lm)["can_project_behind_camera"])


def pixels(lm, intr, n=30, seed=5):
    """pixels within the central 60% of the synthetic camera's imager, where every test model unprojects"""
    rng = np.random.default_rng(seed)
    return intr[2:4] + rng.uniform(-0.6, 0.6, (n, 2)) * intr[2:4]


def closed_form_points(fn, seed=7):
    rng = np.random.default_rng(seed)
    if fn == "project":
        p = rng.uniform(-1., 1., (20, 3))
        p[:, 2] += 3.
        return p
    return rng.uniform(-0.5, 0.5, (20, 2)) * (800., 600.) + (1000., 700.)


FXYCXY = np.array((1100., 1050., 1000., 700.))

# pixels of rays 95, 100 and 110 degrees off the axis. This CAHVORE sees them, but cannot project behind the camera, so
# the Newton solve's ray (z < 0) is flipped to the front, and the gradient path returns another magnitude
FLIPPED_LM = "LENSMODEL_CAHVORE_linearity=-0.25"
FLIPPED_Q = np.array(((4797.88, 2653.98), (-997.18, 2728.30), (4037.52, -2526.89)))


def reference_calls():
    """(key, method, args) of every call these tests make of the restatement"""
    for lm in MODELS:
        intr = _unproject_intrinsics(lm)
        q = pixels(lm, intr)
        for normalize in (False, True):
            yield f"unproject/{lm}/{normalize}", "unproject", (q, lm, intr, normalize, True, behind_ok(lm))
    for normalize in (False, True):
        yield (f"flipped/{FLIPPED_LM}/{normalize}", "unproject",
               (FLIPPED_Q, FLIPPED_LM, _unproject_intrinsics(FLIPPED_LM), normalize, True, behind_ok(FLIPPED_LM)))
    for kind in CLOSED_FORM.values():
        for fn in ("project", "unproject"):
            yield f"closed_form/{fn}_{kind}", "closed_form", (fn, kind, closed_form_points(fn), FXYCXY)


def tol(ref):
    return 1e-9 * (1. + np.abs(ref).max())


@pytest.mark.parametrize("lm", MODELS)
def test_unproject_gradients_match_reference(reference, lm):
    intr = _unproject_intrinsics(lm)
    q = pixels(lm, intr)
    for normalize in (False, True):
        v_ref, dv_dq_ref, dv_di_ref = reference.call(f"unproject/{lm}/{normalize}", "unproject",
                                                     q, lm, intr, normalize, True, behind_ok(lm))
        v, dv_dq, dv_di = mrcal_b200.unproject(q, lm, intr, normalize=normalize, get_gradients=True)
        assert v.shape == (len(q), 3) and dv_dq.shape == (len(q), 3, 2) and dv_di.shape == (len(q), 3, len(intr))
        assert np.abs(v - v_ref).max() <= tol(v_ref)
        assert np.abs(dv_dq - dv_dq_ref).max() <= tol(dv_dq_ref)
        assert np.abs(dv_di - dv_di_ref).max() <= tol(dv_di_ref)


@pytest.mark.parametrize("lm", MODELS)
def test_unproject_gradient_identities(lm):
    intr = _unproject_intrinsics(lm)
    q = pixels(lm, intr)
    v, dv_dq, dv_di = mrcal_b200.unproject(q, lm, intr, get_gradients=True)
    _, dq_dv, dq_di = mrcal_b200.project(v, lm, intr, get_gradients=True)
    assert np.abs(dq_dv @ dv_dq - np.eye(2)).max() < 1e-9
    assert np.abs(dq_dv @ dv_di + dq_di).max() < 1e-9 * (1. + np.abs(dq_di).max())
    # the gradient route: the same direction as the plain unprojection, v = unproject_stereographic(u)
    v0 = mrcal_b200.unproject(q, lm, intr)
    n = lambda a: a / np.linalg.norm(a, axis=-1, keepdims=True)
    assert np.abs(n(v) - n(v0)).max() < 1e-12
    if lm not in CLOSED_FORM:
        assert np.abs(v[:, 2] - (1. - 0.25 * (v[:, :2] ** 2).sum(-1))).max() < 1e-14
    vn, dvn_dq, dvn_di = mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)
    assert np.abs(np.linalg.norm(vn, axis=-1) - 1.).max() < 1e-14
    assert np.abs(np.einsum("ni,nij->nj", vn, dvn_dq)).max() < 1e-12 * np.abs(dvn_dq).max()
    assert np.abs(np.einsum("ni,nij->nj", vn, dvn_di)).max() < 1e-12 * (1. + np.abs(dvn_di).max())
    assert np.abs(mrcal_b200.unproject(q, lm, intr, normalize=True) - vn).max() < 1e-14


def _central_difference(f, x, h):
    J = []
    for k in range(x.size):
        d = np.zeros(x.size)
        d[k] = h[k] if np.ndim(h) else h
        J.append((f(x + d) - f(x - d)) / (2. * d[k]))
    return np.stack(J, -1)


@pytest.mark.parametrize("lm", MODELS)
def test_unproject_gradients_central_differences(lm):
    intr = _unproject_intrinsics(lm)
    q = pixels(lm, intr, n=6)
    v, dv_dq, dv_di = mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)
    for i in range(len(q)):
        Jq = _central_difference(lambda x: mrcal_b200.unproject(x, lm, intr, normalize=True), q[i], 1e-2)
        assert np.abs(Jq - dv_dq[i]).max() <= 1e-6 * np.abs(dv_dq[i]).max()
    if lm.startswith("LENSMODEL_SPLINED"):
        cols = np.r_[0:4, np.flatnonzero(np.abs(dv_di).max(axis=(0, 1)) > 0)[4::7]]
    else:
        cols = np.arange(len(intr))
    if lm.startswith("LENSMODEL_CAHVORE"):
        cols = cols[:-3]   # E stays 0: a noncentral model does not unproject
    for c in cols:
        h = 1e-4 * max(abs(intr[c]), 1e-1)

        def f(x):
            i2 = intr.copy()
            i2[c] = x[0]
            return mrcal_b200.unproject(q, lm, i2, normalize=True)
        Ji = _central_difference(f, np.array([intr[c]]), h)[..., 0]
        scale = np.abs(dv_di[:, :, c]).max()
        assert np.abs(Ji - dv_di[:, :, c]).max() <= 1e-6 * scale + 1e-12, f"column {c}"


def test_unproject_gradients_flipped_point(reference):
    lm, q = FLIPPED_LM, FLIPPED_Q
    intr = _unproject_intrinsics(lm)
    assert not behind_ok(lm)
    v0 = mrcal_b200.unproject(q, lm, intr)
    assert (v0[:, 2] > 0).all()
    for normalize in (False, True):
        refs = reference.call(f"flipped/{lm}/{normalize}", "unproject", q, lm, intr, normalize, True, behind_ok(lm))
        got = mrcal_b200.unproject(q, lm, intr, normalize=normalize, get_gradients=True)
        for a, b in zip(got, refs):
            assert np.all(np.isfinite(a)) and np.abs(a - b).max() <= tol(b)
    # the direction of mrcal_unproject()'s ray, another magnitude: unproject_stereographic(project_stereographic(v0))
    v, dv_dq, _ = mrcal_b200.unproject(q, lm, intr, get_gradients=True)
    n0, n = np.linalg.norm(v0, axis=-1), np.linalg.norm(v, axis=-1)
    assert np.abs(v / n[:, None] - v0 / n0[:, None]).max() < 1e-12
    assert (np.abs(n - n0) > 0.1 * n0).all()
    assert np.abs(v[:, 2] - (1. - 0.25 * (v[:, :2] ** 2).sum(-1))).max() < 1e-14
    # normalized, both paths give the same unit ray
    assert np.abs(mrcal_b200.unproject(q, lm, intr, normalize=True) -
                  mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)[0]).max() < 1e-14


@pytest.mark.parametrize("lm", ("LENSMODEL_LONLAT", "LENSMODEL_LATLON"))
def test_unit_rays_are_not_renormalized(lm):
    intr = _unproject_intrinsics(lm)
    q = pixels(lm, intr)
    v = mrcal_b200.unproject(q, lm, intr)
    assert np.array_equal(mrcal_b200.unproject(q, lm, intr, normalize=True), v)
    g = mrcal_b200.unproject(q, lm, intr, get_gradients=True)
    gn = mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)
    assert all(np.array_equal(a, b) for a, b in zip(g, gn))
    assert np.abs(gn[0] - v).max() <= 1e-15


def test_unproject_gradients_failure_is_nan():
    # the pixel of test_project_gpu.py's test_unproject_reports_failure_as_nan that no ray projects to
    lm = "LENSMODEL_OPENCV8"
    intr = np.array((1000., 1000., 500., 500., 0., 0., 0., 0., 0., 1., 0., 0.))
    q = np.array(((5500., 500.), (600., 520.)))
    for normalize in (False, True):
        v, dv_dq, dv_di = mrcal_b200.unproject(q, lm, intr, normalize=normalize, get_gradients=True)
        assert np.isnan(v[0, :2]).all() and np.isnan(dv_dq[0]).all() and np.isnan(dv_di[0]).all()
        assert np.isfinite(v[1]).all() and np.isfinite(dv_dq[1]).all() and np.isfinite(dv_di[1]).all()
    v = mrcal_b200.unproject(q, lm, intr, normalize=True)
    assert np.array_equal(v[0], (0., 0., 0.)) and abs(np.linalg.norm(v[1]) - 1.) < 1e-14


def test_unproject_gradients_refuse_noncentral_cahvore():
    lm = "LENSMODEL_CAHVORE_linearity=0.37"
    intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
    with pytest.raises(RuntimeError, match="central"):
        mrcal_b200.unproject(np.array(((100., 200.),)), lm, intr, get_gradients=True)


@pytest.mark.parametrize("lm", ("LENSMODEL_OPENCV8", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100",
                                "LENSMODEL_LONLAT"))
def test_unproject_gradients_broadcast(lm):
    intr = _unproject_intrinsics(lm)
    q = pixels(lm, intr, n=24)
    flat = mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True)
    shaped = mrcal_b200.unproject(q.reshape(2, 3, 4, 2), lm, intr, normalize=True, get_gradients=True)
    for a, b, tail in zip(flat, shaped, ((3,), (3, 2), (3, len(intr)))):
        assert b.shape == (2, 3, 4) + tail
        assert np.array_equal(b.reshape(a.shape), a)
    one = mrcal_b200.unproject(q[0], lm, intr, get_gradients=True)
    assert one[0].shape == (3,) and one[1].shape == (3, 2) and one[2].shape == (3, len(intr))


@pytest.mark.parametrize("kind", tuple(CLOSED_FORM.values()))
def test_closed_form_functions(reference, kind):
    for fn in ("project", "unproject"):
        x = closed_form_points(fn)
        out_ref, g_ref = reference.call(f"closed_form/{fn}_{kind}", "closed_form", fn, kind, x, FXYCXY)
        f = getattr(mrcal_b200, f"{fn}_{kind}")
        out, g = f(x, FXYCXY, get_gradients=True)
        assert np.abs(out - out_ref).max() <= tol(out_ref)
        assert np.abs(g - g_ref).max() <= tol(g_ref)
        assert np.array_equal(f(x, FXYCXY), out)
    # the default core is f = 1, c = 0
    p = closed_form_points("project")
    assert np.abs(getattr(mrcal_b200, f"project_{kind}")(p) -
                  getattr(mrcal_b200, f"project_{kind}")(p, np.array((1., 1., 0., 0.)))).max() == 0.
