"""CPU: the restatement the GPU tests of unproject(get_gradients=True), model_resolution__deg_pixel() and
stereo_pair_diff() compare against (tests/unproject_np.py), checked against central differences of the compiled
reference, np.linalg.eigvalsh and the pinhole closed form; and the refusals that come before any device work."""
import numpy as np
import pytest

import mrcal_b200
from test_project_gpu import _unproject_intrinsics

LMS = ("LENSMODEL_PINHOLE", "LENSMODEL_STEREOGRAPHIC", "LENSMODEL_LONLAT", "LENSMODEL_LATLON", "LENSMODEL_OPENCV8",
       "LENSMODEL_CAHVOR", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100")


def _pixels(intr, n=5):
    return intr[2:4] + np.random.default_rng(3).uniform(-0.5, 0.5, (n, 2)) * intr[2:4]


@pytest.mark.parametrize("lm", LMS)
def test_restated_gradients_match_central_differences(ref, lm):
    import unproject_np as U
    intr = _unproject_intrinsics(lm)
    q = _pixels(intr)
    for normalize in (False, True):
        v, dv_dq, dv_di = U.unproject(q, lm, intr, normalize=normalize, get_gradients=True)
        f = lambda qq, ii: U.unproject(qq, lm, ii, normalize=normalize, get_gradients=True)[0]
        for k in range(2):
            h = np.zeros(2)
            h[k] = 1e-2
            num = (f(q + h, intr) - f(q - h, intr)) / 2e-2
            assert np.abs(num - dv_dq[:, :, k]).max() <= 1e-6 * np.abs(dv_dq).max()
        cols = range(len(intr)) if len(intr) < 20 else (0, 1, 2, 3, 30, 41, 57)
        for c in cols:
            h = 1e-4 * max(abs(intr[c]), 1e-1)
            ip, im = intr.copy(), intr.copy()
            ip[c] += h
            im[c] -= h
            num = (f(q, ip) - f(q, im)) / (2 * h)
            assert np.abs(num - dv_di[:, :, c]).max() <= 1e-6 * np.abs(dv_di).max() + 1e-12, f"column {c}"
        if normalize:
            assert np.abs(np.linalg.norm(v, axis=-1) - 1.).max() < 1e-14
            assert np.abs(U.unproject(q, lm, intr, normalize=True) - v).max() < 1e-12


def test_restated_resolution_eigenvalues():
    import unproject_np as U
    rng = np.random.default_rng(0)
    M = rng.normal(size=(50, 2, 2)) * 1000.
    l = np.linalg.eigvalsh(np.swapaxes(M, -1, -2) @ M)
    assert np.allclose(U.resolution_from_M(M, "min"), np.degrees(1. / np.sqrt(l[:, 1])), rtol=1e-12)
    assert np.allclose(U.resolution_from_M(M, "max"), np.degrees(1. / np.sqrt(l[:, 0])), rtol=1e-9)
    # the basis perpendicular to v is orthonormal and perpendicular
    v = rng.normal(size=(20, 3))
    v /= np.linalg.norm(v, axis=-1, keepdims=True)
    B = U.perpendicular_basis(v)
    assert np.abs(np.einsum("ni,nij->nj", v, B)).max() < 1e-14
    assert np.abs(np.swapaxes(B, -1, -2) @ B - np.eye(2)).max() < 1e-14


def test_restated_pinhole_resolution_and_reprojection(ref):
    import unproject_np as U
    f, c = 1234., np.array((499.5, 399.5))
    intr = np.array((f, f, *c))
    r = U.model_resolution(c[None], "LENSMODEL_PINHOLE", intr, "mean")
    assert abs(r[0] - np.degrees(np.arctan(1. / f))) < 1e-6 * r[0]
    # a second pinhole of focal length f2 behind the same rotation-free pose: q1 - c = f2/f (q - c) at infinity; with a
    # baseline t at distance d along the optical axis of the grid's centre, the centre moves by f2 t/d
    q = c + np.random.default_rng(1).uniform(-300., 300., (10, 2))
    f2 = 1100.
    Rt = np.vstack((np.eye(3), np.zeros(3)))
    q1 = U.reproject(q, "LENSMODEL_PINHOLE", intr, "LENSMODEL_PINHOLE", np.array((f2, f2, *c)), Rt, 1.)
    assert np.abs(q1 - (c + f2 / f * (q - c))).max() < 1e-9
    Rt[3] = (0.1, 0., 0.)
    q1 = U.reproject(c[None], "LENSMODEL_PINHOLE", intr, "LENSMODEL_PINHOLE", intr, Rt, 5.)
    assert np.abs(q1[0] - (c + (f * 0.1 / 5., 0.))).max() < 1e-9


def _pinhole(W=1000, H=800):
    return mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", np.array((1000., 1000., (W - 1) / 2., (H - 1) / 2.))),
                                  imagersize=(W, H))


def test_refusals_before_device_work():
    m = _pinhole()
    with pytest.raises(RuntimeError, match=r"Mode must be one of \('min','max','mean','eccentricity'\)"):
        mrcal_b200.model_resolution__deg_pixel(np.zeros(2), m, mode="median")
    with pytest.raises(RuntimeError, match="Exactly 2 model_pairs are expected"):
        mrcal_b200.stereo_pair_diff(((m, m),))
    with pytest.raises(RuntimeError, match="Exactly 2 model_pairs are expected"):
        mrcal_b200.stereo_pair_diff(((m, m), (m, m), (m, m)))
    with pytest.raises(RuntimeError, match="first camera in each given pair MUST have identical imager"):
        mrcal_b200.stereo_pair_diff(((m, m), (_pinhole(1000, 700), m)))
    with pytest.raises(RuntimeError, match="second camera in each given pair must have identical imager"):
        mrcal_b200.stereo_pair_diff(((m, m), (m, _pinhole(1000, 700))))
    cahvore = mrcal_b200.cameramodel(
        intrinsics=("LENSMODEL_CAHVORE_linearity=0.00",
                    np.array((1000., 1000., 499.5, 399.5, 0., 0., 0., 0., 0., 0.01, 0.02, 0.03))),
        imagersize=(1000, 800))
    with pytest.raises(RuntimeError, match="only valid at infinity"):
        mrcal_b200.stereo_pair_diff(((cahvore, m), (m, m)), distance=3.)
