"""match_feature() without a GPU: the numpy restatement of its definition against OpenCV's stored outputs
(tests/golden/match_feature.npz, from make_match_golden.py), the degenerate values of OpenCV's rule, apply_homography()'s
bits and the argument refusals, which are all decided on the host before any launch."""
import os

import numpy as np
import pytest

import mrcal_b200
import match_np
import remap_np

FIXTURE = os.path.join(os.path.dirname(__file__), "golden", "match_feature.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(FIXTURE)


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
@pytest.mark.parametrize("method", range(6))
def test_restatement_matches_opencv(golden, dtype, method):
    """Within 1e-5 of the output's largest magnitude (OpenCV's own float rounding), the same discrete optimum"""
    cut, template = golden[dtype + "_cut"], golden[dtype + "_template"]
    cv = golden[f"{dtype}_m{method}"]
    mine = match_np.match_output(cut, template, method)
    assert mine.shape == cv.shape and mine.dtype == np.float32
    assert np.abs(mine.astype(float) - cv).max() <= 1e-5 * np.abs(cv).max()
    pick = np.argmin if method in (mrcal_b200.TM_SQDIFF, mrcal_b200.TM_SQDIFF_NORMED) else np.argmax
    assert pick(mine) == pick(cv)


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_template_map_and_remap_match_opencv(golden, dtype):
    """The template's map as match_feature() forms it, and the restated remap of it, give OpenCV's template"""
    H10 = golden[dtype + "_H10"].astype(np.float32)
    x0, y0 = golden[dtype + "_q1_template_min"]
    th, tw = golden[dtype + "_template"].shape
    grid = np.stack(np.meshgrid(np.arange(x0, x0 + tw), np.arange(y0, y0 + th)), -1).astype(np.float32)
    mapxy = mrcal_b200.apply_homography(np.linalg.inv(H10), grid)
    np.testing.assert_array_equal(mapxy.view(np.uint32), golden[dtype + "_mapxy"].view(np.uint32))
    np.testing.assert_array_equal(remap_np.remap(golden[dtype + "_image0"], mapxy), golden[dtype + "_template"])


DEGENERATE = {"flat_template": 1., "flat_window": 0., "zero_window_ccorr": 0., "zero_window_sqdiff": 1.,
              "sqdiff_beyond": 1., "band_sqdiff": 1., "band_ccorr": 1., "band_ccoeff": -1.}


@pytest.mark.parametrize("case", sorted(DEGENERATE))
def test_degenerate_values_are_opencvs(golden, case):
    p = f"degenerate_{case}_"
    cut, template, method = golden[p + "cut"], golden[p + "template"], int(golden[p + "method"])
    expected = np.full(golden[p + "result"].shape, DEGENERATE[case], np.float32)
    np.testing.assert_array_equal(golden[p + "result"], expected)
    np.testing.assert_array_equal(match_np.match_output(cut, template, method), expected)
    # the same windows in float32 give the same values
    np.testing.assert_array_equal(match_np.match_output(cut.astype(np.float32), template.astype(np.float32), method),
                                  expected)


def test_band_cases_are_in_the_band(golden):
    """The band cases really have 1 <= |num| / t < 1.125, in exact arithmetic"""
    for case, method in (("band_sqdiff", 1), ("band_ccorr", 3), ("band_ccoeff", 5)):
        p = f"degenerate_{case}_"
        I = golden[p + "cut"].astype(np.int64).ravel()
        T = golden[p + "template"].astype(np.int64).ravel()
        n = I.size
        if method == 1:
            num, t2 = (I - T) @ (I - T), (I @ I) * (T @ T)
        elif method == 3:
            num, t2 = I @ T, (I @ I) * (T @ T)
        else:
            Ic, Tc = n * I - I.sum(), n * T - T.sum()
            num, t2 = Ic @ Tc, (Ic @ Ic) * (Tc @ Tc)
        assert num * num >= t2 and num * num < 1.125 ** 2 * t2, case


def test_opencv_refusals_recorded(golden):
    assert golden["refuses_uint16"] == 1 and golden["refuses_mixed"] == 1 and golden["refuses_small_cut"] == 1


@pytest.mark.parametrize("dtype", [np.float32, np.float64])
def test_apply_homography_bits(dtype):
    """Each operation rounded on its own, in the inputs' precision, broadcasting"""
    rng = np.random.default_rng(3)
    H = rng.normal(size=(5, 1, 3, 3)).astype(dtype)
    q = (rng.uniform(-100, 4000, (7, 2))).astype(dtype)
    r = mrcal_b200.apply_homography(H, q)
    assert r.shape == (5, 7, 2) and r.dtype == dtype
    one = np.dtype(dtype).type
    for i in range(5):
        for j in range(7):
            h, (x, y) = H[i, 0], q[j]
            xyz = [one(one(one(h[k, 0] * x) + one(h[k, 1] * y)) + h[k, 2]) for k in range(3)]
            assert r[i, j, 0] == one(xyz[0] / xyz[2]) and r[i, j, 1] == one(xyz[1] / xyz[2])
    assert mrcal_b200.apply_homography(H.astype(np.float32), q.astype(np.float64)).dtype == np.float64


def test_constants_are_opencvs():
    assert (mrcal_b200.TM_SQDIFF, mrcal_b200.TM_SQDIFF_NORMED, mrcal_b200.TM_CCORR, mrcal_b200.TM_CCORR_NORMED,
            mrcal_b200.TM_CCOEFF, mrcal_b200.TM_CCOEFF_NORMED) == (0, 1, 2, 3, 4, 5)


def test_restated_subpixel_fit_is_the_least_squares_fit():
    """The closed-form pseudo-inverse gives lstsq's coefficients; the peak is that of the fitted quadratic"""
    rng = np.random.default_rng(5)
    mo = rng.uniform(0, 0.5, (5, 6)).astype(np.float32)
    mo[2, 3] = 1.
    status, at, value = match_np.optimum(mo, mrcal_b200.TM_CCORR_NORMED)
    assert status == match_np.MATCH_OK
    x, y = np.meshgrid(np.arange(3) - 1., np.arange(3) - 1.)
    x, y = x.ravel(), y.ravel()
    M = np.stack((np.ones(9), x, y, x * x, x * y, y * y), 1)
    c = np.linalg.lstsq(M, mo[1:4, 2:5].ravel().astype(float), rcond=None)[0]
    xy = -np.array((2 * c[1] * c[5] - c[2] * c[4], 2 * c[2] * c[3] - c[1] * c[4])) / (4 * c[3] * c[5] - c[4] ** 2)
    np.testing.assert_allclose(at, np.array((3., 2.)) + xy, atol=1e-12)


####################################################################################################
# refusals: all decided before any launch
####################################################################################################
def _args(**kw):
    img = np.zeros((40, 50), np.uint8)
    a = dict(image0=img, image1=img, q0=np.array((25., 20.)), search_radius1=3, template_size1=5,
             q1_estimate=np.array((25., 20.)))
    a.update(kw)
    return a


@pytest.mark.parametrize("kw, match", [
    (dict(template_size1=(5, 5, 5)), "of length 2 OR a scalar"),
    (dict(template_size1=0), "integer > 0"),
    (dict(template_size1=5.), "integer > 0"),
    (dict(image0=np.zeros((40, 50, 3), np.uint8)), "grayscale"),
    (dict(image1=np.zeros((40,), np.uint8)), "grayscale"),
    (dict(H10=np.eye(3)), "Exactly one of"),
    (dict(q1_estimate=None), "Exactly one of"),
    (dict(image0=np.zeros((40, 50), np.uint16), image1=np.zeros((40, 50), np.uint16)), "uint8 and float32"),
    (dict(image1=np.zeros((40, 50), np.float32)), "same dtype"),
    (dict(method=6), "TM_"),
    (dict(search_radius1=2.5), "integer"),
    (dict(visualize=True), "gnuplotlib"),
    (dict(q0=np.array((1., 20.)), q1_estimate=np.array((1., 20.))), "left edge in image1"),
    (dict(q0=np.array((25., 1.)), q1_estimate=np.array((25., 1.))), "top edge in image1"),
    (dict(q0=np.array((48., 20.)), q1_estimate=np.array((48., 20.))), "right edge in image1"),
    (dict(q0=np.array((25., 39.)), q1_estimate=np.array((25., 39.))), "bottom edge in image1"),
    (dict(q0=np.array((1., 20.))), "left edge in image0"),
    (dict(q0=np.array((48., 20.))), "right edge in image0"),
    (dict(search_radius1=-1), "smaller than the template"),
])
def test_single_call_refusals(kw, match):
    with pytest.raises(RuntimeError, match=match):
        mrcal_b200.match_feature(**_args(**kw))


@pytest.mark.parametrize("kw, match", [
    (dict(q0=np.array((np.nan, 20.)), q1_estimate=None, H10=np.eye(3)), "left edge in image1"),
    (dict(q0=np.array((25., np.nan)), q1_estimate=None, H10=np.eye(3)), "left edge in image1"),   # 0 * NaN is NaN
    (dict(q1_estimate=np.array((25., np.nan))), "top edge in image1"),
    (dict(q0=np.array((np.inf, 20.)), q1_estimate=None, H10=np.eye(3)), "left edge in image1"),
    (dict(q1_estimate=np.array((np.nan, 20.))), "left edge in image1"),
    (dict(q1_estimate=np.array((1e300, 20.))), "left edge in image1"),
    (dict(q1_estimate=np.array((1e15, 20.))), "right edge in image1"),
    (dict(q1_estimate=None, H10=np.array(((1., 0., np.nan), (0., 1., 0.), (0., 0., 1.)))), "left edge in image1"),
    (dict(q1_estimate=None, H10=np.array(((1., 0., 0.), (0., 1., 0.), (0., 0., 1e-40)))), "left edge in image1"),
])
def test_single_call_refuses_a_nonfinite_estimate(kw, match):
    """A q1_estimate that is not a finite pixel is outside image 1, as the reference's integer cast makes it (NaN, inf
    and anything beyond int64 become INT64_MIN); a batch reports it as a status"""
    with pytest.raises(RuntimeError, match=match):
        mrcal_b200.match_feature(**_args(**kw))
    a = _args(**kw)
    a["q0"] = np.stack((a["q0"], a["q0"]))
    q1, d = mrcal_b200.match_feature(**a)
    assert np.all(np.isnan(q1)) and list(d["status"]) == [mrcal_b200.MATCH_OUTSIDE_IMAGE1] * 2


def test_singular_homography_raises_in_a_single_call():
    H = np.array(((1., 0., 0.), (1., 0., 0.), (0., 0., 1.)))
    a = _args(H10=H, q0=np.array((25., 20.)))
    del a["q1_estimate"]
    a["q0"] = np.array((25., 25.))
    with pytest.raises(np.linalg.LinAlgError):
        mrcal_b200.match_feature(**a)
