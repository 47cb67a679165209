"""match_feature() on the device: its templates against transform_image() and OpenCV's remap, its match output against
the numpy restatement (tests/match_np.py) bit for bit for uint8 and within a float32 ulp for float32, the sub-pixel
optimum within 1e-9 px, every status, template shapes on and off the staged path, NaN, a batch of 20 000 features,
torch tensors, and a rectified pair ranged end to end through stereo_range()."""
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import stereo

import match_np
import remap_np

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(os.path.dirname(__file__), "golden", "match_feature.npz")


def _perspective(rng, N, shift):
    """N homographies near a translation by `shift`: a little rotation, scale, shear and perspective"""
    H = np.tile(np.eye(3), (N, 1, 1))
    H[:, :2, :2] += rng.uniform(-0.06, 0.06, (N, 2, 2))
    H[:, 2, :2] = rng.uniform(-2e-4, 2e-4, (N, 2))
    H[:, :2, 2] = shift + rng.uniform(-1.5, 1.5, (N, 2))
    return H


def _ulps(a, b):
    """|a - b| in float32 ulps of the larger; NaN where exactly one is NaN"""
    a, b = a.astype(np.float64), b.astype(np.float64)
    both_nan = np.isnan(a) & np.isnan(b)
    d = np.abs(a - b) / np.spacing(np.maximum(np.abs(a), np.abs(b)).astype(np.float32)).astype(np.float64)
    return np.where(both_nan | (a == b), 0., d)


def _check_against_restatement(image0, image1, q0, ts, r, method, H10=None, q1_estimate=None, exact=True):
    """A batched call against match_np.match_feature() feature by feature; returns the batched result"""
    res, _, templates = stereo._match_features(image0, image1, q0, r, ts, q1_estimate, H10, method, False,
                                               return_templates=True)
    run = np.flatnonzero(np.isin(res["status"], (stereo.MATCH_OK, stereo.MATCH_EDGE_PEAK)))
    for i in range(len(q0)):
        kw = dict(H10=H10[i] if H10 is not None and np.ndim(H10) == 3 else H10)
        if q1_estimate is not None:
            kw = dict(q1_estimate=q1_estimate[i] if np.ndim(q1_estimate) == 2 else q1_estimate)
        ref = match_np.match_feature(image0, image1, q0[i], search_radius1=r, template_size1=ts, method=method, **kw)
        assert res["status"][i] == ref["status"], i
        if ref["status"] not in (match_np.MATCH_OK, match_np.MATCH_EDGE_PEAK):
            assert res["matchoutput_image"][i] is None and np.all(np.isnan(res["q1"][i]))
            continue
        k = int(np.flatnonzero(run == i)[0])
        np.testing.assert_array_equal(templates[k], ref["template"])
        mo = res["matchoutput_image"][i]
        assert mo.shape == ref["matchoutput"].shape
        if exact:
            np.testing.assert_array_equal(mo.view(np.uint32), ref["matchoutput"].view(np.uint32))
        else:
            assert np.nanmax(_ulps(mo, ref["matchoutput"]), initial=0.) <= 1., i
        if ref["status"] == match_np.MATCH_OK:
            assert np.abs(res["at"][i] - ref["at"]).max() <= 1e-9
            assert np.abs(res["q1"][i] - ref["q1"]).max() <= 1e-9
            assert abs(res["value"][i] - ref["value"]) <= 1e-9 * max(1., abs(ref["value"]))
            np.testing.assert_array_equal(res["qshift"][i], ref["qshift"])
        else:
            assert np.all(np.isnan(res["q1"][i]))
    return res, templates


####################################################################################################
# templates
####################################################################################################
@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_templates_are_opencvs_remap(dtype):
    """The golden case: the device's template is cv2.remap()'s, bit for bit"""
    f = np.load(FIXTURE)
    H10 = f[dtype + "_H10"]
    th, tw = f[dtype + "_template"].shape
    centre = np.array(f[dtype + "_q1_template_min"]) + (np.array((tw, th)) - 1) / 2.
    q0 = mrcal_b200.apply_homography(np.linalg.inv(H10.astype(np.float32)), centre.astype(np.float32))
    res, _, templates = stereo._match_features(f[dtype + "_image0"], f[dtype + "_cut"], q0[None], 3, (tw, th), None,
                                               H10, mrcal_b200.TM_CCORR_NORMED, False, return_templates=True)
    assert res["status"][0] in (stereo.MATCH_OK, stereo.MATCH_EDGE_PEAK)
    np.testing.assert_array_equal(templates[0], f[dtype + "_template"])


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_templates_are_transform_image_on_the_same_maps(dtype):
    rng = np.random.default_rng(1)
    image0 = match_np.textured_image(120, 150, dtype, 3)
    image1 = match_np.textured_image(110, 140, dtype, 4)
    N, ts = 12, (9, 7)
    q0 = rng.uniform(30, 90, (N, 2))
    H10 = _perspective(rng, N, (-4., 3.))
    res, _, templates = stereo._match_features(image0, image1, q0, 5, ts, None, H10, 3, False, return_templates=True)
    run = np.flatnonzero(res["status"] <= stereo.MATCH_EDGE_PEAK)
    assert run.size == N
    H = H10.astype(np.float32)
    q1e = mrcal_b200.apply_homography(H, q0.astype(np.float32))
    tmin = np.round(q1e - (np.array(ts) - 1.) / 2.).astype(int)
    for k, i in enumerate(run):
        grid = np.stack(np.meshgrid(np.arange(tmin[i, 0], tmin[i, 0] + ts[0]),
                                    np.arange(tmin[i, 1], tmin[i, 1] + ts[1])), -1).astype(np.float32)
        mapxy = mrcal_b200.apply_homography(np.linalg.inv(H[i]), grid)
        np.testing.assert_array_equal(templates[k], mrcal_b200.transform_image(image0, mapxy))


####################################################################################################
# the match output and the optimum against the restatement
####################################################################################################
@pytest.mark.parametrize("method", range(6))
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_match_output_against_the_restatement(dtype, method):
    rng = np.random.default_rng(10 + method)
    image0 = match_np.textured_image(160, 200, dtype, 5)
    # image 1: image 0 shifted by (-6.4, 2.7), so the matches have a peak
    yy, xx = np.mgrid[0:150, 0:190].astype(np.float32)
    image1 = remap_np.remap(image0, np.stack((xx + np.float32(6.4), yy - np.float32(2.7)), -1))
    N = 24
    q0 = rng.uniform(25, 150, (N, 2))
    H10 = _perspective(rng, N, (-6.4, 2.7))
    _check_against_restatement(image0, image1, q0, (13, 11), 6, method, H10=H10, exact=dtype == np.uint8)


@pytest.mark.parametrize("ts", [7, 8, (12, 5), (5, 12)])
def test_odd_even_and_nonsquare_templates_with_q1_estimate(ts):
    rng = np.random.default_rng(20)
    image0 = match_np.textured_image(100, 120, np.uint8, 6)
    image1 = np.ascontiguousarray(image0[3:, 5:])
    q0 = rng.uniform(20, 80, (16, 2))
    q1e = q0 - (5., 3.) + rng.uniform(-2, 2, (16, 2))
    _check_against_restatement(image0, image1, q0, ts, 5, mrcal_b200.TM_CCOEFF_NORMED, q1_estimate=q1e)
    # one q1_estimate (2,) for every feature
    _check_against_restatement(image0, image1, q0[:4], ts, 5, mrcal_b200.TM_SQDIFF, q1_estimate=np.array((50., 40.)))


def test_template_too_large_for_the_staged_path():
    """A float32 template of 150 x 140 (84 KB) and its cut's rows exceed the 96 KB the staged path allows, so the kernel
    reads through L2; the output is still the restatement's"""
    image0 = match_np.textured_image(200, 220, np.float32, 7)
    image1 = np.ascontiguousarray(image0[1:, 2:])
    q0 = np.array(((110., 100.), (105., 96.)))
    _check_against_restatement(image0, image1, q0, (150, 140), 3, mrcal_b200.TM_CCORR_NORMED,
                               q1_estimate=q0 - (2., 1.), exact=False)


def test_nan_in_float_images():
    image0 = match_np.textured_image(90, 100, np.float32, 8)
    image1 = image0.copy()
    image1[40, 50] = np.nan
    image0[30:33, 60] = np.nan
    q0 = np.array(((50., 40.), (60., 31.), (30., 30.), (52., 44.)))
    for method in range(6):
        _check_against_restatement(image0, image1, q0, 9, 4, method, q1_estimate=q0 + 0.3, exact=False)


def test_strided_rows():
    big = match_np.textured_image(130, 170, np.uint8, 9)
    image0, image1 = big[5:120, 7:160], big[8:125, 3:150]
    q0 = np.array(((60., 50.), (80., 70.), (40., 90.)))
    _check_against_restatement(image0, image1, q0, 11, 6, mrcal_b200.TM_CCORR_NORMED, q1_estimate=q0 + (4., -3.))


####################################################################################################
# statuses and the single call
####################################################################################################
def test_every_status_and_the_single_calls():
    image0 = match_np.textured_image(100, 130, np.uint8, 12)
    image1 = match_np.textured_image(100, 130, np.uint8, 12)
    ramp = np.add.outer(np.arange(100), np.arange(130)).astype(np.uint8)
    ts, r = 9, 6
    q0 = np.array(((60., 50.),     # ok
                   (2., 50.),      # template outside image 1 (left)
                   (60., 98.),     # ... (bottom)
                   (2., 50.),      # template outside image 0: H10 translates by 60
                   (8., 50.),      # clipped at the left border
                   (124., 50.),    # ... right
                   (60., 7.),      # ... top
                   (60., 94.)))    # ... bottom
    H10 = np.tile(np.eye(3), (len(q0), 1, 1))
    H10[3, 0, 2] = 60.
    res, _ = _check_against_restatement(image0, image1, q0, ts, r, mrcal_b200.TM_CCORR_NORMED, H10=H10)
    assert list(res["status"][:4]) == [stereo.MATCH_OK, stereo.MATCH_OUTSIDE_IMAGE1, stereo.MATCH_OUTSIDE_IMAGE1,
                                       stereo.MATCH_OUTSIDE_IMAGE0]
    shapes = [res["matchoutput_image"][i].shape for i in range(4, 8)]
    assert shapes == [(13, 11), (13, 8), (10, 13), (8, 13)]
    # an edge peak: plain cross-correlation on a ramp peaks at the window's far corner
    res_e, _ = _check_against_restatement(image0, ramp, q0[:1], ts, r, mrcal_b200.TM_CCORR, H10=H10[:1])
    assert res_e["status"][0] == stereo.MATCH_EDGE_PEAK
    # a search region smaller than the template
    res_s, _ = _check_against_restatement(image0, image1, q0[:1], ts, -1, mrcal_b200.TM_CCORR_NORMED, H10=H10[:1])
    assert res_s["status"][0] == stereo.MATCH_SEARCH_TOO_SMALL
    # the single calls: the same bits, the reference's return values
    q1, d = mrcal_b200.match_feature(image0, image1, q0, search_radius1=r, template_size1=ts, H10=H10)
    for i in (0, 4, 5, 6, 7):
        q1i, di = mrcal_b200.match_feature(image0, image1, q0[i], search_radius1=r, template_size1=ts, H10=H10[i])
        assert list(di) == ["matchoutput_image", "matchoutput_optimum_subpixel_at", "matchoutput_optimum_subpixel",
                            "qshift_image1_matchoutput"]
        np.testing.assert_array_equal(q1i, q1[i])
        np.testing.assert_array_equal(di["matchoutput_image"], d["matchoutput_image"][i])
        np.testing.assert_array_equal(di["matchoutput_optimum_subpixel_at"], d["matchoutput_optimum_subpixel_at"][i])
        assert di["matchoutput_optimum_subpixel"] == d["matchoutput_optimum_subpixel"][i]
        np.testing.assert_array_equal(di["qshift_image1_matchoutput"], d["qshift_image1_matchoutput"][i])
    assert np.all(np.isnan(q1[1:4]))
    q1e, de = mrcal_b200.match_feature(image0, ramp, q0[0], search_radius1=r, template_size1=ts, H10=H10[0],
                                       method=mrcal_b200.TM_CCORR)
    assert q1e is None and list(de) == ["matchoutput_image"]
    with pytest.raises(RuntimeError, match="left edge in image0"):
        mrcal_b200.match_feature(image0, image1, q0[3], search_radius1=r, template_size1=ts, H10=H10[3])


def test_a_batch_of_20000_features():
    rng = np.random.default_rng(30)
    image0 = match_np.textured_image(1000, 1200, np.uint8, 13)
    image1 = np.ascontiguousarray(image0[4:, 9:])
    N = 20000
    q0 = rng.uniform(-10, 1210, (N, 2))
    H10 = _perspective(rng, N, (-9., -4.))
    kw = dict(search_radius1=8, template_size1=15, H10=H10)
    q1, d = mrcal_b200.match_feature(image0, image1, q0, **kw)
    q1b, db = mrcal_b200.match_feature(image0, image1, q0, **kw)
    np.testing.assert_array_equal(q1, q1b)
    for i in range(N):
        if d["matchoutput_image"][i] is not None:
            np.testing.assert_array_equal(d["matchoutput_image"][i], db["matchoutput_image"][i])
    # about 2 in 5 of the features are too close to an edge of image 1
    assert np.sum(d["status"] == stereo.MATCH_OK) > N // 3
    assert set(np.unique(d["status"])) >= {stereo.MATCH_OK, stereo.MATCH_OUTSIDE_IMAGE1}
    for i in rng.choice(np.flatnonzero(d["status"] == stereo.MATCH_OK), 25, replace=False):
        q1i, di = mrcal_b200.match_feature(image0, image1, q0[i], search_radius1=8, template_size1=15, H10=H10[i])
        np.testing.assert_array_equal(q1i, q1[i])
        np.testing.assert_array_equal(di["matchoutput_image"], d["matchoutput_image"][i])
    for i in rng.choice(N, 10, replace=False):
        ref = match_np.match_feature(image0, image1, q0[i], search_radius1=8, template_size1=15, H10=H10[i])
        assert ref["status"] == d["status"][i]
        if ref["status"] == match_np.MATCH_OK:
            assert np.abs(ref["q1"] - q1[i]).max() <= 1e-9


def test_a_batch_of_more_features_than_a_grid_dimension_of_65535():
    """100 000 features, over 65 535 of them matched: one call, every row the single call's and the restatement's"""
    rng = np.random.default_rng(31)
    image0 = match_np.textured_image(700, 800, np.uint8, 15)
    image1 = np.ascontiguousarray(image0[2:, 3:])
    N = 100000
    q0 = rng.uniform(8, (785, 685), (N, 2))
    q1e = q0 - (3., 2.) + rng.uniform(-1., 1., (N, 2))
    kw = dict(search_radius1=2, template_size1=5, q1_estimate=q1e, method=mrcal_b200.TM_SQDIFF_NORMED)
    q1, d = mrcal_b200.match_feature(image0, image1, q0, **kw)
    ran = np.flatnonzero(np.isin(d["status"], (stereo.MATCH_OK, stereo.MATCH_EDGE_PEAK)))
    assert ran.size > 65535
    assert np.sum(d["status"] == stereo.MATCH_OK) > 50000
    # the features beyond the first 65 535 that ran, and a few before
    sample = np.concatenate((ran[:5], ran[65535:][rng.choice(ran.size - 65535, 20, replace=False)]))
    for i in sample:
        q1i, di = mrcal_b200.match_feature(image0, image1, q0[i], **{**kw, "q1_estimate": q1e[i]})
        np.testing.assert_array_equal(di["matchoutput_image"], d["matchoutput_image"][i])
        ref = match_np.match_feature(image0, image1, q0[i], search_radius1=2, template_size1=5, q1_estimate=q1e[i],
                                     method=mrcal_b200.TM_SQDIFF_NORMED)
        assert ref["status"] == d["status"][i]
        np.testing.assert_array_equal(d["matchoutput_image"][i].view(np.uint32), ref["matchoutput"].view(np.uint32))
        if ref["status"] == match_np.MATCH_OK:
            np.testing.assert_array_equal(q1i, q1[i])
            assert np.abs(ref["q1"] - q1[i]).max() <= 1e-9
        else:
            assert q1i is None and np.all(np.isnan(q1[i]))


@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_torch_tensors_give_the_numpy_bits(dtype):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(40)
    image0 = match_np.textured_image(200, 230, dtype, 14)
    image1 = np.ascontiguousarray(image0[2:, 3:])
    q0 = rng.uniform(0, 230, (300, 2))
    H10 = _perspective(rng, 300, (-3., -2.))
    kw = dict(search_radius1=5, template_size1=(11, 9), H10=H10, method=mrcal_b200.TM_CCOEFF_NORMED)
    q1, d = mrcal_b200.match_feature(image0, image1, q0, **kw)
    t0, t1 = torch.from_numpy(image0).cuda(), torch.from_numpy(image1).cuda()
    q1t, dt = mrcal_b200.match_feature(t0, t1, q0, **kw)
    np.testing.assert_array_equal(q1, q1t)
    np.testing.assert_array_equal(d["status"], dt["status"])
    for a, b in zip(d["matchoutput_image"], dt["matchoutput_image"]):
        assert (a is None) == (b is None)
        if a is not None:
            np.testing.assert_array_equal(a, b)


####################################################################################################
# end to end: a rectified pair, matched and ranged
####################################################################################################
def test_rectified_pair_matched_and_ranged():
    """A fronto-parallel textured plane at Z = 5 m seen by a rectified pinhole pair with a 0.3 m baseline and f = 121.67
    px: a disparity of 7.3 px everywhere, rendered with transform_image(). The 3x3 quadratic fit pulls a sub-pixel
    optimum toward the whole pixel: on this texture, at a fraction of 0.3 px, the 195 features' largest error is
    0.103 px (H100), and the mean -0.02 px. So disparities are held to 0.15 px, and ranges to the relative error that
    allows, 0.15 / (7.3 - 0.15)"""
    H, W = 240, 320
    f, baseline, Z = 121.67, 0.3, 5.
    d = f * baseline / Z
    fxycxy = np.array((f, f, (W - 1) / 2., (H - 1) / 2.))
    models = (mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", fxycxy), imagersize=(W, H), rt_cam_ref=np.zeros(6)),
              mrcal_b200.cameramodel(intrinsics=("LENSMODEL_PINHOLE", fxycxy), imagersize=(W, H),
                                     rt_cam_ref=np.array((0., 0., 0., -baseline, 0., 0.))))
    texture = match_np.textured_image(H + 40, W + 80, np.float32, 11, blur=3)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    image0 = mrcal_b200.transform_image(texture, np.stack((xx + 20, yy + 20), -1))
    image1 = mrcal_b200.transform_image(texture, np.stack((xx + np.float32(20 + d), yy + 20), -1))
    q0 = np.array([(x, y) for x in range(40, 280, 17) for y in range(40, 200, 13)], float)
    q1, diag = mrcal_b200.match_feature(image0, image1, q0, search_radius1=4, template_size1=15,
                                        q1_estimate=q0 - (7., 0.))
    assert np.all(diag["status"] == stereo.MATCH_OK)
    disparity = q0[:, 0] - q1[:, 0]
    assert np.abs(disparity - d).max() <= 0.15
    assert np.abs(q1[:, 1] - q0[:, 1]).max() <= 0.15
    ranges = mrcal_b200.stereo_range(disparity, models, qrect0=q0)
    v = np.column_stack(((q0 - fxycxy[2:]) / f, np.ones(len(q0))))
    truth = Z * np.linalg.norm(v, axis=1)
    assert np.abs(ranges / truth - 1.).max() <= 0.15 / (d - 0.15)
