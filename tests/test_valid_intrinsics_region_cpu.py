"""The host side of the valid-intrinsics regions (mrcal_b200/regions.py), without a GPU: the restatement of
cv2.findContours(RETR_EXTERNAL, CHAIN_APPROX_SIMPLE) and cv2.contourArea() against what OpenCV 4.13 gave on a few
hundred masks (tests/golden/contours_cv2.npz, from make_contours_golden.py) and against cv2 itself where it imports;
the mask thresholds; close_contour(), imagergrid_using(), the measurements_*() selections given x, and the
cameramodel's region setter."""
import io
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import regions

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "contours_cv2.npz")


def _golden_cases():
    z = np.load(GOLDEN)
    shapes, bits = z["shapes"], np.unpackbits(z["masks"])
    points, lengths, areas = z["points"].astype(np.int64), z["lengths"], z["areas"]
    m0 = p0 = c0 = 0
    for (h, w), n in zip(shapes, z["ncontours"]):
        mask = bits[m0:m0 + h * w].reshape(h, w)
        m0 += h * w
        contours = []
        for L in lengths[c0:c0 + n]:
            contours.append(points[p0:p0 + L].tolist())
            p0 += L
        yield mask, contours, areas[c0:c0 + n].tolist()
        c0 += n


def _as_lists(contours):
    return [[list(map(int, v)) for v in c] for c in contours]


def test_contours_match_opencv_golden():
    n = 0
    for mask, contours, areas in _golden_cases():
        mine = regions.find_external_contours(mask)
        assert _as_lists(mine) == contours, mask
        assert [regions.contour_area(c) for c in mine] == areas
        n += 1
    assert n >= 300


def test_contours_match_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    for i in range(300):
        h, w = ((17, 30), (20, 30), (11, 20))[i % 3]
        mask = (rng.random((h, w)) < rng.uniform(0.1, 0.9)).astype(np.uint8)
        cs = cv2.findContours(mask, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)[-2]
        mine = regions.find_external_contours(mask)
        assert _as_lists(mine) == [c[:, 0, :].tolist() for c in cs]
        assert [regions.contour_area(c) for c in mine] == [cv2.contourArea(c) for c in cs]


def test_contour_cases():
    full = np.ones((17, 30), bool)
    assert _as_lists(regions.find_external_contours(full)) == [[[0, 0], [0, 16], [29, 16], [29, 0]]]
    assert regions.find_external_contours(np.zeros((17, 30), bool)) == []
    one = np.zeros((17, 30), bool)
    one[4, 7] = True
    assert _as_lists(regions.find_external_contours(one)) == [[[7, 4]]]
    assert regions.contour_area([[7, 4]]) == 0.
    # a hole with an island: only the outer border
    m = np.zeros((17, 30), bool)
    m[1:16, 1:29] = True
    m[4:13, 5:25] = False
    m[7:10, 12:18] = True
    assert _as_lists(regions.find_external_contours(m)) == [[[1, 1], [1, 15], [28, 15], [28, 1]]]
    # two blobs: the one met last in the raster scan comes first
    m = np.zeros((17, 30), bool)
    m[2:6, 2:6] = True
    m[10:14, 20:24] = True
    c = regions.find_external_contours(m)
    assert c[0][0] == (20, 10) and c[1][0] == (2, 2)


def test_region_from_mask():
    W, H = 3000, 1700
    full = np.ones((17, 30), bool)
    r = regions._region_from_mask(full, (W, H))
    assert r.dtype == np.int32
    assert r.tolist() == [[0, 0], [0, 1699], [2999, 1699], [2999, 0], [0, 0]]
    for m in (np.zeros((17, 30), bool), np.eye(17, 30, dtype=bool)[:, ::-1] & False):
        assert regions._region_from_mask(m, (W, H)).shape == (0, 2)
    one = np.zeros((17, 30), bool)
    one[3, 3] = True
    assert regions._region_from_mask(one, (W, H)).shape == (0, 2)
    line = np.zeros((17, 30), bool)
    line[5, 3:9] = True                  # 2 vertices, closed: 3 points, too few
    assert regions._region_from_mask(line, (W, H)).shape == (0, 2)
    # equal areas: the first in cv2's order (the blob met last) wins
    m = np.zeros((17, 30), bool)
    m[2:6, 2:6] = True
    m[10:14, 20:24] = True
    r = regions._region_from_mask(m, (30, 17))
    assert r[0].tolist() == [20, 10]
    # the scaling rounds half to even
    m = np.zeros((3, 3), bool)
    m[:2, :2] = True
    r = regions._region_from_mask(m, (4, 6))   # x scale 1.5, y scale 2.5
    assert r.tolist() == [[0, 0], [0, 2], [2, 2], [2, 0], [0, 0]]


def test_region_mask_thresholds():
    rng = np.random.default_rng(3)
    gh, gw = 11, 20
    mean = rng.normal(0, 1, (gh, gw))
    stdev = rng.uniform(0, 3, (gh, gw))
    count = rng.integers(0, 10, (gh, gw)).astype(float)
    unc = rng.uniform(0, 2, (gh, gw))
    unc[0, 0], unc[0, 1], unc[0, 2] = np.nan, np.inf, -np.inf
    thr = (1., 0.5, 1.5, 3)
    base = (np.where(np.isfinite(unc), unc, 1e9) < 1.)
    spl = regions._region_mask("LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=30_Ny=20_fov_x_deg=170", mean, stdev, count,
                               unc, *thr)
    assert np.array_equal(spl, base)
    assert not spl[0, :3].any()
    lean = regions._region_mask("LENSMODEL_OPENCV8", mean, stdev, count, unc, *thr)
    # the signed mean, not its absolute value; count strictly above
    assert np.array_equal(lean, base & (mean < 0.5) & (stdev < 1.5) & (count > 3))
    assert (lean & (mean < -0.5)).any()
    # a huge threshold still rejects the non-finite cells: they become 1e9
    assert not regions._region_mask("LENSMODEL_OPENCV8", mean, stdev, count, unc, 1e9, 1e9, 1e9, -1)[0, :3].any()
    assert regions._region_mask("LENSMODEL_OPENCV8", mean, stdev, count, unc, 1e10, 1e9, 1e9, -1)[0, :3].all()


def test_close_contour_and_using():
    assert regions.close_contour(None) is None
    assert regions.close_contour(np.zeros((0, 3))).shape == (0, 2)
    c = np.array([[0., 0.], [4., 0.], [4., 3.]])
    assert regions.close_contour(c).tolist() == [[0, 0], [4, 0], [4, 3], [0, 0]]
    closed = np.array([[0., 0.], [4., 0.], [4., 3.], [0., 1e-7]])
    assert regions.close_contour(closed) is closed
    assert mrcal_b200.imagergrid_using((3000, 1700), 30) == \
        '($1*{}):($2*{}):3'.format(2999. / 29, 1699. / 16)
    assert mrcal_b200.imagergrid_using((640, 480), 20, 10) == '($1*{}):($2*{}):3'.format(639. / 19, 479. / 9)


def _inputs():
    """A small solve's inputs by hand: 2 cameras, 3 frames, boards of 4x3, some outliers, 2 points"""
    rng = np.random.default_rng(5)
    idx = np.array([[0, 0, -1], [0, 1, 0], [1, 0, -1], [2, 1, 0]], np.int32)
    obs = np.concatenate((rng.uniform(0, 600, (4, 3, 4, 2)), rng.uniform(0.5, 1., (4, 3, 4, 1))), axis=-1)
    obs[1, 0, 2, 2] = -1.
    obs[3, 2, :, 2] = 0.
    obs_pt = np.concatenate((rng.uniform(0, 600, (3, 2)), np.array([[1.], [-1.], [0.7]])), axis=-1)
    return dict(lensmodel="LENSMODEL_OPENCV4", intrinsics=np.tile([500., 500., 320., 240., 0, 0, 0, 0], (2, 1)),
                imagersizes=np.array([[640, 480]] * 2, np.int32), rt_cam_ref=np.zeros((1, 6)),
                rt_ref_frame=np.zeros((3, 6)), points=np.zeros((2, 3)),
                indices_frame_camintrinsics_camextrinsics=idx, observations_board=obs,
                indices_point_camintrinsics_camextrinsics=np.array([[0, 0, -1], [1, 1, 0], [1, 0, -1]], np.int32),
                observations_point=obs_pt, calobject_warp=np.zeros(2), calibration_object_spacing=0.1)


def test_measurements_selection():
    inp = _inputs()
    Nmeas = mrcal_b200.num_measurements(**inp)
    x = np.arange(Nmeas, dtype=float)
    b0 = mrcal_b200.measurement_index_boards(0, **inp)
    xb = x[b0:b0 + 4 * 12 * 2].reshape(4, 3, 4, 2)
    w = inp["observations_board"][..., 2]
    m = mrcal_b200.measurements_board(inp, x=x)
    assert np.array_equal(m, xb[w > 0])
    m, q = mrcal_b200.measurements_board(inp, x=x, icam_intrinsics=1, return_observations=True)
    sel = (w > 0) & (inp["indices_frame_camintrinsics_camextrinsics"][:, 1] == 1)[:, None, None]
    assert np.array_equal(m, xb[sel]) and np.array_equal(q, inp["observations_board"][sel][:, :2])
    assert np.array_equal(mrcal_b200.residuals_board(inp, residuals=x, i_cam=0),
                          mrcal_b200.measurements_board(inp, x=x, icam_intrinsics=0))
    assert mrcal_b200.residuals_chessboard is mrcal_b200.residuals_board
    p0 = mrcal_b200.measurement_index_points(0, **inp)
    xp = x[p0:p0 + 6].reshape(3, 2)
    assert np.array_equal(mrcal_b200.measurements_point(inp, x=x), xp[[0, 2]])
    m, q = mrcal_b200.measurements_point(inp, x=x, icam_intrinsics=0, return_observations=True)
    assert np.array_equal(m, xp[[0, 2]]) and np.array_equal(q, inp["observations_point"][[0, 2], :2])
    assert mrcal_b200.residuals_point(inp, residuals=x, icam_intrinsics=1).shape == (0, 2)   # its one is an outlier
    empty = dict(inp, observations_point=None)
    assert mrcal_b200.measurements_point(empty, x=x).shape == (0, 2)
    a, b = mrcal_b200.measurements_board(dict(inp, observations_board=np.zeros((0, 3, 4, 3))), x=x,
                                         return_observations=True)
    assert a.shape == b.shape == (0, 2)


def test_cameramodel_region_setter():
    m = mrcal_b200.cameramodel(intrinsics=("LENSMODEL_OPENCV4", [500., 500., 320., 240., 0, 0, 0, 0]),
                               imagersize=(640, 480))
    assert m.valid_intrinsics_region() is None
    assert m.valid_intrinsics_region(np.array([[10, 10], [600, 10], [600, 400], [10, 400]])) is True
    r = m.valid_intrinsics_region()
    assert r.dtype == np.float64 and r.tolist() == [[10, 10], [600, 10], [600, 400], [10, 400], [10, 10]]
    r[0, 0] = 99.                                       # the getter gives a copy
    assert m.valid_intrinsics_region()[0, 0] == 10.
    f = io.StringIO()
    m.write(f)
    m2 = mrcal_b200.cameramodel(f.getvalue())
    assert np.array_equal(m2.valid_intrinsics_region(), m.valid_intrinsics_region())
    assert m.valid_intrinsics_region(np.zeros((0, 2))) is True
    assert m.valid_intrinsics_region().shape == (0, 2)
    assert mrcal_b200.cameramodel(io.StringIO(str(m)).getvalue()).valid_intrinsics_region().shape == (0, 2)
    for bad in (np.array([[0, 0], [1, 0], [0, 0]]), np.zeros((5, 3))):
        with pytest.raises(Exception):
            m.valid_intrinsics_region(bad)
    assert m.valid_intrinsics_region().shape == (0, 2)
