"""ref_calibration_object() against the numpy restatement and hand-computed corners, its broadcasting, grids and
refusals; the restatement against tests/golden/synthetic_data.npz; the refusals of the device-backed functions, and
their failure without a device (no GPU needed)."""
import os

import numpy as np
import pytest

import mrcal_b200
from mrcal_b200 import seeding, synthetic
import synthetic_data_np as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "synthetic_data.npz")


def test_ref_calibration_object_values():
    obj = mrcal_b200.ref_calibration_object(10, 6, 0.1)
    assert obj.shape == (6, 10, 3)
    assert np.array_equal(obj, S.ref_calibration_object(10, 6, 0.1))
    assert np.array_equal(obj[0, 0], (0., 0., 0.))
    assert np.array_equal(obj[0, 1], (0.1, 0., 0.))
    assert np.array_equal(obj[5, 9], (9 * 0.1, 5 * 0.1, 0.))
    # warp: the centre of a 3x3 board deflects by both terms, its corners not at all, the edge midpoints by one
    w = np.array((0.01, -0.003))
    obj = mrcal_b200.ref_calibration_object(3, 3, 0.5, calobject_warp=w)
    assert np.array_equal(obj, S.ref_calibration_object(3, 3, 0.5, w))
    assert obj[1, 1, 2] == 0.01 + -0.003 and obj[0, 0, 2] == 0. and obj[0, 1, 2] == 0.01 and obj[1, 0, 2] == -0.003
    # (x, y) spacing, in that order
    obj = mrcal_b200.ref_calibration_object(4, 3, np.array((0.1, 0.2)), calobject_warp=w)
    assert np.array_equal(obj[2, 3, :2], (3 * 0.1, 2 * 0.2))
    assert np.array_equal(obj, S.ref_calibration_object(4, 3, (0.1, 0.2), w))


def test_ref_calibration_object_matches_seeding():
    """seeding uses the public function: the same bits as its former private copy (z starts at 0)"""
    assert seeding.ref_calibration_object is mrcal_b200.ref_calibration_object
    xx, yy = np.meshgrid(np.arange(10, dtype=float), np.arange(9, dtype=float))
    old = np.stack((xx * 0.1, yy * 0.1, np.zeros_like(xx)), -1)
    assert np.array_equal(mrcal_b200.ref_calibration_object(10, 9, 0.1), old)


def test_ref_calibration_object_broadcasting():
    sp = np.array(((0.1, 0.2), (0.3, 0.05), (1., 2.)))
    obj = mrcal_b200.ref_calibration_object(5, 4, sp)
    assert obj.shape == (3, 4, 5, 3)
    for i in range(3):
        assert np.array_equal(obj[i], S.ref_calibration_object(5, 4, sp[i]))
    warp = np.array(((0.01, 0.02), (-0.01, 0.)))[:, None, :]      # (2,1,2) against spacing (3,2)
    obj = mrcal_b200.ref_calibration_object(5, 4, sp, calobject_warp=warp)
    assert obj.shape == (2, 3, 4, 5, 3)
    for i in range(2):
        for j in range(3):
            assert np.array_equal(obj[i, j], S.ref_calibration_object(5, 4, sp[j], warp[i, 0]))
    obj = mrcal_b200.ref_calibration_object(5, 4, 0.1, calobject_warp=warp[:, 0])
    assert obj.shape == (2, 4, 5, 3)
    assert np.array_equal(obj[1], S.ref_calibration_object(5, 4, 0.1, warp[1, 0]))


def test_ref_calibration_object_grids():
    kw = dict(x_corner0=-0.5, x_corner1=4.5, Nx=11, y_corner0=1, y_corner1=2, Ny=3)
    w = np.array((0.002, 0.004))
    obj = mrcal_b200.ref_calibration_object(5, 4, 0.1, calobject_warp=w, **kw)
    assert obj.shape == (3, 11, 3)
    assert np.array_equal(obj, S.ref_calibration_object(5, 4, 0.1, w, **kw))
    assert np.array_equal(obj[0, :, 0], np.linspace(-0.5, 4.5, 11) * 0.1)
    assert np.array_equal(obj[:, 0, 1], np.linspace(1, 2, 3) * 0.1)


def test_ref_calibration_object_from_optimization_inputs():
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=1, Nframes=3, W=6, H=5, spacing=0.07)
    kw["calobject_warp"] = np.array((0.001, -0.002))
    obj = mrcal_b200.ref_calibration_object(optimization_inputs=kw)
    assert np.array_equal(obj, S.ref_calibration_object(6, 5, 0.07, kw["calobject_warp"]))


def test_ref_calibration_object_refusals():
    options = ('W', 'H', 'object_spacing')
    with pytest.raises(Exception, match=f"Options '{options}': ALL must be given, or NONE must be given".replace("(", r"\(").replace(")", r"\)")):
        mrcal_b200.ref_calibration_object(10, 6)
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=1, Nframes=3, W=6, H=5)
    with pytest.raises(Exception, match="and 'optimization_inputs' cannot both be given"):
        mrcal_b200.ref_calibration_object(10, 6, 0.1, optimization_inputs=kw)
    with pytest.raises(Exception, match="and 'optimization_inputs' MUST be given"):
        mrcal_b200.ref_calibration_object()


@pytest.mark.parametrize("key", [k for k, _ in S.cases()])
def test_restatement_matches_golden(ref, key):
    """The restatement, through the compiled reference, still gives the stored answers and RNG state"""
    d = np.load(GOLDEN)
    kw = dict(S.cases())[key]
    q, Rt, margins, Nchunks, digest = S.run_case(kw)
    assert np.array_equal(q, d[f"{key}/q"]) and np.array_equal(Rt, d[f"{key}/Rt_ref_boardref"])
    assert np.array_equal(margins, d[f"{key}/margins"])
    assert Nchunks * kw["Nframes"] * 6 == d[f"{key}/Ndraws"] and digest == str(d[f"{key}/rng"])


def test_golden_inputs_are_the_cases():
    d = np.load(GOLDEN)
    for key, kw in S.cases():
        assert d[f"{key}/seed"] == kw["seed"] and d[f"{key}/Nframes"] == kw["Nframes"]
        assert np.array_equal(d[f"{key}/rt_ref_boardcenter"], kw["rt_ref_boardcenter"])
        assert np.array_equal(d[f"{key}/noiseradius"], kw["noiseradius"])
        assert S.WHICH[int(d[f"{key}/which"])] == kw["which"]
    # the cases cover several chunks, every `which`, and frames partly out of view
    assert max(int(d[f"{k}/Ndraws"]) // (6 * int(d[f"{k}/Nframes"])) for k, _ in S.cases()) >= 3
    assert {int(d[f"{k}/which"]) for k, _ in S.cases()} == {0, 1, 2, 3}


def _model(lm="LENSMODEL_OPENCV4"):
    intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
    return mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=(4000, 2200))


def test_synthesize_refuses_bad_which():
    state = np.random.get_state()
    with pytest.raises(Exception, match="'which' argument must be one of"):
        mrcal_b200.synthesize_board_observations([_model()], object_width_n=5, object_height_n=4, object_spacing=0.1,
                                                 calobject_warp=None, rt_ref_boardcenter=np.array((0, 0, 0, 0, 0, 3.)),
                                                 rt_ref_boardcenter__noiseradius=np.zeros(6), Nframes=3,
                                                 which="most-cameras-must-see-most-of-the-board")
    assert np.array_equal(np.random.get_state()[1], state[1])


def test_hypothesis_refuses_without_boards():
    with pytest.raises(Exception, match="No board observations available"):
        mrcal_b200.hypothesis_board_corner_positions(lensmodel="LENSMODEL_OPENCV4", intrinsics=np.zeros((1, 8)))


@pytest.mark.skipif(mrcal_b200.device_count() > 0, reason="checks the refusal without a device")
def test_device_entry_points_fail_without_a_device():
    kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=2, Nframes=3, W=5, H=4, Npoints=3)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        mrcal_b200.synthesize_board_observations([_model()], object_width_n=5, object_height_n=4, object_spacing=0.1,
                                                 calobject_warp=None, rt_ref_boardcenter=np.array((0, 0, 0, 0, 0, 3.)),
                                                 rt_ref_boardcenter__noiseradius=np.zeros(6), Nframes=3)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        mrcal_b200.hypothesis_board_corner_positions(**kw)
    for sigma in (None, 0.):
        with pytest.raises(RuntimeError, match="no usable CUDA device"):
            mrcal_b200.make_perfect_observations(kw, observed_pixel_uncertainty=sigma)
    # the C entry points themselves, through the binding
    from mrcal_b200._capi import checked
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        checked.mrcal_b200_problem_corners(None, None, None, None, 0, None, 0, None, 0, None, 0, None, 0, None, 0,
                                           None, None, 0)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        checked.mrcal_b200_synthesize_board_observations(None, None, None, None, 0, None, 0, 0, None, None, None, None)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        checked.mrcal_b200_problem_observed_pixel_uncertainty(None, None)
