"""synthesize_board_observations(), hypothesis_board_corner_positions() and make_perfect_observations()
(mrcal_b200/synthetic_data.py, csrc/synthetic_data.cu) against the reference: the answers stored in
tests/golden/synthetic_data.npz, and where oracle/_ref is built, the numpy restatement (tests/synthetic_data_np.py)
run live through the compiled reference. Frames, RNG draws and noise must be the reference's exactly; pixels and
poses agree at the gates of the projection and pose tests."""
import os

import numpy as np
import pytest

import mrcal_b200
import problems
from mrcal_b200 import synthetic
import synthetic_data_np as S

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "synthetic_data.npz")
CASES = dict(S.cases())


def _q_gate(q_ref):
    return 1e-9 * (1. + np.abs(q_ref).max()) if q_ref.size else 0.   # test_project_gpu.py


def _pose_gate(Rt_ref):
    return 1e-12 * (1. + np.abs(Rt_ref).max()) if Rt_ref.size else 0.   # test_poseutils_gpu.py


def _synthesize(kw):
    models = [mrcal_b200.cameramodel(intrinsics=(lm, intr), imagersize=size, rt_cam_ref=rt)
              for lm, intr, rt, size in S.cameras(kw["lensmodels"], kw["seed"])]
    np.random.seed(kw["seed"])
    q, Rt = mrcal_b200.synthesize_board_observations(
        models, object_width_n=kw["W"], object_height_n=kw["H"], object_spacing=kw["spacing"],
        calobject_warp=kw["calobject_warp"], rt_ref_boardcenter=kw["rt_ref_boardcenter"],
        rt_ref_boardcenter__noiseradius=kw["noiseradius"], Nframes=kw["Nframes"],
        max_oblique_angle_deg=kw["max_oblique_angle_deg"], which=kw["which"])
    return q, Rt, S.rng_digest()


def _check(key, q, Rt, digest, q_ref, Rt_ref, digest_ref):
    kw = CASES[key]
    assert q.shape == q_ref.shape == (kw["Nframes"], len(kw["lensmodels"]), kw["H"], kw["W"], 2)
    assert Rt.shape == Rt_ref.shape == (kw["Nframes"], 4, 3)
    assert digest == digest_ref, f"{key}: np.random is not left in the reference's state"
    # the same frames, in the same order: the poses agree at the pose gate, far below their spread
    assert np.abs(Rt - Rt_ref).max() <= _pose_gate(Rt_ref)
    assert np.abs(q - q_ref).max() <= _q_gate(q_ref)


@pytest.mark.parametrize("key", list(CASES))
def test_synthesize_matches_stored_reference(key):
    d = np.load(GOLDEN)
    q_ref, Rt_ref = d[f"{key}/q"], d[f"{key}/Rt_ref_boardref"]
    # every decision of the reference lies farther from its threshold than the gates: the case decides the same way
    # whatever the last bits
    margins = d[f"{key}/margins"]
    assert (margins[:, 0] > _q_gate(q_ref)).all() and (margins[:, 1] > 1e-12).all()
    q, Rt, digest = _synthesize(CASES[key])
    _check(key, q, Rt, digest, q_ref, Rt_ref, str(d[f"{key}/rng"]))


@pytest.mark.parametrize("key", list(CASES))
def test_synthesize_matches_reference_live(ref, key):
    q_ref, Rt_ref, margins, _, digest_ref = S.run_case(CASES[key])
    assert (margins[:, 0] > _q_gate(q_ref)).all() and (margins[:, 1] > 1e-12).all()
    _check(key, *_synthesize(CASES[key]), q_ref, Rt_ref, digest_ref)


def test_synthesize_is_deterministic():
    kw = CASES["mixed"]
    a, b = _synthesize(kw), _synthesize(kw)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2] == b[2]


def _problem(lm="LENSMODEL_OPENCV8", Ncameras=3, Nframes=4, Npoints=0, outliers=3, seed=5):
    kw, truth = synthetic.make_problem(lensmodel=lm, Ncameras=Ncameras, Nframes=Nframes, W=6, H=5, seed=seed,
                                       Npoints=Npoints, pixel_noise=0.3)
    kw["calobject_warp"] = np.array((0.002, -0.001))
    if outliers:
        problems._mark_outliers(kw, outliers, seed)
    return kw, truth


def _clone(kw):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}


def _close(a, b):
    assert a.shape == b.shape
    assert np.abs(a - b).max(initial=0.) <= 1e-12 * (1. + np.abs(b).max(initial=0.))


@pytest.mark.parametrize("lm", ["LENSMODEL_OPENCV8", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100"])
def test_hypothesis_board_corner_positions(ref, lm):
    kw, _ = _problem(lm)
    idx = kw["indices_frame_camintrinsics_camextrinsics"]
    assert (idx[:, 2] == -1).any() and (kw["observations_board"][..., 2] <= 0).any()
    for icam in (None, 0, 2):
        out, out_ref = mrcal_b200.hypothesis_board_corner_positions(icam, **kw), \
            S.hypothesis_board_corner_positions(icam, **kw)
        for a, b in zip(out, out_ref):
            _close(a, b)
    # explicit inliers; with a camera given the array is modified in place, as the reference does
    inl = np.random.default_rng(1).uniform(size=kw["observations_board"].shape[:-1]) > 0.3
    out_ref = S.hypothesis_board_corner_positions(1, inl, **kw)
    given = inl.copy()
    out = mrcal_b200.hypothesis_board_corner_positions(1, given, **kw)
    for a, b in zip(out, out_ref):
        _close(a, b)
    assert not given[idx[:, 1] != 1].any() and np.array_equal(given[idx[:, 1] == 1], inl[idx[:, 1] == 1])
    # bit-identical on a second call
    again = mrcal_b200.hypothesis_board_corner_positions(**kw)
    assert all(np.array_equal(a, b) for a, b in zip(again, mrcal_b200.hypothesis_board_corner_positions(**kw)))


def _perfect_residuals(kw):
    x = mrcal_b200.optimizer_callback(**kw, no_jacobian=True, no_factorization=True)[1]
    rows = []
    for what in ("boards", "points"):
        n = getattr(mrcal_b200, f"num_measurements_{what}")(**kw)
        if n:
            i0 = getattr(mrcal_b200, f"measurement_index_{what}")(0, **kw)
            rows.append(x[i0:i0 + n])
    return np.concatenate(rows)


@pytest.mark.parametrize("lm", ["LENSMODEL_OPENCV8", "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100",
                                "LENSMODEL_CAHVORE_linearity=0.37"])
def test_make_perfect_observations_noiseless(ref, lm):
    kw, _ = _problem(lm, Npoints=6)
    before = _clone(kw)
    qb_ref, qp_ref = S.perfect_projections(kw)
    state = np.random.get_state()
    assert mrcal_b200.make_perfect_observations(kw, observed_pixel_uncertainty=0) is None
    assert np.array_equal(np.random.get_state()[1], state[1]) and np.random.get_state()[2] == state[2]
    assert np.abs(kw["observations_board"][..., :2] - qb_ref).max() <= _q_gate(qb_ref)
    assert np.abs(kw["observations_point"][..., :2] - qp_ref).max() <= _q_gate(qp_ref)
    # only the pixels change: weights (outliers included) and every other key stay
    for k, v in before.items():
        if k in ("observations_board", "observations_point"):
            assert np.array_equal(kw[k][..., 2], v[..., 2])
        elif isinstance(v, np.ndarray):
            assert np.array_equal(kw[k], v), k
        else:
            assert kw[k] == v, k
    # the perfect observations fit the geometry they came from
    assert np.abs(_perfect_residuals(kw)).max() < 1e-9


def _add_noise(kw, sigma, seed):
    """the restatement's noise step on kw, from np.random.seed(seed)"""
    np.random.seed(seed)
    S.add_noise(kw, sigma)


@pytest.mark.parametrize("Npoints", [0, 6])
def test_make_perfect_observations_noise(ref, Npoints):
    kw, truth = _problem(Npoints=Npoints)
    problems.add_triangulated_points(kw, truth, 3, 9)
    tri = (kw["observations_point_triangulated"].copy(), kw["indices_point_triangulated_camintrinsics_camextrinsics"].copy())
    outlier = kw["observations_board"][..., 2] <= 0
    assert outlier.any()
    # the device's perfect observations, plus the restatement's noise drawn from the same seed
    expected = _clone(kw)
    mrcal_b200.make_perfect_observations(expected, observed_pixel_uncertainty=0)
    _add_noise(expected, 0.4, 17)
    digest = S.rng_digest()
    np.random.seed(17)
    mrcal_b200.make_perfect_observations(kw, observed_pixel_uncertainty=0.4)
    assert S.rng_digest() == digest
    assert ("observations_point" in kw) == (Npoints > 0)
    for what in ("observations_board", "observations_point")[:1 + (Npoints > 0)]:
        assert np.array_equal(kw[what], expected[what]), what
    # an outlier's weight becomes 1 in the caller's array, as in the reference
    assert (kw["observations_board"][..., 2][outlier] == 1.).all()
    # triangulated observations are untouched
    assert np.array_equal(kw["observations_point_triangulated"], tri[0])
    assert np.array_equal(kw["indices_point_triangulated_camintrinsics_camextrinsics"], tri[1])
    # the restatement, end to end, agrees
    live = _clone(_problem(Npoints=Npoints)[0])
    np.random.seed(17)
    S.make_perfect_observations(live, 0.4)
    for what in ("observations_board", "observations_point")[:1 + (Npoints > 0)]:
        assert np.abs(kw[what] - live[what]).max() <= _q_gate(live[what])


def test_make_perfect_observations_estimates_sigma():
    kw, _ = _problem(outliers=0)
    P = mrcal_b200.Problem(**_clone(kw))
    try:
        sigma = P.projection_uncertainty(np.array(((0.1, 0.2, 3.),)), 0, method="mean-pcam")[1]
    finally:
        P.close()
    assert sigma > 0
    expected = _clone(kw)
    mrcal_b200.make_perfect_observations(expected, observed_pixel_uncertainty=0)
    _add_noise(expected, sigma, 23)
    np.random.seed(23)
    mrcal_b200.make_perfect_observations(kw)
    assert np.array_equal(kw["observations_board"], expected["observations_board"])


def test_make_perfect_observations_points_only_and_boards_only(ref):
    kw, _ = _problem(Npoints=6, outliers=0)
    boards_only = {k: v for k, v in _clone(kw).items() if "point" not in k and k != "Npoints_fixed"}
    points_only = {k: v for k, v in _clone(kw).items()
                   if k not in ("observations_board", "indices_frame_camintrinsics_camextrinsics", "rt_ref_frame",
                                "calobject_warp", "calibration_object_spacing")}
    points_only["do_optimize_calobject_warp"] = False
    points_only["do_optimize_frames"] = False
    for inputs in (boards_only, points_only):
        qb_ref, qp_ref = S.perfect_projections(inputs)
        mrcal_b200.make_perfect_observations(inputs, observed_pixel_uncertainty=0)
        if qb_ref is not None:
            assert np.abs(inputs["observations_board"][..., :2] - qb_ref).max() <= _q_gate(qb_ref)
        if qp_ref is not None:
            assert np.abs(inputs["observations_point"][..., :2] - qp_ref).max() <= _q_gate(qp_ref)
        assert np.abs(_perfect_residuals(inputs)).max() < 1e-9
        again = _clone(inputs)
        mrcal_b200.make_perfect_observations(again, observed_pixel_uncertainty=0)
        for k in ("observations_board", "observations_point"):
            if k in inputs:
                assert np.array_equal(again[k], inputs[k])


def test_problem_corners_refuses_bad_indices():
    kw, _ = _problem(outliers=0)
    kw["indices_frame_camintrinsics_camextrinsics"] = kw["indices_frame_camintrinsics_camextrinsics"].copy()
    kw["indices_frame_camintrinsics_camextrinsics"][1, 0] = 99
    with pytest.raises(RuntimeError, match="iframe MUST be in"):
        mrcal_b200.hypothesis_board_corner_positions(**kw)
