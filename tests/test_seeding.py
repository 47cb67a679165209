"""Seeding (mrcal_b200/seeding.py; reference: mrcal/calibration.py:622-781,1186-1608).

CPU: the pieces against known answers (an exact pinhole/stereographic camera gives the pose back; a rig seen
through true stereographic lenses seeds close to the truth). GPU: the reference's own end-to-end flow,
test/test-basic-calibration.py:45-209 -- seed_stereographic(), then optimize() in stages with a growing set of
unknowns, noise and gross outliers in the data -- judged by that test's tolerances."""
import numpy as np
import pytest

from mrcal_b200 import seeding as S, synthetic


def test_procrustes_known_answer():
    rng = np.random.default_rng(1)
    p1 = rng.normal(size=(40, 3))
    Rt = S.Rt_from_rt(np.array((0.2, -0.5, 0.1, 1., 2., -3.)))
    p0 = S.transform_point_Rt(Rt, p1)
    assert np.allclose(S.align_procrustes_points_Rt01(p0, p1), Rt, atol=1e-12)


def test_pnp_exact_camera():
    rng = np.random.default_rng(2)
    obj = S.ref_calibration_object(10, 9, 0.1).reshape(-1, 3)
    intr = np.array((1500., 1510., 2000., 1100.))
    for _ in range(10):
        rt = np.concatenate((rng.uniform(-0.6, 0.6, 3), rng.uniform(-1, 1, 2), [rng.uniform(2, 5)]))
        p = S.transform_point_Rt(S.Rt_from_rt(rt), obj)
        u = 2. * p[:, :2] / (np.linalg.norm(p, axis=-1, keepdims=True) + p[:, 2:])
        obs = np.concatenate((u * intr[:2] + intr[2:], np.ones((len(u), 1))), -1)
        Rt = S._estimate_camera_pose_from_fixed_point_observations("LENSMODEL_STEREOGRAPHIC", intr, obs, obj, "test")
        assert np.abs(S.rt_from_Rt(Rt) - rt).max() < 1e-9


def test_traverse_prefers_well_connected_links():
    # 0-1 share 50 frames, 0-2 share 2, 1-2 share 40: camera 2 is reached directly (one hop costs 65536 - n)
    C = np.array(((0, 50, 2), (50, 0, 40), (2, 40, 0)))
    seen = []
    S.traverse_sensor_links(C, lambda i, p: seen.append((i, p)))
    assert seen == [(1, 0), (2, 0)]
    C[0, 2] = C[2, 0] = 0
    seen = []
    S.traverse_sensor_links(C, lambda i, p: seen.append((i, p)))
    assert seen == [(1, 0), (2, 1)]


def test_seed_stereographic_rig():
    kw, truth = synthetic.make_problem(lensmodel="LENSMODEL_STEREOGRAPHIC", Ncameras=4, Nframes=30, W=10, H=9, seed=0,
                                       pixel_noise=0.3, which="some", calobject_warp_true=(0, 0))
    ifc = kw["indices_frame_camintrinsics_camextrinsics"][:, :2]
    intr, rt_cam_ref, rt_ref_frame = S.seed_stereographic(kw["imagersizes"], 1761., ifc, kw["observations_board"],
                                                          kw["calibration_object_spacing"])
    assert intr.shape == (4, 4) and rt_cam_ref.shape == (3, 6) and rt_ref_frame.shape == (30, 6)
    assert np.allclose(intr[:, 2:], (np.array(kw["imagersizes"]) - 1.) / 2.)
    # a seed, not a solution: the true projection centres are ~50 px off the imager centre
    assert np.abs(rt_cam_ref[:, :3] - truth["rt_cam_ref"][:, :3]).max() < np.pi / 180. * 2.
    assert np.abs(rt_cam_ref[:, 3:] - truth["rt_cam_ref"][:, 3:]).max() < 0.15
    assert np.abs(rt_ref_frame[:, :3] - truth["rt_ref_frame"][:, :3]).max() < np.pi / 180. * 5.
    assert np.abs(rt_ref_frame[:, 3:] - truth["rt_ref_frame"][:, 3:]).max() < 0.4


@pytest.mark.gpu
def test_basic_calibration_from_seed():
    """test/test-basic-calibration.py: 4 OPENCV4 cameras, 50 frames of a 10x9 board, 1.5 px noise, 1% of the corners
    off by 20x that, seeded by seed_stereographic(focal 1500), solved in the stages of mrcal-calibrate-cameras
    (:386-826). Tolerances from test-basic-calibration.py:168-330."""
    import mrcal_b200
    pixel_noise = 1.5
    kw, truth = synthetic.make_problem(lensmodel="LENSMODEL_OPENCV4", Ncameras=4, Nframes=50, W=10, H=9, seed=0,
                                       pixel_noise=pixel_noise, weights=(1.0, 1.0))
    rng = np.random.default_rng(5)
    obs = kw["observations_board"]
    flat = obs.reshape(-1, 3)
    iout = rng.choice(flat.shape[0], flat.shape[0] // 100, replace=False)
    flat[iout, :2] += rng.normal(0, 20 * pixel_noise, (len(iout), 2))
    indices = kw["indices_frame_camintrinsics_camextrinsics"]
    intr, rt_cam_ref, rt_ref_frame = S.seed_stereographic(kw["imagersizes"], 1500., indices[:, :2], obs,
                                                          kw["calibration_object_spacing"])
    args = dict(intrinsics=np.ascontiguousarray(intr), rt_cam_ref=np.ascontiguousarray(rt_cam_ref),
                rt_ref_frame=np.ascontiguousarray(rt_ref_frame), points=None, observations_board=obs,
                indices_frame_camintrinsics_camextrinsics=indices, observations_point=None,
                indices_point_camintrinsics_camextrinsics=None, lensmodel="LENSMODEL_STEREOGRAPHIC",
                imagersizes=kw["imagersizes"], calobject_warp=None, calibration_object_spacing=kw["calibration_object_spacing"],
                do_apply_outlier_rejection=False, do_apply_regularization=False, verbose=False)
    # stage 1: geometry only; stage 2: + the core
    mrcal_b200.optimize(**args, do_optimize_intrinsics_core=False, do_optimize_intrinsics_distortions=False,
                        do_optimize_extrinsics=True, do_optimize_frames=True, do_optimize_calobject_warp=False)
    mrcal_b200.optimize(**args, do_optimize_intrinsics_core=True, do_optimize_intrinsics_distortions=False,
                        do_optimize_extrinsics=True, do_optimize_frames=True, do_optimize_calobject_warp=False)
    # stage 3: the real lens model, distortions seeded near 0 (mrcal-calibrate-cameras:601-634)
    intr4 = np.zeros((4, 8))
    intr4[:, :4] = args["intrinsics"]
    intr4[:, 4:] = (rng.random((4, 4)) - 0.5) * 1e-6
    args.update(intrinsics=intr4, lensmodel="LENSMODEL_OPENCV4", do_apply_regularization=True)
    mrcal_b200.optimize(**args, do_optimize_intrinsics_core=True, do_optimize_intrinsics_distortions=True,
                        do_optimize_extrinsics=True, do_optimize_frames=True, do_optimize_calobject_warp=False)
    # stage 4: + the board warp, with outlier rejection
    args.update(calobject_warp=np.zeros(2), do_apply_outlier_rejection=True)
    stats = mrcal_b200.optimize(**args, do_optimize_intrinsics_core=True, do_optimize_intrinsics_distortions=True,
                                do_optimize_extrinsics=True, do_optimize_frames=True, do_optimize_calobject_warp=True)
    # test-basic-calibration.py: rms within 2.5 px (:238), warp to 2e-3 (:243-247), extrinsics to 5 cm / 1 deg (:270-300)
    assert stats["rms_reproj_error__pixels"] < pixel_noise * 1.2
    assert stats["Noutliers_board"] >= 0.7 * len(iout) and stats["Noutliers_board"] <= 3 * len(iout)
    assert np.abs(args["calobject_warp"] - truth["calobject_warp"]).max() < 2e-3
    assert np.abs(args["rt_cam_ref"][:, 3:] - truth["rt_cam_ref"][:, 3:]).max() < 0.05
    assert np.abs(args["rt_cam_ref"][:, :3] - truth["rt_cam_ref"][:, :3]).max() < np.pi / 180.
    assert np.abs(args["intrinsics"][:, :2] / truth["intrinsics"][:, :2] - 1.).max() < 0.01
