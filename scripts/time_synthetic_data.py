"""Time the synthetic-data functions: synthesize_board_observations() for 8 cameras, 10x10 boards and Nframes = 1000
and 10000, with a splined order-3 and an OPENCV8 lens; and make_perfect_observations() on BASELINE config 5
(synthetic.baseline_config(5): 8 splined cameras, 1000 frames, 2000 points). Each: the call time (median, host clock
ending in a device synchronisation), the device time of its kernels from torch.profiler, and, where oracle/_ref was
built, the same computation in numpy with the compiled reference's project() on the CPU (one chunk of frames for the
synthesis). Prints one JSON line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys
import time

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402
from mrcal_b200._poses_host import Rt_from_rt  # noqa: E402
import measure  # noqa: E402
from oracle import ref  # noqa: E402

SPLINED = "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=30_Ny=20_fov_x_deg=170"
IMAGERSIZE = (4000, 2200)
BOARD = dict(object_width_n=10, object_height_n=10, object_spacing=0.1, calobject_warp=np.array((0.002, -0.005)))
RT_CENTER = np.array((0., 0., 0., -1.4, 0., 4.))
RT_RADIUS = np.array((0.3, 0.3, 0.2, 1.5, 1.0, 0.8))


def host_ms(f):
    t0 = time.perf_counter()
    f()
    return 1e3 * (time.perf_counter() - t0)


def cameras(lm):
    intr = synthetic.true_intrinsics(lm, 8, np.random.default_rng(0))
    return [mrcal_b200.cameramodel(intrinsics=(lm, intr[c]), imagersize=IMAGERSIZE,
                                   rt_cam_ref=np.array((0., 0.01 * c, 0., -0.4 * c, 0., 0.))) for c in range(8)]


def synthesize_numpy_ref(models, Nframes):
    """One chunk of synthesize_board_observations() on the CPU: numpy transforms, the reference's project()"""
    W, H, s = BOARD["object_width_n"], BOARD["object_height_n"], BOARD["object_spacing"]
    board = mrcal_b200.ref_calibration_object(W, H, s, calobject_warp=BOARD["calobject_warp"]) - \
        np.array(((W - 1) * s / 2., (H - 1) * s / 2., 0.))
    Rt = Rt_from_rt(RT_CENTER + np.random.uniform(-1., 1., (Nframes, 6)) * RT_RADIUS)
    pref = np.einsum("fij,nj->fni", Rt[:, :3, :], board.reshape(-1, 3)) + Rt[:, None, 3, :]
    q = []
    for m in models:
        Rc = m.Rt_cam_ref()
        pcam = pref @ Rc[:3, :].T + Rc[3]
        q.append(ref.project(pcam.reshape(-1, 3), *m.intrinsics()))
    return q


def make_perfect_numpy_ref(kw):
    """The projections of make_perfect_observations() on the CPU: numpy poses and transforms, the reference's project()"""
    idx = kw["indices_frame_camintrinsics_camextrinsics"]
    board = mrcal_b200.ref_calibration_object(optimization_inputs=kw).reshape(-1, 3)
    Rt_f = Rt_from_rt(kw["rt_ref_frame"])[idx[:, 0]]
    Rt_c = np.concatenate((np.concatenate((np.eye(3), np.zeros((1, 3))))[None], Rt_from_rt(kw["rt_cam_ref"])))
    Rc = Rt_c[idx[:, 2] + 1]
    R = Rc[:, :3, :] @ Rt_f[:, :3, :]
    t = np.einsum("oij,oj->oi", Rc[:, :3, :], Rt_f[:, 3, :]) + Rc[:, 3, :]
    pcam = np.einsum("oij,nj->oni", R, board) + t[:, None, :]
    for c in np.unique(idx[:, 1]):
        ref.project(pcam[idx[:, 1] == c].reshape(-1, 3), kw["lensmodel"], kw["intrinsics"][c])
    ip = kw["indices_point_camintrinsics_camextrinsics"]
    pc = np.einsum("oij,oj->oi", Rt_c[ip[:, 2] + 1][:, :3, :], kw["points"][ip[:, 0]]) + Rt_c[ip[:, 2] + 1][:, 3, :]
    for c in np.unique(ip[:, 1]):
        ref.project(pc[ip[:, 1] == c], kw["lensmodel"], kw["intrinsics"][c])


def chunks_drawn(Nframes):
    """How many chunks of Nframes poses the last call from np.random.seed(0) drew: the np.random state it left is
    that of that many uniform blocks"""
    key = np.random.get_state()[1].copy(), np.random.get_state()[2]
    for k in range(1, 1000):
        np.random.seed(0)
        np.random.uniform(-1., 1., (k * Nframes, 6))
        if np.array_equal(np.random.get_state()[1], key[0]) and np.random.get_state()[2] == key[1]:
            return k
    raise RuntimeError("could not count the chunks")


def main():
    out = {}
    for lm, tag in ((SPLINED, "splined3"), ("LENSMODEL_OPENCV8", "opencv8")):
        models = cameras(lm)
        for Nframes in (1000, 10000):
            def f():
                np.random.seed(0)
                return mrcal_b200.synthesize_board_observations(
                    models, **BOARD, rt_ref_boardcenter=RT_CENTER, rt_ref_boardcenter__noiseradius=RT_RADIUS,
                    Nframes=Nframes, which="some-cameras-must-see-half-board")
            np.random.seed(0)
            f()
            chunks = chunks_drawn(Nframes)
            r = dict(ms_call=measure.median_ms(f, 5),
                     ms_kernels=measure.kernel_ms(f, "synthesize_kernel", "Rt_from_rt_kernel"),
                     ms_device_total=measure.kernel_ms(f, "synthesize_kernel", "Rt_from_rt_kernel", "Memcpy"),
                     projections=8 * 100 * Nframes * chunks, chunks=chunks)
            if ref.available():
                np.random.seed(0)
                r["ms_numpy_ref_one_chunk"] = host_ms(lambda: synthesize_numpy_ref(models, Nframes))
            out[f"synthesize_{tag}_{Nframes}"] = r
    kw, _ = synthetic.baseline_config(5)
    clone = lambda: {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in kw.items()}
    for sigma, tag in ((0., "noiseless"), (0.3, "sigma0.3"), (None, "sigma_estimated")):
        def g():
            np.random.seed(1)
            mrcal_b200.make_perfect_observations(clone(), observed_pixel_uncertainty=sigma)
        r = dict(ms_call=measure.median_ms(g, 3),
                 ms_kernels=measure.kernel_ms(g, "board_corners_kernel", "point_kernel", "observation_poses_kernel"),
                 board_projections=int(kw["observations_board"][..., 0].size),
                 point_projections=int(kw["observations_point"].shape[0]))
        out[f"make_perfect_observations_baseline5_{tag}"] = r
    if ref.available():
        out["make_perfect_observations_baseline5_noiseless"]["ms_numpy_ref"] = host_ms(lambda: make_perfect_numpy_ref(kw))
    measure.emit(out, os.environ.get("TIME_SYNTHETIC_DATA_OUT"))


if __name__ == "__main__":
    main()
