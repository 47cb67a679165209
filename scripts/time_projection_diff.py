"""Time projection_diff() phase by phase: the unprojection of the grid, the uncertainties (where used), the fit of the
implied transformation and the reprojection. Cases: the test models cam0 OPENCV8 against cam0 splined
(tests/golden/cameramodels) at 5 m without uncertainties, on grids 60 and 400 wide; and cameras 0 and 1 of a solved
BASELINE config 3 at infinity, weighted by their uncertainties, on the 60-wide grid. Each fit is also timed on the
route the reference takes, the scipy fit of tests/diff_np.py, followed by mrcal_b200.project() and the difference in
numpy. Times are medians in ms; every timed call ends with a device synchronisation. Prints one JSON line with the
card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import mrcal_b200  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402
import diff_np  # noqa: E402
import measure  # noqa: E402


def reproject(Rt, q0, v, distance, lms, intr):
    """the C entry point with the transform given: upload, reprojection, download"""
    from mrcal_b200 import _capi, api
    N = q0.shape[0] * q0.shape[1]
    difflen, diff = np.zeros(N), np.zeros((N, 2))
    d = None if distance is None else np.array([float(distance)])
    lm = (_capi.Lensmodel * 2)(*[api._lensmodel(x) for x in lms])
    i = np.concatenate(intr)
    vv = np.ascontiguousarray(v.reshape(2, N, 3))
    fc = np.zeros(2)
    assert _capi.lib.mrcal_b200_projection_diff(Rt.ctypes.data, difflen.ctypes.data, diff.ctypes.data, q0.ctypes.data, N,
                                               vv.ctypes.data, 2, None if d is None else d.ctypes.data, 1, lm,
                                               i.ctypes.data, None, fc.ctypes.data, 1., False), _capi.last_error()
    return difflen


def case(models, gridn, distance, use_uncertainties, reps):
    res = {}
    lms = [m.intrinsics()[0] for m in models]
    intr = [m.intrinsics()[1] for m in models]
    W, H = models[0].imagersize()
    atinfinity = distance is None
    d = 1. if atinfinity else distance
    unp = lambda: mrcal_b200.sample_imager_unproject(gridn, None, W, H, lms, intr, normalize=True)
    res["ms_unproject"] = measure.median_ms(unp, reps)
    v, q0 = unp()
    w = None
    if use_uncertainties:
        unc = lambda: [mrcal_b200.projection_uncertainty(v[k] * d, models[k], atinfinity=atinfinity,
                                                         what="worstdirection-stdev") for k in range(2)]
        res["ms_uncertainties"] = measure.median_ms(unc, reps)
        u = unc()
        w = (1. / (u[0] * u[1])) ** 2
        center, radius = ((W - 1) / 2., (H - 1) / 2.), max(W, H) * 100.
    else:
        center, radius = ((W - 1) / 2., (H - 1) / 2.), min(W, H) / 6.
    kw = dict(weights=w, atinfinity=atinfinity, focus_center=center, focus_radius=radius)
    res["ms_fit"] = measure.median_ms(
        lambda: mrcal_b200.implied_Rt10__from_unprojections(q0, v[0] * d, v[1], **kw), reps)
    Rt = mrcal_b200.implied_Rt10__from_unprojections(q0, v[0] * d, v[1], **kw)
    res["ms_reproject"] = measure.median_ms(
        lambda: reproject(Rt, q0, v, None if atinfinity else distance, lms, intr), reps)
    dist = None if atinfinity else distance
    res["ms_total"] = measure.median_ms(lambda: mrcal_b200.projection_diff(models, gridn_width=gridn, distance=dist,
                                                                           use_uncertainties=use_uncertainties), reps)

    def composed():
        Rt_ref = diff_np.fit(q0, v[0] * d, v[1], **kw)
        return mrcal_b200.project(v[0] * d @ Rt_ref[:3].T + Rt_ref[3], lms[1], intr[1]) - q0
    # the scipy fit takes up to a second: one call after the warm-up
    res["ms_composed_fit_and_reproject"] = measure.median_ms(composed, 1)
    Rt_ref = diff_np.fit(q0, v[0] * d, v[1], **kw)
    res["cost_device_over_scipy"] = (diff_np.robust_cost(Rt, q0, v[0] * d, v[1], **kw) /
                                     diff_np.robust_cost(Rt_ref, q0, v[0] * d, v[1], **kw))
    res["grid"] = list(q0.shape[:2])
    return res


def main():
    gold = os.path.join(ROOT, "tests", "golden", "cameramodels")
    m = [mrcal_b200.cameramodel(os.path.join(gold, f)) for f in ("cam0.opencv8.cameramodel", "cam0.splined.cameramodel")]
    out = {}
    out["opencv8_vs_splined_5m_grid60"] = case(m, 60, 5., False, 10)
    out["opencv8_vs_splined_5m_grid400"] = case(m, 400, 5., False, 5)
    kw, _ = synthetic.baseline_config(3, pixel_noise=0.3, seed=0)
    mrcal_b200.optimize(**kw)
    cams = [mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=i) for i in (0, 1)]
    out["config3_cam0_vs_cam1_infinity_uncertainties_grid60"] = case(cams, 60, None, True, 3)
    measure.emit(out)


if __name__ == "__main__":
    main()
