"""Time the stereo functions: rectification_maps() for the splined pair and the OPENCV8 pair of tests/golden/cameramodels
at full resolution (pixels_per_deg = -1), and the dense stereo_range() / stereo_unproject() on a whole rectified image.
For each, the call (arguments, upload, kernels, copy back into numpy) and the device time of its kernels alone
(torch.profiler). Where oracle/_ref was built, the reference's single-threaded C for the same maps and ranges.
Times are medians in ms. Prints one JSON line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
from mrcal_b200._poses_host import Rt_from_rt, compose_Rt, rt_from_Rt  # noqa: E402
from oracle import stereo_ref as ref  # noqa: E402
import measure  # noqa: E402


def pair(names, rt01=(0.1, 0.2, 0.05, 3.0, 0.2, 1.0)):
    gold = os.path.join(ROOT, "tests", "golden", "cameramodels")
    m0, m1 = (mrcal_b200.cameramodel(os.path.join(gold, n)) for n in names)
    m1.rt_ref_cam(rt_from_Rt(compose_Rt(m0.Rt_ref_cam(), Rt_from_rt(rt01))))
    return m0, m1


def case(models, reps):
    res = {}
    rect = mrcal_b200.rectified_system(models, az_fov_deg=90., el_fov_deg=50.)
    W, H = (int(x) for x in rect[0].imagersize())
    res["rectified_imager"] = [W, H]
    maps = lambda: mrcal_b200.rectification_maps(models, rect)
    res["ms_maps_call"] = measure.median_ms(maps, reps)
    res["ms_maps_kernels"] = measure.kernel_ms(maps, "rectification_maps_kernel")
    d = np.random.default_rng(0).integers(0, 2000, size=(H, W)).astype(np.uint16)
    rng = lambda: mrcal_b200.stereo_range(d, rect, disparity_scale=16)
    unp = lambda: mrcal_b200.stereo_unproject(d, rect, disparity_scale=16)
    res["ms_range_call"] = measure.median_ms(rng, reps)
    res["ms_range_kernel"] = measure.kernel_ms(rng, "stereo_range_kernel")
    res["ms_unproject_call"] = measure.median_ms(unp, reps)
    res["ms_unproject_kernel"] = measure.kernel_ms(unp, "stereo_range_kernel")
    if ref.available():
        f, size, r = rect[0].intrinsics()[1], rect[0].imagersize(), rect[0].rt_cam_ref()[:3]
        args = (*models[0].intrinsics(), models[0].rt_cam_ref()[:3], *models[1].intrinsics(), models[1].rt_cam_ref()[:3],
                "LENSMODEL_LATLON", f, size, r)
        # the reference's maps take about a second on one thread: one call after the warm-up
        res["ms_maps_reference_c"] = measure.median_ms(lambda: ref.rectification_maps(*args), 1)
        baseline = float(np.linalg.norm(rect[0].rt_cam_ref()[3:] - rect[1].rt_cam_ref()[3:]))
        res["ms_range_reference_c"] = measure.median_ms(
            lambda: ref.stereo_range_dense(d, 16, 0, 65535, "LENSMODEL_LATLON", f, baseline), 3)
    return res


def main():
    out = {}
    out["splined_pair"] = case(pair(("cam0.splined.cameramodel", "cam1.splined.cameramodel")), 5)
    out["opencv8_pair"] = case(pair(("cam0.opencv8.cameramodel", "cam0.opencv8.cameramodel")), 5)
    measure.emit(out)


if __name__ == "__main__":
    main()
