"""Time the unprojection with gradients and the analyses built on it. Cases: unproject(get_gradients=True,
normalize=True) for the test models cam0 OPENCV8 and cam0 splined (tests/golden/cameramodels, 4000x2200) on a 400-wide
grid (the dense dv/dintrinsics of the splined model's full imager would be about 75 GB); model_resolution__deg_pixel()
at every pixel of the full imager for both; stereo_pair_diff() of the splined cam0/cam1 pair against the OPENCV8 pair
at 5 m on grids 60 and 400 wide. Each: the median call in ms (every timed call ends with a device synchronisation),
and the device time of its kernels from torch.profiler in a separate run. Prints one JSON line with the card's name,
power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
import measure  # noqa: E402


def timed(f, reps, *kernels):
    return dict(ms_call=measure.median_ms(f, reps), ms_kernels=measure.kernel_ms(f, *kernels))


def main():
    gold = os.path.join(ROOT, "tests", "golden", "cameramodels")
    m = {k: [mrcal_b200.cameramodel(os.path.join(gold, f"cam{i}.{k}.cameramodel")) for i in (0, 1)]
         for k in ("opencv8", "splined")}
    out = {}
    for k, (m0, _) in m.items():
        W, H = m0.imagersize()
        lm, intr = m0.intrinsics()
        q = mrcal_b200.sample_imager(400, None, W, H)
        r = timed(lambda: mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True), 5, "unproject_kernel")
        r["grid"] = list(q.shape[:2])
        r["Nintrinsics"] = len(intr)
        out[f"unproject_gradients_{k}_grid400"] = r
        qf = mrcal_b200.sample_imager(W, H, W, H)
        r = timed(lambda: mrcal_b200.model_resolution__deg_pixel(qf, m0), 3, "resolution_kernel")
        r["pixels"] = int(W * H)
        out[f"model_resolution_{k}_full"] = r
    for gridn in (60, 400):
        pairs = (m["splined"], m["opencv8"])
        r = timed(lambda: mrcal_b200.stereo_pair_diff(pairs, gridn_width=gridn, distance=5.), 5,
                  "unproject_kernel", "reproject_diff_kernel")
        out[f"stereo_pair_diff_5m_grid{gridn}"] = r
    measure.emit(out)


if __name__ == "__main__":
    main()
