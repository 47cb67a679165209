"""Time project() and unproject() on torch CUDA tensors against the numpy path of the same calls, for the test models
cam0 OPENCV8 and cam0 splined (tests/golden/cameramodels, 4000x2200). Cases: project() of 10^6 and 10^7 points;
unproject(normalize=True, get_gradients=True) on the 400-wide grid of time_unproject.py; project() of 10^5 points
through 100 stacked intrinsics (each intrinsics row perturbed, broadcast against the points: 10^7 projections). Each:
the median call in ms (every timed call ends with a device synchronisation), the device time of its kernels (and of
the clearing of the dense intrinsics gradient) from torch.profiler in a separate run, the bytes the kernels must move
(every input read once, every output written once) and that traffic as a share of the H100 SXM's 3.35 TB/s data-sheet
bandwidth. Prints one JSON line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
import measure  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def case(f_numpy, f_tensor, nbytes, reps):
    r = {}
    for path, f in (("numpy", f_numpy), ("tensor", f_tensor)):
        ms_kernels = measure.kernel_ms(f, "project_kernel", "Memset")
        r[path] = dict(ms_call=measure.median_ms(f, reps), ms_kernels=ms_kernels)
    r["MB_moved"] = nbytes / 1e6
    r["share_of_peak_bw"] = nbytes / (r["tensor"]["ms_kernels"] * 1e-3) / PEAK_BYTES_PER_S
    return r


def points(n, seed=0):
    rng = np.random.default_rng(seed)
    p = rng.uniform(-1., 1., (n, 3))
    p[:, 2] += 2.
    return p


def main():
    gold = os.path.join(ROOT, "tests", "golden", "cameramodels")
    out = {}
    for k in ("opencv8", "splined"):
        m = mrcal_b200.cameramodel(os.path.join(gold, f"cam0.{k}.cameramodel"))
        W, H = m.imagersize()
        lm, intr = m.intrinsics()
        N = len(intr)
        ti = torch.tensor(intr, device="cuda")
        for n in (10**6, 10**7):
            p = points(n)
            tp = torch.tensor(p, device="cuda")
            out[f"project_{k}_{n}"] = case(lambda: mrcal_b200.project(p, lm, intr),
                                           lambda: mrcal_b200.project(tp, lm, ti), n * (24 + 16), 5)
        q = mrcal_b200.sample_imager(400, None, W, H)
        tq = torch.tensor(q, device="cuda")
        n = q.shape[0] * q.shape[1]
        r = case(lambda: mrcal_b200.unproject(q, lm, intr, normalize=True, get_gradients=True),
                 lambda: mrcal_b200.unproject(tq, lm, ti, normalize=True, get_gradients=True),
                 n * (16 + 24 + 48 + 24 * N), 5)
        r["grid"] = list(q.shape[:2])
        r["Nintrinsics"] = N
        out[f"unproject_gradients_{k}_grid400"] = r
        # 100 intrinsics rows, each perturbed, against 10^5 points
        rows = intr * (1. + 1e-4 * np.random.default_rng(1).standard_normal((100, 1, N)))
        trows = torch.tensor(rows, device="cuda")
        p = points(10**5, 2)
        tp = torch.tensor(p, device="cuda")
        out[f"project_{k}_100x100000"] = case(lambda: mrcal_b200.project(p, lm, rows),
                                              lambda: mrcal_b200.project(tp, lm, trows),
                                              10**5 * 24 + 100 * N * 8 + 10**7 * 16, 5)
        # the last elements of the stacked case agree between the two paths
        assert np.array_equal(mrcal_b200.project(p[-3:], lm, rows[-2:]),
                              mrcal_b200.project(tp[-3:], lm, trows[-2:]).cpu().numpy())
    measure.emit(out)


if __name__ == "__main__":
    main()
