#!/usr/bin/env python3
"""Times match_feature() on the device against the per-feature loop the reference's tools run: a 4096 x 3000 uint8
pair, 10 000 features, a 31 x 31 template, search radius 20, TM_CCORR_NORMED.

The device call (numpy images: upload, kernels, one download) is warmed up, then timed as the median of 5 calls; each
call returns numpy arrays, so it ends in a device synchronisation. The same with the images already on the device as
torch tensors, and the device time of each of its kernels and copies from torch.profiler. The per-feature loops -- the
numpy restatement (tests/match_np.py) and, where cv2 imports, the reference's own sequence of cv2.remap(),
cv2.matchTemplate() and np.linalg.lstsq() -- are timed on a sample of features and extrapolated to all of them. Prints
one JSON line with the card's name, power limit and SM clocks as separate fields (card, power_limit, sm_clock,
max_sm_clock), which replace the one unparsed `gpu` string this line used to carry.

    python scripts/time_match_feature.py [--features 10000] [--sample 100]"""
import argparse
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import mrcal_b200  # noqa: E402
import match_np  # noqa: E402
import measure  # noqa: E402

# what one call with device images runs, in launch order; each is timed from torch.profiler
KERNELS = ("Memcpy HtoD", "template_maps_kernel", "remap_kernel", "template_sums_kernel", "match_kernel",
           "match_optimum_kernel", "Memcpy DtoH")


def cv2_loop(cv2, image0, image1, q0, H10, r, ts):
    """the reference's per-feature sequence (mrcal/stereo.py:1876-2040), restated with cv2 and numpy"""
    x, y = np.meshgrid(np.arange(3) - 1., np.arange(3) - 1.)
    x, y = x.ravel(), y.ravel()
    M = np.stack((np.ones(9), x, y, x * x, x * y, y * y), 1)
    for i in range(len(q0)):
        H = H10[i].astype(np.float32)
        q1e = mrcal_b200.apply_homography(H, q0[i].astype(np.float32))
        tmin = np.round(q1e - (ts - 1.) / 2.).astype(int)
        grid = np.stack(np.meshgrid(np.arange(tmin[0], tmin[0] + ts), np.arange(tmin[1], tmin[1] + ts)),
                        -1).astype(np.float32)
        template = cv2.remap(image0, mrcal_b200.apply_homography(np.linalg.inv(H), grid), None, cv2.INTER_LINEAR)
        qmin = np.maximum(tmin - r, 0)
        qmax = np.minimum(tmin + r + ts - 1, (image1.shape[1] - 1, image1.shape[0] - 1))
        mo = cv2.matchTemplate(image1[qmin[1]:qmax[1] + 1, qmin[0]:qmax[0] + 1], template, cv2.TM_CCORR_NORMED)
        qy, qx = np.unravel_index(np.argmax(mo), mo.shape)
        if 0 < qx < mo.shape[1] - 1 and 0 < qy < mo.shape[0] - 1:
            np.linalg.lstsq(M, mo[qy - 1:qy + 2, qx - 1:qx + 2].ravel(), rcond=None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--features", type=int, default=10000)
    ap.add_argument("--sample", type=int, default=100)
    a = ap.parse_args()
    W, H, ts, r = 4096, 3000, 31, 20
    rng = np.random.default_rng(0)
    image0 = match_np.textured_image(H, W, np.uint8, 1)
    image1 = np.ascontiguousarray(np.pad(image0, ((0, 3), (0, 5)), mode="edge")[3:, 5:])
    q0 = rng.uniform(60, (W - 60, H - 60), (a.features, 2))
    H10 = np.tile(np.eye(3), (a.features, 1, 1))
    H10[:, :2, :2] += rng.uniform(-0.03, 0.03, (a.features, 2, 2))
    H10[:, :2, 2] = (-5., -3.)
    kw = dict(search_radius1=r, template_size1=ts, H10=H10)

    out = dict(features=a.features, image=f"{W}x{H} uint8", template=ts, search_radius=r, method="TM_CCORR_NORMED")
    q1, d = mrcal_b200.match_feature(image0, image1, q0, **kw)
    out["matched"] = int(np.sum(d["status"] == mrcal_b200.MATCH_OK))
    out["device_numpy_ms"] = measure.median_ms(lambda: mrcal_b200.match_feature(image0, image1, q0, **kw), 5)
    t0, t1 = torch.from_numpy(image0).cuda(), torch.from_numpy(image1).cuda()
    device_call = lambda: mrcal_b200.match_feature(t0, t1, q0, **kw)
    out["device_torch_ms"] = measure.median_ms(device_call, 5)
    out["kernels_us"] = {k: round(1e3 * measure.kernel_ms(device_call, k), 1) for k in KERNELS}
    # the host loops take seconds per hundred features: one pass over a sample, extrapolated to all the features
    s = rng.choice(a.features, a.sample, replace=False)
    t = time.perf_counter()
    for i in s:
        match_np.match_feature(image0, image1, q0[i], search_radius1=r, template_size1=ts, H10=H10[i])
    out["restatement_loop_ms_extrapolated"] = 1e3 * (time.perf_counter() - t) / a.sample * a.features
    try:
        import cv2
        t = time.perf_counter()
        cv2_loop(cv2, image0, image1, q0[s], H10[s], r, ts)
        out["cv2_loop_ms_extrapolated"] = 1e3 * (time.perf_counter() - t) / a.sample * a.features
    except ImportError:
        out["cv2_loop_ms_extrapolated"] = None
    measure.emit(out)


if __name__ == "__main__":
    main()
