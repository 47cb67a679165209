#!/usr/bin/env python3
"""Writes tests/golden/match_feature.npz: what OpenCV computes, for the tests of match_feature() to compare against
without importing cv2. Run where cv2 imports:

    python tests/golden/make_match_golden.py

For each of uint8/float32 ("<dtype>_"): seeded textured images image0 (48 x 64) and a cut of image1 (40 x 52), the
float32 map of a perspective H10 over a 17 x 13 template (apply_homography(inv(H10), q1), as match_feature() forms it),
cv2.remap()'s template through that map (INTER_LINEAR, BORDER_CONSTANT 0), and cv2.matchTemplate()'s output of that
template over the cut for each method ("<dtype>_m<method>").

Degenerate cases ("degenerate_<name>_"): a cut, a template, the method and cv2.matchTemplate()'s output:
- flat_template: a constant template, CCOEFF_NORMED: 1 everywhere;
- flat_window: a constant cut, CCOEFF_NORMED: 0;
- zero_window_ccorr / zero_window_sqdiff: an all-zero cut, CCORR_NORMED: 0 and SQDIFF_NORMED: 1;
- sqdiff_beyond: SQDIFF_NORMED with num / t >= 1.125: 1;
- band_sqdiff: SQDIFF_NORMED with 1 <= num / t < 1.125 (the +-1 band of OpenCV's rule): 1. The band and the branch
  beyond it both give 1 for SQDIFF_NORMED, so this case only pins that a ratio just above 1 is not returned as
  num / t; it cannot tell the band from the branch beyond;
- band_ccorr: CCORR_NORMED of a window equal to a template whose energy is a perfect square (num == t): 1. It tells the
  band from a rule without one (which would give 0 for |num| >= t), not from a plain num / t (also 1);
- band_ccoeff: CCOEFF_NORMED of a window 255 - template, its centred energy a perfect square (num == -t): -1. This is
  the case that pins the band: without it the rule gives 0, and only the band gives the sign.
By Cauchy-Schwarz, |num| <= t for the correlation methods, so they reach the band only at equality; only SQDIFF_NORMED
goes strictly inside (1, 1.125). The band cases are 1x1 outputs, so the window is the whole cut.

Refusals ("refuses_<name>", 1 if cv2.matchTemplate() raised): uint16 images, mixed dtypes, a cut smaller than the
template."""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import match_np  # noqa: E402

TW, TH = 17, 13
H10 = np.array(((1.04, 0.06, 3.3), (-0.05, 0.97, -1.7), (2e-4, -1.5e-4, 1.)))
Q1_TEMPLATE_MIN = (20, 14)   # in image1 coordinates; the cut starts at (0, 0)


def _refuses(f):
    try:
        f()
    except cv2.error:
        return 1
    return 0


def _band_sqdiff():
    """a template (a, 0) and a window (p, q) of uint8 with 1 <= (|I|^2 + |T|^2 - 2 I.T) / (|I| |T|) < 1.125, the
    ratio as far inside the band as the search finds"""
    best = None
    a = 100
    for p in range(0, 256):
        for q in range(0, 256):
            ratio = (p * p + q * q + a * a - 2 * a * p) / (a * np.hypot(p, q)) if p or q else 0.
            if 1.02 <= ratio <= 1.1 and (best is None or abs(ratio - 1.06) < abs(best[2] - 1.06)):
                best = (p, q, ratio)
    p, q, _ = best
    T = np.zeros((3, 3), np.uint8)
    T[1, 1] = a
    I = np.zeros((3, 3), np.uint8)
    I[1, 1], I[0, 0] = p, q
    return I, T


def main():
    out = {}
    for name, dtype in (("uint8", np.uint8), ("float32", np.float32)):
        image0 = match_np.textured_image(48, 64, dtype, 1)
        cut = match_np.textured_image(40, 52, dtype, 2)
        grid = np.stack(np.meshgrid(np.arange(Q1_TEMPLATE_MIN[0], Q1_TEMPLATE_MIN[0] + TW),
                                    np.arange(Q1_TEMPLATE_MIN[1], Q1_TEMPLATE_MIN[1] + TH)), -1).astype(np.float32)
        mapxy = match_np.apply_homography(np.linalg.inv(H10.astype(np.float32)), grid)
        template = cv2.remap(image0, mapxy, None, interpolation=cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT,
                             borderValue=0)
        # the template from the map is a textured one; plant it in the cut, a little changed, so the match has a peak
        cut[9:9 + TH, 23:23 + TW] = (template.astype(np.float64) * 0.9 + 10).astype(dtype)
        out.update({f"{name}_image0": image0, f"{name}_cut": cut, f"{name}_mapxy": mapxy,
                    f"{name}_template": template, f"{name}_H10": H10, f"{name}_q1_template_min": Q1_TEMPLATE_MIN})
        for method in range(6):
            out[f"{name}_m{method}"] = cv2.matchTemplate(cut, template, method)

    rng = np.random.default_rng(7)
    tex = rng.integers(0, 256, (9, 9), dtype=np.uint8)
    cases = {
        "flat_template": (tex, np.full((5, 5), 77, np.uint8), cv2.TM_CCOEFF_NORMED),
        "flat_window": (np.full((9, 9), 77, np.uint8), tex[:5, :5].copy(), cv2.TM_CCOEFF_NORMED),
        "zero_window_ccorr": (np.zeros((9, 9), np.uint8), tex[:5, :5].copy(), cv2.TM_CCORR_NORMED),
        "zero_window_sqdiff": (np.zeros((9, 9), np.uint8), tex[:5, :5].copy(), cv2.TM_SQDIFF_NORMED),
    }
    T = np.zeros((3, 3), np.uint8)
    T[1, 1] = 100
    I = np.zeros((3, 3), np.uint8)
    I[0, 0] = 100
    cases["sqdiff_beyond"] = (I, T, cv2.TM_SQDIFF_NORMED)
    cases["band_sqdiff"] = (*_band_sqdiff(), cv2.TM_SQDIFF_NORMED)
    # energy 3^2 + 4^2 + 12^2 = 13^2
    T = np.zeros((3, 3), np.uint8)
    T[0, 0], T[1, 2], T[2, 1] = 3, 4, 12
    cases["band_ccorr"] = (T.copy(), T, cv2.TM_CCORR_NORMED)
    # 100 + (2, 2, -2, -2, 0, 0, 0, 0, 0): centred energy 16, so t = 4 * 4 = 16 = -num for the window 255 - T
    T = (100 + np.array((2, 2, -2, -2, 0, 0, 0, 0, 0))).astype(np.uint8).reshape(3, 3)
    cases["band_ccoeff"] = ((255 - T).astype(np.uint8), T, cv2.TM_CCOEFF_NORMED)
    for key, (cut, template, method) in cases.items():
        p = f"degenerate_{key}_"
        out[p + "cut"], out[p + "template"], out[p + "method"] = cut, template, method
        out[p + "result"] = cv2.matchTemplate(cut, template, method)

    a16 = np.zeros((20, 20), np.uint16)
    out["refuses_uint16"] = _refuses(lambda: cv2.matchTemplate(a16, a16[:5, :5].copy(), cv2.TM_CCORR_NORMED))
    out["refuses_mixed"] = _refuses(lambda: cv2.matchTemplate(np.zeros((20, 20), np.uint8),
                                                              np.zeros((5, 5), np.float32), cv2.TM_CCORR_NORMED))
    out["refuses_small_cut"] = _refuses(lambda: cv2.matchTemplate(np.zeros((4, 20), np.uint8),
                                                                  np.zeros((5, 5), np.uint8), cv2.TM_CCORR_NORMED))
    out["opencv_version"] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, "match_feature.npz"), **out)


if __name__ == "__main__":
    main()
