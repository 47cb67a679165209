#!/usr/bin/env python3
"""Writes tests/golden/transform_image.npz: what OpenCV computes, for the tests of transform_image() and
image_transformation_map() to compare against without importing cv2. Run where cv2 imports:

    python tests/golden/make_transform_golden.py

For each of uint8/uint16/float32 x 1/3 channels x INTER_NEAREST/INTER_LINEAR x BORDER_CONSTANT/BORDER_TRANSPARENT,
key prefix "<dtype>_c<channels>_i<interpolation>_b<border>_": the seeded source image (29 x 37), the map (with the
special values of remap_np.special_map()), the pre-filled out, the border value and cv2.remap()'s result. Then
cv2.initUndistortRectifyMap()'s maps for cam0.opencv8 into pinhole_model_for_reprojection(scale_image=0.1), as the
reference's image_transformation_map() special case computes them, without ("undistort_") and with ("rotated_") a
rotation R_to_from; every 4th row and column of them, to keep the file small."""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import remap_np  # noqa: E402

H, W, HO, WO = 29, 37, 41, 47
DTYPES = {"uint8": np.uint8, "uint16": np.uint16, "float32": np.float32}


def main():
    out = {}
    seed = 0
    for name, dtype in DTYPES.items():
        for channels in (1, 3):
            for interpolation in (cv2.INTER_NEAREST, cv2.INTER_LINEAR):
                for border in (cv2.BORDER_CONSTANT, cv2.BORDER_TRANSPARENT):
                    seed += 1
                    key = f"{name}_c{channels}_i{interpolation}_b{border}_"
                    image = remap_np.seeded_image(H, W, channels, dtype, seed)
                    mapxy = remap_np.special_map(HO, WO, H, W, seed + 100)
                    prefill = remap_np.seeded_image(HO, WO, channels, dtype, seed + 200)
                    value = (7., 200., 3.) if channels == 3 else 11.
                    dst = prefill.copy()
                    r = cv2.remap(image, mapxy, None, interpolation=interpolation, borderMode=border,
                                  borderValue=value, dst=dst)
                    out.update({key + "image": image, key + "mapxy": mapxy, key + "out": prefill,
                                key + "border_value": np.atleast_1d(value), key + "result": r})

    import mrcal_b200
    m = mrcal_b200.cameramodel(os.path.join(HERE, "cameramodels", "cam0.opencv8.cameramodel"))
    pinhole = mrcal_b200.pinhole_model_for_reprojection(m, scale_focal=1., scale_image=0.1)
    lensmodel, intr = m.intrinsics()
    _, intr_to = pinhole.intrinsics()
    K = lambda i: np.array(((i[0], 0, i[2]), (0, i[1], i[3]), (0, 0, 1.)))
    R = cv2.Rodrigues(np.array((0.01, -0.02, 0.015)))[0]
    for key, RR in (("undistort_", None), ("rotated_", R)):
        mx, my = cv2.initUndistortRectifyMap(K(intr), intr[4:], RR, K(intr_to), tuple(int(x) for x in pinhole.imagersize()),
                                             cv2.CV_32FC1)
        out[key + "mapxy"] = np.stack((mx, my), axis=-1)[::4, ::4]
        out[key + "R_to_from"] = np.eye(3) if RR is None else RR
    np.savez_compressed(os.path.join(HERE, "transform_image.npz"), **out)


if __name__ == "__main__":
    main()
