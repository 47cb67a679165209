#!/usr/bin/env python3
"""Writes tests/golden/contours_cv2.npz: what OpenCV's cv2.findContours(mask, RETR_EXTERNAL, CHAIN_APPROX_SIMPLE)
and cv2.contourArea() give on the masks the valid-intrinsics region is traced from, for the host restatement in
mrcal_b200/regions.py to be compared against without importing cv2. Run where cv2 imports:

    python tests/golden/make_contours_golden.py

"shapes" (Nmasks, 2) and "masks" (np.packbits of the masks, raveled and concatenated) give the masks; "ncontours"
the number of contours of each, "lengths" the vertices of each contour, "points" (int16) the vertices of all of them
and "areas" their areas, all in cv2's order. The cases are structured_masks() and then seeded random masks at the grid
shapes the regions use (17x30, 20x30, 11x20), some of them smoothed into blobs."""
import os
import sys

import cv2
import numpy as np


def structured_masks():
    """Full, empty, single pixels, single rows and columns, blobs on the border, diagonal-only links, one-pixel
    necks, holes with islands, blobs of equal area"""
    z = lambda: np.zeros((17, 30), np.uint8)
    out = [np.ones((17, 30), np.uint8), z()]
    m = z(); m[8, 14] = 1; out.append(m)
    m = z(); m[0, 0] = 1; out.append(m)
    m = z(); m[16, 29] = 1; out.append(m)
    m = z(); m[5, 3:20] = 1; out.append(m)
    m = z(); m[2:15, 7] = 1; out.append(m)
    m = z(); m[0, :] = 1; out.append(m)
    m = z(); m[:, 29] = 1; out.append(m)
    m = z(); m[0:6, 0:9] = 1; m[11:17, 21:30] = 1; out.append(m)
    m = z(); m[3:9, 3:9] = 1; m[9:15, 9:15] = 1; out.append(m)               # two squares touching at a corner
    m = z(); [m.__setitem__((i, i + 4), 1) for i in range(12)]; out.append(m)   # a diagonal line
    m = z(); m[4:8, 4:8] = 1; m[8:12, 8:12] = 1; m[4:8, 12:16] = 1; out.append(m)
    m = z(); m[2:8, 2:10] = 1; m[9:15, 2:10] = 1; m[8, 5] = 1; out.append(m)   # a one-pixel neck
    m = z(); m[2:8, 2:10] = 1; m[5, 10:20] = 1; m[2:8, 20:28] = 1; out.append(m)
    m = z(); m[1:16, 1:29] = 1; m[4:13, 5:25] = 0; m[7:10, 12:18] = 1; out.append(m)   # a hole with an island
    m = z(); m[1:16, 1:29] = 1; m[4:13, 5:25] = 0; m[6:11, 8:22] = 1; m[7:10, 10:20] = 0; m[8, 15] = 1; out.append(m)
    m = z(); m[2:6, 2:6] = 1; m[10:14, 20:24] = 1; out.append(m)             # equal areas
    m = z(); m[2:6, 20:24] = 1; m[10:14, 2:6] = 1; m[8, 12] = 1; out.append(m)
    m = z(); m[1:4, 1:4] = 1; m[1:4, 6:9] = 1; m[1:4, 11:14] = 1; out.append(m)
    m = np.ones((17, 30), np.uint8); m[8, 15] = 0; out.append(m)
    m = np.ones((17, 30), np.uint8); m[0, 5:9] = 0; m[16, 20] = 0; m[3:14, 0] = 0; out.append(m)
    m = np.ones((20, 30), np.uint8); m[::2, ::2] = 0; out.append(m)
    m = np.zeros((11, 20), np.uint8); m[::2, ::2] = 1; out.append(m)
    m = np.zeros((11, 20), np.uint8); m[1::2, ::2] = 1; m[::2, 1::2] = 1; out.append(m)   # a checkerboard
    return out


def random_masks(n=360, seed=0):
    rng = np.random.default_rng(seed)
    shapes = ((17, 30), (20, 30), (11, 20))
    out = []
    for i in range(n):
        h, w = shapes[i % 3]
        if i % 2:
            f = rng.random((h, w))
            for _ in range(1 + i % 3):
                f = (f + np.roll(f, 1, 0) + np.roll(f, -1, 0) + np.roll(f, 1, 1) + np.roll(f, -1, 1)) / 5.
            m = f > np.quantile(f, rng.uniform(0.2, 0.8))
        else:
            m = rng.random((h, w)) < rng.uniform(0.1, 0.9)
        out.append(m.astype(np.uint8))
    return out


def main():
    masks = structured_masks() + random_masks()
    shapes, bits, points, lengths, ncontours, areas = [], [], [], [], [], []
    for m in masks:
        cs = cv2.findContours(m, cv2.RETR_EXTERNAL, cv2.CHAIN_APPROX_SIMPLE)[-2]
        shapes.append(m.shape)
        bits.append(m.ravel())
        points += [c[:, 0, :] for c in cs]
        lengths += [len(c) for c in cs]
        ncontours.append(len(cs))
        areas += [cv2.contourArea(c) for c in cs]
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "contours_cv2.npz")
    np.savez_compressed(path, opencv_version=np.array(cv2.__version__), shapes=np.array(shapes, np.int32),
                        masks=np.packbits(np.concatenate(bits)), points=np.concatenate(points).astype(np.int16),
                        lengths=np.array(lengths, np.int32), ncontours=np.array(ncontours, np.int32),
                        areas=np.array(areas, np.float64))
    print(f"wrote {path}: {len(masks)} masks, OpenCV {cv2.__version__}", file=sys.stderr)


if __name__ == "__main__":
    main()
