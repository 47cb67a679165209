"""cv2.remap()'s arithmetic with a float32 (H, W, 2) map, restated in numpy: the reference transform_image() tests
compare against, bit for bit. Vectorised; float32 sums are formed left to right, as numpy does element-wise."""
import numpy as np

INT_MIN = -2 ** 31


def cv_round(v):
    """cvRound(float): round half to even; NaN, +-inf and anything outside int32 give INT_MIN"""
    v = np.asarray(v, np.float32)
    ok = (v >= np.float32(-2147483648.)) & (v < np.float32(2147483648.))
    return np.where(ok, np.rint(np.where(ok, v, np.float32(0))).astype(np.int64), INT_MIN)


def _saturate_short(x):
    return np.clip(x, -32768, 32767)


def border_cval(dtype, value, channels):
    """saturate_cast<T>(Scalar(value)[c]): a number v means (v, 0, 0)"""
    v = np.zeros(3)
    a = np.atleast_1d(np.asarray(value, np.float64))
    v[:min(a.size, 3)] = a[:3]
    v = v[:channels]
    if dtype == np.float32:
        return v.astype(np.float32)
    hi = 255 if dtype == np.uint8 else 65535
    return np.clip(np.rint(v), 0, hi).astype(dtype)


def remap(image, mapxy, *, out=None, border=0, border_value=0, interpolation=1):
    """What cv2.remap(image, mapxy, None, interpolation=..., borderMode=border (0: constant, 5: transparent),
    borderValue=border_value, dst=out) returns. Pixels a transparent border leaves are taken from out (0 if None)"""
    img = image if image.ndim == 3 else image[..., None]
    H, W, CN = img.shape
    Ho, Wo = mapxy.shape[:2]
    res = np.zeros((Ho, Wo, CN), image.dtype) if out is None else \
        (out if out.ndim == 3 else out[..., None]).copy()
    cval = border_cval(image.dtype, border_value, CN)
    mx, my = mapxy[..., 0].astype(np.float32), mapxy[..., 1].astype(np.float32)
    if interpolation == 0:
        sx, sy = _saturate_short(cv_round(mx)), _saturate_short(cv_round(my))
        inside = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
        res[inside] = img[sy[inside], sx[inside]]
        if border == 0:
            res[~inside] = cval
        return res if image.ndim == 3 else res[..., 0]

    X, Y = cv_round(mx * np.float32(32)), cv_round(my * np.float32(32))
    fx, fy = X & 31, Y & 31
    sx, sy = _saturate_short(X >> 5), _saturate_short(Y >> 5)
    x1, y1 = sx + 1, sy + 1
    if border == 0:
        write = ~((sx >= W) | (x1 < 0) | (sy >= H) | (y1 < 0))
        ix0, ix1, iy0, iy1 = sx >= 0, x1 < W, sy >= 0, y1 < H
        valid = (ix0 & iy0, ix1 & iy0, ix0 & iy1, ix1 & iy1)
        res[~write] = cval
    else:
        write = (sx >= 0) & (sx < W) & (sy >= 0) & (sy < H)
        x1, y1 = np.minimum(x1, W - 1), np.minimum(y1, H - 1)
        valid = (write,) * 4
    taps = []
    for (xx, yy), ok in zip(((sx, sy), (x1, sy), (sx, y1), (x1, y1)), valid):
        t = img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)]
        taps.append(np.where(ok[..., None], t, cval))
    fx, fy = fx[..., None], fy[..., None]
    if image.dtype == np.uint8:
        w = ((32 - fy) * (32 - fx) * 32, (32 - fy) * fx * 32, fy * (32 - fx) * 32, fy * fx * 32)
        s = sum(t.astype(np.int64) * wi for t, wi in zip(taps, w))
        v = np.minimum((s + (1 << 14)) >> 15, 255).astype(np.uint8)
    else:
        a, b = fx.astype(np.float32) * np.float32(1. / 32), fy.astype(np.float32) * np.float32(1. / 32)
        one = np.float32(1)
        w = ((one - b) * (one - a), (one - b) * a, b * (one - a), b * a)
        t = [x.astype(np.float32) for x in taps]
        s = ((t[0] * w[0] + t[1] * w[1]) + t[2] * w[2]) + t[3] * w[3]
        v = s if image.dtype == np.float32 else np.clip(cv_round(s), 0, 65535).astype(np.uint16)
    res[write] = v[write]
    return res if image.ndim == 3 else res[..., 0]


def special_map(Ho, Wo, H, W, seed):
    """A map over a source of H x W pixels that exercises every rule: fractional coordinates in and around the image,
    exact ties of the 1/32 grid (x*32 = k + 0.5) and of the integer grid, the last row and column, -1, NaN, +-inf and
    1e9"""
    rng = np.random.default_rng(seed)
    m = np.empty((Ho, Wo, 2), np.float32)
    m[..., 0] = rng.uniform(-3., W + 2., (Ho, Wo))
    m[..., 1] = rng.uniform(-3., H + 2., (Ho, Wo))
    flat = m.reshape(-1, 2)
    n = flat.shape[0]
    idx = rng.permutation(n)
    k = n // 12
    ties = (rng.integers(-64, 32 * W + 64, (k, 2)) + 0.5) / 32.
    ties[:, 1] = (rng.integers(-64, 32 * H + 64, k) + 0.5) / 32.
    flat[idx[:k]] = ties
    flat[idx[k:2 * k]] = rng.integers(-2, max(W, H) + 2, (k, 2)) + 0.5
    flat[idx[2 * k:3 * k], 0] = W - 1 + rng.uniform(-1., 1., k)
    flat[idx[3 * k:4 * k], 1] = H - 1 + rng.uniform(-1., 1., k)
    specials = np.array((-1., np.nan, np.inf, -np.inf, 1e9, -1e9, 6e7, 0., -0.5, -1. / 64), np.float32)
    j = idx[4 * k:5 * k]
    flat[j, rng.integers(0, 2, j.size)] = specials[rng.integers(0, specials.size, j.size)]
    return m


def seeded_image(H, W, channels, dtype, seed):
    rng = np.random.default_rng(seed)
    shape = (H, W) if channels == 1 else (H, W, channels)
    if dtype == np.float32:
        return rng.uniform(-1000., 1000., shape).astype(np.float32)
    return rng.integers(0, np.iinfo(dtype).max + 1, shape, dtype=np.int64).astype(dtype)


def assert_matches_opencv(result, ref, image, mapxy, float_transparent_linear):
    """result == ref, bit for bit. Except for float32 + INTER_LINEAR + BORDER_TRANSPARENT: there OpenCV (4.13) sums
    the taps of pixels that sample the image's last row or column in an order of its own. Those pixels, and only
    those, may differ by the rounding error of a 4-term float32 sum: 4 ulps of the image's largest magnitude"""
    if not float_transparent_linear:
        np.testing.assert_array_equal(result, ref)
        return
    H, W = image.shape[:2]
    differs = result != ref
    if differs.ndim == 3:
        differs = differs.any(axis=-1)
    X, Y = cv_round(mapxy[..., 0] * np.float32(32)) >> 5, cv_round(mapxy[..., 1] * np.float32(32)) >> 5
    assert np.all(((X == W - 1) | (Y == H - 1))[differs])
    tol = 4 * np.spacing(np.float32(np.abs(image).max()))
    assert np.abs(result.astype(np.float64) - ref.astype(np.float64)).max() <= tol
