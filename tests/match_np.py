"""match_feature() restated in numpy, one feature at a time: the reference's control flow (mrcal/stereo.py:1853-2046)
around the device's definition of the match output (DESIGN.md section 4.10) and of the sub-pixel fit. The tests
compare the device with this bit for bit, and this with OpenCV's cv2.matchTemplate() within its rounding."""
import numpy as np

import remap_np

TM_SQDIFF, TM_SQDIFF_NORMED, TM_CCORR, TM_CCORR_NORMED, TM_CCOEFF, TM_CCOEFF_NORMED = range(6)
MATCH_OK, MATCH_EDGE_PEAK, MATCH_OUTSIDE_IMAGE1, MATCH_OUTSIDE_IMAGE0, MATCH_SEARCH_TOO_SMALL = range(5)

TEN_FLT_EPS = float(np.float32(10) * np.finfo(np.float32).eps)
DBL_EPSILON = np.finfo(np.float64).eps

# pinv of the 9x6 design matrix (1, x, y, x^2, xy, y^2 on the 3x3 neighbourhood, x fastest), as integers over a
# denominator per coefficient
FIT_NUM = ((-1, 2, -1, 2, 5, 2, -1, 2, -1),
           (-1, 0, 1, -1, 0, 1, -1, 0, 1),
           (-1, -1, -1, 0, 0, 0, 1, 1, 1),
           (1, -2, 1, 1, -2, 1, 1, -2, 1),
           (1, 0, -1, 0, 0, 0, -1, 0, 1),
           (1, 1, 1, -2, -2, -2, 1, 1, 1))
FIT_DEN = (9., 6., 6., 6., 4., 6.)


def apply_homography(H, q):
    """((H00 x + H01 y) + H02) / ((H20 x + H21 y) + H22), and likewise for y, in the inputs' precision"""
    x, y = q[..., 0], q[..., 1]
    xyz = [(H[..., i, 0] * x + H[..., i, 1] * y) + H[..., i, 2] for i in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.stack((xyz[0] / xyz[2], xyz[1] / xyz[2]), axis=-1)


def _normed(num, diff2, wsum2, tnorm, sqdiff):
    """OpenCV's rule for a small denominator, elementwise"""
    with np.errstate(invalid="ignore", divide="ignore"):
        diff2 = np.where(diff2 < 0., 0., diff2)
        thr = np.fmin(0.5, TEN_FLT_EPS * wsum2)
        t = np.where(diff2 <= thr, 0., np.sqrt(diff2) * tnorm)
        a = np.abs(num)
        beyond = 1. if sqdiff else 0.
        return np.where(a < t, num / t, np.where(a < t * 1.125, np.where(num > 0., 1., -1.), beyond))


def _window_sums(cut, template):
    """(SI, SI2, STI) for every window position: exact int64 for uint8; fp64 summed one element at a time, row-major
    over the template, for float32"""
    th, tw = template.shape
    win = np.lib.stride_tricks.sliding_window_view(cut, (th, tw))
    if cut.dtype == np.uint8:
        w = win.astype(np.int64)
        t = template.astype(np.int64)
        return w.sum((2, 3)), (w * w).sum((2, 3)), (w * t).sum((2, 3))
    oh, ow = win.shape[:2]
    SI, SI2, STI = np.zeros((oh, ow)), np.zeros((oh, ow)), np.zeros((oh, ow))
    for v in range(th):
        for u in range(tw):
            x = win[:, :, v, u].astype(np.float64)
            y = np.float64(template[v, u])
            SI = SI + x
            SI2 = SI2 + x * x
            STI = STI + y * x
    return SI, SI2, STI


def match_output(cut, template, method):
    """The match output (oh, ow), float32, of template over the image cut, as the device defines it"""
    n = template.size
    nd = float(n)
    SI, SI2, STI = _window_sums(cut, template)
    if cut.dtype == np.uint8:
        t = template.astype(np.int64).ravel()
        ST, ST2 = int(t.sum()), int((t * t).sum())
        sq = (SI2 - 2 * STI + ST2).astype(np.float64)
        cc = STI.astype(np.float64)
        co = (n * STI - ST * SI).astype(np.float64) / nd
        eT = float(n * ST2 - ST * ST) / nd
        eI = (n * SI2 - SI * SI).astype(np.float64) / nd
        ST2, SI2 = float(ST2), SI2.astype(np.float64)
    else:
        t = template.astype(np.float64).ravel()
        ST, ST2 = np.add.accumulate(t)[-1], np.add.accumulate(t * t)[-1]
        with np.errstate(invalid="ignore"):
            sq = (SI2 - 2. * STI) + ST2
            sq = np.where(sq < 0., 0., sq)
        cc = STI
        co = (nd * STI - ST * SI) / nd
        eT = (nd * ST2 - ST * ST) / nd
        eI = (nd * SI2 - SI * SI) / nd
    with np.errstate(invalid="ignore"):
        if method == TM_SQDIFF:
            r = sq
        elif method == TM_SQDIFF_NORMED:
            r = _normed(sq, SI2, SI2, np.sqrt(ST2), True)
        elif method == TM_CCORR:
            r = cc
        elif method == TM_CCORR_NORMED:
            r = _normed(cc, SI2, SI2, np.sqrt(ST2), False)
        elif method == TM_CCOEFF:
            r = co
        else:
            r = np.ones_like(co) if eT / nd < DBL_EPSILON else _normed(co, eI, SI2, np.sqrt(eT), False)
    return np.asarray(r, np.float64).astype(np.float32)


def optimum(matchoutput, method):
    """(status, (x, y) of the sub-pixel optimum, its value): numpy's argmin/argmax, the edge test, the quadratic fit
    through the closed-form pseudo-inverse, and the reference's expressions for the optimum"""
    flat = matchoutput.ravel()
    i = int(np.argmin(flat) if method in (TM_SQDIFF, TM_SQDIFF_NORMED) else np.argmax(flat))
    oh, ow = matchoutput.shape
    qy, qx = divmod(i, ow)
    if qx <= 0 or qy <= 0 or qx >= ow - 1 or qy >= oh - 1:
        return MATCH_EDGE_PEAK, None, None
    z = [float(v) for v in matchoutput[qy - 1:qy + 2, qx - 1:qx + 2].ravel()]
    c = []
    for num, den in zip(FIT_NUM, FIT_DEN):
        terms = [a * zj for a, zj in zip(num, z) if a != 0]
        acc = terms[0]
        for term in terms[1:]:
            acc = acc + term
        c.append(acc / den)
    c00, c10, c01, c20, c11, c02 = c
    with np.errstate(all="ignore"):
        det = np.float64(4. * c20 * c02 - c11 * c11)
        x = -np.float64(2. * c10 * c02 - c01 * c11) / det
        y = -np.float64(2. * c01 * c20 - c10 * c11) / det
        value = c00 + c10 * x + c01 * y + c20 * x * x + c11 * x * y + c02 * y * y
    return MATCH_OK, np.array((qx + x, qy + y)), np.float64(value)


def match_feature(image0, image1, q0, *, search_radius1, template_size1, q1_estimate=None, H10=None,
                  method=TM_CCORR_NORMED):
    """One feature, the reference's control flow with the failures as a status instead of an exception. Returns a dict:
    status, and where they exist q1, at, value, qshift, matchoutput, template"""
    ts = np.array(template_size1 if np.ndim(template_size1) else (template_size1, template_size1), dtype=int)
    q0 = np.asarray(q0).astype(np.float32)
    if H10 is None:
        q1e = np.asarray(q1_estimate)
        H10 = np.array(((1., 0., q1e[0] - q0[0]), (0., 1., q1e[1] - q0[1]), (0., 0., 1.)), dtype=np.float32)
        q1e = q1e.astype(np.float32)
    else:
        H10 = np.asarray(H10).astype(np.float32)
        q1e = apply_homography(H10, q0)
    tmin_f = np.round(q1e - (ts - 1.) / 2.)
    H1, W1 = image1.shape
    if not np.all(np.isfinite(tmin_f)):
        return dict(status=MATCH_OUTSIDE_IMAGE1)
    tmin = tmin_f.astype(int)
    tmax = tmin + ts - 1
    for q in (tmin, tmax):
        if q[0] < 0 or q[1] < 0 or q[0] >= W1 or q[1] >= H1:
            return dict(status=MATCH_OUTSIDE_IMAGE1)
    grid = np.stack(np.meshgrid(np.arange(tmin[0], tmax[0] + 1), np.arange(tmin[1], tmax[1] + 1)),
                    axis=-1).astype(np.float32)
    try:
        Hinv = np.linalg.inv(H10)
    except np.linalg.LinAlgError:
        return dict(status=MATCH_OUTSIDE_IMAGE0)
    mapxy = apply_homography(Hinv, grid)
    H0, W0 = image0.shape
    for q in (mapxy[0, 0], mapxy[-1, 0], mapxy[0, -1], mapxy[-1, -1]):
        if q[0] < 0 or q[1] < 0 or q[0] >= W0 or q[1] >= H0:
            return dict(status=MATCH_OUTSIDE_IMAGE0)
    template = remap_np.remap(image0, mapxy)
    qmin = tmin - search_radius1
    qmax = tmin + search_radius1 + ts - 1
    qmin = np.maximum(qmin, 0)
    qmax = np.minimum(qmax, (W1 - 1, H1 - 1))
    if np.any(qmax - qmin + 1 < ts):
        return dict(status=MATCH_SEARCH_TOO_SMALL)
    cut = image1[qmin[1]:qmax[1] + 1, qmin[0]:qmax[0] + 1]
    mo = match_output(cut, template, method)
    status, at, value = optimum(mo, method)
    r = dict(status=status, matchoutput=mo, template=template, mapxy=mapxy)
    if status == MATCH_OK:
        qshift = qmin + q1e - tmin
        r.update(at=at, value=value, qshift=qshift, q1=at + qshift)
    return r


def textured_image(H, W, dtype, seed, blur=2):
    """A seeded image with texture at a few pixels' scale: uniform noise, box-blurred `blur` times"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(0, 1, (H + 8, W + 8))
    for _ in range(blur):
        a = (a[:-2, :-2] + a[:-2, 1:-1] + a[:-2, 2:] + a[1:-1, :-2] + a[1:-1, 1:-1] + a[1:-1, 2:] +
             a[2:, :-2] + a[2:, 1:-1] + a[2:, 2:]) / 9.
    a = a[:H, :W]
    a = (a - a.min()) / (a.max() - a.min())
    if dtype == np.uint8:
        return np.round(a * 255.).astype(np.uint8)
    return (a * 200. - 50.).astype(np.float32)
