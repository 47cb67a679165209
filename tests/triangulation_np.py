"""The answers the triangulation tests compare against, the cases they are asked for, and the comparison rules.

The answers are the compiled reference's own mrcal_triangulate_*() and _mrcal_triangulated_error()
(oracle/triangulation_ref.py) where oracle/_ref is built, and the answers stored in tests/golden/triangulation.npz
(tests/golden/make_triangulation_golden.py) otherwise."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "triangulation.npz")
EPS = np.finfo(float).eps
METHODS = ("geometric", "leecivera_l1", "leecivera_linf", "leecivera_mid2", "leecivera_wmid2", "lindstrom")


def unit(v):
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _rotations(rng, n):
    from scipy.spatial.transform import Rotation
    return Rotation.random(n, random_state=rng.integers(1 << 31)).as_matrix()


def geometries(seed=0):
    """(v0, v1, t01, R01), v0 and v1 in camera 0's coordinates, R01 the rotation of camera 1 (v1 local = R01' v1):
    random convergent rays over baselines 1e-3 .. 10 and ranges 0.1 .. 1e4 with a little angular noise, v scaled
    by 1e-3 .. 1e3; rays on both sides of the 1e-10 thresholds; divergent rays; points behind camera 0, camera 1
    and both; t01 = 0; a zero v; NaN inputs"""
    rng = np.random.default_rng(seed)
    v0s, v1s, ts = [], [], []

    def add(v0, v1, t):
        v0s.append(np.atleast_2d(v0))
        v1s.append(np.atleast_2d(v1))
        ts.append(np.atleast_2d(t))

    n = 240
    b = 10 ** rng.uniform(-3, 1, n)
    r = 10 ** rng.uniform(-1, 4, n)
    t = unit(rng.normal(size=(n, 3))) * b[:, None]
    p = unit(rng.normal(size=(n, 3)) * [0.3, 0.3, 1] + [0, 0, 2]) * r[:, None]
    noise = lambda: rng.normal(size=(n, 3)) * 1e-4   # noqa: E731
    s0, s1 = 10 ** rng.uniform(-3, 3, (2, n, 1))
    v0 = (unit(p) + noise()) * s0
    v1 = (unit(p - t) + noise()) * s1
    add(v0, v1, t)
    # behind camera 0, camera 1, both; divergent (the two rays point away from each other)
    add(-v0[:40], v1[:40], t[:40])
    add(v0[40:80], -v1[40:80], t[40:80])
    add(-v0[80:120], -v1[80:120], t[80:120])
    d = unit(t[120:160])
    add(unit(p[120:160]) - 2 * d, unit(p[120:160] - t[120:160]) + 2 * d, t[120:160])
    # near-parallel: v1 = v0 turned by th about a random axis, th spanning the 1e-10 thresholds on the
    # determinants (|v|^2 th ~ 1e-10) and on geometric's denominator (|v|^4 th^2 ~ 1e-10)
    th = np.concatenate((np.logspace(-12, -3, 37), [1e-5 * (1 - 1e-3), 1e-5 * (1 + 1e-3), 1e-10 * 0.99, 1.01e-10]))
    m = len(th)
    a = unit(rng.normal(size=(m, 3)) * [1, 1, 0.1] + [0, 0, 3])
    axis = unit(np.cross(a, rng.normal(size=(m, 3))))
    w = a * np.cos(th)[:, None] + np.cross(axis, a) * np.sin(th)[:, None]
    tt = unit(rng.normal(size=(m, 3))) * 0.5
    add(a, w, tt)
    add(a * 3, w * 0.5, -tt)
    # t01 = 0, a zero v, NaN
    add(v0[:3], v1[:3], np.zeros((3, 3)))
    add(np.zeros(3), v1[3], t[3])
    add(v0[4], np.zeros(3), t[4])
    add([np.nan, 0, 1], v1[5], t[5])
    add(v0[6], v1[6], [1, np.nan, 0])
    # the error function's cheirality margins in (-3, 0): barely divergent pairs at several scales; and exactly
    # intersecting pairs, whose small-angle error falls below the 1e-21 cut
    k = 30
    dv = np.logspace(-4, 0.5, k)[:, None]
    base = unit(rng.normal(size=(k, 3)) * [0.2, 0.2, 1] + [0, 0, 3])
    tb = np.tile([[1., 0, 0]], (k, 1))
    add(base, base + dv * [1, 0, 0], tb)
    q = np.array([[0.1, 0.2, 5.], [-1, 0.5, 20], [3, -2, 40], [0, 0, 1e3]])
    tq = np.array([[1., 0, 0], [0, 1, 0], [0.5, 0.5, 0], [0.2, 0, 0]])
    add(q, q - tq, tq)
    v0, v1, t = (np.concatenate(x).astype(np.float64) for x in (v0s, v1s, ts))
    R01 = _rotations(rng, len(v0))
    return v0, v1, t, R01


def cases():
    """(key, function, (v0, v1, t01 or Rt01), get_gradients)"""
    v0, v1, t, R01 = geometries()
    Rt01 = np.concatenate((R01, t[:, None, :]), -2)
    v1_local = np.einsum("nji,nj->ni", R01, v1)            # R01' v1
    out = []
    for g in (False, True):
        for m in METHODS:
            args = (v0, v1_local, Rt01) if m == "lindstrom" else (v0, v1, t)
            out.append((f"{m}/{g}", m, args, g))
        out.append((f"_triangulated_error/{g}", "_triangulated_error", (v0, v1, t), g))
    return out


def reference(fname, args, grad):
    from oracle import triangulation_ref as T
    if fname == "_triangulated_error":
        return T.triangulated_error(*args, grad)
    return T.triangulate(fname, *args, grad)


def load():
    """[(key, fname, inputs, get_gradients, answers)], from the compiled reference where it is built, from
    tests/golden/triangulation.npz otherwise"""
    from oracle import ref
    if ref.available():
        return [(k, f, a, g, reference(f, a, g)) for k, f, a, g in cases()]
    z = np.load(GOLDEN)
    out = []
    for k, f, a, g in cases():
        n = sum(1 for key in z.files if key.startswith(k + "/out"))
        out.append((k, f, tuple(z[f"{k}/in{i}"] for i in range(len(a))), g,
                    tuple(z[f"{k}/out{i}"] for i in range(n))))
    return out


def ray_angle(fname, args):
    """the angle between the two rays, in camera 0's coordinates"""
    v0, v1, t = args
    if fname == "lindstrom":
        v1 = np.einsum("nij,nj->ni", t[:, :3, :], v1)
    c = np.cross(v0, v1)
    return np.arctan2(np.linalg.norm(c, axis=-1), np.abs(np.sum(v0 * v1, -1)))


def mid2_point_angle(args):
    """the angle between v0 and the Mid2 point (the first term of _triangulated_error), and the cheirality scale"""
    v0, v1, t = (np.asarray(a, float) for a in args)
    with np.errstate(invalid="ignore", divide="ignore"):
        c2 = _dot(np.cross(v0, v1), np.cross(v0, v1))
        l0 = np.sqrt(_dot(np.cross(v1, t), np.cross(v1, t)) / c2)
        l1 = np.sqrt(_dot(np.cross(v0, t), np.cross(v0, t)) / c2)
        m = (v0 * l0[:, None] + t + v1 * l1[:, None]) / 2
        th = np.arctan2(_norm(np.cross(v0, m)), np.abs(_dot(v0, m)))
        _, scale = _cheirality(l0, v0, l1, v1, t)
    return th, scale


def tolerance(fname, args):
    """Per element, the relative tolerance of values and gradients. The point comes from quotients by |v0 x v1|^2
    (or by determinants of the same order) whose rounding is ~eps |v0|^2 |v1|^2 th, th the angle between the rays:
    a relative error of ~eps/th^2 once the gradients' extra division is counted, in the reference as here. So
    1e-12, widened by 64 eps/th^2"""
    th = ray_angle(fname, args)
    with np.errstate(divide="ignore"):
        return 1e-12 + 64 * EPS / np.maximum(th, 1e-300) ** 2


# Multiples of eps times a quantity's scale within which rounding may decide a comparison. A quantity computed from
# the inputs directly (a determinant, a dot product, a cheirality margin) differs between the device and the reference
# by a few eps times the scale of its terms; NEAR covers that with margin. Lindstrom's determinants come from
# observations corrected through ~40 dependent operations of its niter2 step, so they take NEAR_LINDSTROM
NEAR = 64
NEAR_LINDSTROM = 4096


def _dot(a, b):
    return np.sum(a * b, -1)


def _norm(a):
    return np.linalg.norm(a, axis=-1)


def _near(q, thr, scale, mult):
    """q within mult eps scale of thr; NaN is never near"""
    with np.errstate(invalid="ignore"):
        return np.abs(q - thr) <= mult * EPS * scale


def _intersect(v0, v1, t, mult):
    """the decisions of triangulate_assume_intersect(): (failure near its threshold, branch choice near a tie)"""
    dxz = np.abs(-v0[:, 0] * v1[:, 2] + v0[:, 2] * v1[:, 0])
    dyz = np.abs(-v0[:, 1] * v1[:, 2] + v0[:, 2] * v1[:, 1])
    s = _norm(v0) * _norm(v1)
    branch = _near(dxz - dyz, 0, s, mult)
    a = np.where(dxz > dyz, 0, 1)
    rows = np.arange(len(v0))
    det = np.where(a == 0, dxz, dyz)
    k0num = t[:, 2] * v1[rows, a] - t[rows, a] * v1[:, 2]
    k1num = t[:, 2] * v0[rows, a] - t[rows, a] * v0[:, 2]
    fail = _near(det, 1e-10, s, mult) | _near(det, 0, s, mult) | \
        _near(k0num, 0, _norm(t) * _norm(v1), mult) | _near(k1num, 0, _norm(t) * _norm(v0), mult)
    return fail, branch


def _reject(v, n):
    return v - n * (_dot(v, n) / _dot(n, n))[:, None]


def _cheirality(l0, v0, l1, v1, t):
    """the cheirality margins w0, w1, w01 and their scale"""
    far, near = l1[:, None] * v1, l0[:, None] * v0
    xn = far + t - near
    w = [_dot(x, x) - _dot(xn, xn) for x in (far + t + near, t - far - near, t - far + near)]
    return w, (_norm(far) + _norm(t) + _norm(near)) ** 2


def _unit(v):
    with np.errstate(invalid="ignore", divide="ignore"):
        return v / _norm(v)[:, None]


def decisions(fname, args):
    """Per element, whether rounding may decide (failure, branch): failure, where a quantity the method compares with
    a failure threshold lies within NEAR eps (times the scale of its terms) of it; branch, where a quantity that picks
    one of two ways of computing the point lies as near a tie. Each quantity is computed in numpy from the inputs, as
    the method computes it"""
    with np.errstate(invalid="ignore", divide="ignore"):
        v0, v1, t = (np.asarray(a, float) for a in args)
        n = len(v0)
        none = np.zeros(n, bool)
        if fname == "geometric":
            d00, d11, d01, d0t, d1t = _dot(v0, v0), _dot(v1, v1), _dot(v0, v1), _dot(v0, t), _dot(v1, t)
            denom = d00 * d11 - d01 * d01
            s = d00 * d11
            s_k = d11 * np.sqrt(d00 * _dot(t, t)) + np.sqrt(d00 * d11) * np.sqrt(d11 * _dot(t, t))
            fail = _near(np.abs(denom), 1e-10, s, NEAR) | _near(d11 * d0t - d01 * d1t, 0, s_k, NEAR) | \
                _near(d01 * d0t - d00 * d1t, 0, s_k, NEAR)
            return fail, none
        if fname == "leecivera_l1":
            d00, d11, d0t, d1t = _dot(v0, v0), _dot(v1, v1), _dot(v0, t), _dot(v1, t)
            branch = _near(d0t * d0t * d11 - d1t * d1t * d00, 0, d00 * d11 * _dot(t, t), NEAR)
            first = d0t * d0t * d11 > d1t * d1t * d00
            w0 = np.where(first[:, None], _reject(v0, np.cross(v1, t)), v0)
            w1 = np.where(first[:, None], v1, _reject(v1, np.cross(v0, t)))
            fail, b = _intersect(w0, w1, t, NEAR)
            return fail, branch | b
        if fname == "leecivera_linf":
            u0, u1 = _unit(v0), _unit(v1)
            na, nb = np.cross(u0 + u1, t), np.cross(u0 - u1, t)
            branch = _near(_dot(na, na) - _dot(nb, nb), 0, 4 * _dot(t, t), NEAR)
            nn = np.where((_dot(na, na) > _dot(nb, nb))[:, None], na, nb)
            fail, b = _intersect(_reject(u0, nn), _reject(u1, nn), t, NEAR)
            return fail, branch | b
        if fname in ("leecivera_mid2", "leecivera_wmid2", "_triangulated_error"):
            if fname == "leecivera_wmid2":
                v0, v1 = _unit(v0), _unit(v1)
                c = _norm(np.cross(v0, v1))
                l0, l1 = _norm(np.cross(v1, t)) / c, _norm(np.cross(v0, t)) / c
            else:
                c2 = _dot(np.cross(v0, v1), np.cross(v0, v1))
                l0 = np.sqrt(_dot(np.cross(v1, t), np.cross(v1, t)) / c2)
                l1 = np.sqrt(_dot(np.cross(v0, t), np.cross(v0, t)) / c2)
            w, s = _cheirality(l0, v0, l1, v1, t)
            fail = _near(w[0], 0, s, NEAR) | _near(w[1], 0, s, NEAR) | _near(w[2], 0, s, NEAR)
            return fail, none
        # lindstrom: v0, v1 local; t is Rt01
        R, tt = t[:, :3, :], t[:, 3, :]
        E = np.stack((R[:, 2] * tt[:, 1:2] - R[:, 1] * tt[:, 2:3], R[:, 0] * tt[:, 2:3] - R[:, 2] * tt[:, 0:1],
                      R[:, 1] * tt[:, 0:1] - R[:, 0] * tt[:, 1:2]), 1)             # E = skew(t01) R01
        x0 = v0[:, :2] / v0[:, 2:3]
        x1 = v1[:, :2] / v1[:, 2:3]
        x0h = np.concatenate((x0, np.ones((n, 1))), -1)
        x1h = np.concatenate((x1, np.ones((n, 1))), -1)
        nv = np.einsum("nij,nj->ni", E, x1h)[:, :2]
        nnv = np.einsum("nji,nj->ni", E, x0h)[:, :2]
        E2 = E[:, :2, :2]
        a = np.einsum("ni,nij,nj->n", nv, E2, nnv)
        b = 0.5 * (_dot(nv, nv) + _dot(nnv, nnv))
        cc = np.einsum("ni,nij,nj->n", x0h, E, x1h)
        d = np.sqrt(b * b - a * cc)
        lam = cc / (b + d)
        dx, dxx = lam[:, None] * nv, lam[:, None] * nnv
        nv = nv - np.einsum("nij,nj->ni", E2, dxx)
        nnv = nnv - np.einsum("nji,nj->ni", E2, dx)
        lam = lam / d * 0.5 * (_dot(nv, nv) + _dot(nnv, nnv))
        p0 = np.concatenate((x0 - lam[:, None] * nv, np.ones((n, 1))), -1)
        p1 = np.concatenate((x1 - lam[:, None] * nnv, np.ones((n, 1))), -1)
        return _intersect(p0, np.einsum("nij,nj->ni", R, p1), tt, NEAR_LINDSTROM)
