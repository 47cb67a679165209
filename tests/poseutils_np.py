"""The answers the pose-utility tests compare against, and the cases they are asked for.

Where the compiled reference (oracle/_ref) has the function, the answer is the reference's own mrcal_*_full()
(oracle/poseutils_ref.py). The rest of mrcal/poseutils.py is numpy code in the reference; it is restated here:
skew_symmetric(), R_from_quat() and quat_from_R() (mrcal/_poseutils_scipy.py, scipy's algorithm in the reference's
(w,x,y,z) order), qt_from_Rt(), Rt_from_qt(), and the two tiny-rt gradients built from the reference's functions as
mrcal/poseutils.py builds them. Without oracle/_ref, the answers stored in tests/golden/poseutils.npz
(tests/golden/make_poseutils_golden.py) are used."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "poseutils.npz")
EPS = np.finfo(float).eps


def skew_symmetric(a):
    a = np.asarray(a, float)
    z = np.zeros(a.shape[:-1])
    return np.stack((np.stack((z, -a[..., 2], a[..., 1]), -1), np.stack((a[..., 2], z, -a[..., 0]), -1),
                     np.stack((-a[..., 1], a[..., 0], z), -1)), -2)


def R_from_quat(q):
    w, i, j, k = (q[..., n] for n in range(4))
    return np.stack((np.stack((1 - 2 * (j * j + k * k), 2 * (i * j - k * w), 2 * (i * k + j * w)), -1),
                     np.stack((2 * (i * j + k * w), 1 - 2 * (i * i + k * k), 2 * (j * k - i * w)), -1),
                     np.stack((2 * (i * k - j * w), 2 * (j * k + i * w), 1 - 2 * (i * i + j * j)), -1)), -2)


def quat_from_R(R):
    """scipy's Rotation.from_matrix() algorithm, as mrcal/_poseutils_scipy.py states it: the largest of the diagonal
    and the trace picks the formula (the first on a tie); (w,x,y,z); the sign is not normalized"""
    R = np.asarray(R, float)
    lead = R.shape[:-2]
    R = R.reshape(-1, 3, 3)
    q = np.empty((len(R), 4))
    for n, M in enumerate(R):
        d = np.array([M[0, 0], M[1, 1], M[2, 2], np.trace(M)])
        c = int(np.argmax(d))
        if c != 3:
            i, j, k = c, (c + 1) % 3, (c + 2) % 3
            q[n, i + 1] = 1 - d[3] + 2 * M[i, i]
            q[n, j + 1] = M[j, i] + M[i, j]
            q[n, k + 1] = M[k, i] + M[i, k]
            q[n, 0] = M[k, j] - M[j, k]
        else:
            q[n] = (1 + d[3], M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1])
        q[n] /= np.linalg.norm(q[n])
    return q.reshape(lead + (4,))


def unit(v):
    v = np.asarray(v, float)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _r_set(rng):
    """rotation vectors at every branch of the reference: exactly 0, tiny, both sides of rodrigues()'s series switch
    at 0.1, near, at and beyond a half-turn, and random ones"""
    axes = unit(rng.normal(size=(14, 3)))
    mags = np.array([0., 1e-20, 1e-12, 1e-6, 1e-3, 0.1 - 1e-9, 0.1 + 1e-9, 0.5, 2., np.pi - 1e-6, np.pi,
                     np.pi + 0.3, 4., 5.5])
    r = axes * mags[:, None]
    return np.concatenate((r, rng.normal(size=(8, 3))))


def cases(ref_available=True):
    """(key, function name, inputs, keyword arguments, tags): every function of the reference with and without
    gradients and with every inverted* combination. Tags: "halfturn" where the reference's answer loses digits near
    a half-turn, "small" where its closed-form R_from_r gradient loses digits to cancellation"""
    rng = np.random.default_rng(0)
    r = _r_set(rng)
    t = rng.normal(size=(len(r), 3)) * 3
    rt = np.concatenate((r, t), -1)
    R = np.array([np.eye(3)] * len(r))
    out = []
    add = lambda *c: out.append(c)   # noqa: E731

    # rotation matrices: of the r set, exact half-turns, and traces within 1e-12 of -1
    a = unit(rng.normal(size=(3, 3)))
    R_half = 2 * a[:, :, None] * a[:, None, :] - np.eye(3)
    from oracle import poseutils_ref as P
    if ref_available:
        R = P.R_from_r(r, False)[0]
    Rs = np.concatenate((R, R_half))
    Rts = np.concatenate((Rs, rng.normal(size=(len(Rs), 1, 3))), -2)
    x = rng.normal(size=(len(r), 3)) * 5
    mag = np.linalg.norm(r, axis=-1)
    small = dict(small=mag)
    for g in (False, True):
        add(f"R_from_r/{g}", "R_from_r", (r,), dict(get_gradients=g), small)
        add(f"Rt_from_rt/{g}", "Rt_from_rt", (rt,), dict(get_gradients=g), small)
        add(f"r_from_R/{g}", "r_from_R", (Rs,), dict(get_gradients=g), dict(halfturn=True))
        add(f"rt_from_Rt/{g}", "rt_from_Rt", (Rts,), dict(get_gradients=g), dict(halfturn=True))
        add(f"invert_rt/{g}", "invert_rt", (rt,), dict(get_gradients=g), {})
    add("invert_R", "invert_R", (Rs,), {}, {})
    add("invert_Rt", "invert_Rt", (Rts,), {}, {})

    # composition pairs: random, r and -r, either operand zero, tiny ones, and pairs whose composition lies near,
    # at and beyond a half-turn
    ax = unit(rng.normal(size=(4, 3)))
    r0 = np.concatenate((r, r, np.zeros((3, 3)), r[8:11], [[1e-10, 0, 0]],
                         ax * (np.pi / 2 + 0.3)))
    r1 = np.concatenate((r[::-1], -r, r[8:11], np.zeros((3, 3)), [[0, 2e-10, 0]],
                         ax * (np.pi / 2 - 0.3 + np.array([-1e-3, 0., 1e-7, 1e-3]))[:, None]))
    t0 = rng.normal(size=(len(r0), 3))
    t1 = rng.normal(size=(len(r0), 3))
    Rt0 = np.concatenate((np.concatenate((R, R_half))[:len(r0) % 20 + 3], rng.normal(size=(len(r0) % 20 + 3, 1, 3))),
                         -2)
    for i0 in (False, True):
        for i1 in (False, True):
            kw = dict(inverted0=i0, inverted1=i1)
            for g in (False, True):
                add(f"compose_r/{g}/{i0}/{i1}", "compose_r", (r0, r1), dict(get_gradients=g, **kw),
                    dict(halfturn=True))
                add(f"compose_rt/{g}/{i0}/{i1}", "compose_rt",
                    (np.concatenate((r0, t0), -1), np.concatenate((r1, t1), -1)), dict(get_gradients=g, **kw),
                    dict(halfturn=True))
            add(f"compose_Rt/{i0}/{i1}", "compose_Rt", (Rt0, Rt0[::-1]), kw, {})
    for name, arg in (("compose_r_tinyr0_gradientr0", r), ("compose_r_tinyr1_gradientr1", r),
                      ("compose_rt_tinyrt0_gradientrt0", rt), ("compose_rt_tinyrt1_gradientrt1", rt)):
        add(name, name, (arg,), {}, {})

    for inv in (False, True):
        for g in (False, True):
            kw = dict(get_gradients=g, inverted=inv)
            add(f"rotate_point_r/{g}/{inv}", "rotate_point_r", (r, x), kw, {})
            add(f"rotate_point_R/{g}/{inv}", "rotate_point_R", (R, x), kw, {})
            add(f"transform_point_rt/{g}/{inv}", "transform_point_rt", (rt, x), kw, {})
            add(f"transform_point_Rt/{g}/{inv}", "transform_point_Rt", (Rts[:len(x)], x), kw, {})

    q = unit(rng.normal(size=(10, 4)))
    add("skew_symmetric", "skew_symmetric", (x,), {}, {})
    add("R_from_quat", "R_from_quat", (q,), {}, {})
    add("quat_from_R", "quat_from_R", (Rs,), {}, {})
    add("qt_from_Rt", "qt_from_Rt", (Rts,), {}, {})
    add("Rt_from_qt", "Rt_from_qt", (np.concatenate((q, rng.normal(size=(10, 3))), -1),), {}, {})
    v = np.concatenate((x, [[1., 0, 0], [0.95, 0.1, 0], [0, 0, -2]]))
    add("R_aligned_to_vector", "R_aligned_to_vector", (v,), {}, {})
    return out


def reference(fname, args, kw):
    """The reference's answer: a tuple of arrays, in mrcal/poseutils.py's order and layouts"""
    from oracle import poseutils_ref as P
    g = kw.get("get_gradients", False)
    inv = {k: v for k, v in kw.items() if k.startswith("inverted")}
    if fname in ("R_from_r", "r_from_R", "Rt_from_rt", "rt_from_Rt", "invert_rt"):
        return getattr(P, fname)(*args, g)
    if fname in ("compose_r", "compose_rt", "rotate_point_r", "rotate_point_R", "transform_point_rt",
                 "transform_point_Rt"):
        return getattr(P, fname)(*args, g, **inv)
    if fname == "compose_rt_tinyrt0_gradientrt0":
        # [dr/dr0 0; -skew(t1) I] (mrcal/poseutils.py)
        rt1 = args[0]
        out = np.zeros(rt1.shape + (6,))
        out[..., :3, :3] = P.compose_r_tinyr0_gradientr0(rt1[..., :3])[0]
        out[..., 3:, :3] = -skew_symmetric(rt1[..., 3:])
        out[..., 3:, 3:] = np.eye(3)
        return (out,)
    if fname == "compose_rt_tinyrt1_gradientrt1":
        # drt01/drt1 of compose_rt(rt0, 0) (mrcal/poseutils.py)
        return (P.compose_rt(args[0], np.zeros_like(args[0]), True)[2],)
    if fname == "skew_symmetric":
        return (skew_symmetric(args[0]),)
    if fname == "R_from_quat":
        return (R_from_quat(args[0]),)
    if fname == "quat_from_R":
        return (quat_from_R(args[0]),)
    if fname == "qt_from_Rt":
        return (np.concatenate((quat_from_R(args[0][..., :3, :]), args[0][..., 3, :]), -1),)
    if fname == "Rt_from_qt":
        return (np.concatenate((R_from_quat(args[0][..., :4]), args[0][..., None, 4:]), -2),)
    return getattr(P, fname)(*args, **inv)


ROTATION_VECTOR_RESULT = ("r_from_R", "rt_from_Rt", "compose_r", "compose_rt")


def check_value(key, fname, got, want, R_from_r):
    """Asserts that got, the value output of fname, matches want, the reference's, to 1e-12 of the largest |want|.
    Returns the mask of the elements compared element by element, which is where gradients can be compared too"""
    assert got.shape == want.shape, key
    ok = np.ones(want.shape[:1], bool)
    if fname in ROTATION_VECTOR_RESULT:
        # Within ~1e-3 of a half-turn the reference takes the angle from acos() of a cosine near -1, or from
        # sqrt((1 + R_ii)/2): it loses up to half its digits there, and r and the equivalent rotation of angle
        # |r| - 2 pi are both valid answers. There the results are compared as rotations, to the ~1e-8 that
        # conditioning allows, and the gradients of the rotation part (ill-conditioned) are not compared
        r_ref = want[..., :3]
        near = np.abs(np.linalg.norm(r_ref, axis=-1) - np.pi) < 1e-3
        if near.any():
            Rg = R_from_r(got[near][..., :3])
            Rw = R_from_r(r_ref[near])
            assert np.abs(Rg - Rw).max() < 1e-8, key
            t_err = np.abs(got[near][..., 3:] - want[near][..., 3:])
            assert t_err.size == 0 or t_err.max() <= 1e-8 * (1 + np.abs(want).max()), key
        ok = ~near
    g, w = got[ok], want[ok]
    err = np.abs(g - w).reshape(len(g), -1).max(-1)
    tol = 1e-12 * max(1., np.abs(w).max())
    bad = np.nonzero(err > tol)[0]
    assert len(bad) == 0, f"{key} output 0: element {bad[:3]} error {err[bad[:3]]} > {tol}"
    return ok


def load():
    """[(key, fname, inputs, kwargs, tags, answers)]: the answers from the compiled reference where it is built, from
    tests/golden/poseutils.npz otherwise"""
    from oracle import ref
    if ref.available():
        return [(k, f, a, kw, tags, reference(f, a, kw)) for k, f, a, kw, tags in cases()]
    z = np.load(GOLDEN)
    out = []
    for k, f, a, kw, tags in cases(ref_available=False):
        n = sum(1 for key in z.files if key.startswith(k + "/out"))
        a = tuple(z[f"{k}/in{i}"] for i in range(len(a)))
        out.append((k, f, a, kw, tags, tuple(z[f"{k}/out{i}"] for i in range(n))))
    return out
