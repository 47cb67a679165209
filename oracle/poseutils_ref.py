"""TEST INFRASTRUCTURE ONLY -- the reference's own pose utilities (poseutils.c, poseutils-opencv.c,
poseutils-uses-autodiff.cc, compiled into oracle/_ref/libmrcal_ref.so by oracle/Makefile), called through their
mrcal_*_full() C entry points one element at a time, with the output layouts of mrcal/poseutils.py and
poseutils-genpywrap.py. Every stride is passed as 0: contiguous."""
import ctypes as C

import numpy as np

from . import ref


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _each(f, n_out, *xs):
    """f applied to each element of the leading dimension of xs (already broadcast), outputs stacked"""
    xs = [np.ascontiguousarray(x, dtype=np.float64) for x in xs]
    res = [f(*(x[i] for x in xs)) for i in range(xs[0].shape[0])]
    return tuple(np.array([r[k] for r in res]) for k in range(n_out))


def R_from_r(r, grad):
    def f(r):
        R, J = np.zeros((3, 3)), np.zeros((3, 3, 3)) if grad else None
        ref.lib().mrcal_R_from_r_full(_p(R), 0, 0, _p(J), 0, 0, 0, _p(r), 0)
        return (R, J) if grad else (R,)
    return _each(f, 1 + grad, r)


def r_from_R(R, grad):
    def f(R):
        r, J = np.zeros(3), np.zeros((3, 3, 3)) if grad else None
        ref.lib().mrcal_r_from_R_full(_p(r), 0, _p(J), 0, 0, 0, _p(R), 0, 0)
        return (r, J) if grad else (r,)
    return _each(f, 1 + grad, R)


def Rt_from_rt(rt, grad):
    def f(rt):
        Rt, J = np.zeros((4, 3)), np.zeros((3, 3, 3)) if grad else None
        ref.lib().mrcal_Rt_from_rt_full(_p(Rt), 0, 0, _p(J), 0, 0, 0, _p(rt), 0)
        return (Rt, J) if grad else (Rt,)
    return _each(f, 1 + grad, rt)


def rt_from_Rt(Rt, grad):
    def f(Rt):
        rt, J = np.zeros(6), np.zeros((3, 3, 3)) if grad else None
        ref.lib().mrcal_rt_from_Rt_full(_p(rt), 0, _p(J), 0, 0, 0, _p(Rt), 0, 0)
        return (rt, J) if grad else (rt,)
    return _each(f, 1 + grad, Rt)


def invert_R(R):
    def f(R):
        out = np.zeros((3, 3))
        ref.lib().mrcal_invert_R_full(_p(out), 0, 0, _p(R), 0, 0)
        return (out,)
    return _each(f, 1, R)


def invert_Rt(Rt):
    def f(Rt):
        out = np.zeros((4, 3))
        ref.lib().mrcal_invert_Rt_full(_p(out), 0, 0, _p(Rt), 0, 0)
        return (out,)
    return _each(f, 1, Rt)


def invert_rt(rt, grad):
    def f(rt):
        out, dr, dt = np.zeros(6), np.zeros((3, 3)), np.zeros((3, 3))
        ref.lib().mrcal_invert_rt_full(_p(out), 0, _p(dr) if grad else None, 0, 0, _p(dt) if grad else None, 0, 0,
                                       _p(rt), 0)
        if not grad:
            return (out,)
        # [ -I 0 ; dtout/drin dtout/dtin ] (_invert_rt_withgrad, poseutils-genpywrap.py)
        return out, np.block([[-np.eye(3), np.zeros((3, 3))], [dr, dt]])
    return _each(f, 1 + grad, rt)


def compose_Rt(Rt0, Rt1, inverted0=False, inverted1=False):
    def f(a, b):
        out = np.zeros((4, 3))
        ref.lib().mrcal_compose_Rt_full(_p(out), 0, 0, _p(a), 0, 0, _p(b), 0, 0, C.c_bool(inverted0),
                                        C.c_bool(inverted1))
        return (out,)
    return _each(f, 1, Rt0, Rt1)


def compose_r(r0, r1, grad, inverted0=False, inverted1=False):
    def f(a, b):
        out, d0, d1 = np.zeros(3), np.zeros((3, 3)), np.zeros((3, 3))
        ref.lib().mrcal_compose_r_full(_p(out), 0, _p(d0) if grad else None, 0, 0, _p(d1) if grad else None, 0, 0,
                                       _p(a), 0, _p(b), 0, C.c_bool(inverted0), C.c_bool(inverted1))
        return (out, d0, d1) if grad else (out,)
    return _each(f, 1 + 2 * grad, r0, r1)


def compose_rt(rt0, rt1, grad, inverted0=False, inverted1=False):
    def f(a, b):
        out = np.zeros(6)
        g = [np.zeros((3, 3)) for _ in range(6)]   # dr/dr0 dr/dr1 dt/dr0 dt/dr1 dt/dt0 dt/dt1
        args = []
        for m in g:
            args += [_p(m) if grad else None, 0, 0]
        ref.lib().mrcal_compose_rt_full(_p(out), 0, *args, _p(a), 0, _p(b), 0, C.c_bool(inverted0),
                                        C.c_bool(inverted1))
        if not grad:
            return (out,)
        z = np.zeros((3, 3))
        # [ dr/dr0 0 ; dt/dr0 dt/dt0 ], [ dr/dr1 0 ; dt/dr1 dt/dt1 ] (_compose_rt_withgrad, poseutils-genpywrap.py)
        return out, np.block([[g[0], z], [g[2], g[4]]]), np.block([[g[1], z], [g[3], g[5]]])
    return _each(f, 1 + 2 * grad, rt0, rt1)


def compose_r_tinyr0_gradientr0(r1):
    def f(r):
        out = np.zeros((3, 3))
        ref.lib().mrcal_compose_r_tinyr0_gradientr0_full(_p(out), 0, 0, _p(r), 0)
        return (out,)
    return _each(f, 1, r1)


def compose_r_tinyr1_gradientr1(r0):
    def f(r):
        out = np.zeros((3, 3))
        ref.lib().mrcal_compose_r_tinyr1_gradientr1_full(_p(out), 0, 0, _p(r), 0)
        return (out,)
    return _each(f, 1, r0)


def _point(fn, gshape, pose, x, grad, inverted):
    def f(p, x):
        out, Jp, Jx = np.zeros(3), np.zeros(gshape), np.zeros((3, 3))
        gstrides = (0,) * len(gshape)
        pstrides = (0,) * (p.ndim)
        fn(_p(out), 0, _p(Jp) if grad else None, *gstrides, _p(Jx) if grad else None, 0, 0, _p(p), *pstrides,
           _p(x), 0, C.c_bool(inverted))
        return (out, Jp, Jx) if grad else (out,)
    return _each(f, 1 + 2 * grad, pose, x)


def rotate_point_r(r, x, grad, inverted=False):
    return _point(ref.lib().mrcal_rotate_point_r_full, (3, 3), r, x, grad, inverted)


def rotate_point_R(R, x, grad, inverted=False):
    return _point(ref.lib().mrcal_rotate_point_R_full, (3, 3, 3), R, x, grad, inverted)


def transform_point_rt(rt, x, grad, inverted=False):
    return _point(ref.lib().mrcal_transform_point_rt_full, (3, 6), rt, x, grad, inverted)


def transform_point_Rt(Rt, x, grad, inverted=False):
    return _point(ref.lib().mrcal_transform_point_Rt_full, (3, 4, 3), Rt, x, grad, inverted)


def R_aligned_to_vector(v):
    def f(v):
        out = np.zeros((3, 3))
        ref.lib().mrcal_R_aligned_to_vector(_p(out), _p(v))
        return (out,)
    return _each(f, 1, v)
