"""TEST INFRASTRUCTURE ONLY -- the reference's own triangulation routines (triangulation.cc, compiled into
oracle/_ref/libmrcal_ref.so by oracle/Makefile): mrcal_triangulate_*() and _mrcal_triangulated_error(), called one
element at a time through ctypes, with the output layouts of triangulation-genpywrap.py. The gradient outputs are
zero-initialized: the reference leaves them unwritten where a method fails."""
import ctypes as C

import numpy as np

from . import ref


class _Point3(C.Structure):
    _fields_ = [("xyz", C.c_double * 3)]


METHODS = ("geometric", "leecivera_l1", "leecivera_linf", "leecivera_mid2", "leecivera_wmid2", "lindstrom")


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _fn(name, restype):
    f = getattr(ref.lib(), name)
    f.restype = restype
    f.argtypes = [C.c_void_p] * (5 if restype is C.c_double else 6)
    return f


def triangulate(method, v0, v1, t, grad):
    """method's point p for each element of the (already broadcast, equal-length) v0 (N,3), v1 (N,3) and t01 (N,3)
    (or Rt01 (N,4,3) for lindstrom); with grad: (p, dp/dv0 (N,3,3), dp/dv1 (N,3,3), dp/dt01 (N,3,3) or dp/dRt01
    (N,3,4,3))"""
    f = _fn(f"mrcal_triangulate_{method}", _Point3)
    v0, v1, t = (np.ascontiguousarray(x, dtype=np.float64) for x in (v0, v1, t))
    n = len(v0)
    wt = 12 if method == "lindstrom" else 3
    p = np.zeros((n, 3))
    g = [np.zeros((n, 3, 3)), np.zeros((n, 3, 3)), np.zeros((n, 3, wt))]
    for i in range(n):
        r = f(*((_p(x[i]) for x in g) if grad else (None,) * 3), _p(v0[i]), _p(v1[i]), _p(t[i]))
        p[i] = r.xyz
    if not grad:
        return (p,)
    if method == "lindstrom":
        g[2] = g[2].reshape(n, 3, 4, 3)
    return (p, *g)


def triangulated_error(v0, v1, t01, grad):
    """_mrcal_triangulated_error() for each element: err (N,), and with grad derr/dv1 (N,3), derr/dt01 (N,3)"""
    f = _fn("_mrcal_triangulated_error", C.c_double)
    v0, v1, t01 = (np.ascontiguousarray(x, dtype=np.float64) for x in (v0, v1, t01))
    n = len(v0)
    err, dv1, dt01 = np.zeros(n), np.zeros((n, 3)), np.zeros((n, 3))
    for i in range(n):
        err[i] = f(_p(dv1[i]) if grad else None, _p(dt01[i]) if grad else None, _p(v0[i]), _p(v1[i]), _p(t01[i]))
    return (err, dv1, dt01) if grad else (err,)
