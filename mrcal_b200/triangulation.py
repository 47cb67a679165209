"""The two-view triangulation routines, with the reference's names, keyword arguments, refusals, broadcasting and
output layouts (mrcal/triangulation.py and the generated mrcal._triangulation_npsp).

Each turns a pair of observation rays into a point in camera 0's coordinates: v0 from camera 0, v1 from camera 1,
not necessarily normalized, and camera 1's origin t01 (or the whole transformation Rt01, camera 1 to camera 0).
Where the rays are parallel or divergent, or the point lies behind a camera, the point is (0,0,0), and its gradients
are zeros. Every function runs on the device (csrc/triangulation.cu), one thread per element of the broadcast shape,
through the call frame of the pose utilities: inputs are either all numpy arrays, converted to float64, or all torch
CUDA float64 tensors on one device, enqueued on torch.cuda.current_stream() without waiting. An operand that is
broadcast is read in place, never expanded. out= writes the results into the given array(s) and returns them."""
import numpy as np

from .poseutils import _pose, rotate_point_R

# method codes of include/mrcal_b200.h (MRCAL_B200_TRIANGULATE_*), in order
_METHODS = {name: i for i, name in enumerate((
    "geometric", "leecivera_l1", "leecivera_linf", "leecivera_mid2", "leecivera_wmid2", "lindstrom",
    "_triangulated_error"))}


def _array(x):
    """x, indexable as an array: lists become float64 arrays, arrays and tensors stay as they are"""
    return np.asarray(x, np.float64) if isinstance(x, (list, tuple)) else x


def _parse_args(v1, t01, get_gradients, v_are_local, Rt01):
    """v1 in camera 0's coordinates and t01, from the arguments of the methods that take t01 (the reference's
    _parse_args())"""
    Rt01 = _array(Rt01)
    if Rt01 is not None and t01 is not None:
        raise Exception("Exactly one of Rt01 and t01 must be None. Both were non-None")
    if Rt01 is None and t01 is None:
        raise Exception("Exactly one of Rt01 and t01 must be None. Both were None")
    if v_are_local:
        if get_gradients:
            raise Exception("get_gradients is True, so v_are_local MUST be the default: False")
        if Rt01 is None:
            raise Exception("v_are_local is True, so Rt01 MUST have been given")
        return rotate_point_R(Rt01[..., :3, :], v1), Rt01[..., 3, :]
    if t01 is None:
        if get_gradients:
            raise Exception("get_gradients is True, so t01 MUST have been given")
        return v1, Rt01[..., 3, :]
    return v1, t01


def _call(method, v0, v1, t, proto_t, protos_out, get_gradients, out):
    fname = method if method.startswith("_") else f"triangulate_{method}"
    return _pose(fname, (v0, v1, t), ((3,), (3,), proto_t), protos_out, out, get_gradients,
                 entry="triangulate", op=_METHODS[method])


def _method(method, v0, v1, t01, get_gradients, v_are_local, Rt01, out):
    v1, t01 = _parse_args(v1, t01, get_gradients, v_are_local, Rt01)
    protos_out = ((3,),) + (((3, 3),) * 3 if get_gradients else ())
    return _call(method, v0, v1, t01, (3,), protos_out, get_gradients, out)


def triangulate_geometric(v0, v1, t01=None, *, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """The midpoint of the closest approach of the two rays ("Mid" in Lee and Civera, "Triangulation: Why
    Optimize?"). With get_gradients: (p, dp/dv0 (3,3), dp/dv1 (3,3), dp/dt01 (3,3))"""
    return _method("geometric", v0, v1, t01, get_gradients, v_are_local, Rt01, out)


def triangulate_leecivera_l1(v0, v1, t01=None, *, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """The point minimizing the L1 norm of the angular errors (Lee and Civera, ICCV 2019). With get_gradients:
    (p, dp/dv0 (3,3), dp/dv1 (3,3), dp/dt01 (3,3))"""
    return _method("leecivera_l1", v0, v1, t01, get_gradients, v_are_local, Rt01, out)


def triangulate_leecivera_linf(v0, v1, t01=None, *, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """The point minimizing the L-infinity norm of the angular errors (Lee and Civera, ICCV 2019). With
    get_gradients: (p, dp/dv0 (3,3), dp/dv1 (3,3), dp/dt01 (3,3))"""
    return _method("leecivera_linf", v0, v1, t01, get_gradients, v_are_local, Rt01, out)


def triangulate_leecivera_mid2(v0, v1, t01=None, *, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """Lee and Civera's "Mid2" ("Triangulation: Why Optimize?"). With get_gradients: (p, dp/dv0 (3,3),
    dp/dv1 (3,3), dp/dt01 (3,3))"""
    return _method("leecivera_mid2", v0, v1, t01, get_gradients, v_are_local, Rt01, out)


def triangulate_leecivera_wmid2(v0, v1, t01=None, *, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """Lee and Civera's "wMid2", Mid2 weighted by the inverse ranges ("Triangulation: Why Optimize?"). With
    get_gradients: (p, dp/dv0 (3,3), dp/dv1 (3,3), dp/dt01 (3,3))"""
    return _method("leecivera_wmid2", v0, v1, t01, get_gradients, v_are_local, Rt01, out)


def triangulate_lindstrom(v0, v1, Rt01, *, get_gradients=False, v_are_local=True, out=None):
    """The point minimizing the L2 pinhole reprojection error (Lindstrom, "Triangulation Made Easy", CVPR 2010).
    Unlike the other methods, v0 and v1 are each in their own camera's coordinates by default; with
    v_are_local=False v1 is in camera 0's. With get_gradients (v_are_local only): (p, dp/dv0 (3,3), dp/dv1 (3,3),
    dp/dRt01 (3,4,3))"""
    if not v_are_local:
        if get_gradients:
            raise Exception("get_gradients is True, so v_are_local MUST be True")
        Rt01 = _array(Rt01)
        v1 = rotate_point_R(Rt01[..., :3, :], v1, inverted=True)
    protos_out = ((3,),) + (((3, 3), (3, 3), (3, 4, 3)) if get_gradients else ())
    return _call("lindstrom", v0, v1, Rt01, (4, 3), protos_out, get_gradients, out)


def _triangulated_error(v0, v1, t01=None, get_gradients=False, v_are_local=False, Rt01=None, out=None):
    """The solver's measurement of a triangulated point: twice the small-angle error between v0 and the Mid2 point,
    plus a penalty for pairs that fail the cheirality test (the solver's own per-pair function). With get_gradients:
    (err, derr/dv1 (3,), derr/dt01 (3,)); there is no gradient in v0"""
    v1, t01 = _parse_args(v1, t01, get_gradients, v_are_local, Rt01)
    protos_out = ((),) + (((3,), (3,)) if get_gradients else ())
    return _call("_triangulated_error", v0, v1, t01, (3,), protos_out, get_gradients, out)
