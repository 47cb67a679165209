"""The pose utilities, with the reference's names, keyword arguments, broadcasting, output layouts and gradient
conventions (mrcal/poseutils.py and the generated mrcal._poseutils_npsp):

    rotations:       R (3,3), r (3,): a Rodrigues vector
    transformations: Rt (4,3): R then t; rt (6,): r then t; qt (7,): a unit quaternion (w,x,y,z) then t
    x_out = R x + t

Every function runs on the device: one element-wise kernel per call (csrc/poseutils.cu), one thread per element of
the broadcast shape. Inputs are either all numpy arrays (or lists), converted to float64, or all torch CUDA float64
tensors on one device: the results are then tensors on that device, and the kernel is enqueued on
torch.cuda.current_stream() without waiting for it. Leading dimensions broadcast as in numpy. An operand that is
broadcast is read in place, never expanded. out= writes the results into the given array(s) (a tuple with gradients)
and returns them. identity_*() are host-only.
"""
import ctypes as C
from functools import reduce

import numpy as np

from ._capi import checked
from .api import _ptr, _require_gpu
from .image_transforms import _torch_if_tensors

# operation codes of include/mrcal_b200.h (MRCAL_B200_POSE_*), in order
_OPS = {name: i for i, name in enumerate((
    "R_from_r", "r_from_R", "Rt_from_rt", "rt_from_Rt", "invert_R", "invert_Rt", "invert_rt", "compose_Rt",
    "compose_r", "compose_rt", "compose_r_tinyr0_gradientr0", "compose_r_tinyr1_gradientr1",
    "compose_rt_tinyrt0_gradientrt0", "compose_rt_tinyrt1_gradientrt1", "rotate_point_r", "rotate_point_R",
    "transform_point_rt", "transform_point_Rt", "skew_symmetric", "R_from_quat", "quat_from_R", "qt_from_Rt",
    "Rt_from_qt", "R_aligned_to_vector"))}
_GET_GRADIENTS, _INVERTED0, _INVERTED1 = 1, 2, 4
_MAX_DIMS = 8


def _operand(x, proto, name, fname, torch, device):
    """x as the kernel reads it: float64, its prototype dimensions packed, every stride non-negative"""
    n = len(proto)
    if torch is None:
        x = np.asarray(x, dtype=np.float64)
        shape = x.shape
    else:
        if not x.is_cuda or x.dtype != torch.float64:
            raise ValueError(f"{fname}(): torch tensors must be CUDA float64 tensors; {name} is {x.dtype} on "
                             f"{x.device}")
        if x.device != device:
            raise ValueError(f"{fname}(): all tensors must be on one device; {name} is on {x.device}, not {device}")
        shape = tuple(x.shape)
    if len(shape) < n or tuple(shape[len(shape) - n:]) != tuple(proto):
        raise ValueError(f"{fname}(): {name} must have shape (...,{','.join(map(str, proto))}); got {shape}")
    packed = tuple(int(np.prod(proto[k + 1:])) for k in range(n))
    if torch is None:
        ok = x.strides[len(shape) - n:] == tuple(8 * p for p in packed) and \
            all(s >= 0 and s % 8 == 0 for s in x.strides)
        if not ok:
            x = np.ascontiguousarray(x)
    elif tuple(x.stride()[len(shape) - n:]) != packed:
        x = x.contiguous()
    return x


def _strides(x, lead, nproto, torch):
    """per dimension of the broadcast shape `lead`: x's stride in doubles; 0 where x is repeated"""
    shape = tuple(x.shape)[:len(x.shape) - nproto]
    strides = [s // 8 for s in x.strides] if torch is None else list(x.stride())
    out = np.zeros(len(lead), np.int64)
    skip = len(lead) - len(shape)
    for d in range(len(shape)):
        if shape[d] != 1:
            out[skip + d] = strides[d]
    return out


def _pose(fname, args, protos_in, protos_out, out, get_gradients=False, inverted0=False, inverted1=False,
          entry="poseutils", op=None, lensmodel=None,
          names=("the first input", "the second input", "the third input")):
    """The outputs of operation fname on args: each args[k] of shape (..., *protos_in[k]), the leading dimensions
    broadcast together; the value, then (with get_gradients) the gradients, of shapes (broadcast, *protos_out[k]).
    entry: the C entry point, mrcal_b200_<entry>() (two inputs, three outputs: the pose utilities) or its _device
    flavour; "triangulate" has three inputs and four outputs. op: the operation code (default: fname's pose code).
    lensmodel (a parsed lens model, with entry "project"): the call is mrcal_b200_project[_device]() of that model,
    args the points or pixels and the intrinsics, op its MRCAL_B200_PROJECT_* flags other than the gradients; the
    outputs it is not given are not computed. names: the inputs' names in the messages"""
    outs = tuple(out) if isinstance(out, (tuple, list)) else ((out,) if out is not None else None)
    torch = _torch_if_tensors(*args, *(outs or ()), what=f"{fname}(): the inputs and out")
    device = None if torch is None else args[0].device
    args = [_operand(a, p, names[k], fname, torch, device) for k, (a, p) in enumerate(zip(args, protos_in))]
    leads = [tuple(a.shape)[:len(a.shape) - len(p)] for a, p in zip(args, protos_in)]
    try:
        lead = tuple(int(n) for n in np.broadcast_shapes(*leads))
    except ValueError:
        raise ValueError(f"{fname}(): the leading dimensions {leads} of the inputs do not broadcast") from None
    if len(lead) > _MAX_DIMS:
        raise ValueError(f"{fname}(): at most {_MAX_DIMS} broadcast dimensions are supported; got {len(lead)}")
    shapes = [lead + tuple(p) for p in protos_out]

    if outs is not None:
        if len(outs) != len(shapes):
            raise ValueError(f"{fname}(): out must be {'a tuple of ' + str(len(shapes)) + ' arrays' if len(shapes) > 1 else 'one array'}")
        for o, s in zip(outs, shapes):
            if tuple(o.shape) != s:
                raise ValueError(f"{fname}(): out must have shape {s}; got {tuple(o.shape)}")
            if (o.dtype != np.float64) if torch is None else (o.dtype != torch.float64 or o.device != device):
                raise ValueError(f"{fname}(): out must be float64{'' if torch is None else ' on ' + str(device)}")
            if torch is None and not o.flags.writeable:
                raise ValueError(f"{fname}(): out must be writeable")
    # the kernel writes packed outputs: a given out that is not packed is filled afterwards
    if torch is None:
        direct = [outs is not None and o.flags.c_contiguous for o in (outs or shapes)]
        res = [outs[k] if direct[k] else np.empty(s) for k, s in enumerate(shapes)]
    else:
        direct = [outs is not None and o.is_contiguous() for o in (outs or shapes)]
        res = [outs[k] if direct[k] else torch.empty(s, dtype=torch.float64, device=device)
               for k, s in enumerate(shapes)]

    if int(np.prod(lead)) > 0:
        flags = (_GET_GRADIENTS if get_gradients else 0) | (_INVERTED0 if inverted0 else 0) | \
            (_INVERTED1 if inverted1 else 0)
        nin, nout = (3, 4) if entry == "triangulate" else (2, 3)
        st = [_strides(a, lead, len(p), torch) for a, p in zip(args, protos_in)] + [None] * (nin - len(args))
        shape = np.array(lead, np.int64)
        ptr = (lambda a: a.ctypes.data) if torch is None else (lambda a: a.data_ptr())
        ins = [ptr(a) for a in args] + [None] * (nin - len(args))
        o = [ptr(r) for r in res] + [None] * (nout - len(res))
        call = (_ptr(shape), *(x for k in range(nin) for x in (ins[k], _ptr(st[k]))), *o)
        if lensmodel is None:
            code = _OPS[fname] if op is None else op
        else:
            code, flags = C.byref(lensmodel), flags | op
        if torch is None:
            _require_gpu()
            getattr(checked, f"mrcal_b200_{entry}")(code, flags, len(lead), *call)
        else:
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                getattr(checked, f"mrcal_b200_{entry}_device")(code, flags, len(lead), *call, stream)
    if outs is not None:
        for k in range(len(res)):
            if not direct[k]:
                if torch is None:
                    outs[k][...] = res[k]
                else:
                    outs[k].copy_(res[k])
        res = list(outs)
    return tuple(res) if len(res) > 1 else res[0]


def R_from_r(r, *, get_gradients=False, out=None):
    """Rotation matrix R from Rodrigues vector r; with get_gradients: (R, dR/dr (3,3,3))"""
    return _pose("R_from_r", (r,), ((3,),), ((3, 3),) + (((3, 3, 3),) if get_gradients else ()), out, get_gradients)


def r_from_R(R, *, get_gradients=False, out=None):
    """Rodrigues vector r from rotation matrix R; with get_gradients: (r, dr/dR (3,3,3)), taken within the manifold
    of rotations"""
    return _pose("r_from_R", (R,), ((3, 3),), ((3,),) + (((3, 3, 3),) if get_gradients else ()), out, get_gradients)


def Rt_from_rt(rt, *, get_gradients=False, out=None):
    """Rt from rt; with get_gradients: (Rt, dR/dr (3,3,3)). t is copied"""
    return _pose("Rt_from_rt", (rt,), ((6,),), ((4, 3),) + (((3, 3, 3),) if get_gradients else ()), out,
                 get_gradients)


def rt_from_Rt(Rt, *, get_gradients=False, out=None):
    """rt from Rt; with get_gradients: (rt, dr/dR (3,3,3)). t is copied"""
    return _pose("rt_from_Rt", (Rt,), ((4, 3),), ((6,),) + (((3, 3, 3),) if get_gradients else ()), out,
                 get_gradients)


def invert_R(R, *, out=None):
    """The inverse (the transpose) of rotation matrix R"""
    return _pose("invert_R", (R,), ((3, 3),), ((3, 3),), out)


def invert_Rt(Rt, *, out=None):
    """The inverse of transformation Rt: (R', -R't)"""
    return _pose("invert_Rt", (Rt,), ((4, 3),), ((4, 3),), out)


def invert_rt(rt, *, get_gradients=False, out=None):
    """The inverse of transformation rt; with get_gradients: (rt_out, drt_out/drt_in (6,6))"""
    return _pose("invert_rt", (rt,), ((6,),), ((6,),) + (((6, 6),) if get_gradients else ()), out, get_gradients)


def _compose(fname, xs, proto, get_gradients, out, inverted0, inverted1):
    """compose(x0, reduce(compose, x[1:])), as the reference chains more than two operands"""
    if len(xs) < 2:
        raise ValueError(f"{fname}() needs at least two operands")
    if len(xs) != 2:
        if get_gradients:
            raise Exception(f"{fname}(..., get_gradients=True) is supported only if exactly 2 inputs are given")
        if inverted0 or inverted1:
            raise Exception(f"{fname}(..., inverted...=True) is supported only if exactly 2 inputs are given")
    grads = ((proto[0], proto[0]),) * 2 if get_gradients else ()

    def two(a, b, out=None, inverted0=False, inverted1=False):
        return _pose(fname, (a, b), (proto, proto), (proto,) + grads, out, get_gradients, inverted0, inverted1)

    return two(xs[0], reduce(two, xs[1:]), out=out, inverted0=inverted0, inverted1=inverted1)


def compose_Rt(*Rt, out=None, inverted0=False, inverted1=False):
    """The composition of transformations Rt: compose_Rt(Rt0, Rt1) applies Rt1, then Rt0. With inverted0/inverted1,
    that operand is inverted first (exactly two operands only)"""
    return _compose("compose_Rt", Rt, (4, 3), False, out, inverted0, inverted1)


def compose_r(*r, get_gradients=False, out=None, inverted0=False, inverted1=False):
    """The composition of rotations r; with get_gradients (exactly two operands): (r, dr/dr0, dr/dr1), with respect
    to the operands as given, inverted or not"""
    return _compose("compose_r", r, (3,), get_gradients, out, inverted0, inverted1)


def compose_rt(*rt, get_gradients=False, out=None, inverted0=False, inverted1=False):
    """The composition of transformations rt; with get_gradients (exactly two operands): (rt, drt/drt0 (6,6),
    drt/drt1 (6,6)), with respect to the operands as given, inverted or not"""
    return _compose("compose_rt", rt, (6,), get_gradients, out, inverted0, inverted1)


def compose_r_tinyr0_gradientr0(r1, *, out=None):
    """dr01/dr0 of compose_r(r0, r1) at r0 = 0"""
    return _pose("compose_r_tinyr0_gradientr0", (r1,), ((3,),), ((3, 3),), out)


def compose_r_tinyr1_gradientr1(r0, *, out=None):
    """dr01/dr1 of compose_r(r0, r1) at r1 = 0"""
    return _pose("compose_r_tinyr1_gradientr1", (r0,), ((3,),), ((3, 3),), out)


def compose_rt_tinyrt0_gradientrt0(rt1, *, out=None):
    """drt01/drt0 of compose_rt(rt0, rt1) at rt0 = 0, (6,6)"""
    return _pose("compose_rt_tinyrt0_gradientrt0", (rt1,), ((6,),), ((6, 6),), out)


def compose_rt_tinyrt1_gradientrt1(rt0, *, out=None):
    """drt01/drt1 of compose_rt(rt0, rt1) at rt1 = 0, (6,6)"""
    return _pose("compose_rt_tinyrt1_gradientrt1", (rt0,), ((6,),), ((6, 6),), out)


def _point(fname, pose, proto, dproto, x, get_gradients, out, inverted):
    grads = (dproto, (3, 3)) if get_gradients else ()
    return _pose(fname, (pose, x), (proto, (3,)), ((3,),) + grads, out, get_gradients, inverted)


def rotate_point_r(r, x, *, get_gradients=False, out=None, inverted=False):
    """x rotated by r (by its inverse if inverted); with get_gradients: (x, dx/dr (3,3), dx/dx_in (3,3))"""
    return _point("rotate_point_r", r, (3,), (3, 3), x, get_gradients, out, inverted)


def rotate_point_R(R, x, *, get_gradients=False, out=None, inverted=False):
    """x rotated by R (by R' if inverted); with get_gradients: (x, dx/dR (3,3,3), dx/dx_in (3,3))"""
    return _point("rotate_point_R", R, (3, 3), (3, 3, 3), x, get_gradients, out, inverted)


def transform_point_rt(rt, x, *, get_gradients=False, out=None, inverted=False):
    """x transformed by rt (by its inverse if inverted); with get_gradients: (x, dx/drt (3,6), dx/dx_in (3,3))"""
    return _point("transform_point_rt", rt, (6,), (3, 6), x, get_gradients, out, inverted)


def transform_point_Rt(Rt, x, *, get_gradients=False, out=None, inverted=False):
    """x transformed by Rt (by its inverse if inverted); with get_gradients: (x, dx/dRt (3,4,3), dx/dx_in (3,3))"""
    return _point("transform_point_Rt", Rt, (4, 3), (3, 4, 3), x, get_gradients, out, inverted)


def skew_symmetric(a, *, out=None):
    """The matrix A with A b = cross(a, b)"""
    return _pose("skew_symmetric", (a,), ((3,),), ((3, 3),), out)


def R_from_quat(q, *, out=None):
    """Rotation matrix from unit quaternion q = (w,x,y,z)"""
    return _pose("R_from_quat", (q,), ((4,),), ((3, 3),), out)


def quat_from_R(R, *, out=None):
    """Unit quaternion (w,x,y,z) from rotation matrix R, as the reference computes it (scipy's algorithm; the sign is
    not normalized)"""
    return _pose("quat_from_R", (R,), ((3, 3),), ((4,),), out)


def qt_from_Rt(Rt, *, out=None):
    """qt (7,) from Rt"""
    return _pose("qt_from_Rt", (Rt,), ((4, 3),), ((7,),), out)


def Rt_from_qt(qt, *, out=None):
    """Rt from qt (7,)"""
    return _pose("Rt_from_qt", (qt,), ((7,),), ((4, 3),), out)


def R_aligned_to_vector(v, *, out=None):
    """A rotation matrix whose third row (the z axis) is v normalized"""
    return _pose("R_aligned_to_vector", (v,), ((3,),), ((3, 3),), out)


def _identity(value, out):
    if out is None:
        return value
    out[...] = value
    return out


def identity_R(*, out=None):
    """The (3,3) identity rotation"""
    return _identity(np.eye(3), out)


def identity_r(*, out=None):
    """The (3,) identity rotation"""
    return _identity(np.zeros(3), out)


def identity_Rt(*, out=None):
    """The (4,3) identity transformation"""
    return _identity(np.vstack((np.eye(3), np.zeros((1, 3)))), out)


def identity_rt(*, out=None):
    """The (6,) identity transformation"""
    return _identity(np.zeros(6), out)
