"""The `.cameramodel` file format either side of the solve (SURVEY.md 8f rank 4): what mrcal's tools read
the seed from and write the result to (reference: mrcal/cameramodel.py:160-690, native format only).

A `.cameramodel` is a Python-literal dict with comments:

    {
        'lensmodel':  'LENSMODEL_OPENCV8',
        'intrinsics': [ fx, fy, cx, cy, ... ],
        'rt_cam_ref': [ r0, r1, r2, t0, t1, t2 ],      # 'extrinsics' in files written by mrcal < 2.5
        'imagersize': [ W, H ],
        'valid_intrinsics_region': [ [x,y], ... ],      # optional
        'icam_intrinsics': 0, 'icam_extrinsics': -1,    # with optimization_inputs only
        'optimization_inputs': b'...',                  # optional: base85(npz) of the whole optimize() input
    }

so that a model written here is readable by the reference's tools and vice versa. Pure host code: numpy only,
no GPU. `cameramodel(optimization_inputs=..., icam_intrinsics=i)` is how a solve result becomes a model."""
import ast
import base64
import io

import numpy as np

from ._poses_host import R_from_r as _R_from_r  # noqa: F401  (the private name callers import from this module)
from ._poses_host import Rt_from_rt, invert_rt

_LEGACY_INPUT_NAMES = (("frames_rt_toref", "rt_ref_frame"), ("extrinsics_rt_fromref", "rt_cam_ref"))


class CameramodelParseException(Exception):
    """A `.cameramodel` could not be parsed (the reference's name for it: mrcal/cameramodel.py:150)."""


def serialize_optimization_inputs(optimization_inputs):
    """dict -> the byte string stored under 'optimization_inputs' (mrcal/cameramodel.py:160-307): None becomes '',
    empty new-style arguments are dropped, the pose arrays go under their OLD names (so that older mrcal reads the
    file), np.savez_compressed without pickling, base85."""
    d = {}
    for k, v in optimization_inputs.items():
        if v is None:
            v = ""
        if k in ("do_apply_regularization_unity_cam01", "observations_point_triangulated",
                 "indices_point_triangulated_camintrinsics_camextrinsics"):
            if (isinstance(v, np.ndarray) and v.size == 0) or (not isinstance(v, np.ndarray) and not v):
                continue
        d[k] = v
    for old, new in _LEGACY_INPUT_NAMES:
        vo, vn = d.get(old, ""), d.get(new, "")
        if isinstance(vo, str) and vo.startswith("ERROR:"):
            vo = ""
        empty = lambda x: isinstance(x, str) and x == ""
        if not empty(vo) and not empty(vn) and np.any(np.asarray(vo) - np.asarray(vn)):
            raise RuntimeError(f"optimization_inputs has both keys '{old}' and '{new}', but they're not the same")
        d.pop(new, None)
        d.pop(old, None)
        if not empty(vo) or not empty(vn):
            d[old] = vn if empty(vo) else vo
    f = io.BytesIO()
    np.savez_compressed(f, **d)
    return base64.b85encode(f.getvalue())


def deserialize_optimization_inputs(data_bytes):
    """The inverse (mrcal/cameramodel.py:310-388): 0-d arrays back to Python scalars, '' back to None, the pose
    arrays under their NEW names with the old names poisoned (a string where an array is expected, which
    optimize() takes for "not given"), exactly what the reference hands to code written against it."""
    z = np.load(io.BytesIO(base64.b85decode(data_bytes)), allow_pickle=False)
    d = {}
    for k in z.keys():
        a = z[k]
        if a.shape == ():
            a = a.item()
        if isinstance(a, str) and a == "":
            a = None
        d[k] = a
    for old, new in (("do_optimize_intrinsic_core", "do_optimize_intrinsics_core"),
                     ("do_optimize_intrinsic_distortions", "do_optimize_intrinsics_distortions")):
        if old in d and new not in d:
            d[new] = d.pop(old)
    for old, new in _LEGACY_INPUT_NAMES:
        if old in d and new not in d:
            d[new] = d[old]
        d[old] = f'ERROR: mrcal 2.5 renamed optimization_inputs fields: "{old}" -> "{new}". Please update your code to use the new name'
    d.pop("calibration_object_width_n", None)
    d.pop("calibration_object_height_n", None)
    if d.get("rt_cam_ref") is None:
        d["rt_cam_ref"] = np.zeros((0, 6))
    return d


def _check(lensmodel, intrinsics, imagersize, rt):
    from . import api
    n = api.lensmodel_num_params(lensmodel)   # raises on an unknown model
    if len(intrinsics) != n:
        raise RuntimeError(f"Mismatched intrinsics: {lensmodel} needs {n} values, got {len(intrinsics)}")
    if len(imagersize) != 2 or any(int(x) != x or x <= 0 for x in imagersize):
        raise RuntimeError("imagersize must be two positive integers")
    if len(rt) != 6:
        raise RuntimeError("rt_cam_ref must have 6 values: r (Rodrigues) then t")


class cameramodel:
    """One camera: (lensmodel, intrinsics), imager size, pose, and optionally the optimization it came from."""

    def __init__(self, file_or_model=None, *, intrinsics=None, imagersize=None, rt_cam_ref=None, rt_ref_cam=None,
                 extrinsics_rt_fromref=None, valid_intrinsics_region=None, optimization_inputs=None, icam_intrinsics=None):
        self._valid_intrinsics_region = None
        self._optimization_inputs_string = None
        self._icam_intrinsics = self._icam_extrinsics = None
        if rt_cam_ref is None:
            rt_cam_ref = extrinsics_rt_fromref
        if file_or_model is not None:
            if isinstance(file_or_model, cameramodel):
                self.__dict__.update({k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in file_or_model.__dict__.items()})
            elif isinstance(file_or_model, str) and "{" not in file_or_model:
                with open(file_or_model) as f:
                    self._parse(f.read(), file_or_model)
            else:
                self._parse(file_or_model if isinstance(file_or_model, str) else file_or_model.read(), None)
            return
        if optimization_inputs is not None:
            # a model out of a solve (mrcal/cameramodel.py:1210-1260): camera icam_intrinsics of these inputs
            if icam_intrinsics is None:
                raise RuntimeError("optimization_inputs given, so icam_intrinsics is required too")
            from . import api
            I = optimization_inputs
            icam_e = api.corresponding_icam_extrinsics(icam_intrinsics, **{k: v for k, v in I.items() if v is not None})
            self._intrinsics = (I["lensmodel"], np.array(I["intrinsics"][icam_intrinsics], float))
            self._imagersize = np.array(I["imagersizes"][icam_intrinsics], np.int32)
            rt = I.get("rt_cam_ref", I.get("extrinsics_rt_fromref"))
            self._rt_cam_ref = np.zeros(6) if icam_e < 0 else np.array(rt[icam_e], float)
            self._optimization_inputs_string = serialize_optimization_inputs(I)
            self._icam_intrinsics, self._icam_extrinsics = int(icam_intrinsics), int(icam_e)
        else:
            if intrinsics is None or imagersize is None:
                raise RuntimeError("cameramodel(): give a file/model, or optimization_inputs, or intrinsics + imagersize")
            self._intrinsics = (intrinsics[0], np.array(intrinsics[1], float))
            self._imagersize = np.array(imagersize, np.int32)
            if rt_ref_cam is not None:
                rt_cam_ref = invert_rt(rt_ref_cam)
            self._rt_cam_ref = np.zeros(6) if rt_cam_ref is None else np.array(rt_cam_ref, float)
        if valid_intrinsics_region is not None:
            self._valid_intrinsics_region = np.array(valid_intrinsics_region, float).reshape(-1, 2)
        _check(self._intrinsics[0], self._intrinsics[1], self._imagersize, self._rt_cam_ref)

    def _parse(self, s, name):
        try:
            m = ast.literal_eval(s)
            assert isinstance(m, dict)
        except Exception:
            raise CameramodelParseException("Failed to parse cameramodel" + (f" '{name}'" if name else "!"))
        # names older files use (mrcal/cameramodel.py:593-622)
        for old, new in (("distortion_model", "lensmodel"), ("lens_model", "lensmodel"),
                         ("icam_intrinsics_optimization_inputs", "icam_intrinsics")):
            if old in m and new not in m:
                m[new] = m.pop(old)
        if "extrinsics" in m:
            if "rt_cam_ref" in m and np.abs(np.array(m["extrinsics"]) - np.array(m["rt_cam_ref"])).max() >= 1e-9:
                raise CameramodelParseException("'rt_cam_ref' and 'extrinsics' both given, and they're NOT the same")
            m.setdefault("rt_cam_ref", m["extrinsics"])
        missing = {"lensmodel", "intrinsics", "rt_cam_ref", "imagersize"} - set(m)
        if missing:
            raise CameramodelParseException(f"Model must have at least the keys lensmodel, intrinsics, rt_cam_ref, imagersize; missing: {sorted(missing)}")
        lensmodel = m["lensmodel"].replace("DISTORTION", "LENSMODEL")
        self._intrinsics = (lensmodel, np.array(m["intrinsics"], float))
        self._imagersize = np.array(m["imagersize"], np.int32)
        self._rt_cam_ref = np.array(m["rt_cam_ref"], float)
        _check(lensmodel, self._intrinsics[1], m["imagersize"], self._rt_cam_ref)
        if m.get("valid_intrinsics_region") is not None:
            self._valid_intrinsics_region = np.array(m["valid_intrinsics_region"], float).reshape(-1, 2)
        if "optimization_inputs" in m:
            if not isinstance(m["optimization_inputs"], bytes):
                raise CameramodelParseException("'optimization_inputs' is given, but it's not a byte string")
            if not isinstance(m.get("icam_intrinsics"), int) or m["icam_intrinsics"] < 0:
                raise CameramodelParseException("'optimization_inputs' is given, but icam_intrinsics is not an int >= 0")
            self._optimization_inputs_string = m["optimization_inputs"]
            self._icam_intrinsics = m["icam_intrinsics"]
            self._icam_extrinsics = m.get("icam_extrinsics")
        elif "icam_intrinsics" in m or "icam_extrinsics" in m:
            raise CameramodelParseException("'optimization_inputs' is NOT given, but icam_intrinsics or icam_extrinsics ARE given")

    # ---- accessors (the reference's names)
    def intrinsics(self):
        return self._intrinsics[0], self._intrinsics[1].copy()

    def imagersize(self):
        return self._imagersize.copy()

    def rt_cam_ref(self, rt=None):
        if rt is not None:
            if len(rt) != 6:
                raise RuntimeError("rt_cam_ref must have 6 values")
            self._rt_cam_ref = np.array(rt, float)   # moving the camera keeps the optimization inputs valid
            return None
        return self._rt_cam_ref.copy()

    def rt_ref_cam(self, rt=None):
        if rt is not None:
            return self.rt_cam_ref(invert_rt(rt))
        return invert_rt(self._rt_cam_ref)

    def Rt_cam_ref(self):
        """The pose as a (4,3) Rt transformation: R on top, t in the last row"""
        return Rt_from_rt(self._rt_cam_ref)

    def Rt_ref_cam(self):
        return Rt_from_rt(self.rt_ref_cam())

    extrinsics_rt_fromref = rt_cam_ref
    extrinsics_rt_toref = rt_ref_cam

    def valid_intrinsics_region(self, valid_intrinsics_region=None):
        """The valid-intrinsics region (N,2), or None if the model has none. Given a region, sets it instead (a copy),
        closing an open contour first, and returns True: it must be (N,2) with N >= 4 once closed, or (0,2) for "valid
        nowhere" (mrcal/cameramodel.py:1820-1865)"""
        if valid_intrinsics_region is None:
            return None if self._valid_intrinsics_region is None else self._valid_intrinsics_region.copy()
        from .regions import close_contour
        r = close_contour(np.array(valid_intrinsics_region))
        if not (r.ndim == 2 and r.shape[1] == 2 and (r.shape[0] >= 4 or r.shape[0] == 0)):
            raise RuntimeError("The valid-intrinsics region must be a numpy array of shape (N,2) with N >= 4 or N == 0. "
                               f"Instead got shape {r.shape}")
        self._valid_intrinsics_region = np.array(r, dtype=float)
        return True

    def optimization_inputs(self):
        if self._optimization_inputs_string is None:
            return None
        return deserialize_optimization_inputs(self._optimization_inputs_string)

    def icam_intrinsics(self):
        return self._icam_intrinsics

    def icam_extrinsics(self):
        return self._icam_extrinsics

    # ---- output: key order, number formatting and comments as the reference writes them (mrcal/cameramodel.py:503-559)
    def __str__(self):
        g = lambda a: "".join(f" {float(x):.10g}," for x in a)
        out = ["{", f"    'lensmodel':  '{self._intrinsics[0]}',", "",
               "    # intrinsics are fx,fy,cx,cy,distortion0,distortion1,....",
               f"    'intrinsics': [{g(self._intrinsics[1])}],", ""]
        if self._valid_intrinsics_region is not None:
            out.append("    'valid_intrinsics_region': [")
            out += [f"    [ {x:.10g}, {y:.10g} ]," for x, y in self._valid_intrinsics_region]
            out += ["],", ""]
        out += [f"    'rt_cam_ref': [{g(self._rt_cam_ref)}],",
                f"    'extrinsics': [{g(self._rt_cam_ref)}], # for compatibility with mrcal < 2.5", "",
                f"    'imagersize': [ {int(self._imagersize[0])}, {int(self._imagersize[1])},],", ""]
        if self._icam_intrinsics is not None:
            out.append(f"    'icam_intrinsics': {self._icam_intrinsics:d},")
        if self._icam_extrinsics is not None:
            out.append(f"    'icam_extrinsics': {self._icam_extrinsics:d},")
        out.append("")
        if self._optimization_inputs_string is not None:
            out += ["    # The optimization inputs: everything that went into the solve this model came from (all the",
                    "    # observations of all the cameras), as np.savez_compressed() bytes in base-85",
                    f"    'optimization_inputs': {self._optimization_inputs_string},", ""]
        out.append("}")
        return "\n".join(out) + "\n"

    def write(self, f, note=None):
        text = ("".join("# " + l + "\n" for l in note.splitlines()) if note else "") + str(self)
        if isinstance(f, str):
            with open(f, "w") as fh:
                fh.write(text)
        else:
            f.write(text)
