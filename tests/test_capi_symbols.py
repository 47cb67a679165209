"""The C-ABI library loads, and its binding types every symbol include/mrcal_b200.h declares as the header does
(no GPU needed)."""
import ctypes
import glob
import os
import re

import pytest

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))


def _strip_c(text):
    """C source without comments and preprocessor lines"""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    return "\n".join(l for l in text.splitlines() if not l.lstrip().startswith("#"))


def _prototypes(text, pattern):
    """name -> (return type, [parameter declarations]) of every match of pattern, whose groups are the return type,
    the name and the parameter list"""
    out = {}
    for ret, name, params in re.findall(pattern, _strip_c(text)):
        params = [" ".join(p.split()) for p in params.split(",")]
        out[name] = (" ".join(ret.split()), [] if params == ["void"] else params)
    return out


def _kind(c_type, returned=False):
    """the ctypes type the binding must give a C parameter or return type; an unmapped type fails the test, so a new
    kind has to be added here on purpose"""
    from mrcal_b200 import _capi
    c_type = c_type.replace(" *", "*")
    returns = {"void": None, "const char*": ctypes.c_char_p, "const char* const*": ctypes.POINTER(ctypes.c_char_p),
               "mrcal_stats_t": _capi.Stats, "mrcal_lensmodel_metadata_t": _capi.Metadata}
    if returned and c_type in returns:
        return returns[c_type]
    if "*" in c_type:
        return ctypes.c_void_p
    by_value = {"int": ctypes.c_int, "mrcal_lensmodel_type_t": ctypes.c_int, "double": ctypes.c_double,
                "bool": ctypes.c_bool, "uint16_t": ctypes.c_uint16, "size_t": ctypes.c_size_t,
                "mrcal_problem_selections_t": _capi.Selections}
    base = " ".join(w for w in c_type.split() if w != "const")
    assert base in by_value, f"no ctypes kind for the C type '{c_type}'"
    return by_value[base]


def _parameter_kind(declaration):
    c_type = re.fullmatch(r"(.*?)\s*\b\w+", declaration).group(1)   # without the parameter's name
    return _kind(c_type)


def test_library_loads_and_exports_header_symbols():
    """The library exports every function include/mrcal_b200.h declares, and both handles of the binding type each of
    them, and each test entry mrcal_b200_debug_*() the sources define, with its C arity, argument types and return
    type. Through `checked`, a false bool or a NULL handle raises, except where the caller reads the status itself"""
    from mrcal_b200 import _capi
    declared = _prototypes(open(os.path.join(ROOT, "include", "mrcal_b200.h")).read(),
                           r"([\w\s*]+?)\b(_?mrcal_\w+)\s*\(([^()]*)\)\s*;")
    debug = {}
    for f in glob.glob(os.path.join(ROOT, "mrcal_b200", "csrc", "*.cu")):
        debug.update(_prototypes(open(f).read(),
                                 r'extern\s+"C"\s+([\w\s*]+?)\b(mrcal_b200_debug_\w+)\s*\(([^()]*)\)\s*\{'))
    assert len(declared) > 90 and len(debug) >= 7
    assert set(_capi.EXPORTED_SYMBOLS) == set(declared), set(_capi.EXPORTED_SYMBOLS) ^ set(declared)
    assert set(_capi.DEBUG_SIGNATURES) == set(debug), set(_capi.DEBUG_SIGNATURES) ^ set(debug)
    # the status returns: a lens-model name that does not parse, and no factorization when J'J is not positive definite
    status = {"mrcal_lensmodel_from_name", "mrcal_b200_factorization_create_from_last_callback"}
    for name, (ret, params) in {**declared, **debug}.items():
        for f in (getattr(_capi.lib, name), getattr(_capi.checked, name)):
            assert f.argtypes is not None and list(f.argtypes) == [_parameter_kind(p) for p in params], name
            assert f.restype == _kind(ret, returned=True), name
        raises = ret == "bool" or re.fullmatch(r"mrcal_b200_\w+_create\w*", name) is not None
        assert (getattr(_capi.checked, name).errcheck is not None) == (raises and name not in status), name
        assert getattr(_capi.lib, name).errcheck is None, name


def test_checked_binding_raises_the_library_message():
    """Where the C ABI returns false and sets the message, the package's binding raises it"""
    import mrcal_b200
    from mrcal_b200 import _capi
    if mrcal_b200.device_count() > 0:
        pytest.skip("checks the behaviour without a device")
    args = (None, 0, 2, False, None, 0, -1., None, None)
    assert not _capi.lib.mrcal_b200_problem_projection_uncertainty(*args)
    with pytest.raises(RuntimeError, match=r"^mrcal_b200_problem_projection_uncertainty\(\) failed: .*no usable CUDA "
                                           r"device"):
        _capi.checked.mrcal_b200_problem_projection_uncertainty(*args)


def test_header_is_plain_c(tmp_path):
    """include/mrcal_b200.h is the drop-in boundary: it has to compile as C (gnu11, the reference's dialect: its types use
    anonymous structs, basic-geometry.h:19-60) and as C++"""
    import shutil
    import subprocess
    src = tmp_path / "h.c"
    src.write_text('#include "mrcal_b200.h"\nint main(void) { return (int)sizeof(mrcal_lensmodel_t) - (int)sizeof(mrcal_lensmodel_t); }\n')
    inc = os.path.join(ROOT, "include")
    for cc, std in (("gcc", "-std=gnu11"), ("g++", "-std=c++17")):
        if shutil.which(cc) is None:
            pytest.skip(cc + " not found")
        r = subprocess.run([cc, std, "-Wall", "-Wextra", "-Werror", "-fsyntax-only", "-x", "c" if cc == "gcc" else "c++", "-I", inc, str(src)],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr


def test_struct_sizes_match_reference_abi():
    from mrcal_b200 import _capi
    assert ctypes.sizeof(_capi.Lensmodel) == 16      # types.h:122-136
    assert ctypes.sizeof(_capi.Selections) == 1      # types.h:283-307
    assert ctypes.sizeof(_capi.Stats) == 16          # types.h:320-343
    assert ctypes.sizeof(_capi.Sparse) == 88         # public cholmod_sparse layout


def test_no_gpu_fails_loudly():
    """Without a CUDA device the hot path must raise, never fall back."""
    import mrcal_b200
    from mrcal_b200 import synthetic
    if mrcal_b200.device_count() > 0:
        pytest.skip("a GPU is present")
    inp, _ = synthetic.make_problem(Ncameras=1, Nframes=3, W=4, H=4)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        mrcal_b200.optimizer_callback(**inp)
    with pytest.raises(RuntimeError, match="no usable CUDA device"):
        mrcal_b200.optimize(**inp)


def test_product_does_not_import_oracle():
    """The product must never route through the oracle (test infrastructure)."""
    pkg = os.path.join(ROOT, "mrcal_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cpp", ".h", ".cuh")):
                txt = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
                assert "libmrcal_ref" not in txt, f
