"""The numpy pose conversions of the host-side plumbing (mrcal_b200/_poses_host.py): their values against the
reference's answers (tests/poseutils_np.py: the compiled reference, or tests/golden/poseutils.npz without it), round
trips, and the inverse pose against the compiled reference."""
import numpy as np
import pytest

from mrcal_b200 import _poses_host as P
import poseutils_np as U

FUNCTIONS = ("R_from_r", "r_from_R", "Rt_from_rt", "rt_from_Rt", "invert_Rt", "invert_rt", "compose_Rt",
             "transform_point_Rt")
_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = U.load()
    return _CASES


def _keys():
    return [k for k, f, _, kw, _ in U.cases(ref_available=False)
            if f in FUNCTIONS and not any(v for n, v in kw.items() if n.startswith("inverted"))]


@pytest.mark.parametrize("key", _keys())
def test_against_reference(key):
    _, fname, args, _, _, want = next(c for c in cases() if c[0] == key)
    U.check_value(key, fname, getattr(P, fname)(*args), want[0], P.R_from_r)


def test_pose_utilities_roundtrip():
    rng = np.random.default_rng(0)
    for _ in range(20):
        rt = np.concatenate((rng.uniform(-1.7, 1.7, 3), rng.uniform(-3, 3, 3)))   # |r| < pi
        Rt = P.Rt_from_rt(rt)
        assert np.allclose(P.rt_from_Rt(Rt), rt, atol=1e-12)
        assert np.allclose(P.compose_Rt(Rt, P.invert_Rt(Rt)), np.concatenate((np.eye(3), np.zeros((1, 3)))), atol=1e-12)
    # rotation by almost pi
    r = np.array((0.3, -0.2, 0.9)); r *= (np.pi - 1e-8) / np.linalg.norm(r)
    assert np.allclose(P.R_from_r(P.r_from_R(P.R_from_r(r))), P.R_from_r(r), atol=1e-7)


def test_inverse_pose_matches_reference(ref):
    rng = np.random.default_rng(0)
    for _ in range(5):
        rt = rng.normal(size=6)
        assert np.allclose(P.invert_rt(rt), ref.invert_rt(rt), atol=1e-12)
    assert np.allclose(P.invert_rt(np.array((0., 0., 0., 1., 2., 3.))), (0., 0., 0., -1., -2., -3.))
