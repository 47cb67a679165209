"""CPU: the answers the triangulation GPU tests compare against (tests/triangulation_np.py and the stored
tests/golden/triangulation.npz), and the refusals that come before any device work."""
import numpy as np
import pytest

import mrcal_b200
import triangulation_np as T


def test_golden_matches_the_compiled_reference(ref):
    z = np.load(T.GOLDEN)
    for key, fname, args, g in T.cases():
        for k, a in enumerate(args):
            assert np.array_equal(z[f"{key}/in{k}"], a, equal_nan=True), key
        for k, a in enumerate(T.reference(fname, args, g)):
            assert np.array_equal(z[f"{key}/out{k}"], a, equal_nan=True), f"{key} output {k}"


def test_refusals_before_device_work():
    v, t = np.zeros(3), np.zeros(3)
    Rt = np.zeros((4, 3))
    f = mrcal_b200.triangulate_leecivera_mid2
    with pytest.raises(Exception, match="Both were non-None"):
        f(v, v, t, Rt01=Rt)
    with pytest.raises(Exception, match="Both were None"):
        f(v, v)
    with pytest.raises(Exception, match="v_are_local MUST be the default"):
        mrcal_b200.triangulate_geometric(v, v, Rt01=Rt, v_are_local=True, get_gradients=True)
    with pytest.raises(Exception, match="Rt01 MUST have been given"):
        mrcal_b200.triangulate_leecivera_l1(v, v, t, v_are_local=True)
    with pytest.raises(Exception, match="t01 MUST have been given"):
        mrcal_b200._triangulated_error(v, v, Rt01=Rt, get_gradients=True)
    with pytest.raises(Exception, match="v_are_local MUST be True"):
        mrcal_b200.triangulate_lindstrom(v, v, Rt, v_are_local=False, get_gradients=True)
    with pytest.raises(ValueError, match=r"shape \(\.\.\.,3\)"):
        f(np.zeros(2), v, t)
    with pytest.raises(ValueError, match=r"shape \(\.\.\.,4,3\)"):
        mrcal_b200.triangulate_lindstrom(v, v, np.zeros((3, 3)))
    with pytest.raises(ValueError, match="do not broadcast"):
        mrcal_b200.triangulate_leecivera_wmid2(np.zeros((2, 3)), np.zeros((3, 3)), t)
    with pytest.raises(ValueError, match="out must be a tuple of 4"):
        f(v, v, t, get_gradients=True, out=np.zeros(3))
    with pytest.raises(ValueError, match=r"out must have shape \(\)"):
        mrcal_b200._triangulated_error(v, v, t, out=np.zeros(3))
    torch = pytest.importorskip("torch")
    with pytest.raises(RuntimeError, match="may not be mixed"):
        f(v, torch.zeros(3, dtype=torch.float64), t)
    with pytest.raises(ValueError, match="CUDA float64"):
        f(torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64))
    with pytest.raises(ValueError, match="CUDA float64"):
        f(torch.zeros(3, dtype=torch.float32), torch.zeros(3, dtype=torch.float32), torch.zeros(3, dtype=torch.float32))
