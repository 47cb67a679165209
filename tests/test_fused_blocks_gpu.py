"""The reduced normal equations assembled from the fused evaluation's per-observation blocks (fused_eval.cu, the compact
layout of normal.h) against the same system assembled from the stored Jacobian, and from run to run."""
import numpy as np
import pytest

import mrcal_b200
import problems
from mrcal_b200 import synthetic

pytestmark = pytest.mark.gpu


def _cases():
    golden = dict(problems.golden_cases())
    cases = [(n, golden[n]) for n in ("splined3_2cam_corelocked", "splined2_2cam_corelocked")]
    # the benchmark's configuration at a fraction of its frames: 4 cameras (3 with extrinsics), 10x10 boards, the warp
    kw, _ = synthetic.baseline_config(3, Nframes=24, pixel_noise=0.3)
    cases.append(("config3_24frames", kw))
    return cases


CASES = _cases()


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("lam", [0.0, 1e-3])
def test_fused_matches_stored_jacobian(name, kw, lam):
    P = mrcal_b200.Problem(**kw)
    S_j, g_j, gf_j = P.reduced_system(lam)
    S_f, g_f, gf_f = P.reduced_system(lam, fused=True)
    assert S_f.shape == S_j.shape and S_j.size
    assert np.abs(S_f - S_j).max() <= 1e-9 * np.abs(S_j).max(), "S"
    assert np.abs(g_f - g_j).max() <= 1e-9 * np.abs(gf_j).max(), "g'"
    assert np.abs(gf_f - gf_j).max() <= 1e-9 * np.abs(gf_j).max(), "J'x"
    # the stored-Jacobian path places its blocks anew after the fused one used the pool
    S_j2, g_j2, gf_j2 = P.reduced_system(lam)
    assert np.array_equal(S_j2, S_j) and np.array_equal(g_j2, g_j) and np.array_equal(gf_j2, gf_j)


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_fused_assembly_is_deterministic(name, kw):
    P = mrcal_b200.Problem(**kw)
    a = P.reduced_system(1e-3, fused=True)
    b = P.reduced_system(1e-3, fused=True)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_optimize_keeps_the_fused_path(name, kw, capfd):
    P = mrcal_b200.Problem(**kw)
    P.reset()
    info = P.optimize(max_iterations=20)
    err = capfd.readouterr().err
    assert "disagrees" not in err and "stored-Jacobian path" not in err, err
    assert info["Niterations"] > 0


def test_fused_is_refused_where_it_does_not_apply():
    kw = dict(problems.golden_cases())["opencv8_2cam_all"]
    P = mrcal_b200.Problem(**kw)
    with pytest.raises(RuntimeError, match="fused evaluation"):
        P.reduced_system(0.0, fused=True)
