"""The reduced normal equations are assembled without atomics for every problem (normal.cu, normal_det.cu): the same
problem gives the same system, bit for bit. Also the problems at the edges of that assembly: board
observations wider than the tensor-pipe Gram kernel takes (more than 160 local columns, and more than 255), and
problems with no board or point observations at all."""
import numpy as np
import pytest

import mrcal_b200
import problems
from problems import reduced_reference
from mrcal_b200 import synthetic

pytestmark = pytest.mark.gpu

# A dense spline over a narrow field of view: a board observation spans a large patch of knots
SPL3_DENSE = "LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=30_Ny=20_fov_x_deg=45"


def eliminated_range(P, kw):
    fr0 = mrcal_b200.state_index_frames(0, **kw)
    pt0 = mrcal_b200.state_index_points(0, **kw)
    e0 = fr0 if fr0 is not None else (pt0 if pt0 is not None else P.Nstate)
    e1 = e0 + mrcal_b200.num_states_frames(**kw) * (fr0 is not None) + mrcal_b200.num_states_points(**kw) * (pt0 is not None)
    return e0, e1


def check_reduced(P, kw, lam):
    b, x, J = P.callback()
    S, g, gfull = P.reduced_system(lam)
    e0, e1 = eliminated_range(P, kw)
    S_ref, g_ref, gfull_ref, scale = reduced_reference(J, x, e0, e1, lam)
    assert np.abs(gfull - gfull_ref).max() <= 1e-10 * np.abs(gfull_ref).max(), "J'x"
    act = np.diag(S) != 0
    assert act.sum() > 0
    assert np.abs(S[np.ix_(act, act)] - S_ref[np.ix_(act, act)]).max() <= 1e-9 * scale, "S"
    assert np.abs(g[act] - g_ref[act]).max() <= 1e-9 * np.abs(gfull_ref).max(), "g'"
    return J


CASES = problems.golden_cases()


@pytest.mark.parametrize("name,kw", CASES, ids=[c[0] for c in CASES])
def test_bitwise_repeatable(name, kw):
    P = mrcal_b200.Problem(**kw)
    for lam in (0.0, 1e-3):
        S1, g1, f1 = P.reduced_system(lam)
        S2, g2, f2 = P.reduced_system(lam)
        assert np.array_equal(S1, S2) and np.array_equal(g1, g2) and np.array_equal(f1, f2)


def test_triangulated_only():
    # no board or point observations: the extrinsics x extrinsics block comes from the triangulated rows alone
    name, kw = next(c for c in CASES if c[0] == "tri_pinhole_unity_only")
    P = mrcal_b200.Problem(**kw)
    for lam in (0.0, 1e-3):
        check_reduced(P, kw, lam)


def wide_problem():
    kw, truth = synthetic.make_problem(lensmodel=SPL3_DENSE, Ncameras=2, Nframes=3, W=10, H=8, seed=2, pixel_noise=0.2)
    return kw


def test_wide_observations():
    kw = wide_problem()
    P = mrcal_b200.Problem(**kw)
    J = check_reduced(P, kw, 0.0)
    check_reduced(P, kw, 1e-3)
    # the local columns of each board observation: every column its rows touch (intrinsics, extrinsics, frame, warp)
    rows = 2 * 10 * 8
    Jc = J.tocsr()
    widths = [len(np.unique(Jc[o * rows:(o + 1) * rows].indices)) for o in range(kw["observations_board"].shape[0])]
    # the widest takes the scalar Gram kernel with its block summed in the pool (> 200 columns), past the 8-bit offsets
    # (> 255); the others the same kernel's shared-memory form
    assert max(widths) > 255, widths
    assert min(widths) <= 200, widths
    # ... and their blocks outgrow the pool as the workspace sizes it (a splined board: 160 local columns + the two
    # gradient rows, squared), so it grows before the assembly. A block is (nsh + 2) x (nsh + 2), nsh + 2 rounded up to
    # even, nsh = the columns other than the frame's 6
    need = sum(((w - 6 + 2 + 1) & ~1) ** 2 for w in widths)
    assert need > len(widths) * 162 * 162, (need, widths)
