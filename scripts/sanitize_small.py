#!/usr/bin/env python3
"""A small end-to-end exercise of every kernel family, meant to be run under compute-sanitizer
(memcheck / racecheck / synccheck): callback, solve (persistent Cholesky, potrf_block, Schur, assembly),
factorization object, the dense Cholesky kernels on their own, project/unproject, triangulated points."""
import sys
sys.path.insert(0, ".")
sys.path.insert(0, "tests")
import numpy as np
import mrcal_b200
from mrcal_b200 import synthetic
import problems

cases = dict(problems.golden_cases())
for name in ("opencv8_points_fixed", "splined3_2cam_corelocked", "tri_opencv4_boards_points", "cahvore_points"):
    kw = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in cases[name].items()}
    b, x, J, F = mrcal_b200.optimizer_callback(**kw)
    if F is not None:
        F.solve_xt_JtJ_bt(np.ones((3, J.shape[1])), sys="L")
    kw["do_apply_outlier_rejection"] = False
    r = mrcal_b200.optimize(**kw)
    print(name, "rms", r["rms_reproj_error__pixels"])
kw, _ = synthetic.make_problem(lensmodel="LENSMODEL_SPLINED_STEREOGRAPHIC_order=3_Nx=8_Ny=6_fov_x_deg=100", Ncameras=2, Nframes=12,
                               W=6, H=5, seed=2, pixel_noise=0.2)
P = mrcal_b200.Problem(**kw)
print("solve", P.optimize(max_iterations=6)["Niterations"])
for icam in (-1, 1):
    print("drt_cross_reprojection__dbpacked", icam, np.abs(mrcal_b200.drt_cross_reprojection__dbpacked(icam_intrinsics=icam, **kw)).max())
# the dense Cholesky kernels directly (tests/test_cholesky_gpu.py's entry points): the spine kernel at 1 to 4 blocks
# (its helper CTAs and pre tasks from 3 on, potrf_block's named barriers in every step), the blocked factorization,
# and the solves of chol_solve() (both kernel families) and chol_solve_backward()
import chol_np
import test_cholesky_gpu as tc
for n, path in ((64, 1), (128, 1), (192, 1), (250, 1), (250, 2)):
    f = tc.factor(chol_np.spd_cond(n, 1e2, np.random.default_rng(n)), path)
    B = np.random.default_rng(0).normal(size=(3, f.L.shape[0]))
    for kernel in (1, 2):
        tc.solve(f.L, f.invL, n, B, 3, kernel)
    tc.solve(f.L, f.invL, n, B[:1], 2, 3)
    print("cholesky", n, "path", f.path, "grid", f.grid, "info", f.info)
intr = synthetic.true_intrinsics("LENSMODEL_OPENCV8", 1, np.random.default_rng(0))[0]
q = mrcal_b200.project(np.array(((0.1, 0.2, 2.), (-.3, .1, 3.))), "LENSMODEL_OPENCV8", intr)
print("unproject", mrcal_b200.unproject(q, "LENSMODEL_OPENCV8", intr))
