"""Time projection_uncertainty() at BASELINE config 3 on the default grid of the uncertainty-plotting tool (60 wide,
height in proportion: 60 x 33 on 4000 x 2200), against the route the reference's Python takes composed from this
library's primitives: solve_xt_JtJ_bt() on the dense (2N, Nstate) rows, then one _A_Jt_J_At() per point. Prints one
JSON line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mrcal_b200  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402
import measure  # noqa: E402


def main():
    kw, _ = synthetic.baseline_config(3, pixel_noise=0.3, seed=0)
    mrcal_b200.optimize(**kw)
    icam = 1
    W, H = kw["imagersizes"][icam]
    qx, qy = np.meshgrid(np.linspace(0, W - 1, 60), np.linspace(0, H - 1, 33))
    v = mrcal_b200.unproject(np.stack((qx, qy), -1), kw["lensmodel"], kw["intrinsics"][icam])
    v = (v / np.linalg.norm(v, axis=-1)[..., None]).reshape(-1, 3)
    P = mrcal_b200.Problem(**kw)
    res = {}
    for name, method, pts, inf in (("ccp_10m", "cross-reprojection-ccp", 10. * v, False),
                                   ("ccp_infinity", "cross-reprojection-ccp", v, True),
                                   ("mean_pcam_10m", "mean-pcam", 10. * v, False)):
        res[f"ms_device_{name}"] = measure.median_ms(
            lambda: P.projection_uncertainty(pts, icam, method=method, atinfinity=inf), 5)

    # the composed route. Its cost does not depend on the values of the rows, so they are random here
    b, x, J, F = mrcal_b200.optimizer_callback(**kw)
    Nstate = J.shape[1]
    Nlead = mrcal_b200.num_measurements_boards(**kw) + mrcal_b200.num_measurements_points(**kw)
    rows = np.random.default_rng(0).normal(size=(v.shape[0], 2, Nstate))

    def composed():
        X = F.solve_xt_JtJ_bt(rows)
        return mrcal_b200._A_Jt_J_At__2(X, J.indptr, J.indices, J.data, Nleading_rows_J=Nlead)
    res["ms_composed_primitives"] = measure.median_ms(composed, 1)   # seconds per call: one warm-up, one timed call

    Nrhs = 2 * v.shape[0]
    Nelim = mrcal_b200.num_states_frames(**kw) + mrcal_b200.num_states_points(**kw)
    n_s = Nstate - Nelim
    res.update(Nrhs=Nrhs, Nstate=Nstate, n_shared=n_s,
               # L_S forward + backward (n^2 each per right-hand side) + the forward panels (at most 2 Nelim n_s each)
               gflop_solve=Nrhs * (2. * n_s * n_s + 2. * Nelim * n_s) / 1e9)
    measure.emit(res)


if __name__ == "__main__":
    main()
