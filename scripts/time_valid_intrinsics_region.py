"""Time the valid-intrinsics regions at BASELINE config 3 (4 splined cameras, 400 frames, solved): every camera's
region from valid_intrinsics_regions() (one evaluation and one factorization for all of them) against a loop of
_compute_valid_intrinsics_region() over the cameras (one each), as mrcal-calibrate-cameras runs it, with the tool's
default parameters and the 30-wide grid. Then the regional-statistics kernel alone, from torch.profiler in a run of
its own. Prints one JSON line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mrcal_b200  # noqa: E402
from mrcal_b200 import regions, synthetic  # noqa: E402
import measure  # noqa: E402


def main():
    kw, _ = synthetic.baseline_config(3, pixel_noise=0.3, seed=0)
    mrcal_b200.optimize(**kw)
    Ncameras = len(kw["intrinsics"])
    models = [mrcal_b200.cameramodel(optimization_inputs=kw, icam_intrinsics=i) for i in range(Ncameras)]
    parameters = (1, 0.5, 1.5, 3, 0)
    s = np.std(mrcal_b200.measurements_board(kw).ravel())
    res = {}
    regs = []
    res["ms_valid_intrinsics_regions_all_cameras"] = measure.median_ms(
        lambda: regs.append(mrcal_b200.valid_intrinsics_regions(kw, parameters)), 3)

    def loop():
        return [mrcal_b200._compute_valid_intrinsics_region(m, s, 0.5, 1.5 * s, 3, 0) for m in models]
    res["ms_compute_valid_intrinsics_region_loop"] = measure.median_ms(loop, 3)
    # what the loop pays on the host per camera before any device work: decoding the model's optimization_inputs
    res["ms_decode_optimization_inputs_per_model"] = measure.median_ms(lambda: models[0].optimization_inputs(), 3)
    res["same_regions"] = all(np.array_equal(a, b) for a, b in zip(regs[-1], loop()))
    res["region_vertices"] = [int(r.shape[0]) if r is not None else None for r in regs[-1]]

    # the statistics kernel alone, all cameras in one launch
    W, H = kw["imagersizes"][0]
    gh = int(round(H / W * 30))
    grids = [regions._cell_grid(kw["imagersizes"][i], 30, gh) for i in range(Ncameras)]
    args = (list(range(Ncameras)), np.array([g[0] for g in grids]), np.array([g[1] for g in grids]))
    P = mrcal_b200.Problem(**kw)
    try:
        P.regional_statistics(*args)   # evaluates the residuals that the calls below reuse
        reps = 20
        res["us_regional_statistics_kernel"] = 1e3 / reps * measure.kernel_ms(
            lambda: [P.regional_statistics(*args, evaluate=False) for _ in range(reps)], "regional_statistics_kernel")
    finally:
        P.close()
    Ncorners = int(kw["observations_board"][..., 0].size)
    res.update(Ncameras=Ncameras, grid=[30, gh], Ncorners=Ncorners,
               # every (camera, cell) CTA reads its camera's corners (24 B of observation, 4 B of index) twice at
               # most; the residuals only of the corners in the cell: the L2 traffic that bounds the kernel
               gbytes_l2_scans=2 * 28. * Ncorners * 30 * gh / 1e9)
    measure.emit(res)


if __name__ == "__main__":
    main()
