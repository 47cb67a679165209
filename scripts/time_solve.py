"""Time solve_xt_JtJ_bt() over the number of right-hand sides, for the factors the library makes: the structured factor
optimizer_callback() returns at BASELINE configs 3 and 5, and the dense CHOLMOD_factorization(J) of a random sparse J
(built as tests/test_factorization_gpu.py's test_random_sparse builds it) at n = 1100 and n = 8300.

For each factor, sys in (A, L, Lt) and nrhs: the median wall time of a call (every call ends in a device
synchronisation; it includes the copies of the right-hand sides both ways), after a warm-up call, and the device time
of the call's kernels from torch.profiler in a separate call. One JSON line per point, each with the card's name, power
limit and SM clocks, read as that point is written. --out also writes the lines to a file."""
import argparse
import os
import sys

import numpy as np
import scipy.sparse

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mrcal_b200  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402
import measure  # noqa: E402

NRHS = (1, 2, 8, 32, 64, 128, 256, 512, 3960)
SYSTEMS = ("A", "L", "Lt")
FACTORS = ("config3", "config5", "dense1100", "dense8300")


def make_factor(name):
    if name.startswith("config"):
        kw, _ = synthetic.baseline_config(int(name[len("config"):]), pixel_noise=0.3, seed=0)
        _, _, J, F = mrcal_b200.optimizer_callback(**kw)
        return F, J.shape[1]
    n, m, density = {"dense1100": (1100, 9000, 0.01), "dense8300": (8300, 9000, 0.0005)}[name]
    J = scipy.sparse.random(m, n, density=density, random_state=np.random.RandomState(n), format="csr")
    J = (J + scipy.sparse.vstack([scipy.sparse.eye(n) * 0.5, scipy.sparse.csr_matrix((m - n, n))])).tocsr()
    return mrcal_b200.CHOLMOD_factorization(J), n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--factors", default=",".join(FACTORS))
    ap.add_argument("--nrhs", default=",".join(map(str, NRHS)))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if args.out:
        open(args.out, "w").close()   # emit() appends each point's line
    nrhs_all = [int(v) for v in args.nrhs.split(",")]
    for fname in args.factors.split(","):
        F, n = make_factor(fname)
        bt_all = np.random.default_rng(0).normal(size=(max(nrhs_all), n))
        for sys_ in SYSTEMS:
            for nrhs in nrhs_all:
                bt = bt_all[:nrhs]

                def call():
                    return F.solve_xt_JtJ_bt(bt, sys=sys_)
                # the warm-up call is timed too, to take fewer repetitions of slow calls
                first = measure.median_ms(call, 1, warmup=0)
                ms_call = measure.median_ms(call, 7 if first < 50 else (3 if first < 1000 else 1), warmup=0)
                # every kernel of the library is named *_kernel; the copies of the right-hand sides are left out
                measure.emit(dict(factor=fname, n=n, sys=sys_, nrhs=nrhs, ms_call=round(ms_call, 4),
                                  ms_kernels=round(measure.kernel_ms(call, "_kernel"), 4)), args.out)
        del F


if __name__ == "__main__":
    main()
