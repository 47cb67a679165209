"""Time solve_xt_JtJ_bt() over the number of right-hand sides, for the factors the library makes: the structured factor
optimizer_callback() returns at BASELINE configs 3 and 5, and the dense CHOLMOD_factorization(J) of a random sparse J
(built as tests/test_factorization_gpu.py's test_random_sparse builds it) at n = 1100 and n = 8300.

For each factor, sys in (A, L, Lt) and nrhs: the median wall time of a call (every call ends in a device
synchronisation; it includes the copies of the right-hand sides both ways), after a warm-up call, and the device time
of the call's kernels from torch.profiler in a separate call. One JSON line per point, then one with the card's name
and power limit, read in the same run. --out also writes the lines to a file."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import mrcal_b200  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402

NRHS = (1, 2, 8, 32, 64, 128, 256, 512, 3960)
SYSTEMS = ("A", "L", "Lt")
FACTORS = ("config3", "config5", "dense1100", "dense8300")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception:
        return "unknown", "unknown"


def timed(f):
    """median ms of a call after a warm-up; fewer repetitions for slow calls"""
    t0 = time.perf_counter()
    f()
    first = time.perf_counter() - t0
    reps = 7 if first < 0.05 else (3 if first < 1. else 1)
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t))


def kernel_ms(f):
    """device time of the kernels of one call of f, from torch.profiler"""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.events() if not e.name.startswith(("Memcpy", "Memset")))
    return us / 1e3


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
    lines = []

    def emit(d):
        print(json.dumps(d), flush=True)
        lines.append(json.dumps(d))

    torch.zeros(1, device="cuda")   # the profiler's CUDA context
    nrhs_all = [int(v) for v in args.nrhs.split(",")]
    for fname in args.factors.split(","):
        F, n = make_factor(fname)
        bt_all = np.random.default_rng(0).normal(size=(max(nrhs_all), n))
        for sys_ in SYSTEMS:
            for nrhs in nrhs_all:
                bt = bt_all[:nrhs]

                def call():
                    return F.solve_xt_JtJ_bt(bt, sys=sys_)
                emit(dict(factor=fname, n=n, sys=sys_, nrhs=nrhs, ms_call=round(timed(call), 4),
                          ms_kernels=round(kernel_ms(call), 4)))
        del F
    name, limit = card()
    emit(dict(card=name, power_limit=limit))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
