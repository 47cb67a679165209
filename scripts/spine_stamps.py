#!/usr/bin/env python3
"""Where the spine of the persistent Cholesky (chol_dataflow.cu:chol_spine_kernel) spends its time, per 64-column step."""
import sys
sys.path.insert(0, ".")
import numpy as np
from mrcal_b200 import _capi
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1270
nb = (n + 63) // 64
out = np.zeros(8 * nb, np.int64)
assert _capi.lib.mrcal_b200_debug_spine_stamps(n, out.ctypes.data, out.size)
st = out.reshape(nb, 8)
t0 = st[0, 0]
print("step  start   trsm  diag-ready  potrf  loads-issued  written  step-end | next ready   (cycles; deltas)")
for d in range(nb):
    r = st[d]
    print("%3d %8d %6d %6d %7d %6d %7d %7d | %d" % (d, r[0] - t0, r[1] - r[0] if d else 0, r[2] - (r[1] if d else r[0]), r[3] - r[2], r[4] - r[3], r[5] - r[4], r[6] - r[5], r[7]))
print("total cycles", st[-1, 6] - t0, " mean per step", (st[-1, 6] - t0) / nb)
