#!/usr/bin/env python3
"""Warm device timings of the dense Cholesky: the factorization (net of the refill with an SPD matrix that every call
needs; the persistent kernel up to n = 8192, the multi-kernel chain above) and the persistent backward substitution of
one right-hand side. One line per size, then one JSON line
with the card's name, power limit and SM clocks, read in the same run. usage: time_cholesky.py n [n...]"""
import sys
sys.path.insert(0, ".")
from mrcal_b200 import _capi
import measure
f = _capi.lib.mrcal_b200_debug_time_cholesky


res = {}
for n in [int(a) for a in sys.argv[1:]] or [1268, 4820]:
    factor, backward = f(n, 10, 0), f(n, 20, 1)
    assert factor > 0 and backward > 0, f"n={n}: the timing aid failed"
    gf = n ** 3 / 3 / 1e9
    print(f"n={n}: factorization {factor:.3f} ms ({gf / factor:.1f} TFLOP/s, GFLOP={gf:.2f}); backward substitution {backward:.4f} ms")
    res[n] = {"factor_ms": round(factor, 4), "backward_ms": round(backward, 5)}
measure.emit({"cholesky": res})
