#!/usr/bin/env python3
"""Builds tests/golden/unproject_gradients.npz: the answers of the restatement in tests/unproject_np.py (on the
compiled reference, oracle/_ref) to the calls tests/test_unproject_gradients_gpu.py and tests/test_model_analysis_gpu.py
make of it, so that those tests compare against the reference where oracle/_ref is not built. Needs oracle/_ref:

    make -C oracle ref && python tests/golden/make_unproject_golden.py

Keys: "<key of the call>/in": the fingerprint of its arguments (the sum and the sum of squares of each numeric one);
"<key>/out<k>": its answers in full."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import test_model_analysis_gpu as A  # noqa: E402
import test_unproject_gradients_gpu as T  # noqa: E402

OUT = os.path.join(HERE, "unproject_gradients.npz")


def main():
    store = {}
    R = T.Restatement()
    for module in (T, A):
        for key, method, args in module.reference_calls():
            store[f"{key}/in"] = T.fingerprint(args)
            for k, a in enumerate(R.call(key, method, *args)):
                store[f"{key}/out{k}"] = np.asarray(a, np.float64)
    np.savez_compressed(OUT, **store)
    print(OUT, len(store), "arrays", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
