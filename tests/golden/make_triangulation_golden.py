#!/usr/bin/env python3
"""Builds tests/golden/triangulation.npz: the inputs of the triangulation cases of tests/triangulation_np.py and the
answers of the compiled reference (oracle/_ref) to them, so that tests/test_triangulation_gpu.py compares against the
reference where oracle/_ref is not built. Needs oracle/_ref:

    make -C oracle ref && python tests/golden/make_triangulation_golden.py

Keys: "<key of the case>/in<k>": its inputs; "<key>/out<k>": the reference's answers."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import triangulation_np as T  # noqa: E402

OUT = os.path.join(HERE, "triangulation.npz")


def main():
    store = {}
    for key, fname, args, g in T.cases():
        for k, a in enumerate(args):
            store[f"{key}/in{k}"] = np.asarray(a, np.float64)
        for k, a in enumerate(T.reference(fname, args, g)):
            store[f"{key}/out{k}"] = np.asarray(a, np.float64)
    np.savez_compressed(OUT, **store)
    print(OUT, len(store), "arrays", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
