#!/usr/bin/env python3
"""Builds tests/golden/project_reference.npz: the compiled reference's answers (oracle/_ref) to the calls
tests/test_project_gpu.py makes of it, so that those tests compare against the reference where oracle/_ref is
not built. Needs oracle/_ref:

    make -C oracle ref && python tests/golden/make_project_golden.py

Keys: "<test>/<lens model>/<function>/<n-th call of it in the test>/<in|out><k>"; an argument is stored as a
fingerprint (its sum and its sum of squares), an answer in full. For the last call of test_unproject, whose argument
is the unprojection under test, the reference's own unprojection is the argument. The q and dq/dp that
project_with_intrinsics_gradient() returns are those of project() (one function of the reference): only its
dq/dintrinsics is stored."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref  # noqa: E402
from mrcal_b200 import synthetic  # noqa: E402
import test_project_gpu as T  # noqa: E402

OUT = os.path.join(HERE, "project_reference.npz")


def fingerprint(a):
    a = np.asarray(a, np.float64)
    return np.array((a.sum(), (a * a).sum()))


def main():
    store = {}

    def rec(test, lm, fn, k, inputs, outputs):
        outputs = outputs if isinstance(outputs, tuple) else (outputs,)
        for i, a in enumerate(inputs):
            store[f"{test}/{lm}/{fn}/{k}/in{i}"] = fingerprint(a)
        for i, a in enumerate(outputs):
            store[f"{test}/{lm}/{fn}/{k}/out{i}"] = np.asarray(a, np.float64)
        return outputs

    for lm in T.MODELS:
        intr = synthetic.true_intrinsics(lm, 1, np.random.default_rng(0))[0]
        p = T._points(40, 1)
        rec("test_project_matches_reference", lm, "project", 0, (p, intr), ref.project(p, lm, intr, gradients=True))
        q, dq_dp, dq_dintrinsics = ref.project_with_intrinsics_gradient(p, lm, intr)
        rec("test_project_matches_reference", lm, "project_with_intrinsics_gradient", 0, (p, intr), dq_dintrinsics)
        intr = T._unproject_intrinsics(lm)
        p = T._points(40, 2)
        q, = rec("test_unproject", lm, "project", 0, (p, intr), ref.project(p, lm, intr))
        v, = rec("test_unproject", lm, "unproject", 0, (q, intr), ref.unproject(q, lm, intr))
        rec("test_unproject", lm, "project", 1, (v, intr), ref.project(v, lm, intr))
    np.savez_compressed(OUT, **store)
    print(OUT, len(store), "arrays", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
