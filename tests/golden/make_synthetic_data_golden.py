#!/usr/bin/env python3
"""Builds tests/golden/synthetic_data.npz: the synthesis cases of tests/synthetic_data_np.py, each with its inputs and
seed and the reference's answers as the numpy restatement computes them through the compiled reference (oracle/_ref),
so that tests/test_synthetic_data_gpu.py compares against the reference where oracle/_ref is not built. Needs
oracle/_ref:

    make -C oracle ref && python tests/golden/make_synthetic_data_golden.py

Keys, per case "<key>/": the inputs (seed, W, H, spacing, calobject_warp (empty: None), rt_ref_boardcenter,
noiseradius, Nframes, max_oblique_angle_deg (NaN: None), which), the outputs q and Rt_ref_boardref, Ndraws (the number
of uniform draws: chunks * Nframes * 6), rng (a sha256 of np.random.get_state() after the call) and margins
(Ncandidates, 2): for every candidate frame, the smallest distance of a corner's q from the image bounds and
|costh - cos(max_oblique_angle)|."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, "..", ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synthetic_data_np as S  # noqa: E402

OUT = os.path.join(HERE, "synthetic_data.npz")


def inputs(kw):
    """the stored form of a case's inputs"""
    return dict(seed=kw["seed"], W=kw["W"], H=kw["H"], spacing=kw["spacing"],
                calobject_warp=np.zeros(0) if kw["calobject_warp"] is None else kw["calobject_warp"],
                rt_ref_boardcenter=kw["rt_ref_boardcenter"], noiseradius=kw["noiseradius"], Nframes=kw["Nframes"],
                max_oblique_angle_deg=np.nan if kw["max_oblique_angle_deg"] is None else kw["max_oblique_angle_deg"],
                which=S.WHICH.index(kw["which"]))


def main():
    store = {}
    for key, kw in S.cases():
        for k, v in inputs(kw).items():
            store[f"{key}/{k}"] = np.asarray(v)
        q, Rt, margins, Nchunks, digest = S.run_case(kw)
        store.update({f"{key}/q": q, f"{key}/Rt_ref_boardref": Rt, f"{key}/margins": margins,
                      f"{key}/Ndraws": np.asarray(Nchunks * kw["Nframes"] * 6), f"{key}/rng": np.asarray(digest)})
    np.savez_compressed(OUT, **store)
    print(OUT, len(store), "arrays", os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
