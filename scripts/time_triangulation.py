"""Time the triangulation routines on CUDA tensors: triangulate_leecivera_mid2() with one broadcast t01 and
triangulate_lindstrom() with one broadcast Rt01, over 10^6 and 10^7 ray pairs, with and without gradients; and, for
comparison, the call time of the numpy path (upload, kernel, download) of mid2 at 10^6 pairs. Each: the kernel time
from torch.profiler, the bytes the kernel must move (computed from the shapes: every input element read once, every
output element written once) and the achieved bandwidth against the H100 SXM data-sheet 3.35 TB/s. Prints one JSON
line with the card's name, power limit and SM clocks, read in the same run."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import mrcal_b200  # noqa: E402
import measure  # noqa: E402

PEAK_GBS = 3350.


def kernel(f, nbytes, **info):
    ms = measure.kernel_ms(f, "triangulation_kernel")
    return dict(ms_kernel=ms, bytes=nbytes, GBs=nbytes / ms / 1e6, share_of_datasheet=nbytes / ms / 1e6 / PEAK_GBS,
                **info)


def main():
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    t = torch.tensor([1., 0.1, -0.2], dtype=torch.float64, device=dev)
    Rt = torch.cat((torch.eye(3, dtype=torch.float64, device=dev), t[None]))
    out = {}
    for N in (10**6, 10**7):
        p = torch.randn(N, 3, dtype=torch.float64, device=dev, generator=g) * 0.5 + \
            torch.tensor([0., 0, 10], dtype=torch.float64, device=dev)
        v0 = p + torch.randn(N, 3, dtype=torch.float64, device=dev, generator=g) * 1e-3
        v1 = p - t + torch.randn(N, 3, dtype=torch.float64, device=dev, generator=g) * 1e-3
        for name, f, tin, gout in (("leecivera_mid2", mrcal_b200.triangulate_leecivera_mid2, t, 27),
                                   ("lindstrom", mrcal_b200.triangulate_lindstrom, Rt, 54)):
            out[f"{name}_{N:.0e}"] = kernel(lambda: f(v0, v1, tin), 8 * (tin.numel() + N * 6 + N * 3), N=N)
            out[f"{name}_gradients_{N:.0e}"] = kernel(lambda: f(v0, v1, tin, get_gradients=True),
                                                      8 * (tin.numel() + N * 6 + N * (3 + gout)), N=N)
        del p, v0, v1
        torch.cuda.empty_cache()
    rng = np.random.default_rng(2)
    pn = rng.normal(size=(10**6, 3)) * 0.5 + [0, 0, 10]
    tn = t.cpu().numpy()
    v0n, v1n = pn + rng.normal(size=pn.shape) * 1e-3, pn - tn + rng.normal(size=pn.shape) * 1e-3
    out["leecivera_mid2_numpy_1e+06"] = dict(ms_call=measure.median_ms(
        lambda: mrcal_b200.triangulate_leecivera_mid2(v0n, v1n, tn), 10), N=10**6)
    measure.emit(out, os.environ.get("TIME_TRIANGULATION_OUT"))


if __name__ == "__main__":
    main()
