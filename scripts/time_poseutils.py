"""Time the pose utilities on CUDA tensors: transform_point_rt() of one rt applied to 10^6, 10^7 and 10^8 points, with
and without gradients; compose_rt() with gradients over 10^7 pose pairs; R_from_r() with gradients over 10^7 vectors;
and, for comparison, the call time of the numpy path (upload, kernel, download) at 10^6 points. Each: the kernel time
from torch.profiler, the bytes the kernel must move (computed from the shapes: every input element read once, every
output element written once) and the achieved bandwidth against the H100 SXM data-sheet 3.35 TB/s. The last elements
of the largest case are checked against the numpy path. Prints one JSON line with the card's name, power limit and SM
clocks, read in the same run."""
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
    ms = measure.kernel_ms(f, "poseutils_kernel")
    return dict(ms_kernel=ms, bytes=nbytes, GBs=nbytes / ms / 1e6, share_of_datasheet=nbytes / ms / 1e6 / PEAK_GBS,
                **info)


def main():
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(1)
    rt = torch.tensor([0.3, -1.2, 2.0, 1., 2., 3.], dtype=torch.float64, device=dev)
    out = {}
    for N in (10**6, 10**7, 10**8):
        x = torch.randn(N, 3, dtype=torch.float64, device=dev, generator=g)
        y = torch.empty(N, 3, dtype=torch.float64, device=dev)
        out[f"transform_point_rt_{N:.0e}"] = kernel(lambda: mrcal_b200.transform_point_rt(rt, x, out=y),
                                                    8 * (6 + N * 3 + N * 3), N=N)
        if N == 10**8:
            # 3 + 18 + 9 doubles of output per point: 3e9 doubles, more than 2^31
            outs = (y, torch.empty(N, 3, 6, dtype=torch.float64, device=dev),
                    torch.empty(N, 3, 3, dtype=torch.float64, device=dev))
        else:
            outs = None
        out[f"transform_point_rt_gradients_{N:.0e}"] = kernel(
            lambda: mrcal_b200.transform_point_rt(rt, x, get_gradients=True, out=outs), 8 * (6 + N * 3 + N * 30), N=N)
        if N == 10**8:
            idx = torch.arange(N - 1000, N, device=dev)
            want = mrcal_b200.transform_point_rt(rt.cpu().numpy(), x[idx].cpu().numpy(), get_gradients=True)
            for k in range(3):
                assert np.array_equal(outs[k][idx].cpu().numpy(), want[k]), f"output {k} of the last elements"
            out["last_elements_match_numpy_path"] = True
            del outs
        del x, y
        torch.cuda.empty_cache()
    N = 10**7
    rt0 = torch.randn(N, 6, dtype=torch.float64, device=dev, generator=g)
    rt1 = torch.randn(N, 6, dtype=torch.float64, device=dev, generator=g)
    out["compose_rt_gradients_1e+07"] = kernel(lambda: mrcal_b200.compose_rt(rt0, rt1, get_gradients=True),
                                               8 * N * (6 + 6 + 6 + 36 + 36), N=N)
    out["R_from_r_gradients_1e+07"] = kernel(lambda: mrcal_b200.R_from_r(rt0[:, :3], get_gradients=True),
                                             8 * N * (3 + 9 + 27), N=N)
    del rt0, rt1
    xn = np.random.default_rng(2).normal(size=(10**6, 3))
    rtn = rt.cpu().numpy()
    out["transform_point_rt_numpy_1e+06"] = dict(ms_call=measure.median_ms(
        lambda: mrcal_b200.transform_point_rt(rtn, xn), 10), N=10**6)
    measure.emit(out, os.environ.get("TIME_POSEUTILS_OUT"))


if __name__ == "__main__":
    main()
