"""What the timing scripts share: the card a number is measured on, the median time of a call, the device time of named
kernels, and the one JSON line a script prints. The scripts run as `python scripts/x.py` and `import measure`."""
import json
import subprocess
import time

import numpy as np
import torch


def card():
    """The name, power limit, current SM clock and maximum SM clock of the device in use, read now with an nvidia-smi
    query. Raises if there is no CUDA device or the query fails: a number without its card is not reported."""
    if not torch.cuda.is_available():
        raise RuntimeError("no CUDA device: there is nothing to measure on")
    # by UUID: nvidia-smi numbers the devices without regard to CUDA_VISIBLE_DEVICES
    uuid = torch.cuda.get_device_properties(torch.cuda.current_device()).uuid
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader",
                          "-i", f"GPU-{uuid}"], capture_output=True, text=True, timeout=30, check=True).stdout
    name, power_limit, sm_clock, max_sm_clock = (s.strip() for s in out.strip().split(","))
    return dict(card=name, power_limit=power_limit, sm_clock=sm_clock, max_sm_clock=max_sm_clock)


def median_ms(f, reps, warmup=1):
    """Median host time in ms of `reps` calls of f, each ended by a device synchronisation, after `warmup` untimed
    calls"""
    for _ in range(warmup):
        f()
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        torch.cuda.synchronize()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t))


def kernel_ms(f, *names):
    """Device time in ms, from torch.profiler, of the kernels and copies whose names contain any of `names`, over one
    call of f. f runs once before, so that module loads and first-call set-up stay out of the profiled window."""
    f()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    us = [e.device_time_total for e in prof.events() if any(n in e.name for n in names)]
    if not us:
        raise RuntimeError(f"no kernel named like {names} ran")
    return sum(us) / 1e3


def emit(result, out=None):
    """Print `result` with the card() fields as one JSON line; with `out`, also append the line to that file"""
    line = json.dumps({**result, **card()})
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")
