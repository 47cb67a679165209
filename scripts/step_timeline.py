#!/usr/bin/env python3
"""Per-step device timeline of one BASELINE solve (default config 3).

    python scripts/step_timeline.py [--config 3] [--max-iterations 300] [--out DIR]

The solve runs once unprofiled (3 repeats, the library's own ms_total) and once under torch.profiler with CUDA
activities. The trace is cut at the host's waits (cudaStreamSynchronize): one interval is everything the host enqueued
between two waits, i.e. one trust-region step in a solver that waits once per step. For each interval:

  span       from the end of the device work the previous wait returned on to the end of this interval's last operation
  busy       the union of the interval's kernels, memsets and copies (all streams)
  idle_wait  the gap between the previous interval's last operation and this interval's first one: the host's wake-up,
             decision and first launch
  idle_in    the other idle time inside the interval, split by the phase of the operation that ends the gap
  ops        the number of device operations
  enqueue    host time from the previous wait's return to the last launch call of the interval

Also the number of times the launch geometry that follows the size of the reduced system changes, and the typical
step operation by operation (median idle time before each operation and its duration). Prints one JSON line with the
card's name, power limit and SM clocks, read in the same run; the Chrome trace is written to --out (default: a
temporary directory). Tracing slows the host: the unprofiled ms_per_iteration is the number to quote, the profiled gaps
are upper bounds.
"""
import argparse
import json
import os
import re
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# operation name -> phase (the order of the patterns matters: first match wins)
PHASES = [
    ("evaluate", r"unpack_state|expand_rotations|fused_boards|sum_norm_partials|eval_"),
    ("prepare", r"item_columns|mark_|marks_|compact_scan|item_offsets|item_prepare"),
    ("assemble", r"groups_panels|tile_plan|tile_slots|schur_|reg_blocks|finish_rhs|augment_rhs|set_diagonal|gather_shared|assemble_"),
    ("cauchy", r"dots_kernel|quadform|sum_partials_to|jv_kernel"),
    ("factor", r"potrf|trsm|syrk|spine|chol"),
    ("solve", r"extract_y|solve_|scatter_compact|inactive_step|backsub|cauchy_decide"),
    ("step", r"select_step|combine_step|decide"),
    ("clear/read-back", r"fill_words|read_back"),
    ("memset", r"^Memset"),
    ("memcpy", r"^Memcpy"),
]
# kernels whose grid follows n_c (the size of the reduced system)
NC_KERNELS = r"finish_rhs|scatter_compact|set_diagonal|trsm|tile_plan|unpack_tiles"


def phase_of(name):
    for ph, pat in PHASES:
        if re.search(pat, name):
            return ph
    return "other"


def analyse(trace):
    ev = trace["traceEvents"]
    dev = [e for e in ev if e.get("ph") == "X" and e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")]
    rt = [e for e in ev if e.get("ph") == "X" and e.get("cat") == "cuda_runtime"]
    launch_ts = {}
    for e in rt:
        c = e.get("args", {}).get("correlation")
        if c is not None:
            launch_ts[c] = (e["ts"], e["ts"] + e["dur"])
    syncs = sorted((e["ts"] + e["dur"]) for e in rt if e["name"] in ("cudaStreamSynchronize", "cudaDeviceSynchronize"))
    if not syncs:
        raise SystemExit("no host waits in the trace")
    ops = []
    for e in dev:
        c = e.get("args", {}).get("correlation")
        if c not in launch_ts:
            continue
        ops.append(dict(t0=e["ts"], t1=e["ts"] + e["dur"], name=e["name"], host=launch_ts[c][0], grid=str(e.get("args", {}).get("grid"))))
    ops.sort(key=lambda o: o["t0"])
    # interval k: launches after wait k-1 returned, up to wait k
    edges = np.array(syncs)
    groups = {}
    for o in ops:
        k = int(np.searchsorted(edges, o["host"]))
        groups.setdefault(k, []).append(o)
    keys = sorted(groups)
    rows = []
    prev_end = None
    geometry, changes = None, 0
    for k in keys:
        g = sorted(groups[k], key=lambda o: o["t0"])
        busy, idle_in = 0.0, {}
        cur0, cur1 = g[0]["t0"], g[0]["t1"]
        for o in g[1:]:
            if o["t0"] > cur1:
                busy += cur1 - cur0
                ph = phase_of(o["name"])
                idle_in[ph] = idle_in.get(ph, 0.0) + (o["t0"] - cur1)
                cur0, cur1 = o["t0"], o["t1"]
            else:
                cur1 = max(cur1, o["t1"])
        busy += cur1 - cur0
        end = max(o["t1"] for o in g)
        start = prev_end if prev_end is not None else g[0]["t0"]
        idle_wait = max(0.0, g[0]["t0"] - prev_end) if prev_end is not None else 0.0
        wait_ret = edges[k - 1] if k > 0 else g[0]["host"]
        enqueue = max(o["host"] for o in g) - wait_ret
        geo = tuple(sorted({(o["name"][:40], o["grid"]) for o in g if re.search(NC_KERNELS, o["name"])}))
        if geo:
            if geometry is not None and geo != geometry:
                changes += 1
            geometry = geo
        # per operation: the idle time before it (against everything that ended before it started) and its duration
        seq, last = [], prev_end
        for o in g:
            gap = max(0.0, o["t0"] - last) if last is not None else 0.0
            seq.append((o["name"][:48], gap, o["t1"] - o["t0"]))
            last = o["t1"] if last is None else max(last, o["t1"])
        rows.append(dict(span=end - start, busy=busy, idle_wait=idle_wait, idle_in=idle_in, ops=len(g), enqueue=enqueue, seq=seq))
        prev_end = end
    return rows, changes


def op_table(rows):
    """The typical step (the most common operation count), operation by operation: median idle time before it and
    median duration, in microseconds"""
    steps = rows[1:-1] if len(rows) > 2 else rows
    counts = {}
    for r in steps:
        counts[r["ops"]] = counts.get(r["ops"], 0) + 1
    n = max(counts, key=counts.get)
    typ = [r["seq"] for r in steps if r["ops"] == n]
    return dict(ops=n, steps=len(typ),
                table=[[typ[0][i][0], round(float(np.median([s[i][1] for s in typ])), 2),
                        round(float(np.median([s[i][2] for s in typ])), 2)] for i in range(n)])


def summarise(rows):
    # the trust-region steps: intervals that contain an evaluation (the first and last are set-up and wind-down)
    steps = rows[1:-1] if len(rows) > 2 else rows
    med = lambda k: float(np.median([r[k] for r in steps]))
    phases = sorted({p for r in steps for p in r["idle_in"]})
    return dict(
        steps=len(steps),
        span_us=med("span"), busy_us=med("busy"), idle_wait_us=med("idle_wait"),
        idle_in_us=float(np.median([sum(r["idle_in"].values()) for r in steps])),
        idle_in_by_phase_us={p: float(np.median([r["idle_in"].get(p, 0.0) for r in steps])) for p in phases},
        ops=med("ops"), enqueue_us=med("enqueue"),
        idle_wait_share=float(np.sum([r["idle_wait"] for r in steps]) / np.sum([r["span"] for r in steps])),
        idle_in_share=float(np.sum([sum(r["idle_in"].values()) for r in steps]) / np.sum([r["span"] for r in steps])),
    )


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--config", type=int, default=3)
    ap.add_argument("--max-iterations", type=int, default=300)
    ap.add_argument("--out", default=None, help="directory for the Chrome trace (default: a temporary one)")
    args = ap.parse_args()

    import torch
    import mrcal_b200
    import bench
    import measure

    kw = bench.problem_inputs(args.config)
    P = mrcal_b200.Problem(**kw)
    P.reset()
    P.optimize(max_iterations=args.max_iterations)   # warm-up: module loads, graphs, the one-time self-check
    plain = []
    for _ in range(3):
        P.reset()
        torch.cuda.synchronize()
        plain.append(P.optimize(max_iterations=args.max_iterations))
    out = args.out or tempfile.mkdtemp(prefix="step_timeline_")
    os.makedirs(out, exist_ok=True)
    P.reset()
    torch.cuda.synchronize()
    # not measure.kernel_ms(): the cut at the host's waits needs the whole trace, host calls included
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        info = P.optimize(max_iterations=args.max_iterations)
        torch.cuda.synchronize()
    path = os.path.join(out, "step_timeline.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    rows, changes = analyse(trace)
    ms_it = [p["ms_total"] / p["Niterations"] for p in plain]
    measure.emit(dict(
        config=args.config, device=torch.cuda.get_device_name(),
        unprofiled=dict(ms_per_iteration=ms_it, Niterations=plain[-1]["Niterations"], Nsyncs=plain[-1]["Nsyncs"],
                        Nevaluations=plain[-1]["Nevaluations"], Nfactorizations=plain[-1]["Nfactorizations"]),
        profiled=dict(intervals=len(rows), Niterations=info["Niterations"], Nsyncs=info["Nsyncs"],
                      nc_geometry_changes=changes, per_step=summarise(rows), typical_step=op_table(rows)),
        trace=path))
    return 0


if __name__ == "__main__":
    sys.exit(main())
