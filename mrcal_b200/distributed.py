"""Multi-GPU solves: one process per GPU, the frames (and the discrete points)
sharded across ranks, the shared unknowns (all intrinsics, all extrinsics, the
board warp) replicated.

Per trust-region iteration every rank evaluates and assembles its own frames,
eliminates them locally (Schur complement), and ONE NCCL all-reduce sums the
reduced normal equations (plus a few scalars); every rank then factors the same
reduced system and back-substitutes its own frames (SURVEY.md 8e). The
collective itself is issued by libmrcal_b200.so on the solver's stream;
torch.distributed is only the plumbing that carries the NCCL unique id between
the processes and gathers the per-rank frame poses at the end.

    kw_local, shard = shard_inputs(kw, rank, world)
    init_comm(rank, world, local_rank)          # once per process, after dist.init_process_group()
    P = mrcal_b200.Problem(**kw_local); attach(P, shard)
    stats = P.optimize()
    solution = gather_solution(P, shard)        # full-size arrays on every rank
"""
import ctypes as C
import glob
import os

import numpy as np

from ._capi import checked


def _frame_ranges(Nframes, world):
    edges = [(Nframes * r) // world for r in range(world + 1)]
    return [(edges[r], edges[r + 1]) for r in range(world)]


def shard_inputs(kw, rank, world):
    """This rank's slice of a full optimization_inputs dict. Frames are split into
    contiguous ranges (the board observations are already sorted by frame,
    mrcal-pywrap.c:1063-1127); non-fixed points likewise; fixed points and their
    observations stay on rank 0. Regularization stays on in every rank (the rows are
    replicated, and counted once: the library makes rank 0 their owner)."""
    Nframes = 0 if kw.get("rt_ref_frame") is None else kw["rt_ref_frame"].shape[0]
    if Nframes and world > Nframes:
        raise RuntimeError(f"cannot shard {Nframes} frames over {world} ranks")
    out = dict(kw)
    shard = dict(rank=rank, world=world, Nframes=Nframes, f0=0, f1=Nframes, p0=0, p1=0, Npoints=0)
    if Nframes:
        f0, f1 = _frame_ranges(Nframes, world)[rank]
        idx = kw["indices_frame_camintrinsics_camextrinsics"]
        sel = (idx[:, 0] >= f0) & (idx[:, 0] < f1)
        loc = idx[sel].copy()
        loc[:, 0] -= f0
        out["indices_frame_camintrinsics_camextrinsics"] = np.ascontiguousarray(loc)
        out["observations_board"] = np.ascontiguousarray(kw["observations_board"][sel])
        out["rt_ref_frame"] = np.ascontiguousarray(kw["rt_ref_frame"][f0:f1])
        shard.update(f0=f0, f1=f1, board_sel=sel)
    pts = kw.get("points")
    if pts is not None and pts.shape[0]:
        Npf = int(kw.get("Npoints_fixed", 0) or 0)
        Nvar = pts.shape[0] - Npf
        p0, p1 = _frame_ranges(Nvar, world)[rank] if Nvar else (0, 0)
        ip = kw["indices_point_camintrinsics_camextrinsics"]
        sel = (ip[:, 0] >= p0) & (ip[:, 0] < p1)
        loc = ip[sel].copy()
        loc[:, 0] -= p0
        obs = kw["observations_point"][sel]
        points = pts[p0:p1]
        if rank == 0 and Npf:
            self_fixed = ip[:, 0] >= Nvar
            locf = ip[self_fixed].copy()
            locf[:, 0] = locf[:, 0] - Nvar + (p1 - p0)
            loc = np.concatenate((loc, locf))
            obs = np.concatenate((obs, kw["observations_point"][self_fixed]))
            points = np.concatenate((points, pts[Nvar:]))
            out["Npoints_fixed"] = Npf
        else:
            out["Npoints_fixed"] = 0
        if points.shape[0] == 0:
            for k in ("points", "indices_point_camintrinsics_camextrinsics", "observations_point", "Npoints_fixed"):
                out.pop(k, None)
        else:
            out["points"] = np.ascontiguousarray(points)
            out["indices_point_camintrinsics_camextrinsics"] = np.ascontiguousarray(loc.astype(np.int32))
            out["observations_point"] = np.ascontiguousarray(obs)
        shard.update(p0=p0, p1=p1, Npoints=pts.shape[0], Npoints_variable=Nvar)
    # the selections must not depend on what happens to exist on one rank
    for name, default in (("do_optimize_intrinsics_core", True), ("do_optimize_intrinsics_distortions", True),
                          ("do_optimize_extrinsics", kw.get("rt_cam_ref") is not None and kw["rt_cam_ref"].shape[0] > 0),
                          ("do_optimize_frames", Nframes > 0),
                          ("do_optimize_calobject_warp", kw.get("observations_board") is not None)):
        if out.get(name) is None:
            out[name] = default
    # outlier rejection works sharded (the statistics and the "found" flag are all-reduced, outliers.cu); the
    # default must be spelled out so that every rank takes the same path
    if out.get("do_apply_outlier_rejection") is None:
        out["do_apply_outlier_rejection"] = True
    for k in ("intrinsics", "rt_cam_ref", "calobject_warp"):
        if out.get(k) is not None:
            out[k] = out[k].copy()
    return out, shard


def _find_nccl():
    try:
        import torch
        base = os.path.dirname(os.path.dirname(torch.__file__))
        hits = glob.glob(os.path.join(base, "nvidia", "nccl", "lib", "libnccl.so*"))
        if hits:
            return sorted(hits)[0]
    except Exception:
        pass
    return None


def init_comm(rank, world, local_rank):
    """Create the library's NCCL communicator. The unique id is made by rank 0 and
    broadcast with torch.distributed (any initialised backend)."""
    import torch
    import torch.distributed as dist
    if "MRCAL_B200_NCCL_LIB" not in os.environ:
        p = _find_nccl()
        if p:
            os.environ["MRCAL_B200_NCCL_LIB"] = p
    buf = (C.c_char * 128)()
    if rank == 0:
        checked.mrcal_b200_nccl_get_unique_id(buf)
    dev = torch.device("cuda", local_rank) if dist.get_backend() == "nccl" else torch.device("cpu")
    t = torch.frombuffer(bytearray(bytes(buf)), dtype=torch.uint8).clone().to(dev)
    dist.broadcast(t, src=0)
    raw = bytes(t.cpu().numpy().tobytes())
    checked.mrcal_b200_nccl_comm_init(raw, rank, world, local_rank)


def attach(problem, shard):
    checked.mrcal_b200_problem_set_sharding(problem._h, shard["f0"], shard["Nframes"], shard["p0"],
                                            shard.get("Npoints", 0))


def gather_solution(problem, shard):
    """Full-size solution arrays on every rank: shared unknowns from the local copy
    (identical on all ranks), frame poses and points all-gathered."""
    import torch
    import torch.distributed as dist
    out = problem.download(into_inputs=False)
    dev = torch.device("cuda") if dist.get_backend() == "nccl" else torch.device("cpu")

    def allgather_rows(a):
        n = torch.tensor([a.shape[0]], device=dev)
        ns = [torch.zeros_like(n) for _ in range(shard["world"])]
        dist.all_gather(ns, n)
        m = int(max(x.item() for x in ns))
        pad = np.zeros((m,) + a.shape[1:])
        pad[:a.shape[0]] = a
        t = torch.from_numpy(pad).to(dev)
        ts = [torch.zeros_like(t) for _ in range(shard["world"])]
        dist.all_gather(ts, t)
        return np.concatenate([ts[r].cpu().numpy()[:int(ns[r].item())] for r in range(shard["world"])])

    res = dict(intrinsics=out["intrinsics"], rt_cam_ref=out["rt_cam_ref"], calobject_warp=out["calobject_warp"])
    if shard["Nframes"]:
        res["rt_ref_frame"] = allgather_rows(out["rt_ref_frame"])
    if shard.get("Npoints", 0):
        pts = out["points"] if out["points"] is not None else np.zeros((0, 3))
        nloc = shard["p1"] - shard["p0"]
        var = allgather_rows(pts[:nloc])
        fixed = allgather_rows(pts[nloc:])   # only rank 0 has any
        res["points"] = np.concatenate((var, fixed))
    return res
