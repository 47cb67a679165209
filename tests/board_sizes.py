"""The board-size cases of test_board_sizes_gpu.py and test_board_sizes_cpu.py, and the extended-precision reference of
the reduced normal equations they are checked against.

The board kernels change how they work with the number of corners W*H of a board:
    eval_boards_kernel (eval.cu)       clamp(round_up_32(W*H), 128, 256) threads; above 256 corners several chunks of
                                       corners, which reuse the staging buffer and the per-corner window starts
    fused_boards_kernel (fused_eval.cu) 128 threads, one per corner, for W*H <= 128; K = round_up_4(W*H) rows in its
                                       tensor-pipe products (K - W*H zero rows of padding), 8 (104 K + 2324) bytes of
                                       shared memory; each observation's patch of nk <= 64 knots in 8x8 tiles
Every case here is a small seeded problem (2 cameras, 3-6 frames), so that the dense references stay cheap. Each case
states the coverage it claims; test_board_sizes_cpu.py checks those claims against the compiled reference's Jacobian."""
import numpy as np

from chol_np import LD, cholesky_ld, solve_lower_ld
from mrcal_b200 import synthetic
from problems import SPL2, SPL3

OPENCV8 = "LENSMODEL_OPENCV8"


def spl(order, Nx, Ny, fov):
    return f"LENSMODEL_SPLINED_STEREOGRAPHIC_order={order}_Nx={Nx}_Ny={Ny}_fov_x_deg={fov}"


def eval_threads(nwh):
    """the block size eval.cu's board kernel launches with"""
    return min(max((nwh + 31) // 32 * 32, 128), 256)


def eval_chunks(nwh):
    return -(-nwh // eval_threads(nwh))


def fused_K(nwh):
    return (nwh + 3) & ~3


def fused_smem_bytes(K):
    """dynamic shared memory of fused_boards_kernel for K rows (fused_eval.cu: fused_smem_bytes)"""
    return 8 * (104 * K + 2324)


def make(lensmodel, W, H, seed=1, Nframes=3, core=None, extr=True, warp=True, outlier_frame=False):
    """One problem: 2 cameras, Nframes frames seen by both, W x H boards. core: optimize the intrinsics core (None: the
    default, locked for splined models). outlier_frame: the last frame keeps only its first observation, with every
    corner marked as an outlier, so that nothing constrains that frame"""
    kw, _ = synthetic.make_problem(lensmodel=lensmodel, Ncameras=2, Nframes=Nframes, W=W, H=H, seed=seed,
                                   pixel_noise=0.3, do_optimize_intrinsics_core=core)
    kw["calobject_warp"] = np.array((1e-3, -2e-3))   # away from 0 so that its gradient is exercised
    kw["do_optimize_extrinsics"] = extr
    kw["do_optimize_calobject_warp"] = warp
    if outlier_frame:
        idx = kw["indices_frame_camintrinsics_camextrinsics"]
        last = np.flatnonzero(idx[:, 0] == Nframes - 1)
        keep = np.ones(len(idx), bool)
        keep[last[1:]] = False
        kw["indices_frame_camintrinsics_camextrinsics"] = np.ascontiguousarray(idx[keep])
        obs = np.ascontiguousarray(kw["observations_board"][keep])
        obs[-1, ..., 2] = -1.   # (the observations are sorted by frame: the last is the last frame's)
        kw["observations_board"] = obs
    return kw


# ---- the cost function at the sizes of eval_boards_kernel: (corners, shape) x lens configurations
EVAL_SHAPES = [(10, 10), (16, 8), (12, 11), (16, 16), (13, 20), (20, 20)]
EVAL_LENSES = {"opencv8": (OPENCV8, True),
               "splined3_corelocked": (SPL3, False),
               # the widest row (16 knots, the core, camera, frame, warp): the largest staging stride at 256 threads
               "splined3_core": (SPL3, True)}


def eval_cases():
    """(name, W, H, optimization_inputs)"""
    out = []
    for (W, H) in EVAL_SHAPES:
        for lens, (lm, core) in EVAL_LENSES.items():
            out.append((f"{lens}_{W}x{H}", W, H, make(lm, W, H, core=core)))
    return out


# ---- the fused evaluation. claims: what each case exercises, checked by test_board_sizes_cpu.py
#   pad       K - W*H, the zero rows of the tensor-pipe products
#   fits      8 (104 K + 2324) <= the 112 640 bytes the kernel was limited to before it was sized by K
#   nk        (lo, hi): the knots of the widest observation's patch
#   ncam0     no camera columns (extrinsics locked)     nwarp0   no warp columns
#   outlier_frame   one frame's only observation is all outliers
FUSED = {
    "pad3_5x5": dict(lens=SPL3, W=5, H=5, claims=dict(pad=3)),
    "pad2_7x6": dict(lens=SPL3, W=7, H=6, claims=dict(pad=2)),
    "pad1_9x7": dict(lens=SPL3, W=9, H=7, claims=dict(pad=1)),
    "order2_pad2_7x6": dict(lens=SPL2, W=7, H=6, claims=dict(pad=2)),
    "board100_10x10": dict(lens=SPL3, W=10, H=10, claims=dict(pad=0, fits=True)),
    "largest_fit_14x8": dict(lens=SPL3, W=14, H=8, claims=dict(pad=0, fits=True)),
    # 113 is prime: the smallest board above 112 corners with W, H > 1 is 19x6, whose K = 116 is the K of 113 corners
    "over_19x6": dict(lens=SPL3, W=19, H=6, claims=dict(pad=2, fits=False)),
    "over_11x11": dict(lens=SPL3, W=11, H=11, claims=dict(pad=3, fits=False)),
    "over_16x8": dict(lens=SPL3, W=16, H=8, claims=dict(pad=0, fits=False)),
    "order2_over_11x11": dict(lens=SPL2, W=11, H=11, claims=dict(pad=3, fits=False)),
    "noextr_10x10": dict(lens=SPL3, W=10, H=10, extr=False, claims=dict(ncam0=True)),
    "nowarp_10x10": dict(lens=SPL3, W=10, H=10, warp=False, claims=dict(nwarp0=True)),
    "outlier_frame_10x10": dict(lens=SPL3, W=10, H=10, outlier_frame=True, claims=dict(outlier_frame=True)),
    # dense splines over a narrow field of view: the widest patch fills its last 8x8 tile partly, or reaches 64 knots
    "nk57to63": dict(lens=spl(3, 24, 16, 80), W=10, H=10, seed=0, claims=dict(nk=(57, 63))),
    "nk64": dict(lens=spl(3, 24, 16, 100), W=10, H=10, seed=2, claims=dict(nk=(64, 64))),
    "order2_nk57to63": dict(lens=spl(2, 24, 16, 70), W=10, H=10, seed=1, claims=dict(nk=(57, 63))),
    "order2_nk64": dict(lens=spl(2, 24, 16, 60), W=10, H=10, seed=0, claims=dict(nk=(64, 64))),
}


def fused_case(name):
    c = FUSED[name]
    return make(c["lens"], c["W"], c["H"], seed=c.get("seed", 1), extr=c.get("extr", True), warp=c.get("warp", True),
                outlier_frame=c.get("outlier_frame", False))


# the fallback: a core-locked splined problem whose widest observations touch more than 64 knots
FALLBACK = dict(lens=spl(3, 24, 16, 60), W=10, H=10, seed=0, Nframes=6)
# a solve on the fused path at 121 corners
SOLVE121 = dict(lens=SPL3, W=11, H=11, seed=1, Nframes=4)


def fallback_case():
    c = FALLBACK
    return make(c["lens"], c["W"], c["H"], seed=c["seed"], Nframes=c["Nframes"])


def solve121_case():
    c = SOLVE121
    return make(c["lens"], c["W"], c["H"], seed=c["seed"], Nframes=c["Nframes"])


# ---- what the reference's Jacobian says about a case
def observation_knots(P, kw, J):
    """per board observation: the number of spline knots its rows touch (from J's column pattern; P an oracle Problem)"""
    i0 = P.state_index("intrinsics", 0)
    n = P.num_states_of("intrinsics")
    W, H = P.W, P.H
    rows = 2 * W * H
    Jc = J.tocsr()
    out = []
    for o in range(P.Nobs_board):
        c = np.unique(Jc.indices[Jc.indptr[o * rows]:Jc.indptr[(o + 1) * rows]])
        c = c[(c >= i0) & (c < i0 + n)]
        out.append(len(c) // 2)   # an x and a y control value per knot
    return out


def observation_columns(P, J, what):
    """per board observation: how many of the columns of `what` ("extrinsics", "calobject_warp") its rows touch"""
    n = P.num_states_of(what)
    if n == 0:
        return [0] * P.Nobs_board
    i0 = P.state_index(what) if what == "calobject_warp" else P.state_index(what, 0)
    rows = 2 * P.W * P.H
    Jc = J.tocsr()
    out = []
    for o in range(P.Nobs_board):
        c = Jc.indices[Jc.indptr[o * rows]:Jc.indptr[(o + 1) * rows]]
        out.append(len(np.unique(c[(c >= i0) & (c < i0 + n)])))
    return out


def unconstrained_frames(P, J):
    """frames whose columns of J are all zero"""
    if P.num_states_of("frames") == 0:
        return []
    f0 = P.state_index("frames", 0)
    Jc = J.tocsc()
    return [f for f in range(P.Nframes)
            if not np.any(Jc[:, f0 + 6 * f:f0 + 6 * f + 6].data != 0)]


# ---- the reduced normal equations in extended precision
def normal_ld(J, x):
    """J'J and J'x in np.longdouble, accumulated from J's nonzeros row by row (J sparse)"""
    J = J.tocsr()
    n = J.shape[1]
    H = np.zeros(n * n, dtype=LD)
    g = np.zeros(n, dtype=LD)
    lens = np.diff(J.indptr)
    rows = np.repeat(np.arange(J.shape[0]), lens)
    v = J.data.astype(LD)
    np.add.at(g, J.indices, v * np.asarray(x, dtype=LD)[rows])
    # rows of equal length together: their outer products in one array
    for L in np.unique(lens):
        if L == 0:
            continue
        r = np.flatnonzero(lens == L)
        idx = J.indptr[r][:, None] + np.arange(L)[None, :]
        V, C = v[idx], J.indices[idx].astype(np.int64)
        np.add.at(H, (C[:, :, None] * n + C[:, None, :]).ravel(), (V[:, :, None] * V[:, None, :]).ravel())
    return H.reshape(n, n), g


def eliminated_groups(P):
    """(e0, e1, sizes): the eliminated range of the state and the size of each of its blocks, frames (6) then points (3)"""
    nf, npt = P.num_states_of("frames"), P.num_states_of("points")
    if nf == 0 and npt == 0:
        return P.num_states(), P.num_states(), []
    e0 = P.state_index("frames", 0) if nf else P.state_index("points", 0)
    return e0, e0 + nf + npt, [6] * (nf // 6) + [3] * (npt // 3)


def reduced_reference_ld(J, x, P, lam=0.0):
    """S, g', J'x (float64) and the scale of S's accuracy: the normal equations accumulated in np.longdouble, each frame's
    (and point's) block eliminated by its longdouble Cholesky factor. Groups that nothing constrains (zero rows of J'J:
    a frame seen only through outliers, at lambda = 0) drop out, as problems.reduced_reference leaves them out"""
    H, g = normal_ld(J, x)
    n = H.shape[0]
    H[np.arange(n), np.arange(n)] += LD(lam)
    e0, e1, sizes = eliminated_groups(P)
    sh = np.r_[0:e0, e1:n]
    A = H[np.ix_(sh, sh)].copy()
    gs = g[sh].copy()
    k = e0
    for s in sizes:
        el = np.arange(k, k + s)
        k += s
        if not np.any(H[el] != 0):
            continue
        Lg = cholesky_ld(H[np.ix_(el, el)])
        Y = solve_lower_ld(Lg, H[np.ix_(el, sh)])   # L^-1 B'
        z = solve_lower_ld(Lg, g[el])
        A -= Y.T @ Y
        gs -= Y.T @ z
    scale = float(np.abs(H[np.ix_(sh, sh)]).max()) if len(sh) else 1.
    return A.astype(np.float64), gs.astype(np.float64), g.astype(np.float64), scale


def cauchy_reference_ld(J, x):
    """(|g|^2, |J g|^2), g = J'x, in np.longdouble"""
    J = J.tocsr()
    v = J.data.astype(LD)
    rows = np.repeat(np.arange(J.shape[0]), np.diff(J.indptr))
    g = np.zeros(J.shape[1], dtype=LD)
    np.add.at(g, J.indices, v * np.asarray(x, dtype=LD)[rows])
    Jg = np.zeros(J.shape[0], dtype=LD)
    np.add.at(Jg, rows, v * g[J.indices])
    return float(g @ g), float(Jg @ Jg)
