"""The cases of test_structured_factor_gpu.py and test_structured_factor_cpu.py: problems whose structured factor
(factorization_schur.cu) takes each path of its solve kernels, what each case claims about its shape, and the
extended-precision reference the factor is checked against.

The factor is  P J'J P' = L L',  L = [L_D 0 0; Y' L_S 0; 0 0 L_I]:
    L_D   the 6x6 (frame) and 3x3 (point) Cholesky factors of the eliminated groups, in group order
    Y'    the panels, one per (group, 64-column block of L_S) that the group reaches
    L_S   the dense factor of the n_c coupled shared unknowns, padded to nblk 64-column blocks. Compact rows n_c and n_c + 1
          carry the solver's right-hand side and become padding in the factor: the padded size is round_up_64(n_c + 2)
    L_I   the 2x2 (spline knot) and 1x1 (distortion, centre pixel) factors of the regularization blocks of the shared
          unknowns that no observation touches
and P orders the unknowns [eliminated (state order) | coupled (state order) | uncoupled (state order)].

Where the kernels change path:
    panels_forward_tiled_kernel   per 64-block, the groups that reach it, 8 per stage, from presence words of 32 groups:
                                  1 group, a full stage (8), a second stage (9), a full word (32), a second word (33),
                                  three words (65); frame groups (6 unknowns) and point groups (3) in one stage. Every
                                  group reaches the block of compact column n_c (the solver's right-hand side)
    clear_aug_rows_kernel         rows n_c, n_c + 1: in one block (n_c = 62), across two (63), both in the next (64, 65)
    chol_solve()                  per-block kernels below 8 nblk right-hand sides, the tiled kernel from 8 nblk on; one
                                  right-hand side through a CUDA graph cached on the device addresses
    the tiles of 32 right-hand sides of the panels and of chol_solve's tiled kernel: 31, 32, 33 rows
    inactive_tri_kernel           2x2 blocks (a knot, ia_first 1 then 2) and 1x1 blocks (ia_first 3)
    diag_minmax_rest_kernel       rcond()'s smallest pivot in L_D, L_S or L_I

Not covered: n_c > 2048, more than 32 blocks, where grp_blkmask takes a second word (a dense longdouble reference at that
size takes minutes); sharded problems, which have no structured factor.

Every case here is a seeded synthetic.make_problem() with selection flags. test_structured_factor_cpu.py proves each
claim from the Jacobian of the compiled reference (oracle/_ref); the GPU tests use the Jacobian optimizer_callback()
returns, which the factor was built from."""
import numpy as np

from chol_np import LD, cholesky_ld, padded, solve_lower_ld, solve_upper_ld
from board_sizes import normal_ld
from mrcal_b200 import synthetic
from problems import SPL3

OPENCV4, OPENCV5, OPENCV8, OPENCV12 = (f"LENSMODEL_OPENCV{n}" for n in (4, 5, 8, 12))
SPLINED_CORE = SPL3   # 11 x 8 knots: with the core optimized, two cameras give a few hundred coupled unknowns


def _select(kw, core=None, dist=True, extr=None, frames=True, warp=True, reg=True):
    if core is not None:
        kw["do_optimize_intrinsics_core"] = core
    kw["do_optimize_intrinsics_distortions"] = dist
    if extr is not None:
        kw["do_optimize_extrinsics"] = extr
    kw["do_optimize_frames"] = frames
    kw["do_optimize_calobject_warp"] = warp
    kw["do_apply_regularization"] = reg
    return kw


def _points_only(kw):
    """drop the board observations: the points are the only eliminated groups"""
    for k in ("observations_board", "indices_frame_camintrinsics_camextrinsics", "rt_ref_frame"):
        kw.pop(k)
    kw["calobject_warp"] = None
    kw["do_optimize_calobject_warp"] = False
    return kw


def _outlier_point(kw, ip):
    """every observation of point ip an outlier: nothing constrains it (D = 0)"""
    obs = kw["observations_point"].copy()
    obs[kw["indices_point_camintrinsics_camextrinsics"][:, 0] == ip, 2] = -1.
    kw["observations_point"] = obs
    return kw


def _unobserved_camera(kw, icam):
    """camera icam keeps its intrinsics but loses its observations"""
    idx = kw["indices_frame_camintrinsics_camextrinsics"]
    keep = idx[:, 1] != icam
    kw["indices_frame_camintrinsics_camextrinsics"] = np.ascontiguousarray(idx[keep])
    kw["observations_board"] = np.ascontiguousarray(kw["observations_board"][keep])
    return kw


def _weighted(kw, boards=None, points=None):
    """board observations' weights times `boards`; point ip's observations' weights times points[ip]"""
    if boards is not None:
        obs = kw["observations_board"].copy()
        obs[..., 2] *= boards
        kw["observations_board"] = obs
    for ip, f in (points or {}).items():
        obs = kw["observations_point"].copy()
        obs[kw["indices_point_camintrinsics_camextrinsics"][:, 0] == ip, 2] *= f
        kw["observations_point"] = obs
    return kw


def _make(lensmodel, Ncameras, Nframes, W=6, H=5, seed=1, which="all", Npoints=0, Npoints_fixed=0, core=None, **sel):
    kw, _ = synthetic.make_problem(lensmodel=lensmodel, Ncameras=Ncameras, Nframes=Nframes, W=W, H=H, seed=seed,
                                   pixel_noise=0.3, which=which, Npoints=Npoints, Npoints_fixed=Npoints_fixed,
                                   do_optimize_intrinsics_core=core)
    kw["calobject_warp"] = np.array((1e-3, -2e-3))
    return _select(kw, **sel)


# ---- the cases. claims (each proved from J by test_structured_factor_cpu.py):
#   n_c, nelim          coupled shared unknowns, eliminated unknowns
#   groups              (frame groups, point groups)
#   nblk                64-column blocks of L_S;  reach  {block: the number of groups that reach it}
#   mixed_stage         some stage of 8 groups holds frame and point groups
#   n_i                 uncoupled shared unknowns;  kinds  the set of ia_first values among them (1, 2: a 2x2 block; 3: 1x1)
#   min_pivot           where rcond()'s smallest diagonal entry of L lies: "D", "S" or "I"; min_kind: its ia_first in L_I
#   singular            J'J is singular: the factor is refused
CASES = {
    # panel stages: one 64-block, which every group reaches
    "stage1": dict(make=lambda: _make(OPENCV4, 3, 1, core=False, dist=False),
                   claims=dict(n_c=14, groups=(1, 0), reach={0: 1})),
    "stage8": dict(make=lambda: _make(OPENCV4, 2, 8), claims=dict(n_c=24, groups=(8, 0), reach={0: 8})),
    "stage9": dict(make=lambda: _make(OPENCV4, 2, 9), claims=dict(n_c=24, groups=(9, 0), reach={0: 9})),
    "stage32": dict(make=lambda: _make(OPENCV4, 2, 32), claims=dict(n_c=24, groups=(32, 0), reach={0: 32})),
    "stage33": dict(make=lambda: _make(OPENCV4, 2, 33), claims=dict(n_c=24, groups=(33, 0), reach={0: 33})),
    "stage65": dict(make=lambda: _make(OPENCV4, 2, 65), claims=dict(n_c=24, groups=(65, 0), reach={0: 65})),
    "stage_mixed": dict(make=lambda: _make(OPENCV8, 2, 3, Npoints=12),
                        claims=dict(n_c=32, groups=(3, 12), reach={0: 15}, mixed_stage=True)),
    # (the fixed points hold the scale that the boards hold elsewhere)
    "points_only": dict(make=lambda: _points_only(_make(OPENCV4, 3, 1, Npoints=30, Npoints_fixed=8)),
                        claims=dict(n_c=36, groups=(0, 17), reach={0: 17})),
    # n_c at the 64-column edge, from the layout alone: 16 x 3 + 6 x 2 + 2, 9 x 7, 16 x 4, 9 x 7 + 2
    "nc62": dict(make=lambda: _make(OPENCV12, 3, 4), claims=dict(n_c=62, nblk=1, reach={0: 4})),
    "nc63": dict(make=lambda: _make(OPENCV5, 7, 24, which="some", extr=False, warp=False),
                 claims=dict(n_c=63, nblk=2, reach={0: 24, 1: 0})),
    "nc64": dict(make=lambda: _make(OPENCV12, 4, 6, extr=False, warp=False),
                 claims=dict(n_c=64, nblk=2, reach={0: 6, 1: 6})),
    "nc65": dict(make=lambda: _make(OPENCV5, 7, 24, which="some", extr=False),
                 claims=dict(n_c=65, nblk=2, reach={0: 24, 1: 24})),
    "multiblock": dict(make=lambda: _make(SPLINED_CORE, 3, 6, W=10, H=10, core=True),
                       claims=dict(n_c=238, nblk=4, reach={0: 6, 1: 6, 2: 6, 3: 6}, kinds={1, 2})),
    "nc0_frames_only": dict(make=lambda: _make(OPENCV4, 2, 4, core=False, dist=False, extr=False, warp=False),
                            claims=dict(n_c=0, nelim=24, groups=(4, 0), n_i=0, min_pivot="D")),
    "nelim0_intrinsics_only": dict(make=lambda: _make(OPENCV4, 2, 6, extr=False, frames=False, warp=False),
                                   claims=dict(n_c=16, nelim=0, groups=(0, 0), n_i=0, min_pivot="S")),
    # uncoupled unknowns: the knots no observation touches (2x2 blocks), the distortions of a camera nobody observes
    # (1x1 blocks; its core and extrinsics locked, else nothing would hold them)
    "uncoupled_knots": dict(make=lambda: _make(SPL3, 2, 4), claims=dict(kinds={1, 2}, min_pivot="S")),
    "uncoupled_1x1": dict(make=lambda: _unobserved_camera(_make(OPENCV4, 3, 4, core=False, extr=False), 2),
                          claims=dict(n_c=10, n_i=4, kinds={3}, min_pivot="I")),
    # rcond()'s smallest pivot: a point group weighted down to 1e-4 (L_D, next to L_S); the board observations weighted
    # up 10 times, which lifts L_S above the regularization of the untouched knots (L_I, the second pivot of a 2x2 block)
    "pivot_in_LD": dict(make=lambda: _weighted(_make(OPENCV4, 2, 3, Npoints=6), points={0: 1e-4}),
                        claims=dict(n_c=24, groups=(3, 5), mixed_stage=True, min_pivot="D")),
    "pivot_in_LI": dict(make=lambda: _weighted(_make(SPL3, 2, 8, W=10, H=10), boards=10.),
                        claims=dict(kinds={1, 2}, min_pivot="I", min_kind=2)),
    # refusals: J has a zero column
    "refuse_outlier_point": dict(make=lambda: _outlier_point(_make(OPENCV4, 2, 3, Npoints=6), 2),
                                 claims=dict(groups=(3, 5), mixed_stage=True, singular=True)),
    "refuse_unregularized_knot": dict(make=lambda: _make(SPL3, 2, 4, reg=False), claims=dict(singular=True)),
}


def case(name):
    return CASES[name]["make"]()


SOLVABLE = [n for n, c in CASES.items() if not c["claims"].get("singular")]
REFUSED = [n for n, c in CASES.items() if c["claims"].get("singular")]


# ---- the shape of a problem, from its J and its layout
class Shape:
    """What the structured factor of the problem kw looks like, from J's sparsity pattern and the layout functions
    (mrcal_b200.state_index_*(), which need no device):
        e0, e1        the eliminated range of the state;  group_cols  each group's state columns, frames then points
        coupled       shared state columns that an observation row touches, in state order (compact numbering)
        uncoupled     the other shared state columns, in state order;  kinds  their ia_first (1/2: first/second of a
                      knot's 2x2 block, 3: a 1x1 block)
        perm          P as an index vector: row i of P b is b[perm[i]]
        reach[b]      the groups that reach 64-block b of L_S, in group order"""

    def __init__(self, kw, J):
        import mrcal_b200 as m
        J = J.tocsr()
        n = J.shape[1]
        assert n == m.num_states(**kw)
        nf, npt = m.num_states_frames(**kw), m.num_states_points(**kw)
        self.e0 = (m.state_index_frames(0, **kw) if nf else m.state_index_points(0, **kw)) if nf + npt else n
        self.e1 = self.e0 + nf + npt
        self.group_cols = [np.arange(self.e0 + 6 * g, self.e0 + 6 * g + 6) for g in range(nf // 6)] + \
                          [np.arange(self.e0 + nf + 3 * p, self.e0 + nf + 3 * p + 3) for p in range(npt // 3)]
        self.Nframe_groups = nf // 6
        shared = np.r_[0:self.e0, self.e1:n]
        m_reg = m.measurement_index_regularization(**kw) if m.num_measurements_regularization(**kw) else J.shape[0]
        touched = np.zeros(n, bool)
        touched[J.indices[:J.indptr[m_reg]]] = True
        self.coupled = shared[touched[shared]]
        self.uncoupled = shared[~touched[shared]]
        self.n_c = len(self.coupled)
        self.nelim = self.e1 - self.e0
        self.nblk = padded(self.n_c + 2) // 64
        self.perm = np.r_[np.arange(self.e0, self.e1), self.coupled, self.uncoupled].astype(int)
        compact = -np.ones(n, int)
        compact[self.coupled] = np.arange(self.n_c)
        # a group reaches the blocks of the coupled columns of its observations' rows, and the block of column n_c
        Jc = J.tocsc()
        self.reach = {b: [] for b in range(self.nblk)}
        for g, cols in enumerate(self.group_cols):
            rows = np.unique(np.concatenate([Jc.indices[Jc.indptr[c]:Jc.indptr[c + 1]] for c in cols]))
            rows = rows[rows < m_reg]
            cc = np.unique(np.concatenate([J.indices[J.indptr[r]:J.indptr[r + 1]] for r in rows])) if len(rows) else []
            for b in {int(compact[c]) // 64 for c in cc if compact[c] >= 0} | {self.n_c // 64}:
                self.reach[b].append(g)
        for b in self.reach:
            self.reach[b].sort()
        # the uncoupled unknowns' blocks: a knot's two columns (x then y), or one column
        i0 = m.state_index_intrinsics(0, **kw)
        ni = m.num_states_intrinsics(**kw) // len(kw["intrinsics"]) if i0 is not None else 0
        ncore = 4 if kw.get("do_optimize_intrinsics_core", True) else 0
        splined = kw["lensmodel"].startswith("LENSMODEL_SPLINED")
        self.kinds = [(1 + (c - i0 - ncore) % ni % 2 if splined and (c - i0) % ni >= ncore else 3)
                      for c in self.uncoupled]

    def stages(self, b):
        """the stages of 8 groups panels_forward_tiled_kernel runs for block b"""
        g = self.reach[b]
        return [g[i:i + 8] for i in range(0, len(g), 8)]


# ---- the reference
def jtj_ld(J):
    """J'J in np.longdouble"""
    H, _ = normal_ld(J, np.zeros(J.shape[0]))
    return H


class Reference:
    """The exact answers of every system for the factor P J'J P' = L L', L the longdouble Cholesky factor of the
    longdouble P J'J P' (unique for a given P). perm: P as an index vector (Shape.perm, or what sys="P" reveals)"""

    def __init__(self, J, perm):
        self.perm = np.asarray(perm)
        H = jtj_ld(J)
        self.H = H
        self.PHP = H[np.ix_(self.perm, self.perm)]
        self.L = cholesky_ld(self.PHP)
        self.Hf = (J.T @ J).toarray()
        self.PHPf = self.Hf[np.ix_(self.perm, self.perm)]

    def pivots(self):
        return np.diag(self.L)

    def rcond(self):
        d = self.pivots()
        return float((d.min() / d.max()) ** 2)

    def solve(self, sys, bt, L=None, lower=None):
        """the rows of bt solved with system `sys` (longdouble); L: another factor (float64) to solve with instead"""
        L = self.L if L is None else L
        B = np.asarray(bt, dtype=LD if L.dtype == LD else float).T
        lo = solve_lower_ld if L.dtype == LD else _lower64
        up = solve_upper_ld if L.dtype == LD else _upper64
        inv = np.argsort(self.perm)
        if sys == "A":
            X = up(L, lo(L, B[self.perm]))[inv]
        elif sys == "LDLt":
            X = up(L, lo(L, B))
        elif sys in ("L", "LD"):
            X = lo(L, B)
        elif sys in ("Lt", "DLt"):
            X = up(L, B)
        elif sys == "D":
            X = B
        elif sys == "P":
            X = B[self.perm]
        elif sys == "Pt":
            X = B[inv]
        else:
            raise ValueError(sys)
        return np.ascontiguousarray(X.T)


def _lower64(L, B):
    import scipy.linalg
    return scipy.linalg.solve_triangular(L, B, lower=True)


def _upper64(L, B):
    import scipy.linalg
    return scipy.linalg.solve_triangular(L, B, lower=True, trans="T")


SYSTEMS = ("A", "LDLt", "LD", "DLt", "L", "Lt", "D", "P", "Pt")


def rhs_counts(nblk):
    """1 (the graph), 7, the per-block/tiled crossover of chol_solve() (8 nblk), the tile edge (32), a partial tile"""
    return sorted({1, 7, 8 * nblk - 1, 8 * nblk, 31, 32, 33, 100})
