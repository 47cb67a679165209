// Internal: the normal equations of the trust-region step, reduced to the shared unknowns by Schur elimination.
// normal.cu: which shared unknowns the rows touch, and the per-item blocks; normal_schur.cu: their sum into S, and the
// back-substitution of the eliminated unknowns
#pragma once
#include "chol.h"
#include "problem_impl.h"

namespace mb200 {

// All device pointers. "work item" = one board observation or one point
// observation; "group" = one eliminated block (a frame: 6 unknowns, or a
// non-fixed point: 3 unknowns) with the work items that see it.
constexpr int kYld = 68;              // row stride of the panels of Ypan (doubles)
constexpr int kYpanel = 6 * kYld;     // one (group, block) panel

// The compact block of a board observation of the fused evaluation. Its local columns are numbered as in the full layout:
// knot k is columns 2k (x surface) and 2k+1 (y surface), then the nsh - 2 nk geometry columns (camera r,t | warp). The
// knot x knot part of the Gram matrix is fx^2 M on the x surface, fy^2 M on the y surface and zero across, M = Dk'Dk (nk x
// nk), so M is stored once and the two gradient rows of the full layout (equal) once. In doubles:
//   [0] fx*fx, [1] fy*fy
//   [2 ..)                   M, packed lower triangle: M[k1][k2], k2 <= k1, at 2 + k1 (k1 + 1) / 2 + k2
//   [compact_geo0(nk) ..)    rows 2nk .. nsh-1 of the full layout, nsh doubles each (columns 0 .. row valid)
//   then                     -J'x over the nsh columns: rows nsh and nsh+1 of the full layout
// The entries of the full layout are (fx*fx) * M[k1][k2] and (fy*fy) * M[k1][k2], rounded as written.
constexpr int kCompactMaxKnots = 64;  // knots of one observation's patch (the fused kernel gives up beyond)
constexpr int kCompactMaxGeo = 8;     // geometry columns: camera extrinsics 6, board warp 2
__host__ __device__ constexpr int compact_geo0(int nk) { return 2 + nk * (nk + 1) / 2; }
// the fixed slot of one board observation in the pool (the fused kernel writes board w at w * kCompactSlot)
constexpr long long kCompactSlot = compact_geo0(kCompactMaxKnots) + (kCompactMaxGeo + 1) * (2 * kCompactMaxKnots + kCompactMaxGeo);

struct NormalBuffers
{
    double* S;        // [ldS][ldS] row-major, lower: reduced normal matrix over the ACTIVE shared unknowns
                      // (compact numbering), then its Cholesky factor
    int     ldS;      // n_c padded to a multiple of 64 (changes per assembly)
    int     ldS_max;  // n_r padded: the allocation
    int     n_r;      // number of shared (non-eliminated) unknowns
    int     n_c;      // ... of which touched by some observation: the coupled ("active") ones
    int     max_ntot; // widest work item (local columns) at the operating point of the last normal_prepare()
    double* gs;       // [ldS_max] reduced gradient g' (compact numbering)
    int*    active;   // [n_r] flag
    int*    cidx;     // [n_r] reduced -> compact index, -1 if inactive
    int*    cinv;     // [ldS_max] compact -> reduced index
    int*    stat;     // device: [0] n_c, [1] widest item (local columns), [2] the items' blocks outgrow the pool,
                      // [3] the fused evaluation gave up on an observation
    int*    h_stat;   // pinned host mirror of stat
    bool    splined;
    double* g_full;   // [Nstate] J'x, state numbering
    int*    info;     // 0, or a code for the first non-PD block found
    int     e0, e1;   // eliminated state range [e0,e1)

    int     cap;      // capacity (columns) of one work item's B rows
    int*    wi_nsh;   // [Nwi] shared columns the item touches
    int*    wi_cols;  // [Nwi][cap] their reduced indices, increasing
    double* wi_B;     // [Nwi][6][cap] (eliminated x shared) block of the item's Gram matrix
    double* wi_D;     // [Nwi][36]
    double* wi_gf;    // [Nwi][6]

    int     Ngroups, Nframe_groups;
    int*    grp_ptr;    // [Ngroups+1]
    int*    grp_items;  // work item ids

    // ---- the sum into S (normal_schur.cu): every entry of S is summed by ONE thread in a fixed order
    bool    fused;        // the board rows are evaluated by fused_eval.cu: blocks straight from the projection, no J
    double* norm_part;    // [Nobs_board] per-observation |x|^2
    double* qf_part;      // [Nobs_board] per-observation g'(J'J)g
    cudaStream_t s_side[2];               // forked streams: the Gram kernel's size classes; [0] also the step's Cauchy sums
    cudaEvent_t  ev_fork, ev_join[2];
    int     capA;         // most local columns (incl. the two gradient rows) an item may have in the A pool
    double* wi_A;         // pool of per-item Gram blocks over the shared columns, in one of two layouts (wi_lda says which):
                          //  full    [lda][lda] row-major, lower triangle; rows nsh, nsh+1: -J'x over the item's shared columns
                          //  compact the board observations of the fused evaluation (fused_eval.cu); see kCompactSlot
    long long* wi_Aoff;   // [Nwi] offset of each item's block in the pool (doubles)
    long long  A_pool;    // pool size (doubles); grows when the items' blocks do not fit (normal_adopt_sizes)
    long long* pool_need; // device: what the last placement of the items needed (doubles)
    bool    replace_items;   // the pool grew since the items were placed: place them again before the next assembly
    int*    wi_lda;       // [Nwi] full layout: nsh + 2 rounded up to even. Compact layout: ~nk (< 0)
    unsigned short* wi_ccol;    // [Nwi][capA] compact index of each local column (increasing); then n_c, n_c+1
    unsigned short* wi_segoff;  // [Nwi][nblk_max+1] first local column of each 64-column block of S
    int     nblk_max;     // ldS_max / 64
    double* Ypan;         // [Ngroups][nblk_max][6][kYld] inv(L_D) B of each group, dense per 64-column block (present blocks
                          // only). Rows padded to kYld: a panel goes to shared memory as ONE bulk copy and lands with a
                          // row stride whose DMMA fragment loads are free of bank conflicts
    unsigned* grp_present;   // [nblk_max][gwords] bit g: group g has columns in this block
    unsigned* wi_present;    // [nblk_max][wwords]
    unsigned* grp_blkmask;   // [Ngroups][bwords] the blocks a group is present in
    int     gwords, wwords, bwords;
    double* grp_Linv;     // [Ngroups][36] inverse of the Cholesky factor of D (lower)
    double* grp_h;        // [Ngroups][6]  inv(L_D) gf
    double* part_scratch; // partial tiles of the tiles whose contributors are split over several CTAs
    int*    part_arrive;  // their arrival counters
    double* S_packed;     // sharded solves: the lower-triangle tiles of S, each 64x64 contiguous: what is all-reduced

    __host__ __device__ int reduced_index(int c) const { return c < e0 ? c : c - (e1 - e0); }
    __host__ __device__ int state_index(int r) const { return r < e0 ? r : r + (e1 - e0); }

    // Where state column c lives in the three pieces of a permuted vector (the structured factor's right-hand sides,
    // factorization_schur.cu): piece 0 = Bf[.][i] (eliminated), 1 = Bs[.][i] (coupled, compact numbering),
    // 2 = Bi[.][i] (uncoupled, reduced numbering)
    struct Slot { int piece, i; };
    __device__ Slot slot(int c) const
    {
        if(c >= e0 && c < e1) return {0, c - e0};
        const int r = reduced_index(c);
        return cidx[r] >= 0 ? Slot{1, cidx[r]} : Slot{2, r};
    }
    // that slot of right-hand side `rhs`
    template <typename T>
    __device__ T* at(Slot s, T* Bf, int Nelim, T* Bs, T* Bi, size_t rhs) const
    {
        return s.piece == 0 ? &Bf[rhs * Nelim + s.i] : s.piece == 1 ? &Bs[rhs * ldS + s.i] : &Bi[rhs * n_r + s.i];
    }
};

// The first eliminated column of group grp, relative to e0
__host__ __device__ inline int group_col0(const NormalBuffers& N, int grp)
{
    return grp < N.Nframe_groups ? 6 * grp : 6 * N.Nframe_groups + 3 * (grp - N.Nframe_groups);
}

// The regularization block of an uncoupled shared unknown (state column c), the only rows that touch it: H = J'J over
// its 1 or 2 columns and, if x is given, J'x. n = 0: no row touches c
struct UncoupledBlock { int n, which; double Hxx, Hyy, Hxy, gx, gy; };
__device__ __forceinline__ UncoupledBlock uncoupled_block(const DevProblem& P, bool splined, int c, const double* __restrict__ Jval,
                                                          const double* __restrict__ x)
{
    UncoupledBlock u{};
    const int b = reg_block_of_column(P, splined, c, &u.which);
    if(b < 0) return u;
    const RegBlock rb = reg_block(P, splined, b);
    u.n = rb.ncol;
    if(rb.ncol == 2)
    {
        // rows (radial, tangential) of the knot; entries [d/dx, d/dy] each
        const double* e0 = &Jval[rb.j0];
        const double* e1 = e0 + 2;
        u.Hxx = e0[0] * e0[0] + e1[0] * e1[0];
        u.Hyy = e0[1] * e0[1] + e1[1] * e1[1];
        u.Hxy = e0[0] * e0[1] + e1[0] * e1[1];
        if(x != nullptr)
        {
            const double x0 = x[rb.m0], x1 = x[rb.m0 + 1];
            u.gx = e0[0] * x0 + e1[0] * x1;
            u.gy = e0[1] * x0 + e1[1] * x1;
        }
    }
    else
    {
        const double e = Jval[rb.j0];
        u.Hxx = e * e;
        if(x != nullptr) u.gx = e * x[rb.m0];
    }
    return u;
}

// The buffers of the normal equations of problem P (its layout, its observations): allocated in `arena`, except for
// what may grow or is not memory (the pool of the items' blocks, the side streams and their events), which
// normal_buffers_destroy() releases. N.h_stat is the caller's to set
bool normal_buffers_create(NormalBuffers* N, const mrcal_b200_problem* P, DeviceArena& arena);
void normal_buffers_destroy(NormalBuffers* N);

// The evaluation at `op` that the assembly needs: the fused one when N.fused (the board observations' blocks straight
// from the projection, the other rows as usual), the stored-Jacobian one otherwise. normal_prepare() comes next
bool normal_evaluate(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, cudaStream_t s, int* nlaunch);
// The same in pieces, for a caller that wants to pick its own moment to wait for the device:
// prepare (device work + an async copy of the sizes) -> [synchronise the stream] -> adopt_sizes -> finish
// (copy_sizes = false: the caller copies stat[] to h_stat itself, together with its own scalars)
bool normal_prepare(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, cudaStream_t s, int* nlaunch, bool boards_done,
                    double* rider = nullptr, bool* rider_summed = nullptr, bool copy_sizes = true);
bool normal_adopt_sizes(NormalBuffers& N, cudaStream_t s);   // (s: the stream the pool is used on, when it grows)
// also_clear: n doubles of the caller's that are zeroed with the assembly's own accumulators (one launch)
bool normal_finish(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                   double lambda, cudaStream_t s, int* nlaunch, bool boards_done, double* also_clear = nullptr, int also_clear_n = 0);
// fused_eval.cu
bool launch_fused_boards(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& out, double* norm_part, cudaStream_t s, int* nlaunch);
bool launch_quadform_boards(const DevProblem& dp, const NormalBuffers& N, const double* g_full, double* part, double* out, cudaStream_t s, int* nlaunch);
// S, g', g_full at the operating point `op` (needs its x and Jacobian). lambda: diagonal loading.
// Updates N.n_c / N.ldS (one small device->host read)
bool normal_assemble(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                     double lambda, cudaStream_t s, int* nlaunch);
// rhs <- y, L y = -g': read from the augmented row of the factor (valid after chol_factor)
bool normal_extract_y(const NormalBuffers& N, double* rhs, cudaStream_t s, int* nlaunch);
// full-length Gauss-Newton step from the compact solution: active shared unknowns, inactive shared
// unknowns (from their regularization blocks), eliminated unknowns (back-substitution).
bool normal_expand_step(const DevProblem& dp, const NormalBuffers& N, const EvalBuffers& op, double lambda,
                        const double* sol, double* step_full, cudaStream_t s, int* nlaunch);

// normal_schur.cu. S, g' and J'x from the items' blocks at `op` (normal_finish() runs it)
bool normal_schur_sum(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                      double lambda, cudaStream_t s, int* nlaunch);
// the eliminated unknowns of the step from the compact solution (normal_expand_step() runs it)
bool normal_schur_backsub(const NormalBuffers& N, const double* sol_compact, double* step_full, cudaStream_t s, int* nlaunch);
// what its buffers need for a system of up to nblk_max 64-column blocks
struct NormalSchurSizes { size_t part_scratch_doubles; int part_arrive_ints; size_t packed_doubles; };
NormalSchurSizes normal_schur_sizes(int nblk_max);

}  // namespace mb200
