// Internal: what the assembly kernels of normal.cu, normal_schur.cu and fused_eval.cu share.
#pragma once
#include "normal.h"
#include "ptx.cuh"
#include "reduce.cuh"

namespace mb200 {

constexpr int kMaxRowNnz = 40;     // widest row: 16 intrinsics + 6 + 6 + 2 (any model here <= 30)
constexpr int kGramMax   = 200;
constexpr int RCH        = 16;     // rows staged per chunk in assemble_items_kernel (RCH*kMaxRowNnz <= 3*256)    // largest local column count whose Gram matrix lives in shared memory

struct ItemDesc
{
    int rows, nnz_row, nI, j0, m0;
    int cbase, clen;       // the camera's intrinsics block in the state vector
    int cam0;              // first extrinsics column, or -1
    int elim0, nelim;      // first eliminated column, count (6 frame / 3 point / 0)
    int warp0;             // first warp column or -1
    int group;             // elimination group or -1
};

__device__ __forceinline__ ItemDesc describe_item(const DevProblem& P, int w, int Nframe_groups)
{
    ItemDesc d;
    d.nI = P.nnz_row_intr;
    d.clen = P.Nintr_state;
    if(w < P.Nobs_board)
    {
        const int icam_i = P.obs_board[3 * w + 0], icam_e = P.obs_board[3 * w + 1], iframe = P.obs_board[3 * w + 2];
        d.rows = 2 * P.W * P.H;
        d.j0 = P.board_j0[w];
        d.nnz_row = (P.board_j0[w + 1] - d.j0) / d.rows;
        d.m0 = d.rows * w;
        d.cbase = P.i_intr0 + icam_i * P.Nintr_state;
        d.cam0 = (P.opt_extr && icam_e >= 0) ? P.i_extr0 + 6 * icam_e : -1;
        d.nelim = P.opt_frames ? 6 : 0;
        d.elim0 = P.opt_frames ? P.i_frame0 + 6 * iframe : -1;
        d.warp0 = P.opt_warp ? P.i_warp0 : -1;
        d.group = P.opt_frames ? iframe : -1;
    }
    else
    {
        const int o = w - P.Nobs_board;
        const int icam_i = P.obs_point[3 * o + 0], icam_e = P.obs_point[3 * o + 1], ipt = P.obs_point[3 * o + 2];
        const bool in_state = P.opt_frames && ipt < P.Npoints_variable;
        d.rows = 2;
        d.j0 = P.point_j0[o];
        d.nnz_row = (P.point_j0[o + 1] - d.j0) / 2;
        d.m0 = P.m_point0 + 2 * o;
        d.cbase = P.i_intr0 + icam_i * P.Nintr_state;
        d.cam0 = (P.opt_extr && icam_e >= 0) ? P.i_extr0 + 6 * icam_e : -1;
        d.nelim = in_state ? 3 : 0;
        d.elim0 = in_state ? P.i_point0 + 3 * ipt : -1;
        d.warp0 = -1;
        d.group = in_state ? Nframe_groups + ipt : -1;
    }
    return d;
}

__device__ __forceinline__ int tri(int a, int b) { return a * (a + 1) / 2 + b; }   // a >= b

// the inverse of tri(): q -> (r >= c) with tri(r, c) == q. The float square root is a first guess, corrected exactly
__device__ __forceinline__ void tri_row_col(int q, int& r, int& c)
{
    r = (int)((sqrtf(8.f * q + 1.f) - 1.f) * 0.5f);
    while(r * (r + 1) / 2 > q) r--;
    while((r + 1) * (r + 2) / 2 <= q) r++;
    c = q - r * (r + 1) / 2;
}

}  // namespace mb200
