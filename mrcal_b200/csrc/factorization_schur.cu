// The factorization object of a CALIBRATION PROBLEM, with the structure the solver itself uses instead of a
// dense Nstate x Nstate matrix: the 4th return value of mrcal.optimizer_callback() (mrcal-pywrap.c:1980-1988),
// consumed by the projection-uncertainty code through solve_xt_JtJ_bt(bt, sys=...) (mrcal-pywrap.c:425-578,
// mrcal/model_analysis.py:716-870) with hundreds of right-hand sides.
//
// In the order  P = [ eliminated unknowns (frames, points) | coupled shared unknowns (compact) | uncoupled shared
// unknowns ]  the normal matrix factors as  P JtJ P' = L L'  with
//
//         [ L_D            ]     L_D  block diagonal: the 6x6 / 3x3 Cholesky factors of the groups
//     L = [ Y'   L_S       ]     Y    = inv(L_D) B, held as dense 6x64 panels per (group, 64-column block)
//         [           L_I  ]     L_S  the dense Cholesky factor of the reduced system (DMMA kernels, chol*.cu)
//                                L_I  2x2 / 1x1 factors of the regularization blocks of unknowns no observation touches
//
// a genuine lower-triangular Cholesky factor, so every system of the reference -- A, LDLt, LD, DLt, L, Lt, D (= I), P,
// Pt -- has its meaning, and the identities between them that the callers rely on hold. At BASELINE config 3 this is
// 1268^3/3 flops and ~40 MB instead of 7220^3/3 flops and 417 MB.
//
// The object OWNS the device problem it was made from (the one the last mrcal_optimizer_callback() call left in the
// cache): mrcal_b200_factorization_create_from_last_callback().
#include "comm.h"
#include "ptx.cuh"
#include "reduce.cuh"
#include "solver_internal.h"

namespace mb200 {

mrcal_b200_problem_t* capi_steal_cached_problem();   // capi.cu

namespace {
constexpr int TB = 64;

// rows n_c, n_c+1 of the factor carry the solver's right-hand side: here they become plain padding -- in L and in the
// stored inverses of its diagonal blocks (row m of the inverse of a lower-triangular block depends on rows <= m only)
__global__ void clear_aug_rows_kernel(NormalBuffers N, int n_c, double* __restrict__ invL)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= N.ldS) return;
    for(int r = n_c; r < n_c + 2 && r < N.ldS; r++)
    {
        N.S[(size_t)r * N.ldS + c] = (c == r) ? 1. : 0.;
        if((c >> 6) == (r >> 6)) invL[(size_t)(r >> 6) * (TB * TB) + (r & 63) * TB + (c & 63)] = (c == r) ? 1. : 0.;
    }
}

// Cholesky factors of the regularization blocks of the uncoupled shared unknowns (what inactive_step_kernel inverts)
__global__ void inactive_blocks_kernel(DevProblem P, NormalBuffers N, const double* __restrict__ Jval,
                                       double* __restrict__ ia_L, int* __restrict__ ia_first, int* __restrict__ bad)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if(r >= N.n_r) return;
    ia_first[r] = 0;
    if(N.cidx[r] >= 0) return;
    const int c = N.state_index(r);
    const UncoupledBlock u = uncoupled_block(P, N.splined, c, Jval, nullptr);
    if(u.n == 2)
    {
        const double l11 = sqrt(u.Hxx), l21 = u.Hxy / l11, d = u.Hyy - l21 * l21;
        if(!(u.Hxx > 0.) || !(d > 0.)) { atomicExch(bad, 1); return; }
        ia_first[r] = u.which == 0 ? 1 : 2;
        ia_L[3 * r] = l11; ia_L[3 * r + 1] = l21; ia_L[3 * r + 2] = sqrt(d);
        return;
    }
    const double H = u.Hxx;
    if(!(H > 0.)) { atomicExch(bad, 1); return; }   // an unknown nothing constrains: JtJ is singular
    ia_first[r] = 3;
    ia_L[3 * r] = sqrt(H); ia_L[3 * r + 1] = 0.; ia_L[3 * r + 2] = 0.;
}

// state-ordered right-hand sides <-> the three pieces of the permuted vector. bt, out: [Nrhs][Nstate]
// Bf: [Nrhs][Nelim]   Bs: [Nrhs][ldS] (compact, zero padded)   Bi: [Nrhs][n_r] (reduced numbering; active slots unused)
__global__ void split_state_kernel(NormalBuffers N, const double* __restrict__ bt, int Nstate, int Nrhs,
                                   double* __restrict__ Bf, int Nelim, double* __restrict__ Bs, double* __restrict__ Bi)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrhs * Nstate) return;
    const int rhs = (int)(idx / Nstate), c = (int)(idx - (long)rhs * Nstate);
    *N.at(N.slot(c), Bf, Nelim, Bs, Bi, rhs) = bt[idx];
}
__global__ void join_state_kernel(NormalBuffers N, double* __restrict__ out, int Nstate, int Nrhs,
                                  const double* __restrict__ Bf, int Nelim, const double* __restrict__ Bs, const double* __restrict__ Bi)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrhs * Nstate) return;
    const int rhs = (int)(idx / Nstate), c = (int)(idx - (long)rhs * Nstate);
    out[idx] = *N.at(N.slot(c), Bf, Nelim, Bs, Bi, rhs);
}
// the same two maps for vectors that are ALREADY in the permuted order [eliminated | compact | uncoupled (reduced order)]
__global__ void split_permuted_kernel(NormalBuffers N, const double* __restrict__ bt, int Nstate, int Nrhs, bool to_pieces,
                                      double* __restrict__ Bf, int Nelim, double* __restrict__ Bs, double* __restrict__ Bi,
                                      const int* __restrict__ ia_rank /*[n_r] rank of each uncoupled unknown among the uncoupled*/,
                                      double* __restrict__ out)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrhs * Nstate) return;
    const int rhs = (int)(idx / Nstate), c = (int)(idx - (long)rhs * Nstate);
    // c is a STATE index; its place in the permuted vector:
    const NormalBuffers::Slot sl = N.slot(c);
    const int perm = sl.piece == 0 ? sl.i : sl.piece == 1 ? Nelim + sl.i : Nelim + N.n_c + ia_rank[sl.i];
    double* piece = N.at(sl, Bf, Nelim, Bs, Bi, rhs);
    if(to_pieces) *piece = bt[(size_t)rhs * Nstate + perm];
    else          out[(size_t)rhs * Nstate + perm] = *piece;
}

// L_D z = b (forward) or L_D' x = z (backward) per group and right-hand side, in place in Bf
__global__ void groups_tri_kernel(NormalBuffers N, double* __restrict__ Bf, int Nelim, int Nrhs, bool forward)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrhs * N.Ngroups) return;
    const int rhs = (int)(idx / N.Ngroups), grp = (int)(idx - (long)rhs * N.Ngroups);
    const int nelim = grp < N.Nframe_groups ? 6 : 3;
    const double* Li = N.grp_Linv + (size_t)grp * 36;   // inv(L_D), lower
    double* b = Bf + (size_t)rhs * Nelim + group_col0(N, grp);
    double v[6], o[6];
    for(int p = 0; p < nelim; p++) v[p] = b[p];
    for(int p = 0; p < nelim; p++)
    {
        double t = 0.;
        if(forward) for(int q = 0; q <= p; q++) t += Li[p * 6 + q] * v[q];          // inv(L) b
        else        for(int q = p; q < nelim; q++) t += Li[q * 6 + p] * v[q];       // inv(L)' z
        o[p] = t;
    }
    for(int p = 0; p < nelim; p++) b[p] = o[p];
}

// Forward panels: Bs[r][64 blk + col] -= sum over the groups g that reach block blk of  Zf[r][g] Y_g[blk][:, col].
// One CTA per (block, tile of kSolveTile right-hand sides); the groups in index order, 8 per stage, each padded to 8
// unknowns. (The panels carry the solver's right-hand-side column at compact index n_c: not part of the factor)
__global__ void __launch_bounds__(256)
panels_forward_tiled_kernel(NormalBuffers N, const double* __restrict__ Bf, int Nelim, double* __restrict__ Bs, int Nrhs)
{
    extern __shared__ __align__(16) double dsm[];
    double (*sA)[kSolveTileLd] = reinterpret_cast<double (*)[kSolveTileLd]>(dsm);
    double (*sM)[kSolveTileLd] = reinterpret_cast<double (*)[kSolveTileLd]>(dsm + kSolveTile * kSolveTileLd);
    const int blk = blockIdx.x, r0 = blockIdx.y * kSolveTile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g8 = lane >> 2, t4 = lane & 3;
    const int mt = warp >> 1, nt0 = (warp & 1) * 4;   // warp: rows mt*8.., n-tiles nt0..nt0+3
    double acc[4][2] = {};
    const unsigned* present = N.grp_present + (size_t)blk * N.gwords;
    int gid[8], nb = 0;
    auto stage = [&]()
    {
        for(int e = tid; e < kSolveTile * 64; e += 256)
        {
            const int r = e >> 6, kk = e & 63, q = kk >> 3, pp = kk & 7;
            double v = 0.;
            if(q < nb && r0 + r < Nrhs)
            {
                const int g = gid[q], ne = g < N.Nframe_groups ? 6 : 3;
                if(pp < ne) v = Bf[(size_t)(r0 + r) * Nelim + group_col0(N, g) + pp];
            }
            sA[r][kk] = v;
        }
        for(int e = tid; e < 64 * TB; e += 256)
        {
            const int kk = e >> 6, col = e & 63, q = kk >> 3, pp = kk & 7;
            double v = 0.;
            if(q < nb)
            {
                const int g = gid[q], ne = g < N.Nframe_groups ? 6 : 3;
                if(pp < ne) v = N.Ypan[((size_t)g * N.nblk_max + blk) * kYpanel + pp * kYld + col];
            }
            sM[kk][col] = v;
        }
        __syncthreads();
        const int ksteps = 2 * nb;
        for(int ks = 0; ks < ksteps; ks++)
        {
            const double a = sA[mt * 8 + g8][ks * 4 + t4];
#pragma unroll
            for(int j = 0; j < 4; j++) dmma(acc[j][0], acc[j][1], a, sM[ks * 4 + t4][(nt0 + j) * 8 + g8]);
        }
        __syncthreads();
        nb = 0;
    };
    for(int w = 0; w < N.gwords; w++)
    {
        unsigned m = present[w];
        while(m)
        {
            gid[nb++] = 32 * w + __ffs(m) - 1;
            m &= m - 1;
            if(nb == 8) stage();
        }
    }
    if(nb > 0) stage();
    const int r = r0 + mt * 8 + g8;
    if(r >= Nrhs) return;
#pragma unroll
    for(int j = 0; j < 4; j++)
        for(int h = 0; h < 2; h++)
        {
            const int col = TB * blk + (nt0 + j) * 8 + 2 * t4 + h;
            if(col < N.n_c) Bs[(size_t)r * N.ldS + col] -= acc[j][h];
        }
}
// z_g -= Y_g x_s  (backward, after L_S'): one warp per (group, right-hand side)
__global__ void __launch_bounds__(256)
panels_backward_kernel(NormalBuffers N, double* __restrict__ Bf, int Nelim, const double* __restrict__ Bs, int Nrhs, int nblk)
{
    const long wid = ((long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if(wid >= (long)Nrhs * N.Ngroups) return;
    const int rhs = (int)(wid / N.Ngroups), grp = (int)(wid - (long)rhs * N.Ngroups);
    const double* Yg = N.Ypan + (size_t)grp * N.nblk_max * kYpanel;
    const double* xs = Bs + (size_t)rhs * N.ldS;
    double t[6] = {0., 0., 0., 0., 0., 0.};
    for(int b = 0; b < nblk; b++)
    {
        if(!((N.grp_blkmask[(size_t)grp * N.bwords + (b >> 5)] >> (b & 31)) & 1u)) continue;
        const double d0 = xs[TB * b + lane], d1 = xs[TB * b + 32 + lane];
#pragma unroll
        for(int p = 0; p < 6; p++) t[p] += Yg[(size_t)b * kYpanel + p * kYld + lane] * d0 + Yg[(size_t)b * kYpanel + p * kYld + 32 + lane] * d1;
    }
    warp_sum(t);
    const int nelim = grp < N.Nframe_groups ? 6 : 3;
    if(lane < nelim) Bf[(size_t)rhs * Nelim + group_col0(N, grp) + lane] -= t[lane];
}

// the uncoupled unknowns: L_I z = b / L_I' x = z, per block
__global__ void inactive_tri_kernel(NormalBuffers N, const double* __restrict__ ia_L, const int* __restrict__ ia_first,
                                    double* __restrict__ Bi, int Nrhs, bool forward)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrhs * N.n_r) return;
    const int rhs = (int)(idx / N.n_r), r = (int)(idx - (long)rhs * N.n_r);
    const int kind = ia_first[r];
    double* b = Bi + (size_t)rhs * N.n_r;
    if(kind == 3) b[r] /= ia_L[3 * r];
    else if(kind == 1)
    {
        // the block (r, r+1): [l11 0; l21 l22]
        const double l11 = ia_L[3 * r], l21 = ia_L[3 * r + 1], l22 = ia_L[3 * r + 2];
        const double b0 = b[r], b1 = b[r + 1];
        if(forward) { const double z0 = b0 / l11; b[r] = z0; b[r + 1] = (b1 - l21 * z0) / l22; }
        else        { const double x1 = b1 / l22; b[r + 1] = x1; b[r] = (b0 - l21 * x1) / l11; }
    }
}

// d_out2[0] = min, [1] = max over the diagonal of L_D and L_I (L_S is done by chol_diag_minmax)
__global__ void diag_minmax_rest_kernel(NormalBuffers N, const double* __restrict__ ia_L, const int* __restrict__ ia_first, double* __restrict__ out2)
{
    // one thread: called once per rcond(); the arrays are short
    if(threadIdx.x != 0 || blockIdx.x != 0) return;
    double mn = out2[0], mx = out2[1];
    for(int g = 0; g < N.Ngroups; g++)
    {
        const int nelim = g < N.Nframe_groups ? 6 : 3;
        for(int p = 0; p < nelim; p++)
        {
            const double d = 1. / N.grp_Linv[(size_t)g * 36 + p * 6 + p];
            mn = fmin(mn, d); mx = fmax(mx, d);
        }
    }
    for(int r = 0; r < N.n_r; r++)
    {
        const int k = ia_first[r];
        if(k == 3 || k == 1) { mn = fmin(mn, ia_L[3 * r]); mx = fmax(mx, ia_L[3 * r]); }
        if(k == 1) { mn = fmin(mn, ia_L[3 * r + 2]); mx = fmax(mx, ia_L[3 * r + 2]); }
    }
    out2[0] = mn; out2[1] = mx;
}

}  // namespace

bool schur_solve_pieces(const mrcal_b200_factorization* F, double* Bf, double* Bs, double* Bi, int Nrhs, bool forward,
                        BackSolve backward, cudaStream_t s)
{
    const SolverWorkspace* ws = F->P->ws.get();
    const NormalBuffers& N = ws->N;
    const int Nelim = F->Nelim, nblk = N.ldS / TB;
    const long gr = (long)Nrhs * N.Ngroups, ir = (long)Nrhs * N.n_r;
    if(forward)
    {
        if(N.Ngroups > 0)
        {
            groups_tri_kernel<<<(unsigned)((gr + 127) / 128), 128, 0, s>>>(N, Bf, Nelim, Nrhs, true);
            panels_forward_tiled_kernel<<<dim3(nblk, (Nrhs + kSolveTile - 1) / kSolveTile), 256, kSolveTileSmem, s>>>(N, Bf, Nelim, Bs, Nrhs);
        }
        if(N.n_c > 0 && !chol_solve(N.S, N.ldS, N.n_c, ws->invL, Bs, N.ldS, Nrhs, s, nullptr, 1)) return false;
        if(N.n_r > N.n_c) inactive_tri_kernel<<<(unsigned)((ir + 255) / 256), 256, 0, s>>>(N, F->ia_L, F->ia_first, Bi, Nrhs, true);
    }
    if(backward != BackSolve::none)
    {
        if(N.n_r > N.n_c) inactive_tri_kernel<<<(unsigned)((ir + 255) / 256), 256, 0, s>>>(N, F->ia_L, F->ia_first, Bi, Nrhs, false);
        if(N.n_c > 0 && !chol_solve(N.S, N.ldS, N.n_c, ws->invL, Bs, N.ldS, Nrhs, s, nullptr, 2)) return false;
        if(backward == BackSolve::all && N.Ngroups > 0)
        {
            panels_backward_kernel<<<(unsigned)((gr * 32 + 255) / 256), 256, 0, s>>>(N, Bf, Nelim, Bs, Nrhs, nblk);
            groups_tri_kernel<<<(unsigned)((gr + 127) / 128), 128, 0, s>>>(N, Bf, Nelim, Nrhs, false);
        }
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

bool schur_factorization_solve(mrcal_b200_factorization* F, double* out, const double* bt, int Nrhs, const SysSteps& st)
{
    mrcal_b200_problem* P = F->P;
    NormalBuffers& N = P->ws->N;
    cudaStream_t s = P->stream;
    const int Nstate = P->L.Nstate, Nelim = F->Nelim;
    DeviceArena tmp;
    double *d_in, *d_out, *Bf, *Bs, *Bi;
    if(!tmp.alloc(&d_in, (size_t)Nrhs * Nstate) || !tmp.alloc(&d_out, (size_t)Nrhs * Nstate) ||
       !tmp.alloc(&Bf, (size_t)Nrhs * (Nelim > 0 ? Nelim : 1), true) || !tmp.alloc(&Bs, (size_t)Nrhs * N.ldS, true) ||
       !tmp.alloc(&Bi, (size_t)Nrhs * (N.n_r > 0 ? N.n_r : 1), true))
        return false;
    MB200_CUDA_CHECK(cudaMemcpyAsync(d_in, bt, (size_t)Nrhs * Nstate * sizeof(double), cudaMemcpyHostToDevice, s));
    const long tot = (long)Nrhs * Nstate;
    const unsigned gtot = (unsigned)((tot + 255) / 256);
    if(st.permuted_in) split_permuted_kernel<<<gtot, 256, 0, s>>>(N, d_in, Nstate, Nrhs, true, Bf, Nelim, Bs, Bi, F->ia_first + N.n_r, nullptr);
    else            split_state_kernel<<<gtot, 256, 0, s>>>(N, d_in, Nstate, Nrhs, Bf, Nelim, Bs, Bi);
    if(!schur_solve_pieces(F, Bf, Bs, Bi, Nrhs, st.fwd, st.bwd ? BackSolve::all : BackSolve::none, s)) return false;
    if(st.permuted_out) split_permuted_kernel<<<gtot, 256, 0, s>>>(N, nullptr, Nstate, Nrhs, false, Bf, Nelim, Bs, Bi, F->ia_first + N.n_r, d_out);
    else             join_state_kernel<<<gtot, 256, 0, s>>>(N, d_out, Nstate, Nrhs, Bf, Nelim, Bs, Bi);
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpyAsync(out, d_out, (size_t)Nrhs * Nstate * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

double schur_factorization_rcond(mrcal_b200_factorization* F)
{
    mrcal_b200_problem* P = F->P;
    NormalBuffers& N = P->ws->N;
    cudaStream_t s = P->stream;
    double mm[2] = {1e300, 0.};
    if(N.n_c > 0) { if(!chol_diag_minmax(N.S, N.ldS, N.n_c, F->minmax, s)) return -1.; }
    else if(cudaMemcpyAsync(F->minmax, mm, sizeof(mm), cudaMemcpyHostToDevice, s) != cudaSuccess) return -1.;
    diag_minmax_rest_kernel<<<1, 32, 0, s>>>(N, F->ia_L, F->ia_first, F->minmax);
    if(cudaMemcpyAsync(mm, F->minmax, sizeof(mm), cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) return -1.;
    if(!(mm[1] > 0.)) return 0.;
    const double r = mm[0] / mm[1];
    return r * r;
}

void schur_factorization_release(mrcal_b200_factorization* F)
{
    if(F->P) { cudaStreamSynchronize(F->P->stream); }
    F->arena.release();
    if(F->P) mrcal_b200_problem_destroy(F->P);
    F->P = nullptr;
}

__global__ void rank_inactive_kernel(NormalBuffers N, int* __restrict__ ia_rank)
{
    // one thread: n_r <= a few 10^4
    if(threadIdx.x != 0 || blockIdx.x != 0) return;
    int k = 0;
    for(int r = 0; r < N.n_r; r++) ia_rank[r] = N.cidx[r] < 0 ? k++ : -1;
}

// Builds the structured factor of P at its current state into F (F->P is set by the caller; F does not own P here).
// False, with the reason in the error string, if P is sharded or JtJ is not positive definite. The device problem's
// solver workspace holds L_S and the panels afterwards (they are what the next solver iteration overwrites)
bool schur_factor_build(mrcal_b200_problem* P, mrcal_b200_factorization* F)
{
    if(comm_active() || P->sharded) { set_error("structured factorization: not available for sharded problems"); return false; }
    if(!solver_build_workspace(P)) return false;
    // every solve with the factor takes the forward panels' tiles (schur_solve_pieces): more than 48 KB of shared memory
    if(!set_max_dynamic_smem<panels_forward_tiled_kernel>((int)kSolveTileSmem)) return false;
    SolverWorkspace* ws = P->ws.get();
    NormalBuffers& N = ws->N;
    cudaStream_t s = P->stream;
    int nl = 0;
    if(!problem_evaluate(P, P->cur, true, true) ||
       !normal_assemble(P->dp, N, P->op[P->cur], P->d_rowptr, 0., s, &nl)) return false;
    int h_info[2] = {0, 0}, h_bad = 0;
    if(N.n_c > 0 && !chol_factor(N.S, N.ldS, N.n_c, ws->invL, N.info + 1, s, &nl, &ws->chol)) return false;
    clear_aug_rows_kernel<<<(N.ldS + 255) / 256, 256, 0, s>>>(N, N.n_c, ws->invL);
    int* d_bad = nullptr;
    F->arena.release();
    if(!F->arena.alloc(&F->ia_L, 3 * (size_t)(N.n_r > 0 ? N.n_r : 1), true) || !F->arena.alloc(&F->ia_first, 2 * (size_t)(N.n_r > 0 ? N.n_r : 1), true) ||
       !F->arena.alloc(&F->minmax, 2) || !F->arena.alloc(&d_bad, 1, true)) return false;
    if(N.n_r > 0)
    {
        inactive_blocks_kernel<<<(N.n_r + 255) / 256, 256, 0, s>>>(P->dp, N, P->op[P->cur].Jval, F->ia_L, F->ia_first, d_bad);
        rank_inactive_kernel<<<1, 32, 0, s>>>(N, F->ia_first + N.n_r);
    }
    if(cudaMemcpyAsync(h_info, N.info, sizeof(h_info), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
       cudaMemcpyAsync(&h_bad, d_bad, sizeof(int), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
       cudaStreamSynchronize(s) != cudaSuccess)
    { set_error("structured factorization: device failure"); return false; }
    if(h_info[0] != 0 || h_info[1] != 0 || h_bad != 0) { set_error("JtJ is not positive definite"); return false; }
    F->n = P->L.Nstate;
    F->Nelim = N.e1 - N.e0;
    return true;
}

}  // namespace mb200
using namespace mb200;

// The structured factorization of the problem the LAST mrcal_optimizer_callback() call evaluated (this call takes that
// device problem over). NULL -- with mrcal_b200_last_error() saying why -- if there is none, if it is sharded, or if
// JtJ is not positive definite (which, as in the reference, is not an error for the caller: mrcal-pywrap.c:1981-1988)
extern "C" mrcal_b200_factorization_t* mrcal_b200_factorization_create_from_last_callback(void)
{
    mrcal_b200_problem_t* P = capi_steal_cached_problem();
    if(P == nullptr) { set_error("no mrcal_optimizer_callback() problem to factor"); return nullptr; }
    std::unique_ptr<mrcal_b200_factorization> F(new mrcal_b200_factorization());
    F->P = P;
    if(!schur_factor_build(P, F.get()))
    {
        const std::string why = get_error();
        schur_factorization_release(F.get());
        set_error("%s", why.c_str());
        return nullptr;
    }
    return F.release();
}
