// Internal: the solver workspace (solver.cu) for the pieces that build on it (factorization_schur.cu)
#pragma once
#include <vector>

#include "chol.h"
#include "normal.h"
#include "problem_impl.h"

namespace mb200 {

struct SolverWorkspace
{
    DeviceArena arena;
    NormalBuffers N{};
    double* invL = nullptr;
    double* rhs = nullptr;        // [ldS] compact solution
    double* step_gn = nullptr;    // [Nstate]
    double* step = nullptr;       // [Nstate]
    double* scal = nullptr;       // [64] device scalars
    double* h_scal = nullptr;     // pinned mirror
    int*    h_info = nullptr;     // pinned
    int*    ictl = nullptr;       // [8] device control flags of the step logic
    int*    h_ictl = nullptr;     // pinned
    double* h_scal_dev = nullptr; // the device's addresses of the pinned mirrors (read_back_kernel writes them directly)
    int*    h_info_dev = nullptr;
    CholScratch chol;             // this workspace's own flags of the persistent factorization kernels
    std::vector<cudaEvent_t> ev;
    ~SolverWorkspace()
    {
        chol_forget_graphs(N.S);
        if(N.wi_A) cudaFree(N.wi_A);
        for(int k = 0; k < 2; k++)
        {
            if(N.s_side[k]) cudaStreamDestroy(N.s_side[k]);
            if(N.ev_join[k]) cudaEventDestroy(N.ev_join[k]);
        }
        if(N.ev_fork) cudaEventDestroy(N.ev_fork);
        if(h_scal) cudaFreeHost(h_scal);
        if(h_info) cudaFreeHost(h_info);
        chol_scratch_destroy(&chol);
        for(auto e : ev) cudaEventDestroy(e);
    }
};

bool solver_build_workspace(mrcal_b200_problem* P);   // solver.cu

}  // namespace mb200

// The factorization object of the C-ABI: either a dense Cholesky of JtJ for an arbitrary CSR J (factorization.cu),
// or the structured factor of a calibration problem (factorization_schur.cu), which owns that problem
struct mrcal_b200_factorization
{
    mb200::DeviceArena arena;
    cudaStream_t stream = nullptr;
    int n = 0, npad = 0;
    double* H = nullptr;      // npad x npad, lower: L after factorization
    double* invL = nullptr;
    int*    info = nullptr;
    double* minmax = nullptr;
    mb200::CholScratch chol;  // this object's own flags of the persistent kernels
    // structured variant
    mrcal_b200_problem* P = nullptr;   // owned
    double* ia_L = nullptr;            // [n_r][3] Cholesky factor (l11, l21, l22) of each inactive unknown's regularization block
    int*    ia_first = nullptr;        // [n_r] is this the first unknown of its block (1), the second (2), alone (3), or active (0)
    int     Nelim = 0;
};

namespace mb200 {
// What solve_xt_JtJ_bt(sys=...) does with a factor P JtJ P' = L L' (D = I): the solve with L, the one with L', and
// whether the input and the output are in the permuted order. The dense factor has P = I.
// sys_steps (factorization.cu): false, with the error set, for an unknown sys
struct SysSteps { bool fwd, bwd, permuted_in, permuted_out; };
bool sys_steps(int sys, SysSteps* st);

bool schur_factorization_solve(mrcal_b200_factorization* F, double* out, const double* bt, int Nrhs, const SysSteps& st);
double schur_factorization_rcond(mrcal_b200_factorization* F);
void schur_factorization_release(mrcal_b200_factorization* F);
bool schur_factor_build(mrcal_b200_problem* P, mrcal_b200_factorization* F);
// The triangular solves with the structured factor, in place on the pieces of the permuted right-hand sides as
// NormalBuffers::slot() lays them out. forward: L_D, the panels, L_S, L_I. backward: L_I', L_S', then (all) the panels
// and L_D'; `shared` stops after L_S', with X on the shared unknowns only
enum class BackSolve { none, shared, all };
bool schur_solve_pieces(const mrcal_b200_factorization* F, double* Bf, double* Bs, double* Bi, int Nrhs, bool forward,
                        BackSolve backward, cudaStream_t s);
// csr_ops.cu
bool csr_stable_transpose(const int* p, const int* col, int Nrows, int nnz, int Ncols, DeviceArena& arena,
                          int** tp, int** tsrc, int** trow, cudaStream_t s);
// cross_reprojection.cu: K = drt/db_packed (6 x Nstate, row-major) into device memory; evaluate: evaluate the
// Jacobian at the current state first (false: the caller just did)
bool cross_reprojection_K(mrcal_b200_problem* P, int icam_intrinsics, bool evaluate, double* d_K);
}  // namespace mb200
