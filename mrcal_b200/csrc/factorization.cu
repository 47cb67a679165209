// The factorization object: Cholesky of JtJ for an arbitrary CSR J, on the GPU.
// Stands in for mrcal.CHOLMOD_factorization (mrcal-pywrap.c:110-649): built
// from J (:196-212), solve_xt_JtJ_bt(sys='A') (:425-578), rcond (:580-593).
// The known-answer test is the reference's test/test-CHOLMOD-factorization.py.
//
// J is arbitrary here (the object is also constructible from user matrices), so
// no block structure is assumed: JtJ is accumulated densely and factored with
// the same DMMA Cholesky the solver uses.
#include "solver_internal.h"

namespace mb200 {

// one warp per row of J: lower triangle of the row's outer product
__global__ void jtj_rows_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const double* __restrict__ val,
                                int Nrows, double* __restrict__ H, int ld)
{
    const int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if(row >= Nrows) return;
    const int j0 = rowptr[row], nn = rowptr[row + 1] - j0;
    for(int e = lane; e < nn * nn; e += 32)
    {
        const int a = e / nn, b = e - a * nn;
        const int ca = col[j0 + a], cb = col[j0 + b];
        // each unordered pair once; duplicates of a column within a row are legal in CSR
        if(b > a) continue;
        const double v = val[j0 + a] * val[j0 + b];
        if(v == 0.) continue;
        if(ca == cb) atomicAdd(&H[(size_t)ca * ld + ca], (a == b) ? v : 2. * v);
        else if(ca > cb) atomicAdd(&H[(size_t)ca * ld + cb], v);
        else             atomicAdd(&H[(size_t)cb * ld + ca], v);
    }
}

__global__ void pad_diagonal_kernel(double* H, int ld, int n, int npad)
{
    const int i = n + blockIdx.x * blockDim.x + threadIdx.x;
    if(i < npad) H[(size_t)i * ld + i] = 1.;
}

}  // namespace mb200
using namespace mb200;

extern "C" mrcal_b200_factorization_t*
mrcal_b200_factorization_create(const int32_t* Jrowptr, const int32_t* Jcolidx, const double* Jval, int Nrows, int Ncols)
{
    if(mrcal_b200_device_count() <= 0) { set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback"); return nullptr; }
    if(Nrows < 0 || Ncols <= 0 || Jrowptr == nullptr) { set_error("factorization: bad J"); return nullptr; }
    const int nnz = Jrowptr[Nrows];
    for(int i = 0; i < nnz; i++)
        if(Jcolidx[i] < 0 || Jcolidx[i] >= Ncols) { set_error("factorization: J has a column index out of range"); return nullptr; }

    std::unique_ptr<mrcal_b200_factorization> F(new mrcal_b200_factorization());
    F->n = Ncols;
    F->npad = chol_padded(Ncols);
    if(cudaStreamCreateWithFlags(&F->stream, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate failed"); return nullptr; }
    cudaStream_t s = F->stream;
    int *d_p, *d_i; double* d_x;
    DeviceArena tmp;
    if(!(F->arena.alloc(&F->H, (size_t)F->npad * F->npad, true) &&
         F->arena.alloc(&F->invL, (size_t)F->npad * kCholBlock) && F->arena.alloc(&F->info, 1, true) &&
         F->arena.alloc(&F->minmax, 2) &&
         tmp.alloc(&d_p, (size_t)Nrows + 1) && tmp.alloc(&d_i, nnz) && tmp.alloc(&d_x, nnz)))
    { cudaStreamDestroy(s); return nullptr; }
    cudaMemcpyAsync(d_p, Jrowptr, ((size_t)Nrows + 1) * sizeof(int), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_i, Jcolidx, (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_x, Jval, (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice, s);
    if(Nrows > 0) jtj_rows_kernel<<<((size_t)Nrows * 32 + 255) / 256, 256, 0, s>>>(d_p, d_i, d_x, Nrows, F->H, F->npad);
    if(F->npad > F->n) pad_diagonal_kernel<<<(F->npad - F->n + 255) / 256, 256, 0, s>>>(F->H, F->npad, F->n, F->npad);
    int info = -1;
    bool ok = chol_scratch_create(&F->chol, F->npad) && chol_factor(F->H, F->npad, F->n, F->invL, F->info, s, nullptr, &F->chol) &&
              cudaMemcpyAsync(&info, F->info, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
              cudaStreamSynchronize(s) == cudaSuccess;
    if(!ok)
    {
        set_error("factorization failed on the device: %s", cudaGetErrorString(cudaGetLastError()));
        chol_scratch_destroy(&F->chol);
        cudaStreamDestroy(s);
        return nullptr;
    }
    if(info != 0)
    {
        // the reference reports this the same way: no object (mrcal-pywrap.c:199-212)
        set_error("JtJ is not positive definite (pivot %d)", info - 1);
        chol_scratch_destroy(&F->chol);
        cudaStreamDestroy(s);
        return nullptr;
    }
    return F.release();
}

extern "C" void mrcal_b200_factorization_destroy(mrcal_b200_factorization_t* F)
{
    if(F == nullptr) return;
    if(F->P != nullptr) { schur_factorization_release(F); delete F; return; }
    if(F->stream) { cudaStreamSynchronize(F->stream); }
    chol_forget_graphs(F->H);
    chol_scratch_destroy(&F->chol);
    F->arena.release();
    if(F->stream) cudaStreamDestroy(F->stream);
    delete F;
}

extern "C" bool mrcal_b200_factorization_solve_xt_JtJ_bt(mrcal_b200_factorization_t* F, double* out, const double* bt, int Nrhs)
{
    return mrcal_b200_factorization_solve_sys(F, out, bt, Nrhs, MRCAL_B200_SYS_A);
}

// The factorization is P JtJ P' = L D L' with P = I (no fill-reducing permutation: the matrix is dense here),
// L the Cholesky factor and D = I. The reference's CHOLMOD has its own P and a genuine D (simplicial LDL'), so
// the individual pieces differ from CHOLMOD's -- but every identity between them holds, which is what callers
// use (mrcal/model_analysis.py:837-841: sys='P', then 'L', then 'D')
namespace mb200 {
bool sys_steps(int sys, SysSteps* st)
{
    switch(sys)
    {
    case MRCAL_B200_SYS_A:    *st = {true,  true,  false, false}; return true;
    case MRCAL_B200_SYS_LDLt: *st = {true,  true,  true,  true};  return true;
    case MRCAL_B200_SYS_LD: case MRCAL_B200_SYS_L:   *st = {true,  false, true, true}; return true;
    case MRCAL_B200_SYS_DLt: case MRCAL_B200_SYS_Lt: *st = {false, true,  true, true}; return true;
    case MRCAL_B200_SYS_D:    *st = {false, false, true,  true};  return true;
    case MRCAL_B200_SYS_P:    *st = {false, false, false, true};  return true;   // out = P b
    case MRCAL_B200_SYS_Pt:   *st = {false, false, true,  false}; return true;   // out = P' b
    default: set_error("Unknown sys %d given", sys); return false;
    }
}
}  // namespace mb200

extern "C" bool mrcal_b200_factorization_solve_sys(mrcal_b200_factorization_t* F, double* out, const double* bt, int Nrhs, int sys)
{
    if(Nrhs <= 0) return true;
    SysSteps st;
    if(!sys_steps(sys, &st)) return false;
    if(F->P != nullptr) return schur_factorization_solve(F, out, bt, Nrhs, st);
    const int parts = (st.fwd ? 1 : 0) | (st.bwd ? 2 : 0);
    if(parts == 0)
    {
        if(out != bt) memcpy(out, bt, (size_t)Nrhs * F->n * sizeof(double));
        return true;
    }
    DeviceArena tmp;
    double* d_b;
    if(!tmp.alloc(&d_b, (size_t)Nrhs * F->npad, true)) return false;
    cudaStream_t s = F->stream;
    MB200_CUDA_CHECK(cudaMemcpy2DAsync(d_b, (size_t)F->npad * sizeof(double), bt, (size_t)F->n * sizeof(double),
                                       (size_t)F->n * sizeof(double), Nrhs, cudaMemcpyHostToDevice, s));
    if(!chol_solve(F->H, F->npad, F->n, F->invL, d_b, F->npad, Nrhs, s, nullptr, parts)) return false;
    MB200_CUDA_CHECK(cudaMemcpy2DAsync(out, (size_t)F->n * sizeof(double), d_b, (size_t)F->npad * sizeof(double),
                                       (size_t)F->n * sizeof(double), Nrhs, cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" double mrcal_b200_factorization_rcond(mrcal_b200_factorization_t* F)
{
    // For an LL' factorization cholmod_rcond() returns (min diag(L) / max diag(L))^2
    if(F->P != nullptr) return schur_factorization_rcond(F);
    double mm[2] = {0., 0.};
    if(!chol_diag_minmax(F->H, F->npad, F->n, F->minmax, F->stream)) return -1.;
    if(cudaMemcpyAsync(mm, F->minmax, sizeof(mm), cudaMemcpyDeviceToHost, F->stream) != cudaSuccess ||
       cudaStreamSynchronize(F->stream) != cudaSuccess)
        return -1.;
    if(!(mm[1] > 0.)) return 0.;
    const double r = mm[0] / mm[1];
    return r * r;
}

// Timing aid for kernel development (scripts/time_cholesky.py); not declared in the public header.
// what: 0 the factorization, 1 the backward substitution
extern "C" double mrcal_b200_debug_time_cholesky(int n, int reps, int what)
{
    return chol_debug_time(n, reps, what);
}
namespace mb200 { bool chol_debug_spine_stamps(int n, long long* out, int nmax); }
extern "C" bool mrcal_b200_debug_spine_stamps(int n, long long* out, int nmax) { return mb200::chol_debug_spine_stamps(n, out, nmax); }
extern "C" bool mrcal_b200_debug_potrf_stamps(long long* out64)
{
    return chol_debug_potrf_stamps(out64);
}
// Test entry points of the dense Cholesky kernels (tests/test_cholesky_gpu.py); not declared in the public header
extern "C" bool mrcal_b200_debug_cholesky(const double* A, int n, int nreal, int path, double* L_out, double* invL_out,
                                          int* info_out, int* grid_out)
{
    return chol_debug_factor(A, n, nreal, path, L_out, invL_out, info_out, grid_out);
}
extern "C" bool mrcal_b200_debug_chol_solve(const double* L, const double* invL, int npad, int nreal, double* B, int nrhs,
                                            int parts, int kernel)
{
    return chol_debug_solve(L, invL, npad, nreal, B, nrhs, parts, kernel);
}
