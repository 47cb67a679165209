// Internal: dense Cholesky on the device (chol_dataflow.cu, chol.cu)
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

constexpr int kCholBlock = 64;
inline int chol_padded(int n) { return ((n + kCholBlock - 1) / kCholBlock) * kCholBlock; }

// Up to 8 device ranges of 32-bit words, each set to one value, in ONE launch (fill_words, chol.cu). The trust-region
// step clears its flags, counters and accumulators a few words at a time; one cudaMemsetAsync per buffer costs a launch
// gap each on the step's critical path
struct WordFill
{
    unsigned* p[8];
    long long n[8];
    unsigned v[8];
    int count = 0;
    void add(void* ptr, size_t bytes, unsigned value = 0u)
    {
        if(bytes == 0) return;
        p[count] = (unsigned*)ptr; n[count] = (long long)(bytes / 4); v[count] = value; count++;
    }
};
bool fill_words(const WordFill& f, cudaStream_t s);

// Scratch of the persistent kernels (tile flags, the solution slots of the backward substitution) for systems of up to
// npad_max unknowns: one per owner of a factorization, so that two factorizations in flight never share flags
struct CholScratch { int* flags = nullptr; double* xbuf = nullptr; int npad_max = 0; };
bool chol_scratch_create(CholScratch* sc, int npad_max);
void chol_scratch_destroy(CholScratch* sc);

// chol_dataflow.cu, one persistent kernel each (the factorization: up to npad = 8192):
//
// A: row-major npad x npad, lower triangle holds the matrix; rows/cols >= nreal
// are padding (1 on the diagonal). On return the lower triangle holds L.
// invL: [npad/64][64*64] inverses of the diagonal blocks of L.
// d_info: device int; 0 if positive definite, else 1 + index of the first bad pivot.
// scratch: the caller's, for at least npad. d_run_if: device flag; 0 there = do nothing (nullptr: always run)
bool chol_factor(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch,
                 CholScratch* scratch, const int* d_run_if = nullptr);

// Only the backward half, L' Z = B in place, one right-hand side B[0..npad). d_info (may be the factorization's): set
// to -9 if the persistent kernel gave up waiting (never expected; the alternative would be to hang the GPU)
bool chol_solve_backward(const double* L, int npad, const double* invL, double* B, int* d_info, cudaStream_t s, int* nlaunch,
                         CholScratch* scratch, const int* d_run_if = nullptr);

// chol.cu: the multi-kernel factorization, which chol_factor runs above npad = 8192 (same arguments; no scratch)
bool chol_factor_blocked(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch);

// Right-hand sides per tile of the many-right-hand-side DMMA kernels (chol.cu's tiled solve, the structured factor's
// forward panels), the row stride (doubles) of their tiles staged in shared memory, and that shared memory
constexpr int kSolveTile = 32, kSolveTileLd = 68;
constexpr size_t kSolveTileSmem = (size_t)(kSolveTile + kCholBlock) * kSolveTileLd * sizeof(double);

// chol.cu: solve L L' X = B in place for nrhs right-hand sides stored as rows B[r][0..npad); unknowns >= nreal are
// padding, read as zero whatever B holds there. parts: 1 = only L Y = B, 2 = only L' X = B, 3 = both. The kernels are
// chosen by nrhs; kernels (tests only): 1 forces the per-block kernels, 2 the tiled one
bool chol_solve(const double* L, int npad, int nreal, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s,
                int* nlaunch, int parts = 3, int kernels = 0);

// drop cached CUDA graphs that reference this buffer (call before freeing it)
void chol_forget_graphs(const void* A);

double chol_debug_time(int n, int reps, int what);
bool chol_debug_potrf_stamps(long long* out64);
// test aids: chol_dataflow.cu, chol.cu
bool chol_debug_factor(const double* A0, int n, int nreal, int path, double* L_out, double* invL_out, int* info_out, int* grid_out);
bool chol_debug_solve(const double* L, const double* invL, int npad, int nreal, double* B, int nrhs, int parts, int kernel);

// d_out2[0] = min, d_out2[1] = max of diag(L)[0..nreal)
bool chol_diag_minmax(const double* L, int npad, int nreal, double* d_out2, cudaStream_t s);

}  // namespace mb200
