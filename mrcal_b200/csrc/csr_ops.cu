// Consumers of the sparse Jacobian downstream of the solve: Jt*x and A Jt J At
// for a CSR J held on the GPU. These are what the reference's projection-
// uncertainty code calls through its numpysane wrappers
//     _Jt_x           mrcal-genpywrap.py:640-731
//     _A_Jt_J_At      mrcal-genpywrap.py:477-567
//     _A_Jt_J_At__2   mrcal-genpywrap.py:569-638   (the same with A.shape = (2,Nstate))
// (mrcal/model_analysis.py:716-870 is the caller).
//
// Both results are sums over the rows of J. They are formed in a FIXED order:
//   Jt x       through a stable transpose of J (built once per matrix): every output sums its
//              column's entries in row order -- the order the reference's loop adds them in,
//              so the result is bit-identical to the reference's.
//   A Jt J At  M = J A' (one thread per row and output column), then M'M by per-block partial
//              sums over contiguous row ranges, added up in block order.
#include <memory>

#include "problem_impl.h"

struct mrcal_b200_csr
{
    mb200::DeviceArena arena;
    cudaStream_t stream = nullptr;
    int Nrows = 0, Ncols = 0, nnz = 0;
    int* p = nullptr; int* i = nullptr; double* x = nullptr;
    // stable transpose (CSC): built on first use
    bool have_t = false;
    int* tp = nullptr;      // [Ncols+1]
    int* tsrc = nullptr;    // [nnz] position in the CSR arrays
    int* trow = nullptr;    // [nnz] row of each entry
};

namespace mb200 {

constexpr int kTChunks = 2048;

// entry e belongs to row r: rows[e] = r
__global__ void csr_expand_rows_kernel(const int* __restrict__ p, int Nrows, int* __restrict__ rows)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if(r >= Nrows) return;
    for(int e = p[r]; e < p[r + 1]; e++) rows[e] = r;
}
// chunk c of the entries: how many fall in each column (one thread per chunk, sequential: order matters below)
__global__ void csr_chunk_hist_kernel(const int* __restrict__ col, int nnz, int Ncols, int* __restrict__ hist /*[kTChunks][Ncols]*/)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= kTChunks) return;
    const long per = ((long)nnz + kTChunks - 1) / kTChunks;
    const long e0 = (long)c * per, e1 = min((long)nnz, e0 + per);
    int* h = hist + (size_t)c * Ncols;
    for(long e = e0; e < e1; e++) h[col[e]]++;
}
// per column: exclusive scan over the chunks; column totals -> tp[col+1]
__global__ void csr_chunk_scan_kernel(int Ncols, int* __restrict__ hist, int* __restrict__ tp)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= Ncols) return;
    int run = 0;
    for(int k = 0; k < kTChunks; k++) { const int v = hist[(size_t)k * Ncols + c]; hist[(size_t)k * Ncols + c] = run; run += v; }
    tp[c + 1] = run;
}
__global__ void csr_colptr_scan_kernel(int Ncols, int* __restrict__ tp)
{
    // one thread: Ncols is the number of state variables (<= a few 10^4)
    if(blockIdx.x != 0 || threadIdx.x != 0) return;
    tp[0] = 0;
    for(int c = 0; c < Ncols; c++) tp[c + 1] += tp[c];
}
__global__ void csr_chunk_fill_kernel(const int* __restrict__ col, const int* __restrict__ rows, int nnz, int Ncols,
                                      int* __restrict__ hist, const int* __restrict__ tp, int* __restrict__ tsrc, int* __restrict__ trow)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= kTChunks) return;
    const long per = ((long)nnz + kTChunks - 1) / kTChunks;
    const long e0 = (long)c * per, e1 = min((long)nnz, e0 + per);
    int* h = hist + (size_t)c * Ncols;
    for(long e = e0; e < e1; e++)
    {
        const int cc = col[e];
        const int pos = tp[cc] + h[cc]++;
        tsrc[pos] = (int)e;
        trow[pos] = rows[e];
    }
}

// y[c] = sum over the entries of column c, in row order. One warp per column would reorder the sum: one thread each.
// Product and sum are rounded separately (no fused multiply-add), as the reference's x86 loop does
// (mrcal-genpywrap.py:505-520): the result is the same to the last bit
__global__ void csr_jt_x_kernel(const int* __restrict__ tp, const int* __restrict__ tsrc, const int* __restrict__ trow,
                                const double* __restrict__ val, const double* __restrict__ x, int Ncols, double* __restrict__ y)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= Ncols) return;
    double s = 0.;
    for(int k = tp[c]; k < tp[c + 1]; k++) s = __dadd_rn(s, __dmul_rn(val[tsrc[k]], x[trow[k]]));
    y[c] = s;
}

// M[r][k] = sum_e J[r][e] A[k][col_e]
__global__ void csr_j_at_kernel(const int* __restrict__ p, const int* __restrict__ col, const double* __restrict__ val,
                                const double* __restrict__ A, int Nx, int Nstate, int Nrows, double* __restrict__ M)
{
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrows * Nx) return;
    const int r = (int)(idx / Nx), k = (int)(idx - (long)r * Nx);
    const double* a = A + (size_t)k * Nstate;
    double s = 0.;
    for(int e = p[r]; e < p[r + 1]; e++) s += a[col[e]] * val[e];
    M[idx] = s;
}
// partial[b][i][j] = sum over the rows of block b of M[r][i] M[r][j]; thread (i,j) walks the rows in order
__global__ void csr_mtm_partial_kernel(const double* __restrict__ M, int Nx, int Nrows, int rows_per_block, double* __restrict__ partial)
{
    const int r0 = blockIdx.x * rows_per_block, r1 = min(Nrows, r0 + rows_per_block);
    for(int e = threadIdx.x; e < Nx * Nx; e += blockDim.x)
    {
        const int i = e / Nx, j = e - i * Nx;
        double s = 0.;
        if(j >= i)
            for(int r = r0; r < r1; r++) s += M[(size_t)r * Nx + i] * M[(size_t)r * Nx + j];
        partial[(size_t)blockIdx.x * Nx * Nx + e] = s;
    }
}
__global__ void csr_mtm_final_kernel(const double* __restrict__ partial, int Nx, int nblocks, double* __restrict__ out)
{
    const int e = blockIdx.x * blockDim.x + threadIdx.x;
    if(e >= Nx * Nx) return;
    const int i = e / Nx, j = e - i * Nx;
    const int src = j >= i ? e : j * Nx + i;   // the upper triangle was computed; mirror it
    double s = 0.;
    for(int b = 0; b < nblocks; b++) s += partial[(size_t)b * Nx * Nx + src];
    out[e] = s;
}

// The stable transpose (CSC) of a device CSR matrix: column c's entries in row order at [tp[c], tp[c+1]), with their
// positions in the CSR arrays (tsrc) and their rows (trow). The arrays are allocated from `arena`
bool csr_stable_transpose(const int* p, const int* col, int Nrows, int nnz, int Ncols, DeviceArena& arena,
                          int** tp, int** tsrc, int** trow, cudaStream_t s)
{
    DeviceArena tmp;
    int *rows = nullptr, *hist = nullptr;
    if(!arena.alloc(tp, (size_t)Ncols + 1, true) || !arena.alloc(tsrc, nnz) || !arena.alloc(trow, nnz) ||
       !tmp.alloc(&rows, nnz) || !tmp.alloc(&hist, (size_t)kTChunks * Ncols, true))
        return false;
    if(Nrows > 0) csr_expand_rows_kernel<<<(Nrows + 255) / 256, 256, 0, s>>>(p, Nrows, rows);
    csr_chunk_hist_kernel<<<(kTChunks + 127) / 128, 128, 0, s>>>(col, nnz, Ncols, hist);
    csr_chunk_scan_kernel<<<(Ncols + 127) / 128, 128, 0, s>>>(Ncols, hist, *tp);
    csr_colptr_scan_kernel<<<1, 32, 0, s>>>(Ncols, *tp);
    csr_chunk_fill_kernel<<<(kTChunks + 127) / 128, 128, 0, s>>>(col, rows, nnz, Ncols, hist, *tp, *tsrc, *trow);
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));   // tmp goes out of scope
    return true;
}

static bool build_transpose(mrcal_b200_csr* J)
{
    if(J->have_t) return true;
    if(!csr_stable_transpose(J->p, J->i, J->Nrows, J->nnz, J->Ncols, J->arena, &J->tp, &J->tsrc, &J->trow, J->stream)) return false;
    J->have_t = true;
    return true;
}

}  // namespace mb200
using namespace mb200;

extern "C" mrcal_b200_csr_t* mrcal_b200_csr_create(const int32_t* Jrowptr, const int32_t* Jcolidx, const double* Jval, int Nrows, int Ncols)
{
    if(mrcal_b200_device_count() <= 0) { set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback"); return nullptr; }
    if(Nrows < 0 || Ncols <= 0 || Jrowptr == nullptr) { set_error("csr: bad J"); return nullptr; }
    const int nnz = Jrowptr[Nrows];
    for(int r = 0; r < Nrows; r++)
        if(Jrowptr[r + 1] < Jrowptr[r]) { set_error("csr: row pointers must not decrease"); return nullptr; }
    for(int e = 0; e < nnz; e++)
        if(Jcolidx[e] < 0 || Jcolidx[e] >= Ncols) { set_error("csr: J has a column index out of range"); return nullptr; }
    std::unique_ptr<mrcal_b200_csr> J(new mrcal_b200_csr());
    J->Nrows = Nrows; J->Ncols = Ncols; J->nnz = nnz;
    if(cudaStreamCreateWithFlags(&J->stream, cudaStreamNonBlocking) != cudaSuccess) { set_error("cudaStreamCreate failed"); return nullptr; }
    bool ok = J->arena.alloc(&J->p, (size_t)Nrows + 1) && J->arena.alloc(&J->i, nnz) && J->arena.alloc(&J->x, nnz) &&
              cudaMemcpyAsync(J->p, Jrowptr, ((size_t)Nrows + 1) * sizeof(int), cudaMemcpyHostToDevice, J->stream) == cudaSuccess &&
              (nnz == 0 || (cudaMemcpyAsync(J->i, Jcolidx, (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice, J->stream) == cudaSuccess &&
                            cudaMemcpyAsync(J->x, Jval, (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice, J->stream) == cudaSuccess)) &&
              cudaStreamSynchronize(J->stream) == cudaSuccess;
    if(!ok) { set_error("csr: upload failed: %s", cudaGetErrorString(cudaGetLastError())); cudaStreamDestroy(J->stream); return nullptr; }
    return J.release();
}

extern "C" void mrcal_b200_csr_destroy(mrcal_b200_csr_t* J)
{
    if(J == nullptr) return;
    if(J->stream) cudaStreamSynchronize(J->stream);
    J->arena.release();
    if(J->stream) cudaStreamDestroy(J->stream);
    delete J;
}

extern "C" bool mrcal_b200_csr_Jt_x(mrcal_b200_csr_t* J, double* out, const double* xt)
{
    if(!build_transpose(J)) return false;
    DeviceArena tmp;
    double *d_x, *d_y;
    if(!tmp.alloc(&d_x, J->Nrows) || !tmp.alloc(&d_y, J->Ncols)) return false;
    cudaStream_t s = J->stream;
    if(J->Nrows > 0) MB200_CUDA_CHECK(cudaMemcpyAsync(d_x, xt, (size_t)J->Nrows * sizeof(double), cudaMemcpyHostToDevice, s));
    csr_jt_x_kernel<<<(J->Ncols + 127) / 128, 128, 0, s>>>(J->tp, J->tsrc, J->trow, J->x, d_x, J->Ncols, d_y);
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpyAsync(out, d_y, (size_t)J->Ncols * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" bool mrcal_b200_csr_A_Jt_J_At(mrcal_b200_csr_t* J, double* out, const double* A, int Nx, int Nleading_rows_J)
{
    if(Nleading_rows_J <= 0) { set_error("Nleading_rows_J must be passed, and must be > 0"); return false; }
    if(Nleading_rows_J > J->Nrows) { set_error("Nleading_rows_J = %d exceeds the %d rows of J", Nleading_rows_J, J->Nrows); return false; }
    if(Nx <= 0) { set_error("A must have at least one row"); return false; }
    const int Nrows = Nleading_rows_J;
    const int rows_per_block = 2048;
    const int nblocks = (Nrows + rows_per_block - 1) / rows_per_block;
    DeviceArena tmp;
    double *d_A, *d_M, *d_part, *d_out;
    if(!tmp.alloc(&d_A, (size_t)Nx * J->Ncols) || !tmp.alloc(&d_M, (size_t)Nrows * Nx) ||
       !tmp.alloc(&d_part, (size_t)nblocks * Nx * Nx) || !tmp.alloc(&d_out, (size_t)Nx * Nx))
        return false;
    cudaStream_t s = J->stream;
    MB200_CUDA_CHECK(cudaMemcpyAsync(d_A, A, (size_t)Nx * J->Ncols * sizeof(double), cudaMemcpyHostToDevice, s));
    const long total = (long)Nrows * Nx;
    csr_j_at_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(J->p, J->i, J->x, d_A, Nx, J->Ncols, Nrows, d_M);
    csr_mtm_partial_kernel<<<nblocks, 256, 0, s>>>(d_M, Nx, Nrows, rows_per_block, d_part);
    csr_mtm_final_kernel<<<(Nx * Nx + 127) / 128, 128, 0, s>>>(d_part, Nx, nblocks, d_out);
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpyAsync(out, d_out, (size_t)Nx * Nx * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}
