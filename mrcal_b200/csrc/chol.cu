// Kernel family 2b: dense Cholesky factorization and triangular solves of the
// reduced (camera) normal equations, fp64, on the DMMA (fp64 tensor) pipe.
//
// Stands in for what the reference gets from CHOLMOD through libdogleg
// (cholmod_factorize / cholmod_solve; call sites mrcal.c:6435 and
// mrcal-pywrap.c:196-212, 557). The reference factors the full sparse JtJ with
// a simplicial LDL'; here the frame/point blocks have already been eliminated
// (normal.cu), what is left is small and dense, and it is factored as L L'
// with a two-level blocked right-looking algorithm:
//
//   for each 256-column outer panel:
//       for each 64-column inner block of it:
//           potrf_diag   one CTA: factor the 64x64 diagonal block in shared
//                        memory, and invert the factor (potrf_block.cuh)
//           trsm         rows below: X <- A inv(L_kk)'   (small GEMM)
//           syrk (K=64)  update of the REST OF THE PANEL only
//       syrk (K=256)     one DMMA update of the whole trailing matrix
//
// Storage: row-major n x n, lower triangle, n padded to a multiple of 64 (the
// caller puts 1 on the padding diagonal). Rows are K-contiguous, which is what
// mma.sync.m8n8k4.row.col.f64 wants for both operands of  C -= P P'.
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

#include "chol.h"
#include "potrf_block.cuh"
#include "problem.h"

namespace mb200 {

constexpr int NB = 64;     // inner block
constexpr int NBO = 256;   // outer panel

////////////////////////////////////////////////////////////////////////////////
// diagonal block: Cholesky + inverse of the factor, one CTA (potrf_block.cuh)
////////////////////////////////////////////////////////////////////////////////
template <bool STAMP>
__global__ void __launch_bounds__(256, 1)
potrf_diag_kernel(double* __restrict__ A, int ld, int k0, double* __restrict__ invL, int* __restrict__ info, int nreal, long long* stamps)
{
    extern __shared__ __align__(16) unsigned char dsm_raw[];
    PotrfSmem& sm = *reinterpret_cast<PotrfSmem*>(dsm_raw);
    const int tid = threadIdx.x;
    if(STAMP && tid == 0) stamps[30] = clock64();
    {
        // all 16 loads of a thread in flight at once
        double v[NB * NB / 256];
#pragma unroll
        for(int q = 0; q < NB * NB / 256; q++)
        {
            const int e = tid + q * 256, r = e / NB, c = e % NB;
            v[q] = c <= r ? A[(size_t)(k0 + r) * ld + k0 + c] : 0.;
        }
#pragma unroll
        for(int q = 0; q < NB * NB / 256; q++)
        {
            const int e = tid + q * 256;
            sm.L[(e / NB) * PLD + e % NB] = v[q];
        }
    }
    potrf_block<STAMP>(sm, info, k0, nreal, stamps);
    for(int e = tid; e < NB * NB; e += 256)
    {
        const int r = e / NB, c = e % NB;
        if(c <= r) A[(size_t)(k0 + r) * ld + k0 + c] = sm.L[r * PLD + c];
        invL[e] = sm.X[r * PLD + c];
    }
    if(STAMP && tid == 0) stamps[31] = clock64();
}

////////////////////////////////////////////////////////////////////////////////
// panel: X[i][c] = sum_m A[i][k0+m] invL[c][m], rows i >= k0+64, in place.
// 64x64 tile per CTA, 4x4 outputs per thread; a thread's 4 columns are 16 apart so
// that a warp's shared-memory reads of invL rows fall in distinct banks
////////////////////////////////////////////////////////////////////////////////
__global__ void __launch_bounds__(256)
trsm_kernel(double* __restrict__ A, int ld, int k0, const double* __restrict__ invL, int n)
{
    extern __shared__ __align__(16) double dsm[];
    double (*sa)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(dsm);
    double (*sl)[NB + 1] = reinterpret_cast<double (*)[NB + 1]>(dsm + NB * (NB + 1));
    const int row0 = k0 + NB + blockIdx.x * NB;
    const int tid = threadIdx.x;
    for(int e = tid; e < NB * NB; e += 256)
    {
        const int i = e / NB, j = e % NB;
        sa[i][j] = A[(size_t)(row0 + i) * ld + k0 + j];
        sl[i][j] = invL[e];
    }
    __syncthreads();
    const int ti = (tid / 16) * 4, tc = tid % 16;
    double acc[4][4] = {};
#pragma unroll 8
    for(int m = 0; m < NB; m++)
    {
        double a[4], l[4];
#pragma unroll
        for(int r = 0; r < 4; r++) { a[r] = sa[ti + r][m]; l[r] = sl[tc + 16 * r][m]; }
#pragma unroll
        for(int r = 0; r < 4; r++)
#pragma unroll
            for(int c = 0; c < 4; c++) acc[r][c] += a[r] * l[c];
    }
#pragma unroll
    for(int r = 0; r < 4; r++)
#pragma unroll
        for(int c = 0; c < 4; c++) A[(size_t)(row0 + ti + r) * ld + k0 + tc + 16 * c] = acc[r][c];
    (void)n;
}

////////////////////////////////////////////////////////////////////////////////
// C(i,j) -= sum_{m in [k0,k1)} A(i,m) A(j,m)   for j in [c0,c1), i in [c0,n), i >= j
// 128x128 tiles, 8 warps (4 x 2), warp tile 32 x 64 = 4 x 8 DMMA.8x8x4 tiles.
// Operands staged through shared memory with cp.async, 3 stages of BK=16.
////////////////////////////////////////////////////////////////////////////////
constexpr int BM = 128, BK = 16, LDS = BK + 4, STAGES = 3;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid)
{
    const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    const int sz = valid ? 16 : 0;   // src-size 0: zero-fill
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// TILE = 128: 8 warps as 4 x 2, warp tile 32 x 64 (4 x 8 DMMA tiles)   -- large trailing matrices
// TILE =  64: 8 warps as 4 x 2, warp tile 16 x 32 (2 x 4 DMMA tiles)   -- small ones: 4x the CTAs, so the
//             update spreads over the whole chip instead of a few dozen SMs
template <int TILE>
__global__ void __launch_bounds__(256, TILE == 128 ? 1 : 2)
syrk_dmma_kernel(double* __restrict__ A, int ld, int n, int c0, int c1, int k0, int k1)
{
    constexpr int MI = TILE / 32, NJ = TILE / 16;    // DMMA tiles per warp along m, n
    constexpr int WM = TILE / 4, WN = TILE / 2;      // warp tile
    const int tj = blockIdx.x, ti = blockIdx.y;
    if(ti < tj) return;
    extern __shared__ __align__(16) double smem[];
    double* sA = smem;                                 // [STAGES][TILE][LDS]
    double* sB = smem + (size_t)STAGES * TILE * LDS;   // [STAGES][TILE][LDS]

    const int row0 = c0 + ti * TILE, col0 = c0 + tj * TILE;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int wm = warp >> 1, wn = warp & 1;   // 4 x 2 warps
    const int g = lane >> 2, t = lane & 3;

    double acc[MI][NJ][2];
#pragma unroll
    for(int i = 0; i < MI; i++)
#pragma unroll
        for(int j = 0; j < NJ; j++) acc[i][j][0] = acc[i][j][1] = 0.;

    const int nk = (k1 - k0) / BK;
    // TILE rows x 8 chunks of 16 B per operand per stage
    auto load_stage = [&](int stage, int kb)
    {
        const int kk = k0 + kb * BK;
#pragma unroll
        for(int it = 0; it < TILE / 32; it++)
        {
            const int chunk = tid + it * 256;
            const int r = chunk >> 3, cc = (chunk & 7) * 2;
            const int gi = row0 + r, gj = col0 + r;
            cp_async16(&sA[((size_t)stage * TILE + r) * LDS + cc], &A[(size_t)(gi < n ? gi : 0) * ld + kk + cc], gi < n);
            cp_async16(&sB[((size_t)stage * TILE + r) * LDS + cc], &A[(size_t)(gj < c1 ? gj : 0) * ld + kk + cc], gj < c1);
        }
    };
#pragma unroll
    for(int s = 0; s < STAGES - 1; s++)
    {
        if(s < nk) load_stage(s, s);
        cp_async_commit();
    }
    for(int kb = 0; kb < nk; kb++)
    {
        cp_async_wait<STAGES - 2>();
        __syncthreads();
        {
            const int nxt = kb + STAGES - 1;
            if(nxt < nk) load_stage(nxt % STAGES, nxt);
            cp_async_commit();
        }
        const double* a_s = &sA[((size_t)(kb % STAGES) * TILE + wm * WM) * LDS];
        const double* b_s = &sB[((size_t)(kb % STAGES) * TILE + wn * WN) * LDS];
#pragma unroll
        for(int ks = 0; ks < BK / 4; ks++)
        {
            double af[MI], bf[NJ];
#pragma unroll
            for(int i = 0; i < MI; i++) af[i] = a_s[(i * 8 + g) * LDS + ks * 4 + t];
#pragma unroll
            for(int j = 0; j < NJ; j++) bf[j] = b_s[(j * 8 + g) * LDS + ks * 4 + t];
#pragma unroll
            for(int i = 0; i < MI; i++)
#pragma unroll
                for(int j = 0; j < NJ; j++) dmma(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
        }
    }
    cp_async_wait<0>();

    // C -= acc, lower triangle only
#pragma unroll
    for(int i = 0; i < MI; i++)
    {
        const int gi = row0 + wm * WM + i * 8 + g;
        if(gi >= n) continue;
#pragma unroll
        for(int j = 0; j < NJ; j++)
        {
            const int gj = col0 + wn * WN + j * 8 + 2 * t;
            if(gj >= c1) continue;
            double* p = &A[(size_t)gi * ld + gj];
            if(gj + 1 <= gi)
            {
                double2 v = *reinterpret_cast<double2*>(p);
                v.x -= acc[i][j][0];
                v.y -= acc[i][j][1];
                *reinterpret_cast<double2*>(p) = v;
            }
            else if(gj <= gi)
                p[0] -= acc[i][j][0];
        }
    }
}

static const size_t kSyrkSmem = (size_t)2 * STAGES * BM * LDS * sizeof(double);   // TILE = 128; half of it for TILE = 64
static const size_t kBlockSmem = (size_t)2 * NB * (NB + 1) * sizeof(double);   // trsm
static const size_t kPotrfSmem = sizeof(PotrfSmem);

static bool configure_kernels()
{
    // cudaFuncSetAttribute is per device
    static bool configured_dev[kMaxDevices] = {};
    int dev = 0;
    MB200_CUDA_CHECK(cudaGetDevice(&dev));
    if(dev < 0 || dev >= kMaxDevices) { set_error("device index %d out of range", dev); return false; }
    bool& configured = configured_dev[dev];
    if(configured) return true;
    MB200_CUDA_CHECK(cudaFuncSetAttribute(syrk_dmma_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
    MB200_CUDA_CHECK(cudaFuncSetAttribute(syrk_dmma_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSyrkSmem));
    MB200_CUDA_CHECK(cudaFuncSetAttribute(trsm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBlockSmem));
    MB200_CUDA_CHECK(cudaFuncSetAttribute(potrf_diag_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
    MB200_CUDA_CHECK(cudaFuncSetAttribute(potrf_diag_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPotrfSmem));
    configured = true;
    return true;
}

static bool syrk_update(double* A, int ld, int n, int c0, int c1, int k0, int k1, cudaStream_t s, int* nlaunch)
{
    if(c1 <= c0 || n <= c0) return true;
    // big tiles when they fill the chip twice over, small tiles otherwise
    const long nt128 = (long)((c1 - c0 + 127) / 128) * ((n - c0 + 127) / 128);
    if(nt128 >= 2L * device_sm_count())
    {
        dim3 grid((c1 - c0 + 127) / 128, (n - c0 + 127) / 128);
        syrk_dmma_kernel<128><<<grid, 256, kSyrkSmem, s>>>(A, ld, n, c0, c1, k0, k1);
    }
    else
    {
        dim3 grid((c1 - c0 + 63) / 64, (n - c0 + 63) / 64);
        syrk_dmma_kernel<64><<<grid, 256, kSyrkSmem / 2, s>>>(A, ld, n, c0, c1, k0, k1);
    }
    if(nlaunch) (*nlaunch)++;
    return true;
}

static bool chol_factor_enqueue(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch, int kinds = 7);
static bool chol_solve_enqueue(const double* L, int npad, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s, int* nlaunch, int parts = 3);

// The factorization is ~3 short kernels per 64-column block, all with launch-time-constant
// arguments: replaying a captured CUDA graph takes the host out of the loop (the host would
// otherwise bound the rate at which the chain of tiny kernels is issued).
struct GraphKey { const void* a; const void* b; int npad, nreal, kind; };
struct GraphEntry { GraphKey key; cudaGraphExec_t exec; int launches; unsigned long stamp; };
static std::vector<GraphEntry> g_graphs;
static unsigned long g_stamp = 0;

template <typename F>
static bool run_graphed(const GraphKey& key, cudaStream_t s, int* nlaunch, F enqueue)
{
    for(auto& e : g_graphs)
        if(e.key.a == key.a && e.key.b == key.b && e.key.npad == key.npad && e.key.nreal == key.nreal && e.key.kind == key.kind)
        {
            e.stamp = ++g_stamp;
            MB200_CUDA_CHECK(cudaGraphLaunch(e.exec, s));
            if(nlaunch) *nlaunch += e.launches;
            return true;
        }
    int n = 0;
    cudaGraph_t graph = nullptr;
    MB200_CUDA_CHECK(cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal));
    const bool ok = enqueue(&n);
    cudaError_t e1 = cudaStreamEndCapture(s, &graph);
    if(!ok || e1 != cudaSuccess || graph == nullptr)
    {
        if(graph) cudaGraphDestroy(graph);
        set_error("CUDA graph capture of the factorization failed: %s", cudaGetErrorString(e1));
        return false;
    }
    GraphEntry ent{key, nullptr, n, ++g_stamp};
    MB200_CUDA_CHECK(cudaGraphInstantiate(&ent.exec, graph, 0));
    cudaGraphDestroy(graph);
    if(g_graphs.size() >= 16)
    {
        size_t old = 0;
        for(size_t i = 1; i < g_graphs.size(); i++) if(g_graphs[i].stamp < g_graphs[old].stamp) old = i;
        cudaGraphExecDestroy(g_graphs[old].exec);
        g_graphs.erase(g_graphs.begin() + old);
    }
    g_graphs.push_back(ent);
    MB200_CUDA_CHECK(cudaGraphLaunch(ent.exec, s));
    if(nlaunch) *nlaunch += n;
    return true;
}

void chol_forget_graphs(const void* A)
{
    for(size_t i = 0; i < g_graphs.size();)
        if(g_graphs[i].key.a == A || g_graphs[i].key.b == A) { cudaGraphExecDestroy(g_graphs[i].exec); g_graphs.erase(g_graphs.begin() + i); }
        else i++;
}

bool chol_factor(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch,
                 CholScratch* scratch, const int* d_run_if)
{
    if(!configure_kernels()) return false;
    if(chol_dataflow_usable(npad)) return chol_factor_dataflow(A, npad, nreal, invL, d_info, s, nlaunch, scratch, d_run_if);
    // (the multi-kernel fallback always runs: a factorization nobody asked for costs time, not correctness)
    return run_graphed(GraphKey{A, d_info, npad, nreal, 0}, s, nlaunch,
                       [&](int* n) { return chol_factor_enqueue(A, npad, nreal, invL, d_info, s, n); });
}

bool chol_solve(const double* L, int npad, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s, int* nlaunch, int parts)
{
    if(nrhs != 1) return chol_solve_enqueue(L, npad, invL, B, ldb, nrhs, s, nlaunch, parts);
    return run_graphed(GraphKey{L, B, npad, ldb, 1 + 16 * parts}, s, nlaunch,
                       [&](int* n) { return chol_solve_enqueue(L, npad, invL, B, ldb, 1, s, n, parts); });
}

static bool chol_solve_bwd_enqueue(const double* L, int npad, const double* invL, double* B, int ldb, cudaStream_t s, int* nlaunch);

// L' z = y only (the forward half came out of the factorization itself: see normal_assemble's augmented row)
bool chol_solve_backward(const double* L, int npad, const double* invL, double* B, int ldb, int* d_info, cudaStream_t s, int* nlaunch,
                         CholScratch* scratch, const int* d_run_if)
{
    if(chol_dataflow_usable(npad)) return chol_solve_backward_dataflow(L, npad, invL, B, d_info, s, nlaunch, scratch, d_run_if);
    return run_graphed(GraphKey{L, B, npad, ldb, 2}, s, nlaunch,
                       [&](int* n) { return chol_solve_bwd_enqueue(L, npad, invL, B, ldb, s, n); });
}

static bool chol_factor_enqueue(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch, int kinds)
{
    if(!configure_kernels()) return false;
    MB200_CUDA_CHECK(cudaMemsetAsync(d_info, 0, sizeof(int), s));
    for(int K0 = 0; K0 < npad; K0 += NBO)
    {
        const int K1 = K0 + NBO < npad ? K0 + NBO : npad;
        for(int k0 = K0; k0 < K1; k0 += NB)
        {
            if(kinds & 1)
            {
                potrf_diag_kernel<false><<<1, 256, kPotrfSmem, s>>>(A, npad, k0, invL + (size_t)(k0 / NB) * NB * NB, d_info, nreal, nullptr);
                if(nlaunch) (*nlaunch)++;
            }
            const int nrows_below = npad - (k0 + NB);
            if(nrows_below > 0)
            {
                if(kinds & 2)
                {
                    trsm_kernel<<<nrows_below / NB, 256, kBlockSmem, s>>>(A, npad, k0, invL + (size_t)(k0 / NB) * NB * NB, npad);
                    if(nlaunch) (*nlaunch)++;
                }
                // rest of this outer panel only
                if((kinds & 4) && !syrk_update(A, npad, npad, k0 + NB, K1, k0, k0 + NB, s, nlaunch)) return false;
            }
        }
        // the whole trailing matrix, K = width of the panel
        if((kinds & 8 || kinds == 7) && !syrk_update(A, npad, npad, K1, npad, K0, K1, s, nlaunch)) return false;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

////////////////////////////////////////////////////////////////////////////////
// triangular solves, Nrhs right-hand sides stored as rows: B[rhs][n]
////////////////////////////////////////////////////////////////////////////////
// y_k = invL_kk b_k  (transpose=false)  or  invL_kk' b_k (transpose=true); one CTA per rhs
__global__ void __launch_bounds__(64)
solve_diag_kernel(const double* __restrict__ invL, double* __restrict__ B, int ldb, int k0, bool transpose)
{
    __shared__ double b[NB];
    double* v = B + (size_t)blockIdx.x * ldb + k0;
    const int i = threadIdx.x;
    b[i] = v[i];
    __syncthreads();
    double acc = 0.;
    if(!transpose) { for(int m = 0; m <= i; m++) acc += invL[i * NB + m] * b[m]; }
    else           { for(int m = i; m < NB; m++) acc += invL[m * NB + i] * b[m]; }
    v[i] = acc;
}

// forward:  b_i -= L(i, k0:k0+64) y_k for rows i >= k0+64. One warp per row, all rhs
__global__ void __launch_bounds__(256)
solve_update_fwd_kernel(const double* __restrict__ L, int ld, int n, double* __restrict__ B, int ldb, int nrhs, int k0)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int i = k0 + NB + warp;
    if(i >= n) return;
    const double l0 = L[(size_t)i * ld + k0 + lane], l1 = L[(size_t)i * ld + k0 + 32 + lane];
    for(int r = 0; r < nrhs; r++)
    {
        const double* y = B + (size_t)r * ldb + k0;
        double acc = l0 * y[lane] + l1 * y[32 + lane];
#pragma unroll
        for(int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if(lane == 0) B[(size_t)r * ldb + i] -= acc;
    }
}

// backward: b_j -= sum_r L(k0+r, j) z_k[r] for columns j < k0. One thread per column, all rhs
__global__ void __launch_bounds__(256)
solve_update_bwd_kernel(const double* __restrict__ L, int ld, double* __restrict__ B, int ldb, int nrhs, int k0)
{
    __shared__ double z[NB];
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    for(int r = 0; r < nrhs; r++)
    {
        __syncthreads();
        if(threadIdx.x < NB) z[threadIdx.x] = B[(size_t)r * ldb + k0 + threadIdx.x];
        __syncthreads();
        if(j < k0)
        {
            double acc = 0.;
#pragma unroll 8
            for(int m = 0; m < NB; m++) acc += L[(size_t)(k0 + m) * ld + j] * z[m];
            B[(size_t)r * ldb + j] -= acc;
        }
    }
}

static bool chol_solve_enqueue(const double* L, int npad, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s, int* nlaunch, int parts)
{
    const int nblk = npad / NB;
    for(int k = 0; k < nblk && (parts & 1); k++)
    {
        const int k0 = k * NB;
        solve_diag_kernel<<<nrhs, NB, 0, s>>>(invL + (size_t)k * NB * NB, B, ldb, k0, false);
        if(nlaunch) (*nlaunch)++;
        const int below = npad - k0 - NB;
        if(below > 0)
        {
            solve_update_fwd_kernel<<<(below * 32 + 255) / 256, 256, 0, s>>>(L, npad, npad, B, ldb, nrhs, k0);
            if(nlaunch) (*nlaunch)++;
        }
    }
    for(int k = nblk - 1; k >= 0 && (parts & 2); k--)
    {
        const int k0 = k * NB;
        solve_diag_kernel<<<nrhs, NB, 0, s>>>(invL + (size_t)k * NB * NB, B, ldb, k0, true);
        if(nlaunch) (*nlaunch)++;
        if(k0 > 0)
        {
            solve_update_bwd_kernel<<<(k0 + 255) / 256, 256, 0, s>>>(L, npad, B, ldb, nrhs, k0);
            if(nlaunch) (*nlaunch)++;
        }
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

__global__ void debug_fill_spd_kernel(double* A, int n)
{
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(e >= (size_t)n * n) return;
    const int i = (int)(e / n), j = (int)(e % n);
    A[e] = i == j ? (double)n : 1. / (1. + (double)((i * 31 + j * 17) % 97));
}

void chol_debug_fill_spd(double* A, int npad, cudaStream_t s)
{
    debug_fill_spd_kernel<<<(unsigned)(((size_t)npad * npad + 255) / 256), 256, 0, s>>>(A, npad);
}

// Timing aid (not on any product path): device time of `reps` factorizations of an n x n matrix,
// restricted to the kernel kinds in the mask (1 potrf_diag, 2 trsm, 4 panel syrk, 8 trailing syrk;
// 15 = everything), launched directly (graph=0) or as a captured graph (graph=1)
double chol_debug_time(int n, int reps, int kinds, int graph)
{
    const int npad = chol_padded(n);
    double *A, *invL; int* info;
    if(cudaMalloc(&A, (size_t)npad * npad * sizeof(double)) != cudaSuccess) return -1.;
    cudaMalloc(&invL, (size_t)npad * NB * sizeof(double));
    cudaMalloc(&info, sizeof(int));
    cudaStream_t s; cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    configure_kernels();
    debug_fill_spd_kernel<<<(unsigned)(((size_t)npad * npad + 255) / 256), 256, 0, s>>>(A, npad);
    cudaGraphExec_t exec = nullptr;
    if(graph)
    {
        cudaGraph_t g;
        cudaStreamBeginCapture(s, cudaStreamCaptureModeThreadLocal);
        chol_factor_enqueue(A, npad, n, invL, info, s, nullptr, kinds == 15 ? 7 : kinds);
        cudaStreamEndCapture(s, &g);
        cudaGraphInstantiate(&exec, g, 0);
        cudaGraphDestroy(g);
    }
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    double* rhs = nullptr;
    if(kinds >= 32)
    {
        // 32: persistent factorization; 64: persistent backward substitution; 128: multi-kernel backward substitution
        cudaMalloc(&rhs, (size_t)npad * sizeof(double));
        cudaMemsetAsync(rhs, 0, (size_t)npad * sizeof(double), s);
        chol_factor_dataflow(A, npad, n, invL, info, s, nullptr);
    }
    for(int r = -1; r < reps; r++)
    {
        if(r == 0) cudaEventRecord(e0, s);
        if(kinds == 32)
        {
            if(r >= 0) debug_fill_spd_kernel<<<(unsigned)(((size_t)npad * npad + 255) / 256), 256, 0, s>>>(A, npad);
            chol_factor_dataflow(A, npad, n, invL, info, s, nullptr);
        }
        else if(kinds == 33) debug_fill_spd_kernel<<<(unsigned)(((size_t)npad * npad + 255) / 256), 256, 0, s>>>(A, npad);
        else if(kinds == 64) chol_solve_backward_dataflow(A, npad, invL, rhs, info, s, nullptr);
        else if(kinds == 128) run_graphed(GraphKey{A, rhs, npad, npad, 2}, s, nullptr, [&](int* nn) { return chol_solve_bwd_enqueue(A, npad, invL, rhs, npad, s, nn); });
        else if(graph) cudaGraphLaunch(exec, s);
        else      chol_factor_enqueue(A, npad, n, invL, info, s, nullptr, kinds == 15 ? 7 : kinds);
    }
    cudaEventRecord(e1, s);
    cudaEventSynchronize(e1);
    float ms = 0.f; cudaEventElapsedTime(&ms, e0, e1);
    if(exec) cudaGraphExecDestroy(exec);
    cudaEventDestroy(e0); cudaEventDestroy(e1);
    chol_forget_graphs(A);
    cudaStreamDestroy(s);
    cudaFree(A); cudaFree(invL); cudaFree(info); cudaFree(rhs);
    return ms / reps;
}

// Debugging aid: clock64() stamps of the phases of one diagonal-block factorization (64 values)
bool chol_debug_potrf_stamps(long long* out64)
{
    const int npad = 128;
    double *A, *invL; int* info; long long* st;
    if(!configure_kernels()) return false;
    MB200_CUDA_CHECK(cudaMalloc(&A, (size_t)npad * npad * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&invL, (size_t)npad * NB * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&info, sizeof(int)));
    MB200_CUDA_CHECK(cudaMalloc(&st, 64 * sizeof(long long)));
    debug_fill_spd_kernel<<<(npad * npad + 255) / 256, 256>>>(A, npad);
    for(int r = 0; r < 3; r++)
    {
        cudaMemset(st, 0, 64 * sizeof(long long));
        potrf_diag_kernel<true><<<1, 256, kPotrfSmem>>>(A, npad, 0, invL, info, npad, st);
    }
    MB200_CUDA_CHECK(cudaDeviceSynchronize());
    MB200_CUDA_CHECK(cudaMemcpy(out64, st, 64 * sizeof(long long), cudaMemcpyDeviceToHost));
    cudaFree(A); cudaFree(invL); cudaFree(info); cudaFree(st);
    return true;
}

static bool chol_solve_bwd_enqueue(const double* L, int npad, const double* invL, double* B, int ldb, cudaStream_t s, int* nlaunch)
{
    const int nblk = npad / NB;
    for(int k = nblk - 1; k >= 0; k--)
    {
        const int k0 = k * NB;
        solve_diag_kernel<<<1, NB, 0, s>>>(invL + (size_t)k * NB * NB, B, ldb, k0, true);
        if(nlaunch) (*nlaunch)++;
        if(k0 > 0)
        {
            solve_update_bwd_kernel<<<(k0 + 255) / 256, 256, 0, s>>>(L, npad, B, ldb, 1, k0);
            if(nlaunch) (*nlaunch)++;
        }
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// min/max of the diagonal of L (for rcond)
__global__ void diag_minmax_kernel(const double* __restrict__ L, int ld, int n, double* out)
{
    __shared__ double smin[256], smax[256];
    double mn = 1e300, mx = 0.;
    for(int i = threadIdx.x; i < n; i += blockDim.x)
    {
        const double d = L[(size_t)i * ld + i];
        mn = d < mn ? d : mn;
        mx = d > mx ? d : mx;
    }
    smin[threadIdx.x] = mn; smax[threadIdx.x] = mx;
    __syncthreads();
    for(int o = 128; o > 0; o >>= 1)
    {
        if(threadIdx.x < o)
        {
            smin[threadIdx.x] = fmin(smin[threadIdx.x], smin[threadIdx.x + o]);
            smax[threadIdx.x] = fmax(smax[threadIdx.x], smax[threadIdx.x + o]);
        }
        __syncthreads();
    }
    if(threadIdx.x == 0) { out[0] = smin[0]; out[1] = smax[0]; }
}

bool chol_diag_minmax(const double* L, int npad, int nreal, double* d_out2, cudaStream_t s)
{
    diag_minmax_kernel<<<1, 256, 0, s>>>(L, npad, nreal, d_out2);
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace mb200
