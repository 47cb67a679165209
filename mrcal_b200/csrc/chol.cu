// Kernel family 2b: what the dense Cholesky needs besides its two persistent kernels (chol_dataflow.cu: the
// factorization up to n = 8192, and the backward substitution of one right-hand side):
//   - the factorization above n = 8192, where a chain of short kernels per 64 columns is faster than the persistent
//     kernel (DESIGN section 9). A two-level blocked right-looking algorithm:
//
//       for each 256-column outer panel:
//           for each 64-column inner block of it:
//               potrf_diag   one CTA: factor the 64x64 diagonal block in shared
//                            memory, and invert the factor (potrf_block.cuh)
//               trsm         rows below: X <- A inv(L_kk)'   (small GEMM)
//               syrk (K=64)  update of the REST OF THE PANEL only
//           syrk (K=256)     one DMMA update of the whole trailing matrix
//
//   - triangular solves with the factor for nrhs right-hand sides (the factorization objects' solves, and through the
//     structured factor projection_uncertainty()'s), chosen by nrhs and the number of 64-column blocks: two short
//     kernels per block and direction, or a DMMA kernel that takes a tile of kSolveTile right-hand sides per CTA
//   - min/max of diag(L), for rcond
//   - fill_words: a few ranges of flags and counters cleared in one launch
//   - timing and debugging aids
//
// Stands in for cholmod_factorize / cholmod_solve as the reference calls them (mrcal.c:6435, mrcal-pywrap.c:196-212,
// 557). Storage: row-major npad x npad, lower triangle, npad a multiple of 64 (the caller puts 1 on the padding
// diagonal). Rows are K-contiguous, which is what dmma() (ptx.cuh, row x col) wants for both operands of  C -= P P'.
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

#include "chol.h"
#include "potrf_block.cuh"
#include "problem.h"
#include "ptx.cuh"
#include "reduce.cuh"

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

////////////////////////////////////////////////////////////////////////////////
// triangular solves, Nrhs right-hand sides stored as rows: B[rhs][n]
////////////////////////////////////////////////////////////////////////////////
// y_k = invL_kk b_k  (transpose=false)  or  invL_kk' b_k (transpose=true); one CTA per rhs. Unknowns >= nreal are
// read as zero: whatever the padding holds (NaN included) never reaches a real unknown, and the padding unknowns of
// the solution come out zero in the backward direction
__global__ void __launch_bounds__(64)
solve_diag_kernel(const double* __restrict__ invL, double* __restrict__ B, int ldb, int k0, int nreal, bool transpose)
{
    __shared__ double b[NB];
    double* v = B + (size_t)blockIdx.x * ldb + k0;
    const int i = threadIdx.x;
    b[i] = k0 + i < nreal ? v[i] : 0.;
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
        const double acc = warp_sum(l0 * y[lane] + l1 * y[32 + lane]);
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

// L y = b (BWD = false) or L' x = b (BWD = true) for a tile of kSolveTile right-hand sides B[r][0..ldb), in place,
// left-looking over 64-blocks: block i takes the GEMM of every already-solved block k with L's block (i,k) (or (k,i)'),
// then the GEMM with the stored inverse of its diagonal block. Unknowns >= nreal are treated as zero
template <bool BWD>
__global__ void __launch_bounds__(256)
ls_solve_tiled_kernel(const double* __restrict__ L, int ld, const double* __restrict__ invL, double* __restrict__ B, int ldb,
                      int Nrhs, int nblk, int nreal)
{
    extern __shared__ __align__(16) double dsm[];
    double (*sA)[kSolveTileLd] = reinterpret_cast<double (*)[kSolveTileLd]>(dsm);
    double (*sM)[kSolveTileLd] = reinterpret_cast<double (*)[kSolveTileLd]>(dsm + kSolveTile * kSolveTileLd);
    const int r0 = blockIdx.x * kSolveTile;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g8 = lane >> 2, t4 = lane & 3;
    const int mt = warp >> 1, nt0 = (warp & 1) * 4;
    auto gemm = [&](double (&acc)[4][2], bool trans)
    {
#pragma unroll 4
        for(int ks = 0; ks < NB / 4; ks++)
        {
            const double a = sA[mt * 8 + g8][ks * 4 + t4];
#pragma unroll
            for(int j = 0; j < 4; j++)
            {
                const int n = (nt0 + j) * 8 + g8, k = ks * 4 + t4;
                dmma(acc[j][0], acc[j][1], a, trans ? sM[k][n] : sM[n][k]);
            }
        }
    };
    auto load_rhs = [&](int kb)
    {
        for(int e = tid; e < kSolveTile * NB; e += 256)
        {
            const int r = e >> 6, m = e & 63, c = kb * NB + m;
            sA[r][m] = (r0 + r < Nrhs && c < nreal) ? B[(size_t)(r0 + r) * ldb + c] : 0.;
        }
    };
    for(int step = 0; step < nblk; step++)
    {
        const int i = BWD ? nblk - 1 - step : step;
        double acc[4][2] = {};
        for(int s = 0; s < step; s++)
        {
            const int k = BWD ? nblk - 1 - s : s;
            load_rhs(k);
            // forward: sM[n][m] = L(i*64+n, k*64+m);  backward: sM[m][n] = L(k*64+m, i*64+n)
            for(int e = tid; e < NB * NB; e += 256)
            {
                const int a = e >> 6, b = e & 63;
                const int row = BWD ? k * NB + a : i * NB + a, col = BWD ? i * NB + b : k * NB + b;
                sM[a][b] = (row < nreal && col < nreal) ? L[(size_t)row * ld + col] : 0.;
            }
            __syncthreads();
            gemm(acc, BWD);
            __syncthreads();
        }
        load_rhs(i);
        for(int e = tid; e < NB * NB; e += 256) sM[e >> 6][e & 63] = invL[(size_t)i * NB * NB + e];
        __syncthreads();
#pragma unroll
        for(int j = 0; j < 4; j++)
        {
            sA[mt * 8 + g8][(nt0 + j) * 8 + 2 * t4] -= acc[j][0];
            sA[mt * 8 + g8][(nt0 + j) * 8 + 2 * t4 + 1] -= acc[j][1];
            acc[j][0] = acc[j][1] = 0.;
        }
        __syncthreads();
        // forward: y[n] = sum_m invL[n][m] b[m];  backward: x[n] = sum_m invL[m][n] b[m]
        gemm(acc, BWD);
        const int r = r0 + mt * 8 + g8;
        if(r < Nrhs)
#pragma unroll
            for(int j = 0; j < 4; j++)
                for(int h = 0; h < 2; h++)
                {
                    const int c = i * NB + (nt0 + j) * 8 + 2 * t4 + h;
                    if(c < nreal) B[(size_t)r * ldb + c] = acc[j][h];
                }
        __syncthreads();
    }
}

__global__ void fill_words_kernel(WordFill f)
{
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
    for(int k = 0; k < f.count; k++)
    {
        unsigned* p = f.p[k];
        const unsigned v = f.v[k];
        for(long long i = t; i < f.n[k]; i += stride) p[i] = v;
    }
}

bool fill_words(const WordFill& f, cudaStream_t s)
{
    if(f.count == 0) return true;
    long long widest = 0;
    for(int k = 0; k < f.count; k++) widest = f.n[k] > widest ? f.n[k] : widest;
    const long long blocks = (widest + 255) / 256;
    fill_words_kernel<<<(unsigned)(blocks < 1 ? 1 : (blocks > 512 ? 512 : blocks)), 256, 0, s>>>(f);
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

static const size_t kSyrkSmem = (size_t)2 * STAGES * BM * LDS * sizeof(double);   // TILE = 128; half of it for TILE = 64
static const size_t kBlockSmem = (size_t)2 * NB * (NB + 1) * sizeof(double);   // trsm
static const size_t kPotrfSmem = sizeof(PotrfSmem);

static bool configure_kernels()
{
    return set_max_dynamic_smem<syrk_dmma_kernel<128>>((int)kSyrkSmem) && set_max_dynamic_smem<syrk_dmma_kernel<64>>((int)kSyrkSmem) &&
           set_max_dynamic_smem<trsm_kernel>((int)kBlockSmem) &&
           set_max_dynamic_smem<potrf_diag_kernel<false>>((int)kPotrfSmem) && set_max_dynamic_smem<potrf_diag_kernel<true>>((int)kPotrfSmem) &&
           set_max_dynamic_smem<ls_solve_tiled_kernel<false>>((int)kSolveTileSmem) &&
           set_max_dynamic_smem<ls_solve_tiled_kernel<true>>((int)kSolveTileSmem);
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

// The multi-kernel factorization is ~3 short kernels per 64-column block, a solve 2 per block and direction, all with
// launch-time-constant arguments: replaying a captured CUDA graph takes the host out of the loop (the host would
// otherwise bound the rate at which the chain of tiny kernels is issued).
// m: ldb (solve; unused by the factorization); kind: 0 the factorization, else the solve's parts
struct GraphKey { const void* a; const void* b; int npad, nreal, m, kind; };
struct GraphEntry { GraphKey key; cudaGraphExec_t exec; int launches; unsigned long stamp; };
static std::vector<GraphEntry> g_graphs;
static unsigned long g_stamp = 0;

template <typename F>
static bool run_graphed(const GraphKey& key, cudaStream_t s, int* nlaunch, F enqueue)
{
    for(auto& e : g_graphs)
        if(e.key.a == key.a && e.key.b == key.b && e.key.npad == key.npad && e.key.nreal == key.nreal && e.key.m == key.m &&
           e.key.kind == key.kind)
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

bool chol_factor_blocked(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch)
{
    if(!configure_kernels()) return false;
    return run_graphed(GraphKey{A, d_info, npad, nreal, 0, 0}, s, nlaunch, [&](int* n)
    {
        MB200_CUDA_CHECK(cudaMemsetAsync(d_info, 0, sizeof(int), s));
        for(int K0 = 0; K0 < npad; K0 += NBO)
        {
            const int K1 = K0 + NBO < npad ? K0 + NBO : npad;
            for(int k0 = K0; k0 < K1; k0 += NB)
            {
                potrf_diag_kernel<false><<<1, 256, kPotrfSmem, s>>>(A, npad, k0, invL + (size_t)(k0 / NB) * NB * NB, d_info, nreal, nullptr);
                (*n)++;
                const int nrows_below = npad - (k0 + NB);
                if(nrows_below > 0)
                {
                    trsm_kernel<<<nrows_below / NB, 256, kBlockSmem, s>>>(A, npad, k0, invL + (size_t)(k0 / NB) * NB * NB, npad);
                    (*n)++;
                    // rest of this outer panel only
                    if(!syrk_update(A, npad, npad, k0 + NB, K1, k0, k0 + NB, s, n)) return false;
                }
            }
            // the whole trailing matrix, K = width of the panel
            if(!syrk_update(A, npad, npad, K1, npad, K0, K1, s, n)) return false;
        }
        MB200_CUDA_CHECK(cudaGetLastError());
        return true;
    });
}

static bool chol_solve_enqueue(const double* L, int npad, int nreal, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s,
                               int* nlaunch, int parts)
{
    const int nblk = npad / NB;
    for(int k = 0; k < nblk && (parts & 1); k++)
    {
        const int k0 = k * NB;
        solve_diag_kernel<<<nrhs, NB, 0, s>>>(invL + (size_t)k * NB * NB, B, ldb, k0, nreal, false);
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
        solve_diag_kernel<<<nrhs, NB, 0, s>>>(invL + (size_t)k * NB * NB, B, ldb, k0, nreal, true);
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

// The per-block kernels parallelise over the rows under each 64-block and loop over the right-hand sides: their time
// grows as nblk x nrhs. The tiled kernel runs one CTA per kSolveTile right-hand sides through all nblk^2/2 block pairs:
// its time grows as nblk^2 and hardly with nrhs. So the crossover moves with nblk. Measured on H100 (DESIGN section
// 9), the tiled kernel wins from 2 to 3 nblk right-hand sides on for L' and 4 to 7 nblk for L; it takes over at 8 nblk
constexpr int kTiledSolveRhsPerBlock = 8;

bool chol_solve(const double* L, int npad, int nreal, const double* invL, double* B, int ldb, int nrhs, cudaStream_t s,
                int* nlaunch, int parts, int kernels)
{
    if(kernels == 2 || (kernels == 0 && nrhs >= kTiledSolveRhsPerBlock * (npad / NB)))
    {
        if(!configure_kernels()) return false;
        const unsigned tiles = (unsigned)((nrhs + kSolveTile - 1) / kSolveTile);
        if(parts & 1) ls_solve_tiled_kernel<false><<<tiles, 256, kSolveTileSmem, s>>>(L, npad, invL, B, ldb, nrhs, npad / NB, nreal);
        if(parts & 2) ls_solve_tiled_kernel<true><<<tiles, 256, kSolveTileSmem, s>>>(L, npad, invL, B, ldb, nrhs, npad / NB, nreal);
        if(nlaunch) *nlaunch += (parts & 1) + (parts >> 1);
        MB200_CUDA_CHECK(cudaGetLastError());
        return true;
    }
    if(nrhs != 1) return chol_solve_enqueue(L, npad, nreal, invL, B, ldb, nrhs, s, nlaunch, parts);
    return run_graphed(GraphKey{L, B, npad, nreal, ldb, parts}, s, nlaunch,
                       [&](int* n) { return chol_solve_enqueue(L, npad, nreal, invL, B, ldb, 1, s, n, parts); });
}

// Test aid (not on any product path): solve with a host factor (L: npad x npad, invL: npad/64 blocks of 64 x 64) for
// nrhs host right-hand sides B[r][0..npad), in place. kernel: 0 chol_solve()'s own choice, 1 its per-block kernels,
// 2 its tiled kernel, 3 chol_solve_backward() (nrhs = 1, parts = 2: the whole padded system)
bool chol_debug_solve(const double* L, const double* invL, int npad, int nreal, double* B, int nrhs, int parts, int kernel)
{
    if(npad <= 0 || npad % NB != 0 || nreal < 0 || nreal > npad || nrhs <= 0 || parts < 1 || parts > 3 || kernel < 0 ||
       kernel > 3 || (kernel == 3 && (nrhs != 1 || parts != 2)))
    {
        set_error("chol_debug_solve: bad arguments (npad %d, nreal %d, nrhs %d, parts %d, kernel %d)", npad, nreal, nrhs, parts, kernel);
        return false;
    }
    double *dL = nullptr, *dinv = nullptr, *dB = nullptr; int* info = nullptr;
    cudaStream_t s = nullptr;
    CholScratch sc;
    int h_info = 0;
    bool ok = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&dL, (size_t)npad * npad * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&dinv, (size_t)npad * NB * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&dB, (size_t)nrhs * npad * sizeof(double)) == cudaSuccess && cudaMalloc(&info, sizeof(int)) == cudaSuccess &&
              cudaMemcpyAsync(dL, L, (size_t)npad * npad * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemcpyAsync(dinv, invL, (size_t)npad * NB * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemcpyAsync(dB, B, (size_t)nrhs * npad * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemsetAsync(info, 0, sizeof(int), s) == cudaSuccess;
    if(ok && kernel == 3)
        ok = chol_scratch_create(&sc, npad) && chol_solve_backward(dL, npad, dinv, dB, info, s, nullptr, &sc);
    else if(ok)
        ok = chol_solve(dL, npad, nreal, dinv, dB, npad, nrhs, s, nullptr, parts, kernel);
    ok = ok && cudaMemcpyAsync(B, dB, (size_t)nrhs * npad * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(&h_info, info, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess;
    if(!ok) set_error("chol_debug_solve failed: %s", cudaGetErrorString(cudaGetLastError()));
    else if(h_info != 0) { set_error("chol_debug_solve: the backward substitution reported %d", h_info); ok = false; }
    if(s) cudaStreamSynchronize(s);
    chol_forget_graphs(dL);   // one right-hand side: a graph keyed on dL and dB
    chol_scratch_destroy(&sc);
    cudaFree(dL); cudaFree(dinv); cudaFree(dB); cudaFree(info);
    if(s) cudaStreamDestroy(s);
    return ok;
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

// Timing aid (not on any product path): device time of chol_factor for an n x n matrix (what = 0; net of the refill
// with an SPD matrix that every repetition needs) or of chol_solve_backward (what = 1), per call, averaged over reps
// calls; -1 on failure
double chol_debug_time(int n, int reps, int what)
{
    const int npad = chol_padded(n);
    double *A = nullptr, *invL = nullptr, *rhs = nullptr; int* info = nullptr;
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CholScratch sc;
    bool ok = cudaMalloc(&A, (size_t)npad * npad * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&invL, (size_t)npad * NB * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&rhs, (size_t)npad * sizeof(double)) == cudaSuccess && cudaMalloc(&info, sizeof(int)) == cudaSuccess &&
              cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess &&
              cudaEventCreate(&e0) == cudaSuccess && cudaEventCreate(&e1) == cudaSuccess && chol_scratch_create(&sc, npad);
    // ms per call of: 0 the refill, 1 the refill and the factorization, 2 the backward substitution
    auto timed = [&](int kind) -> double
    {
        for(int r = -1; r < reps && ok; r++)
        {
            if(r == 0) ok = cudaEventRecord(e0, s) == cudaSuccess;
            if(kind <= 1) chol_debug_fill_spd(A, npad, s);
            if(kind == 1) ok = ok && chol_factor(A, npad, n, invL, info, s, nullptr, &sc);
            if(kind == 2) ok = ok && chol_solve_backward(A, npad, invL, rhs, info, s, nullptr, &sc);
        }
        float ms = 0.f;
        ok = ok && cudaEventRecord(e1, s) == cudaSuccess && cudaEventSynchronize(e1) == cudaSuccess &&
             cudaEventElapsedTime(&ms, e0, e1) == cudaSuccess;
        return ms / reps;
    };
    double ms = -1.;
    if(ok && what == 0)
    {
        const double fill = timed(0), both = timed(1);
        if(ok) ms = both - fill;
    }
    else if(ok && what == 1)
    {
        chol_debug_fill_spd(A, npad, s);
        ok = cudaMemsetAsync(rhs, 0, (size_t)npad * sizeof(double), s) == cudaSuccess &&
             chol_factor(A, npad, n, invL, info, s, nullptr, &sc);
        const double bwd = timed(2);
        if(ok) ms = bwd;
    }
    if(s) cudaStreamSynchronize(s);
    chol_scratch_destroy(&sc);
    if(e0) cudaEventDestroy(e0);
    if(e1) cudaEventDestroy(e1);
    if(s) cudaStreamDestroy(s);
    cudaFree(A); cudaFree(invL); cudaFree(rhs); cudaFree(info);
    return ms;
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
