// Kernel family 2c: the dense Cholesky factorization and the backward substitution
// of every dense system, as ONE persistent kernel each.
//
// Left-looking tile algorithm, 64x64 tiles, one CTA per SM. The owner of tile (i,j) computes
//       C = A_ij - sum_{k<j} L_ik L_jk'          (DMMA, operands staged with cp.async)
//       i == j:  L_jj = chol(C), and its inverse (potrf_block.cuh)
//       i >  j:  L_ij = C inv(L_jj)'             (DMMA)
// and then raises a flag in global memory (st.release). Consumers poll the flags of the
// tiles they need (ld.acquire) and pull them from L2. The diagonal tiles and the tiles
// left of them -- the critical path -- belong to one CTA, the spine (chol_spine_kernel).
// All CTAs are co-resident (cooperative launch) and every CTA walks its tasks in an order
// in which each depends only on earlier ones: the scheme cannot deadlock. Waits are
// bounded all the same (a wedged GPU box costs more than a wrong answer that the caller
// can detect): on timeout *info = -9.
//
// Stands in for cholmod_factorize / cholmod_solve as libdogleg calls them (call site
// mrcal.c:6435); the reference has no counterpart of this structure.
#include <cuda_runtime.h>
#include <cstdint>
#include <vector>

#include "chol.h"
#include "potrf_block.cuh"
#include "problem.h"

namespace mb200 {

namespace {

constexpr int T = 64;
constexpr long long kSpinLimit = 4000000000ll;   // ~2 s of SM clocks

struct DfSmem
{
    PotrfSmem pb;          // pb.L doubles as the C tile of a diagonal tile
    double C2[T * PLD];    // the C tile of an off-diagonal tile
    double opA[T * PLD];
    double opB[T * PLD];
    int ok;
};

__device__ __forceinline__ int ld_acquire(const int* p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int* p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// 64x64 tile, row stride ld in global -> [64][PLD] in shared. 2048 16-byte chunks, 8 per thread
__device__ __forceinline__ void tile_to_smem(double* dst, const double* src, size_t ld)
{
#pragma unroll
    for(int q = 0; q < 8; q++)
    {
        const int chunk = threadIdx.x + q * 256, r = chunk >> 5, c = (chunk & 31) * 2;
        cp_async16(&dst[r * PLD + c], &src[(size_t)r * ld + c]);
    }
}

// thread 0 waits for up to two flags; everybody learns whether it worked
__device__ __forceinline__ bool wait_flags(DfSmem& sm, const int* f0, const int* f1, int* abort_flag, int* info)
{
    if(threadIdx.x == 0)
    {
        int ok = 1;
        const long long t0 = clock64();
        while(ld_acquire(f0) == 0 || (f1 && ld_acquire(f1) == 0))
        {
            if(ld_acquire(abort_flag) != 0 || clock64() - t0 > kSpinLimit)
            {
                st_release(abort_flag, 1);
                atomicExch(info, -9);
                ok = 0;
                break;
            }
        }
        sm.ok = ok;
    }
    __syncthreads();
    const bool ok = sm.ok != 0;
    __syncthreads();
    return ok;
}

// acc += A B' for two [64][PLD] operands; 8 warps as 4 x 2, warp tile 16 x 32
__device__ __forceinline__ void tile_mma(double (&acc)[2][4][2], const double* A, const double* B)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
    const double* a_s = A + (wm * 16) * PLD;
    const double* b_s = B + (wn * 32) * PLD;
#pragma unroll 4
    for(int ks = 0; ks < T / 4; ks++)
    {
        double af[2], bf[4];
#pragma unroll
        for(int i = 0; i < 2; i++) af[i] = a_s[(i * 8 + g) * PLD + ks * 4 + t];
#pragma unroll
        for(int j = 0; j < 4; j++) bf[j] = b_s[(j * 8 + g) * PLD + ks * 4 + t];
#pragma unroll
        for(int i = 0; i < 2; i++)
#pragma unroll
            for(int j = 0; j < 4; j++) dmma(acc[i][j][0], acc[i][j][1], af[i], bf[j]);
    }
}
__device__ __forceinline__ void acc_zero(double (&acc)[2][4][2])
{
#pragma unroll
    for(int a = 0; a < 2; a++)
#pragma unroll
        for(int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.;
}
// C -= acc for a [64][PLD] tile in shared memory (each thread its own fragment elements)
__device__ __forceinline__ void tile_sub(double* C, const double (&acc)[2][4][2])
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
#pragma unroll
    for(int a = 0; a < 2; a++)
#pragma unroll
        for(int b = 0; b < 4; b++)
        {
            double2* c = reinterpret_cast<double2*>(&C[(wm * 16 + a * 8 + g) * PLD + wn * 32 + b * 8 + 2 * t]);
            double2 v = *c;
            v.x -= acc[a][b][0];
            v.y -= acc[a][b][1];
            *c = v;
        }
}

// X = C W' for a LOWER TRIANGULAR W (the inverse of a diagonal block): 8 warps as 8 x 1, warp tile 8 x 64, and
// column tile j only needs k < 8 (j+1): 72 instead of 128 DMMAs per warp. X goes to global memory (row stride
// ld) and, if Xs is given, to a [64][PLD] tile in shared memory too
__device__ __forceinline__ void tile_trsm(const double* C, const double* W, double* __restrict__ Xg, size_t ld, double* Xs)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    double acc[8][2];
#pragma unroll
    for(int j = 0; j < 8; j++) acc[j][0] = acc[j][1] = 0.;
    const double* a_s = C + (warp * 8) * PLD;
#pragma unroll
    for(int ks = 0; ks < T / 4; ks++)
    {
        const double af = a_s[g * PLD + ks * 4 + t];
#pragma unroll
        for(int j = 0; j < 8; j++)
            if(ks * 4 < 8 * (j + 1))
                dmma(acc[j][0], acc[j][1], af, W[(j * 8 + g) * PLD + ks * 4 + t]);
    }
#pragma unroll
    for(int j = 0; j < 8; j++)
    {
        const int r = warp * 8 + g, c = j * 8 + 2 * t;
        const double2 v = make_double2(acc[j][0], acc[j][1]);
        *reinterpret_cast<double2*>(&Xg[(size_t)r * ld + c]) = v;
        if(Xs) *reinterpret_cast<double2*>(&Xs[r * PLD + c]) = v;
    }
}

__device__ __forceinline__ int tile_flag(int i, int j, int nb) { return j * nb - (j * (j - 1)) / 2 + (i - j); }

// C = D - A A' on the 8x8 granules of the LOWER triangle only (36 of 64: what potrf_block reads), dealt to the 8 warps
// in row-major order: 5 or 4 granules per warp instead of 8
__device__ __forceinline__ void tile_syrk_lower_sub(double* C, const double* D, const double* A)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    int gr[5], gc[5];
    double acc[5][2][2];   // two chains per granule (K halves): the DMMA latency, not its rate, is what a chain of 16 costs
#pragma unroll
    for(int m = 0; m < 5; m++)
    {
        const int idx = warp + 8 * m;
        int r = 0;
        while((r + 1) * (r + 2) / 2 <= idx) r++;
        gr[m] = idx < 36 ? r : 0;
        gc[m] = idx < 36 ? idx - r * (r + 1) / 2 : 0;
        acc[m][0][0] = acc[m][0][1] = acc[m][1][0] = acc[m][1][1] = 0.;
    }
    const bool five = warp + 32 < 36;
#pragma unroll 4
    for(int ks = 0; ks < T / 8; ks++)
    {
#pragma unroll
        for(int h = 0; h < 2; h++)
#pragma unroll
            for(int m = 0; m < 5; m++)
                if(m < 4 || five)
                    dmma(acc[m][h][0], acc[m][h][1], A[(gr[m] * 8 + g) * PLD + (ks + h * (T / 8)) * 4 + t],
                         A[(gc[m] * 8 + g) * PLD + (ks + h * (T / 8)) * 4 + t]);
    }
#pragma unroll
    for(int m = 0; m < 5; m++)
        if(m < 4 || five)
        {
            const int e = (gr[m] * 8 + g) * PLD + gc[m] * 8 + 2 * t;
            const double2 v = *reinterpret_cast<const double2*>(&D[e]);
            *reinterpret_cast<double2*>(&C[e]) = make_double2(v.x - (acc[m][0][0] + acc[m][1][0]), v.y - (acc[m][0][1] + acc[m][1][1]));
        }
}
// [64][PLD] tile in shared memory -> global (row stride ld); lower_only: the entries c <= r
__device__ __forceinline__ void tile_to_global(double* __restrict__ dst, size_t ld, const double* src, bool lower_only)
{
    for(int e = threadIdx.x; e < T * T / 2; e += 256)
    {
        const int r = e >> 5, c = (e & 31) * 2;
        const double2 v = *reinterpret_cast<const double2*>(&src[r * PLD + c]);
        if(!lower_only || c + 1 <= r) *reinterpret_cast<double2*>(&dst[(size_t)r * ld + c]) = v;
        else if(c <= r) dst[(size_t)r * ld + c] = v.x;
    }
}

// The factorization, with the SPINE -- the diagonal tiles and the tiles left of them, whose chain of
// potrf_block -> triangular product -> last rank-64 update IS the critical path -- on one CTA that does nothing else:
// the inverse of a diagonal block goes from potrf_block to the next triangular product through shared memory, and the
// spine CTA never spends time on the earlier updates of its tiles. Those are "pre" tasks of the other CTAs:
//   pre(d):  A_{d,d-1} -= sum_{k<=d-2} L_dk L_{d-1,k}',   A_dd -= sum_{k<=d-2} L_dk L_dk'      in place, then flag pre[d]
// which the spine picks up when potrf_block of step d-1 is done (they have had that long to finish).
// Helper tasks in the order every helper CTA walks them, column by column j = 0 .. nb-3:
//   tile (j+2, j);  pre(j+2);  tiles (i, j), i = j+3 .. nb-1
// (none for nb <= 2: steps 0 and 1 have no pre task, and the spine CTA runs alone).
// Every task depends on spine steps and on EARLIER helper tasks only; the spine depends on its own past and on pre
// tasks: no cycles, all CTAs co-resident, every CTA walks its list in order: no deadlock. Waits are bounded as above.
// (registers capped -- no spills at 160 -- so that the small kernels of the Cauchy side fit next to a CTA of this one)
__global__ void __maxnreg__(160)
chol_spine_kernel(double* __restrict__ A, int ld, int nb, int nreal, double* __restrict__ invL, int* __restrict__ info,
                  int* __restrict__ flags, int* __restrict__ pre, int* __restrict__ abort_flag,
                  long long* __restrict__ stamps /* debugging aid: 8 clock64() values per spine step, or NULL */)
{
#define SPINE_STAMP(k) do { if(stamps != nullptr && tid == 0) stamps[8 * d + (k)] = clock64(); } while(0)
    extern __shared__ __align__(16) unsigned char dsm_raw[];
    DfSmem& sm = *reinterpret_cast<DfSmem*>(dsm_raw);
    const int tid = threadIdx.x;
    double acc[2][4][2];

    if(blockIdx.x == 0)
    {
        ////////////////////////////// the spine
        tile_to_smem(sm.pb.L, A, ld);
        cp_async_commit();
        cp_async_wait<0>();
        for(int d = 0; d < nb; d++)
        {
            double* Add = A + (size_t)d * T * ld + (size_t)d * T;
            SPINE_STAMP(0);
            if(d > 0)
            {
                // C2 = the pre-updated A_{d,d-1}, opB = the pre-updated A_dd: loaded at the end of the last step
                double* Aij = A + (size_t)d * T * ld + (size_t)(d - 1) * T;
                tile_trsm(sm.C2, sm.pb.X, Aij, ld, sm.opA);     // L_{d,d-1} = C2 inv(L_{d-1,d-1})': to global and to opA
                __syncthreads();
                // (the barrier orders everybody's stores before the release store of the one thread that raises the
                // flag -- a thread of the last warp, the chain warp of potrf_block has better things to do)
                if(tid == 255) st_release(flags + tile_flag(d, d - 1, nb), 1);
                SPINE_STAMP(1);
                tile_syrk_lower_sub(sm.pb.L, sm.opB, sm.opA);
            }
            SPINE_STAMP(2);
            potrf_block(sm.pb, info, d * T, nreal);
            SPINE_STAMP(3);
            // the next step's tiles, if they are ready: their loads run under the write-out below. (Fetching them under the
            // last panel of potrf_block by its idle warps was tried: the loads finish no earlier, and the barriers of the
            // panel come later.)
            bool loading = false;
            if(d + 1 < nb)
            {
                if(tid == 0) sm.ok = (d + 1 < 2 || ld_acquire(pre + d + 1) != 0) ? 1 : 0;
                __syncthreads();
                loading = sm.ok != 0;
                if(loading)
                {
                    tile_to_smem(sm.C2, A + (size_t)(d + 1) * T * ld + (size_t)d * T, ld);
                    tile_to_smem(sm.opB, A + (size_t)(d + 1) * T * ld + (size_t)(d + 1) * T, ld);
                    cp_async_commit();
                }
            }
            SPINE_STAMP(4);
            tile_to_global(Add, ld, sm.pb.L, true);
            {
                double* invLd = invL + (size_t)d * T * T;
                for(int e = tid; e < T * T / 2; e += 256)
                {
                    const int r = e >> 5, c = (e & 31) * 2;
                    *reinterpret_cast<double2*>(&invLd[r * T + c]) = *reinterpret_cast<const double2*>(&sm.pb.X[r * PLD + c]);
                }
            }
            SPINE_STAMP(5);
            if(stamps != nullptr && tid == 0) stamps[8 * d + 7] = loading ? 1 : 0;
            if(d + 1 < nb && !loading)
            {
                __syncthreads();
                if(tid == 255) st_release(flags + tile_flag(d, d, nb), 1);
                if(!wait_flags(sm, pre + d + 1, nullptr, abort_flag, info)) return;
                tile_to_smem(sm.C2, A + (size_t)(d + 1) * T * ld + (size_t)d * T, ld);
                tile_to_smem(sm.opB, A + (size_t)(d + 1) * T * ld + (size_t)(d + 1) * T, ld);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
            }
            else
            {
                cp_async_wait<0>();
                __syncthreads();
                if(tid == 255) st_release(flags + tile_flag(d, d, nb), 1);
            }
            SPINE_STAMP(6);
        }
        return;
    }
#undef SPINE_STAMP

    ////////////////////////////// the helpers
    const int nhelpers = gridDim.x - 1;
    const int ntasks = (nb - 1) * nb / 2 - 1;       // sum over j = 0 .. nb-3 of (nb - 1 - j)
    for(int tl = blockIdx.x - 1; tl < ntasks; tl += nhelpers)
    {
        int j = 0, rem = tl;
        while(rem >= nb - 1 - j) { rem -= nb - 1 - j; j++; }
        const bool is_pre = rem == 1;
        if(!is_pre)
        {
            // ---- the tile (i, j), i >= j+2
            const int i = rem == 0 ? j + 2 : j + 1 + rem;
            double* Aij = A + (size_t)i * T * ld + (size_t)j * T;
            tile_to_smem(sm.C2, Aij, ld);
            cp_async_commit();
            for(int k = 0; k < j; k++)
            {
                if(!wait_flags(sm, flags + tile_flag(i, k, nb), flags + tile_flag(j, k, nb), abort_flag, info)) return;
                tile_to_smem(sm.opA, A + (size_t)i * T * ld + (size_t)k * T, ld);
                tile_to_smem(sm.opB, A + (size_t)j * T * ld + (size_t)k * T, ld);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
                acc_zero(acc);
                tile_mma(acc, sm.opA, sm.opB);
                tile_sub(sm.C2, acc);
                __syncthreads();
            }
            if(!wait_flags(sm, flags + tile_flag(j, j, nb), nullptr, abort_flag, info)) return;
            tile_to_smem(sm.opB, invL + (size_t)j * T * T, T);
            cp_async_commit();
            cp_async_wait<0>();
            __syncthreads();
            tile_trsm(sm.C2, sm.opB, Aij, ld, nullptr);
            __threadfence();
            __syncthreads();
            if(tid == 0) st_release(flags + tile_flag(i, j, nb), 1);
        }
        else
        {
            // ---- pre(d), d = j+2: everything the spine's two tiles of step d get from the columns k <= d-2
            const int d = j + 2;
            double* Aij = A + (size_t)d * T * ld + (size_t)(d - 1) * T;
            double* Add = A + (size_t)d * T * ld + (size_t)d * T;
            tile_to_smem(sm.C2, Aij, ld);
            tile_to_smem(sm.pb.L, Add, ld);
            cp_async_commit();
            for(int k = 0; k <= d - 2; k++)
            {
                if(!wait_flags(sm, flags + tile_flag(d, k, nb), flags + tile_flag(d - 1, k, nb), abort_flag, info)) return;
                tile_to_smem(sm.opA, A + (size_t)d * T * ld + (size_t)k * T, ld);
                tile_to_smem(sm.opB, A + (size_t)(d - 1) * T * ld + (size_t)k * T, ld);
                cp_async_commit();
                cp_async_wait<0>();
                __syncthreads();
                acc_zero(acc);
                tile_mma(acc, sm.opA, sm.opB);
                tile_sub(sm.C2, acc);
                acc_zero(acc);
                tile_mma(acc, sm.opA, sm.opA);
                tile_sub(sm.pb.L, acc);
                __syncthreads();
            }
            tile_to_global(Aij, ld, sm.C2, false);
            tile_to_global(Add, ld, sm.pb.L, true);
            __threadfence();
            __syncthreads();
            if(tid == 0) st_release(pre + d, 1);
        }
        __syncthreads();
    }
}

// Backward substitution L' x = y, one right-hand side, one CTA per 64-row block (walking
// down from the last block). Block i needs x_j for all j > i: it polls the x values
// themselves (the slots hold a sentinel until written), so a hop between consecutive
// blocks costs one L2 round trip. The tiles L_ji are prefetched into registers before
// the wait.
__global__ void __launch_bounds__(256, 1)
chol_backward_dataflow_kernel(const double* __restrict__ L, int ld, int nb, const double* __restrict__ invL,
                              double* __restrict__ B, double* __restrict__ xbuf, int* __restrict__ abort_flag, int* __restrict__ info)
{
    __shared__ double xs[T];
    __shared__ double red[4][T];
    __shared__ double tv[T];
    __shared__ int okflag;
    const int tid = threadIdx.x, c = tid & 63, q = tid >> 6;
    if(tid == 0) okflag = 1;
    __syncthreads();
    for(int i = nb - 1 - (int)blockIdx.x; i >= 0; i -= gridDim.x)
    {
        double part = 0.;
        for(int jb = nb - 1; jb > i; jb--)
        {
            double v[16];
#pragma unroll
            for(int r = 0; r < 16; r++) v[r] = __ldcg(&L[(size_t)(jb * T + q * 16 + r) * ld + i * T + c]);
            if(tid < T)
            {
                const volatile double* src = xbuf + jb * T + tid;
                double x = *src;
                int ok = 1;
                const long long t0 = clock64();
                while(__double_as_longlong(x) == -1ll)
                {
                    if(clock64() - t0 > kSpinLimit || *(volatile int*)abort_flag != 0) { *(volatile int*)abort_flag = 1; atomicExch(info, -9); ok = 0; break; }
                    x = *src;
                }
                xs[tid] = x;
                if(!ok) okflag = 0;
            }
            __syncthreads();
            if(*(volatile int*)&okflag == 0) return;
#pragma unroll
            for(int r = 0; r < 16; r++) part = fma(v[r], xs[q * 16 + r], part);
            __syncthreads();
        }
        red[q][c] = part;
        __syncthreads();
        if(tid < T) tv[tid] = B[i * T + tid] - (red[0][tid] + red[1][tid] + red[2][tid] + red[3][tid]);
        __syncthreads();
        // x_i = inv(L_ii)' t:  x[c] = sum_{m >= c} invL[m][c] t[m]
        const double* Li = invL + (size_t)i * T * T;
        double acc = 0.;
#pragma unroll
        for(int r = 0; r < 16; r++)
        {
            const int m = q * 16 + r;
            acc = fma(__ldcg(&Li[m * T + c]), tv[m], acc);   // zeros above the diagonal
        }
        red[q][c] = acc;
        __syncthreads();
        if(tid < T)
        {
            const double x = red[0][tid] + red[1][tid] + red[2][tid] + red[3][tid];
            B[i * T + tid] = x;
            *(volatile double*)(xbuf + i * T + tid) = x;
        }
        __syncthreads();
    }
}

// SMs of the current device, once the kernels are set up for it (cached per device)
int g_num_sms[kMaxDevices];

// the SM count; 0 (and set_error) if the persistent kernels cannot run on the current device
int configure()
{
    int dev = 0;
    if(cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices)
    {
        set_error("the persistent Cholesky kernels: no usable current device: %s", cudaGetErrorString(cudaGetLastError()));
        return 0;
    }
    if(g_num_sms[dev] > 0) return g_num_sms[dev];
    int coop = 0, sms = 0;
    cudaError_t e = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
    if(e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if(e == cudaSuccess) e = cudaFuncSetAttribute(chol_spine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DfSmem));
    // (the spine needs a second CTA for its pre tasks from nb = 3 on)
    if(e != cudaSuccess || !coop || sms < 2)
    {
        cudaGetLastError();
        set_error("the persistent Cholesky kernels cannot run on device %d (cooperative launch: %d, SMs: %d): %s", dev, coop, sms,
                  cudaGetErrorString(e));
        return 0;
    }
    return g_num_sms[dev] = sms;
}

bool scratch_fits(const CholScratch* sc, int npad)
{
    if(sc != nullptr && npad <= sc->npad_max) return true;
    set_error("Cholesky of a %d x %d system with a scratch for at most %d x %d", npad, npad, sc ? sc->npad_max : 0, sc ? sc->npad_max : 0);
    return false;
}

long long* g_debug_stamps = nullptr;   // set by chol_debug_spine_stamps() only
int* g_debug_grid = nullptr;           // set by chol_debug_factor() only: the spine kernel's grid goes there

// the persistent factorization (chol_factor up to npad = 8192)
bool chol_factor_spine(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch,
                       CholScratch* scratch)
{
    const int num_sms = configure();
    if(num_sms == 0) return false;
    int nb = npad / T, ld = npad;
    const int ntiles = nb * (nb + 1) / 2;
    int* abort_flag = scratch->flags;
    int* flags = abort_flag + 1;
    int* pre = flags + ntiles;
    WordFill clear;
    clear.add(d_info, sizeof(int));
    clear.add(abort_flag, (size_t)(1 + ntiles + nb) * sizeof(int));
    if(!fill_words(clear, s)) return false;
    long long* stamps = g_debug_stamps;
    void* args[] = {&A, &ld, &nb, &nreal, &invL, &d_info, &flags, &pre, &abort_flag, &stamps};
    // the spine CTA and up to one helper CTA per helper task (see the kernel; none for nb <= 2) on the other SMs
    const int nhelper_tasks = nb >= 3 ? (nb - 1) * nb / 2 - 1 : 0;
    const int grid = 1 + (nhelper_tasks < num_sms - 1 ? nhelper_tasks : num_sms - 1);
    MB200_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)chol_spine_kernel, dim3(grid), dim3(256), args, sizeof(DfSmem), s));
    if(nlaunch) (*nlaunch)++;
    if(g_debug_grid) *g_debug_grid = grid;
    return true;
}

}  // namespace

// flags: the abort flag, then for a system of nb blocks one flag per tile of the lower triangle and the spine's nb
// pre counters; xbuf: the solution slots of the backward substitution
bool chol_scratch_create(CholScratch* sc, int npad_max)
{
    const size_t nb = (size_t)(npad_max / T);
    sc->flags = nullptr; sc->xbuf = nullptr; sc->npad_max = 0;
    if(cudaMalloc(&sc->flags, (1 + nb * (nb + 1) / 2 + nb) * sizeof(int)) != cudaSuccess ||
       cudaMalloc(&sc->xbuf, nb * T * sizeof(double)) != cudaSuccess)
    {
        set_error("cudaMalloc of the factorization scratch failed: %s", cudaGetErrorString(cudaGetLastError()));
        chol_scratch_destroy(sc);
        return false;
    }
    sc->npad_max = npad_max;
    return true;
}
void chol_scratch_destroy(CholScratch* sc)
{
    if(sc->flags) cudaFree(sc->flags);
    if(sc->xbuf) cudaFree(sc->xbuf);
    sc->flags = nullptr; sc->xbuf = nullptr; sc->npad_max = 0;
}

bool chol_factor(double* A, int npad, int nreal, double* invL, int* d_info, cudaStream_t s, int* nlaunch,
                 CholScratch* scratch)
{
    if(!scratch_fits(scratch, npad)) return false;
    // Above 8192 unknowns the multi-kernel factorization (chol.cu) is faster: 39 against 43 ms at n = 12000, 159
    // against 187 ms at n = 19376 (DESIGN section 9)
    if(npad > 8192) return chol_factor_blocked(A, npad, nreal, invL, d_info, s, nlaunch);
    return chol_factor_spine(A, npad, nreal, invL, d_info, s, nlaunch, scratch);
}

bool chol_solve_backward(const double* L, int npad, const double* invL, double* B, int* d_info, cudaStream_t s, int* nlaunch,
                         CholScratch* scratch)
{
    const int num_sms = configure();
    if(num_sms == 0 || !scratch_fits(scratch, npad)) return false;
    int nb = npad / T, ld = npad;
    int* abort_flag = scratch->flags;
    WordFill clear;   // the solution slots to all-ones bytes (not yet written), the abort flag to 0
    clear.add(scratch->xbuf, (size_t)nb * T * sizeof(double), 0xffffffffu);
    clear.add(abort_flag, sizeof(int));
    if(!fill_words(clear, s)) return false;
    double* xbuf = scratch->xbuf;
    void* args[] = {&L, &ld, &nb, &invL, &B, &xbuf, &abort_flag, &d_info};
    const int grid = nb < num_sms ? nb : num_sms;
    MB200_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)chol_backward_dataflow_kernel, dim3(grid), dim3(256), args, 0, s));
    if(nlaunch) (*nlaunch)++;
    return true;
}

// Debugging aid (not on any product path): clock64() stamps of the spine of one factorization of an n x n matrix:
// out[8 d + k], k = 0 step start, 1 triangular product done, 2 diagonal tile ready, 3 potrf_block done, 4 next loads
// issued, 5 written out and flagged, 6 step end, 7 whether the next tiles were ready when asked
void chol_debug_fill_spd(double* A, int npad, cudaStream_t s);   // chol.cu
bool chol_debug_spine_stamps(int n, long long* out, int nmax)
{
    const int npad = chol_padded(n), nb = npad / T;
    if(nmax < 8 * nb) return false;
    double *A = nullptr, *invL = nullptr; int* info = nullptr; long long* st = nullptr;
    cudaStream_t s;
    MB200_CUDA_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    MB200_CUDA_CHECK(cudaMalloc(&A, (size_t)npad * npad * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&invL, (size_t)npad * T * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&info, sizeof(int)));
    MB200_CUDA_CHECK(cudaMalloc(&st, (size_t)8 * nb * sizeof(long long)));
    MB200_CUDA_CHECK(cudaMemsetAsync(st, 0, (size_t)8 * nb * sizeof(long long), s));
    CholScratch sc;
    bool ok = chol_scratch_create(&sc, npad);
    for(int rep = 0; rep < 3 && ok; rep++)
    {
        chol_debug_fill_spd(A, npad, s);
        g_debug_stamps = rep == 2 ? st : nullptr;
        ok = chol_factor(A, npad, n, invL, info, s, nullptr, &sc);
        g_debug_stamps = nullptr;
    }
    ok = ok && cudaMemcpyAsync(out, st, (size_t)8 * nb * sizeof(long long), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaStreamSynchronize(s) == cudaSuccess;
    chol_scratch_destroy(&sc);
    cudaFree(A); cudaFree(invL); cudaFree(info); cudaFree(st);
    cudaStreamDestroy(s);
    return ok;
}

// Test aid (not on any product path): factor the lower triangle of the host n x n matrix A0 (row-major), padded to
// npad = chol_padded(n) with 1 on the padding diagonal; pivots >= nreal are not reported. path: 0 what chol_factor
// picks, 1 the spine kernel (npad <= 8192), 2 chol_factor_blocked. Out: L_out (npad x npad, the whole buffer),
// invL_out (npad/64 blocks of 64 x 64), *info_out, grid_out[4] = {path that ran, CTAs of the spine kernel's cooperative
// launch (0: not launched), SMs of the device, helper tasks of the spine kernel}
bool chol_debug_factor(const double* A0, int n, int nreal, int path, double* L_out, double* invL_out, int* info_out, int* grid_out)
{
    const int npad = chol_padded(n), nb = npad / T;
    if(n <= 0 || nreal < 0 || nreal > n || path < 0 || path > 2 || (path == 1 && npad > 8192))
    {
        set_error("chol_debug_factor: bad arguments (n %d, nreal %d, path %d)", n, nreal, path);
        return false;
    }
    const int sms = configure();
    if(sms == 0) return false;
    std::vector<double> h((size_t)npad * npad, 0.);
    for(int i = 0; i < npad; i++)
        for(int j = 0; j <= i; j++) h[(size_t)i * npad + j] = i < n ? A0[(size_t)i * n + j] : (i == j ? 1. : 0.);
    double *A = nullptr, *invL = nullptr; int* info = nullptr;
    cudaStream_t s = nullptr;
    CholScratch sc;
    int grid = 0;
    bool ok = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&A, (size_t)npad * npad * sizeof(double)) == cudaSuccess &&
              cudaMalloc(&invL, (size_t)npad * T * sizeof(double)) == cudaSuccess && cudaMalloc(&info, sizeof(int)) == cudaSuccess &&
              chol_scratch_create(&sc, npad) &&
              cudaMemcpyAsync(A, h.data(), h.size() * sizeof(double), cudaMemcpyHostToDevice, s) == cudaSuccess &&
              cudaMemsetAsync(invL, 0xff, (size_t)npad * T * sizeof(double), s) == cudaSuccess;   // NaN: every entry must be written
    if(ok)
    {
        g_debug_grid = &grid;
        ok = path == 0 ? chol_factor(A, npad, nreal, invL, info, s, nullptr, &sc)
           : path == 1 ? chol_factor_spine(A, npad, nreal, invL, info, s, nullptr, &sc)
                       : chol_factor_blocked(A, npad, nreal, invL, info, s, nullptr);
        g_debug_grid = nullptr;
    }
    ok = ok && cudaMemcpyAsync(L_out, A, (size_t)npad * npad * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(invL_out, invL, (size_t)npad * T * sizeof(double), cudaMemcpyDeviceToHost, s) == cudaSuccess &&
         cudaMemcpyAsync(info_out, info, sizeof(int), cudaMemcpyDeviceToHost, s) == cudaSuccess && cudaStreamSynchronize(s) == cudaSuccess;
    if(!ok) set_error("chol_debug_factor failed: %s", cudaGetErrorString(cudaGetLastError()));
    grid_out[0] = grid > 0 ? 1 : 2;
    grid_out[1] = grid;
    grid_out[2] = sms;
    grid_out[3] = nb >= 3 ? (nb - 1) * nb / 2 - 1 : 0;
    if(s) cudaStreamSynchronize(s);
    chol_forget_graphs(A);   // the blocked path caches a graph keyed on A
    chol_scratch_destroy(&sc);
    cudaFree(A); cudaFree(invL); cudaFree(info);
    if(s) cudaStreamDestroy(s);
    return ok;
}

}  // namespace mb200
