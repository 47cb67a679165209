// Internal: the fixed-order sums and the block-wide scans of the kernels.
//
// Every floating-point sum here adds its operands in an order that depends only on the launch shape, never on timing:
// the same inputs give the same bits from run to run. Each helper states its association; a kernel that needs another
// one (zero padding, pairwise combinations of a few partials) writes it out where it is used.
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

// Butterfly over the 32 lanes of a warp (all of them active): at step o = 16, 8, 4, 2, 1 every lane adds the value of
// lane ^ o to its own. Every lane ends with the same bits (a + b == b + a): for lane 0,
// (((v0 + v16) + (v8 + v24)) + ((v4 + v20) + (v12 + v28))) + ...,  a balanced tree over the lanes in bit-reversed order
template <typename T>
__device__ __forceinline__ T warp_sum(T v)
{
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// the same for each of N values, in place (their shuffles interleaved)
template <typename T, int N>
__device__ __forceinline__ void warp_sum(T (&v)[N])
{
#pragma unroll
    for(int o = 16; o > 0; o >>= 1)
#pragma unroll
        for(int k = 0; k < N; k++) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
}

// Block sums of NV values per thread, over the warps of the block (all threads call it): each warp's warp_sum() goes to
// s[k][warp], and after a barrier thread k < NV adds the nw partials of value k in warp order onto zero,
// ((0 + s[k][0]) + s[k][1]) + ... + s[k][nw - 1]  (so a sum of -0 partials is +0). Returns the sum in threads k < NV
template <int NV, int NW, typename T>
__device__ __forceinline__ T block_sum_by_warps(T (&v)[NV], T (*s)[NW], int nw = NW)
{
    warp_sum(v);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if(lane == 0)
#pragma unroll
        for(int k = 0; k < NV; k++) s[k][w] = v[k];
    __syncthreads();
    T t = 0;
    if(threadIdx.x < NV)
        for(int i = 0; i < nw; i++) t += s[threadIdx.x][i];
    return t;
}

// Halving tree over the NT slots of s (NT threads, a power of two; all of them call it): thread i stores v to s[i],
// then at step o = NT/2, ..., 1 slot i < o adds slot i + o. Afterwards s[0] holds the sum, visible to every thread:
// for NT = 4, (s0 + s2) + (s1 + s3)
template <int NT, typename T>
__device__ __forceinline__ void tree_sum(T* s, T v)
{
    const int tid = threadIdx.x;
    s[tid] = v;
    __syncthreads();
    for(int o = NT / 2; o > 0; o >>= 1) { if(tid < o) s[tid] += s[tid + o]; __syncthreads(); }
}

// *out += the sum of part[0, n), one CTA of NT threads: thread i adds a contiguous stretch of ceil(n / NT) partials in
// index order onto zero, and tree_sum() adds the NT stretch sums
template <int NT>
__global__ void __launch_bounds__(NT) sum_partials_kernel(const double* __restrict__ part, int n, double* __restrict__ out)
{
    __shared__ double s[NT];
    const int tid = threadIdx.x;
    const int per = (n + NT - 1) / NT;
    double a = 0.;
    for(int i = tid * per; i < min(n, (tid + 1) * per); i++) a += part[i];
    tree_sum<NT>(s, a);
    if(tid == 0) *out += s[0];
}

// Exclusive prefix sum of v over the NT threads of the block (all of them call it; an integer type), through s[NT] in
// shared memory (Hillis-Steele). Returns the sum of the values of the threads before this one; *total <- the block's sum.
// s may be written again after the next barrier
template <typename T, int NT>
__device__ __forceinline__ T block_exclusive_scan(T v, T* s, T& total)
{
    const int tid = threadIdx.x;
    s[tid] = v;
    __syncthreads();
    for(int o = 1; o < NT; o <<= 1)
    {
        const T u = tid >= o ? s[tid - o] : T(0);
        __syncthreads();
        s[tid] += u;
        __syncthreads();
    }
    total = s[NT - 1];
    return s[tid] - v;
}

}  // namespace mb200
