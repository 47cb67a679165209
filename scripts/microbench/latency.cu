// Dependent-issue latencies (SM cycles) of the instructions on the pivot chain of potrf_block.cuh.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o latency latency.cu && ./latency
#include <cstdio>
#include <cuda_runtime.h>
constexpr int N = 512;
template <int KIND> __global__ void chain(double* out, long long* cyc, double seed)
{
    double x = seed + threadIdx.x * 1e-9, y = 1.0000001;
    long long t0 = clock64();
#pragma unroll 1
    for(int it = 0; it < N / 16; it++)
    {
#pragma unroll
        for(int u = 0; u < 16; u++)
        {
            if(KIND == 0) x = fma(x, y, 1e-9);                               // DFMA
            if(KIND == 1) x = x * y;                                          // DMUL
            if(KIND == 2) x = x + y;                                          // DADD
            if(KIND == 3) x = __shfl_sync(0xffffffffu, x, (u * 7 + 1) & 31);  // SHFL x2 (64 bit)
            if(KIND == 4) asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(x) : "d"(x));   // MUFU.RCP64H
            if(KIND == 5) asm volatile("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(x) : "d"(x));
            if(KIND == 6) x = (x > 0.5) ? x : y;                              // DSETP + SEL
            if(KIND == 7) { const int hi = __double2hiint(x); x = (hi >= 0x03f00000 && hi < 0x7ff00000) ? x : y; x = __longlong_as_double(__double_as_longlong(x) + 1); }
            if(KIND == 8) { float f = (float)x; f = f * 1.0001f; x = (double)f; }   // F2F round trip + FMUL
            if(KIND == 9) x = __drcp_rn(x);
            if(KIND == 10) { int v = __shfl_sync(0xffffffffu, __double2loint(x), (u * 7 + 1) & 31); x = __hiloint2double(__double2hiint(x), v); }   // one SHFL
            if(KIND == 11) { float f = __int_as_float(__double2loint(x)); f = fmaf(f, 1.0001f, 1e-9f); x = __hiloint2double(__double2hiint(x), __float_as_int(f)); }  // FFMA
        }
    }
    long long t1 = clock64();
    out[threadIdx.x] = x;
    if(threadIdx.x == 0) cyc[KIND] = t1 - t0;
}
int main()
{
    double* out; long long* cyc;
    cudaMalloc(&out, 32 * 8); cudaMallocManaged(&cyc, 16 * 8);
    const char* names[] = {"DFMA", "DMUL", "DADD", "SHFL.64 (2 shfl)", "rcp.approx.f64 (MUFU.RCP64H)", "rsqrt.approx.f64", "DSETP+SEL", "ISETP x2+SEL+IADD64", "F2F.F32.F64+FMUL+F2F.F64.F32", "__drcp_rn", "SHFL.32", "FFMA"};
    for(int rep = 0; rep < 2; rep++)
    {
        chain<0><<<1, 32>>>(out, cyc, 1.); chain<1><<<1, 32>>>(out, cyc, 1.); chain<2><<<1, 32>>>(out, cyc, 1.); chain<3><<<1, 32>>>(out, cyc, 1.);
        chain<4><<<1, 32>>>(out, cyc, 1.5); chain<5><<<1, 32>>>(out, cyc, 1.5); chain<6><<<1, 32>>>(out, cyc, 1.); chain<7><<<1, 32>>>(out, cyc, 1.);
        chain<8><<<1, 32>>>(out, cyc, 1.); chain<9><<<1, 32>>>(out, cyc, 1.5); chain<10><<<1, 32>>>(out, cyc, 1.); chain<11><<<1, 32>>>(out, cyc, 1.);
        cudaDeviceSynchronize();
    }
    for(int k = 0; k < 12; k++) printf("%-34s %7.1f cycles per step\n", names[k], (double)cyc[k] / N);
    return 0;
}
