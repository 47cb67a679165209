// Microbenchmark: sustained FP64 throughput of the vector pipe (DFMA) and of the
// tensor pipe (DMMA.8x8x4) on this GPU. Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_rate fp64_rate.cu
#include <cstdio>
#include <cuda_runtime.h>

__global__ void dfma_kernel(double* out, int iters)
{
    double a0 = threadIdx.x, a1 = 1.0, a2 = 2.0, a3 = 3.0, a4 = 4., a5 = 5., a6 = 6., a7 = 7.;
    const double b = 1.0000001, c = 0.5;
    for(int i = 0; i < iters; i++)
    {
        a0 = a0 * b + c; a1 = a1 * b + c; a2 = a2 * b + c; a3 = a3 * b + c;
        a4 = a4 * b + c; a5 = a5 * b + c; a6 = a6 * b + c; a7 = a7 * b + c;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

__global__ void dmma_kernel(double* out, int iters)
{
    double c[8][2] = {};
    double a = threadIdx.x * 1e-3, b = 1.0 + threadIdx.x * 1e-6;
    for(int i = 0; i < iters; i++)
    {
#pragma unroll
        for(int j = 0; j < 8; j++)
            asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                         : "+d"(c[j][0]), "+d"(c[j][1]) : "d"(a), "d"(b));
    }
    double s = 0;
    for(int j = 0; j < 8; j++) s += c[j][0] + c[j][1];
    out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void ffma_kernel(float* out, int iters)
{
    float a0 = threadIdx.x, a1 = 1.f, a2 = 2.f, a3 = 3.f, a4 = 4.f, a5 = 5.f, a6 = 6.f, a7 = 7.f;
    const float b = 1.0000001f, c = 0.5f;
    for(int i = 0; i < iters; i++)
    {
        a0 = a0 * b + c; a1 = a1 * b + c; a2 = a2 * b + c; a3 = a3 * b + c;
        a4 = a4 * b + c; a5 = a5 * b + c; a6 = a6 * b + c; a7 = a7 * b + c;
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
}

int main()
{
    cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
    const int blocks = p.multiProcessorCount * 8, threads = 256, iters = 20000;
    double* d; cudaMalloc(&d, sizeof(double) * blocks * threads);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    float ms;
    for(int rep = 0; rep < 2; rep++)
    {
        cudaEventRecord(e0); dfma_kernel<<<blocks, threads>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if(rep) printf("DFMA   : %.2f TFLOP/s\n", 2.0 * 8 * iters * (double)blocks * threads / (ms * 1e-3) / 1e12);
        cudaEventRecord(e0); dmma_kernel<<<blocks, threads>>>(d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if(rep) printf("DMMA   : %.2f TFLOP/s\n", 2.0 * 8 * 256 * iters * (double)blocks * (threads / 32) / (ms * 1e-3) / 1e12);
        cudaEventRecord(e0); ffma_kernel<<<blocks, threads>>>((float*)d, iters); cudaEventRecord(e1); cudaEventSynchronize(e1);
        cudaEventElapsedTime(&ms, e0, e1);
        if(rep) printf("FFMA   : %.2f TFLOP/s\n", 2.0 * 8 * iters * (double)blocks * threads / (ms * 1e-3) / 1e12);
    }
    printf("%s, %d SMs\n", p.name, p.multiProcessorCount);
    return 0;
}
