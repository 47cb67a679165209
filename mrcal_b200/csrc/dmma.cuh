// Internal: one fp64 tensor-core product, mma.sync.m8n8k4 (row x col): {c0, c1} += a b over the 8x8x4 fragment
#pragma once

namespace mb200 {

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b)
{
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

}  // namespace mb200
