// The triangulation routines of mrcal.triangulation on the device: one element-wise kernel family, templated on the
// method and on whether it gives gradients. Each thread takes one element of the broadcast shape (broadcast.cuh):
// it reads v0, v1 and t01 (or Rt01) through their strides, runs the method of triangulation.cuh (or the solver's own
// triangulated_error() of triangulated.cuh) in fp64 registers and writes the point and any gradients, packed.
#include "broadcast.cuh"
#include "triangulation.cuh"

namespace mb200 {

namespace {

enum { F_GRAD = MRCAL_B200_TRIANGULATE_GET_GRADIENTS, ERROR = MRCAL_B200_TRIANGULATE_TRIANGULATED_ERROR,
       LINDSTROM = MRCAL_B200_TRIANGULATE_LINDSTROM };

// doubles per element of the third input (t01 or Rt01) and of each output; nvars: the inputs the gradients are taken
// with respect to; pass: derivative components carried at once (the gradients take nvars / pass passes)
struct MethodShape
{
    int in2, out0, out1, out2, out3, nvars, pass;
};

__host__ __device__ constexpr MethodShape method_shape(int method)
{
    return method == LINDSTROM ? MethodShape{12, 3, 9, 9, 36, 18, 3}
         : method == ERROR     ? MethodShape{3, 1, 3, 3, 0, 6, 6}
                               : MethodShape{3, 3, 9, 9, 9, 9, 9};
}

struct TriArgs : Broadcast<3>
{
    double* out[4];                     // packed: element e's output k at out[k] + e * out_k
};

// the point m of method M, with derivative components first .. first + N - 1; false where the method fails
template <int M, int N>
__device__ __forceinline__ bool triangulate(Dual<N> m[3], const double* x0, const double* x1, const double* x2,
                                            int first)
{
    Dual<N> v0[3], v1[3], t01[3];
    tri_load(v0, x0, 0, first);
    tri_load(v1, x1, 3, first);
    if constexpr(M == LINDSTROM)
    {
        Dual<N> R01[9];
#pragma unroll
        for(int i = 0; i < 9; i++) R01[i] = Dual<N>::var(x2[i], 6 + i - first);
        tri_load(t01, &x2[9], 15, first);
        return tri_lindstrom(m, v0, v1, R01, t01);
    }
    else
    {
        tri_load(t01, x2, 6, first);
        if constexpr(M == MRCAL_B200_TRIANGULATE_GEOMETRIC) return tri_geometric(m, v0, v1, t01);
        else if constexpr(M == MRCAL_B200_TRIANGULATE_LEECIVERA_L1) return tri_leecivera_l1(m, v0, v1, t01);
        else if constexpr(M == MRCAL_B200_TRIANGULATE_LEECIVERA_LINF) return tri_leecivera_linf(m, v0, v1, t01);
        else if constexpr(M == MRCAL_B200_TRIANGULATE_LEECIVERA_MID2) return tri_leecivera_mid2(m, v0, v1, t01);
        else return tri_leecivera_wmid2(m, v0, v1, t01);
    }
}

// x, through an instruction the compiler neither moves nor merges with another
__device__ __forceinline__ double opaque(double x)
{
    double y;
    asm volatile("mov.b64 %0, %1;" : "=d"(y) : "d"(x));
    return y;
}

// the point, and the gradients dp/dv0, dp/dv1 and dp/dt01 (or dp/dRt01), zeros where the method fails, in passes over
// the derivative components first .. first + pass - 1. The point is written by the first pass: the point and its
// gradients come from one instantiation, so they agree on whether the method failed. Each pass recomputes the values
// from copies of the inputs the compiler cannot see through, rather than keeping them live across the passes (which
// spills Lindstrom's)
template <int M>
__device__ __forceinline__ void gradients(const TriArgs& a, int64_t e, const double* x0, const double* x1,
                                          const double* x2)
{
    constexpr MethodShape S = method_shape(M);
    constexpr int W3 = S.out3 / 3;
#pragma unroll 1
    for(int first = 0; first < S.nvars; first += S.pass)
    {
        double y0[3], y1[3], y2[S.in2];
#pragma unroll
        for(int i = 0; i < 3; i++)
        {
            y0[i] = opaque(x0[i]);
            y1[i] = opaque(x1[i]);
        }
#pragma unroll
        for(int i = 0; i < S.in2; i++) y2[i] = opaque(x2[i]);
        Dual<S.pass> m[3];
        const bool ok = triangulate<M, S.pass>(m, y0, y1, y2, first);
        if(first == 0)
#pragma unroll
            for(int i = 0; i < 3; i++) a.out[0][e * 3 + i] = ok ? m[i].x : 0.;
#pragma unroll
        for(int c = 0; c < S.pass; c++)
        {
            const int k = first + c;
            if(k >= S.nvars) break;
            double* p = k < 3 ? a.out[1] + e * 9 + k : k < 6 ? a.out[2] + e * 9 + k - 3 : a.out[3] + e * S.out3 + k - 6;
            const int w = k < 6 ? 3 : W3;
#pragma unroll
            for(int i = 0; i < 3; i++) p[w * i] = ok ? m[i].j[c] : 0.;
        }
    }
}

template <int M, bool G> __global__ void __launch_bounds__(256) triangulation_kernel(const TriArgs a)
{
    constexpr MethodShape S = method_shape(M);
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(e >= a.N) return;
    int64_t o[3];
    broadcast_offsets(a, e, o);
    double x0[3], x1[3], x2[S.in2];
#pragma unroll
    for(int i = 0; i < 3; i++)
    {
        x0[i] = __ldg(&a.in[0][o[0] + i]);
        x1[i] = __ldg(&a.in[1][o[1] + i]);
    }
#pragma unroll
    for(int i = 0; i < S.in2; i++) x2[i] = __ldg(&a.in[2][o[2] + i]);

    if constexpr(M == ERROR)
    {
        // the solver's per-pair error itself; v0 carries no gradient
        double dv1[3], dt01[3];
        a.out[0][e] = triangulated_error(dv1, dt01, x0, x1, x2);
        if constexpr(G)
#pragma unroll
            for(int i = 0; i < 3; i++)
            {
                a.out[1][e * 3 + i] = dv1[i];
                a.out[2][e * 3 + i] = dt01[i];
            }
    }
    else if constexpr(G)
        gradients<M>(a, e, x0, x1, x2);
    else
    {
        // the point alone carries no derivative components
        Dual<0> m[3];
        const bool ok = triangulate<M, 0>(m, x0, x1, x2, 0);
#pragma unroll
        for(int i = 0; i < 3; i++) a.out[0][e * 3 + i] = ok ? m[i].x : 0.;
    }
}

template <int M> void launch_method(const TriArgs& a, cudaStream_t stream)
{
    const unsigned blocks = (unsigned)((a.N + 255) / 256);
    if(a.flags & F_GRAD) triangulation_kernel<M, true><<<blocks, 256, 0, stream>>>(a);
    else triangulation_kernel<M, false><<<blocks, 256, 0, stream>>>(a);
}

template <int M = 0> void dispatch(int method, const TriArgs& a, cudaStream_t stream)
{
    if constexpr(M < MRCAL_B200_TRIANGULATE_NUM_METHODS)
    {
        if(method == M) launch_method<M>(a, stream);
        else dispatch<M + 1>(method, a, stream);
    }
}

// The checks both flavours make, and the broadcast frame of the launch. Pointers are not filled in
bool prepare(TriArgs& a, int method, int flags, int ndim, const int64_t* shape, const int64_t* strides0,
             const int64_t* strides1, const int64_t* strides2)
{
    if(method < 0 || method >= MRCAL_B200_TRIANGULATE_NUM_METHODS)
    {
        set_error("triangulate: unknown method %d", method);
        return false;
    }
    if(flags & ~F_GRAD)
    {
        set_error("triangulate: unknown flags 0x%x", flags);
        return false;
    }
    const int64_t* const st[3] = {strides0, strides1, strides2};
    const int width[3] = {3, 3, method_shape(method).in2};
    a = TriArgs{};
    return broadcast_prepare<3>(a, "triangulate", flags, ndim, shape, st, width);
}

}  // namespace

}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_triangulate(int method, int flags, int ndim, const int64_t* shape, const double* v0,
                                       const int64_t* strides0, const double* v1, const int64_t* strides1,
                                       const double* t01_or_Rt01, const int64_t* strides2, double* out0,
                                       double* out1, double* out2, double* out3)
{
    TriArgs a;
    if(!prepare(a, method, flags, ndim, shape, strides0, strides1, strides2)) return false;
    if(a.N == 0) return true;
    const MethodShape S = method_shape(method);
    const bool G = flags & F_GRAD;
    const size_t n[4] = {a.N * (size_t)S.out0, G ? a.N * (size_t)S.out1 : 0, G ? a.N * (size_t)S.out2 : 0,
                         G ? a.N * (size_t)S.out3 : 0};
    double* host_out[4] = {out0, out1, out2, out3};
    const double* host_in[3] = {v0, v1, t01_or_Rt01};
    const int width[3] = {3, 3, S.in2};
    DeviceCall D;
    if(!D.start()) return false;
    for(int k = 0; k < 3; k++)
        if(!D.upload((double**)&a.in[k], host_in[k], broadcast_extent(a, k, width[k]))) return false;
    for(int k = 0; k < 4; k++)
        if(n[k] && !D.alloc(&a.out[k], n[k])) return false;
    dispatch(method, a, D.stream);
    MB200_CUDA_CHECK(cudaGetLastError());
    for(int k = 0; k < 4; k++)
        if(n[k] && !D.download(host_out[k], a.out[k], n[k])) return false;
    return D.finish();
}

extern "C" bool mrcal_b200_triangulate_device(int method, int flags, int ndim, const int64_t* shape, const double* v0,
                                              const int64_t* strides0, const double* v1, const int64_t* strides1,
                                              const double* t01_or_Rt01, const int64_t* strides2, double* out0,
                                              double* out1, double* out2, double* out3, void* stream)
{
    TriArgs a;
    if(!prepare(a, method, flags, ndim, shape, strides0, strides1, strides2)) return false;
    if(a.N == 0) return true;
    if(!have_device()) return false;
    a.in[0] = v0;
    a.in[1] = v1;
    a.in[2] = t01_or_Rt01;
    a.out[0] = out0;
    a.out[1] = out1;
    a.out[2] = out2;
    a.out[3] = out3;
    dispatch(method, a, (cudaStream_t)stream);
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}
