// A value and its gradient with respect to N inputs: the forward-mode arithmetic of the reference's val_withgrad_t
// (_autodiff.hh), so that a function restated with it takes the reference's branches and gives its gradients
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

template <int N> struct Dual
{
    double x;
    double j[N > 0 ? N : 1];
    __device__ Dual(double v = 0.) : x(v)
    {
#pragma unroll
        for(int i = 0; i < N; i++) j[i] = 0.;
    }
    // input number k of the N
    __device__ static Dual var(double v, int k)
    {
        Dual d(v);
#pragma unroll
        for(int i = 0; i < N; i++) d.j[i] = i == k ? 1. : 0.;
        return d;
    }
};

template <int N> __device__ __forceinline__ Dual<N> operator+(const Dual<N>& a, const Dual<N>& b)
{
    Dual<N> y(a.x + b.x);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] + b.j[i];
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& a, const Dual<N>& b)
{
    Dual<N> y(a.x - b.x);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] - b.j[i];
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator*(const Dual<N>& a, const Dual<N>& b)
{
    Dual<N> y(a.x * b.x);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] * b.x + a.x * b.j[i];
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator*(const Dual<N>& a, double b)
{
    Dual<N> y(a.x * b);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] * b;
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator/(const Dual<N>& a, const Dual<N>& b)
{
    Dual<N> y(a.x / b.x);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = (a.j[i] * b.x - a.x * b.j[i]) / (b.x * b.x);
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator/(const Dual<N>& a, double b) { return a * (1. / b); }
// a constant changes the value only
template <int N> __device__ __forceinline__ Dual<N> operator+(const Dual<N>& a, double b)
{
    Dual<N> y = a;
    y.x += b;
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& a, double b)
{
    Dual<N> y = a;
    y.x -= b;
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> operator-(const Dual<N>& a) { return a * -1.; }
template <int N> __device__ __forceinline__ Dual<N> dsqrt(const Dual<N>& a)
{
    Dual<N> y(sqrt(a.x));
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] / (2. * y.x);
    return y;
}
template <int N> __device__ __forceinline__ void dsincos(const Dual<N>& a, Dual<N>& s, Dual<N>& c)
{
    double sv, cv;
    sincos(a.x, &sv, &cv);
    s = Dual<N>(sv);
    c = Dual<N>(cv);
#pragma unroll
    for(int i = 0; i < N; i++) { s.j[i] = cv * a.j[i]; c.j[i] = -sv * a.j[i]; }
}
template <int N> __device__ __forceinline__ Dual<N> dtan(const Dual<N>& a)
{
    double sv, cv;
    sincos(a.x, &sv, &cv);
    Dual<N> y(sv / cv);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = a.j[i] / (cv * cv);
    return y;
}
template <int N> __device__ __forceinline__ Dual<N> dacos(const Dual<N>& a)
{
    Dual<N> y(acos(a.x));
    const double d = -1. / sqrt(1. - a.x * a.x);
#pragma unroll
    for(int i = 0; i < N; i++) y.j[i] = d * a.j[i];
    return y;
}

}  // namespace mb200
