// The triangulated-point measurement: the angular misfit of a pair of observation
// rays of the same (unparametrized) point, as the reference defines it in
// _mrcal_triangulated_error() (triangulation.cc:958-1123): the Lee-Civera "Mid2"
// midpoint, the small-angle ray-to-midpoint error doubled, and a smooth penalty
// for pairs that fail the cheirality test.
//
// The reference gets the gradients by forward-mode automatic differentiation over
// 6 inputs; so does this file, with the same dual-number type (dual.cuh): the function has
// branches whose derivatives are defined by "whatever the operations taken produce",
// and carrying the derivatives through the same operations is the one way to agree
// with that to rounding everywhere, branch boundaries included.
//
// The helpers are templates on the number of derivative components: the Mid2 ranges and the cheirality test here
// are also the ones triangulate_leecivera_mid2() and _wmid2() use (triangulation.cuh), over 9 inputs.
#pragma once
#include <cuda_runtime.h>

#include "dual.cuh"

namespace mb200 {

template <int N> __device__ __forceinline__ Dual<N> d_dot(const Dual<N> a[3], const Dual<N> b[3])
{
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2];
}
template <int N> __device__ __forceinline__ Dual<N> d_cross_norm2(const Dual<N> a[3], const Dual<N> b[3])
{
    const Dual<N> c0 = a[1] * b[2] - a[2] * b[1];
    const Dual<N> c1 = a[2] * b[0] - a[0] * b[2];
    const Dual<N> c2 = a[0] * b[1] - a[1] * b[0];
    return c0 * c0 + c1 * c1 + c2 * c2;
}

// angle between two vectors, small-angle form th = sqrt(2 (1 - |cos|)); exactly 0 (value and gradient)
// below 1e-21 (triangulation.cc:781-817)
template <int N> __device__ __forceinline__ Dual<N> d_angle_small(const Dual<N> a[3], const Dual<N> b[3])
{
    Dual<N> costh = d_dot(a, b) / dsqrt(d_dot(a, a) * d_dot(b, b));
    if(costh.x < 0.) costh = -costh;
    const Dual<N> th_sq = costh * (-2.) + 2.;
    if(th_sq.x < 1e-21) return Dual<N>(0.);
    return dsqrt(th_sq);
}

// 0 below 0, 1 above the knee, two parabolas in between (triangulation.cc:893-947)
template <int N> __device__ __forceinline__ Dual<N> d_sigmoid(const Dual<N>& x, double knee)
{
    if(x.x <= 0.) return Dual<N>(0.);
    if(knee <= x.x) return Dual<N>(1.);
    const double b = 2. / knee;
    const double a = (x.x < knee / 2. ? 2. : -2.) / knee / knee;
    const Dual<N> dx = x - knee / 2.;
    return dx * (dx * a + b) + 0.5;
}

// The Lee-Civera Mid2 ranges: l0 along v0 and l1 along v1 (from t01) of the two estimates of the point
// (triangulation.cc:662-665 and 986-989)
template <int N>
__device__ __forceinline__ void mid2_ranges(Dual<N>& l0, Dual<N>& l1, const Dual<N> v0[3], const Dual<N> v1[3],
                                            const Dual<N> t01[3])
{
    const Dual<N> p_norm2_recip = Dual<N>(1.) / d_cross_norm2(v0, v1);
    l0 = dsqrt(d_cross_norm2(v1, t01) * p_norm2_recip);
    l1 = dsqrt(d_cross_norm2(v0, t01) * p_norm2_recip);
}

// cheirality: does flipping the sign of l0, l1 or both bring the two estimates l0 v0 and t01 + l1 v1 of the point
// closer? w0, w1, w01: how much each flip worsens the fit; true if every flip worsens it (triangulation.cc:576-621)
template <int N>
__device__ __forceinline__ bool cheirality(Dual<N>& w0, Dual<N>& w1, Dual<N>& w01, const Dual<N>& l0,
                                           const Dual<N> v0[3], const Dual<N>& l1, const Dual<N> v1[3],
                                           const Dual<N> t01[3])
{
    w0 = w1 = w01 = Dual<N>(0.);
#pragma unroll
    for(int i = 0; i < 3; i++)
    {
        const Dual<N> far = l1 * v1[i], near = l0 * v0[i];
        const Dual<N> xn  = (far + t01[i]) - near;
        const Dual<N> x0  = (far + t01[i]) + near;
        const Dual<N> x1  = (t01[i] - far) - near;
        const Dual<N> x01 = (t01[i] - far) + near;
        const Dual<N> n2 = xn * xn;
        w0  = w0 + (x0 * x0 - n2);
        w1  = w1 + (x1 * x1 - n2);
        w01 = w01 + (x01 * x01 - n2);
    }
    return w0.x > 0. && w1.x > 0. && w01.x > 0.;
}

// err(v_fixed, a, t) with derr/da, derr/dt. In the reference's naming (triangulation.cc:960-975):
// v_fixed = _v0 (no gradient), a = _v1, t = _t01; all in the coordinate system of v_fixed's camera
__device__ inline double triangulated_error(double derr_da[3], double derr_dt[3],
                                            const double v_fixed[3], const double a_in[3], const double t_in[3])
{
    // values and gradients with respect to (a[0..2], t[0..2])
    Dual<6> v0[3], v1[3], t01[3];
#pragma unroll
    for(int i = 0; i < 3; i++)
    {
        v0[i] = Dual<6>(v_fixed[i]);
        v1[i] = Dual<6>::var(a_in[i], i);
        t01[i] = Dual<6>::var(t_in[i], 3 + i);
    }
    Dual<6> l0, l1;
    mid2_ranges(l0, l1, v0, v1, t01);
    Dual<6> m[3];
#pragma unroll
    for(int i = 0; i < 3; i++) m[i] = (v0[i] * l0 + t01[i] + v1[i] * l1) * 0.5;
    Dual<6> err = d_angle_small(v0, m) * 2.;

    Dual<6> w0, w1, w01;
    if(!cheirality(w0, w1, w01, l0, v0, l1, v1, t01))
    {
        const Dual<6> to_vanishing_point = d_angle_small(v0, v1);
        err = err + to_vanishing_point * (d_sigmoid(-w0, 3.) + d_sigmoid(-w1, 3.) + d_sigmoid(-w01, 3.));
    }
#pragma unroll
    for(int i = 0; i < 3; i++) { derr_da[i] = err.j[i]; derr_dt[i] = err.j[3 + i]; }
    return err.x;
}

}  // namespace mb200
