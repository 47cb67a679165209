// The two-view triangulation methods of the reference (triangulation.cc), restated operation by operation over the
// dual numbers of dual.cuh so that they take the reference's branches and give its gradients:
//
//   geometric, leecivera_l1, leecivera_linf, leecivera_mid2, leecivera_wmid2: v0, v1, t01, all in camera 0's
//     coordinates; 9 inputs in the order v0 (0-2), v1 (3-5), t01 (6-8)
//   lindstrom: v0 and v1 in their own cameras' coordinates, and Rt01; 18 inputs: v0, v1, then Rt01's 12 (R01
//     row-major, then t01)
//
// Each returns false (the point is (0,0,0)) where the reference does: parallel or divergent rays, a point behind a
// camera. Input k carries derivative component k - first where that lies in [0, N), and no derivative otherwise: a
// caller that needs all the gradients but cannot hold them at once calls the method again with another first. In
// forward mode each derivative component depends only on the values and on itself, so passes of one instantiation
// (one N) give the same bits as one pass would, and take the same branches. Instantiations with different N are
// compiled separately, and the compiler may fuse multiplies and adds differently in each: their values can differ
// in the last bits, and so, within rounding of a threshold, their branches.
#pragma once
#include <cuda_runtime.h>

#include "triangulated.cuh"

namespace mb200 {

template <int N> __device__ __forceinline__ void tri_load(Dual<N> v[3], const double x[3], int k0, int first)
{
#pragma unroll
    for(int i = 0; i < 3; i++) v[i] = Dual<N>::var(x[i], k0 + i - first);
}

template <int N> __device__ __forceinline__ void d_cross(Dual<N> c[3], const Dual<N> a[3], const Dual<N> b[3])
{
    c[0] = a[1] * b[2] - a[2] * b[1];
    c[1] = a[2] * b[0] - a[0] * b[2];
    c[2] = a[0] * b[1] - a[1] * b[0];
}

// v /= |v|
template <int N> __device__ __forceinline__ void d_normalize(Dual<N> v[3])
{
    const Dual<N> mag = dsqrt(d_dot(v, v));
#pragma unroll
    for(int i = 0; i < 3; i++) v[i] = v[i] / mag;
}

// v -= n (v.n) / |n|^2: v projected onto the plane normal to n
template <int N> __device__ __forceinline__ void d_reject(Dual<N> v[3], const Dual<N> n[3])
{
    const Dual<N> vn = d_dot(n, v), nn = d_dot(n, n);
#pragma unroll
    for(int i = 0; i < 3; i++) v[i] = v[i] - n[i] * vn / nn;
}

// The intersection of two rays assumed to intersect, from their components A (x or y) and z
template <int A, int N>
__device__ __forceinline__ bool intersect_with(Dual<N> m[3], double fabs_det, const Dual<N> v0[3],
                                               const Dual<N> v1[3], const Dual<N> t01[3])
{
    if(fabs_det <= 1e-10) return false;
    const Dual<N> det = v1[A] * v0[2] - v0[A] * v1[2];
    const Dual<N> k0 = (t01[2] * v1[A] - t01[A] * v1[2]) / det;
    if(k0.x <= 0.) return false;
    const bool k1_negative = (t01[2].x * v0[A].x > t01[A].x * v0[2].x) ^ (det.x > 0);
    if(k1_negative) return false;
#pragma unroll
    for(int i = 0; i < 3; i++) m[i] = v0[i] * k0;
    return true;
}

// The intersection of two rays assumed to intersect, from the x and z or the y and z components, whichever has the
// larger determinant (triangulate_assume_intersect(), triangulation.cc:16-101). The two branches index the rays with
// constants, so the rays stay in registers
template <int N>
__device__ __forceinline__ bool assume_intersect(Dual<N> m[3], const Dual<N> v0[3], const Dual<N> v1[3],
                                                 const Dual<N> t01[3])
{
    const double fabs_det_xz = fabs(-v0[0].x * v1[2].x + v0[2].x * v1[0].x);
    const double fabs_det_yz = fabs(-v0[1].x * v1[2].x + v0[2].x * v1[1].x);
    if(fabs_det_xz > fabs_det_yz) return intersect_with<0>(m, fabs_det_xz, v0, v1, t01);
    return intersect_with<1>(m, fabs_det_yz, v0, v1, t01);
}

// the midpoint of the closest approach of the two rays (mrcal_triangulate_geometric(), triangulation.cc:106-209)
template <int N>
__device__ __forceinline__ bool tri_geometric(Dual<N> m[3], const Dual<N> v0[3], const Dual<N> v1[3],
                                              const Dual<N> t01[3])
{
    const Dual<N> dot_v0v0 = d_dot(v0, v0), dot_v1v1 = d_dot(v1, v1), dot_v0v1 = d_dot(v1, v0);
    const Dual<N> dot_v0t = d_dot(t01, v0), dot_v1t = d_dot(t01, v1);
    const Dual<N> denom = dot_v0v0 * dot_v1v1 - dot_v0v1 * dot_v0v1;
    if(-1e-10 <= denom.x && denom.x <= 1e-10) return false;
    const Dual<N> denom_recip = Dual<N>(1.) / denom;
    const Dual<N> k0 = denom_recip * (dot_v1v1 * dot_v0t - dot_v0v1 * dot_v1t);
    if(k0.x <= 0.) return false;
    const Dual<N> k1 = denom_recip * (dot_v0v1 * dot_v0t - dot_v0v0 * dot_v1t);
    if(k1.x <= 0.) return false;
#pragma unroll
    for(int i = 0; i < 3; i++) m[i] = (v0[i] * k0 + v1[i] * k1 + t01[i]) * 0.5;
    return true;
}

// L1 angular error: the ray more nearly perpendicular to t01 keeps its direction, the other is projected onto the
// epipolar plane (equations (12), (13); mrcal_triangulate_leecivera_l1(), triangulation.cc:436-510)
template <int N>
__device__ __forceinline__ bool tri_leecivera_l1(Dual<N> m[3], Dual<N> v0[3], Dual<N> v1[3], const Dual<N> t01[3])
{
    const double v0v0 = d_dot(v0, v0).x, v1v1 = d_dot(v1, v1).x;
    const double v0t = d_dot(t01, v0).x, v1t = d_dot(t01, v1).x;
    Dual<N> n[3];
    if(v0t * v0t * v1v1 > v1t * v1t * v0v0)
    {
        d_cross(n, v1, t01);
        d_reject(v0, n);
    }
    else
    {
        d_cross(n, v0, t01);
        d_reject(v1, n);
    }
    return assume_intersect(m, v0, v1, t01);
}

// L-infinity angular error: both rays projected onto the plane of the larger of cross(v0 +- v1, t01)
// (mrcal_triangulate_leecivera_linf(), triangulation.cc:515-573)
template <int N>
__device__ __forceinline__ bool tri_leecivera_linf(Dual<N> m[3], Dual<N> v0[3], Dual<N> v1[3], const Dual<N> t01[3])
{
    d_normalize(v0);
    d_normalize(v1);
    Dual<N> s[3], n[3], nb[3];
#pragma unroll
    for(int i = 0; i < 3; i++) s[i] = v0[i] + v1[i];
    d_cross(n, s, t01);
#pragma unroll
    for(int i = 0; i < 3; i++) s[i] = v0[i] - v1[i];
    d_cross(nb, s, t01);
    if(!(d_dot(n, n).x > d_dot(nb, nb).x))
#pragma unroll
        for(int i = 0; i < 3; i++) n[i] = nb[i];
    d_reject(v0, n);
    d_reject(v1, n);
    return assume_intersect(m, v0, v1, t01);
}

// Mid2: the midpoint of the two range estimates (mrcal_triangulate_leecivera_mid2(), triangulation.cc:640-689)
template <int N>
__device__ __forceinline__ bool tri_leecivera_mid2(Dual<N> m[3], const Dual<N> v0[3], const Dual<N> v1[3],
                                                   const Dual<N> t01[3])
{
    Dual<N> l0, l1, w0, w1, w01;
    mid2_ranges(l0, l1, v0, v1, t01);
    if(!cheirality(w0, w1, w01, l0, v0, l1, v1, t01)) return false;
#pragma unroll
    for(int i = 0; i < 3; i++) m[i] = (v0[i] * l0 + t01[i] + v1[i] * l1) * 0.5;
    return true;
}

// wMid2: the range estimates of unit rays, weighted by their inverse ranges (mrcal_triangulate_leecivera_wmid2(),
// triangulation.cc:710-764)
template <int N>
__device__ __forceinline__ bool tri_leecivera_wmid2(Dual<N> m[3], Dual<N> v0[3], Dual<N> v1[3], const Dual<N> t01[3])
{
    d_normalize(v0);
    d_normalize(v1);
    const Dual<N> p_mag_recip = Dual<N>(1.) / dsqrt(d_cross_norm2(v0, v1));
    const Dual<N> l0 = dsqrt(d_cross_norm2(v1, t01)) * p_mag_recip;
    const Dual<N> l1 = dsqrt(d_cross_norm2(v0, t01)) * p_mag_recip;
    Dual<N> w0, w1, w01;
    if(!cheirality(w0, w1, w01, l0, v0, l1, v1, t01)) return false;
    const Dual<N> sum = l0 + l1;
#pragma unroll
    for(int i = 0; i < 3; i++) m[i] = (v0[i] * l0 * l1 + t01[i] * l0 + v1[i] * l0 * l1) / sum;
    return true;
}

// Lindstrom's niter2 (Listing 3 of "Triangulation Made Easy", CVPR 2010): both observations corrected to satisfy
// the epipolar constraint, then intersected (mrcal_triangulate_lindstrom(), triangulation.cc:214-431).
// v0, v1: local; R01 row-major; t01
template <int N>
__device__ __forceinline__ bool tri_lindstrom(Dual<N> m[3], const Dual<N> v0[3], const Dual<N> v1[3],
                                              const Dual<N> R01[9], const Dual<N> t01[3])
{
    const Dual<N> E[9] = {R01[6] * t01[1] - R01[3] * t01[2], R01[7] * t01[1] - R01[4] * t01[2],
                          R01[8] * t01[1] - R01[5] * t01[2],

                          R01[0] * t01[2] - R01[6] * t01[0], R01[1] * t01[2] - R01[7] * t01[0],
                          R01[2] * t01[2] - R01[8] * t01[0],

                          R01[3] * t01[0] - R01[0] * t01[1], R01[4] * t01[0] - R01[1] * t01[1],
                          R01[5] * t01[0] - R01[2] * t01[1]};
    const Dual<N> x0[2] = {v0[0] / v0[2], v0[1] / v0[2]};
    const Dual<N> x1[2] = {v1[0] / v1[2], v1[1] / v1[2]};

    Dual<N> n[2] = {E[0] * x1[0] + E[1] * x1[1] + E[2], E[3] * x1[0] + E[4] * x1[1] + E[5]};
    Dual<N> nn[2] = {E[0] * x0[0] + E[3] * x0[1] + E[6], E[1] * x0[0] + E[4] * x0[1] + E[7]};
    const Dual<N> a = n[0] * E[0] * nn[0] + n[0] * E[1] * nn[1] + n[1] * E[3] * nn[0] + n[1] * E[4] * nn[1];
    const Dual<N> b = (n[0] * n[0] + n[1] * n[1] + nn[0] * nn[0] + nn[1] * nn[1]) * 0.5;
    const Dual<N> n_2 = E[6] * x1[0] + E[7] * x1[1] + E[8];
    const Dual<N> c = n[0] * x0[0] + n[1] * x0[1] + n_2;
    const Dual<N> d = dsqrt(b * b - a * c);
    Dual<N> l = c / (b + d);
    Dual<N> dx[2] = {l * n[0], l * n[1]};
    Dual<N> dxx[2] = {l * nn[0], l * nn[1]};
    n[0] = n[0] - E[0] * dxx[0] - E[1] * dxx[1];
    n[1] = n[1] - E[3] * dxx[0] - E[4] * dxx[1];
    nn[0] = nn[0] - E[0] * dx[0] - E[3] * dx[1];
    nn[1] = nn[1] - E[1] * dx[0] - E[4] * dx[1];
    const Dual<N> bb = (n[0] * n[0] + n[1] * n[1] + nn[0] * nn[0] + nn[1] * nn[1]) * 0.5;
    l = l / d * bb;
    dx[0] = l * n[0];
    dx[1] = l * n[1];
    dxx[0] = l * nn[0];
    dxx[1] = l * nn[1];

    const Dual<N> one(1.);
    const Dual<N> p0[3] = {x0[0] - dx[0], x0[1] - dx[1], one};
    const Dual<N> p1[3] = {x1[0] - dxx[0], x1[1] - dxx[1], one};
    Dual<N> Rp1[3];
#pragma unroll
    for(int i = 0; i < 3; i++) Rp1[i] = R01[3 * i] * p1[0] + R01[3 * i + 1] * p1[1] + R01[3 * i + 2] * p1[2];
    return assume_intersect(m, p0, Rp1, t01);
}

}  // namespace mb200
