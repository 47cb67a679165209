// Device pose functions: Rodrigues in both directions, composition with its gradients, the tiny-composition gradients,
// inversion, rotation and transformation of points, and the quaternion conversions. Every function works on one pose in
// registers, fp64, and follows the branches of the reference (poseutils.c, poseutils-opencv.c,
// poseutils-uses-autodiff.cc, mrcal/_poseutils_scipy.py; cited per function). Layouts are the reference's: R is
// row-major (3,3); Rt is (4,3), R then t; rt is (6,), r then t; a quaternion is (w,x,y,z). The ones marked __host__
// serve the host code too (stereo.cu).
#pragma once
#include <cuda_runtime.h>

#include "device_math.cuh"
#include "dual.cuh"

namespace mb200 {

// x rotated by r (by -r if inverted), the Rodrigues formula of rotate_point_r_core() (poseutils-uses-autodiff.cc:17-81),
// with its small-angle limit for |r|^2 < 1e-10
template <int N>
__device__ __forceinline__ void rotate_point_r_core(Dual<N> out[3], const Dual<N> r[3], const Dual<N> x[3], bool inverted)
{
    const double sign = inverted ? -1. : 1.;
    const Dual<N> th2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    const Dual<N> cross[3] = {(r[1] * x[2] - r[2] * x[1]) * sign, (r[2] * x[0] - r[0] * x[2]) * sign,
                              (r[0] * x[1] - r[1] * x[0]) * sign};
    const Dual<N> inner = r[0] * x[0] + r[1] * x[1] + r[2] * x[2];
    if(th2.x < 1e-10)
    {
#pragma unroll
        for(int i = 0; i < 3; i++) out[i] = x[i] + cross[i] + r[i] * inner / 2.;
        return;
    }
    const Dual<N> th = dsqrt(th2);
    Dual<N> s, c;
    dsincos(th, s, c);
#pragma unroll
    for(int i = 0; i < 3; i++) out[i] = x[i] * c + cross[i] * s / th + r[i] * inner * (Dual<N>(1.) - c) / th2;
}

// x rotated by r; with Jr, Jx: the (3,3) gradients with respect to r and x, row-major
__device__ __forceinline__ void rotate_point_r(double out[3], double* Jr, double* Jx, const double r[3],
                                               const double x[3], bool inverted)
{
    if(Jr == nullptr)
    {
        Dual<0> rg[3], xg[3], o[3];
#pragma unroll
        for(int i = 0; i < 3; i++) { rg[i] = Dual<0>(r[i]); xg[i] = Dual<0>(x[i]); }
        rotate_point_r_core(o, rg, xg, inverted);
#pragma unroll
        for(int i = 0; i < 3; i++) out[i] = o[i].x;
        return;
    }
    Dual<6> rg[3], xg[3], o[3];
#pragma unroll
    for(int i = 0; i < 3; i++) { rg[i] = Dual<6>::var(r[i], i); xg[i] = Dual<6>::var(x[i], 3 + i); }
    rotate_point_r_core(o, rg, xg, inverted);
#pragma unroll
    for(int i = 0; i < 3; i++)
    {
        out[i] = o[i].x;
#pragma unroll
        for(int k = 0; k < 3; k++) { Jr[3 * i + k] = o[i].j[k]; Jx[3 * i + k] = o[i].j[3 + k]; }
    }
}

// r01 = compose(r0, r1), compose_r_core() (poseutils-uses-autodiff.cc:279-607): Altmann's half-angle formulas, with
// the reference's branches for a tiny operand, and for a result near zero or near a half-turn
template <int N> __device__ __forceinline__ void compose_r_core(Dual<N> r[3], const Dual<N> r0[3], const Dual<N> r1[3])
{
    const Dual<N> A = dsqrt(r0[0] * r0[0] + r0[1] * r0[1] + r0[2] * r0[2]) / 2.;
    const Dual<N> B = dsqrt(r1[0] * r1[0] + r1[1] * r1[1] + r1[2] * r1[2]) / 2.;
    const Dual<N> inner = r0[0] * r1[0] + r0[1] * r1[1] + r0[2] * r1[2];
    const Dual<N> cross[3] = {r0[1] * r1[2] - r0[2] * r1[1], r0[2] * r1[0] - r0[0] * r1[2],
                              r0[0] * r1[1] - r0[1] * r1[0]};
    const double eps = 1e-8;
    if(A.x < eps / 2.)
    {
        if(B.x < eps)
        {
#pragma unroll
            for(int i = 0; i < 3; i++) r[i] = r0[i] + r1[i];
            return;
        }
        const Dual<N> BtB = B / dtan(B);
#pragma unroll
        for(int i = 0; i < 3; i++)
            r[i] = r1[i] * (Dual<N>(1.) - inner * (BtB - Dual<N>(1.)) / (B * B * 4.)) + r0[i] * BtB + cross[i] / 2.;
        return;
    }
    if(B.x < eps)
    {
        const Dual<N> AtA = A / dtan(A);
#pragma unroll
        for(int i = 0; i < 3; i++)
            r[i] = r0[i] * (Dual<N>(1.) - inner * (AtA - Dual<N>(1.)) / (A * A * 4.)) + r1[i] * AtA + cross[i] / 2.;
        return;
    }
    Dual<N> sA, cA, sB, cB;
    dsincos(A, sA, cA);
    dsincos(B, sB, cB);
    // sin(x)/x is taken as the constant 1 below 1e-5, as the reference's sinx_over_x() does
    const Dual<N> sAA = fabs(A.x) < 1e-5 ? Dual<N>(1.) : sA / A;
    const Dual<N> sBB = fabs(B.x) < 1e-5 ? Dual<N>(1.) : sB / B;
    const Dual<N> cosC = cA * cB - sAA * sBB * inner / 4.;
#pragma unroll
    for(int i = 0; i < 3; i++) r[i] = sAA * cB * r0[i] + sBB * cA * r1[i] + sAA * sBB * cross[i] / 2.;
    if(cosC.x - 1. > -eps * eps / 2.)
        return;   // C ~ 0: C/sin(C) = 1
    if(cosC.x + 1. < eps * eps / 2.)
    {
        // C ~ pi: the equivalent rotation of angle 2C - 2pi, (C - pi)/sin(C) ~ -1
#pragma unroll
        for(int i = 0; i < 3; i++) r[i] = r[i] * -1.;
        return;
    }
    const Dual<N> C = dacos(cosC);
    const Dual<N> sC = dsqrt(Dual<N>(1.) - cosC * cosC);
    const Dual<N> f = cosC.x < 0. ? (C - Dual<N>(M_PI)) / sC : C / sC;
#pragma unroll
    for(int i = 0; i < 3; i++) r[i] = r[i] * f;
}

// compose(r0, r1), r0 and r1 taken as -r0, -r1 where inverted; with dr0, dr1: the (3,3) gradients with respect to
// r0 and r1 as given
__device__ __forceinline__ void compose_r(double out[3], double* dr0, double* dr1, const double r0[3],
                                          const double r1[3], bool inverted0, bool inverted1)
{
    const double s0 = inverted0 ? -1. : 1., s1 = inverted1 ? -1. : 1.;
    if(dr0 == nullptr)
    {
        Dual<0> a[3], b[3], o[3];
#pragma unroll
        for(int i = 0; i < 3; i++) { a[i] = Dual<0>(r0[i] * s0); b[i] = Dual<0>(r1[i] * s1); }
        compose_r_core(o, a, b);
#pragma unroll
        for(int i = 0; i < 3; i++) out[i] = o[i].x;
        return;
    }
    Dual<6> a[3], b[3], o[3];
#pragma unroll
    for(int i = 0; i < 3; i++) { a[i] = Dual<6>::var(r0[i], i) * s0; b[i] = Dual<6>::var(r1[i], 3 + i) * s1; }
    compose_r_core(o, a, b);
#pragma unroll
    for(int i = 0; i < 3; i++)
    {
        out[i] = o[i].x;
#pragma unroll
        for(int k = 0; k < 3; k++) { dr0[3 * i + k] = o[i].j[k]; dr1[3 * i + k] = o[i].j[3 + k]; }
    }
}

// (internal linkage, as each translation unit compiles its own device code)
namespace {

// dr01/dr0 at r0 = 0 (poseutils.c:1003-1062): -r r' (B/tanB - 1)/(4 B^2) + (B/tanB) I - skew(r)/2, B = |r|/2
__device__ void compose_r_tinyr0_gradient(double Dr[9], const double r[3])
{
    const double n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    if(n2 < 2e-8 * 2e-8)
    {
        for(int i = 0; i < 9; i++) Dr[i] = (i % 4 == 0) ? 1. : 0.;
        return;
    }
    const double B = sqrt(n2) / 2., BtB = B / tan(B);
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++) Dr[3 * i + j] = -r[i] * r[j] * (BtB - 1.) / (4. * B * B) + (i == j ? BtB : 0.);
    Dr[1] += r[2] / 2.; Dr[2] -= r[1] / 2.;
    Dr[3] -= r[2] / 2.; Dr[5] += r[0] / 2.;
    Dr[6] += r[1] / 2.; Dr[7] -= r[0] / 2.;
}

}  // namespace

// dr01/dr1 at r1 = 0 (poseutils.c:1071-1137): the same with A = |r0|/2 and +skew(r0)/2
__device__ __forceinline__ void compose_r_tinyr1_gradient(double Dr[9], const double r[3])
{
    const double n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    if(n2 < 2e-8 * 2e-8)
    {
        for(int i = 0; i < 9; i++) Dr[i] = (i % 4 == 0) ? 1. : 0.;
        return;
    }
    const double A = sqrt(n2) / 2., AtA = A / tan(A);
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++) Dr[3 * i + j] = -r[i] * r[j] * (AtA - 1.) / (4. * A * A) + (i == j ? AtA : 0.);
    Dr[1] -= r[2] / 2.; Dr[2] += r[1] / 2.;
    Dr[3] += r[2] / 2.; Dr[5] -= r[0] / 2.;
    Dr[6] -= r[1] / 2.; Dr[7] += r[0] / 2.;
}

// R from r (mrcal_R_from_r_full, poseutils-opencv.c:42-155), with J[i][j][k] = dR_ij/dr_k. Below |r| = DBL_EPSILON
// the reference's exact branch: I and the constant gradient. Otherwise rodrigues(), whose series below |r| = 0.1 is
// accurate where the reference's closed form loses digits to cancellation
__host__ __device__ __forceinline__ void R_from_r(double R[9], double* J, const double r[3])
{
    const double n2 = r[0] * r[0] + r[1] * r[1] + r[2] * r[2];
    if(n2 < 2.220446049250313e-16 * 2.220446049250313e-16)
    {
        for(int i = 0; i < 9; i++) R[i] = (i % 4 == 0) ? 1. : 0.;
        if(J)
        {
            for(int i = 0; i < 27; i++) J[i] = 0.;
            J[9 * 1 + 3 * 2 + 0] = -1.; J[9 * 2 + 3 * 0 + 1] = -1.; J[9 * 0 + 3 * 1 + 2] = -1.;
            J[9 * 2 + 3 * 1 + 0] = 1.;  J[9 * 0 + 3 * 2 + 1] = 1.;  J[9 * 1 + 3 * 0 + 2] = 1.;
        }
        return;
    }
    if(J == nullptr)
    {
        rodrigues(R, nullptr, r);
        return;
    }
    double dR[27];   // [k][i][j]
    rodrigues(R, dR, r);
#pragma unroll
    for(int k = 0; k < 3; k++)
#pragma unroll
        for(int ij = 0; ij < 9; ij++) J[3 * ij + k] = dR[9 * k + ij];
}

// r from R (mrcal_r_from_R_full, poseutils.c:1140-1437): the axis from R - R', the angle from the trace, with the
// reference's small-angle branch and its branch near a half-turn. J[k][i][j] = dr_k/dR_ij: the pseudo-inverse of
// dR/dr at the result, the gradient within the manifold of rotations
__host__ __device__ __forceinline__ void r_from_R(double r[3], double* J, const double R[9])
{
    const double tr = R[0] + R[4] + R[8];
    const double u[3] = {R[7] - R[5], R[2] - R[6], R[3] - R[1]};
    const double costh = (tr - 1.) / 2.;
    const double eps = 1e-8;
    const double norm2u = u[0] * u[0] + u[1] * u[1] + u[2] * u[2];
    if(norm2u > 4. * eps * eps && 1. - fabs(costh) > eps * eps / 2.)
    {
        const double sinth = sqrt(norm2u) / 2;
        const double th = (sinth > sqrt(2.) / 2.) ? acos(costh) : (costh > 0 ? asin(sinth) : (M_PI - asin(sinth)));
        for(int i = 0; i < 3; i++) r[i] = u[i] / sqrt(norm2u) * th;
    }
    else if(costh > 0)
    {
        for(int i = 0; i < 3; i++) r[i] = u[i] / 2.;
    }
    else
    {
        // near a half-turn: |v_i| = sqrt((1 + R_ii)/2), the signs from the symmetric part
        double v[3];
        for(int i = 0; i < 3; i++)
        {
            r[i] = u[i] / -2.;
            const double vsq = (R[4 * i] + 1.) / 2.;
            v[i] = vsq > 0. ? sqrt(vsq) : 0.;
        }
        if(v[0] > 0.1)
        {
            if(R[1] + R[3] < 0) v[1] *= -1.;
            if(R[2] + R[6] < 0) v[2] *= -1.;
        }
        else if(v[1] > 0.1)
        {
            if(R[3] + R[1] < 0) v[0] *= -1.;
            if(R[5] + R[7] < 0) v[2] *= -1.;
        }
        else
        {
            if(R[6] + R[2] < 0) v[0] *= -1.;
            if(R[7] + R[5] < 0) v[1] *= -1.;
        }
        for(int i = 0; i < 3; i++) r[i] += v[i] * M_PI;
    }
    if(J == nullptr) return;

    // dr/dR = inv(D' D) D' with D = dR/dr (9,3) at r
    double Rr[9], D[27];   // D[ij][k]
    R_from_r(Rr, D, r);
    double M[6] = {};      // D'D, upper triangle: 00 01 02 11 12 22
    for(int ij = 0; ij < 9; ij++)
    {
        const double* d = &D[3 * ij];
        M[0] += d[0] * d[0]; M[1] += d[0] * d[1]; M[2] += d[0] * d[2];
        M[3] += d[1] * d[1]; M[4] += d[1] * d[2]; M[5] += d[2] * d[2];
    }
    // the inverse of the symmetric M from its cofactors
    const double c00 = M[3] * M[5] - M[4] * M[4], c01 = M[2] * M[4] - M[1] * M[5], c02 = M[1] * M[4] - M[2] * M[3];
    const double c11 = M[0] * M[5] - M[2] * M[2], c12 = M[1] * M[2] - M[0] * M[4], c22 = M[0] * M[3] - M[1] * M[1];
    const double inv_det = 1. / (M[0] * c00 + M[1] * c01 + M[2] * c02);
    const double Mi[9] = {c00, c01, c02, c01, c11, c12, c02, c12, c22};
    for(int ij = 0; ij < 9; ij++)
        for(int k = 0; k < 3; k++)
            J[9 * k + ij] = (Mi[3 * k] * D[3 * ij] + Mi[3 * k + 1] * D[3 * ij + 1] + Mi[3 * k + 2] * D[3 * ij + 2]) *
                            inv_det;
}

// element (i,j) of R or, if transposed, of R'
__host__ __device__ __forceinline__ double Rij(const double* R, bool transposed, int i, int j)
{
    return transposed ? R[3 * j + i] : R[3 * i + j];
}

__host__ __device__ __forceinline__ void invert_R(double out[9], const double R[9])
{
    for(int i = 0; i < 9; i++) out[i] = R[3 * (i % 3) + i / 3];
}

// (R', -R' t); out must not alias Rt
__host__ __device__ __forceinline__ void invert_Rt(double out[12], const double Rt[12])
{
    invert_R(out, Rt);
    for(int i = 0; i < 3; i++) out[9 + i] = -(out[3 * i] * Rt[9] + out[3 * i + 1] * Rt[10] + out[3 * i + 2] * Rt[11]);
}

// R x + t (mrcal_transform_point_Rt_full, poseutils.c:271-424, not inverted). out must not alias x
__host__ __device__ __forceinline__ void transform_point_Rt(double out[3], const double Rt[12], const double x[3])
{
    for(int i = 0; i < 3; i++) out[i] = Rt[3 * i] * x[0] + Rt[3 * i + 1] * x[1] + Rt[3 * i + 2] * x[2] + Rt[9 + i];
}

// x -> Rt0(Rt1(x)), Rt0 and Rt1 taken inverted where asked: the four cases of mrcal_compose_Rt_full
// (poseutils.c:603-738). out must not alias Rt0 or Rt1
__host__ __device__ __forceinline__ void compose_Rt(double out[12], const double Rt0[12], const double Rt1[12],
                                                    bool inverted0, bool inverted1)
{
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++)
            out[3 * i + j] = Rij(Rt0, inverted0, i, 0) * Rij(Rt1, inverted1, 0, j) +
                             Rij(Rt0, inverted0, i, 1) * Rij(Rt1, inverted1, 1, j) +
                             Rij(Rt0, inverted0, i, 2) * Rij(Rt1, inverted1, 2, j);
    const double* t0 = &Rt0[9];
    const double* t1 = &Rt1[9];
    for(int i = 0; i < 3; i++)
    {
        if(!inverted0 && !inverted1)
            out[9 + i] = Rt0[3 * i] * t1[0] + Rt0[3 * i + 1] * t1[1] + Rt0[3 * i + 2] * t1[2] + t0[i];
        else if(inverted0 && !inverted1)
            out[9 + i] = Rt0[i] * (t1[0] - t0[0]) + Rt0[3 + i] * (t1[1] - t0[1]) + Rt0[6 + i] * (t1[2] - t0[2]);
        else
        {
            const double Rt = out[3 * i] * t1[0] + out[3 * i + 1] * t1[1] + out[3 * i + 2] * t1[2];
            out[9 + i] = inverted0 ? -Rt - (Rt0[i] * t0[0] + Rt0[3 + i] * t0[1] + Rt0[6 + i] * t0[2]) : -Rt + t0[i];
        }
    }
}

__device__ __forceinline__ void skew_symmetric(double S[9], const double a[3])
{
    S[0] = 0.;    S[1] = -a[2]; S[2] = a[1];
    S[3] = a[2];  S[4] = 0.;    S[5] = -a[0];
    S[6] = -a[1]; S[7] = a[0];  S[8] = 0.;
}

// R from the unit quaternion q = (w, x, y, z) (R_from_quat, poseutils-genpywrap.py)
__device__ __forceinline__ void R_from_quat(double R[9], const double q[4])
{
    const double w = q[0], i = q[1], j = q[2], k = q[3];
    R[0] = 1. - 2. * (j * j + k * k); R[1] = 2. * (i * j - k * w);      R[2] = 2. * (i * k + j * w);
    R[3] = 2. * (i * j + k * w);      R[4] = 1. - 2. * (i * i + k * k); R[5] = 2. * (j * k - i * w);
    R[6] = 2. * (i * k - j * w);      R[7] = 2. * (j * k + i * w);      R[8] = 1. - 2. * (i * i + j * j);
}

// the unit quaternion (w, x, y, z) of R (quat_from_R, mrcal/_poseutils_scipy.py): the largest of the diagonal and the
// trace picks the formula, the first one on a tie; the sign is not normalized
__device__ __forceinline__ void quat_from_R(double q[4], const double R[9])
{
    const double tr = R[0] + R[4] + R[8];
    int choice = 0;
    double best = R[0];
    if(R[4] > best) { choice = 1; best = R[4]; }
    if(R[8] > best) { choice = 2; best = R[8]; }
    if(tr > best) choice = 3;
    if(choice != 3)
    {
        const int i = choice, j = (i + 1) % 3, k = (j + 1) % 3;
        q[i + 1] = 1. - tr + 2. * R[4 * i];
        q[j + 1] = R[3 * j + i] + R[3 * i + j];
        q[k + 1] = R[3 * k + i] + R[3 * i + k];
        q[0] = R[3 * k + j] - R[3 * j + k];
    }
    else
    {
        q[1] = R[7] - R[5];
        q[2] = R[2] - R[6];
        q[3] = R[3] - R[1];
        q[0] = 1. + tr;
    }
    const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    for(int i = 0; i < 4; i++) q[i] /= n;
}

// a rotation whose z axis is v (mrcal_R_aligned_to_vector, poseutils.c:1650-1695): rows x, y, z of R
__device__ __forceinline__ void R_aligned_to_vector(double R[9], const double v[3])
{
    const double magv = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    double* x = &R[0];
    double* y = &R[3];
    double* z = &R[6];
    for(int i = 0; i < 3; i++) { x[i] = 0.; z[i] = v[i] / magv; }
    double inner_x_z;
    if(fabs(z[0]) < .9) { x[0] = 1.; inner_x_z = z[0]; }
    else                { x[1] = 1.; inner_x_z = z[1]; }
    for(int i = 0; i < 3; i++) x[i] -= inner_x_z * z[i];
    const double magx = sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2]);
    for(int i = 0; i < 3; i++) x[i] /= magx;
    y[0] = z[1] * x[2] - z[2] * x[1];
    y[1] = z[2] * x[0] - z[0] * x[2];
    y[2] = z[0] * x[1] - z[1] * x[0];
}

}  // namespace mb200
