// projection_diff(): the comparison of camera models, as mrcal.projection_diff() and
// mrcal.implied_Rt10__from_unprojections() compute it (mrcal/model_analysis.py:27-395, 1520-1928).
//
// The fit of the transformation the two sets of intrinsics imply is one CTA per pair of models, all pairs in one launch.
// It minimizes the reference's objective, sum over kept points of huber((w th2)^2) with th2 = 2 (1 - cos(angle between
// the transformed p0 and v1)) and the huber threshold C = (5 deg)^2 (scipy's loss='huber', f_scale=C), from zero
// parameters, by damped robust Gauss-Newton, accepting a step only if the robust cost decreases. The whole
// iteration stays on the device. Every per-iteration sum runs in a fixed order without atomics (a fixed stride of
// points per thread, warp shuffles, then the warps in index order), so two calls give bit-identical results.
//
// The gradient is exact: sum rho'(f^2) f J. The curvature model keeps the term plain Gauss-Newton drops. th2 is a
// squared angle, th2 ~ |e|^2 for the angular error e, so f d2f is as large as J'J and, unlike J'J (rank one per point,
// along e), it spans every direction: without it the fit crawls wherever the errors share a direction, as the
// systematic differences between two lens models do. Per point the model is
//   (rho' + 2 rho'' s) J'J + rho' f w 2 D'(I - v v')D,   D = d(a/|a|)/dparams,
// the second term the curvature of th2 with the second derivative of the rotation left out (exact at a = v). Below
// huber's threshold the first weight is 1, beyond it 0, as in scipy's robust least squares. Near a perfect fit the
// model is Newton's on a quartic, which still converges only linearly: the iteration limit is generous. 2 (1 - cos)
// resolves angles only down to ~1e-8 rad in fp64, so below that the cost is rounding noise: steps stop
// decreasing it, are rejected, and the damping grows past its cap. A gradient that is exactly zero (a model diffed with
// itself at infinity) stops the fit at once, at the exact identity.
#include <cuda_runtime.h>

#include "common.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "problem_impl.h"
#include "reduce.cuh"

namespace mb200 {
namespace {

constexpr int kFitThreads = 256;
constexpr int kFitWarps = kFitThreads / 32;
constexpr int kFitMaxPasses = 1000;
constexpr double kHuberC = (5. * M_PI / 180.) * (5. * M_PI / 180.);
constexpr double kLambda0 = 1e-6, kLambdaMin = 1e-12, kLambdaMax = 1e16;
constexpr double kFlatCost = 1e-14;   // an accepted step, damped by at most kLambda0, that lowers the cost by less than
                                      // this, relative, ends the fit

enum { FIT_OK = 0, FIT_TOO_FEW_POINTS = 1 };

// One fit's inputs. Point (m, i): p0 = p0[m][i], or p0[i] * dist[m] if dist is given; v1[i]; weight w[m][i] (1 if w is
// NULL). Kept if |q0[i] - center|^2 < r2 and p0, v1 and the weight are finite.
struct FitArgs
{
    const double* q0;   // [N][2]
    const double* p0;   // + fit * p0_stride
    const double* dist; // [M] or NULL
    const double* v1;   // + fit * v1_stride
    const double* w;    // + fit * w_stride, or NULL
    size_t p0_stride, v1_stride, w_stride;
    int N, M;
    double cx, cy, r2;
    double* Rt10;       // [Nfits][4][3]
    int* status;        // [Nfits]
};

__device__ __forceinline__ bool finite3(const double* a) { return isfinite(a[0]) && isfinite(a[1]) && isfinite(a[2]); }

// without contraction into FMAs: u = dR_k p and v.u come out exactly 0 at r = 0 when p == v, so diffing a model with
// itself at infinity has an exactly zero gradient
__device__ __forceinline__ double dot3_rn(const double* a, const double* b)
{
    return __dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]));
}

__device__ __forceinline__ bool kept(const FitArgs& A, int i)
{
    const double dx = A.q0[2 * i] - A.cx, dy = A.q0[2 * i + 1] - A.cy;
    return __dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)) < A.r2;   // as numpy evaluates it
}

// the weighted residual f = w th2, its gradient J over (r, t) and the columns U of d(a/|a|)/d(r, t)
template <int NP>
__device__ __forceinline__ void residual(double* f, double J[NP], double U[NP][3], const double* p, const double* v,
                                         double w, const double* R, const double* dR, const double* t)
{
    double a[3], u[3][3];
    mat3_vec(a, R, p);
#pragma unroll
    for(int k = 0; k < 3; k++)
    {
        const double* D = dR + 9 * k;
        u[k][0] = dot3_rn(D, p); u[k][1] = dot3_rn(D + 3, p); u[k][2] = dot3_rn(D + 6, p);
    }
    if constexpr(NP == 3)
    {
        // |a| = 1: the reference divides by nothing
        *f = w * (2. * (1. - (a[0] * v[0] + a[1] * v[1] + a[2] * v[2])));
#pragma unroll
        for(int k = 0; k < 3; k++)
        {
            J[k] = -2. * w * dot3_rn(v, u[k]);
            U[k][0] = u[k][0]; U[k][1] = u[k][1]; U[k][2] = u[k][2];
        }
    }
    else
    {
        a[0] += t[0]; a[1] += t[1]; a[2] += t[2];
        const double mag = sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]);
        const double inner = a[0] * v[0] + a[1] * v[1] + a[2] * v[2];
        *f = w * (2. * (1. - inner / mag));
        // dth2/da = -2 (v - inner a / |a|^2) / |a|
        const double s = -2. * w / mag, c = inner / (mag * mag);
        const double g[3] = {s * (v[0] - c * a[0]), s * (v[1] - c * a[1]), s * (v[2] - c * a[2])};
#pragma unroll
        for(int k = 0; k < 3; k++) { J[k] = dot3_rn(g, u[k]); J[3 + k] = g[k]; }
        // d(a/|a|)/dx = (I - a a'/|a|^2) da/dx / |a|; da/dt = I
        const double im = 1. / mag;
#pragma unroll
        for(int c = 0; c < 6; c++)
        {
            double d[3] = {0., 0., 0.};
            if(c < 3) { d[0] = u[c][0]; d[1] = u[c][1]; d[2] = u[c][2]; }
            else d[c - 3] = 1.;
            const double ad = (a[0] * d[0] + a[1] * d[1] + a[2] * d[2]) * im * im;
            U[c][0] = (d[0] - ad * a[0]) * im; U[c][1] = (d[1] - ad * a[1]) * im; U[c][2] = (d[2] - ad * a[2]) * im;
        }
    }
}

// Block-wide sum of NS per-thread values in a fixed order: warp_sum(), then thread 0 adds the other warps' sums to its
// own in warp order, ((w0 + w1) + w2) + ... (no zero in front: block_sum_by_warps() would add a +0 first, and thread 0
// needs all NS sums). The result is valid in thread 0 only
template <int NS>
__device__ __forceinline__ void block_sum(double (&acc)[NS], double (*red)[NS])
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    warp_sum(acc);
    if(lane == 0)
#pragma unroll
        for(int j = 0; j < NS; j++) red[warp][j] = acc[j];
    __syncthreads();
    if(threadIdx.x == 0)
        for(int w = 1; w < kFitWarps; w++)
#pragma unroll
            for(int j = 0; j < NS; j++) acc[j] += red[w][j];
}

// In place: A (NP x NP, row-major) -> its Cholesky factor L, then x = -A^-1 g. False if A is not positive definite
template <int NP>
__device__ __forceinline__ bool chol_solve_neg(double* __restrict__ A, const double* __restrict__ g, double* __restrict__ x)
{
    for(int j = 0; j < NP; j++)
    {
        double d = A[j * NP + j];
        for(int k = 0; k < j; k++) d -= A[j * NP + k] * A[j * NP + k];
        if(!(d > 0.) || !isfinite(d)) return false;
        d = sqrt(d);
        A[j * NP + j] = d;
        for(int i = j + 1; i < NP; i++)
        {
            double s = A[i * NP + j];
            for(int k = 0; k < j; k++) s -= A[i * NP + k] * A[j * NP + k];
            A[i * NP + j] = s / d;
        }
    }
    for(int i = 0; i < NP; i++)
    {
        double s = -g[i];
        for(int k = 0; k < i; k++) s -= A[i * NP + k] * x[k];
        x[i] = s / A[i * NP + i];
    }
    for(int i = NP - 1; i >= 0; i--)
    {
        double s = x[i];
        for(int k = i + 1; k < NP; k++) s -= A[k * NP + i] * x[k];
        x[i] = s / A[i * NP + i];
    }
    return true;
}

// One CTA per fit (blockIdx.x). NP = 3: rotation only (at infinity); NP = 6: rotation and translation
template <int NP>
__global__ void __launch_bounds__(kFitThreads) implied_fit_kernel(FitArgs A)
{
    constexpr int NH = NP * (NP + 1) / 2, NS = 1 + NP + NH;   // cost, gradient, upper triangle of J'J
    __shared__ double red[kFitWarps][NS];
    __shared__ double R[9], dR[27], t[3];
    // thread 0's iteration state: the parameters, the sums at them, the step being tried, the damped system
    __shared__ double x[NP], cur[NS], step[NP], xt[NP], H[NP * NP];
    __shared__ int s_done, s_count[1][kFitWarps];
    const int fit = blockIdx.x, tid = threadIdx.x;
    const double* p0 = A.p0 + fit * A.p0_stride;
    const double* v1 = A.v1 + fit * A.v1_stride;
    const double* wt = A.w ? A.w + fit * A.w_stride : nullptr;

    // the focus region must hold at least 3 points (model_analysis.py:213-217)
    int count = 0;
    for(int i = tid; i < A.N; i += kFitThreads) count += kept(A, i);
    int v[1] = {count};
    const int total = block_sum_by_warps(v, s_count);
    if(tid == 0)
    {
        A.status[fit] = total < 3 ? FIT_TOO_FEW_POINTS : FIT_OK;
        s_done = total < 3;
    }
    __syncthreads();
    if(s_done) return;

    double lambda = kLambda0;
    int pass = 0;
    if(tid == 0)
    {
        for(int a = 0; a < NP; a++) x[a] = 0.;
        rodrigues(R, dR, x);
        t[0] = t[1] = t[2] = 0.;
    }
    __syncthreads();
    for(;;)
    {
        // evaluate at the parameters in R, dR, t
        double acc[NS];
#pragma unroll
        for(int j = 0; j < NS; j++) acc[j] = 0.;
        for(int m = 0; m < A.M; m++)
        for(int i = tid; i < A.N; i += kFitThreads)
        {
            const size_t j = (size_t)m * A.N + i;
            if(!kept(A, i)) continue;
            double p[3], v[3];
            if(A.dist)
            {
                const double d = A.dist[m];
                p[0] = p0[3 * i] * d; p[1] = p0[3 * i + 1] * d; p[2] = p0[3 * i + 2] * d;
            }
            else { p[0] = p0[3 * j]; p[1] = p0[3 * j + 1]; p[2] = p0[3 * j + 2]; }
            v[0] = v1[3 * i]; v[1] = v1[3 * i + 1]; v[2] = v1[3 * i + 2];
            const double w = wt ? wt[j] : 1.;
            if(!finite3(p) || !finite3(v) || !isfinite(w)) continue;
            double f, J[NP], U[NP][3];
            residual<NP>(&f, J, U, p, v, w, R, dR, t);
            // huber: rho(s) = s below C^2, 2 C sqrt(s) - C^2 above
            const double af = fabs(f);
            const bool quad = af <= kHuberC;
            const double rho = quad ? f * f : 2. * kHuberC * af - kHuberC * kHuberC;
            const double rp = quad ? 1. : kHuberC / af, hw = quad ? 1. : 0., kw = 2. * rp * f * w;
            double vU[NP];
#pragma unroll
            for(int a = 0; a < NP; a++) vU[a] = v[0] * U[a][0] + v[1] * U[a][1] + v[2] * U[a][2];
            acc[0] += rho;
            int h = 1 + NP;
#pragma unroll
            for(int a = 0; a < NP; a++)
            {
                acc[1 + a] += rp * f * J[a];
#pragma unroll
                for(int b = a; b < NP; b++)
                    acc[h++] += hw * J[a] * J[b] +
                                kw * (U[a][0] * U[b][0] + U[a][1] * U[b][1] + U[a][2] * U[b][2] - vU[a] * vU[b]);
            }
        }
        block_sum<NS>(acc, red);

        if(tid == 0)
        {
            bool done = false;
            if(pass == 0)
                for(int j = 0; j < NS; j++) cur[j] = acc[j];
            else if(acc[0] < cur[0])
            {
                // only an undamped step says the cost is flat: a heavily damped one is short by design
                const bool flat = cur[0] - acc[0] <= kFlatCost * cur[0] && lambda <= kLambda0;
                for(int a = 0; a < NP; a++) x[a] = xt[a];
                for(int j = 0; j < NS; j++) cur[j] = acc[j];
                lambda = fmax(lambda * 0.1, kLambdaMin);
                done = flat;
            }
            else lambda *= 10.;
            pass++;
            bool zero_gradient = true;
            for(int a = 0; a < NP; a++) zero_gradient = zero_gradient && cur[1 + a] == 0.;
            done = done || zero_gradient || pass >= kFitMaxPasses || lambda > kLambdaMax;
            // the next trial: (H + lambda diag(H)) step = -g
            while(!done)
            {
                int h = 1 + NP;
                for(int a = 0; a < NP; a++)
                    for(int b = a; b < NP; b++, h++) H[a * NP + b] = H[b * NP + a] = cur[h];
                for(int a = 0; a < NP; a++)
                {
                    const double d = H[a * NP + a];
                    H[a * NP + a] += lambda * (d > 0. ? d : 1.);
                }
                if(chol_solve_neg<NP>(H, cur + 1, step)) break;
                lambda *= 10.;
                done = lambda > kLambdaMax;
            }
            for(int a = 0; a < NP; a++) xt[a] = done ? x[a] : x[a] + step[a];
            rodrigues(R, dR, xt);
            if constexpr(NP == 6) { t[0] = xt[3]; t[1] = xt[4]; t[2] = xt[5]; }
            s_done = done;
            if(done)
            {
                double* out = A.Rt10 + 12 * fit;
                for(int k = 0; k < 9; k++) out[k] = R[k];
                for(int k = 0; k < 3; k++) out[9 + k] = NP == 6 ? xt[3 + k] : 0.;
            }
        }
        __syncthreads();
        if(s_done) return;
    }
}

// (1/(u_0 u_k))^2 for pair k = 1..Nmodels-1 (model_analysis.py:1821-1829); non-finite values are cleaned up by the fit
__global__ void diff_weights_kernel(const double* __restrict__ U, int Nmodels, long NdN, double* __restrict__ w)
{
    const long j = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if(j >= NdN) return;
    const double u0 = U[j];
    for(int k = 1; k < Nmodels; k++)
    {
        double x = 1. / (u0 * U[k * NdN + j]);
        w[(k - 1) * NdN + j] = x * x;
    }
}

// q1 = project_k(R (v0 d) + t) for every (distance, grid point). Two models: diff = q1 - q0 and |diff|. More: |diff|^2
// into this model's slice of the scratch
template <int KIND>
__global__ void reproject_diff_kernel(LensArgs a, const double* __restrict__ Rt, const double* __restrict__ q0,
                                      const double* __restrict__ v0, const double* __restrict__ dist, int N, int Nd,
                                      double* __restrict__ diff, double* __restrict__ difflen, double* __restrict__ norm2)
{
    const long j = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if(j >= (long)Nd * N) return;
    const int m = (int)(j / N), i = (int)(j - (long)m * N);
    const double d = dist ? dist[m] : 1.;
    const double p[3] = {v0[3 * i] * d, v0[3 * i + 1] * d, v0[3 * i + 2] * d};
    double pc[3], q[2], g[2][3];
    mat3_vec(pc, Rt, p);
    pc[0] += Rt[9]; pc[1] += Rt[10]; pc[2] += Rt[11];
    project_any<KIND>(q, g, pc, a);
    const double dx = q[0] - q0[2 * i], dy = q[1] - q0[2 * i + 1];
    const double n2 = dx * dx + dy * dy;
    if(norm2) norm2[j] = n2;
    else
    {
        diff[2 * j] = dx; diff[2 * j + 1] = dy;
        difflen[j] = sqrt(n2);
    }
}

// sqrt(mean_k |q_k - q0|^2), summed in model order
__global__ void diff_stdev_kernel(const double* __restrict__ norm2, int K, long NdN, double* __restrict__ difflen)
{
    const long j = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if(j >= NdN) return;
    double s = 0.;
    for(int k = 0; k < K; k++) s += norm2[k * NdN + j];
    difflen[j] = sqrt(s / K);
}

bool have_device()
{
    if(mrcal_b200_device_count() > 0) return true;
    set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback");
    return false;
}

template <typename T>
bool upload(DeviceArena& mem, T** d, const T* h, size_t n, cudaStream_t s)
{
    if(!mem.alloc(d, n)) return false;
    MB200_CUDA_CHECK(cudaMemcpyAsync(*d, h, n * sizeof(T), cudaMemcpyHostToDevice, s));
    return true;
}

void launch_fit(const FitArgs& A, int Nfits, bool atinfinity, cudaStream_t s)
{
    if(atinfinity) implied_fit_kernel<3><<<Nfits, kFitThreads, 0, s>>>(A);
    else           implied_fit_kernel<6><<<Nfits, kFitThreads, 0, s>>>(A);
}

bool fit_status(const std::vector<int>& status)
{
    for(int st : status)
        if(st == FIT_TOO_FEW_POINTS) { set_error("Focus region contained too few points"); return false; }
    return true;
}

struct Stream
{
    cudaStream_t s = nullptr;
    ~Stream() { if(s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); } }
};

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_implied_Rt10__from_unprojections(double* Rt10, const mrcal_point2_t* q0, int N,
                                                            const mrcal_point3_t* p0, int M, const mrcal_point3_t* v1,
                                                            const double* weights, bool atinfinity,
                                                            const double* focus_center, double focus_radius)
{
    if(!have_device()) return false;
    if(N < 0 || M < 1) { set_error("implied_Rt10__from_unprojections: need N >= 0 and M >= 1"); return false; }
    DeviceArena mem;   // freed after the stream has drained
    Stream S;
    MB200_CUDA_CHECK(cudaStreamCreateWithFlags(&S.s, cudaStreamNonBlocking));
    FitArgs A{};
    double *d_q0, *d_p0, *d_v1, *d_w = nullptr, *d_Rt;
    int* d_status;
    const size_t MN = (size_t)M * N;
    if(!upload(mem, &d_q0, (const double*)q0, 2 * (size_t)N, S.s) || !upload(mem, &d_p0, (const double*)p0, 3 * MN, S.s) ||
       !upload(mem, &d_v1, (const double*)v1, 3 * (size_t)N, S.s) || (weights && !upload(mem, &d_w, weights, MN, S.s)) ||
       !mem.alloc(&d_Rt, 12) || !mem.alloc(&d_status, 1))
        return false;
    A.q0 = d_q0; A.p0 = d_p0; A.v1 = d_v1; A.w = d_w;
    A.N = N; A.M = M;
    A.cx = focus_center[0]; A.cy = focus_center[1]; A.r2 = focus_radius * focus_radius;
    A.Rt10 = d_Rt; A.status = d_status;
    launch_fit(A, 1, atinfinity, S.s);
    MB200_CUDA_CHECK(cudaGetLastError());
    std::vector<int> status(1);
    MB200_CUDA_CHECK(cudaMemcpyAsync(Rt10, d_Rt, 12 * sizeof(double), cudaMemcpyDeviceToHost, S.s));
    MB200_CUDA_CHECK(cudaMemcpyAsync(status.data(), d_status, sizeof(int), cudaMemcpyDeviceToHost, S.s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(S.s));
    return fit_status(status);
}

extern "C" bool mrcal_b200_projection_diff(double* Rt10, double* difflen, double* diff,
                                           const mrcal_point2_t* q0, int N, const mrcal_point3_t* v, int Nmodels,
                                           const double* distance, int Nd,
                                           const mrcal_lensmodel_t* lensmodels, const double* intrinsics,
                                           const double* uncertainties, const double* focus_center, double focus_radius,
                                           bool fit_Rt10)
{
    if(!have_device()) return false;
    if(Nmodels < 2) { set_error("At least 2 models are required to compute the diff"); return false; }
    if(N < 0 || Nd < 1 || (distance == nullptr && Nd != 1))
    {
        set_error("projection_diff: need N >= 0, and Nd >= 1 (Nd == 1 at infinity)");
        return false;
    }
    std::vector<int> kinds(Nmodels), Nintr(Nmodels);
    std::vector<LensArgs> lens(Nmodels);
    size_t Nintr_all = 0;
    for(int k = 0; k < Nmodels; k++)
    {
        kinds[k] = lens_kind_of(&lensmodels[k]);
        if(kinds[k] < 0) { set_error("this lens model has no CUDA implementation"); return false; }
        if(!lens_args_setup(&lens[k], kinds[k], &lensmodels[k])) return false;
        Nintr[k] = mrcal_lensmodel_num_params(&lensmodels[k]);
        Nintr_all += Nintr[k];
    }
    const int Npairs = Nmodels - 1;
    const long NdN = (long)Nd * N;
    DeviceArena mem;   // freed after the stream has drained
    Stream S;
    MB200_CUDA_CHECK(cudaStreamCreateWithFlags(&S.s, cudaStreamNonBlocking));
    double *d_q0, *d_v, *d_dist = nullptr, *d_intr, *d_U = nullptr, *d_w = nullptr, *d_Rt, *d_diff = nullptr, *d_len,
           *d_n2 = nullptr;
    int* d_status = nullptr;
    if(!upload(mem, &d_q0, (const double*)q0, 2 * (size_t)N, S.s) ||
       !upload(mem, &d_v, (const double*)v, 3 * (size_t)Nmodels * N, S.s) ||
       (distance && !upload(mem, &d_dist, distance, (size_t)Nd, S.s)) ||
       !upload(mem, &d_intr, intrinsics, Nintr_all, S.s) || !mem.alloc(&d_Rt, 12 * (size_t)Npairs) ||
       !mem.alloc(&d_len, (size_t)NdN))
        return false;
    if(Nmodels == 2) { if(!mem.alloc(&d_diff, 2 * (size_t)NdN)) return false; }
    else if(!mem.alloc(&d_n2, (size_t)Npairs * NdN)) return false;
    std::vector<int> status;
    if(fit_Rt10)
    {
        if(!mem.alloc(&d_status, (size_t)Npairs)) return false;
        if(uncertainties)
        {
            if(!upload(mem, &d_U, uncertainties, (size_t)Nmodels * NdN, S.s) || !mem.alloc(&d_w, (size_t)Npairs * NdN))
                return false;
            if(NdN > 0) diff_weights_kernel<<<(unsigned)((NdN + 255) / 256), 256, 0, S.s>>>(d_U, Nmodels, NdN, d_w);
        }
        FitArgs A{};
        A.q0 = d_q0; A.p0 = d_v; A.dist = d_dist; A.v1 = d_v + 3 * (size_t)N; A.w = d_w;
        A.p0_stride = 0; A.v1_stride = 3 * (size_t)N; A.w_stride = (size_t)NdN;
        A.N = N; A.M = Nd;
        A.cx = focus_center[0]; A.cy = focus_center[1]; A.r2 = focus_radius * focus_radius;
        A.Rt10 = d_Rt; A.status = d_status;
        launch_fit(A, Npairs, distance == nullptr, S.s);
        status.resize(Npairs);
    }
    else MB200_CUDA_CHECK(cudaMemcpyAsync(d_Rt, Rt10, 12 * (size_t)Npairs * sizeof(double), cudaMemcpyHostToDevice, S.s));
    if(NdN > 0)
    {
        const unsigned blocks = (unsigned)((NdN + 127) / 128);
        const double* intr = d_intr + Nintr[0];
        for(int k = 1; k < Nmodels; k++)
        {
            LensArgs a = lens[k];
            a.intr = intr;
            intr += Nintr[k];
            const double* Rt = d_Rt + 12 * (k - 1);
            double* n2 = d_n2 ? d_n2 + (k - 1) * NdN : nullptr;
            if(!dispatch_lens_kind(kinds[k], [&](auto kk)
               {
                   reproject_diff_kernel<decltype(kk)::value><<<blocks, 128, 0, S.s>>>(a, Rt, d_q0, d_v, d_dist, N, Nd,
                                                                                     d_diff, d_len, n2);
               }))
                return false;
        }
        if(d_n2) diff_stdev_kernel<<<(unsigned)((NdN + 255) / 256), 256, 0, S.s>>>(d_n2, Npairs, NdN, d_len);
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    if(fit_Rt10)
    {
        MB200_CUDA_CHECK(cudaMemcpyAsync(Rt10, d_Rt, 12 * (size_t)Npairs * sizeof(double), cudaMemcpyDeviceToHost, S.s));
        MB200_CUDA_CHECK(cudaMemcpyAsync(status.data(), d_status, Npairs * sizeof(int), cudaMemcpyDeviceToHost, S.s));
    }
    MB200_CUDA_CHECK(cudaMemcpyAsync(difflen, d_len, NdN * sizeof(double), cudaMemcpyDeviceToHost, S.s));
    if(diff && d_diff) MB200_CUDA_CHECK(cudaMemcpyAsync(diff, d_diff, 2 * NdN * sizeof(double), cudaMemcpyDeviceToHost, S.s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(S.s));
    return fit_status(status);
}
