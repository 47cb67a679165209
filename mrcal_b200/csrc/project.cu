// mrcal_project() / mrcal_unproject(): the reference's point-wise entry points
// (mrcal.h:165-224, mrcal.c:2866-3080 and :3082-3270), host buffers in and out,
// one thread per point on the device. They use the same lens-model device functions
// as the residual kernels (device_math.cuh); the unprojection is unproject.cuh's. With them, the unprojection with
// gradients (mrcal/projections.py:112-397) and model_resolution__deg_pixel() (mrcal/model_analysis.py:2152-2246).
#include <cuda_runtime.h>

#include "common.h"
#include "device_call.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "unproject.cuh"

namespace mb200 {
namespace {

// dq_di: dense (N,2,Nintr), zeroed by the caller, or NULL; IntrinsicsGradient::scatter() fills its nonzero entries
template <int KIND>
__global__ void project_kernel(LensArgs a, const double* __restrict__ p, int N, double* __restrict__ q, double* __restrict__ dq_dp,
                               double* __restrict__ dq_di, int Nintr)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= N) return;
    double qq[2], g[2][3];
    const double pp[3] = {p[3 * i], p[3 * i + 1], p[3 * i + 2]};
    if(dq_di == nullptr) project_any<KIND>(qq, g, pp, a);
    else
    {
        IntrinsicsGradient<KIND> G;
        G.project(g, pp, a);
        qq[0] = G.q[0]; qq[1] = G.q[1];
        double* out = dq_di + (size_t)i * 2 * Nintr;
        G.scatter(a, [&](int k, int col, double val) { out[k * Nintr + col] = val; });
    }
    q[2 * i] = qq[0]; q[2 * i + 1] = qq[1];
    if(dq_dp)
        for(int r = 0; r < 2; r++)
            for(int c = 0; c < 3; c++) dq_dp[6 * i + 3 * r + c] = g[r][c];
}

// The resolution of the model at each pixel, as mrcal.model_resolution__deg_pixel() computes it
// (mrcal/model_analysis.py:2152-2246), fused: the unit ray v, dq/dv there, M = dq/dv [u0 u1] for an orthonormal basis
// of the plane perpendicular to v, and the eigenvalues of M'M in closed form. Those do not depend on the basis, so any
// basis does: u0 is perpendicular to v and to the axis least aligned with it, u1 = v x u0. mode: MB200_RESOLUTION_*
template <int KIND>
__global__ void resolution_kernel(LensArgs a, const double* __restrict__ q, int N, double* __restrict__ out, int mode,
                                  bool behind_ok)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= N) return;
    double v[3], qq[2], g[2][3];
    unproject_any<KIND>(v, q[2 * i], q[2 * i + 1], a, behind_ok);
    normalize_or_zero<KIND>(v);
    project_any<KIND>(qq, g, v, a);
    const double ax[3] = {fabs(v[0]), fabs(v[1]), fabs(v[2])};
    const int e = ax[0] <= ax[1] && ax[0] <= ax[2] ? 0 : (ax[1] <= ax[2] ? 1 : 2);
    // u0 = e x v / |e x v|
    double u0[3] = {0., 0., 0.};
    u0[(e + 1) % 3] = -v[(e + 2) % 3];
    u0[(e + 2) % 3] = v[(e + 1) % 3];
    const double n0 = 1. / sqrt(u0[0] * u0[0] + u0[1] * u0[1] + u0[2] * u0[2]);
    for(int k = 0; k < 3; k++) u0[k] *= n0;
    const double u1[3] = {v[1] * u0[2] - v[2] * u0[1], v[2] * u0[0] - v[0] * u0[2], v[0] * u0[1] - v[1] * u0[0]};
    double M[2][2];
    for(int r = 0; r < 2; r++)
    {
        M[r][0] = g[r][0] * u0[0] + g[r][1] * u0[1] + g[r][2] * u0[2];
        M[r][1] = g[r][0] * u1[0] + g[r][1] * u1[1] + g[r][2] * u1[2];
    }
    const double A = M[0][0] * M[0][0] + M[1][0] * M[1][0];
    const double B = M[0][0] * M[0][1] + M[1][0] * M[1][1];
    const double C = M[0][1] * M[0][1] + M[1][1] * M[1][1];
    const double sd = sqrt((A - C) * (A - C) / 4. + B * B);
    const double lmax = (A + C) / 2. + sd;
    double lmin = (A + C) / 2. - sd;
    if(lmin < 1e-6) lmin = 1e-6;   // roundoff, as the reference
    // the reciprocals swap min and max
    const double rmax = 1. / sqrt(lmin) * 180. / M_PI, rmin = 1. / sqrt(lmax) * 180. / M_PI;
    out[i] = mode == MB200_RESOLUTION_MIN ? rmin : mode == MB200_RESOLUTION_MAX ? rmax :
             mode == MB200_RESOLUTION_ECCENTRICITY ? rmax / rmin : (rmin + rmax) / 2.;
}

enum Call { PROJECT, UNPROJECT, RESOLUTION };

// PROJECT: p [N][3] -> q [N][2], dq_dp [N][2][3], dq_di [N][2][Nintr]. UNPROJECT: q [N][2] -> v [N][3], dv_dq
// [N][3][2], dv_di [N][3][Nintr], normalized if opt. RESOLUTION: q [N][2] -> [N] in mode opt. The gradients may be NULL
bool run(Call call, double* out, double* grad, double* gi, const double* in, int N, const mrcal_lensmodel_t* lensmodel,
         const double* intrinsics, int opt = 0)
{
    DeviceCall D;
    HostLens L;
    if(!D.start() || !lens_setup(&L, lensmodel)) return false;
    if(N <= 0) return true;
    if(call != PROJECT && !central_projection(L, intrinsics)) return false;
    const int Nintr = L.Nintr;
    const size_t nin = (size_t)N * (call == PROJECT ? 3 : 2), nout = (size_t)N * (call == PROJECT ? 2 : call == UNPROJECT ? 3 : 1);
    const size_t ngi = (size_t)N * (call == PROJECT ? 2 : 3) * Nintr;
    double *d_intr, *d_in, *d_out, *d_grad = nullptr, *d_gi = nullptr;
    if(!D.upload(&d_intr, intrinsics, (size_t)Nintr) || !D.upload(&d_in, in, nin) || !D.alloc(&d_out, nout) ||
       (grad && !D.alloc(&d_grad, (size_t)N * 6)) || (gi && !D.alloc(&d_gi, ngi)))
        return false;
    if(gi) MB200_CUDA_CHECK(cudaMemsetAsync(d_gi, 0, ngi * sizeof(double), D.stream));
    L.a.intr = d_intr;
    const mrcal_lensmodel_metadata_t meta = mrcal_lensmodel_metadata(lensmodel);
    const int threads = 128, blocks = (N + threads - 1) / threads;
    const bool ok = dispatch_lens_kind(L.kind, [&](auto k)
    {
        constexpr int K = decltype(k)::value;
        if(call == UNPROJECT)
            unproject_kernel<K><<<blocks, threads, 0, D.stream>>>(L.a, d_in, N, d_out, d_grad, d_gi, Nintr,
                                                                  meta.can_project_behind_camera, opt != 0);
        else if(call == PROJECT)
            project_kernel<K><<<blocks, threads, 0, D.stream>>>(L.a, d_in, N, d_out, d_grad, d_gi, Nintr);
        else
            resolution_kernel<K><<<blocks, threads, 0, D.stream>>>(L.a, d_in, N, d_out, opt, meta.can_project_behind_camera);
    });
    if(!ok) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(out, d_out, nout) && (!grad || D.download(grad, d_grad, (size_t)N * 6)) &&
           (!gi || D.download(gi, d_gi, ngi)) && D.finish();
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// replaces mrcal.h:165-191. dq_dp (N,2,3) and dq_dintrinsics (N,2,Nintrinsics; dense, mrcal.c:2866-2992) may be NULL
extern "C" bool mrcal_project(mrcal_point2_t* q, mrcal_point3_t* dq_dp, double* dq_dintrinsics,
                              const mrcal_point3_t* p, int N, const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(PROJECT, (double*)q, (double*)dq_dp, dq_dintrinsics, (const double*)p, N, lensmodel, intrinsics);
}

// replaces mrcal.h:193-224
extern "C" bool mrcal_unproject(mrcal_point3_t* out, const mrcal_point2_t* q, int N,
                                const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(UNPROJECT, (double*)out, nullptr, nullptr, (const double*)q, N, lensmodel, intrinsics);
}

extern "C" bool mrcal_b200_unproject_with_gradients(mrcal_point3_t* v, double* dv_dq, double* dv_dintrinsics,
                                                    const mrcal_point2_t* q, int N, const mrcal_lensmodel_t* lensmodel,
                                                    const double* intrinsics, bool normalize)
{
    return run(UNPROJECT, (double*)v, dv_dq, dv_dintrinsics, (const double*)q, N, lensmodel, intrinsics, normalize);
}

extern "C" bool mrcal_b200_model_resolution__deg_pixel(double* resolution, const mrcal_point2_t* q, int N,
                                                       const mrcal_lensmodel_t* lensmodel, const double* intrinsics,
                                                       int mode)
{
    if(mode < MB200_RESOLUTION_MEAN || mode > MB200_RESOLUTION_ECCENTRICITY)
    {
        set_error("Mode must be one of ('min','max','mean','eccentricity')");
        return false;
    }
    return run(RESOLUTION, resolution, nullptr, nullptr, (const double*)q, N, lensmodel, intrinsics, mode);
}
