// mrcal_project() / mrcal_unproject(): the reference's point-wise entry points
// (mrcal.h:165-224, mrcal.c:2866-3080 and :3082-3270), host buffers in and out,
// one thread per point on the device. They use the same lens-model device functions
// as the residual kernels (device_math.cuh); the unprojection is unproject.cuh's.
#include <cuda_runtime.h>

#include "common.h"
#include "device_call.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "unproject.cuh"

namespace mb200 {
namespace {

// dq_di: dense (N,2,Nintr), zeroed by the caller, or NULL. The layout of mrcal.c:2936-2992: the core (dq/df
// on its own axis only, dq/dc = I), then the distortions -- dense for the parametric models, the RUN x RUN touched
// control points of the matching surface for the splined ones
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
        double* out = dq_di + (size_t)i * 2 * Nintr;
        if constexpr(LensTraits<KIND>::SPLINED)
        {
            constexpr int RUN = LensTraits<KIND>::RUN;
            double wx[4], wy[4], upd[2];
            int ivar0;
            project_splined<RUN>(qq, g, wx, wy, &ivar0, upd, pp, a.intr, a.Nx, a.Ny, a.segments_per_u);
            out[0] = upd[0]; out[Nintr + 1] = upd[1];
            for(int k = 0; k < 2; k++)
                for(int iy = 0; iy < RUN; iy++)
                    for(int ix = 0; ix < RUN; ix++)
                        out[k * Nintr + ivar0 + 2 * a.Nx * iy + 2 * ix + k] = wx[ix] * wy[iy] * a.intr[k];
        }
        else
        {
            constexpr int ND = LensTraits<KIND>::NDIST;
            double ddist[2][ND > 0 ? ND : 1];
            project_parametric<KIND>(qq, g, ddist, pp, a.intr, a.cfg);
            out[0] = (qq[0] - a.intr[2]) / a.intr[0];          // mrcal.c:1427-1431
            out[Nintr + 1] = (qq[1] - a.intr[3]) / a.intr[1];
            for(int k = 0; k < 2; k++)
                for(int d = 0; d < ND; d++) out[k * Nintr + 4 + d] = ddist[k][d];
        }
        out[2] = 1.; out[Nintr + 3] = 1.;
    }
    q[2 * i] = qq[0]; q[2 * i + 1] = qq[1];
    if(dq_dp)
        for(int r = 0; r < 2; r++)
            for(int c = 0; c < 3; c++) dq_dp[6 * i + 3 * r + c] = g[r][c];
}

template <int KIND>
__global__ void unproject_kernel(LensArgs a, const double* __restrict__ q, int N, double* __restrict__ v, bool behind_ok)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= N) return;
    double out[3];
    unproject_any<KIND>(out, q[2 * i], q[2 * i + 1], a, behind_ok);
    v[3 * i] = out[0]; v[3 * i + 1] = out[1]; v[3 * i + 2] = out[2];
}

bool run(bool unproject, double* out, double* dq_dp, double* dq_di, const double* in, int N, const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    DeviceCall D;
    HostLens L;
    if(!D.start() || !lens_setup(&L, lensmodel)) return false;
    if(N <= 0) return true;
    if(unproject && !central_projection(L, intrinsics)) return false;
    const int Nintr = L.Nintr;
    const size_t nin = (size_t)N * (unproject ? 2 : 3), nout = (size_t)N * (unproject ? 3 : 2);
    double *d_intr, *d_in, *d_out, *d_grad = nullptr, *d_gi = nullptr;
    if(!D.upload(&d_intr, intrinsics, (size_t)Nintr) || !D.upload(&d_in, in, nin) || !D.alloc(&d_out, nout) ||
       (dq_dp && !D.alloc(&d_grad, (size_t)N * 6)) || (dq_di && !D.alloc(&d_gi, (size_t)N * 2 * Nintr)))
        return false;
    if(dq_di) MB200_CUDA_CHECK(cudaMemsetAsync(d_gi, 0, (size_t)N * 2 * Nintr * sizeof(double), D.stream));
    L.a.intr = d_intr;
    const mrcal_lensmodel_metadata_t meta = mrcal_lensmodel_metadata(lensmodel);
    const int threads = 128, blocks = (N + threads - 1) / threads;
    const bool ok = dispatch_lens_kind(L.kind, [&](auto k)
    {
        constexpr int K = decltype(k)::value;
        if(unproject) unproject_kernel<K><<<blocks, threads, 0, D.stream>>>(L.a, d_in, N, d_out, meta.can_project_behind_camera);
        else          project_kernel<K><<<blocks, threads, 0, D.stream>>>(L.a, d_in, N, d_out, d_grad, d_gi, Nintr);
    });
    if(!ok) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(out, d_out, nout) && (!dq_dp || D.download(dq_dp, d_grad, (size_t)N * 6)) &&
           (!dq_di || D.download(dq_di, d_gi, (size_t)N * 2 * Nintr)) && D.finish();
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// replaces mrcal.h:165-191. dq_dp (N,2,3) and dq_dintrinsics (N,2,Nintrinsics; dense, mrcal.c:2866-2992) may be NULL
extern "C" bool mrcal_project(mrcal_point2_t* q, mrcal_point3_t* dq_dp, double* dq_dintrinsics,
                              const mrcal_point3_t* p, int N, const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(false, (double*)q, (double*)dq_dp, dq_dintrinsics, (const double*)p, N, lensmodel, intrinsics);
}

// replaces mrcal.h:193-224
extern "C" bool mrcal_unproject(mrcal_point3_t* out, const mrcal_point2_t* q, int N,
                                const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(true, (double*)out, nullptr, nullptr, (const double*)q, N, lensmodel, intrinsics);
}
