// mrcal_project() / mrcal_unproject(): the reference's point-wise entry points
// (mrcal.h:165-224, mrcal.c:2866-3080 and :3082-3270), host buffers in and out,
// one thread per point on the device. They use the same lens-model device functions
// as the residual kernels (device_math.cuh); the unprojection is unproject.cuh's.
#include <cuda_runtime.h>

#include "common.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "problem.h"
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

struct Scratch
{
    double *d_intr = nullptr, *d_in = nullptr, *d_out = nullptr, *d_grad = nullptr, *d_gi = nullptr;
    ~Scratch() { cudaFree(d_intr); cudaFree(d_in); cudaFree(d_out); cudaFree(d_grad); cudaFree(d_gi); }
};

bool run(bool unproject, double* out, double* dq_dp, double* dq_di, const double* in, int N, const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    int ndev = 0;
    if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0)
    {
        cudaGetLastError();
        set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback");
        return false;
    }
    const int kind = lens_kind_of(lensmodel);
    if(kind < 0) { set_error("this lens model has no CUDA implementation"); return false; }
    const int Nintr = mrcal_lensmodel_num_params(lensmodel);
    if(N <= 0) return true;
    LensArgs a;
    if(!lens_args_setup(&a, kind, lensmodel)) return false;
    if(kind == LENS_CAHVORE && unproject)
        for(int i = Nintr - 3; i < Nintr; i++)
            if(intrinsics[i] != 0.)
            {
                // the reference's rule (mrcal.c:3203-3214)
                set_error("unproject() currently only works with a central projection. So I cannot unproject(CAHVORE,E!=0)");
                return false;
            }
    Scratch S;
    const size_t nin = (size_t)N * (unproject ? 2 : 3), nout = (size_t)N * (unproject ? 3 : 2);
    MB200_CUDA_CHECK(cudaMalloc(&S.d_intr, Nintr * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&S.d_in, nin * sizeof(double)));
    MB200_CUDA_CHECK(cudaMalloc(&S.d_out, nout * sizeof(double)));
    if(dq_dp) MB200_CUDA_CHECK(cudaMalloc(&S.d_grad, (size_t)N * 6 * sizeof(double)));
    if(dq_di)
    {
        MB200_CUDA_CHECK(cudaMalloc(&S.d_gi, (size_t)N * 2 * Nintr * sizeof(double)));
        MB200_CUDA_CHECK(cudaMemset(S.d_gi, 0, (size_t)N * 2 * Nintr * sizeof(double)));
    }
    MB200_CUDA_CHECK(cudaMemcpy(S.d_intr, intrinsics, Nintr * sizeof(double), cudaMemcpyHostToDevice));
    MB200_CUDA_CHECK(cudaMemcpy(S.d_in, in, nin * sizeof(double), cudaMemcpyHostToDevice));
    a.intr = S.d_intr;
    const mrcal_lensmodel_metadata_t meta = mrcal_lensmodel_metadata(lensmodel);
    const int threads = 128, blocks = (N + threads - 1) / threads;
    const bool ok = dispatch_lens_kind(kind, [&](auto k)
    {
        constexpr int K = decltype(k)::value;
        if(unproject) unproject_kernel<K><<<blocks, threads>>>(a, S.d_in, N, S.d_out, meta.can_project_behind_camera);
        else          project_kernel<K><<<blocks, threads>>>(a, S.d_in, N, S.d_out, S.d_grad, S.d_gi, Nintr);
    });
    if(!ok) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpy(out, S.d_out, nout * sizeof(double), cudaMemcpyDeviceToHost));
    if(dq_dp) MB200_CUDA_CHECK(cudaMemcpy(dq_dp, S.d_grad, (size_t)N * 6 * sizeof(double), cudaMemcpyDeviceToHost));
    if(dq_di) MB200_CUDA_CHECK(cudaMemcpy(dq_di, S.d_gi, (size_t)N * 2 * Nintr * sizeof(double), cudaMemcpyDeviceToHost));
    return true;
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
