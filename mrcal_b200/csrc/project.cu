// mrcal_project() / mrcal_unproject(): the reference's point-wise entry points
// (mrcal.h:165-224, mrcal.c:2866-3080 and :3082-3270), host buffers in and out,
// one thread per point on the device. They use the same lens-model device functions
// as the residual kernels (device_math.cuh).
//
// Unprojection of the models without a closed form follows the reference's scheme
// (mrcal.c:3106-3270): search the 2D stereographic coordinates u of the ray so that
// project(unproject_stereographic(u)) = q, seeded from the pinhole ray. The
// reference hands that 2x2 problem to libdogleg; here it is a damped Newton
// iteration. Same fixed point, same failure rule (residual^2/2 > 1e-4 -> NaN).
#include <cuda_runtime.h>

#include "common.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "problem.h"

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
    const double fx = a.intr[0], fy = a.intr[1], cx = a.intr[2], cy = a.intr[3];
    const double x = (q[2 * i] - cx) / fx, y = (q[2 * i + 1] - cy) / fy;
    double out[3];
    if constexpr(KIND == LENS_PINHOLE) { out[0] = x; out[1] = y; out[2] = 1.; }
    else if constexpr(KIND == LENS_STEREOGRAPHIC) { out[0] = x; out[1] = y; out[2] = 1. - 0.25 * (x * x + y * y); }
    else if constexpr(KIND == LENS_LONLAT)
    {
        double sl, cl, sb, cb;
        sincos(x, &sl, &cl);   // lon
        sincos(y, &sb, &cb);   // lat
        out[0] = cb * sl; out[1] = sb; out[2] = cb * cl;
    }
    else if constexpr(KIND == LENS_LATLON)
    {
        double sl, cl, sb, cb;
        sincos(x, &sb, &cb);   // lat
        sincos(y, &sl, &cl);   // lon
        out[0] = sb; out[1] = cb * sl; out[2] = cb * cl;
    }
    else
    {
        // u: normalised stereographic coordinates of the ray; seed: the pinhole ray (x, y, 1)
        const double mag = sqrt(x * x + y * y + 1.);
        double u[2] = {2. * x / (mag + 1.), 2. * y / (mag + 1.)};
        auto residual = [&](const double uu[2], double r[2], double J[2][2])
        {
            const double vv[3] = {uu[0], uu[1], 1. - 0.25 * (uu[0] * uu[0] + uu[1] * uu[1])};
            double qq[2], g[2][3];
            project_any<KIND>(qq, g, vv, a);
            r[0] = qq[0] - q[2 * i]; r[1] = qq[1] - q[2 * i + 1];
            for(int k = 0; k < 2; k++)
            {
                J[k][0] = g[k][0] - 0.5 * uu[0] * g[k][2];
                J[k][1] = g[k][1] - 0.5 * uu[1] * g[k][2];
            }
        };
        double r[2], J[2][2];
        residual(u, r, J);
        double n2 = r[0] * r[0] + r[1] * r[1];
        for(int it = 0; it < 100 && n2 > 1e-24; it++)
        {
            const double det = J[0][0] * J[1][1] - J[0][1] * J[1][0];
            if(!(fabs(det) > 0.)) break;
            double du[2] = {-(J[1][1] * r[0] - J[0][1] * r[1]) / det, -(-J[1][0] * r[0] + J[0][0] * r[1]) / det};
            double un[2], rn[2], Jn[2][2], n2n = n2;
            bool better = false;
            for(int half = 0; half < 20; half++)
            {
                un[0] = u[0] + du[0]; un[1] = u[1] + du[1];
                residual(un, rn, Jn);
                n2n = rn[0] * rn[0] + rn[1] * rn[1];
                if(n2n < n2) { better = true; break; }
                du[0] *= 0.5; du[1] *= 0.5;
            }
            if(!better) break;
            u[0] = un[0]; u[1] = un[1]; r[0] = rn[0]; r[1] = rn[1]; n2 = n2n;
            for(int k = 0; k < 2; k++) { J[k][0] = Jn[k][0]; J[k][1] = Jn[k][1]; }
        }
        out[0] = u[0]; out[1] = u[1]; out[2] = 1. - 0.25 * (u[0] * u[0] + u[1] * u[1]);
        if(!(n2 / 2. <= 1e-4)) { out[0] = nan(""); out[1] = nan(""); }
        else if(!behind_ok && out[2] < 0.) { out[0] = -out[0]; out[1] = -out[1]; out[2] = -out[2]; }
    }
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
