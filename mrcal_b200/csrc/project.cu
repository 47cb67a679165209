// mrcal_project() / mrcal_unproject(): the reference's point-wise entry points (mrcal.h:165-224, mrcal.c:2866-3080
// and :3082-3270), and mrcal_b200_project(): the same projections broadcast over stacked intrinsics, with host or device
// buffers. One thread per element on the device, in the broadcast frame of unproject.cuh (LensBroadcast): the
// entries for one intrinsics vector repeat it through stride 0. They use the same lens-model device functions as the
// residual kernels (device_math.cuh); the unprojection is unproject.cuh's. With them, the unprojection with gradients
// (mrcal/projections.py:112-397) and model_resolution__deg_pixel() (mrcal/model_analysis.py:2152-2246).
#include <cuda_runtime.h>

#include "broadcast.cuh"
#include "common.h"
#include "device_call.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "unproject.cuh"

namespace mb200 {
namespace {

enum { F_GRAD = MRCAL_B200_PROJECT_GET_GRADIENTS, F_UNPROJECT = MRCAL_B200_PROJECT_UNPROJECT,
       F_NORMALIZE = MRCAL_B200_PROJECT_NORMALIZE };

// One thread per point: q (2), and if given, dq_dp (2,3) = out[1] and dq_di (2,Nintr) = out[2] (zeroed by the caller;
// IntrinsicsGradient::scatter() fills its nonzero entries)
template <int KIND>
__global__ void project_kernel(const LensBroadcast b)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= b.N) return;
    int64_t o[2];
    const LensArgs a = lens_element(b, i, o);
    double* __restrict__ q = b.out[0];
    double* __restrict__ dq_dp = b.out[1];
    double* __restrict__ dq_di = b.out[2];
    const int Nintr = b.Nintr;
    double qq[2], g[2][3];
    const double pp[3] = {b.in[0][o[0]], b.in[0][o[0] + 1], b.in[0][o[0] + 2]};
    if(dq_di == nullptr) project_any<KIND>(qq, g, pp, a);
    else
    {
        IntrinsicsGradient<KIND> G;
        G.project(g, pp, a);
        qq[0] = G.q[0]; qq[1] = G.q[1];
        double* out = dq_di + i * 2 * Nintr;
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

// flag = 1 if any intrinsics row of r (CAHVORE, Nintr) has E != 0. One thread per row
__global__ void noncentral_kernel(const Broadcast<1> r, int Nintr, int* flag)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= r.N) return;
    int64_t o[1];
    broadcast_offsets(r, i, o);
    const double* E = r.in[0] + o[0] + Nintr - 3;
    if(E[0] != 0. || E[1] != 0. || E[2] != 0.) *flag = 1;
}

// The checks both flavours of mrcal_b200_project() make, and the broadcast frame of the call; the operands and outputs
// are not filled in
bool prepare(LensBroadcast& b, HostLens& L, const mrcal_lensmodel_t* lensmodel, int flags, int ndim,
             const int64_t* shape, const int64_t* strides_in, const int64_t* strides_intrinsics)
{
    if(flags & ~(F_GRAD | F_UNPROJECT | F_NORMALIZE) || ((flags & F_NORMALIZE) && !(flags & F_UNPROJECT)))
    {
        set_error("project: invalid flags 0x%x", flags);
        return false;
    }
    if(!lens_setup(&L, lensmodel)) return false;
    const int64_t* const st[2] = {strides_in, strides_intrinsics};
    const int width[2] = {flags & F_UNPROJECT ? 2 : 3, L.Nintr};
    b = LensBroadcast{};
    if(!broadcast_prepare<2>(b, "project", flags, ndim, shape, st, width)) return false;
    b.lens = L.a;
    b.Nintr = L.Nintr;
    b.behind_ok = mrcal_lensmodel_metadata(lensmodel).can_project_behind_camera;
    b.normalize = flags & F_NORMALIZE;
    return true;
}

// The projection (or with F_UNPROJECT the unprojection) of every element of b on stream, b's operands and outputs on
// the device. out[2], the dense intrinsics gradient, is zeroed first: the kernels write only its nonzero entries
bool launch(const LensBroadcast& b, int kind, int flags, cudaStream_t stream)
{
    const size_t rows = flags & F_UNPROJECT ? 3 : 2;
    if(b.out[2]) MB200_CUDA_CHECK(cudaMemsetAsync(b.out[2], 0, (size_t)b.N * rows * b.Nintr * sizeof(double), stream));
    const bool ok = dispatch_lens_kind(kind, [&](auto k)
    {
        constexpr int K = decltype(k)::value;
        if(flags & F_UNPROJECT) launch_unproject<K>(b, stream);
        else project_kernel<K><<<(unsigned)((b.N + 127) / 128), 128, 0, stream>>>(b);
    });
    if(!ok) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// mrcal_project(), mrcal_unproject(), mrcal_b200_unproject_with_gradients(): N points or pixels of one intrinsics
// vector, host buffers. flags: F_*; the gradients may be NULL
bool run(int flags, double* out, double* grad, double* gi, const double* in, int N, const mrcal_lensmodel_t* lensmodel,
         const double* intrinsics)
{
    // shape (N,): the points packed, the intrinsics repeated
    const int w_in = flags & F_UNPROJECT ? 2 : 3, w_out = 5 - w_in;
    const int64_t shape[1] = {N > 0 ? N : 0}, st_in[1] = {w_in}, st_intr[1] = {0};
    DeviceCall D;
    HostLens L;
    LensBroadcast b;
    if(!D.start() || !prepare(b, L, lensmodel, flags, 1, shape, st_in, st_intr)) return false;
    if(N <= 0) return true;
    if((flags & F_UNPROJECT) && !central_projection(L, intrinsics)) return false;
    const size_t nin = (size_t)N * w_in, nout = (size_t)N * w_out, ngi = (size_t)N * w_out * L.Nintr;
    double *d_intr, *d_in, *d_out, *d_grad = nullptr, *d_gi = nullptr;
    if(!D.upload(&d_intr, intrinsics, (size_t)L.Nintr) || !D.upload(&d_in, in, nin) || !D.alloc(&d_out, nout) ||
       (grad && !D.alloc(&d_grad, (size_t)N * 6)) || (gi && !D.alloc(&d_gi, ngi)))
        return false;
    b.in[0] = d_in;
    b.in[1] = d_intr;
    b.out[0] = d_out;
    b.out[1] = d_grad;
    b.out[2] = d_gi;
    return launch(b, L.kind, flags, D.stream) && D.download(out, d_out, nout) &&
           (!grad || D.download(grad, d_grad, (size_t)N * 6)) && (!gi || D.download(gi, d_gi, ngi)) && D.finish();
}

}  // namespace
}  // namespace mb200

using namespace mb200;

// replaces mrcal.h:165-191. dq_dp (N,2,3) and dq_dintrinsics (N,2,Nintrinsics; dense, mrcal.c:2866-2992) may be NULL
extern "C" bool mrcal_project(mrcal_point2_t* q, mrcal_point3_t* dq_dp, double* dq_dintrinsics,
                              const mrcal_point3_t* p, int N, const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(F_GRAD, (double*)q, (double*)dq_dp, dq_dintrinsics, (const double*)p, N, lensmodel, intrinsics);
}

// replaces mrcal.h:193-224
extern "C" bool mrcal_unproject(mrcal_point3_t* out, const mrcal_point2_t* q, int N,
                                const mrcal_lensmodel_t* lensmodel, const double* intrinsics)
{
    return run(F_UNPROJECT, (double*)out, nullptr, nullptr, (const double*)q, N, lensmodel, intrinsics);
}

extern "C" bool mrcal_b200_unproject_with_gradients(mrcal_point3_t* v, double* dv_dq, double* dv_dintrinsics,
                                                    const mrcal_point2_t* q, int N, const mrcal_lensmodel_t* lensmodel,
                                                    const double* intrinsics, bool normalize)
{
    return run(F_GRAD | F_UNPROJECT | (normalize ? F_NORMALIZE : 0), (double*)v, dv_dq, dv_dintrinsics,
               (const double*)q, N, lensmodel, intrinsics);
}

extern "C" bool mrcal_b200_project(const mrcal_lensmodel_t* lensmodel, int flags, int ndim, const int64_t* shape,
                                   const double* in, const int64_t* strides_in, const double* intrinsics,
                                   const int64_t* strides_intrinsics, double* out, double* dout_din,
                                   double* dout_dintrinsics)
{
    LensBroadcast b;
    HostLens L;
    if(!prepare(b, L, lensmodel, flags, ndim, shape, strides_in, strides_intrinsics)) return false;
    if(b.N == 0) return true;
    if(flags & F_UNPROJECT)
    {
        // every intrinsics row the call reads must be central
        b.in[1] = intrinsics;
        const Broadcast<1> rows = broadcast_rows(b, 1);
        for(int64_t r = 0; r < rows.N; r++)
        {
            int64_t o[1];
            broadcast_offsets(rows, r, o);
            if(!central_projection(L, intrinsics + o[0])) return false;
        }
    }
    const bool G = flags & F_GRAD;
    const int w_in = flags & F_UNPROJECT ? 2 : 3, w_out = 5 - w_in;
    const size_t n0 = b.N * w_out, n1 = G && dout_din ? b.N * 6 : 0, n2 = G && dout_dintrinsics ? b.N * w_out * L.Nintr : 0;
    DeviceCall D;
    const double *d_in, *d_intr;
    double *d_out, *d_grad = nullptr, *d_gi = nullptr;
    if(!D.start() || !D.upload((double**)&d_in, in, broadcast_extent(b, 0, w_in)) ||
       !D.upload((double**)&d_intr, intrinsics, broadcast_extent(b, 1, L.Nintr)) || !D.alloc(&d_out, n0) ||
       (n1 && !D.alloc(&d_grad, n1)) || (n2 && !D.alloc(&d_gi, n2)))
        return false;
    b.in[0] = d_in;
    b.in[1] = d_intr;
    b.out[0] = d_out;
    b.out[1] = d_grad;
    b.out[2] = d_gi;
    return launch(b, L.kind, flags, D.stream) && D.download(out, d_out, n0) &&
           (!n1 || D.download(dout_din, d_grad, n1)) && (!n2 || D.download(dout_dintrinsics, d_gi, n2)) && D.finish();
}

extern "C" bool mrcal_b200_project_device(const mrcal_lensmodel_t* lensmodel, int flags, int ndim, const int64_t* shape,
                                          const double* in, const int64_t* strides_in, const double* intrinsics,
                                          const int64_t* strides_intrinsics, double* out, double* dout_din,
                                          double* dout_dintrinsics, void* stream)
{
    LensBroadcast b;
    HostLens L;
    if(!prepare(b, L, lensmodel, flags, ndim, shape, strides_in, strides_intrinsics)) return false;
    if(b.N == 0) return true;
    if(!have_device()) return false;
    b.in[0] = in;
    b.in[1] = intrinsics;
    if((flags & F_UNPROJECT) && L.kind == LENS_CAHVORE)
    {
        // every intrinsics row the call reads must be central: one flag back to the host, so this call waits
        DeviceCall D;
        int *d_flag, flag = 0;
        if(!D.start((cudaStream_t)stream) || !D.alloc(&d_flag, 1)) return false;
        MB200_CUDA_CHECK(cudaMemsetAsync(d_flag, 0, sizeof(int), D.stream));
        const Broadcast<1> rows = broadcast_rows(b, 1);
        noncentral_kernel<<<(unsigned)((rows.N + 127) / 128), 128, 0, D.stream>>>(rows, L.Nintr, d_flag);
        MB200_CUDA_CHECK(cudaGetLastError());
        if(!D.download(&flag, d_flag, 1) || !D.finish()) return false;
        if(flag) return refuse_noncentral();
    }
    const bool G = flags & F_GRAD;
    b.out[0] = out;
    b.out[1] = G ? dout_din : nullptr;
    b.out[2] = G ? dout_dintrinsics : nullptr;
    return launch(b, L.kind, flags, (cudaStream_t)stream);
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
    DeviceCall D;
    HostLens L;
    if(!D.start() || !lens_setup(&L, lensmodel)) return false;
    if(N <= 0) return true;
    if(!central_projection(L, intrinsics)) return false;
    double *d_intr, *d_q, *d_out;
    if(!D.upload(&d_intr, intrinsics, (size_t)L.Nintr) || !D.upload(&d_q, (const double*)q, 2 * (size_t)N) ||
       !D.alloc(&d_out, (size_t)N))
        return false;
    L.a.intr = d_intr;
    const bool behind_ok = mrcal_lensmodel_metadata(lensmodel).can_project_behind_camera;
    const int threads = 128, blocks = (N + threads - 1) / threads;
    if(!dispatch_lens_kind(L.kind, [&](auto k)
       {
           resolution_kernel<decltype(k)::value><<<blocks, threads, 0, D.stream>>>(L.a, d_q, N, d_out, mode, behind_ok);
       }))
        return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(resolution, d_out, (size_t)N) && D.finish();
}
