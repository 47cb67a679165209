// Lens-model dispatch: the per-call lens arguments and their host setup, one projection call for every kind, and the
// runtime kind -> template instantiation switch, for the point-wise kernels (project.cu, diff.cu, image_transforms.cu,
// stereo.cu) and the problem's own (eval.cu, uncertainty.cu).
#pragma once
#include <type_traits>

#include "common.h"
#include "device_math.cuh"

namespace mb200 {

bool spline_segments_per_u(double* out, const mrcal_lensmodel_t* lm);   // layout.cpp
int lens_kind_of(const mrcal_lensmodel_t* lm);                          // problem.cu

// intr: device pointer to the intrinsics, set by the caller
struct LensArgs { const double* intr; int Nx, Ny; double segments_per_u, cfg; };

template <int KIND>
__device__ __forceinline__ void project_any(double q[2], double dq_dp[2][3], const double* p, const LensArgs& a)
{
    if constexpr(LensTraits<KIND>::SPLINED)
    {
        double wx[4], wy[4], upd[2];
        int ivar0;
        project_splined<LensTraits<KIND>::RUN>(q, dq_dp, wx, wy, &ivar0, upd, p, a.intr, a.Nx, a.Ny, a.segments_per_u);
    }
    else
        project_parametric<KIND>(q, dq_dp, nullptr, p, a.intr, a.cfg);
}

// A projection with its gradient in the intrinsics, kept in the compact form the model computes it in. scatter() hands
// every nonzero entry of dq/dintrinsics to emit(row, column, value), in the dense layout of mrcal.c:2936-2992: the core
// (dq/df on its own axis only, from q; dq/dc = I), then the distortions -- dense for the parametric models, the RUN x RUN
// touched control points of the matching surface for the splined ones
template <int KIND>
struct IntrinsicsGradient
{
    static constexpr int ND = LensTraits<KIND>::NDIST, RUN = LensTraits<KIND>::RUN;
    double q[2];
    double ddist[2][ND > 0 ? ND : 1];
    double wx[4], wy[4], upd[2];
    int ivar0;

    __device__ __forceinline__ void project(double dq_dp[2][3], const double* p, const LensArgs& a)
    {
        if constexpr(LensTraits<KIND>::SPLINED)
            project_splined<RUN>(q, dq_dp, wx, wy, &ivar0, upd, p, a.intr, a.Nx, a.Ny, a.segments_per_u);
        else
            project_parametric<KIND>(q, dq_dp, ddist, p, a.intr, a.cfg);
    }

    template <class F>
    __device__ __forceinline__ void scatter(const LensArgs& a, F&& emit) const
    {
        if constexpr(LensTraits<KIND>::SPLINED)
        {
            emit(0, 0, upd[0]); emit(1, 1, upd[1]);
            for(int k = 0; k < 2; k++)
                for(int iy = 0; iy < RUN; iy++)
                    for(int ix = 0; ix < RUN; ix++)
                        emit(k, ivar0 + 2 * a.Nx * iy + 2 * ix + k, wx[ix] * wy[iy] * a.intr[k]);
        }
        else
        {
            emit(0, 0, (q[0] - a.intr[2]) / a.intr[0]);          // mrcal.c:1427-1431
            emit(1, 1, (q[1] - a.intr[3]) / a.intr[1]);
            for(int k = 0; k < 2; k++)
                for(int d = 0; d < ND; d++) emit(k, 4 + d, ddist[k][d]);
        }
        emit(0, 2, 1.); emit(1, 3, 1.);
    }
};

// A lens model as the point-wise kernels take it. a.intr is left for the caller to point at the uploaded intrinsics
struct HostLens { int kind; LensArgs a; int Nintr; };

// false + set_error() for a lens model without a kernel or with an invalid spline grid
inline bool lens_setup(HostLens* L, const mrcal_lensmodel_t* lensmodel)
{
    *L = HostLens{lens_kind_of(lensmodel), LensArgs{}, mrcal_lensmodel_num_params(lensmodel)};
    if(L->kind < 0) { set_error("this lens model has no CUDA implementation"); return false; }
    if(L->kind == LENS_SPLINED3 || L->kind == LENS_SPLINED2)
    {
        L->a.Nx = lensmodel->LENSMODEL_SPLINED_STEREOGRAPHIC__config.Nx;
        L->a.Ny = lensmodel->LENSMODEL_SPLINED_STEREOGRAPHIC__config.Ny;
        if(!spline_segments_per_u(&L->a.segments_per_u, lensmodel)) return false;
    }
    if(L->kind == LENS_CAHVORE) L->a.cfg = lensmodel->LENSMODEL_CAHVORE__config.linearity;
    return true;
}

// unproject() needs a central projection: the refusal of CAHVORE with E != 0, the reference's rule (mrcal.c:3203-3214)
inline bool refuse_noncentral()
{
    set_error("unproject() currently only works with a central projection. So I cannot unproject(CAHVORE,E!=0)");
    return false;
}

// false + refuse_noncentral() for CAHVORE with E != 0 in the (host) intrinsics
inline bool central_projection(const HostLens& L, const double* intrinsics)
{
    if(L.kind == LENS_CAHVORE)
        for(int i = L.Nintr - 3; i < L.Nintr; i++)
            if(intrinsics[i] != 0.) return refuse_noncentral();
    return true;
}

// f(std::integral_constant<int, KIND>{}) for the runtime kind; false + set_error() for a kind without a kernel
template <class F>
bool dispatch_lens_kind(int kind, F&& f)
{
#define MB200_LENS_CASE(K) case K: f(std::integral_constant<int, K>{}); return true;
    switch(kind)
    {
        MB200_LENS_CASE(LENS_PINHOLE) MB200_LENS_CASE(LENS_STEREOGRAPHIC) MB200_LENS_CASE(LENS_LONLAT) MB200_LENS_CASE(LENS_LATLON)
        MB200_LENS_CASE(LENS_OPENCV4) MB200_LENS_CASE(LENS_OPENCV5) MB200_LENS_CASE(LENS_OPENCV8) MB200_LENS_CASE(LENS_OPENCV12)
        MB200_LENS_CASE(LENS_SPLINED3) MB200_LENS_CASE(LENS_SPLINED2) MB200_LENS_CASE(LENS_CAHVOR) MB200_LENS_CASE(LENS_CAHVORE)
    default: set_error("lens model kind %d has no CUDA implementation", kind); return false;
    }
#undef MB200_LENS_CASE
}

}  // namespace mb200
