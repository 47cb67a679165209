// Lens-model dispatch shared by the point-wise kernels (project.cu, diff.cu): the per-call lens arguments, one
// projection call for every kind, and the runtime kind -> template instantiation switch.
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

// Everything of LensArgs but intr, for a lens model whose kind has been checked (lens_kind_of() >= 0)
inline bool lens_args_setup(LensArgs* a, int kind, const mrcal_lensmodel_t* lensmodel)
{
    *a = LensArgs{};
    if(kind == LENS_SPLINED3 || kind == LENS_SPLINED2)
    {
        a->Nx = lensmodel->LENSMODEL_SPLINED_STEREOGRAPHIC__config.Nx;
        a->Ny = lensmodel->LENSMODEL_SPLINED_STEREOGRAPHIC__config.Ny;
        if(!spline_segments_per_u(&a->segments_per_u, lensmodel)) return false;
    }
    if(kind == LENS_CAHVORE) a->cfg = lensmodel->LENSMODEL_CAHVORE__config.linearity;
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
