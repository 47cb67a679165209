// The per-point unprojection of every lens kind, shared by mrcal_unproject() (project.cu) and the reprojection maps
// (image_transforms.cu).
//
// Unprojection of the models without a closed form follows the reference's scheme (mrcal.c:3106-3270): search the 2D
// stereographic coordinates u of the ray so that project(unproject_stereographic(u)) = q, seeded from the pinhole
// ray. The reference hands that 2x2 problem to libdogleg; here it is a damped Newton iteration. Same fixed point,
// same failure rule (residual^2/2 > 1e-4 -> NaN).
#pragma once
#include "device_math.cuh"
#include "lens_dispatch.cuh"

namespace mb200 {

// out: the (not normalised) observation ray of pixel (qx, qy). behind_ok: the model can project points behind the
// camera; otherwise a solution with z < 0 is flipped to the front
template <int KIND>
__device__ __forceinline__ void unproject_any(double out[3], double qx, double qy, const LensArgs& a, bool behind_ok)
{
    const double fx = a.intr[0], fy = a.intr[1], cx = a.intr[2], cy = a.intr[3];
    const double x = (qx - cx) / fx, y = (qy - cy) / fy;
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
            r[0] = qq[0] - qx; r[1] = qq[1] - qy;
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
}

}  // namespace mb200
