// The per-point unprojection of every lens kind: unproject_any(), used by the reprojection maps (image_transforms.cu)
// and model_resolution__deg_pixel() (project.cu); its gradients, unproject_gradient(); the normalizations; the
// broadcast frame of the point-wise lens kernels, LensBroadcast; and unproject_kernel, which runs every unprojection
// entry of project.cu and the unprojections of mrcal_b200_stereo_pair_reproject() (diff.cu).
//
// Unprojection of the models without a closed form follows the reference's scheme (mrcal.c:3106-3270): search the 2D
// stereographic coordinates u of the ray so that project(unproject_stereographic(u)) = q, seeded from the pinhole
// ray. The reference hands that 2x2 problem to libdogleg; here it is a damped Newton iteration. Same fixed point,
// same failure rule (residual^2/2 > 1e-4 -> NaN).
#pragma once
#include "broadcast.cuh"
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

// The ray of pixel (qx, qy) and dv/dq, as the reference's unproject(get_gradients=True) returns them
// (mrcal/projections.py:250-397), and G: the projection at v with its intrinsics gradient, for dv/dintrinsics =
// -dv/dq dq/dintrinsics.
// - The closed-form kinds: their ray and its closed-form derivative (mrcal.c:1475-1880). G holds only the core, from
//   the given q, as the reference's dv/dintrinsics uses it.
// - The others, the reference's "q -> vs -> u -> v": the ray vs of unproject_any() is taken to its stereographic
//   coordinates u and back, v = unproject_stereographic(u), and dv/dq = dv/du (dq/du)^-1 with dq/du = dq/dv dv/du (2x2).
//   A ray that unproject_any() flipped to the front comes back with another magnitude, as in the reference. A singular
//   dq/du gives NaN dv/dq
template <int KIND>
__device__ __forceinline__ void unproject_gradient(double v[3], double dv_dq[3][2], IntrinsicsGradient<KIND>& G,
                                                   double qx, double qy, const LensArgs& a, bool behind_ok)
{
    unproject_any<KIND>(v, qx, qy, a, behind_ok);
    const double fxr = 1. / a.intr[0], fyr = 1. / a.intr[1];
    if constexpr(KIND == LENS_PINHOLE || KIND == LENS_STEREOGRAPHIC || KIND == LENS_LONLAT || KIND == LENS_LATLON)
    {
        G.q[0] = qx; G.q[1] = qy;
        const double x = (qx - a.intr[2]) * fxr, y = (qy - a.intr[3]) * fyr;
        if constexpr(KIND == LENS_PINHOLE || KIND == LENS_STEREOGRAPHIC)
        {
            dv_dq[0][0] = fxr; dv_dq[0][1] = 0.;
            dv_dq[1][0] = 0.;  dv_dq[1][1] = fyr;
            dv_dq[2][0] = KIND == LENS_PINHOLE ? 0. : -x / 2. * fxr;
            dv_dq[2][1] = KIND == LENS_PINHOLE ? 0. : -y / 2. * fyr;
        }
        else if constexpr(KIND == LENS_LONLAT)
        {
            double slon, clon, slat, clat;
            sincos(x, &slon, &clon);
            sincos(y, &slat, &clat);
            dv_dq[0][0] = fxr * clat * clon;  dv_dq[0][1] = -fyr * slat * slon;
            dv_dq[1][0] = 0.;                 dv_dq[1][1] = fyr * clat;
            dv_dq[2][0] = -fxr * clat * slon; dv_dq[2][1] = -fyr * slat * clon;
        }
        else
        {
            double slat, clat, slon, clon;
            sincos(x, &slat, &clat);
            sincos(y, &slon, &clon);
            dv_dq[0][0] = fxr * clat;         dv_dq[0][1] = 0.;
            dv_dq[1][0] = -fxr * slat * slon; dv_dq[1][1] = fyr * clat * clon;
            dv_dq[2][0] = -fxr * slat * clon; dv_dq[2][1] = -fyr * clat * slon;
        }
    }
    else
    {
        // u = project_stereographic(vs), v = unproject_stereographic(u) (mrcal.c:1511-1600, f = 1, c = 0)
        const double mag = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        const double scale = 2. / (mag + v[2]);
        const double u[2] = {v[0] * scale, v[1] * scale};
        v[0] = u[0]; v[1] = u[1]; v[2] = 1. - 0.25 * (u[0] * u[0] + u[1] * u[1]);
        const double dv_du[3][2] = {{1., 0.}, {0., 1.}, {-u[0] / 2., -u[1] / 2.}};
        double dq_dv[2][3];
        G.project(dq_dv, v, a);
        double J[2][2];
        for(int r = 0; r < 2; r++)
            for(int c = 0; c < 2; c++) J[r][c] = dq_dv[r][0] * dv_du[0][c] + dq_dv[r][1] * dv_du[1][c] + dq_dv[r][2] * dv_du[2][c];
        const double det = J[0][0] * J[1][1] - J[0][1] * J[1][0];
        const double id = det != 0. ? 1. / det : nan("");
        const double Ji[2][2] = {{J[1][1] * id, -J[0][1] * id}, {-J[1][0] * id, J[0][0] * id}};
        for(int r = 0; r < 3; r++)
            for(int c = 0; c < 2; c++) dv_dq[r][c] = dv_du[r][0] * Ji[0][c] + dv_du[r][1] * Ji[1][c];
    }
}

// LONLAT and LATLON rays are unit vectors already: normalize leaves them as they are (mrcal/projections.py:259-276)
template <int KIND>
constexpr bool unit_rays = KIND == LENS_LONLAT || KIND == LENS_LATLON;

// v/|v|, or the zero vector for a ray that is not finite, as the reference's unproject(normalize=True) without
// gradients (mrcal/projections.py:334-344); unit rays unchanged
template <int KIND>
__device__ __forceinline__ void normalize_or_zero(double v[3])
{
    if constexpr(unit_rays<KIND>) return;
    if(isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]))
    {
        const double m = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        v[0] /= m; v[1] /= m; v[2] /= m;
    }
    else v[0] = v[1] = v[2] = 0.;
}

// v -> v/|v| and each column d of dv/dq -> (I - v v'/|v|^2) d / |v|, mrcal/projections.py:220-247. The same projector
// taken through dv/dintrinsics = -dv/dq dq/dintrinsics normalizes that too
__device__ __forceinline__ void normalize_with_gradient(double v[3], double dv_dq[3][2])
{
    const double r = 1. / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
    for(int k = 0; k < 3; k++) v[k] *= r;
    for(int c = 0; c < 2; c++)
    {
        const double d[3] = {dv_dq[0][c] * r, dv_dq[1][c] * r, dv_dq[2][c] * r};
        const double vd = v[0] * d[0] + v[1] * d[1] + v[2] * d[2];
        for(int k = 0; k < 3; k++) dv_dq[k][c] = d[k] - v[k] * vd;
    }
}

// The frame of project_kernel (project.cu) and unproject_kernel: one thread per element of the broadcast shape, two
// operands read in place through Broadcast<2> -- in[0] the point (3) or pixel (2), in[1] the intrinsics row (Nintr),
// repeated through stride 0 where one row serves many elements. Every row shares one lens model: lens holds its spline
// grid and configuration, and each thread points its own copy's intr at its row. out[0] the value, out[1] its gradient
// in the point or pixel, out[2] its gradient in the intrinsics (dense, zeroed by the caller: only its nonzero entries
// are written); packed, element e's at out[k] + e * (its size). The gradients may be NULL
struct LensBroadcast : Broadcast<2>
{
    LensArgs lens;
    int Nintr;
    bool behind_ok, normalize;   // unprojection only
    double* out[3];
};

// The lens arguments of element e: the call's, pointed at e's intrinsics row. o: e's offsets into the two operands
__device__ __forceinline__ LensArgs lens_element(const LensBroadcast& b, int64_t e, int64_t o[2])
{
    broadcast_offsets(b, e, o);
    LensArgs a = b.lens;
    a.intr = b.in[1] + o[1];
    return a;
}

// One thread per pixel: v (3), and if dv_dq (3,2) = out[1] or dv_di (3,Nintr) = out[2] is given, the gradients of
// unproject_gradient() (dv_di zeroed by the caller: only its nonzero columns are written). normalize: unit rays, and
// the gradients of the unit rays. A ray or dv/dq that is not finite gives NaN gradients
template <int KIND>
__global__ void unproject_kernel(const LensBroadcast b)
{
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= b.N) return;
    int64_t o[2];
    const LensArgs a = lens_element(b, i, o);
    const double qx = b.in[0][o[0]], qy = b.in[0][o[0] + 1];
    double* __restrict__ v = b.out[0];
    double* __restrict__ dv_dq = b.out[1];
    double* __restrict__ dv_di = b.out[2];
    const int Nintr = b.Nintr;
    double out[3];
    if(dv_dq == nullptr && dv_di == nullptr)
    {
        unproject_any<KIND>(out, qx, qy, a, b.behind_ok);
        if(b.normalize) normalize_or_zero<KIND>(out);
        v[3 * i] = out[0]; v[3 * i + 1] = out[1]; v[3 * i + 2] = out[2];
        return;
    }
    double D[3][2];
    IntrinsicsGradient<KIND> G;
    unproject_gradient<KIND>(out, D, G, qx, qy, a, b.behind_ok);
    if(b.normalize && !unit_rays<KIND>) normalize_with_gradient(out, D);
    bool ok = isfinite(out[0]) && isfinite(out[1]) && isfinite(out[2]);
    for(int r = 0; r < 3; r++)
        for(int c = 0; c < 2; c++) ok = ok && isfinite(D[r][c]);
    if(!ok)
        for(int r = 0; r < 3; r++) D[r][0] = D[r][1] = nan("");
    v[3 * i] = out[0]; v[3 * i + 1] = out[1]; v[3 * i + 2] = out[2];
    if(dv_dq)
        for(int r = 0; r < 3; r++) { dv_dq[6 * i + 2 * r] = D[r][0]; dv_dq[6 * i + 2 * r + 1] = D[r][1]; }
    if(dv_di)
    {
        double* row = dv_di + i * 3 * Nintr;
        if(!ok)
            for(int j = 0; j < 3 * Nintr; j++) row[j] = nan("");
        else
            G.scatter(a, [&](int k, int col, double val)
            {
                for(int r = 0; r < 3; r++) row[r * Nintr + col] -= D[r][k] * val;
            });
    }
}

// The launch of unproject_kernel over b on stream: 128 threads per block
template <int KIND> void launch_unproject(const LensBroadcast& b, cudaStream_t stream)
{
    unproject_kernel<KIND><<<(unsigned)((b.N + 127) / 128), 128, 0, stream>>>(b);
}

}  // namespace mb200
