// Stereo rectification and ranging, as the reference's stereo.h/stereo.c define them (stereo.c:19-972, 1242-1417):
// the geometry of a rectified pair (host), the rectification maps (one thread per rectified pixel per camera) and the
// conversion of disparities to ranges and to points (one thread per element).
//
// The maps form each rectified ray directly from its pixel, as mrcal_unproject_latlon()/_pinhole() define it; the
// reference's incremental sin/cos recurrence across a row (stereo.c:880-942) only saves CPU time. Each map kernel is
// instantiated per (lens kind, rectification model) and launched once per camera.
#include <cuda_runtime.h>
#include <cfloat>

#include "common.h"
#include "device_call.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "pose.cuh"

namespace mb200 {
namespace {

enum { RECT_LATLON = 0, RECT_PINHOLE = 1 };

struct Mat3 { double m[9]; };
struct Fxycxy { double fx, fy, cx, cy; };

// the rectified ray of pixel (x, y): mrcal_unproject_latlon() (x -> latitude, y -> longitude; unit length) or
// mrcal_unproject_pinhole() (z = 1)
template <int RECT>
__device__ __forceinline__ void rectified_ray(double v[3], double x, double y, const Fxycxy& f)
{
    const double a = (x - f.cx) / f.fx, b = (y - f.cy) / f.fy;
    if constexpr(RECT == RECT_LATLON)
    {
        double sa, ca, sb, cb;
        sincos(a, &sa, &ca);
        sincos(b, &sb, &cb);
        v[0] = sa; v[1] = ca * sb; v[2] = ca * cb;
    }
    else { v[0] = a; v[1] = b; v[2] = 1.; }
}

// map[i][j] = project_cam(R_cam_rect unproject_rect(j, i)), stored as a float32 pair (stereo.c:783-822)
template <int KIND, int RECT>
__global__ void rectification_maps_kernel(LensArgs a, Mat3 R, Fxycxy f, int Naz, long Npix, float2* __restrict__ map)
{
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= Npix) return;
    const int i = (int)(k / Naz), j = (int)(k - (long)i * Naz);
    double v[3];
    rectified_ray<RECT>(v, (double)j, (double)i, f);
    const double p[3] = {R.m[0] * v[0] + R.m[1] * v[1] + R.m[2] * v[2],
                         R.m[3] * v[0] + R.m[4] * v[1] + R.m[5] * v[2],
                         R.m[6] * v[0] + R.m[7] * v[1] + R.m[8] * v[2]};
    double q[2], g[2][3];
    project_any<KIND>(q, g, p, a);
    map[k] = make_float2((float)q[0], (float)q[1]);
}

// _stereo_range_one() (stereo.c:1263-1308): the range to the point seen at qrect0 with this disparity; 0 if that is
// not finite
template <int RECT>
__device__ __forceinline__ double range_one(double disparity, double qx, double qy, const Fxycxy& f, double baseline)
{
    double r;
    if constexpr(RECT == RECT_LATLON)
    {
        const double az0 = (qx - f.cx) / f.fx, disparity_rad = disparity / f.fx;
        r = baseline * cos(az0 - disparity_rad) / sin(disparity_rad);
    }
    else
    {
        const double tanaz0 = (qx - f.cx) / f.fx, tanel = (qy - f.cy) / f.fy;
        const double s_sq_recip = tanel * tanel + 1.;
        const double dtan = disparity / f.fx, tanaz1 = tanaz0 - dtan;
        r = baseline / sqrt(s_sq_recip + tanaz0 * tanaz0) * ((s_sq_recip + tanaz0 * tanaz1) / dtan + tanaz0);
    }
    return isfinite(r) ? r : 0.;
}

// Where the disparities come from. Dense: a uint16 image (row-packed on the device), scaled, with its pixel grid as
// qrect0. Sparse: doubles with their qrect0, or the pixel grid of width W if qrect0 is NULL. Ranges: given, no
// disparities at all
struct RangeInput
{
    const uint16_t* d16 = nullptr;
    double scale = 1.;
    uint16_t smin = 0, smax = 0;
    const double* d = nullptr;
    double dmin = 0., dmax = 0.;
    const double* ranges = nullptr;
    const double* q = nullptr;
    int W = 0;
};

template <int RECT>
__device__ __forceinline__ double element_range(const RangeInput& in, long k, double qx, double qy, const Fxycxy& f,
                                                double baseline)
{
    if(in.ranges) return in.ranges[k];
    if(in.d16)
    {
        // stereo.c:1399-1412
        const uint16_t s = in.d16[k];
        if(s == 0 || s < in.smin || s > in.smax) return 0.;
        return range_one<RECT>((double)s / in.scale, qx, qy, f, baseline);
    }
    // stereo.c:1337-1348
    const double d = in.d[k];
    if(d <= 0. || d < in.dmin || d > in.dmax) return 0.;
    return range_one<RECT>(d, qx, qy, f, baseline);
}

__device__ __forceinline__ void element_q(const RangeInput& in, long k, double* qx, double* qy)
{
    if(in.q) { *qx = in.q[2 * k]; *qy = in.q[2 * k + 1]; }
    else
    {
        const long i = k / in.W;
        *qx = (double)(k - i * in.W); *qy = (double)i;
    }
}

// range[k]; and if p != NULL, p[k] = range[k] normalize(unproject_rect(qrect0[k])) ((0,0,0) where the range is 0)
template <int RECT>
__global__ void stereo_range_kernel(RangeInput in, Fxycxy f, double baseline, long N, double* __restrict__ range,
                                    double* __restrict__ p)
{
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= N) return;
    double qx, qy;
    element_q(in, k, &qx, &qy);
    const double r = element_range<RECT>(in, k, qx, qy, f, baseline);
    if(range) range[k] = r;
    if(p)
    {
        double v[3];
        rectified_ray<RECT>(v, qx, qy, f);
        const double s = r / sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        p[3 * k] = v[0] * s; p[3 * k + 1] = v[1] * s; p[3 * k + 2] = v[2] * s;
    }
}

////////////////////////////////////////////////////////////////////////////////
// host: the real roots of the pinhole quartic (stereo.c:175-272). The reference asks LAPACK's dgeev for the
// eigenvalues of the companion matrix; this is the same computation without LAPACK: the companion matrix is already
// upper Hessenberg, and Francis double-shift QR iterations reduce it to quasi-triangular form
////////////////////////////////////////////////////////////////////////////////
constexpr int kMaxPoly = 4;

// eigenvalues of the n x n upper Hessenberg matrix a (row-major, destroyed). false if an eigenvalue does not converge
bool hessenberg_eigenvalues(double a[kMaxPoly][kMaxPoly], int n, double* wr, double* wi)
{
    double anorm = 0.;
    for(int i = 0; i < n; i++)
        for(int j = (i > 0 ? i - 1 : 0); j < n; j++) anorm += fabs(a[i][j]);
    int nn = n - 1, its = 0;
    double t = 0.;   // accumulated exceptional shifts
    while(nn >= 0)
    {
        // the lowest l with a negligible subdiagonal element a[l][l-1] splits off the active block l..nn
        int l = nn;
        for(; l >= 1; l--)
        {
            double s = fabs(a[l - 1][l - 1]) + fabs(a[l][l]);
            if(s == 0.) s = anorm;
            if(fabs(a[l][l - 1]) + s == s) { a[l][l - 1] = 0.; break; }
        }
        double x = a[nn][nn];
        if(l == nn)
        {
            wr[nn] = x + t; wi[nn] = 0.;
            nn--; its = 0;
            continue;
        }
        double y = a[nn - 1][nn - 1], w = a[nn][nn - 1] * a[nn - 1][nn];
        if(l == nn - 1)
        {
            // a 2x2 block: its two eigenvalues in closed form
            const double p = 0.5 * (y - x), q = p * p + w, z = sqrt(fabs(q));
            x += t;
            if(q >= 0.)
            {
                const double zz = p + copysign(z, p);
                wr[nn - 1] = wr[nn] = x + zz;
                if(zz != 0.) wr[nn] = x - w / zz;
                wi[nn - 1] = wi[nn] = 0.;
            }
            else
            {
                wr[nn - 1] = wr[nn] = x + p;
                wi[nn - 1] = z; wi[nn] = -z;
            }
            nn -= 2; its = 0;
            continue;
        }
        if(its == 60) return false;
        if(its == 10 || its == 20)
        {
            // exceptional shift, to break a cycle
            t += x;
            for(int i = 0; i <= nn; i++) a[i][i] -= x;
            const double s = fabs(a[nn][nn - 1]) + fabs(a[nn - 1][nn - 2]);
            x = y = 0.75 * s;
            w = -0.4375 * s * s;
        }
        its++;
        // the first column of the double-shift polynomial, started at the lowest m where two consecutive subdiagonal
        // elements are small enough to leave the block unchanged above it
        int m = nn - 2;
        double p = 0., q = 0., r = 0., z;
        for(; m >= l; m--)
        {
            z = a[m][m];
            const double rr = x - z, ss = y - z;
            p = (rr * ss - w) / a[m + 1][m] + a[m][m + 1];
            q = a[m + 1][m + 1] - z - rr - ss;
            r = a[m + 2][m + 1];
            const double s = fabs(p) + fabs(q) + fabs(r);
            p /= s; q /= s; r /= s;
            if(m == l) break;
            const double u = fabs(a[m][m - 1]) * (fabs(q) + fabs(r));
            const double v = fabs(p) * (fabs(a[m - 1][m - 1]) + fabs(z) + fabs(a[m + 1][m + 1]));
            if(u + v == v) break;
        }
        for(int i = m + 2; i <= nn; i++)
        {
            a[i][i - 2] = 0.;
            if(i != m + 2) a[i][i - 3] = 0.;
        }
        // chase the bulge with 3x3 Householder reflections, rows and columns l..nn
        for(int k = m; k <= nn - 1; k++)
        {
            if(k != m)
            {
                p = a[k][k - 1]; q = a[k + 1][k - 1]; r = k != nn - 1 ? a[k + 2][k - 1] : 0.;
                x = fabs(p) + fabs(q) + fabs(r);
                if(x != 0.) { p /= x; q /= x; r /= x; }
            }
            const double s = copysign(sqrt(p * p + q * q + r * r), p);
            if(s == 0.) continue;
            if(k == m) { if(l != m) a[k][k - 1] = -a[k][k - 1]; }
            else a[k][k - 1] = -s * x;
            p += s;
            x = p / s; y = q / s; z = r / s;
            q /= p; r /= p;
            for(int j = k; j <= nn; j++)
            {
                double pp = a[k][j] + q * a[k + 1][j];
                if(k != nn - 1) { pp += r * a[k + 2][j]; a[k + 2][j] -= pp * z; }
                a[k + 1][j] -= pp * y;
                a[k][j] -= pp * x;
            }
            const int imax = nn < k + 3 ? nn : k + 3;
            for(int i = l; i <= imax; i++)
            {
                double pp = x * a[i][k] + y * a[i][k + 1];
                if(k != nn - 1) { pp += z * a[i][k + 2]; a[i][k + 2] -= pp * r; }
                a[i][k + 1] -= pp * q;
                a[i][k] -= pp;
            }
        }
    }
    return true;
}

// The real roots of c[0] + c[1] x + ... + c[n-1] x^(n-1) + x^n; real: |imaginary part| <= 1e-7, as stereo.c:266-269.
// Returns their number, <0 on failure
int roots_real_polynomial(double* roots, int n, const double* c)
{
    double a[kMaxPoly][kMaxPoly] = {};
    for(int i = 1; i < n; i++) a[i][i - 1] = 1.;
    for(int i = 0; i < n; i++) a[i][n - 1] = -c[i];
    double wr[kMaxPoly], wi[kMaxPoly];
    if(!hessenberg_eigenvalues(a, n, wr, wi))
    {
        set_error("ERROR: the eigenvalue iteration did not converge");
        return -1;
    }
    int nroots = 0;
    for(int i = 0; i < n; i++)
        if(fabs(wi[i]) <= 1e-7) roots[nroots++] = wr[i];
    return nroots;
}

// cx (or cy) of a rectified pinhole: tan(az0) fx + cx = (Naz-1)/2 and the angle between the rays of pixels 0 and
// Naz-1 is the fov (stereo.c:274-385, where the quartic in C = cx/fx is derived). Of its real roots, keep those with
// the sign of cos(fov) right and a positive imager, then the most positive of the sign condition
void remove_root(double* C, int* nroots, int* i)
{
    if(*i != *nroots - 1) { C[*i] = C[*nroots - 1]; (*i)--; }
    (*nroots)--;
}

bool compute_pinhole_cxy(double* cxy, double fxy, double tanazel0, double fov_deg)
{
    const double cosfov = cos(fov_deg * M_PI / 180.);
    const double cos2fov = cosfov * cosfov;
    const double K = 2. * tanazel0;
    const double c[4] = {K * K + 1. + K * K / (cos2fov - 1), 2. * K + K * 4. / (cos2fov - 1),
                         K * K + 2 + 4. / (cos2fov - 1), 2. * K};
    double C[4];
    int nroots = roots_real_polynomial(C, 4, c);
    if(nroots <= 0) return false;
    for(int i = 0; i < nroots; i++)
        if(!(cosfov * (1. - K * C[i] - C[i] * C[i]) >= -1e-9)) remove_root(C, &nroots, &i);
    if(nroots <= 0) return false;
    for(int i = 0; i < nroots; i++)
        if(!((tanazel0 * fxy + C[i] * fxy) * 2. + 1. > 0)) remove_root(C, &nroots, &i);
    if(nroots <= 0) return false;
    double val_max = -DBL_MAX;
    int i_max = -1;
    for(int i = 0; i < nroots; i++)
    {
        const double val = cosfov * (1. - K * C[i] - C[i] * C[i]);
        if(val > val_max) { val_max = val; i_max = i; }
    }
    *cxy = C[i_max] * fxy;
    return true;
}

bool valid_rectification_model(mrcal_lensmodel_type_t t)
{
    if(t == MRCAL_LENSMODEL_LATLON || t == MRCAL_LENSMODEL_PINHOLE) return true;
    mrcal_lensmodel_t lm{};
    lm.type = t;
    const char* name = mrcal_lensmodel_name_unconfigured(&lm);
    if(name == nullptr) set_error("Unknown rectification_model_type=%d", (int)t);
    else set_error("Invalid rectification_model_type for rectification: %s; I know about MRCAL_LENSMODEL_LATLON and "
                   "MRCAL_LENSMODEL_PINHOLE", name);
    return false;
}

template <class F>
void dispatch_rect(mrcal_lensmodel_type_t t, F&& f)
{
    if(t == MRCAL_LENSMODEL_LATLON) f(std::integral_constant<int, RECT_LATLON>{});
    else f(std::integral_constant<int, RECT_PINHOLE>{});
}

// The ranges (and the points) of N elements, on a stream of their own. range and p are host buffers; either may be
// NULL. p is packed (N, 3); range has rows of W elements range_stride bytes apart (range_stride = 0: packed)
bool run_range(const RangeInput& host_in, const uint16_t* d16_host, int d16_stride, int W, long N,
               double* range, int range_stride, double* p, mrcal_lensmodel_type_t rect, const double* fxycxy,
               double baseline)
{
    DeviceCall D;
    if(!D.start()) return false;
    if(N <= 0) return true;
    RangeInput in = host_in;
    const long H = W > 0 ? N / W : 0;
    uint16_t* d_d16 = nullptr;
    double *d_d = nullptr, *d_ranges = nullptr, *d_q = nullptr, *d_range = nullptr, *d_p = nullptr;
    if((d16_host && !D.upload(&d_d16, d16_host, (size_t)d16_stride, (size_t)W, (size_t)H)) ||
       (host_in.d && !D.upload(&d_d, host_in.d, (size_t)N)) ||
       (host_in.ranges && !D.upload(&d_ranges, host_in.ranges, (size_t)N)) ||
       (host_in.q && !D.upload(&d_q, host_in.q, 2 * (size_t)N)) || (range && !D.alloc(&d_range, (size_t)N)) ||
       (p && !D.alloc(&d_p, 3 * (size_t)N)))
        return false;
    in.d16 = d_d16; in.d = d_d; in.ranges = d_ranges; in.q = d_q;
    const Fxycxy f{fxycxy[0], fxycxy[1], fxycxy[2], fxycxy[3]};
    const unsigned blocks = (unsigned)((N + 255) / 256);
    dispatch_rect(rect, [&](auto r)
    {
        stereo_range_kernel<decltype(r)::value><<<blocks, 256, 0, D.stream>>>(in, f, baseline, N, d_range, d_p);
    });
    MB200_CUDA_CHECK(cudaGetLastError());
    if(range && !(range_stride > 0 ? D.download(range, (size_t)range_stride, d_range, (size_t)W, (size_t)H)
                                   : D.download(range, d_range, (size_t)N)))
        return false;
    return (!p || D.download(p, d_p, 3 * (size_t)N)) && D.finish();
}

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_rectified_resolution(double* pixels_per_deg_az, double* pixels_per_deg_el,
                                           const mrcal_lensmodel_t* lensmodel, const double* intrinsics,
                                           const mrcal_point2_t* azel_fov_deg, const mrcal_point2_t* azel0_deg,
                                           const double* R_cam0_rect0, const mrcal_lensmodel_type_t rectification_model_type)
{
    const mrcal_lensmodel_type_t rect = rectification_model_type;
    if(*pixels_per_deg_az < 0 || *pixels_per_deg_el < 0)
    {
        // the resolution of camera 0 at the centre of the rectified view: |dq/daz| and |dq/del| there
        // (stereo.c:37-150)
        const double az0 = azel0_deg->x * M_PI / 180., el0 = azel0_deg->y * M_PI / 180.;
        double v[3], dv_daz[3], dv_del[3];
        if(rect == MRCAL_LENSMODEL_LATLON)
        {
            // v = (sin az, cos az sin el, cos az cos el)
            const double sa = sin(az0), ca = cos(az0), se = sin(el0), ce = cos(el0);
            v[0] = sa;       v[1] = ca * se;       v[2] = ca * ce;
            dv_daz[0] = ca;  dv_daz[1] = -sa * se; dv_daz[2] = -sa * ce;
            dv_del[0] = 0.;  dv_del[1] = ca * ce;  dv_del[2] = -ca * se;
        }
        else if(rect == MRCAL_LENSMODEL_LONLAT)
        {
            // v = (cos el sin az, sin el, cos el cos az)
            const double sa = sin(az0), ca = cos(az0), se = sin(el0), ce = cos(el0);
            v[0] = ce * sa;       v[1] = se; v[2] = ce * ca;
            dv_daz[0] = ce * ca;  dv_daz[1] = 0.; dv_daz[2] = -ce * sa;
            dv_del[0] = -se * sa; dv_del[1] = ce; dv_del[2] = -se * ca;
        }
        else if(rect == MRCAL_LENSMODEL_PINHOLE)
        {
            // v = (tan az, tan el, 1); d tan(th)/dth = 1/cos^2(th)
            const double ca = cos(az0), ce = cos(el0);
            v[0] = tan(az0); v[1] = tan(el0); v[2] = 1.;
            dv_daz[0] = 1. / (ca * ca); dv_daz[1] = 0.; dv_daz[2] = 0.;
            dv_del[0] = 0.; dv_del[1] = 1. / (ce * ce); dv_del[2] = 0.;
        }
        else
        {
            set_error("Unsupported rectification model");
            return false;
        }
        mrcal_point3_t v0;
        double dv0_daz[3], dv0_del[3];
        for(int j = 0; j < 3; j++)
        {
            v0.xyz[j] = dv0_daz[j] = dv0_del[j] = 0.;
            for(int k = 0; k < 3; k++)
            {
                v0.xyz[j] += R_cam0_rect0[3 * j + k] * v[k];
                dv0_daz[j] += R_cam0_rect0[3 * j + k] * dv_daz[k];
                dv0_del[j] += R_cam0_rect0[3 * j + k] * dv_del[k];
            }
        }
        mrcal_point2_t q;
        mrcal_point3_t dq_dv0[2];
        if(!mrcal_project(&q, dq_dv0, nullptr, &v0, 1, lensmodel, intrinsics)) return false;
        double n2_az = 0., n2_el = 0.;
        for(int i = 0; i < 2; i++)
        {
            double a = 0., e = 0.;
            for(int k = 0; k < 3; k++) { a += dq_dv0[i].xyz[k] * dv0_daz[k]; e += dq_dv0[i].xyz[k] * dv0_del[k]; }
            n2_az += a * a; n2_el += e * e;
        }
        if(*pixels_per_deg_az < 0) *pixels_per_deg_az *= -sqrt(n2_az) * M_PI / 180.;
        if(*pixels_per_deg_el < 0) *pixels_per_deg_el *= -sqrt(n2_el) * M_PI / 180.;
    }
    // even angular spacing: fit a whole number of pixels into the field of view (stereo.c:153-169)
    if(rect == MRCAL_LENSMODEL_LATLON || rect == MRCAL_LENSMODEL_LONLAT)
    {
        const int Naz = (int)round(azel_fov_deg->x * (*pixels_per_deg_az));
        const int Nel = (int)round(azel_fov_deg->y * (*pixels_per_deg_el));
        *pixels_per_deg_az = (double)Naz / azel_fov_deg->x;
        *pixels_per_deg_el = (double)Nel / azel_fov_deg->y;
    }
    return true;
}

extern "C" bool mrcal_rectified_system2(unsigned int* imagersize_rectified, double* fxycxy_rectified, double* rt_rect0_ref,
                                        double* baseline, double* pixels_per_deg_az, double* pixels_per_deg_el,
                                        mrcal_point2_t* azel_fov_deg, mrcal_point2_t* azel0_deg,
                                        const double az_edge_margin_deg, const mrcal_lensmodel_t* lensmodel0,
                                        const double* intrinsics0, const double* rt_cam0_ref, const double* rt_cam1_ref,
                                        const mrcal_lensmodel_type_t rectification_model_type, bool az0_deg_autodetect,
                                        bool el0_deg_autodetect, bool az_fov_deg_autodetect, bool el_fov_deg_autodetect)
{
    // the refusals of stereo.c:424-485, in its order and with its messages
    if(el0_deg_autodetect) { set_error("el0_deg_autodetect is not yet supported"); return false; }
    if(az_fov_deg_autodetect) { set_error("az_fov_deg_autodetect is not yet supported"); return false; }
    if(el_fov_deg_autodetect) { set_error("el_fov_deg_autodetect is not yet supported"); return false; }
    if(!(rectification_model_type == MRCAL_LENSMODEL_LATLON || rectification_model_type == MRCAL_LENSMODEL_PINHOLE))
    {
        mrcal_lensmodel_t lm{};
        lm.type = rectification_model_type;
        const char* name = mrcal_lensmodel_name_unconfigured(&lm);
        set_error("Unsupported rectification model '%s'. Only LENSMODEL_LATLON and LENSMODEL_PINHOLE are supported",
                  name ? name : "(null)");
        return false;
    }
    if(mrcal_lensmodel_metadata(lensmodel0).noncentral)
    {
        if(lensmodel0->type == MRCAL_LENSMODEL_CAHVORE)
        {
            const int Nintrinsics = mrcal_lensmodel_num_params(lensmodel0);
            for(int i = Nintrinsics - 3; i < Nintrinsics; i++)
                if(intrinsics0[i] != 0)
                {
                    set_error("Stereo rectification is only possible with a central projection. Please centralize your "
                              "models. This is CAHVORE, so set E=0 to centralize. This will ignore all noncentral "
                              "effects near the lens");
                    return false;
                }
        }
        else
        {
            set_error("Stereo rectification is only possible with a central projection. Please centralize your models");
            return false;
        }
    }
    if(*pixels_per_deg_az == 0)
    {
        set_error("pixels_per_deg_az == 0 is illegal. Must be >0 if we're trying to specify a value, or <0 to autodetect");
        return false;
    }
    if(*pixels_per_deg_el == 0)
    {
        set_error("pixels_per_deg_el == 0 is illegal. Must be >0 if we're trying to specify a value, or <0 to autodetect");
        return false;
    }
    if(azel_fov_deg->x <= 0. || azel_fov_deg->y <= 0.)
    {
        set_error("az_fov_deg, el_fov_deg must be > 0. No auto-detection implemented yet");
        return false;
    }

    // The rectified frame, in camera-0 coordinates (stereo.c:488-550): x ("right") along the baseline towards camera
    // 1, z ("forward") the mean of the two optical axes without its component along x, y ("down") completing it
    double Rt_cam0_ref[12], Rt_cam1_ref[12], Rt_ref_cam1[12], Rt01[12];
    R_from_r(Rt_cam0_ref, nullptr, rt_cam0_ref);
    R_from_r(Rt_cam1_ref, nullptr, rt_cam1_ref);
    for(int i = 0; i < 3; i++) { Rt_cam0_ref[9 + i] = rt_cam0_ref[3 + i]; Rt_cam1_ref[9 + i] = rt_cam1_ref[3 + i]; }
    invert_Rt(Rt_ref_cam1, Rt_cam1_ref);
    compose_Rt(Rt01, Rt_cam0_ref, Rt_ref_cam1, false, false);

    double Rt_rect0_cam0[12] = {};
    double* right = &Rt_rect0_cam0[0];
    double* down = &Rt_rect0_cam0[3];
    double* forward = &Rt_rect0_cam0[6];
    *baseline = 0.;
    for(int i = 0; i < 3; i++) { right[i] = Rt01[9 + i]; *baseline += right[i] * right[i]; }
    *baseline = sqrt(*baseline);
    if(*baseline < 1e-6)
    {
        set_error("The stereo pair has a unnaturally small baseline. Did you accidentally pass the same model for the "
                  "two cameras?");
        return false;
    }
    for(int i = 0; i < 3; i++) right[i] /= *baseline;
    const double forward01[3] = {Rt01[2], Rt01[5], Rt01[8] + 1.};
    double forward01_proj_right = 0., norm2_forward = 0.;
    for(int i = 0; i < 3; i++) forward01_proj_right += forward01[i] * right[i];
    for(int i = 0; i < 3; i++) { forward[i] = forward01[i] - forward01_proj_right * right[i]; norm2_forward += forward[i] * forward[i]; }
    for(int i = 0; i < 3; i++) forward[i] /= sqrt(norm2_forward);
    down[0] = forward[1] * right[2] - forward[2] * right[1];
    down[1] = forward[2] * right[0] - forward[0] * right[2];
    down[2] = forward[0] * right[1] - forward[1] * right[0];

    // az0, and the margin the view must keep from the baseline direction (stereo.c:555-627). The checks are loosened
    // a little, so that a corrected az0 passes them despite rounding
    const double margin_loose = az_edge_margin_deg - 1e-3;
    double az0 = azel0_deg->x * M_PI / 180.;
    const double el0 = azel0_deg->y * M_PI / 180.;
    auto in_bounds = [&]()
    {
        return azel0_deg->x - azel_fov_deg->x / 2. > -90. + margin_loose &&
               azel0_deg->x + azel_fov_deg->x / 2. < 90. - margin_loose;
    };
    if(az0_deg_autodetect)
    {
        // the mean forward direction of the cameras, which need not be perpendicular to the baseline
        double norm2_forward01 = 0.;
        for(int i = 0; i < 3; i++) norm2_forward01 += forward01[i] * forward01[i];
        az0 = asin(forward01_proj_right / sqrt(norm2_forward01));
        azel0_deg->x = az0 * 180. / M_PI;
        if(!in_bounds())
        {
            if(azel_fov_deg->x > 180. - 2. * az_edge_margin_deg)
            {
                set_error("ERROR: rectified view cannot avoid looking along the baseline vector: az_fov_deg is too "
                          "large. Have az_fov=%.1fdeg angle_margin=%.1fdeg", azel_fov_deg->x, az_edge_margin_deg);
                return false;
            }
            if(!(azel0_deg->x - azel_fov_deg->x / 2. > -90. + margin_loose))
                azel0_deg->x = -90. + az_edge_margin_deg + azel_fov_deg->x / 2.;
            else
                azel0_deg->x = 90. - az_edge_margin_deg - azel_fov_deg->x / 2.;
            az0 = azel0_deg->x / 180. * M_PI;
        }
    }
    else if(!in_bounds())
    {
        set_error("ERROR: rectified view looks along the baseline vector. Reduce az_fov_deg or move az0_deg closer to "
                  "the center. Have az0=%.1fdeg az_fov=%.1fdeg angle_margin=%.1fdeg",
                  azel0_deg->x, azel_fov_deg->x, az_edge_margin_deg);
        return false;
    }

    double R_cam0_rect0[9];
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++) R_cam0_rect0[3 * i + j] = Rt_rect0_cam0[3 * j + i];
    if(!mrcal_rectified_resolution(pixels_per_deg_az, pixels_per_deg_el, lensmodel0, intrinsics0, azel_fov_deg,
                                   azel0_deg, R_cam0_rect0, rectification_model_type))
        return false;

    // fx, fy from the resolution; then cx, cy and the imager (stereo.c:645-702)
    fxycxy_rectified[0] = *pixels_per_deg_az / M_PI * 180.;
    fxycxy_rectified[1] = *pixels_per_deg_el / M_PI * 180.;
    if(rectification_model_type == MRCAL_LENSMODEL_LATLON)
    {
        // even angular spacing: the imager's centre is (az0, el0)
        imagersize_rectified[0] = (int)round(azel_fov_deg->x * (*pixels_per_deg_az));
        imagersize_rectified[1] = (int)round(azel_fov_deg->y * (*pixels_per_deg_el));
        fxycxy_rectified[2] = ((double)(imagersize_rectified[0] - 1)) / 2 - az0 * fxycxy_rectified[0];
        fxycxy_rectified[3] = ((double)(imagersize_rectified[1] - 1)) / 2 - el0 * fxycxy_rectified[1];
    }
    else
    {
        // pinhole: the resolution is highest at the centre, dq/dth = f/cos^2(th); the imager is asymmetric, so cx and
        // Naz (cy and Nel) come from the quartic
        const double cos_az0 = cos(az0), cos_el0 = cos(el0);
        fxycxy_rectified[0] *= cos_az0 * cos_az0;
        fxycxy_rectified[1] *= cos_el0 * cos_el0;
        const double tanaz0 = tan(az0), tanel0 = tan(el0);
        if(!compute_pinhole_cxy(&fxycxy_rectified[2], fxycxy_rectified[0], tanaz0, azel_fov_deg->x))
        {
            set_error("Couldn't compute the rectified pinhole cx. Something is wrong.");
            return false;
        }
        if(!compute_pinhole_cxy(&fxycxy_rectified[3], fxycxy_rectified[1], tanel0, azel_fov_deg->y))
        {
            set_error("Couldn't compute the rectified pinhole cy. Something is wrong.");
            return false;
        }
        imagersize_rectified[0] = (int)round((tanaz0 * fxycxy_rectified[0] + fxycxy_rectified[2]) * 2.) + 1;
        imagersize_rectified[1] = (int)round((tanel0 * fxycxy_rectified[1] + fxycxy_rectified[3]) * 2.) + 1;
    }
    if((int)imagersize_rectified[1] <= 0)
    {
        set_error("Resulting stereo geometry has Nel=%d. This is nonsensical. You should examine the geometry or adjust "
                  "the elevation bounds or pixels-per-deg", (int)imagersize_rectified[1]);
        return false;
    }

    double Rt_rect0_ref[12];
    compose_Rt(Rt_rect0_ref, Rt_rect0_cam0, Rt_cam0_ref, false, false);
    r_from_R(rt_rect0_ref, nullptr, Rt_rect0_ref);
    for(int i = 0; i < 3; i++) rt_rect0_ref[3 + i] = Rt_rect0_ref[9 + i];
    return true;
}

extern "C" bool mrcal_rectified_system(unsigned int* imagersize_rectified, double* fxycxy_rectified, double* rt_rect0_ref,
                                       double* baseline, double* pixels_per_deg_az, double* pixels_per_deg_el,
                                       mrcal_point2_t* azel_fov_deg, mrcal_point2_t* azel0_deg,
                                       const mrcal_lensmodel_t* lensmodel0, const double* intrinsics0,
                                       const double* rt_cam0_ref, const double* rt_cam1_ref,
                                       const mrcal_lensmodel_type_t rectification_model_type, bool az0_deg_autodetect,
                                       bool el0_deg_autodetect, bool az_fov_deg_autodetect, bool el_fov_deg_autodetect)
{
    return mrcal_rectified_system2(imagersize_rectified, fxycxy_rectified, rt_rect0_ref, baseline, pixels_per_deg_az,
                                   pixels_per_deg_el, azel_fov_deg, azel0_deg, 10.0, lensmodel0, intrinsics0,
                                   rt_cam0_ref, rt_cam1_ref, rectification_model_type, az0_deg_autodetect,
                                   el0_deg_autodetect, az_fov_deg_autodetect, el_fov_deg_autodetect);
}

extern "C" bool mrcal_rectification_maps(float* rectification_maps,
                                         const mrcal_lensmodel_t* lensmodel0, const double* intrinsics0,
                                         const double* r_cam0_ref,
                                         const mrcal_lensmodel_t* lensmodel1, const double* intrinsics1,
                                         const double* r_cam1_ref,
                                         const mrcal_lensmodel_type_t rectification_model_type,
                                         const double* fxycxy_rectified, const unsigned int* imagersize_rectified,
                                         const double* r_rect0_ref)
{
    if(!(rectification_model_type == MRCAL_LENSMODEL_LATLON || rectification_model_type == MRCAL_LENSMODEL_PINHOLE))
    {
        set_error("mrcal_rectification_maps() supports MRCAL_LENSMODEL_LATLON and MRCAL_LENSMODEL_PINHOLE only");
        return false;
    }
    DeviceCall D;
    if(!D.start()) return false;
    const double* intr[2] = {intrinsics0, intrinsics1};
    const double* r_cam_ref[2] = {r_cam0_ref, r_cam1_ref};
    HostLens L[2];
    if(!lens_setup(&L[0], lensmodel0) || !lens_setup(&L[1], lensmodel1)) return false;
    const int Naz = (int)imagersize_rectified[0], Nel = (int)imagersize_rectified[1];
    const long Npix = (long)Naz * Nel;
    if(Npix <= 0) return true;
    // R_cam_rect = R_cam_ref R_rect0_ref' (stereo.c:850-862)
    double R_rect0_ref[9];
    R_from_r(R_rect0_ref, nullptr, r_rect0_ref);
    Mat3 R[2];
    for(int c = 0; c < 2; c++)
    {
        double R_cam_ref[9];
        R_from_r(R_cam_ref, nullptr, r_cam_ref[c]);
        for(int i = 0; i < 3; i++)
            for(int j = 0; j < 3; j++)
            {
                double s = 0.;
                for(int k = 0; k < 3; k++) s += R_cam_ref[3 * i + k] * R_rect0_ref[3 * j + k];
                R[c].m[3 * i + j] = s;
            }
    }
    const Fxycxy f{fxycxy_rectified[0], fxycxy_rectified[1], fxycxy_rectified[2], fxycxy_rectified[3]};
    float2* d_map;
    if(!D.alloc(&d_map, 2 * (size_t)Npix)) return false;
    const unsigned blocks = (unsigned)((Npix + 127) / 128);
    for(int c = 0; c < 2; c++)
    {
        double* d_intr;
        if(!D.upload(&d_intr, intr[c], (size_t)L[c].Nintr)) return false;
        L[c].a.intr = d_intr;
        float2* out = d_map + c * Npix;
        bool ok = false;
        dispatch_rect(rectification_model_type, [&](auto r)
        {
            constexpr int RECT = decltype(r)::value;
            ok = dispatch_lens_kind(L[c].kind, [&](auto k)
            {
                rectification_maps_kernel<decltype(k)::value, RECT><<<blocks, 128, 0, D.stream>>>(
                    L[c].a, R[c], f, Naz, Npix, out);
            });
        });
        if(!ok) return false;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download((float2*)rectification_maps, d_map, 2 * (size_t)Npix) && D.finish();
}

extern "C" bool mrcal_stereo_range_sparse(double* range, const double* disparity, const mrcal_point2_t* qrect0, const int N,
                                          const double disparity_min, const double disparity_max,
                                          const mrcal_lensmodel_type_t rectification_model_type,
                                          const double* fxycxy_rectified, const double baseline)
{
    if(!valid_rectification_model(rectification_model_type)) return false;
    if(disparity_min >= disparity_max) { set_error("Must have disparity_max > disparity_min"); return false; }
    RangeInput in;
    in.d = disparity; in.q = (const double*)qrect0; in.dmin = disparity_min; in.dmax = disparity_max;
    return run_range(in, nullptr, 0, 0, N, range, 0, nullptr, rectification_model_type, fxycxy_rectified, baseline);
}

extern "C" bool mrcal_stereo_range_dense(mrcal_image_double_t* range, const mrcal_image_uint16_t* disparity_scaled,
                                         const uint16_t disparity_scale, const uint16_t disparity_scaled_min,
                                         const uint16_t disparity_scaled_max,
                                         const mrcal_lensmodel_type_t rectification_model_type,
                                         const double* fxycxy_rectified, const double baseline)
{
    if(!valid_rectification_model(rectification_model_type)) return false;
    if(disparity_scaled_min >= disparity_scaled_max)
    {
        set_error("Must have disparity_scaled_max > disparity_scaled_min");
        return false;
    }
    if(range->width != disparity_scaled->width || range->height != disparity_scaled->height)
    {
        set_error("range and disparity_scaled MUST have the same dimensions. Got (W,H): (%d,%d) and (%d,%d) respectively",
                  range->width, range->height, disparity_scaled->width, disparity_scaled->height);
        return false;
    }
    RangeInput in;
    in.scale = (double)disparity_scale; in.smin = disparity_scaled_min; in.smax = disparity_scaled_max;
    in.W = disparity_scaled->width;
    return run_range(in, disparity_scaled->data, disparity_scaled->stride, disparity_scaled->width,
                     (long)disparity_scaled->width * disparity_scaled->height, range->data, range->stride, nullptr,
                     rectification_model_type, fxycxy_rectified, baseline);
}

extern "C" bool mrcal_b200_stereo_unproject(mrcal_point3_t* p, double* range,
                                            const mrcal_image_uint16_t* disparity_scaled, uint16_t disparity_scale,
                                            uint16_t disparity_scaled_min, uint16_t disparity_scaled_max,
                                            const double* disparity, const double* ranges, const mrcal_point2_t* qrect0,
                                            int N, int W, double disparity_min, double disparity_max,
                                            mrcal_lensmodel_type_t rectification_model_type,
                                            const double* fxycxy_rectified, double baseline)
{
    if(!valid_rectification_model(rectification_model_type)) return false;
    if((disparity_scaled != nullptr) + (disparity != nullptr) + (ranges != nullptr) != 1)
    {
        set_error("Exactly one of (disparity_scaled, disparity, ranges) must be non-NULL");
        return false;
    }
    RangeInput in;
    if(disparity_scaled)
    {
        if(disparity_scaled_min >= disparity_scaled_max)
        {
            set_error("Must have disparity_scaled_max > disparity_scaled_min");
            return false;
        }
        in.scale = (double)disparity_scale; in.smin = disparity_scaled_min; in.smax = disparity_scaled_max;
        in.W = disparity_scaled->width;
        return run_range(in, disparity_scaled->data, disparity_scaled->stride, disparity_scaled->width,
                         (long)disparity_scaled->width * disparity_scaled->height, range, 0, (double*)p,
                         rectification_model_type, fxycxy_rectified, baseline);
    }
    if(qrect0 == nullptr && (W <= 0 || N % W != 0))
    {
        set_error("Without qrect0 the elements are the pixel grid: need W > 0 dividing N");
        return false;
    }
    if(disparity && disparity_min >= disparity_max) { set_error("Must have disparity_max > disparity_min"); return false; }
    in.d = disparity; in.ranges = ranges; in.q = (const double*)qrect0; in.W = W;
    in.dmin = disparity_min; in.dmax = disparity_max;
    return run_range(in, nullptr, 0, W, N, range, 0, (double*)p, rectification_model_type, fxycxy_rectified, baseline);
}
