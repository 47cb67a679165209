// Device-side geometry and lens models for the residual/Jacobian kernels.
//
// What is computed follows the reference (file:line cited per function); how it
// is computed does not. In particular the reference builds the camera*frame
// "joint" transform with mrcal_compose_rt() + mrcal_R_from_r() and chains
// forward-mode autodiff gradients through it (mrcal.c:2659-2702, 2304-2417).
// Here the two rotations are kept separate: p_cam = Rc (Rf p + tf) + tc, and
// the analytic dR/dr tensors of the two Rodrigues vectors are applied per
// corner. Same function of (rc,tc,rf,tf), hence the same gradients, with ~6x
// fewer flops per observation and no per-observation serial prologue.
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

// R(r) (row-major 3x3) and dR[k][i][j] = dR_ij/dr_k for a Rodrigues vector r.
// Same quantity as mrcal_R_from_r_full (poseutils-opencv.c:42-155); the
// near-zero branch there (:64-84) is replaced by series that are accurate to
// roundoff for all |r| < 0.1
__host__ __device__ __forceinline__ void rodrigues(double* __restrict__ R, double* __restrict__ dR, const double* __restrict__ r)
{
    const double rx = r[0], ry = r[1], rz = r[2];
    const double t2 = rx * rx + ry * ry + rz * rz;
    double a, b, c, B, C;   // cos, sin/th, (1-cos)/th^2, d(b)/d(th^2)*2, d(c)/d(th^2)*2
    if(t2 < 1e-2)
    {
        // Taylor series in th^2; truncation error < 1e-17 at th^2 = 1e-2
        b = 1. + t2 * (-1. / 6. + t2 * (1. / 120. + t2 * (-1. / 5040. + t2 * (1. / 362880. - t2 / 39916800.))));
        c = 0.5 + t2 * (-1. / 24. + t2 * (1. / 720. + t2 * (-1. / 40320. + t2 * (1. / 3628800. - t2 / 479001600.))));
        a = 1. - t2 * c;
        B = -1. / 3. + t2 * (1. / 30. + t2 * (-1. / 840. + t2 * (1. / 45360. + t2 * (-1. / 3991680. + t2 / 518918400.))));
        C = -1. / 12. + t2 * (1. / 180. + t2 * (-1. / 6720. + t2 * (1. / 453600. + t2 * (-1. / 47900160. + t2 / 7264857600.))));
    }
    else
    {
        const double th = sqrt(t2);
        double s;
        sincos(th, &s, &a);
        b = s / th;
        c = (1. - a) / t2;
        B = (a - b) / t2;
        C = (b - 2. * c) / t2;
    }
    // R = a I + b [r]x + c r r^T
    R[0] = a + c * rx * rx;   R[1] = -b * rz + c * rx * ry; R[2] = b * ry + c * rx * rz;
    R[3] = b * rz + c * ry * rx; R[4] = a + c * ry * ry;   R[5] = -b * rx + c * ry * rz;
    R[6] = -b * ry + c * rz * rx; R[7] = b * rx + c * rz * ry; R[8] = a + c * rz * rz;
    if(dR == nullptr) return;

    const double rr[3] = {rx, ry, rz};
    // [r]x
    const double K[9] = {0., -rz, ry, rz, 0., -rx, -ry, rx, 0.};
#pragma unroll
    for(int k = 0; k < 3; k++)
    {
        const double rk = rr[k];
        double* D = &dR[9 * k];
        // da/dr_k = -b r_k ; db/dr_k = B r_k ; dc/dr_k = C r_k
#pragma unroll
        for(int i = 0; i < 3; i++)
#pragma unroll
            for(int j = 0; j < 3; j++)
            {
                double v = B * rk * K[3 * i + j] + C * rk * rr[i] * rr[j];
                if(i == j) v -= b * rk;
                if(i == k) v += c * rr[j];
                if(j == k) v += c * rr[i];
                D[3 * i + j] = v;
            }
        // b * d[r]x/dr_k
        const int i1 = (k + 1) % 3, i2 = (k + 2) % 3;
        D[3 * i2 + i1] += b;
        D[3 * i1 + i2] -= b;
    }
}

__device__ __forceinline__ void mat3_vec(double* out, const double* __restrict__ M, const double* __restrict__ v)
{
    out[0] = M[0] * v[0] + M[1] * v[1] + M[2] * v[2];
    out[1] = M[3] * v[0] + M[4] * v[1] + M[5] * v[2];
    out[2] = M[6] * v[0] + M[7] * v[1] + M[8] * v[2];
}

////////////////////////////////////////////////////////////////////////////////
// Lens models. Each returns q and dq/dp (2x3). Parametric models also fill
// dq_ddist[2][NDIST]; the splined model returns its 1D basis vectors and the
// index of the first control point it touches.
////////////////////////////////////////////////////////////////////////////////
enum LensKind
{
    LENS_PINHOLE = 0, LENS_STEREOGRAPHIC, LENS_LONLAT, LENS_LATLON,
    LENS_OPENCV4, LENS_OPENCV5, LENS_OPENCV8, LENS_OPENCV12,
    LENS_SPLINED3, LENS_SPLINED2,
    LENS_CAHVOR,
    LENS_CAHVORE,
    LENS_NKINDS
};

template <int KIND> struct LensTraits { static constexpr int NDIST = 0; static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_OPENCV4>  { static constexpr int NDIST = 4;  static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_OPENCV5>  { static constexpr int NDIST = 5;  static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_OPENCV8>  { static constexpr int NDIST = 8;  static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_OPENCV12> { static constexpr int NDIST = 12; static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_CAHVOR>   { static constexpr int NDIST = 5;  static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_CAHVORE>  { static constexpr int NDIST = 8;  static constexpr bool SPLINED = false; static constexpr int RUN = 0; };
template <> struct LensTraits<LENS_SPLINED3> { static constexpr int NDIST = 0;  static constexpr bool SPLINED = true;  static constexpr int RUN = 4; };
template <> struct LensTraits<LENS_SPLINED2> { static constexpr int NDIST = 0;  static constexpr bool SPLINED = true;  static constexpr int RUN = 3; };

// The normalised (f=1, c=0) stereographic projection u = 2 p_xy/(|p|+p_z) and
// du/dp. mrcal.c:1528-1544 (model) and :2132-2153 (inside the splined model)
__device__ __forceinline__ void stereographic_u(double* u, double du_dp[2][3], const double* p)
{
    const double mag = sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
    const double scale = 2.0 / (mag + p[2]);
    const double A = -0.5 * scale * scale;
    const double Bm = A / mag;
    u[0] = p[0] * scale;
    u[1] = p[1] * scale;
    du_dp[0][0] = p[0] * Bm * p[0] + scale; du_dp[0][1] = p[0] * Bm * p[1];         du_dp[0][2] = p[0] * (Bm * p[2] + A);
    du_dp[1][0] = p[1] * Bm * p[0];         du_dp[1][1] = p[1] * Bm * p[1] + scale; du_dp[1][2] = p[1] * (Bm * p[2] + A);
}

// Parametric models with a closed form. intr = fx,fy,cx,cy,distortions...; cfg: the model's configuration
// scalar (CAHVORE: linearity)
template <int KIND>
__device__ __forceinline__ void project_parametric(double q[2], double dq_dp[2][3],
                                                   double (*dq_ddist)[LensTraits<KIND>::NDIST > 0 ? LensTraits<KIND>::NDIST : 1],
                                                   const double* p, const double* __restrict__ intr, double cfg = 0.)
{
    const double fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
    if constexpr(KIND == LENS_PINHOLE)
    {
        // mrcal.c:1436-1468
        const double zi = 1. / p[2];
        q[0] = p[0] * zi * fx + cx;
        q[1] = p[1] * zi * fy + cy;
        dq_dp[0][0] = fx * zi; dq_dp[0][1] = 0.;      dq_dp[0][2] = -fx * p[0] * zi * zi;
        dq_dp[1][0] = 0.;      dq_dp[1][1] = fy * zi; dq_dp[1][2] = -fy * p[1] * zi * zi;
    }
    else if constexpr(KIND == LENS_STEREOGRAPHIC)
    {
        // mrcal.c:1503-1546
        double u[2], du[2][3];
        stereographic_u(u, du, p);
        q[0] = u[0] * fx + cx;
        q[1] = u[1] * fy + cy;
#pragma unroll
        for(int j = 0; j < 3; j++) { dq_dp[0][j] = fx * du[0][j]; dq_dp[1][j] = fy * du[1][j]; }
    }
    else if constexpr(KIND == LENS_LONLAT)
    {
        // q = (atan2(x,z), asin(y/|p|)) * f + c.  mrcal.c:1687-1725
        const double n2i = 1. / (p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
        const double ni = sqrt(n2i);
        const double xz2i = 1. / (p[0] * p[0] + p[2] * p[2]);
        const double xzi = sqrt(xz2i);
        dq_dp[0][0] = fx * xz2i * p[2]; dq_dp[0][1] = 0.; dq_dp[0][2] = -fx * xz2i * p[0];
        dq_dp[1][0] = -fy * xzi * (p[1] * p[0] * n2i);
        dq_dp[1][1] = -fy * xzi * (p[1] * p[1] * n2i - 1.);
        dq_dp[1][2] = -fy * xzi * (p[1] * p[2] * n2i);
        q[0] = atan2(p[0], p[2]) * fx + cx;
        q[1] = asin(p[1] * ni) * fy + cy;
    }
    else if constexpr(KIND == LENS_LATLON)
    {
        // q = (asin(x/|p|), atan2(y,z)) * f + c.  mrcal.c:1774-1810
        const double n2i = 1. / (p[0] * p[0] + p[1] * p[1] + p[2] * p[2]);
        const double ni = sqrt(n2i);
        const double yz2i = 1. / (p[1] * p[1] + p[2] * p[2]);
        const double yzi = sqrt(yz2i);
        dq_dp[0][0] = -fx * yzi * (p[0] * p[0] * n2i - 1.);
        dq_dp[0][1] = -fx * yzi * (p[0] * p[1] * n2i);
        dq_dp[0][2] = -fx * yzi * (p[0] * p[2] * n2i);
        dq_dp[1][0] = 0.; dq_dp[1][1] = fy * yz2i * p[2]; dq_dp[1][2] = -fy * yz2i * p[1];
        q[0] = asin(p[0] * ni) * fx + cx;
        q[1] = atan2(p[1], p[2]) * fy + cy;
    }
    else if constexpr(KIND == LENS_CAHVOR)
    {
        // JPL CAHVOR in mrcal's parametrisation (mrcal.c:1067-1240): distortions (alpha, beta, r0, r1, r2).
        //   o = optical axis from (alpha,beta); w = p.o ; tau = |p|^2/w^2 - 1 ; mu = r0 + r1 tau + r2 tau^2
        //   p' = p + mu (p - w o) ; q = pinhole(p')
        const double al = intr[4], be = intr[5], r0 = intr[6], r1 = intr[7], r2 = intr[8];
        double sa, ca, sb, cb;
        sincos(al, &sa, &ca);
        sincos(be, &sb, &cb);
        const double o[3]   = {sa * cb, sb, ca * cb};
        const double o_a[3] = {ca * cb, 0., -sa * cb};
        const double o_b[3] = {-sa * sb, cb, -ca * sb};
        const double n2 = p[0] * p[0] + p[1] * p[1] + p[2] * p[2];
        const double w = p[0] * o[0] + p[1] * o[1] + p[2] * o[2];
        const double wi = 1. / w;
        const double tau = n2 * wi * wi - 1.;
        const double mu = r0 + tau * (r1 + tau * r2);
        const double dmu = r1 + 2. * tau * r2;                       // d mu / d tau
        double u[3], pd[3], dmu_dp[3];
#pragma unroll
        for(int i = 0; i < 3; i++)
        {
            u[i] = p[i] - w * o[i];
            pd[i] = p[i] + mu * u[i];
            dmu_dp[i] = dmu * (2. * p[i] * wi * wi - 2. * n2 * wi * wi * wi * o[i]);
        }
        const double zi = 1. / pd[2];
        q[0] = pd[0] * zi * fx + cx;
        q[1] = pd[1] * zi * fy + cy;
        // dq/dp' (pinhole) then dp'/dp = (1+mu) I - mu o o' + u dmu_dp'
        const double gx[3] = {fx * zi, 0., -fx * pd[0] * zi * zi};
        const double gy[3] = {0., fy * zi, -fy * pd[1] * zi * zi};
#pragma unroll
        for(int j = 0; j < 3; j++)
        {
            double cxj = 0., cyj = 0.;
#pragma unroll
            for(int i = 0; i < 3; i++)
            {
                const double d = (i == j ? 1. + mu : 0.) - mu * o[i] * o[j] + u[i] * dmu_dp[j];
                cxj += gx[i] * d;
                cyj += gy[i] * d;
            }
            dq_dp[0][j] = cxj;
            dq_dp[1][j] = cyj;
        }
        if(dq_ddist != nullptr)
        {
            // dp'/d(alpha,beta): w_t = p.o_t ; tau_t = -2 |p|^2 w_t / w^3 ; dp' = dmu tau_t u - mu (w_t o + w o_t)
            const double w_a = p[0] * o_a[0] + p[1] * o_a[1] + p[2] * o_a[2];
            const double w_b = p[0] * o_b[0] + p[1] * o_b[1] + p[2] * o_b[2];
            const double mu_a = dmu * (-2. * n2 * wi * wi * wi) * w_a;
            const double mu_b = dmu * (-2. * n2 * wi * wi * wi) * w_b;
            double d[5][3];
#pragma unroll
            for(int i = 0; i < 3; i++)
            {
                d[0][i] = mu_a * u[i] - mu * (w_a * o[i] + w * o_a[i]);
                d[1][i] = mu_b * u[i] - mu * (w_b * o[i] + w * o_b[i]);
                d[2][i] = u[i];
                d[3][i] = tau * u[i];
                d[4][i] = tau * tau * u[i];
            }
#pragma unroll
            for(int k = 0; k < 5; k++)
            {
                dq_ddist[0][k] = gx[0] * d[k][0] + gx[2] * d[k][2];
                dq_ddist[1][k] = gy[1] * d[k][1] + gy[2] * d[k][2];
            }
        }
    }
    else if constexpr(KIND == LENS_CAHVORE)
    {
        // JPL CAHVORE (noncentral) in mrcal's parametrisation: distortions (alpha, beta, r0,r1,r2, e0,e1,e2) and
        // the configuration value "linearity". Same model and the same Newton iteration for theta as
        // cahvore.cc:36-158; the reference pushes forward-mode derivatives through every operation, here theta
        // carries its derivatives with respect to the five scalars it depends on (zeta, l, e0, e1, e2) through the
        // iteration (so the gradients agree with the reference's to rounding, not just to the Newton tolerance)
        // and everything after that is chained by hand.
        //   zeta = p.o ; ll = p - zeta o ; l = |ll|
        //   theta:  zeta sin - l cos - (theta - sin)(e0 + e1 theta^2 + e2 theta^4) = 0
        //   chi = theta | sin(lin theta)/lin | tan(lin theta)/lin ; mu = r0 + r1 chi^2 + r2 chi^4
        //   p' = o l/chi + ll (1 + mu) ; q = pinhole(p')
        const double al = intr[4], be = intr[5], r0 = intr[6], r1 = intr[7], r2 = intr[8], e0 = intr[9], e1 = intr[10], e2 = intr[11];
        const double lin = cfg;
        double sa, ca, sb, cb;
        sincos(al, &sa, &ca);
        sincos(be, &sb, &cb);
        const double o[3]   = {sa * cb, sb, ca * cb};
        const double o_a[3] = {ca * cb, 0., -sa * cb};
        const double o_b[3] = {-sa * sb, cb, -ca * sb};
        const double zeta = p[0] * o[0] + p[1] * o[1] + p[2] * o[2];
        const double ll[3] = {p[0] - zeta * o[0], p[1] - zeta * o[1], p[2] - zeta * o[2]};
        const double l = sqrt(ll[0] * ll[0] + ll[1] * ll[1] + ll[2] * ll[2]);
        double th = atan2(l, zeta);
        double dth[5];   // d theta / d (zeta, l, e0, e1, e2)
        {
            const double n2i = 1. / (zeta * zeta + l * l);
            dth[0] = -l * n2i; dth[1] = zeta * n2i; dth[2] = dth[3] = dth[4] = 0.;
        }
        bool failed = true;
        for(int it = 0; it < 100; it++)
        {
            double s, c;
            sincos(th, &s, &c);
            const double th2 = th * th, th3 = th * th2, th4 = th * th3;
            const double E = e0 + e1 * th2 + e2 * th4, E1 = 2. * e1 * th + 4. * e2 * th3, E2 = 2. * e1 + 12. * e2 * th2;
            const double ts = th - s;
            const double g = zeta * s - l * c - ts * E;
            const double ups = zeta * c + l * s + (c - 1.) * E - ts * E1;
            const double ups_th = -zeta * s + l * c - s * E + 2. * (c - 1.) * E1 - ts * E2;
            const double step = g / ups;
            const double g_x[5]   = {s, -c, -ts, -ts * th2, -ts * th4};
            const double ups_x[5] = {c, s, c - 1., (c - 1.) * th2 - ts * 2. * th, (c - 1.) * th4 - ts * 4. * th3};
#pragma unroll
            for(int k = 0; k < 5; k++)
            {
                const double dg = ups * dth[k] + g_x[k];
                const double du = ups_th * dth[k] + ups_x[k];
                dth[k] -= (dg - step * du) / ups;
            }
            th -= step;
            if(fabs(step) < 1e-8) { failed = false; break; }
        }
        if(failed || th * fabs(lin) > 1.5707963267948966)
        {
            // the reference refuses the whole evaluation here (cahvore.cc:104-116); the poisoned measurement does the same
            th = nan("");
        }
        double pd[3], J_p[3][3], J_i[3][8];   // p', dp'/dp, dp'/d(alpha,beta,r0,r1,r2,e0,e1,e2)
        if(th > 1e-8)
        {
            const double linth = th * lin;
            double chi, chi_th;
            if(lin < -1e-15)     { chi = sin(linth) / lin; chi_th = cos(linth); }
            else if(lin > 1e-15) { chi = tan(linth) / lin; const double ci = 1. / cos(linth); chi_th = ci * ci; }
            else                 { chi = th; chi_th = 1.; }
            const double chi2 = chi * chi, chi3 = chi * chi2, chi4 = chi2 * chi2;
            const double zp = l / chi;
            const double mu = r0 + r1 * chi2 + r2 * chi4;
            const double mu_chi = 2. * r1 * chi + 4. * r2 * chi3;
#pragma unroll
            for(int i = 0; i < 3; i++) pd[i] = o[i] * zp + ll[i] * (mu + 1.);
            // partials of p' with respect to (zeta, l, e0, e1, e2) at fixed o, ll
            double F[5][3];
#pragma unroll
            for(int k = 0; k < 5; k++)
            {
                const double chi_x = chi_th * dth[k];
                const double zp_x = (k == 1 ? 1. / chi : 0.) - l * chi_x / chi2;
                const double mu_x = mu_chi * chi_x;
#pragma unroll
                for(int i = 0; i < 3; i++) F[k][i] = o[i] * zp_x + ll[i] * mu_x;
            }
            const double li = 1. / l;
            // wrt p: zeta_p = o, l_p = ll/l, ll_p = I - o o'
#pragma unroll
            for(int i = 0; i < 3; i++)
#pragma unroll
                for(int j = 0; j < 3; j++)
                    J_p[i][j] = F[0][i] * o[j] + F[1][i] * ll[j] * li + (mu + 1.) * ((i == j ? 1. : 0.) - o[i] * o[j]);
            // wrt alpha, beta
#pragma unroll
            for(int ab = 0; ab < 2; ab++)
            {
                const double* ot = ab == 0 ? o_a : o_b;
                const double zeta_t = p[0] * ot[0] + p[1] * ot[1] + p[2] * ot[2];
                const double l_t = -zeta * (ll[0] * ot[0] + ll[1] * ot[1] + ll[2] * ot[2]) * li;
#pragma unroll
                for(int i = 0; i < 3; i++)
                    J_i[i][ab] = zp * ot[i] + (mu + 1.) * (-zeta_t * o[i] - zeta * ot[i]) + F[0][i] * zeta_t + F[1][i] * l_t;
            }
#pragma unroll
            for(int i = 0; i < 3; i++)
            {
                J_i[i][2] = ll[i]; J_i[i][3] = ll[i] * chi2; J_i[i][4] = ll[i] * chi4;
                J_i[i][5] = F[2][i]; J_i[i][6] = F[3][i]; J_i[i][7] = F[4][i];
            }
        }
        else
        {
            // small-angle branch (cahvore.cc:118-149): p' = p. (NaN theta lands here too: poison p')
#pragma unroll
            for(int i = 0; i < 3; i++)
            {
                pd[i] = th == th ? p[i] : th;
#pragma unroll
                for(int j = 0; j < 3; j++) J_p[i][j] = i == j ? 1. : 0.;
#pragma unroll
                for(int k = 0; k < 8; k++) J_i[i][k] = 0.;
            }
        }
        const double zi = 1. / pd[2];
        q[0] = pd[0] * zi * fx + cx;
        q[1] = pd[1] * zi * fy + cy;
        const double gx[3] = {fx * zi, 0., -fx * pd[0] * zi * zi};
        const double gy[3] = {0., fy * zi, -fy * pd[1] * zi * zi};
#pragma unroll
        for(int j = 0; j < 3; j++)
        {
            dq_dp[0][j] = gx[0] * J_p[0][j] + gx[2] * J_p[2][j];
            dq_dp[1][j] = gy[1] * J_p[1][j] + gy[2] * J_p[2][j];
        }
        if(dq_ddist != nullptr)
        {
#pragma unroll
            for(int k = 0; k < 8; k++)
            {
                dq_ddist[0][k] = gx[0] * J_i[0][k] + gx[2] * J_i[2][k];
                dq_ddist[1][k] = gy[1] * J_i[1][k] + gy[2] * J_i[2][k];
            }
        }
    }
    else
    {
        // OpenCV rational + tangential + thin-prism model. Same model as
        // opencv.c:50-152; the gradients are written here in terms of the
        // normalised image coordinates (x,y) and chained once
        constexpr int ND = LensTraits<KIND>::NDIST;
        double k[12];
#pragma unroll
        for(int i = 0; i < 12; i++) k[i] = i < ND ? intr[4 + i] : 0.;
        const double zi = 1. / p[2];
        const double x = p[0] * zi, y = p[1] * zi;
        const double r2 = x * x + y * y, r4 = r2 * r2, r6 = r4 * r2;
        const double num = 1. + k[0] * r2 + k[1] * r4 + k[4] * r6;
        const double deni = 1. / (1. + k[5] * r2 + k[6] * r4 + k[7] * r6);
        const double s = num * deni;
        const double a1 = 2. * x * y, a2 = r2 + 2. * x * x, a3 = r2 + 2. * y * y;
        const double xd = x * s + k[2] * a1 + k[3] * a2 + k[8] * r2 + k[9] * r4;
        const double yd = y * s + k[2] * a3 + k[3] * a1 + k[10] * r2 + k[11] * r4;
        q[0] = xd * fx + cx;
        q[1] = yd * fy + cy;

        // ds/dr2
        const double dnum = k[0] + 2. * k[1] * r2 + 3. * k[4] * r4;
        const double dden = k[5] + 2. * k[6] * r2 + 3. * k[7] * r4;
        const double ds = (dnum - s * dden) * deni;
        const double px = k[8] + 2. * k[9] * r2;    // thin prism d/dr2
        const double py = k[10] + 2. * k[11] * r2;
        const double dxd_dx = s + 2. * x * x * ds + 2. * k[2] * y + 6. * k[3] * x + 2. * x * px;
        const double dxd_dy = 2. * x * y * ds + 2. * k[2] * x + 2. * k[3] * y + 2. * y * px;
        const double dyd_dx = 2. * x * y * ds + 2. * k[2] * x + 2. * k[3] * y + 2. * x * py;
        const double dyd_dy = s + 2. * y * y * ds + 6. * k[2] * y + 2. * k[3] * x + 2. * y * py;
        // d(x,y)/dp = [zi 0 -x zi; 0 zi -y zi]
        dq_dp[0][0] = fx * dxd_dx * zi; dq_dp[0][1] = fx * dxd_dy * zi; dq_dp[0][2] = -fx * zi * (dxd_dx * x + dxd_dy * y);
        dq_dp[1][0] = fy * dyd_dx * zi; dq_dp[1][1] = fy * dyd_dy * zi; dq_dp[1][2] = -fy * zi * (dyd_dx * x + dyd_dy * y);

        if(dq_ddist != nullptr)
        {
            double gx[12], gy[12];
            gx[0] = x * deni * r2; gy[0] = y * deni * r2;
            gx[1] = x * deni * r4; gy[1] = y * deni * r4;
            gx[2] = a1;            gy[2] = a3;
            gx[3] = a2;            gy[3] = a1;
            gx[4] = x * deni * r6; gy[4] = y * deni * r6;
            const double m = -s * deni;
            gx[5] = x * m * r2; gy[5] = y * m * r2;
            gx[6] = x * m * r4; gy[6] = y * m * r4;
            gx[7] = x * m * r6; gy[7] = y * m * r6;
            gx[8] = r2; gy[8] = 0.;
            gx[9] = r4; gy[9] = 0.;
            gx[10] = 0.; gy[10] = r2;
            gx[11] = 0.; gy[11] = r4;
#pragma unroll
            for(int i = 0; i < ND; i++) { dq_ddist[0][i] = fx * gx[i]; dq_ddist[1][i] = fy * gy[i]; }
        }
    }
}

// Uniform B-spline basis and its derivative. Cubic: t in [0,1] between the 2nd
// and 3rd of 4 control points; quadratic: t in [-1/2,1/2] about the middle of 3.
// mrcal.c:902-917, 991-1002 (derived in the reference's analyses/splines/bsplines.py)
template <int RUN>
__device__ __forceinline__ void bspline_basis(double* w, double* dw, double t)
{
    const double t2 = t * t;
    if constexpr(RUN == 4)
    {
        const double t3 = t2 * t;
        w[0] = (-t3 + 3. * t2 - 3. * t + 1.) / 6.;
        w[1] = (3. * t3 / 2. - 3. * t2 + 2.) / 3.;
        w[2] = (-3. * t3 + 3. * t2 + 3. * t + 1.) / 6.;
        w[3] = t3 / 6.;
        dw[0] = -t2 / 2. + t - 0.5;
        dw[1] = 3. * t2 / 2. - 2. * t;
        dw[2] = -3. * t2 / 2. + t + 0.5;
        dw[3] = t2 / 2.;
    }
    else
    {
        w[0] = (4. * t2 - 4. * t + 1.) / 8.;
        w[1] = (3. - 4. * t2) / 4.;
        w[2] = (4. * t2 + 4. * t + 1.) / 8.;
        dw[0] = t - 0.5;
        dw[1] = -2. * t;
        dw[2] = t + 0.5;
    }
}

// LENSMODEL_SPLINED_STEREOGRAPHIC: q = (u + deltau(u)) f + c, with deltau two
// interleaved B-spline surfaces over the stereographic u. mrcal.c:2075-2293.
//   wx, wy  basis weights along x and y (RUN each): d deltau_k / d knot(ix,iy,k) = wx[ix] wy[iy]
//   ivar0   index in the camera's intrinsics vector of control point (0,0) of the
//           touched RUNxRUN window (x surface); includes the 4 core values
//   upd[2]  u + deltau  (= dq/df)
template <int RUN>
__device__ __forceinline__ void project_splined(double q[2], double dq_dp[2][3],
                                                double* wx, double* wy, int* ivar0, double upd[2],
                                                const double* p, const double* __restrict__ intr,
                                                int Nx, int Ny, double segments_per_u)
{
    double u[2], du[2][3];
    stereographic_u(u, du, p);
    const double ix = u[0] * segments_per_u + (double)(Nx - 1) / 2.;
    const double iy = u[1] * segments_per_u + (double)(Ny - 1) / 2.;
    int ix0, iy0;
    if constexpr(RUN == 4)
    {
        // (int) truncates toward zero, as in the reference (:2171-2172)
        ix0 = (int)ix; iy0 = (int)iy;
        ix0 = ix0 < 1 ? 1 : (ix0 > Nx - 3 ? Nx - 3 : ix0);
        iy0 = iy0 < 1 ? 1 : (iy0 > Ny - 3 ? Ny - 3 : iy0);
    }
    else
    {
        ix0 = (int)(ix + 0.5); iy0 = (int)(iy + 0.5);
        ix0 = ix0 < 1 ? 1 : (ix0 > Nx - 2 ? Nx - 2 : ix0);
        iy0 = iy0 < 1 ? 1 : (iy0 > Ny - 2 ? Ny - 2 : iy0);
    }
    *ivar0 = 4 + 2 * ((iy0 - 1) * Nx + (ix0 - 1));

    double dwx[RUN], dwy[RUN];
    bspline_basis<RUN>(wx, dwx, ix - (double)ix0);
    bspline_basis<RUN>(wy, dwy, iy - (double)iy0);

    // sample both surfaces and their derivatives wrt (ix,iy)
    const double* __restrict__ c = &intr[*ivar0];
    double v[2] = {0., 0.}, vx[2] = {0., 0.}, vy[2] = {0., 0.};
#pragma unroll
    for(int jy = 0; jy < RUN; jy++)
    {
        double rv[2] = {0., 0.}, rdx[2] = {0., 0.};
#pragma unroll
        for(int jx = 0; jx < RUN; jx++)
        {
            const double c0 = __ldg(&c[jy * 2 * Nx + jx * 2 + 0]);
            const double c1 = __ldg(&c[jy * 2 * Nx + jx * 2 + 1]);
            rv[0] += wx[jx] * c0;   rv[1] += wx[jx] * c1;
            rdx[0] += dwx[jx] * c0; rdx[1] += dwx[jx] * c1;
        }
#pragma unroll
        for(int k = 0; k < 2; k++)
        {
            v[k]  += wy[jy] * rv[k];
            vx[k] += wy[jy] * rdx[k];
            vy[k] += dwy[jy] * rv[k];
        }
    }
    const double fx = intr[0], fy = intr[1], cx = intr[2], cy = intr[3];
    upd[0] = u[0] + v[0];
    upd[1] = u[1] + v[1];
    q[0] = upd[0] * fx + cx;
    q[1] = upd[1] * fy + cy;
    // d deltau / du = d deltau / d(ix,iy) * segments_per_u
    const double dxx = vx[0] * segments_per_u, dxy = vy[0] * segments_per_u;   // d deltau_x / du_x, / du_y
    const double dyx = vx[1] * segments_per_u, dyy = vy[1] * segments_per_u;   // d deltau_y / du_x, / du_y
#pragma unroll
    for(int j = 0; j < 3; j++)
    {
        dq_dp[0][j] = fx * (du[0][j] * (1. + dxx) + dxy * du[1][j]);
        dq_dp[1][j] = fy * (du[1][j] * (1. + dyy) + dyx * du[0][j]);
    }
}

}  // namespace mb200
