// Projection uncertainty: Var(q) of a camera's projection of query points, from the noise of the calibration's pixel
// observations propagated through the solve -- the reference's mrcal.projection_uncertainty()
// (mrcal/model_analysis.py:1192-1517, with _propagate_calibration_uncertainty() :560-869), on the device end to end.
//
// For each query point, F = q(p_cam) depends on the solved state through the rows dF/db_packed (2 x Nstate):
//     intrinsics  dq/dintrinsics                                               every method
//     extrinsics  dq/dpcam dpcam/drt_cam_ref / Ne                              mean-pcam, rrp-Jfp
//     frames      mean over the extrinsics j of dq/dpref_j dpref/drt_ref_frame / Nframes   mean-pcam
//     K term      [dq/dpcam skew(p_cam) | -dq/dpcam] K_ccp   or   [dq/dpref skew(p_ref) | -dq/dpref] K_rrp
// (at infinity only the rotations: translations drop out). The direct columns are in unpacked units and are multiplied
// by the pack scales; K = drt/db_packed is already per packed unknown. The rows go straight into the pieces of the
// permuted right-hand side of the structured factor P JtJ P' = L L' (factorization_schur.cu), and
//
//     Z = inv(L) P dF'                    Var0 = Z'Z = dF inv(JtJ) dF'
//     X = inv(L') Z  (shared part only)   Var  = sigma^2 (Var0 - (Jr X)'(Jr X))
//
// The second form is the reference's  dF inv(JtJ) Jo'Jo inv(JtJ) dF'  (:750-766) with Jo'Jo = JtJ - Jr'Jr: Jr, the
// regularization rows, touches shared unknowns only (the intrinsics; with unity_cam01 also an extrinsics vector), which
// are never eliminated, so X is needed only on the shared unknowns and the backward pass stops after L_S' (the panels
// are not needed in that direction). Without regularization rows Var = sigma^2 Z'Z (:784-843).
//
// The triangular solves are the structured factor's own (schur_solve_pieces(), factorization_schur.cu), which take
// tiles of kSolveTile right-hand sides when there are many. The 2x2 per point is reduced by one warp in a fixed order:
// no atomics anywhere, two calls give bit-identical results.
#include <algorithm>
#include <vector>

#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "reduce.cuh"
#include "solver_internal.h"

namespace mb200 {

namespace {

struct RowArgs
{
    int method;           // MRCAL_B200_UNCERTAINTY_*
    bool atinfinity;
    int icam;             // icam_intrinsics
    int e_first, Ne;      // the camera's consecutive extrinsics; Ne = 0: at the reference
    int intr_col0;        // state column of the camera's first intrinsics unknown, -1 if none
    int intr_arg0;        // which intrinsics parameter that is (4 if the core is not optimized)
    int Nelim;
    const double* scale;  // [Nstate] pack scales
};

// transform_point_rt(rt, p) and its gradient in r: R p + t, d(R p)/dr (3x3). rotation only: R p
__device__ __forceinline__ void pose_apply(double out[3], double d_dr[3][3], const double R[9], const double dR[27], const double* t, const double p[3])
{
    mat3_vec(out, R, p);
    if(t) for(int i = 0; i < 3; i++) out[i] += t[i];
    for(int i = 0; i < 3; i++)
        for(int k = 0; k < 3; k++) d_dr[i][k] = dR[9 * k + 3 * i] * p[0] + dR[9 * k + 3 * i + 1] * p[1] + dR[9 * k + 3 * i + 2] * p[2];
}
// p = R'(x - t)  (t == nullptr: R' x)
__device__ __forceinline__ void pose_invert_apply(double p[3], const double R[9], const double* t, const double x[3])
{
    const double v[3] = {x[0] - (t ? t[0] : 0.), x[1] - (t ? t[1] : 0.), x[2] - (t ? t[2] : 0.)};
    for(int i = 0; i < 3; i++) p[i] = R[i] * v[0] + R[3 + i] * v[1] + R[6 + i] * v[2];
}

// One thread per query point: the direct columns of its two rows, and the 2x6 coefficients G of the K term
template <int KIND>
__global__ void __launch_bounds__(128)
uncertainty_rows_kernel(DevProblem P, NormalBuffers N, RowArgs A, const double* __restrict__ pcam, int Npts,
                        double* __restrict__ Bf, double* __restrict__ Bs, double* __restrict__ Bi, double* __restrict__ G)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= Npts) return;
    const double p[3] = {pcam[3 * i], pcam[3 * i + 1], pcam[3 * i + 2]};
    const double* intr = P.u_intr + (size_t)A.icam * P.Nintr;
    const int r0 = 2 * i;
    auto put = [&](int row, int c, double v) { *N.at(N.slot(c), Bf, A.Nelim, Bs, Bi, row) = v * A.scale[c]; };
    // intrinsics parameter k (of the model's Nintr) -> its state column, or -1
    auto intr_col = [&](int k) { const int j = k - A.intr_arg0; return (A.intr_col0 >= 0 && j >= 0 && j < P.Nintr_state) ? A.intr_col0 + j : -1; };

    double q[2], dq_dp[2][3];
    if constexpr(LensTraits<KIND>::SPLINED)
    {
        constexpr int RUN = LensTraits<KIND>::RUN;
        double wx[4], wy[4], upd[2];
        int ivar0;
        project_splined<RUN>(q, dq_dp, wx, wy, &ivar0, upd, p, intr, P.Nx, P.Ny, P.segments_per_u);
        int c;
        if((c = intr_col(0)) >= 0) put(r0, c, upd[0]);
        if((c = intr_col(1)) >= 0) put(r0 + 1, c, upd[1]);
        if((c = intr_col(2)) >= 0) put(r0, c, 1.);
        if((c = intr_col(3)) >= 0) put(r0 + 1, c, 1.);
        for(int k = 0; k < 2; k++)
            for(int iy = 0; iy < RUN; iy++)
                for(int ix = 0; ix < RUN; ix++)
                    if((c = intr_col(ivar0 + 2 * P.Nx * iy + 2 * ix + k)) >= 0) put(r0 + k, c, wx[ix] * wy[iy] * intr[k]);
    }
    else
    {
        constexpr int ND = LensTraits<KIND>::NDIST;
        double ddist[2][ND > 0 ? ND : 1];
        project_parametric<KIND>(q, dq_dp, ddist, p, intr, P.lens_cfg);
        int c;
        if((c = intr_col(0)) >= 0) put(r0, c, (q[0] - intr[2]) / intr[0]);
        if((c = intr_col(1)) >= 0) put(r0 + 1, c, (q[1] - intr[3]) / intr[1]);
        if((c = intr_col(2)) >= 0) put(r0, c, 1.);
        if((c = intr_col(3)) >= 0) put(r0 + 1, c, 1.);
        for(int k = 0; k < 2; k++)
            for(int d = 0; d < ND; d++)
                if((c = intr_col(4 + d)) >= 0) put(r0 + k, c, ddist[k][d]);
    }

    const bool inf = A.atinfinity;
    const int Ne = A.Ne > 0 ? A.Ne : 1;
    // per extrinsics j: p_ref_j, and dq/dpref_j = dq/dpcam R_j. The extrinsics columns as we go
    double Gk[2][6] = {};
    const bool want_e = A.method != MRCAL_B200_UNCERTAINTY_CCP && A.Ne > 0 && P.opt_extr;
    const bool want_f = A.method == MRCAL_B200_UNCERTAINTY_MEAN_PCAM && P.opt_frames && P.i_frame0 >= 0;
    // the frames columns accumulate over j: zeroed here, written once at the end of each j
    for(int j = 0; j < Ne; j++)
    {
        double R[9] = {1., 0., 0., 0., 1., 0., 0., 0., 1.}, dR[27] = {};
        const double* t = nullptr;
        if(A.Ne > 0)
        {
            const double* rt = P.u_rtcam + 6 * (size_t)(A.e_first + j);
            rodrigues(R, dR, rt);
            t = inf ? nullptr : rt + 3;
        }
        double pref[3];
        pose_invert_apply(pref, R, t, p);
        double dqr[2][3];   // dq/dpref = dq/dpcam R
        for(int a = 0; a < 2; a++)
            for(int k = 0; k < 3; k++) dqr[a][k] = dq_dp[a][0] * R[k] + dq_dp[a][1] * R[3 + k] + dq_dp[a][2] * R[6 + k];
        if(want_e)
        {
            double pc[3], d_dr[3][3];
            pose_apply(pc, d_dr, R, dR, nullptr, pref);
            const int c0 = P.i_extr0 + 6 * (A.e_first + j);
            for(int a = 0; a < 2; a++)
            {
                for(int k = 0; k < 3; k++)
                    put(r0 + a, c0 + k, (dq_dp[a][0] * d_dr[0][k] + dq_dp[a][1] * d_dr[1][k] + dq_dp[a][2] * d_dr[2][k]) / A.Ne);
                if(!inf)
                    for(int k = 0; k < 3; k++) put(r0 + a, c0 + 3 + k, dq_dp[a][k] / A.Ne);
            }
        }
        if(want_f)
        {
            for(int f = 0; f < P.Nframes; f++)
            {
                const double* rtf = P.u_rtframe + 6 * (size_t)f;
                double Rf[9], dRf[27];
                rodrigues(Rf, dRf, rtf);
                double pf[3], pr[3], d_dr[3][3];
                pose_invert_apply(pf, Rf, inf ? nullptr : rtf + 3, pref);
                pose_apply(pr, d_dr, Rf, dRf, nullptr, pf);
                const int c0 = P.i_frame0 + 6 * f;
                const double w = 1. / ((double)Ne * (double)P.Nframes);
                for(int a = 0; a < 2; a++)
                {
                    double v[6];
                    for(int k = 0; k < 3; k++) v[k] = (dqr[a][0] * d_dr[0][k] + dqr[a][1] * d_dr[1][k] + dqr[a][2] * d_dr[2][k]) * w;
                    for(int k = 0; k < 3; k++) v[3 + k] = inf ? 0. : dqr[a][k] * w;
                    for(int k = 0; k < 6; k++)
                    {
                        double* s = N.at(N.slot(c0 + k), Bf, A.Nelim, Bs, Bi, r0 + a);
                        const double add = v[k] * A.scale[c0 + k];
                        *s = j == 0 ? add : *s + add;
                    }
                }
            }
        }
        if(A.method != MRCAL_B200_UNCERTAINTY_MEAN_PCAM && j == 0)
        {
            // [dq/dx skew(x) | -dq/dx]: x = p_cam with dq/dpcam (ccp), x = p_ref with dq/dpref (rrp)
            const bool ccp = A.method == MRCAL_B200_UNCERTAINTY_CCP;
            const double* x = ccp ? p : pref;
            for(int a = 0; a < 2; a++)
            {
                const double* g = ccp ? dq_dp[a] : dqr[a];
                // (g skew(x))_k, skew(x) = [0 -x2 x1; x2 0 -x0; -x1 x0 0]
                Gk[a][0] = g[1] * x[2] - g[2] * x[1];
                Gk[a][1] = -g[0] * x[2] + g[2] * x[0];
                Gk[a][2] = g[0] * x[1] - g[1] * x[0];
                for(int k = 0; k < 3; k++) Gk[a][3 + k] = inf ? 0. : -g[k];
            }
        }
    }
    if(G)
        for(int a = 0; a < 2; a++)
            for(int k = 0; k < 6; k++) G[(size_t)(r0 + a) * 6 + k] = Gk[a][k];
}

// rows += G K over the columns [c0, Nstate) K can be nonzero in: one thread per (row, column)
__global__ void uncertainty_K_kernel(NormalBuffers N, int Nelim, const double* __restrict__ G, const double* __restrict__ K,
                                     int Nstate, int c0, int Nrows, double* __restrict__ Bf, double* __restrict__ Bs, double* __restrict__ Bi)
{
    const int w = Nstate - c0;
    const long idx = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(idx >= (long)Nrows * w) return;
    const int row = (int)(idx / w), c = c0 + (int)(idx - (long)row * w);
    double v = 0.;
#pragma unroll
    for(int k = 0; k < 6; k++) v += G[(size_t)row * 6 + k] * K[(size_t)k * Nstate + c];
    *N.at(N.slot(c), Bf, Nelim, Bs, Bi, row) += v;
}

// Var0 = Z'Z per point: one warp per point, lanes over the unknowns, then a butterfly (fixed order)
__global__ void ztz_kernel(const NormalBuffers N, const double* __restrict__ Bf, int Nelim, const double* __restrict__ Bs,
                           const double* __restrict__ Bi, int nBi, int Npts, double* __restrict__ V /*[Npts][3]*/)
{
    const int pt = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if(pt >= Npts) return;
    double s[3] = {0., 0., 0.};
    auto acc = [&](const double* a, const double* b, int n)
    {
        for(int c = lane; c < n; c += 32) { const double x = a[c], y = b[c]; s[0] += x * x; s[1] += x * y; s[2] += y * y; }
    };
    const size_t ra = 2 * (size_t)pt, rb = ra + 1;
    acc(Bf + ra * Nelim, Bf + rb * Nelim, Nelim);
    acc(Bs + ra * N.ldS, Bs + rb * N.ldS, N.n_c);
    acc(Bi + ra * nBi, Bi + rb * nBi, nBi);
    warp_sum(s);
    if(lane == 0) { V[3 * pt] = s[0]; V[3 * pt + 1] = s[1]; V[3 * pt + 2] = s[2]; }
}

// Var = sigma^2 (Var0 - (Jr X)'(Jr X)): one warp per point, lanes over the regularization rows. X lives in Bs / Bi
// (shared unknowns); a regularization entry on an eliminated unknown sets *bad
__global__ void finish_kernel(const NormalBuffers N, const double* __restrict__ Bs, const double* __restrict__ Bi,
                              const int* __restrict__ rowptr, const int* __restrict__ Jcol, const double* __restrict__ Jval,
                              int m0, int m1, int Npts, const double* __restrict__ V, const double* __restrict__ sigma,
                              double* __restrict__ out /*[Npts][2][2]*/, int* __restrict__ bad)
{
    const int pt = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if(pt >= Npts) return;
    double s[3] = {0., 0., 0.};
    for(int m = m0 + lane; m < m1; m += 32)
    {
        double a = 0., b = 0.;
        for(int e = rowptr[m]; e < rowptr[m + 1]; e++)
        {
            const NormalBuffers::Slot sl = N.slot(Jcol[e]);
            if(sl.piece == 0) { *bad = 1; continue; }
            const double xa = *N.at<const double>(sl, nullptr, 0, Bs, Bi, 2 * pt);
            const double xb = *N.at<const double>(sl, nullptr, 0, Bs, Bi, 2 * pt + 1);
            a += Jval[e] * xa; b += Jval[e] * xb;
        }
        s[0] += a * a; s[1] += a * b; s[2] += b * b;
    }
    warp_sum(s);
    if(lane != 0) return;
    const double s2 = sigma[0] * sigma[0];
    const double v00 = (V[3 * pt] - s[0]) * s2, v01 = (V[3 * pt + 1] - s[1]) * s2, v11 = (V[3 * pt + 2] - s[2]) * s2;
    out[4 * pt] = v00; out[4 * pt + 1] = v01; out[4 * pt + 2] = v01; out[4 * pt + 3] = v11;
}

// sigma = sqrt(sum x^2 / Nobs) / sqrt(1 - Nstate/Nobs) over the board and point measurements (model_analysis.py:491-556).
// One CTA, fixed order
__global__ void __launch_bounds__(256) sigma_kernel(const double* __restrict__ x, int m_board0, int Nboard, int m_point0, int Npoint,
                                                    int Nstate, double given, double* __restrict__ sigma)
{
    __shared__ double part[256];
    double s = 0.;
    for(int i = threadIdx.x; i < Nboard; i += 256) s += x[m_board0 + i] * x[m_board0 + i];
    for(int i = threadIdx.x; i < Npoint; i += 256) s += x[m_point0 + i] * x[m_point0 + i];
    tree_sum<256>(part, s);
    if(threadIdx.x == 0)
    {
        const double n = (double)(Nboard + Npoint);
        sigma[0] = given > 0. ? given : sqrt(part[0] / n) / sqrt(1. - (double)Nstate / n);
    }
}

bool launch_rows(const DevProblem& dp, const NormalBuffers& N, const RowArgs& A, const double* pcam, int Npts,
                 double* Bf, double* Bs, double* Bi, double* G, cudaStream_t s)
{
    const unsigned blocks = (unsigned)((Npts + 127) / 128);
    if(!dispatch_lens_kind(dp.lens_kind, [&](auto k)
       { uncertainty_rows_kernel<decltype(k)::value><<<blocks, 128, 0, s>>>(dp, N, A, pcam, Npts, Bf, Bs, Bi, G); }))
        return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// The extrinsics of camera icam as the reference finds them (model_analysis.py:1460-1495): the sorted distinct
// icam_extrinsics of its observations, which must be one camera at the reference or a consecutive block
bool camera_extrinsics(const mrcal_b200_problem* P, int icam, int* e_first, int* Ne)
{
    std::vector<int> e;
    for(size_t o = 0; o < P->h_obs_board.size() / 3; o++) if(P->h_obs_board[3 * o] == icam) e.push_back(P->h_obs_board[3 * o + 1]);
    for(size_t o = 0; o < P->h_obs_point.size() / 3; o++) if(P->h_obs_point[3 * o] == icam) e.push_back(P->h_obs_point[3 * o + 1]);
    std::sort(e.begin(), e.end());
    e.erase(std::unique(e.begin(), e.end()), e.end());
    if(e.empty()) { set_error("No extrinsics corresponding to icam_intrinsics=%d. I don't know what to do", icam); return false; }
    for(size_t k = 1; k < e.size(); k++)
        if(e[k] != e[k - 1] + 1) { set_error("At this point I'm only supporting consecutive block of extrinsics for a given icam_intrinsics"); return false; }
    if(e[0] < 0)
    {
        if(e.size() > 1) { set_error("Have moving camera, some poses are at the reference. This isn't supported yet"); return false; }
        *e_first = -1; *Ne = 0;
        return true;
    }
    *e_first = e[0]; *Ne = (int)e.size();
    return true;
}

// What the reference refuses whatever the camera, for a known method (model_analysis.py:727-734, 1447-1452, 901-902)
bool uncertainty_method_ok(const mrcal_b200_problem* P, int method)
{
    const Layout& L = P->L;
    const DevProblem& dp = P->dp;
    if(dp.Ntri > 0) { set_error("Some measurements other than boards, points and regularization are present. Don't know what to do"); return false; }
    if(L.Nmeas_board + L.Nmeas_point == 0)
    { set_error("observed_pixel_uncertainty cannot be computed because we don't have any board or point observations"); return false; }
    if(L.Nmeas_reg > 0 && L.Nmeas_board + L.Nmeas_point == 0) { set_error("No non-regularization measurements. Don't know what to do"); return false; }
    if(method == MRCAL_B200_UNCERTAINTY_MEAN_PCAM && dp.opt_frames && dp.Nobs_point > 0)
    { set_error("We have point observations that we are optimizing; only cross-reprojection uncertainty can work here. Have method='mean-pcam'"); return false; }
    return true;
}

// One camera's query points: what the reference refuses for it (model_analysis.py:1460-1483), and its extrinsics
struct CameraQuery
{
    int icam, Npts;
    int e_first = -1, Ne = 0;
    size_t p0 = 0;   // its first point among all the cameras' points
};
bool camera_query_ok(const mrcal_b200_problem* P, int method, CameraQuery* Q)
{
    // (ccp does not look at the camera's extrinsics: model_analysis.py:1347-1417 returns before that)
    if(method != MRCAL_B200_UNCERTAINTY_CCP && !camera_extrinsics(P, Q->icam, &Q->e_first, &Q->Ne)) return false;
    if(method == MRCAL_B200_UNCERTAINTY_RRP_JFP && Q->Ne > 1) { set_error("I only handle stationary cameras for now"); return false; }
    return true;
}

// The part every camera shares: the Jacobian at the current state, the structured factor of JtJ, and sigma
struct UncertaintyFactor
{
    mrcal_b200_factorization F;   // its buffers only: it does not own the problem here
    DeviceArena mem;
    double* sigma = nullptr;
    int* bad = nullptr;
    double* K = nullptr;          // [6][Nstate] for the cross-reprojection methods
    int c0K = 0;                  // the first column K can be nonzero in
};
bool uncertainty_factor(mrcal_b200_problem* P, int method, double observed_pixel_uncertainty, UncertaintyFactor* U)
{
    const Layout& L = P->L;
    const DevProblem& dp = P->dp;
    U->F.P = P;
    if(!schur_factor_build(P, &U->F)) return false;
    if(!U->mem.alloc(&U->sigma, 1) || !U->mem.alloc(&U->bad, 1, true)) return false;
    U->c0K = L.Nstate;
    if(method != MRCAL_B200_UNCERTAINTY_MEAN_PCAM)
    {
        if(!U->mem.alloc(&U->K, (size_t)6 * L.Nstate)) return false;
        for(int c : {dp.i_extr0, dp.i_frame0, dp.i_point0, dp.i_warp0}) if(c >= 0 && c < U->c0K) U->c0K = c;
    }
    const EvalBuffers& op = P->op[P->cur];
    sigma_kernel<<<1, 256, 0, P->stream>>>(op.x, L.m_board0, L.Nmeas_board, L.m_point0, L.Nmeas_point, L.Nstate,
                                           observed_pixel_uncertainty, U->sigma);
    return true;
}

// The points in a chunk of the solves: as many as a fixed memory budget holds, at most Npts
int uncertainty_chunk(const UncertaintyFactor& U, const NormalBuffers& N, int Npts)
{
    const size_t per_rhs = (size_t)(U.F.Nelim > 0 ? U.F.Nelim : 1) + N.ldS + (N.n_r > 0 ? N.n_r : 1);
    const size_t budget = (size_t)512 << 20;
    int chunk = (int)(budget / (2 * per_rhs * sizeof(double)));
    chunk = chunk < kSolveTile ? kSolveTile : (chunk / kSolveTile) * kSolveTile;
    return chunk > Npts ? Npts : chunk;
}

// Var of one camera's points pts [Npts][3] (device) into out [Npts][2][2] (device): its rows, the solves and the
// 2x2 reductions, chunk points at a time. Bf .. V hold a chunk
bool uncertainty_camera(mrcal_b200_problem* P, const UncertaintyFactor& U, int method, bool atinfinity,
                        const CameraQuery& Q, const double* pts, double* Bf, double* Bs, double* Bi, double* G,
                        double* V, double* out)
{
    const Layout& L = P->L;
    const DevProblem& dp = P->dp;
    const NormalBuffers N = P->ws->N;
    const int Nelim = U.F.Nelim, nBi = N.n_r, Nstate = L.Nstate;
    const EvalBuffers& op = P->op[P->cur];
    cudaStream_t s = P->stream;
    // K of the cross-reprojection methods (the Jacobian was evaluated by the factorization)
    if(U.K && !cross_reprojection_K(P, method == MRCAL_B200_UNCERTAINTY_CCP ? Q.icam : -1, false, U.K)) return false;

    RowArgs A{};
    A.method = method; A.atinfinity = atinfinity; A.icam = Q.icam; A.e_first = Q.e_first; A.Ne = Q.Ne;
    A.intr_col0 = (dp.i_intr0 >= 0 && dp.Nintr_state > 0) ? dp.i_intr0 + Q.icam * dp.Nintr_state : -1;
    A.intr_arg0 = dp.opt_core ? 0 : 4;
    A.Nelim = Nelim;
    A.scale = P->d_scale;

    const int chunk = uncertainty_chunk(U, N, Q.Npts);
    const bool reg = L.Nmeas_reg > 0;
    for(int p0 = 0; p0 < Q.Npts; p0 += chunk)
    {
        const int np = Q.Npts - p0 < chunk ? Q.Npts - p0 : chunk, nr = 2 * np;
        MB200_CUDA_CHECK(cudaMemsetAsync(Bf, 0, (size_t)nr * (Nelim > 0 ? Nelim : 1) * sizeof(double), s));
        MB200_CUDA_CHECK(cudaMemsetAsync(Bs, 0, (size_t)nr * N.ldS * sizeof(double), s));
        MB200_CUDA_CHECK(cudaMemsetAsync(Bi, 0, (size_t)nr * (nBi > 0 ? nBi : 1) * sizeof(double), s));
        if(!launch_rows(dp, N, A, pts + 3 * (size_t)p0, np, Bf, Bs, Bi, U.K ? G : nullptr, s)) return false;
        if(U.K && U.c0K < Nstate)
        {
            const long tot = (long)nr * (Nstate - U.c0K);
            uncertainty_K_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, s>>>(N, Nelim, G, U.K, Nstate, U.c0K, nr, Bf, Bs, Bi);
        }
        // Z = inv(L) P dF'
        if(!schur_solve_pieces(&U.F, Bf, Bs, Bi, nr, true, BackSolve::none, s)) return false;
        ztz_kernel<<<(unsigned)((np * 32 + 255) / 256), 256, 0, s>>>(N, Bf, Nelim, Bs, Bi, nBi, np, V);
        // X on the shared unknowns = inv(L_S') Z_s, inv(L_I') Z_i
        if(reg && !schur_solve_pieces(&U.F, Bf, Bs, Bi, nr, false, BackSolve::shared, s)) return false;
        finish_kernel<<<(unsigned)((np * 32 + 255) / 256), 256, 0, s>>>(N, Bs, Bi, P->d_rowptr, op.Jcol, op.Jval, L.m_reg0,
                                                                         reg ? L.m_reg0 + L.Nmeas_reg : L.m_reg0, np, V, U.sigma,
                                                                         out + 4 * (size_t)p0, U.bad);
        MB200_CUDA_CHECK(cudaGetLastError());
    }
    return true;
}

// Var of the cameras Q[Ncams] from one factorization: p_cam and Var hold every camera's points, camera after camera
bool uncertainty_cameras(mrcal_b200_problem* P, int method, bool atinfinity, std::vector<CameraQuery>& Q,
                         const mrcal_point3_t* p_cam, double observed_pixel_uncertainty, double* Var, double* sigma_used)
{
    if(method < MRCAL_B200_UNCERTAINTY_MEAN_PCAM || method > MRCAL_B200_UNCERTAINTY_CCP)
    { set_error("Unknown uncertainty method %d", method); return false; }
    for(const CameraQuery& q : Q)
    {
        if(q.icam < 0 || q.icam >= P->dp.Ncam_i) { set_error("icam_intrinsics = %d is out of range", q.icam); return false; }
        if(q.Npts < 0) { set_error("projection_uncertainty: N < 0"); return false; }
    }
    if(!uncertainty_method_ok(P, method)) return false;
    size_t Ntotal = 0;
    for(CameraQuery& q : Q)
    {
        if(!camera_query_ok(P, method, &q)) return false;
        q.p0 = Ntotal;
        Ntotal += (size_t)q.Npts;
    }
    cudaStream_t s = P->stream;
    UncertaintyFactor U;
    if(!uncertainty_factor(P, method, observed_pixel_uncertainty, &U)) return false;
    if(Ntotal > 0)
    {
        const NormalBuffers N = P->ws->N;
        int maxchunk = 0;
        for(const CameraQuery& q : Q) maxchunk = std::max(maxchunk, uncertainty_chunk(U, N, q.Npts));
        const int maxrhs = 2 * maxchunk, Nelim = U.F.Nelim, nBi = N.n_r;
        DeviceArena& mem = U.mem;
        double *Bf, *Bs, *Bi, *G, *pts, *V, *out;
        if(!mem.alloc(&Bf, (size_t)maxrhs * (Nelim > 0 ? Nelim : 1)) || !mem.alloc(&Bs, (size_t)maxrhs * N.ldS) ||
           !mem.alloc(&Bi, (size_t)maxrhs * (nBi > 0 ? nBi : 1)) || !mem.alloc(&G, (size_t)maxrhs * 6) ||
           !mem.alloc(&pts, 3 * Ntotal) || !mem.alloc(&V, (size_t)3 * maxchunk) || !mem.alloc(&out, 4 * Ntotal))
            return false;
        MB200_CUDA_CHECK(cudaMemcpyAsync(pts, p_cam, 3 * Ntotal * sizeof(double), cudaMemcpyHostToDevice, s));
        for(const CameraQuery& q : Q)
            if(q.Npts > 0 && !uncertainty_camera(P, U, method, atinfinity, q, pts + 3 * q.p0, Bf, Bs, Bi, G, V, out + 4 * q.p0))
                return false;
        MB200_CUDA_CHECK(cudaMemcpyAsync(Var, out, 4 * Ntotal * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    int h_bad = 0;
    MB200_CUDA_CHECK(cudaMemcpyAsync(&h_bad, U.bad, sizeof(int), cudaMemcpyDeviceToHost, s));
    if(sigma_used) MB200_CUDA_CHECK(cudaMemcpyAsync(sigma_used, U.sigma, sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    if(h_bad) { set_error("projection_uncertainty: a regularization term touches an eliminated unknown"); return false; }
    return true;
}

}  // namespace
}  // namespace mb200
using namespace mb200;

extern "C" bool mrcal_b200_problem_projection_uncertainty(mrcal_b200_problem_t* P, int icam, int method, bool atinfinity,
                                                          const mrcal_point3_t* p_cam, int Npts, double observed_pixel_uncertainty,
                                                          double* Var, double* sigma_used)
{
    if(mrcal_b200_device_count() <= 0) { set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback"); return false; }
    if(P == nullptr) { set_error("projection_uncertainty: no problem"); return false; }
    std::vector<CameraQuery> Q(1);
    Q[0].icam = icam; Q[0].Npts = Npts;
    return uncertainty_cameras(P, method, atinfinity, Q, p_cam, observed_pixel_uncertainty, Var, sigma_used);
}

extern "C" bool mrcal_b200_problem_observed_pixel_uncertainty(mrcal_b200_problem_t* P, double* sigma)
{
    if(mrcal_b200_device_count() <= 0) { set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback"); return false; }
    if(P == nullptr) { set_error("observed_pixel_uncertainty: no problem"); return false; }
    const Layout& L = P->L;
    if(L.Nmeas_board + L.Nmeas_point == 0)
    { set_error("observed_pixel_uncertainty cannot be computed because we don't have any board or point observations"); return false; }
    DeviceArena mem;
    double* d_sigma;
    if(!mem.alloc(&d_sigma, 1)) return false;
    // the evaluation schur_factor_build() makes, so that the residuals, and sigma, are those projection_uncertainty() uses
    if(!problem_evaluate(P, P->cur, true, true)) return false;
    const EvalBuffers& op = P->op[P->cur];
    sigma_kernel<<<1, 256, 0, P->stream>>>(op.x, L.m_board0, L.Nmeas_board, L.m_point0, L.Nmeas_point, L.Nstate, -1.,
                                           d_sigma);
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpyAsync(sigma, d_sigma, sizeof(double), cudaMemcpyDeviceToHost, P->stream));
    MB200_CUDA_CHECK(cudaStreamSynchronize(P->stream));
    return true;
}

extern "C" bool mrcal_b200_problem_projection_uncertainty_cameras(mrcal_b200_problem_t* P, const int* icam_intrinsics,
                                                                  const int* N, int Ncameras, int method, bool atinfinity,
                                                                  const mrcal_point3_t* p_cam,
                                                                  double observed_pixel_uncertainty, double* Var,
                                                                  double* sigma_used)
{
    if(mrcal_b200_device_count() <= 0) { set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback"); return false; }
    if(P == nullptr) { set_error("projection_uncertainty: no problem"); return false; }
    if(Ncameras < 0) { set_error("projection_uncertainty: Ncameras < 0"); return false; }
    std::vector<CameraQuery> Q(Ncameras);
    for(int c = 0; c < Ncameras; c++) { Q[c].icam = icam_intrinsics[c]; Q[c].Npts = N[c]; }
    return uncertainty_cameras(P, method, atinfinity, Q, p_cam, observed_pixel_uncertainty, Var, sigma_used);
}
