// Kernel family 1: the cost function. residuals x and the block-sparse
// Jacobian dx/db_packed, written in the reference's CSR order.
//
// What these kernels compute is the reference's optimizer_callback()
// (mrcal.c:4444-5970): board rows (:4604-4900), discrete-point rows
// (:4902-5176), regularization rows (:5655-5955). How: the unit of parallel
// work is the board OBSERVATION (one CTA) and the board CORNER (one thread);
// the two Rodrigues rotations of an observation are expanded once per CTA into
// shared memory; each thread evaluates its corner's projection and gradients
// in registers and writes its two fixed-width Jacobian rows. Row positions are
// analytic (fixed nnz per row class), so there is no serial fill pointer.
#include "observation.cuh"
#include "ptx.cuh"
#include "triangulated.cuh"

namespace mb200 {

// b_packed -> unpacked intrinsics / poses / points / warp, falling back to the
// seed values for whatever is not being optimised (mrcal.c:4534-4601)
__global__ void unpack_state_kernel(DevProblem P, const double* __restrict__ b)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int n_intr = P.Ncam_i * P.Nintr;
    const int n_cam  = P.Ncam_e * 6;
    const int n_frm  = P.Nframes * 6;
    const int n_pt   = P.Npoints * 3;
    int i = t;
    if(i < n_intr)
    {
        const int cam = i / P.Nintr, k = i - cam * P.Nintr;
        double v;
        if(k < 4)
        {
            if(P.opt_core) v = b[P.i_intr0 + cam * P.Nintr_state + k] * (k < 2 ? kScaleFocal : kScaleCenter);
            else           v = P.in_intrinsics[i];
        }
        else
        {
            if(P.opt_dist) v = b[P.i_intr0 + cam * P.Nintr_state + P.Ncore_state + (k - 4)] * kScaleDistortion;
            else           v = P.in_intrinsics[i];
        }
        P.u_intr[i] = v;
        return;
    }
    i -= n_intr;
    if(i < n_cam)
    {
        const int k = i % 6;
        P.u_rtcam[i] = P.opt_extr ? b[P.i_extr0 + i] * (k < 3 ? kScaleRotCam : kScaleTransCam) : P.in_rt_cam[i];
        return;
    }
    i -= n_cam;
    if(i < n_frm)
    {
        const int k = i % 6;
        P.u_rtframe[i] = P.opt_frames ? b[P.i_frame0 + i] * (k < 3 ? kScaleRotFrame : kScaleTransFrame) : P.in_rt_frame[i];
        return;
    }
    i -= n_frm;
    if(i < n_pt)
    {
        const int ipt = i / 3;
        P.u_points[i] = (P.opt_frames && ipt < P.Npoints_variable) ? b[P.i_point0 + i] * kScalePoint : P.in_points[i];
        return;
    }
    i -= n_pt;
    if(i < 2)
    {
        if(P.opt_warp)        P.u_warp[i] = b[P.i_warp0 + i] * kScaleWarp;
        else if(P.have_warp)  P.u_warp[i] = P.in_warp[i];
        else                  P.u_warp[i] = 0.;
    }
}

// R and dR/dr of every frame and camera pose, one thread each: the board kernel's CTAs then only
// load 36 doubles instead of one of their threads evaluating sincos and 27 derivatives serially
__global__ void expand_rotations_kernel(DevProblem P)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i < P.Nframes)                  rodrigues(&P.u_rot_frame[36 * i], &P.u_rot_frame[36 * i + 9], &P.u_rtframe[6 * i]);
    else if(i < P.Nframes + P.Ncam_e)  { const int c = i - P.Nframes; rodrigues(&P.u_rot_cam[36 * c], &P.u_rot_cam[36 * c + 9], &P.u_rtcam[6 * c]); }
}

__device__ __forceinline__ double block_sum(double v, double* sh /* >= 32 doubles */)
{
#pragma unroll
    for(int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if(lane == 0) sh[warp] = v;
    __syncthreads();
    if(warp == 0)
    {
        v = lane < (int)((blockDim.x + 31) >> 5) ? sh[lane] : 0.;
#pragma unroll
        for(int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    }
    return v;   // valid in thread 0
}

// Intrinsics part of one measurement row. i_xy selects the x or the y row.
//   g_f      dq_k/df_k (core)
//   ddist    dense distortion gradient of this row (parametric models)
//   wx,wy    spline basis (splined models); ivar0s = knot offset within the STATE block
template <int KIND>
__device__ __forceinline__ int emit_intrinsics(double* __restrict__ jv, int* __restrict__ jc,
                                               const DevProblem& P, int i_var_intr, int i_xy, double w, bool zero,
                                               double g_f, const double* ddist,
                                               const double* wx, const double* wy, int ivar0s, double f_xy)
{
    int n = 0;
    if(P.opt_core)
    {
        if(jc) jc[n] = i_var_intr + i_xy;
        jv[n] = zero ? 0. : g_f * w * kScaleFocal;  n++;
        if(jc) jc[n] = i_var_intr + i_xy + 2;
        jv[n] = zero ? 0. : w * kScaleCenter;       n++;
    }
    if(P.opt_dist)
    {
        if constexpr(LensTraits<KIND>::SPLINED)
        {
            constexpr int RUN = LensTraits<KIND>::RUN;
#pragma unroll
            for(int iy = 0; iy < RUN; iy++)
#pragma unroll
                for(int ix = 0; ix < RUN; ix++)
                {
                    if(jc) jc[n] = i_var_intr + ivar0s + iy * 2 * P.Nx + ix * 2 + i_xy;
                    jv[n] = zero ? 0. : wx[ix] * wy[iy] * f_xy * w * kScaleDistortion;
                    n++;
                }
        }
        else
        {
            constexpr int ND = LensTraits<KIND>::NDIST;
#pragma unroll
            for(int i = 0; i < ND; i++)
            {
                if(jc) jc[n] = i_var_intr + P.Ncore_state + i;
                jv[n] = zero ? 0. : ddist[i] * w * kScaleDistortion;
                n++;
            }
        }
    }
    return n;
}

// One CTA per board observation, one thread per corner (strided if W*H > blockDim)
template <int KIND, bool WITH_J>
__global__ void __maxnreg__(160)   // 3 CTAs of 128 threads per SM
eval_boards_kernel(DevProblem P, double* __restrict__ x, double* __restrict__ Jval, int* __restrict__ Jcol,
                   double* __restrict__ norm2)
{
    __shared__ ObsPoses G;
    __shared__ double red[32];
    __shared__ int s_ivar0[256];   // per corner: where its spline window starts (the only data-dependent column index)
    __shared__ __align__(8) int s_pat[2 * 256]; // per entry of a corner's two rows: its column for a window at 0, and whether the window's
                                   // start adds to it (pattern[2 e], pattern[2 e + 1]): the same for every corner of the view
    // Jacobian staging: each thread (corner) deposits the VALUES of its two rows here -- 2*nnz_row contiguous
    // doubles, which is also how they sit in J -- and hands them to the TMA: one bulk shared->global copy per
    // corner (cp.async.bulk), no thread spends time on the value stores. The column indices are not staged at all:
    // they are a function of (corner, entry) and are written straight from registers, coalesced, a warp per corner.
    // The row stride is 2 (mod 4) doubles: 16-byte aligned for the bulk copy, 2-way bank conflicts at worst
    extern __shared__ __align__(16) double stage_v[];

    const int iobs   = blockIdx.x;
    const int icam_i = P.obs_board[3 * iobs + 0];
    const int icam_e = P.obs_board[3 * iobs + 1];
    const int iframe = P.obs_board[3 * iobs + 2];
    const bool cam_identity = icam_e < 0;

    load_obs_poses(G, P, iframe, icam_e, threadIdx.x);
    __syncthreads();

    const double* __restrict__ intr = &P.u_intr[(size_t)icam_i * P.Nintr];
    const int i_var_intr  = P.i_intr0 + icam_i * P.Nintr_state;
    const int i_var_cam   = P.i_extr0 + 6 * icam_e;
    const int i_var_frame = P.i_frame0 + 6 * iframe;
    const bool emit_cam   = P.opt_extr && !cam_identity;
    const int nnz_row     = P.nnz_row_intr + (emit_cam ? 6 : 0) + P.nnz_row_board_geom;
    const int NWH         = P.W * P.H;
    const double wx2 = P.u_warp[0], wy2 = P.u_warp[1];

    const int row2 = 2 * nnz_row;
    int stride = row2;
    while((stride & 3) != 2) stride++;
    const int nI = P.nnz_row_intr;
    if constexpr(WITH_J)
    {
        // the column pattern of this view's rows (mrcal.c:4575-4760 lay the rows out in this order): once per CTA
        const int ncore = P.opt_core ? 2 : 0;
        for(int e = threadIdx.x; e < row2 && e < 256; e += blockDim.x)
        {
            const int i_xy = e >= nnz_row ? 1 : 0, k = e - i_xy * nnz_row;
            int col, dep = 0;
            if(k < nI)
            {
                if(k < ncore) col = i_var_intr + i_xy + 2 * k;
                else if constexpr(LensTraits<KIND>::SPLINED)
                {
                    constexpr int RUN = LensTraits<KIND>::RUN;
                    const int kk = k - ncore, iy = kk / RUN, ix = kk - iy * RUN;
                    col = i_var_intr + iy * 2 * P.Nx + ix * 2 + i_xy;
                    dep = 1;
                }
                else col = i_var_intr + P.Ncore_state + (k - ncore);
            }
            else
            {
                int kk = k - nI;
                if(emit_cam && kk < 6) col = i_var_cam + kk;
                else
                {
                    if(emit_cam) kk -= 6;
                    if(P.opt_frames && kk < 6) col = i_var_frame + kk;
                    else { if(P.opt_frames) kk -= 6; col = P.i_warp0 + kk; }
                }
            }
            s_pat[2 * e] = col;
            s_pat[2 * e + 1] = dep;
        }
        // (visible to everybody after the barrier that precedes the first use below)
    }

    double sumsq = 0.;
    for(int ipt0 = 0; ipt0 < NWH; ipt0 += blockDim.x)
    {
      const int ipt = ipt0 + threadIdx.x;
      if(ipt < NWH)
      {
        double pt[3], dz[2], v[3], p[3];
        board_corner(pt, dz, v, p, P, G, cam_identity, ipt % P.W, ipt / P.W, wx2, wy2);

        double q[2], dq_dp[2][3];
        double ddist[2][LensTraits<KIND>::NDIST > 0 ? LensTraits<KIND>::NDIST : 1];
        double wx[4], wy[4], upd[2] = {0., 0.};
        int ivar0 = 0;
        if constexpr(LensTraits<KIND>::SPLINED)
            project_splined<LensTraits<KIND>::RUN>(q, dq_dp, wx, wy, &ivar0, upd, p, intr, P.Nx, P.Ny, P.segments_per_u);
        else
            project_parametric<KIND>(q, dq_dp, WITH_J ? ddist : nullptr, p, intr, P.lens_cfg);

        const size_t ifeat = (size_t)iobs * NWH + ipt;
        const double qx_obs = P.obs_board_pool[3 * ifeat + 0];
        const double qy_obs = P.obs_board_pool[3 * ifeat + 1];
        const double w      = P.obs_board_pool[3 * ifeat + 2];
        const bool outlier  = !(w >= 0.0);   // mrcal.c:4695
        const double e0 = outlier ? 0. : (q[0] - qx_obs) * w;
        const double e1 = outlier ? 0. : (q[1] - qy_obs) * w;
        x[2 * ifeat + 0] = e0;
        x[2 * ifeat + 1] = e1;
        sumsq += e0 * e0 + e1 * e1;

        if constexpr(WITH_J)
        {
            // G2 = dq/dv : gradient wrt the point in reference coords
            double G2[2][3];
            if(cam_identity)
            {
#pragma unroll
                for(int k = 0; k < 2; k++) { G2[k][0] = dq_dp[k][0]; G2[k][1] = dq_dp[k][1]; G2[k][2] = dq_dp[k][2]; }
            }
            else
            {
#pragma unroll
                for(int k = 0; k < 2; k++)
#pragma unroll
                    for(int j = 0; j < 3; j++)
                        G2[k][j] = dq_dp[k][0] * G.Rc[j] + dq_dp[k][1] * G.Rc[3 + j] + dq_dp[k][2] * G.Rc[6 + j];
            }
            // frame rotation: dv/drf_k = dRf[k] pt
            double dq_drf[2][3], dq_drc[2][3];
            if(P.opt_frames)
            {
#pragma unroll
                for(int k = 0; k < 3; k++)
                {
                    double dv[3];
                    mat3_vec(dv, &G.dRf[9 * k], pt);
                    dq_drf[0][k] = G2[0][0] * dv[0] + G2[0][1] * dv[1] + G2[0][2] * dv[2];
                    dq_drf[1][k] = G2[1][0] * dv[0] + G2[1][1] * dv[1] + G2[1][2] * dv[2];
                }
            }
            if(emit_cam)
            {
#pragma unroll
                for(int k = 0; k < 3; k++)
                {
                    double dp[3];
                    mat3_vec(dp, &G.dRc[9 * k], v);
                    dq_drc[0][k] = dq_dp[0][0] * dp[0] + dq_dp[0][1] * dp[1] + dq_dp[0][2] * dp[2];
                    dq_drc[1][k] = dq_dp[1][0] * dp[0] + dq_dp[1][1] * dp[1] + dq_dp[1][2] * dp[2];
                }
            }
            // warp: dpt_z/dwarp_i = dz[i], and d v/d pt_z = Rf[:,2]  (mrcal.c:2529-2558)
            double dq_dz[2];
#pragma unroll
            for(int k = 0; k < 2; k++) dq_dz[k] = G2[k][0] * G.Rf[2] + G2[k][1] * G.Rf[5] + G2[k][2] * G.Rf[8];

            const int ivar0s = ivar0 - (P.opt_core ? 0 : 4);
#pragma unroll
            for(int i_xy = 0; i_xy < 2; i_xy++)
            {
                double* jv = stage_v + (size_t)threadIdx.x * stride + i_xy * nnz_row;
                int*    jc = nullptr;
                double g_f;
                if constexpr(LensTraits<KIND>::SPLINED) g_f = upd[i_xy];
                else                                    g_f = (q[i_xy] - intr[2 + i_xy]) / intr[i_xy];   // mrcal.c:1427-1431
                int n = emit_intrinsics<KIND>(jv, jc, P, i_var_intr, i_xy, w, outlier, g_f, ddist[i_xy], wx, wy, ivar0s, intr[i_xy]);
                if(emit_cam)
                {
#pragma unroll
                    for(int k = 0; k < 3; k++) { jv[n] = outlier ? 0. : dq_drc[i_xy][k] * w * kScaleRotCam;   n++; }
#pragma unroll
                    for(int k = 0; k < 3; k++) { jv[n] = outlier ? 0. : dq_dp[i_xy][k] * w * kScaleTransCam;  n++; }
                }
                if(P.opt_frames)
                {
#pragma unroll
                    for(int k = 0; k < 3; k++) { jv[n] = outlier ? 0. : dq_drf[i_xy][k] * w * kScaleRotFrame; n++; }
#pragma unroll
                    for(int k = 0; k < 3; k++) { jv[n] = outlier ? 0. : G2[i_xy][k] * w * kScaleTransFrame;   n++; }
                }
                if(P.opt_warp)
                {
#pragma unroll
                    for(int k = 0; k < 2; k++) { jv[n] = outlier ? 0. : dq_dz[i_xy] * dz[k] * w * kScaleWarp; n++; }
                }
            }
            s_ivar0[threadIdx.x] = ivar0s;
            // this corner's 2 rows: one bulk copy, shared -> global, issued by the thread that wrote them. The fence makes
            // the generic-proxy writes above visible to the async proxy that reads them
            {
                fence_proxy_async();
                bulk_store(Jval + (size_t)P.board_j0[iobs] + (size_t)ipt * row2, stage_v + (size_t)threadIdx.x * stride, row2 * 8);
                bulk_commit();
            }
        }
      }
      if constexpr(WITH_J)
      {
        // the column indices of this chunk of corners: a warp per corner, a lane per entry (coalesced stores): the view's
        // pattern plus, for the entries of the spline window, where this corner's window starts
        __syncthreads();
        const int nhere = min((int)blockDim.x, NWH - ipt0);
        const size_t gbase = (size_t)P.board_j0[iobs] + (size_t)ipt0 * row2;
        const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
        for(int t = wib; t < nhere; t += nwarps)
        {
            const int iv0 = s_ivar0[t];
            for(int e = lane; e < row2; e += 32)
            {
                const int2 pd = *reinterpret_cast<const int2*>(&s_pat[2 * e]);
                Jcol[gbase + (size_t)t * row2 + e] = pd.x + (pd.y ? iv0 : 0);
            }
        }
        // the staging buffer is reused by the next chunk of corners: wait until the TMA has READ it
        bulk_wait_read();
        __syncthreads();
      }
    }
    const double s = block_sum(sumsq, red);
    if(threadIdx.x == 0 && s != 0.) atomicAdd(norm2, s);
}

// One thread per discrete-point observation (two rows). mrcal.c:4902-5176
template <int KIND, bool WITH_J>
__global__ void __launch_bounds__(128)
eval_points_kernel(DevProblem P, double* __restrict__ x, double* __restrict__ Jval, int* __restrict__ Jcol,
                   double* __restrict__ norm2)
{
    __shared__ double red[32];
    const int iobs = blockIdx.x * blockDim.x + threadIdx.x;
    double sumsq = 0.;
    if(iobs < P.Nobs_point)
    {
        const int icam_i  = P.obs_point[3 * iobs + 0];
        const int icam_e  = P.obs_point[3 * iobs + 1];
        const int i_point = P.obs_point[3 * iobs + 2];
        const bool cam_identity = icam_e < 0;
        const bool point_in_state = P.opt_frames && i_point < P.Npoints_variable;
        const bool emit_cam = P.opt_extr && !cam_identity;
        const double* __restrict__ intr = &P.u_intr[(size_t)icam_i * P.Nintr];
        const int i_var_intr  = P.i_intr0 + icam_i * P.Nintr_state;
        const int i_var_cam   = P.i_extr0 + 6 * icam_e;
        const int i_var_point = P.i_point0 + 3 * i_point;
        const int nnz_row = P.nnz_row_intr + (emit_cam ? 6 : 0) + (point_in_state ? 3 : 0);

        const double w = P.obs_point_pool[3 * iobs + 2];
        const bool outlier = w <= 0.0;   // mrcal.c:4918 (note: <=, unlike boards)
        const int m = P.m_point0 + 2 * iobs;

        double q[2] = {0., 0.}, dq_dp[2][3] = {};
        double ddist[2][LensTraits<KIND>::NDIST > 0 ? LensTraits<KIND>::NDIST : 1] = {};
        double wx[4] = {}, wy[4] = {}, upd[2] = {0., 0.};
        double Rc[9], dRc[27], pr[3] = {0., 0., 0.};
        int ivar0 = 4;   // outliers name the first control points (mrcal.c:4965-4975)
        if(!outlier)
        {
            pr[0] = P.u_points[3 * i_point + 0];
            pr[1] = P.u_points[3 * i_point + 1];
            pr[2] = P.u_points[3 * i_point + 2];
            double p[3] = {pr[0], pr[1], pr[2]};
            if(!cam_identity)
            {
                const double* rt = &P.u_rtcam[6 * icam_e];
                rodrigues(Rc, WITH_J ? dRc : nullptr, rt);
                mat3_vec(p, Rc, pr);
                p[0] += rt[3]; p[1] += rt[4]; p[2] += rt[5];
            }
            if constexpr(LensTraits<KIND>::SPLINED)
                project_splined<LensTraits<KIND>::RUN>(q, dq_dp, wx, wy, &ivar0, upd, p, intr, P.Nx, P.Ny, P.segments_per_u);
            else
                project_parametric<KIND>(q, dq_dp, WITH_J ? ddist : nullptr, p, intr, P.lens_cfg);
        }
        const double e0 = outlier ? 0. : (q[0] - P.obs_point_pool[3 * iobs + 0]) * w;
        const double e1 = outlier ? 0. : (q[1] - P.obs_point_pool[3 * iobs + 1]) * w;
        x[m + 0] = e0;
        x[m + 1] = e1;
        sumsq = e0 * e0 + e1 * e1;

        if constexpr(WITH_J)
        {
            const int ivar0s = ivar0 - (P.opt_core ? 0 : 4);
            const size_t jbase = (size_t)P.point_j0[iobs];
#pragma unroll
            for(int i_xy = 0; i_xy < 2; i_xy++)
            {
                double* jv = Jval + jbase + (size_t)i_xy * nnz_row;
                int*    jc = Jcol + jbase + (size_t)i_xy * nnz_row;
                double g_f = 0.;
                if(!outlier)
                {
                    if constexpr(LensTraits<KIND>::SPLINED) g_f = upd[i_xy];
                    else                                    g_f = (q[i_xy] - intr[2 + i_xy]) / intr[i_xy];
                }
                int n;
                if(outlier && LensTraits<KIND>::SPLINED)
                {
                    // structural zeros at the first RUN*RUN distortion columns, contiguous (mrcal.c:4960-4976)
                    n = 0;
                    if(P.opt_core)
                    {
                        jc[n] = i_var_intr + i_xy;     jv[n] = 0.; n++;
                        jc[n] = i_var_intr + i_xy + 2; jv[n] = 0.; n++;
                    }
                    if(P.opt_dist)
                        for(int i = 0; i < LensTraits<KIND>::RUN * LensTraits<KIND>::RUN; i++)
                        { jc[n] = i_var_intr + P.Ncore_state + i; jv[n] = 0.; n++; }
                }
                else
                    n = emit_intrinsics<KIND>(jv, jc, P, i_var_intr, i_xy, w, outlier, g_f, ddist[i_xy], wx, wy, ivar0s, intr[i_xy]);
                if(emit_cam)
                {
#pragma unroll
                    for(int k = 0; k < 3; k++)
                    {
                        double val = 0.;
                        if(!outlier)
                        {
                            double dp[3];
                            mat3_vec(dp, &dRc[9 * k], pr);
                            val = (dq_dp[i_xy][0] * dp[0] + dq_dp[i_xy][1] * dp[1] + dq_dp[i_xy][2] * dp[2]) * w * kScaleRotCam;
                        }
                        jc[n] = i_var_cam + k; jv[n] = val; n++;
                    }
#pragma unroll
                    for(int k = 0; k < 3; k++) { jc[n] = i_var_cam + 3 + k; jv[n] = outlier ? 0. : dq_dp[i_xy][k] * w * kScaleTransCam; n++; }
                }
                if(point_in_state)
                {
#pragma unroll
                    for(int k = 0; k < 3; k++)
                    {
                        double val = 0.;
                        if(!outlier)
                        {
                            if(cam_identity) val = dq_dp[i_xy][k];
                            else             val = dq_dp[i_xy][0] * Rc[k] + dq_dp[i_xy][1] * Rc[3 + k] + dq_dp[i_xy][2] * Rc[6 + k];
                            val *= w * kScalePoint;
                        }
                        jc[n] = i_var_point + k; jv[n] = val; n++;
                    }
                }
            }
        }
    }
    const double s = block_sum(sumsq, red);
    if(threadIdx.x == 0 && s != 0.) atomicAdd(norm2, s);
}

// Regularization rows, one thread each. mrcal.c:5655-5955
template <bool WITH_J>
__global__ void __launch_bounds__(128)
eval_regularization_kernel(DevProblem P, bool splined, double* __restrict__ x, double* __restrict__ Jval,
                           int* __restrict__ Jcol, double* __restrict__ norm2)
{
    __shared__ double red[32];
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    const int Ndist_rows = P.Nreg_dist, Ncenter_rows = P.Nreg_center, Nunity_rows = P.Nreg_unity;
    const double nominal_pixel_error = 0.1;
    double err = 0.;
    if(t < Ndist_rows)
    {
        const int m = P.m_reg0 + t;
        if(splined)
        {
            // per knot: a radial row then a (10x heavier) tangential row (:5709-5786)
            const double scale = nominal_pixel_error / 10.0;
            const int per_cam = P.Ndist_state;
            const int cam = t / per_cam, r = t - cam * per_cam;
            const int knot = r >> 1, which = r & 1;
            const int iy = knot / P.Nx, ix = knot - iy * P.Nx;
            const double* d = &P.u_intr[(size_t)cam * P.Nintr + 4 + 2 * knot];
            double ux = (double)(2 * ix - P.Nx + 1), uy = (double)(2 * iy - P.Ny + 1);
            bool anisotropic = true;
            if(2 * ix == P.Nx - 1 && 2 * iy == P.Ny - 1) { ux = 1.0; anisotropic = false; }
            else { const double mag = sqrt(ux * ux + uy * uy); ux /= mag; uy /= mag; }
            const int col = P.i_intr0 + cam * P.Nintr_state + P.Ncore_state + 2 * knot;
            double g0, g1;
            if(which == 0) { err = scale * (d[0] * ux + d[1] * uy); g0 = scale * ux; g1 = scale * uy; }
            else
            {
                const double extra = anisotropic ? 10. : 1.;
                err = scale * extra * (d[0] * uy - d[1] * ux);
                g0 = scale * extra * uy; g1 = -scale * extra * ux;
            }
            x[m] = err;
            if constexpr(WITH_J)
            {
                const size_t j = reg_row_j0(P, true, t);
                Jcol[j] = col;     Jval[j]     = g0 * kScaleDistortion;
                Jcol[j + 1] = col + 1; Jval[j + 1] = g1 * kScaleDistortion;
            }
        }
        else
        {
            // L2 on each distortion; the rational denominator terms of OPENCV8+ 5x heavier (:5787-5850)
            const double scale = nominal_pixel_error / 1.0;
            const int per_cam = P.Ndist_state;
            const int cam = t / per_cam, j = t - cam * per_cam;
            const double scale_here = (P.opencv8plus && 5 <= j && j <= 7) ? scale * 5. : scale;
            err = scale_here * P.u_intr[(size_t)cam * P.Nintr + 4 + j];
            x[m] = err;
            if constexpr(WITH_J)
            {
                const size_t jj = reg_row_j0(P, false, t);
                Jcol[jj] = P.i_intr0 + cam * P.Nintr_state + P.Ncore_state + j;
                Jval[jj] = scale_here * kScaleDistortion;
            }
        }
    }
    else if(t < Ndist_rows + Ncenter_rows)
    {
        // optical centre near the middle of the imager (:5853-5901). The scale is
        // derived from camera 0's width for every camera, as in the reference
        const int r = t - Ndist_rows;
        const int cam = r >> 1, k = r & 1;
        const double scale = nominal_pixel_error / ((double)P.imagersizes[0] * 0.1);
        const double target = 0.5 * (double)(P.imagersizes[2 * cam + k] - 1);
        err = scale * (P.u_intr[(size_t)cam * P.Nintr + 2 + k] - target);
        x[P.m_reg0 + t] = err;
        if constexpr(WITH_J)
        {
            const size_t jj = reg_row_j0(P, splined, t);
            Jcol[jj] = P.i_intr0 + cam * P.Nintr_state + 2 + k;
            Jval[jj] = scale * kScaleCenter;
        }
    }
    else if(t < Ndist_rows + Ncenter_rows + Nunity_rows)
    {
        // |t_cam0|^2 -> 1 (:5903-5954)
        const double scale = nominal_pixel_error / 0.01;
        const double* tt = &P.u_rtcam[3];
        err = scale * (tt[0] * tt[0] + tt[1] * tt[1] + tt[2] * tt[2] - 1.);
        x[P.m_reg0 + t] = err;
        if constexpr(WITH_J)
        {
            const size_t jj = reg_row_j0(P, splined, t);
            for(int i = 0; i < 3; i++)
            {
                Jcol[jj + i] = P.i_extr0 + 3 + i;
                Jval[jj + i] = scale * kScaleTransCam * 2. * tt[i];
            }
        }
    }
    const double s = block_sum(err * err, red);
    if(threadIdx.x == 0 && s != 0. && P.reg_owner) atomicAdd(norm2, s);
}

// One thread per triangulated measurement = per pair (i0 < i1) of observations of the same point
// (mrcal.c:5180-5653). The point has no state: the rows depend on the extrinsics of the two cameras only.
//   v0_ref = R_0r' v0,  t_r0 = -R_0r' t_0r        (camera 0 -> reference)
//   v0_cam1 = R_1r v0_ref,  t_10 = R_1r t_r0 + t_1r
//   x = err(v1, v0_cam1, t_10)
// Row layout as the reference writes it: [r_0r, t_0r] if camera 0 has extrinsics, then [r_1r, t_1r] likewise.
template <bool WITH_J>
__global__ void __launch_bounds__(128)
eval_triangulated_kernel(DevProblem P, double* __restrict__ x, double* __restrict__ Jval, int* __restrict__ Jcol,
                         double* __restrict__ norm2)
{
    __shared__ double red[32];
    const int ip = blockIdx.x * blockDim.x + threadIdx.x;
    double sumsq = 0.;
    if(ip < P.Ntri)
    {
        const int i0 = P.tri_pairs[2 * ip], i1 = P.tri_pairs[2 * ip + 1];
        const int e0 = P.tri_cam_e[i0], e1 = P.tri_cam_e[i1];
        const bool outlier = P.tri_outlier[i0] || P.tri_outlier[i1];
        double err = 0.;
        double J0[6] = {}, J1[6] = {};
        if(!outlier)
        {
            const double* v0 = &P.tri_px[3 * i0];
            const double* v1 = &P.tri_px[3 * i1];
            double R0[9], dR0[27], R1[9], dR1[27];
            double v0_ref[3], t_r0[3] = {0., 0., 0.}, v0_cam1[3], t_10[3];
            const double* rt0 = e0 >= 0 ? &P.u_rtcam[6 * e0] : nullptr;
            const double* rt1 = e1 >= 0 ? &P.u_rtcam[6 * e1] : nullptr;
            if(rt0)
            {
                rodrigues(R0, WITH_J ? dR0 : nullptr, rt0);
#pragma unroll
                for(int c = 0; c < 3; c++)
                {
                    v0_ref[c] = R0[c] * v0[0] + R0[3 + c] * v0[1] + R0[6 + c] * v0[2];
                    t_r0[c] = -(R0[c] * rt0[3] + R0[3 + c] * rt0[4] + R0[6 + c] * rt0[5]);
                }
            }
            else
                for(int c = 0; c < 3; c++) v0_ref[c] = v0[c];
            if(rt1)
            {
                rodrigues(R1, WITH_J ? dR1 : nullptr, rt1);
                mat3_vec(v0_cam1, R1, v0_ref);
                mat3_vec(t_10, R1, t_r0);
                t_10[0] += rt1[3]; t_10[1] += rt1[4]; t_10[2] += rt1[5];
            }
            else
                for(int c = 0; c < 3; c++) { v0_cam1[c] = v0_ref[c]; t_10[c] = t_r0[c]; }

            double g_v[3], g_t[3];
            err = triangulated_error(g_v, g_t, v1, v0_cam1, t_10);
            if constexpr(WITH_J)
            {
                // gradients pulled back to the reference frame: R_1r' g  (R_1r = I for a camera at the reference)
                double gv_ref[3], gt_ref[3];
                for(int c = 0; c < 3; c++)
                {
                    gv_ref[c] = rt1 ? R1[c] * g_v[0] + R1[3 + c] * g_v[1] + R1[6 + c] * g_v[2] : g_v[c];
                    gt_ref[c] = rt1 ? R1[c] * g_t[0] + R1[3 + c] * g_t[1] + R1[6 + c] * g_t[2] : g_t[c];
                }
                if(rt0)
                {
                    for(int k = 0; k < 3; k++)
                    {
                        // d v0_ref / d r_k = dR0_k' v0 ; d t_r0 / d r_k = -dR0_k' t_0r
                        const double* D = &dR0[9 * k];
                        double acc = 0.;
                        for(int c = 0; c < 3; c++)
                        {
                            const double dv = D[c] * v0[0] + D[3 + c] * v0[1] + D[6 + c] * v0[2];
                            const double dt = -(D[c] * rt0[3] + D[3 + c] * rt0[4] + D[6 + c] * rt0[5]);
                            acc += gv_ref[c] * dv + gt_ref[c] * dt;
                        }
                        J0[k] = acc * kScaleRotCam;
                        // d t_r0 / d t_0r = -R0'  ->  derr/dt_0r[k] = -sum_c gt_ref[c] R0[k][c]
                        J0[3 + k] = -(R0[3 * k] * gt_ref[0] + R0[3 * k + 1] * gt_ref[1] + R0[3 * k + 2] * gt_ref[2]) * kScaleTransCam;
                    }
                }
                if(rt1)
                {
                    for(int k = 0; k < 3; k++)
                    {
                        double dv[3], dt[3];
                        mat3_vec(dv, &dR1[9 * k], v0_ref);
                        mat3_vec(dt, &dR1[9 * k], t_r0);
                        J1[k] = (g_v[0] * dv[0] + g_v[1] * dv[1] + g_v[2] * dv[2] + g_t[0] * dt[0] + g_t[1] * dt[1] + g_t[2] * dt[2]) * kScaleRotCam;
                        J1[3 + k] = g_t[k] * kScaleTransCam;
                    }
                }
            }
        }
        x[P.m_tri0 + ip] = err;
        sumsq = err * err;
        if constexpr(WITH_J)
        {
            int j = P.tri_j0[ip];
            if(e0 >= 0) for(int k = 0; k < 6; k++) { Jcol[j] = P.i_extr0 + 6 * e0 + k; Jval[j] = J0[k]; j++; }
            if(e1 >= 0) for(int k = 0; k < 6; k++) { Jcol[j] = P.i_extr0 + 6 * e1 + k; Jval[j] = J1[k]; j++; }
        }
    }
    const double s = block_sum(sumsq, red);
    if(threadIdx.x == 0 && s != 0.) atomicAdd(norm2, s);
}

// CSR row pointers. Analytic: every row of an observation has the same width
__global__ void fill_rowptr_kernel(DevProblem P, bool splined, int nnz_total, int* __restrict__ rowptr)
{
    const int m = blockIdx.x * blockDim.x + threadIdx.x;
    if(m > P.Nmeas) return;
    if(m == P.Nmeas) { rowptr[m] = nnz_total; return; }
    if(m < P.m_point0)
    {
        const int per_obs = 2 * P.W * P.H;
        const int iobs = m / per_obs, r = m - iobs * per_obs;
        const int j0 = P.board_j0[iobs], j1 = P.board_j0[iobs + 1];
        rowptr[m] = j0 + r * ((j1 - j0) / per_obs);
    }
    else if(m < P.m_tri0)
    {
        const int r = m - P.m_point0;
        const int iobs = r >> 1;
        const int j0 = P.point_j0[iobs], j1 = P.point_j0[iobs + 1];
        rowptr[m] = j0 + (r & 1) * ((j1 - j0) / 2);
    }
    else if(m < P.m_reg0)
        rowptr[m] = P.tri_j0[m - P.m_tri0];
    else
        rowptr[m] = reg_row_j0(P, splined, m - P.m_reg0);
}

template <int KIND>
static bool launch_kind(const DevProblem& dp, const EvalBuffers& out, bool with_j, cudaStream_t stream, int* nlaunch, bool boards)
{
    if(dp.Nobs_board > 0 && boards)
    {
        int threads = ((dp.W * dp.H + 31) / 32) * 32;
        if(threads > 256) threads = 256;
        if(threads < 128) threads = 128;
        if(with_j)
        {
            // widest row: extrinsics present
            const int row2 = 2 * (dp.nnz_row_intr + (dp.opt_extr ? 6 : 0) + dp.nnz_row_board_geom);
            int stride = row2;
            while((stride & 3) != 2) stride++;
            const size_t smem = (size_t)threads * stride * sizeof(double) + 16;
            if(!set_max_dynamic_smem<eval_boards_kernel<KIND, true>>(200 * 1024)) return false;
            if(smem > 200 * 1024) { set_error("Jacobian rows of %d entries are too wide for the staging buffer", row2 / 2); return false; }
            eval_boards_kernel<KIND, true ><<<dp.Nobs_board, threads, smem, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        }
        else
            eval_boards_kernel<KIND, false><<<dp.Nobs_board, threads, 0, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        (*nlaunch)++;
        MB200_CUDA_CHECK(cudaGetLastError());
    }
    if(dp.Nobs_point > 0)
    {
        const int threads = 128, blocks = (dp.Nobs_point + threads - 1) / threads;
        if(with_j) eval_points_kernel<KIND, true ><<<blocks, threads, 0, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        else       eval_points_kernel<KIND, false><<<blocks, threads, 0, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        (*nlaunch)++;
    }
    return true;
}

bool launch_unpack_state(const DevProblem& dp, const double* b_packed, cudaStream_t stream, int* nlaunch)
{
    const int n = dp.Ncam_i * dp.Nintr + dp.Ncam_e * 6 + dp.Nframes * 6 + dp.Npoints * 3 + 2;
    unpack_state_kernel<<<(n + 255) / 256, 256, 0, stream>>>(dp, b_packed);
    if(nlaunch) (*nlaunch)++;
    if(dp.Nframes + dp.Ncam_e > 0 && dp.Nobs_board > 0)
    {
        expand_rotations_kernel<<<(dp.Nframes + dp.Ncam_e + 127) / 128, 128, 0, stream>>>(dp);
        if(nlaunch) (*nlaunch)++;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// boards = false: everything but the board observations (the fused evaluation of fused_eval.cu does those, and has
// already unpacked the state and started |x|^2)
bool launch_evaluate(const DevProblem& dp, const EvalBuffers& out, bool with_jacobian,
                     int* Jrowptr, cudaStream_t stream, int* nlaunch, bool boards)
{
    int dummy = 0;
    if(nlaunch == nullptr) nlaunch = &dummy;
    if(boards)
    {
        MB200_CUDA_CHECK(cudaMemsetAsync(out.norm2, 0, sizeof(double), stream));
        if(!launch_unpack_state(dp, out.p, stream, nlaunch)) return false;
    }
    switch(dp.lens_kind)
    {
    case LENS_PINHOLE:       if(!launch_kind<LENS_PINHOLE>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_STEREOGRAPHIC: if(!launch_kind<LENS_STEREOGRAPHIC>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_LONLAT:        if(!launch_kind<LENS_LONLAT>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_LATLON:        if(!launch_kind<LENS_LATLON>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_OPENCV4:       if(!launch_kind<LENS_OPENCV4>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_OPENCV5:       if(!launch_kind<LENS_OPENCV5>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_OPENCV8:       if(!launch_kind<LENS_OPENCV8>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_OPENCV12:      if(!launch_kind<LENS_OPENCV12>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_SPLINED3:      if(!launch_kind<LENS_SPLINED3>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_SPLINED2:      if(!launch_kind<LENS_SPLINED2>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_CAHVOR:        if(!launch_kind<LENS_CAHVOR>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    case LENS_CAHVORE:       if(!launch_kind<LENS_CAHVORE>(dp, out, with_jacobian, stream, nlaunch, boards)) return false; break;
    default: set_error("lens model kind %d has no CUDA implementation", dp.lens_kind); return false;
    }
    if(dp.Ntri > 0)
    {
        const int threads = 128, blocks = (dp.Ntri + threads - 1) / threads;
        if(with_jacobian) eval_triangulated_kernel<true ><<<blocks, threads, 0, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        else              eval_triangulated_kernel<false><<<blocks, threads, 0, stream>>>(dp, out.x, out.Jval, out.Jcol, out.norm2);
        (*nlaunch)++;
    }
    const bool splined = dp.lens_kind == LENS_SPLINED3 || dp.lens_kind == LENS_SPLINED2;
    const int Nreg = dp.Nmeas - dp.m_reg0;
    if(Nreg > 0)
    {
        const int threads = 128, blocks = (Nreg + threads - 1) / threads;
        if(with_jacobian) eval_regularization_kernel<true ><<<blocks, threads, 0, stream>>>(dp, splined, out.x, out.Jval, out.Jcol, out.norm2);
        else              eval_regularization_kernel<false><<<blocks, threads, 0, stream>>>(dp, splined, out.x, out.Jval, out.Jcol, out.norm2);
        (*nlaunch)++;
    }
    if(Jrowptr != nullptr)
    {
        fill_rowptr_kernel<<<(dp.Nmeas + 1 + 255) / 256, 256, 0, stream>>>(dp, splined, reg_nnz_total(dp, splined), Jrowptr);
        (*nlaunch)++;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// development / test aid (not in the public header): the triangulated-point error function on its own
__global__ void debug_triangulated_error_kernel(const double* __restrict__ in, int N, double* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= N) return;
    double g_v[3], g_t[3];
    // in: v0 (the ray without gradient), v1, t01 -- the reference's argument names (triangulation.cc:960-975)
    const double err = triangulated_error(g_v, g_t, &in[9 * i], &in[9 * i + 3], &in[9 * i + 6]);
    out[7 * i] = err;
    for(int k = 0; k < 3; k++) { out[7 * i + 1 + k] = g_v[k]; out[7 * i + 4 + k] = g_t[k]; }
}

}  // namespace mb200

extern "C" bool mrcal_b200_debug_triangulated_error(const double* v0_v1_t01 /*[N][9]*/, int N, double* err_dv1_dt01 /*[N][7]*/)
{
    double *d_in = nullptr, *d_out = nullptr;
    bool ok = cudaMalloc(&d_in, (size_t)N * 9 * sizeof(double)) == cudaSuccess && cudaMalloc(&d_out, (size_t)N * 7 * sizeof(double)) == cudaSuccess &&
              cudaMemcpy(d_in, v0_v1_t01, (size_t)N * 9 * sizeof(double), cudaMemcpyHostToDevice) == cudaSuccess;
    if(ok)
    {
        mb200::debug_triangulated_error_kernel<<<(N + 127) / 128, 128>>>(d_in, N, d_out);
        ok = cudaMemcpy(err_dv1_dt01, d_out, (size_t)N * 7 * sizeof(double), cudaMemcpyDeviceToHost) == cudaSuccess;
    }
    if(!ok) mb200::set_error("debug_triangulated_error: %s", cudaGetErrorString(cudaGetLastError()));
    cudaFree(d_in); cudaFree(d_out);
    return ok;
}
