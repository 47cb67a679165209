// K = drt_ref_refperturbed/db_packed (icam_intrinsics < 0: "rrp") or drt_cam_camperturbed/db_packed for one camera
// (icam_intrinsics >= 0: "ccp"): the reference's _mrcal_drt_cross_reprojection__dbpacked() (uncertainty.c:798-1577,
// called from mrcal.drt_cross_reprojection__dbpacked(), mrcal-pywrap.c:2016-2110), the heart of its cross-reprojection
// uncertainty method (mrcal/model_analysis.py:1379,1441):
//
//     K = -inv(Jcross' Jcross) Jcross' J_packed[extrinsics | frames | points | calobject_warp]        shape (6, Nstate)
//
// where every measurement row contributes  jcross = j_this Dinv M_this : "this" is the frame the row sees (rrp; or ccp
// for a camera at the reference), its point, or (ccp) the camera's extrinsics;  M_this = d compose(tiny, this)/d tiny.
//
// The reference walks the rows of J one after the other, cutting them into runs with the same (camera, frame, point).
// Here the unit is the OBSERVATION (a board view: 2 W H rows; a point view: 2 rows), one warp each:
//   1. G = sum over its rows of the outer products of the row's "this" block with itself and with the other blocks
//      (frame x frame, frame x warp | point x point | extrinsics x extrinsics, x frame, x point, x warp), straight
//      from the Jacobian the evaluation kernels left on the device (eval.cu) -- the one pass over J;
//   2. everything the reference's accumulate_rt_block()/accumulate_point() (uncertainty.c:132-776) do with a run is
//      LINEAR in G, so it is applied per observation, in matrix form:
//            C_this  = M' Dinv G_this,this      C_thing = M' Dinv G_this,thing      JJ = M' Dinv G Dinv M
//      with M = [dr/dr0 0; -skew(t) I] (poses; dr/dr0 = mrcal_compose_r_tinyr0_gradientr0, poseutils.c:1003) or
//      M = [-skew(p) I] (points), Dinv = the pack scales;
//   3. the columns of K: one thread per frame / point / camera adds the C of its observations IN OBSERVATION ORDER
//      (fixed order: the result does not depend on scheduling), one warp adds JJ and the warp columns;
//   4. 6x6 Cholesky of JJ, K = -inv(JJ) C, per column.
// Accepts what the reference accepts and refuses what it refuses (uncertainty.c:944-989).
#include "device_math.cuh"
#include "pose.cuh"
#include "problem_impl.h"
#include "reduce.cuh"

namespace mb200 {

namespace {

struct ObsOut
{
    int    key_e, key_f, key_p;   // state index of the block the columns belong to, or -1
    int    has_cw;
    double Ce[36], Cf[36], Cp[18], Ccw[12], JJ[21];   // row-major (6 x n); JJ: upper triangle, row-major
};

__device__ __forceinline__ int sym6(int i, int j) { return i <= j ? i * 6 - i * (i - 1) / 2 + (j - i) : j * 6 - j * (j - 1) / 2 + (i - j); }

// M' = [Dr' skew(t); 0 I] applied to a 6 x n block X (row-major, leading dimension n) whose rows were already scaled by
// Dinv: out (6 x n) = M' X
__device__ void apply_Mt_pose(double* out, const double* X, int n, const double Dr[9], const double t[3])
{
    for(int j = 0; j < n; j++)
    {
        const double xr[3] = {X[0 * n + j], X[1 * n + j], X[2 * n + j]};
        const double xt[3] = {X[3 * n + j], X[4 * n + j], X[5 * n + j]};
        // Dr' xr + t x xt
        out[0 * n + j] = Dr[0] * xr[0] + Dr[3] * xr[1] + Dr[6] * xr[2] + (t[1] * xt[2] - t[2] * xt[1]);
        out[1 * n + j] = Dr[1] * xr[0] + Dr[4] * xr[1] + Dr[7] * xr[2] + (t[2] * xt[0] - t[0] * xt[2]);
        out[2 * n + j] = Dr[2] * xr[0] + Dr[5] * xr[1] + Dr[8] * xr[2] + (t[0] * xt[1] - t[1] * xt[0]);
        out[3 * n + j] = xt[0];
        out[4 * n + j] = xt[1];
        out[5 * n + j] = xt[2];
    }
}

// One warp per observation. icam < 0: rrp. Otherwise ccp for camera icam: the other cameras' observations contribute nothing
__global__ void __launch_bounds__(128)
cross_observations_kernel(DevProblem P, const double* __restrict__ b, const double* __restrict__ Jval, int icam, ObsOut* __restrict__ out)
{
    const int o = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if(o >= P.Nobs_board + P.Nobs_point) return;
    const bool board = o < P.Nobs_board;
    const int* idx = board ? &P.obs_board[3 * o] : &P.obs_point[3 * (o - P.Nobs_board)];
    const int icam_i = idx[0], icam_e = idx[1], ithing = idx[2];
    ObsOut* O = &out[o];
    if(lane == 0) { O->key_e = O->key_f = O->key_p = -1; O->has_cw = 0; }
    if(icam >= 0 && icam_i != icam) return;   // (the record stays empty: all keys -1)

    const bool have_e = P.opt_extr && icam_e >= 0;
    const bool have_f = board && P.opt_frames;
    const bool have_p = !board && P.opt_frames && ithing < P.Npoints_variable;
    const bool have_cw = board && P.opt_warp;
    const int ne = have_e ? 6 : 0;
    const int rowlen = P.nnz_row_intr + ne + (board ? P.nnz_row_board_geom : (have_p ? 3 : 0));
    const int Nrows = board ? 2 * P.W * P.H : 2;
    const long j0 = board ? P.board_j0[o] : P.point_j0[o - P.Nobs_board];
    // which block is "this" (uncertainty.c:1290-1310): ccp with extrinsics -> the camera; else the frame / the point
    const bool this_e = icam >= 0 && have_e;
    if(!this_e && !have_f && !have_p) return;

    // ---- 1. the Gram blocks: lane over rows, then a butterfly
    double Gtt[21], Gtf[36], Gtc[12];   // this x this (upper), this x (frame | point), this x warp
    const int nthis = (this_e || have_f) ? 6 : 3;
    const int nsome = this_e ? (have_f ? 6 : (have_p ? 3 : 0)) : 0;
#pragma unroll
    for(int i = 0; i < 21; i++) Gtt[i] = 0.;
#pragma unroll
    for(int i = 0; i < 36; i++) Gtf[i] = 0.;
#pragma unroll
    for(int i = 0; i < 12; i++) Gtc[i] = 0.;
    for(int k = lane; k < Nrows; k += 32)
    {
        const double* row = Jval + j0 + (long)k * rowlen;
        const double* je = row + P.nnz_row_intr;
        const double* jf = je + ne;             // frame (6) or point (3)
        const double* jc = jf + (have_f ? 6 : 0);   // warp (boards only)
        const double* jt = this_e ? je : jf;
        double v[6];
#pragma unroll
        for(int i = 0; i < 6; i++) v[i] = i < nthis ? jt[i] : 0.;
        int q = 0;
#pragma unroll
        for(int i = 0; i < 6; i++)
#pragma unroll
            for(int j = i; j < 6; j++, q++) Gtt[q] += v[i] * v[j];
        if(nsome > 0)
#pragma unroll
            for(int i = 0; i < 6; i++)
#pragma unroll
                for(int j = 0; j < 6; j++)
                    if(j < nsome) Gtf[6 * i + j] += v[i] * jf[j];
        if(have_cw)
#pragma unroll
            for(int i = 0; i < 6; i++) { Gtc[2 * i] += v[i] * jc[0]; Gtc[2 * i + 1] += v[i] * jc[1]; }
    }
    warp_sum(Gtt);
    warp_sum(Gtf);
    warp_sum(Gtc);
    if(lane != 0) return;

    // ---- 2. the transform
    if(nthis == 6)
    {
        const int key = this_e ? P.i_extr0 + 6 * icam_e : P.i_frame0 + 6 * ithing;
        const double sr = this_e ? kScaleRotCam : kScaleRotFrame, st = this_e ? kScaleTransCam : kScaleTransFrame;
        const double r[3] = {b[key] * sr, b[key + 1] * sr, b[key + 2] * sr};
        const double t[3] = {b[key + 3] * st, b[key + 4] * st, b[key + 5] * st};
        double Dr[9];
        compose_r_tinyr0_gradient(Dr, r);
        const double dinv[6] = {1. / sr, 1. / sr, 1. / sr, 1. / st, 1. / st, 1. / st};
        double X[36], Cthis[36];
        for(int i = 0; i < 6; i++)
            for(int j = 0; j < 6; j++) X[6 * i + j] = Gtt[sym6(i, j)] * dinv[i];
        apply_Mt_pose(Cthis, X, 6, Dr, t);
        double* Cdst = this_e ? O->Ce : O->Cf;
        for(int i = 0; i < 36; i++) Cdst[i] = Cthis[i];
        if(this_e) O->key_e = key; else O->key_f = key;
        if(nsome > 0)
        {
            double Xs[36], Cs[36];
            for(int i = 0; i < 6; i++)
                for(int j = 0; j < nsome; j++) Xs[nsome * i + j] = Gtf[6 * i + j] * dinv[i];
            apply_Mt_pose(Cs, Xs, nsome, Dr, t);
            if(nsome == 6) { for(int i = 0; i < 36; i++) O->Cf[i] = Cs[i]; O->key_f = P.i_frame0 + 6 * ithing; }
            else           { for(int i = 0; i < 18; i++) O->Cp[i] = Cs[i]; O->key_p = P.i_point0 + 3 * ithing; }
        }
        if(have_cw)
        {
            double Xc[12], Cc[12];
            for(int i = 0; i < 6; i++) { Xc[2 * i] = Gtc[2 * i] * dinv[i]; Xc[2 * i + 1] = Gtc[2 * i + 1] * dinv[i]; }
            apply_Mt_pose(Cc, Xc, 2, Dr, t);
            for(int i = 0; i < 12; i++) O->Ccw[i] = Cc[i];
            O->has_cw = 1;
        }
        // JJ = Cthis Dinv M,  M = [Dr 0; -skew(t) I]: column j < 3 of (Y M) = Y[:, :3] Dr[:, j] - (Y[:, 3:] skew(t))[:, j]
        for(int i = 0; i < 6; i++)
        {
            const double y[6] = {Cthis[6 * i] * dinv[0], Cthis[6 * i + 1] * dinv[1], Cthis[6 * i + 2] * dinv[2],
                                 Cthis[6 * i + 3] * dinv[3], Cthis[6 * i + 4] * dinv[4], Cthis[6 * i + 5] * dinv[5]};
            // (y_t skew(t))_j = sum_k y_t[k] skew[k][j];  skew = [0 -t2 t1; t2 0 -t0; -t1 t0 0]
            const double ys[3] = {y[4] * t[2] - y[5] * t[1], -y[3] * t[2] + y[5] * t[0], y[3] * t[1] - y[4] * t[0]};
            double rowv[6];
            for(int j = 0; j < 3; j++) rowv[j] = y[0] * Dr[j] + y[1] * Dr[3 + j] + y[2] * Dr[6 + j] - ys[j];
            rowv[3] = y[3]; rowv[4] = y[4]; rowv[5] = y[5];
            for(int j = i; j < 6; j++) O->JJ[sym6(i, j)] = rowv[j];
        }
    }
    else
    {
        // a point: M = [-skew(p) I] (3 x 6), Dinv = 1/scale
        const int key = P.i_point0 + 3 * ithing;
        const double sp = kScalePoint;
        const double p[3] = {b[key] * sp, b[key + 1] * sp, b[key + 2] * sp};
        double G[9];
        for(int i = 0; i < 3; i++)
            for(int j = 0; j < 3; j++) G[3 * i + j] = Gtt[sym6(i, j)] / sp;
        // C (6 x 3) = M' G = [skew(p) G; G]
        double Cp[18];
        for(int j = 0; j < 3; j++)
        {
            const double g[3] = {G[j], G[3 + j], G[6 + j]};
            Cp[0 * 3 + j] = p[1] * g[2] - p[2] * g[1];
            Cp[1 * 3 + j] = p[2] * g[0] - p[0] * g[2];
            Cp[2 * 3 + j] = p[0] * g[1] - p[1] * g[0];
            Cp[3 * 3 + j] = g[0]; Cp[4 * 3 + j] = g[1]; Cp[5 * 3 + j] = g[2];
        }
        for(int i = 0; i < 18; i++) O->Cp[i] = Cp[i];
        O->key_p = key;
        // JJ = C (1/sp) M: columns 0..2 = -(C/sp) skew(p), columns 3..5 = C/sp
        for(int i = 0; i < 6; i++)
        {
            const double y[3] = {Cp[3 * i] / sp, Cp[3 * i + 1] / sp, Cp[3 * i + 2] / sp};
            const double ys[3] = {y[1] * p[2] - y[2] * p[1], -y[0] * p[2] + y[2] * p[0], y[0] * p[1] - y[1] * p[0]};
            const double rowv[6] = {-ys[0], -ys[1], -ys[2], y[0], y[1], y[2]};
            for(int j = i; j < 6; j++) O->JJ[sym6(i, j)] = rowv[j];
        }
    }
}

// The columns of one block of K: thread (blk, e) adds entry e of the C of the observations with that key, in order
__global__ void cross_columns_kernel(const ObsOut* __restrict__ obs, int Nobs, int which /*0 e, 1 f, 2 p*/, int key0, int width, int Nblocks,
                                     double* __restrict__ C /*[6][Nstate]*/, int Nstate)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if(t >= Nblocks * 6 * width) return;
    const int blk = t / (6 * width), e = t - blk * 6 * width, i = e / width, j = e - i * width;
    const int key = key0 + width * blk;
    double s = 0.;
    for(int o = 0; o < Nobs; o++)
    {
        const int k = which == 0 ? obs[o].key_e : which == 1 ? obs[o].key_f : obs[o].key_p;
        if(k != key) continue;
        s += which == 0 ? obs[o].Ce[e] : which == 1 ? obs[o].Cf[e] : obs[o].Cp[e];
    }
    C[(size_t)i * Nstate + key + j] = s;
}
// JJ (21) and the warp columns (12): one thread per value, observations in order
__global__ void cross_totals_kernel(const ObsOut* __restrict__ obs, int Nobs, int i_warp0, double* __restrict__ C, int Nstate, double* __restrict__ JJ)
{
    const int t = threadIdx.x;
    if(blockIdx.x != 0 || t >= 33) return;
    double s = 0.;
    for(int o = 0; o < Nobs; o++)
    {
        if(obs[o].key_e < 0 && obs[o].key_f < 0 && obs[o].key_p < 0) continue;
        if(t < 21) s += obs[o].JJ[t];
        else if(obs[o].has_cw) s += obs[o].Ccw[t - 21];
    }
    if(t < 21) JJ[t] = s;
    else if(i_warp0 >= 0) C[(size_t)((t - 21) / 2) * Nstate + i_warp0 + ((t - 21) & 1)] = s;
}
// K[:, c] = -inv(JJ) C[:, c]: Cholesky of the 6x6 (every thread its own copy), one column per thread. info: 1 = singular
__global__ void cross_solve_kernel(const double* __restrict__ JJ, double* __restrict__ K, int Nstate, int c0, int c1, int* __restrict__ info)
{
    const int c = c0 + blockIdx.x * blockDim.x + threadIdx.x;
    double L[6][6];
    for(int j = 0; j < 6; j++)
    {
        double d = JJ[sym6(j, j)];
        for(int k = 0; k < j; k++) d -= L[j][k] * L[j][k];
        if(!(d > 0.)) { if(c == c0) *info = 1; return; }
        d = sqrt(d);
        L[j][j] = d;
        for(int i = j + 1; i < 6; i++)
        {
            double v = JJ[sym6(i, j)];
            for(int k = 0; k < j; k++) v -= L[i][k] * L[j][k];
            L[i][j] = v / d;
        }
    }
    if(c >= c1) return;
    double x[6];
    for(int i = 0; i < 6; i++) { double v = K[(size_t)i * Nstate + c]; for(int k = 0; k < i; k++) v -= L[i][k] * x[k]; x[i] = v / L[i][i]; }
    for(int i = 5; i >= 0; i--) { double v = x[i]; for(int k = i + 1; k < 6; k++) v -= L[k][i] * x[k]; x[i] = v / L[i][i]; }
    for(int i = 0; i < 6; i++) K[(size_t)i * Nstate + c] = -x[i];
}

}  // namespace

// K into d_K (device, [6][Nstate]), zero outside the extrinsics / frames / points / calobject_warp columns
bool cross_reprojection_K(mrcal_b200_problem* P, int icam_intrinsics, bool evaluate, double* d_K)
{
    const Layout& L = P->L;
    const DevProblem& dp = P->dp;
    if(P->sharded) { set_error("drt_cross_reprojection__dbpacked: not available for sharded problems"); return false; }
    // what the reference refuses (uncertainty.c:944-989, 1189-1197)
    if(dp.i_frame0 >= 0 && dp.i_warp0 >= 0 && dp.i_warp0 != dp.i_frame0 + 6 * dp.Nframes)
    {
        set_error("I assume that the calobject_warp state variables follow the frame state variables immediately");
        return false;
    }
    if(dp.i_frame0 < 0 && dp.i_extr0 < 0)
    {
        set_error("Cross-reprojection uncertainty requires either the extrinsics or the frames/points to be optimized. Otherwise the direct method looking at the intrinsics subset of J works fine");
        return false;
    }
    if(dp.i_warp0 >= 0 && dp.Nobs_point > 0)
    {
        set_error("Unexpected jacobian structure. There's no calobject_warp gradient in measurement %d, but the user asked for it", dp.m_point0);
        return false;
    }
    if(icam_intrinsics >= dp.Ncam_i) { set_error("icam_intrinsics = %d is out of range", icam_intrinsics); return false; }
    if(icam_intrinsics >= 0 && dp.Nintr_state == 0)
    {
        set_error("ERROR: I was asked to report the uncertainty for a given icam_intrinsics, but saw a measurement with unknown icam_intrinsics. The intrinsics are probably fixed, and this implementation can't handle that. Please fix it");
        return false;
    }
    if(dp.Ntri > 0) { set_error("drt_cross_reprojection__dbpacked: triangulated points are not supported (nor are they by the reference)"); return false; }
    cudaStream_t s = P->stream;
    if(evaluate && !problem_evaluate(P, P->cur, true, false)) return false;
    const int Nobs = dp.Nobs_board + dp.Nobs_point, Nstate = L.Nstate;
    if(Nobs == 0) { set_error("no observations"); return false; }
    DeviceArena tmp;
    ObsOut* obs = nullptr;
    double* JJ = nullptr;
    int* info = nullptr;
    if(!tmp.alloc(&obs, (size_t)Nobs) || !tmp.alloc(&JJ, 21, true) || !tmp.alloc(&info, 1, true))
        return false;
    double* K = d_K;
    MB200_CUDA_CHECK(cudaMemsetAsync(K, 0, (size_t)6 * Nstate * sizeof(double), s));
    const EvalBuffers& op = P->op[P->cur];
    cross_observations_kernel<<<(Nobs * 32 + 127) / 128, 128, 0, s>>>(dp, op.p, op.Jval, icam_intrinsics, obs);
    if(dp.i_extr0 >= 0 && dp.Ncam_e > 0 && icam_intrinsics >= 0)
        cross_columns_kernel<<<(dp.Ncam_e * 36 + 127) / 128, 128, 0, s>>>(obs, Nobs, 0, dp.i_extr0, 6, dp.Ncam_e, K, Nstate);
    if(dp.i_frame0 >= 0 && dp.Nframes > 0)
        cross_columns_kernel<<<(dp.Nframes * 36 + 127) / 128, 128, 0, s>>>(obs, Nobs, 1, dp.i_frame0, 6, dp.Nframes, K, Nstate);
    if(dp.i_point0 >= 0 && dp.Npoints_variable > 0)
        cross_columns_kernel<<<(dp.Npoints_variable * 18 + 127) / 128, 128, 0, s>>>(obs, Nobs, 2, dp.i_point0, 3, dp.Npoints_variable, K, Nstate);
    cross_totals_kernel<<<1, 64, 0, s>>>(obs, Nobs, dp.opt_warp ? dp.i_warp0 : -1, K, Nstate, JJ);
    // the columns that can be nonzero: from the first extrinsics / frame / point column to the end of the state
    int c0 = Nstate;
    if(dp.i_extr0 >= 0) c0 = dp.i_extr0 < c0 ? dp.i_extr0 : c0;
    if(dp.i_frame0 >= 0) c0 = dp.i_frame0 < c0 ? dp.i_frame0 : c0;
    if(dp.i_point0 >= 0) c0 = dp.i_point0 < c0 ? dp.i_point0 : c0;
    if(dp.i_warp0 >= 0) c0 = dp.i_warp0 < c0 ? dp.i_warp0 : c0;
    cross_solve_kernel<<<(Nstate - c0 + 127) / 128, 128, 0, s>>>(JJ, K, Nstate, c0, Nstate, info);
    P->launches += 6;
    int h_info = 0;
    MB200_CUDA_CHECK(cudaGetLastError());
    MB200_CUDA_CHECK(cudaMemcpyAsync(&h_info, info, sizeof(int), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    if(h_info != 0) { set_error("Singular Jcross_t Jcross!"); return false; }
    return true;
}

}  // namespace mb200
using namespace mb200;

// K_out: [6][Nstate] (host), zero outside the extrinsics / frames / points / calobject_warp columns. The Jacobian is
// evaluated at the problem's current state (as mrcal.drt_cross_reprojection__dbpacked() does, mrcal-pywrap.c:1931-1990)
extern "C" bool mrcal_b200_problem_drt_cross_reprojection__dbpacked(mrcal_b200_problem_t* P, int icam_intrinsics, double* K_out)
{
    DeviceArena tmp;
    double* K = nullptr;
    if(!tmp.alloc(&K, (size_t)6 * P->L.Nstate)) return false;
    if(!cross_reprojection_K(P, icam_intrinsics, true, K)) return false;
    MB200_CUDA_CHECK(cudaMemcpyAsync(K_out, K, (size_t)6 * P->L.Nstate * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
    MB200_CUDA_CHECK(cudaStreamSynchronize(P->stream));
    return true;
}
