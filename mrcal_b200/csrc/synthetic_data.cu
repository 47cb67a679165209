// Synthetic calibration data on the device: the projections behind mrcal.synthesize_board_observations()
// (mrcal/synthetic_data.py:236-554), and the hypothetical board corners and perfect observations of a problem behind
// mrcal.hypothesis_board_corner_positions() (mrcal/utils.py:440-584) and mrcal.make_perfect_observations()
// (mrcal/synthetic_data.py:594-750). Each keeps the reference's order of pose operations: the synthesized boards are
// transformed twice (board -> ref -> camera), the problem's corners through the composed Rt_cam_frame. The random
// draws, the host-side arithmetic that must keep the reference's bits and the frame selection stay in Python
// (mrcal_b200/synthetic_data.py).
#include <cuda_runtime.h>

#include <vector>

#include "common.h"
#include "device_call.h"
#include "lens_dispatch.cuh"
#include "pose.cuh"

namespace mb200 {
namespace {

constexpr int kThreads = 128;

// Rt[i] = Rt_from_rt(rt[i])
__device__ __forceinline__ void Rt_from_rt(double Rt[12], const double* rt)
{
    const double r[3] = {rt[0], rt[1], rt[2]};
    R_from_r(Rt, nullptr, r);
    for(int k = 0; k < 3; k++) Rt[9 + k] = rt[3 + k];
}

__global__ void __launch_bounds__(kThreads) Rt_from_rt_kernel(const double* __restrict__ rt, int N,
                                                              double* __restrict__ Rt)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= N) return;
    double R[12];
    Rt_from_rt(R, rt + 6 * (size_t)i);
    for(int k = 0; k < 12; k++) Rt[12 * (size_t)i + k] = R[k];
}

// One CTA per frame f, for camera icam of Ncam: every board corner p is taken to the reference and then to the camera,
// Rt_cam_ref(Rt_ref_boardref[f](p)), and projected into q [Nframes][Ncam][Npt][2]. Nvisible [Nframes][Ncam] counts the
// corners with 0 <= q <= imagersize - 1 on both axes (no test of z, as in the reference): integers, so the count is
// exact in any order
template <int KIND>
__global__ void __launch_bounds__(kThreads) synthesize_kernel(LensArgs a, const double* __restrict__ Rt_ref_boardref,
                                                              const double* __restrict__ board, int Npt,
                                                              const double* __restrict__ Rt_cam_ref, int icam,
                                                              int Ncam, double xmax, double ymax,
                                                              double* __restrict__ q, int* __restrict__ Nvisible)
{
    const int f = blockIdx.x;
    double Rf[12], Rc[12];
    for(int k = 0; k < 12; k++) { Rf[k] = Rt_ref_boardref[12 * (size_t)f + k]; Rc[k] = Rt_cam_ref[k]; }
    double* qf = q + ((size_t)f * Ncam + icam) * Npt * 2;
    int count = 0;
    for(int base = 0; base < Npt; base += kThreads)
    {
        const int i = base + threadIdx.x;
        bool visible = false;
        if(i < Npt)
        {
            const double p[3] = {board[3 * i], board[3 * i + 1], board[3 * i + 2]};
            double pref[3], pcam[3], qq[2], g[2][3];
            transform_point_Rt(pref, Rf, p);
            transform_point_Rt(pcam, Rc, pref);
            project_any<KIND>(qq, g, pcam, a);
            qf[2 * i] = qq[0];
            qf[2 * i + 1] = qq[1];
            visible = qq[0] >= 0. && qq[1] >= 0. && qq[0] <= xmax && qq[1] <= ymax;
        }
        count += __syncthreads_count(visible);
    }
    if(threadIdx.x == 0) Nvisible[(size_t)f * Ncam + icam] = count;
}

// Rt_cam_frame [Nobs][12] of each board observation (iframe, icam_intrinsics, icam_extrinsics):
// compose_Rt(Rt_cam_ref, Rt_ref_frame), with the identity for icam_extrinsics = -1, as the reference composes it
__global__ void __launch_bounds__(kThreads) observation_poses_kernel(const int* __restrict__ indices, int Nobs,
                                                                     const double* __restrict__ rt_ref_frame,
                                                                     const double* __restrict__ rt_cam_ref,
                                                                     double* __restrict__ Rt_cam_frame)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if(o >= Nobs) return;
    const int iframe = indices[3 * o], ie = indices[3 * o + 2];
    double Rf[12], Rc[12], out[12];
    Rt_from_rt(Rf, rt_ref_frame + 6 * (size_t)iframe);
    if(ie < 0)
        for(int k = 0; k < 12; k++) Rc[k] = (k < 9 && k % 4 == 0) ? 1. : 0.;
    else
        Rt_from_rt(Rc, rt_cam_ref + 6 * (size_t)ie);
    compose_Rt(out, Rc, Rf, false, false);
    for(int k = 0; k < 12; k++) Rt_cam_frame[12 * (size_t)o + k] = out[k];
}

// One thread per (board observation, corner): pcam = Rt_cam_frame(corner) into pcam [Nobs][Npt][3] (if not NULL) and,
// for KIND >= 0, its projection through the observing camera's intrinsics into q [Nobs][Npt][2]
template <int KIND>
__global__ void __launch_bounds__(kThreads) board_corners_kernel(LensArgs a, int Nintr, const int* __restrict__ indices,
                                                                 const double* __restrict__ Rt_cam_frame, int Nobs,
                                                                 const double* __restrict__ board, int Npt,
                                                                 double* __restrict__ pcam_out, double* __restrict__ q)
{
    const size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(e >= (size_t)Nobs * Npt) return;
    const size_t o = e / Npt;
    const int i = (int)(e % Npt);
    double R[12];
    for(int k = 0; k < 12; k++) R[k] = Rt_cam_frame[12 * o + k];
    const double p[3] = {board[3 * i], board[3 * i + 1], board[3 * i + 2]};
    double pcam[3];
    transform_point_Rt(pcam, R, p);
    if(pcam_out)
        for(int k = 0; k < 3; k++) pcam_out[3 * e + k] = pcam[k];
    if constexpr(KIND >= 0)
    {
        LensArgs l = a;
        l.intr += (size_t)indices[3 * o + 1] * Nintr;
        double qq[2], g[2][3];
        project_any<KIND>(qq, g, pcam, l);
        q[2 * e] = qq[0];
        q[2 * e + 1] = qq[1];
    }
}

// One thread per point observation (i_point, icam_intrinsics, icam_extrinsics): Rt_cam_ref(points[i_point]), the
// identity for icam_extrinsics = -1, projected into q [Nobs][2]
template <int KIND>
__global__ void __launch_bounds__(kThreads) point_kernel(LensArgs a, int Nintr, const int* __restrict__ indices, int Nobs,
                                                         const double* __restrict__ points,
                                                         const double* __restrict__ rt_cam_ref, double* __restrict__ q)
{
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if(o >= Nobs) return;
    const int ipt = indices[3 * o], ie = indices[3 * o + 2];
    const double p[3] = {points[3 * (size_t)ipt], points[3 * (size_t)ipt + 1], points[3 * (size_t)ipt + 2]};
    double pcam[3];
    if(ie < 0)
        for(int k = 0; k < 3; k++) pcam[k] = p[k];
    else
    {
        double Rc[12];
        Rt_from_rt(Rc, rt_cam_ref + 6 * (size_t)ie);
        transform_point_Rt(pcam, Rc, p);
    }
    LensArgs l = a;
    l.intr += (size_t)indices[3 * o + 1] * Nintr;
    double qq[2], g[2][3];
    project_any<KIND>(qq, g, pcam, l);
    q[2 * o] = qq[0];
    q[2 * o + 1] = qq[1];
}

unsigned blocks_for(size_t n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// false + set_error() unless every row of indices [N][3] has column 0 in [0, N0), column 1 in [0, N1) (unless N1 < 0)
// and column 2 in [-1, N2)
bool indices_ok(const char* what, const int* indices, int N, int N0, const char* name0, int N1, int N2)
{
    for(int o = 0; o < N; o++)
    {
        const int* r = indices + 3 * o;
        if(r[0] < 0 || r[0] >= N0) { set_error("%s: %s MUST be in [0,%d]; row %d has %d", what, name0, N0 - 1, o, r[0]); return false; }
        if(N1 >= 0 && (r[1] < 0 || r[1] >= N1))
        { set_error("%s: icam_intrinsics MUST be in [0,%d]; row %d has %d", what, N1 - 1, o, r[1]); return false; }
        if(r[2] < -1 || r[2] >= N2)
        { set_error("%s: icam_extrinsics MUST be in [-1,%d]; row %d has %d", what, N2 - 1, o, r[2]); return false; }
    }
    return true;
}

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_synthesize_board_observations(double* q, int* Nvisible, double* Rt_ref_boardref,
                                                         const double* rt_ref_boardref, int Nframes,
                                                         const double* board, int Npoints, int Ncameras,
                                                         const mrcal_lensmodel_t* lensmodels, const double* intrinsics,
                                                         const double* Rt_cam_ref, const int* imagersizes)
{
    if(Nframes < 0 || Npoints < 0 || Ncameras < 0)
    {
        set_error("synthesize_board_observations: Nframes, Npoints and Ncameras must be >= 0");
        return false;
    }
    DeviceCall D;
    if(!D.start()) return false;
    std::vector<HostLens> lens(Ncameras);
    size_t Nintr_all = 0;
    for(int c = 0; c < Ncameras; c++)
    {
        if(!lens_setup(&lens[c], &lensmodels[c])) return false;
        Nintr_all += lens[c].Nintr;
    }
    if(Nframes == 0) return true;
    const size_t Nq = (size_t)Nframes * Ncameras * Npoints * 2;
    double *d_rt, *d_Rt, *d_board, *d_intr, *d_Rc, *d_q;
    int* d_Nvis;
    if(!D.upload(&d_rt, rt_ref_boardref, (size_t)Nframes * 6) || !D.alloc(&d_Rt, (size_t)Nframes * 12) ||
       !D.upload(&d_board, board, (size_t)Npoints * 3) || !D.upload(&d_intr, intrinsics, Nintr_all) ||
       !D.upload(&d_Rc, Rt_cam_ref, (size_t)Ncameras * 12) || !D.alloc(&d_q, Nq) ||
       !D.alloc(&d_Nvis, (size_t)Nframes * Ncameras))
        return false;
    Rt_from_rt_kernel<<<blocks_for(Nframes), kThreads, 0, D.stream>>>(d_rt, Nframes, d_Rt);
    size_t i0 = 0;
    for(int c = 0; c < Ncameras; c++)
    {
        HostLens& L = lens[c];
        L.a.intr = d_intr + i0;
        i0 += L.Nintr;
        const double xmax = imagersizes[2 * c] - 1, ymax = imagersizes[2 * c + 1] - 1;
        if(!dispatch_lens_kind(L.kind, [&](auto k)
           {
               synthesize_kernel<decltype(k)::value><<<Nframes, kThreads, 0, D.stream>>>(
                   L.a, d_Rt, d_board, Npoints, d_Rc + 12 * c, c, Ncameras, xmax, ymax, d_q, d_Nvis);
           }))
            return false;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(q, d_q, Nq) && D.download(Nvisible, d_Nvis, (size_t)Nframes * Ncameras) &&
           D.download(Rt_ref_boardref, d_Rt, (size_t)Nframes * 12) && D.finish();
}

extern "C" bool mrcal_b200_problem_corners(double* pcam_board, double* q_board, double* q_point,
                                           const int32_t* indices_frame_camintrinsics_camextrinsics,
                                           int Nobservations_board, const double* board, int Npoints_board,
                                           const int32_t* indices_point_camintrinsics_camextrinsics,
                                           int Nobservations_point, const double* points, int Npoints,
                                           const double* rt_ref_frame, int Nframes, const double* rt_cam_ref,
                                           int Ncameras_extrinsics, const mrcal_lensmodel_t* lensmodel,
                                           const double* intrinsics, int Ncameras_intrinsics)
{
    const bool project = q_board != nullptr || q_point != nullptr;
    if(Nobservations_board < 0 || Nobservations_point < 0 || Npoints_board < 0 || Ncameras_intrinsics < 0)
    {
        set_error("problem_corners: negative counts");
        return false;
    }
    if(Nobservations_point > 0 && q_point == nullptr)
    {
        set_error("problem_corners: point observations are only projected: q_point must be given");
        return false;
    }
    if(project && (lensmodel == nullptr || intrinsics == nullptr))
    {
        set_error("problem_corners: projecting needs the lens model and the intrinsics");
        return false;
    }
    const int N1 = project ? Ncameras_intrinsics : -1;
    if(!indices_ok("problem_corners", indices_frame_camintrinsics_camextrinsics, Nobservations_board, Nframes, "iframe",
                   N1, Ncameras_extrinsics) ||
       !indices_ok("problem_corners", indices_point_camintrinsics_camextrinsics, Nobservations_point, Npoints, "i_point",
                   N1, Ncameras_extrinsics))
        return false;
    DeviceCall D;
    HostLens L{};
    if(!D.start() || (project && !lens_setup(&L, lensmodel))) return false;
    const size_t Nb = (size_t)Nobservations_board * Npoints_board;
    if(Nb == 0 && Nobservations_point == 0) return true;
    int *d_ib, *d_ip;
    double *d_intr = nullptr, *d_rtf, *d_rtc, *d_board, *d_points, *d_Rt, *d_pcam = nullptr, *d_qb = nullptr,
           *d_qp = nullptr;
    if(!D.upload(&d_ib, indices_frame_camintrinsics_camextrinsics, (size_t)Nobservations_board * 3) ||
       !D.upload(&d_ip, indices_point_camintrinsics_camextrinsics, (size_t)Nobservations_point * 3) ||
       (project && !D.upload(&d_intr, intrinsics, (size_t)Ncameras_intrinsics * L.Nintr)) ||
       !D.upload(&d_rtf, rt_ref_frame, (size_t)Nframes * 6) ||
       !D.upload(&d_rtc, rt_cam_ref, (size_t)Ncameras_extrinsics * 6) ||
       !D.upload(&d_board, board, (size_t)Npoints_board * 3) || !D.upload(&d_points, points, (size_t)Npoints * 3) ||
       !D.alloc(&d_Rt, (size_t)Nobservations_board * 12) || (pcam_board && !D.alloc(&d_pcam, Nb * 3)) ||
       (q_board && !D.alloc(&d_qb, Nb * 2)) || (q_point && !D.alloc(&d_qp, (size_t)Nobservations_point * 2)))
        return false;
    L.a.intr = d_intr;
    if(Nb > 0)
    {
        observation_poses_kernel<<<blocks_for(Nobservations_board), kThreads, 0, D.stream>>>(d_ib, Nobservations_board,
                                                                                             d_rtf, d_rtc, d_Rt);
        if(q_board == nullptr)
            board_corners_kernel<-1><<<blocks_for(Nb), kThreads, 0, D.stream>>>(L.a, L.Nintr, d_ib, d_Rt, Nobservations_board,
                                                                               d_board, Npoints_board, d_pcam, nullptr);
        else if(!dispatch_lens_kind(L.kind, [&](auto k)
                {
                    board_corners_kernel<decltype(k)::value><<<blocks_for(Nb), kThreads, 0, D.stream>>>(
                        L.a, L.Nintr, d_ib, d_Rt, Nobservations_board, d_board, Npoints_board, d_pcam, d_qb);
                }))
            return false;
    }
    if(Nobservations_point > 0 &&
       !dispatch_lens_kind(L.kind, [&](auto k)
       {
           point_kernel<decltype(k)::value><<<blocks_for(Nobservations_point), kThreads, 0, D.stream>>>(
               L.a, L.Nintr, d_ip, Nobservations_point, d_points, d_rtc, d_qp);
       }))
        return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return (!pcam_board || D.download(pcam_board, d_pcam, Nb * 3)) && (!q_board || D.download(q_board, d_qb, Nb * 2)) &&
           (!q_point || D.download(q_point, d_qp, (size_t)Nobservations_point * 2)) && D.finish();
}
