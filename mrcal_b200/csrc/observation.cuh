// The geometry of a board observation, shared by the two kernels that evaluate it (eval_boards_kernel in eval.cu,
// fused_boards_kernel in fused_eval.cu): the two poses in shared memory and the corner point.
#pragma once
#include "device_math.cuh"
#include "problem.h"

namespace mb200 {

// The two poses of a board observation, in shared memory: R, dR/dr and t of the frame and of the camera
struct ObsPoses
{
    double Rf[9], dRf[27], tf[3];
    double Rc[9], dRc[27], tc[3];
};

// Cooperative load of the expanded poses (expand_rotations_kernel) by the first 100 threads of the CTA; the camera's
// only if it has extrinsics (icam_e >= 0). t is the thread's index in the CTA, in the caller's own type (threadIdx.x or
// an int copy): the index arithmetic follows it, so each kernel compiles as it did with the load written inline. The
// caller synchronizes
template <class Index>
__device__ __forceinline__ void load_obs_poses(ObsPoses& G, const DevProblem& P, int iframe, int icam_e, Index t)
{
    if(t < 36) { const double v = P.u_rot_frame[36 * iframe + t]; if(t < 9) G.Rf[t] = v; else G.dRf[t - 9] = v; }
    else if(t < 39) G.tf[t - 36] = P.u_rtframe[6 * iframe + 3 + t - 36];
    if(icam_e >= 0)
    {
        if(t >= 64 && t < 100) { const int k = t - 64; const double v = P.u_rot_cam[36 * icam_e + k]; if(k < 9) G.Rc[k] = v; else G.dRc[k - 9] = v; }
        else if(t >= 40 && t < 43) G.tc[t - 40] = P.u_rtcam[6 * icam_e + 3 + t - 40];
    }
}

// Corner (cx, cy) of the board: the board point pt with the parabolic warp (mrcal.c:2794-2819), dz[i] = dpt_z/dwarp_i,
// v = Rf pt + tf in reference coordinates and p = Rc v + tc in camera coordinates
__device__ __forceinline__ void board_corner(double pt[3], double dz[2], double v[3], double p[3], const DevProblem& P,
                                             const ObsPoses& G, bool cam_identity, int cx, int cy, double warp_x, double warp_y)
{
    pt[0] = (double)cx * P.spacing; pt[1] = (double)cy * P.spacing; pt[2] = 0.;
    dz[0] = 0.; dz[1] = 0.;
    if(P.have_warp)
    {
        const double xr = (double)cx / (double)(P.W - 1), yr = (double)cy / (double)(P.H - 1);
        dz[0] = 4. * xr * (1. - xr);
        dz[1] = 4. * yr * (1. - yr);
        pt[2] += warp_x * dz[0];
        pt[2] += warp_y * dz[1];
    }
    mat3_vec(v, G.Rf, pt);
    v[0] += G.tf[0]; v[1] += G.tf[1]; v[2] += G.tf[2];
    if(cam_identity) { p[0] = v[0]; p[1] = v[1]; p[2] = v[2]; }
    else { mat3_vec(p, G.Rc, v); p[0] += G.tc[0]; p[1] += G.tc[1]; p[2] += G.tc[2]; }
}

}  // namespace mb200
