// Internal: the device-resident problem and the kernels' parameter block.
#pragma once
#include <cuda_runtime.h>

#include "common.h"

namespace mb200 {

#define MB200_CUDA_CHECK(expr)                                                            \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if(_e != cudaSuccess)                                                             \
        {                                                                                 \
            mb200::set_error("CUDA error %s at %s:%d: %s", cudaGetErrorName(_e), __FILE__, __LINE__, \
                             cudaGetErrorString(_e));                                     \
            return false;                                                                 \
        }                                                                                 \
    } while(0)

constexpr int kMaxDevices = 64;   // per-device one-time kernel configuration flags

// SMs of the current device (cached per device); 0 if it cannot be queried
int device_sm_count();

// Read-only description handed to every kernel BY VALUE (lives in the constant
// bank; ~300 bytes). All pointers are device pointers.
struct DevProblem
{
    int Ncam_i, Ncam_e, Nframes, Npoints, Npoints_variable, Nobs_board, Nobs_point;
    int W, H;
    int Nintr, Ncore_state, Ndist_state, Nintr_state;
    int i_intr0, i_extr0, i_frame0, i_point0, i_warp0, Nstate;
    int m_point0, m_reg0, Nmeas;
    int lens_kind;             // LensKind
    int Nx, Ny;
    double segments_per_u;
    double lens_cfg;           // the lens model's configuration scalar (CAHVORE: linearity)
    double spacing;
    bool opt_core, opt_dist, opt_extr, opt_frames, opt_warp;
    bool have_warp;            // a calobject_warp was given (optimised or not)
    bool reg, reg_unity;
    bool reg_owner;            // this rank adds the (replicated) regularization rows to cross-rank sums
    int  opencv8plus;          // regularisation of the rational denominators (mrcal.c:5806-5834)
    int  nnz_row_intr;         // per board/point row
    int  nnz_row_board_geom;   // frames + warp

    // the seed / fixed values, unpacked units
    const double* in_intrinsics;   // [Ncam_i][Nintr]
    const double* in_rt_cam;       // [Ncam_e][6]
    const double* in_rt_frame;     // [Nframes][6]
    const double* in_points;       // [Npoints][3]
    const double* in_warp;         // [2]
    const int*    imagersizes;     // [Ncam_i][2]

    const int*    obs_board;       // [Nobs_board][3] = icam_intrinsics, icam_extrinsics, iframe
    const double* obs_board_pool;  // [Nobs_board*W*H][3] = qx, qy, weight
    const int*    obs_point;       // [Nobs_point][3] = icam_intrinsics, icam_extrinsics, i_point
    const double* obs_point_pool;  // [Nobs_point][3]
    const int*    board_j0;        // [Nobs_board+1] index of each observation's first Jacobian entry
    const int*    point_j0;        // [Nobs_point+1]
    int           reg_j0;          // first Jacobian entry of the regularization rows
    // triangulated points (mrcal.c:5180-5653): observation rays in camera coordinates, pairs of them
    int           m_tri0, Ntri;    // first measurement, number of measurements (= pairs)
    const double* tri_px;          // [Nobs_tri][3]
    const int*    tri_cam_e;       // [Nobs_tri] icam_extrinsics (-1: at the reference)
    int*          tri_outlier;     // [Nobs_tri] flags; outlier rejection adds to them (outliers.cu)
    const int*    tri_pairs;       // [Ntri][2] observation indices i0 < i1
    const int*    tri_j0;          // [Ntri+1] first Jacobian entry of each pair's row
    const int*    tri_cam_ptr;     // [Ncam_e+1] the pairs that see camera e: tri_cam_rows[tri_cam_ptr[e] .. tri_cam_ptr[e+1])
    const int*    tri_cam_rows;    // pair indices, increasing within each camera
    int           Ntri_sets;       // triangulated points (sets of consecutive observations)
    const int*    tri_set_obs0;    // [Ntri_sets+1] first observation of each set
    const int*    tri_set_m0;      // [Ntri_sets] first measurement (pair) of each set, relative to m_tri0

    // the current state, unpacked (written by unpack_state_kernel each evaluation)
    double* u_intr;      // [Ncam_i][Nintr]
    double* u_rtcam;     // [Ncam_e][6]
    double* u_rtframe;   // [Nframes][6]
    double* u_points;    // [Npoints][3]
    double* u_warp;      // [2]
    double* u_rot_frame; // [Nframes][36]  R (9) then dR/dr (27) of each frame's Rodrigues vector
    double* u_rot_cam;   // [Ncam_e][36]   same for each camera
};

// One set of evaluation outputs ("operating point" in libdogleg's language)
struct EvalBuffers
{
    double* p     = nullptr;   // [Nstate] packed state
    double* x     = nullptr;   // [Nmeas]
    double* Jval  = nullptr;   // [nnz]   CSR order
    int*    Jcol  = nullptr;   // [nnz]
    double* norm2 = nullptr;   // [1] |x|^2
};

struct Problem;   // problem.cu

// eval.cu
bool launch_unpack_state(const DevProblem& dp, const double* b_packed, cudaStream_t stream, int* launch_counter);
bool launch_evaluate(const DevProblem& dp, const EvalBuffers& out, bool with_jacobian,
                     int* Jrowptr /* device, may be null */, cudaStream_t stream, int* launch_counter, bool boards = true);

}  // namespace mb200
