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

// Raises the limit of `kernel`'s dynamic shared memory to `bytes`, once per device (the attribute is per device)
template <auto kernel>
bool set_max_dynamic_smem(int bytes)
{
    static bool configured[kMaxDevices] = {};
    int dev = 0;
    MB200_CUDA_CHECK(cudaGetDevice(&dev));
    if(dev < 0 || dev >= kMaxDevices) { set_error("device index %d out of range", dev); return false; }
    if(!configured[dev])
    {
        MB200_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
        configured[dev] = true;
    }
    return true;
}

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
    int           Nreg_dist, Nreg_center, Nreg_unity;   // the regularization rows, from m_reg0 on (see reg_row_j0())
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

// The regularization rows (mrcal.c:5655-5955) follow all other rows, from measurement m_reg0 and Jacobian entry reg_j0
// on, in three runs:
//   Nreg_dist    on the distortions, Ndist_state per camera. Splined models: a radial and a tangential row per knot,
//                each with 2 entries (the knot's two surfaces); the others: 1 entry
//   Nreg_center  on the centre pixels, 2 per camera, 1 entry each
//   Nreg_unity   on the translation of camera 0, 3 entries
// The first Jacobian entry of regularization row t
__host__ __device__ __forceinline__ int reg_row_j0(const DevProblem& P, bool splined, int t)
{
    const int wd = splined ? 2 : 1;
    if(t < P.Nreg_dist)                 return P.reg_j0 + wd * t;
    if(t < P.Nreg_dist + P.Nreg_center) return P.reg_j0 + wd * P.Nreg_dist + (t - P.Nreg_dist);
    return P.reg_j0 + wd * P.Nreg_dist + P.Nreg_center;
}
// the Jacobian's entries: all of them, the regularization's last
__host__ __device__ __forceinline__ int reg_nnz_total(const DevProblem& P, bool splined)
{
    return P.reg_j0 + (splined ? 2 : 1) * P.Nreg_dist + P.Nreg_center + 3 * P.Nreg_unity;
}
// The regularization rows by the unknowns they couple: a spline knot's two rows over its two surfaces, every other row
// alone. Block b: rows m0 .. m0 + nrows - 1, entries from j0 on, ncol per row
struct RegBlock { int m0, nrows, j0, ncol; };
__host__ __device__ __forceinline__ int reg_block_count(const DevProblem& P, bool splined)
{
    return (splined ? P.Nreg_dist / 2 : P.Nreg_dist) + P.Nreg_center + P.Nreg_unity;
}
__host__ __device__ __forceinline__ RegBlock reg_block(const DevProblem& P, bool splined, int b)
{
    const int Ndist_blocks = splined ? P.Nreg_dist / 2 : P.Nreg_dist;
    const int wd = splined ? 2 : 1;
    RegBlock r;
    if(b < Ndist_blocks)
    {
        if(splined) { r.m0 = P.m_reg0 + 2 * b; r.nrows = 2; r.j0 = P.reg_j0 + 4 * b; r.ncol = 2; }
        else        { r.m0 = P.m_reg0 + b;     r.nrows = 1; r.j0 = P.reg_j0 + b;     r.ncol = 1; }
    }
    else if(b < Ndist_blocks + P.Nreg_center)
    {
        const int rr = b - Ndist_blocks;
        r.m0 = P.m_reg0 + P.Nreg_dist + rr; r.nrows = 1; r.j0 = P.reg_j0 + wd * P.Nreg_dist + rr; r.ncol = 1;
    }
    else { r.m0 = P.m_reg0 + P.Nreg_dist + P.Nreg_center; r.nrows = 1; r.j0 = P.reg_j0 + wd * P.Nreg_dist + P.Nreg_center; r.ncol = 3; }
    return r;
}
// The block of state column c when it is a shared unknown that only its own regularization block touches (a distortion
// or a centre pixel), and c's place among the block's columns (*which); -1: no regularization row touches c
__host__ __device__ __forceinline__ int reg_block_of_column(const DevProblem& P, bool splined, int c, int* which)
{
    *which = 0;
    if(!P.reg || c >= P.Ncam_i * P.Nintr_state) return -1;
    const int cam = c / P.Nintr_state, k = c - cam * P.Nintr_state;
    if(k >= P.Ncore_state)
    {
        const int t = cam * P.Ndist_state + (k - P.Ncore_state);
        if(!splined) return t;
        *which = t & 1;
        return t >> 1;
    }
    if(k >= 2) return (splined ? P.Nreg_dist / 2 : P.Nreg_dist) + 2 * cam + (k - 2);
    return -1;
}

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
