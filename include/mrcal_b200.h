// mrcal_b200: C-ABI of the H100-native implementation of mrcal's calibration
// solve (the optimizer_callback residual/Jacobian evaluator and the
// trust-region normal-equations solve).
//
// This is the drop-in boundary. Part 1 re-declares, with IDENTICAL names,
// argument order, struct layouts and error behaviour, the subset of the
// reference's C API that its Python wrapper (mrcal-pywrap.c) binds for this
// path; each declaration cites the reference interface it replaces
// (file:line into the reference tree). A build of the reference that links
// libmrcal_b200.so instead of compiling the corresponding functions of mrcal.c
// gets the GPU path with no source change (INTEGRATION.md).
//
// Part 2 (prefix mrcal_b200_) is the extension surface that has no counterpart
// in the reference: a device-resident problem handle (so repeated solves and
// the benchmark can keep inputs in HBM), the factorization object that stands
// in for mrcal.CHOLMOD_factorization, multi-GPU initialisation and
// introspection.
//
// Plain C: pointers and sizes only. No torch, no C++ types.
#pragma once

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

////////////////////////////////////////////////////////////////////////////////
// Part 1a. Types. Layout-compatible with the reference (x86-64 SysV)
////////////////////////////////////////////////////////////////////////////////

// replaces basic-geometry.h:17-91
typedef union { struct { double x, y; };    double xy[2];  } mrcal_point2_t;
typedef union { struct { double x, y, z; }; double xyz[3]; } mrcal_point3_t;
typedef struct { mrcal_point3_t r, t; } mrcal_pose_t;   // rt: Rodrigues r, then t

// replaces types.h:33-121. Values are the X-macro order of MRCAL_LENSMODEL_LIST
typedef enum
{
    MRCAL_LENSMODEL_INVALID_TYPE          = -4,
    MRCAL_LENSMODEL_INVALID_MISSINGCONFIG = -3,
    MRCAL_LENSMODEL_INVALID               = -2,
    MRCAL_LENSMODEL_INVALID_BADCONFIG     = -1,
    MRCAL_LENSMODEL_PINHOLE               = 0,
    MRCAL_LENSMODEL_STEREOGRAPHIC         = 1,
    MRCAL_LENSMODEL_LONLAT                = 2,
    MRCAL_LENSMODEL_LATLON                = 3,
    MRCAL_LENSMODEL_OPENCV4               = 4,
    MRCAL_LENSMODEL_OPENCV5               = 5,
    MRCAL_LENSMODEL_OPENCV8               = 6,
    MRCAL_LENSMODEL_OPENCV12              = 7,
    MRCAL_LENSMODEL_CAHVOR                = 8,
    MRCAL_LENSMODEL_CAHVORE               = 9,
    MRCAL_LENSMODEL_SPLINED_STEREOGRAPHIC = 10
} mrcal_lensmodel_type_t;

// replaces types.h:66-92
typedef struct { double   linearity;                } mrcal_LENSMODEL_CAHVORE__config_t;
typedef struct { uint16_t order, Nx, Ny, fov_x_deg; } mrcal_LENSMODEL_SPLINED_STEREOGRAPHIC__config_t;

// replaces types.h:122-136. sizeof == 16; the configuration lives at offset 8
typedef struct
{
    mrcal_lensmodel_type_t type;
    union
    {
        mrcal_LENSMODEL_CAHVORE__config_t               LENSMODEL_CAHVORE__config;
        mrcal_LENSMODEL_SPLINED_STEREOGRAPHIC__config_t LENSMODEL_SPLINED_STEREOGRAPHIC__config;
    };
} mrcal_lensmodel_t;

// replaces types.h:175-182
typedef struct
{
    bool has_core                  : 1;
    bool can_project_behind_camera : 1;
    bool has_gradients             : 1;
    bool noncentral                : 1;
} mrcal_lensmodel_metadata_t;

// replaces types.h:139-148
typedef union { struct { double x2, y2; }; double values[2]; } mrcal_calobject_warp_t;
#define MRCAL_NSTATE_CALOBJECT_WARP 2

// replaces types.h:196-228. NOTE the order differs from the Python index arrays
// (iframe, icam_intrinsics, icam_extrinsics): mrcal-pywrap.c:1255-1261
typedef struct { int intrinsics; int extrinsics; /* <0: at the reference */ } mrcal_camera_index_t;
typedef struct { mrcal_camera_index_t icam; int iframe;  } mrcal_observation_board_t;
typedef struct { mrcal_camera_index_t icam; int i_point; } mrcal_observation_point_t;

// replaces types.h:243-263
typedef struct
{
    mrcal_camera_index_t icam;
    bool                 last_in_set : 1;
    bool                 outlier     : 1;
    mrcal_point3_t       px;
} mrcal_observation_point_triangulated_t;

// replaces types.h:283-307. One byte, passed BY VALUE
typedef struct
{
    bool do_optimize_intrinsics_core         : 1;
    bool do_optimize_intrinsics_distortions  : 1;
    bool do_optimize_extrinsics              : 1;
    bool do_optimize_frames                  : 1;
    bool do_optimize_calobject_warp          : 1;
    bool do_apply_regularization             : 1;
    bool do_apply_outlier_rejection          : 1;
    bool do_apply_regularization_unity_cam01 : 1;
} mrcal_problem_selections_t;

// replaces types.h:313-315 (empty in the reference; sizeof 0 in GNU C, 1 in C++.
// Only ever passed by pointer, and never dereferenced)
typedef struct mrcal_problem_constants_t mrcal_problem_constants_t;

// replaces types.h:320-343
typedef struct
{
    double rms_reproj_error__pixels;   // <0 on error
    int    Noutliers_board;
    int    Noutliers_triangulated_point;
} mrcal_stats_t;

// Stands in for CHOLMOD's cholmod_sparse, which is what the reference passes
// as "Jt" (mrcal.h:548, mrcal.c:4461-4463). The transpose of J in
// compressed-column form == J in CSR. Only p, i, x are read by this library;
// field order and sizes follow the public CHOLMOD struct so that a
// cholmod_sparse* can be passed as is
typedef struct
{
    size_t nrow, ncol, nzmax;   // nrow = Nstate, ncol = Nmeasurements
    void*  p;                   // int32[Nmeasurements+1]   row pointers of J
    void*  i;                   // int32[nnz]               column indices of J
    void*  nz;
    void*  x;                   // double[nnz]              values of J
    void*  z;
    int    stype, itype, xtype, dtype, sorted, packed;
} mrcal_b200_sparse_t;

////////////////////////////////////////////////////////////////////////////////
// Part 1b. Lens-model description (host only)
////////////////////////////////////////////////////////////////////////////////

// replaces internal.h:30-49, 85 (mrcal.c:1904-1965): quantities derived from the model configuration, computed
// once. Only the splined model has one: segments_per_u = (Nx - 1 - margin) / (2 * 2 tan(fov_x/4)), margin 2 (cubic)
// or 1 (quadratic)
typedef struct
{
    bool ready;
    union
    {
        struct { double segments_per_u; } LENSMODEL_SPLINED_STEREOGRAPHIC__precomputed;
    };
} mrcal_projection_precomputed_t;
void _mrcal_precompute_lensmodel_data(mrcal_projection_precomputed_t* precomputed, const mrcal_lensmodel_t* lensmodel);

// replaces mrcal.h:98-102 (mrcal.c:156-214)
bool mrcal_lensmodel_from_name(mrcal_lensmodel_t* lensmodel, const char* name);
// replaces mrcal.h:87 (mrcal.c:219-250)
mrcal_lensmodel_type_t mrcal_lensmodel_type_from_name(const char* name);
// replaces mrcal.h:76-77 (mrcal.c:92-114)
bool mrcal_lensmodel_name(char* out, int size, const mrcal_lensmodel_t* lensmodel);
// replaces mrcal.h:59 (mrcal.c:47-71)
const char* mrcal_lensmodel_name_unconfigured(const mrcal_lensmodel_t* lensmodel);
// replaces mrcal.h:108 (mrcal.c:252-288)
mrcal_lensmodel_metadata_t mrcal_lensmodel_metadata(const mrcal_lensmodel_t* lensmodel);
// replaces mrcal.h:113 (mrcal.c:312-334)
int mrcal_lensmodel_num_params(const mrcal_lensmodel_t* lensmodel);
// replaces mrcal.h (mrcal.c:137-153)
const char* const* mrcal_supported_lensmodel_names(void);
// replaces mrcal.h (mrcal.c:1966-1998)
bool mrcal_knots_for_splined_models(double* ux, double* uy, const mrcal_lensmodel_t* lensmodel);

////////////////////////////////////////////////////////////////////////////////
// Part 1c. State-vector and measurement-vector layout (host only, pure integer)
////////////////////////////////////////////////////////////////////////////////

// replaces mrcal.h:729-790 (mrcal.c:352-379, 3737-3880)
int mrcal_num_intrinsics_optimization_params(mrcal_problem_selections_t problem_selections,
                                             const mrcal_lensmodel_t* lensmodel);
int mrcal_num_states(int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                     int Npoints, int Npoints_fixed, int Nobservations_board,
                     mrcal_problem_selections_t problem_selections,
                     const mrcal_lensmodel_t* lensmodel);
int mrcal_num_states_intrinsics(int Ncameras_intrinsics,
                                mrcal_problem_selections_t problem_selections,
                                const mrcal_lensmodel_t* lensmodel);
int mrcal_num_states_extrinsics(int Ncameras_extrinsics, mrcal_problem_selections_t problem_selections);
int mrcal_num_states_frames(int Nframes, mrcal_problem_selections_t problem_selections);
int mrcal_num_states_points(int Npoints, int Npoints_fixed, mrcal_problem_selections_t problem_selections);
int mrcal_num_states_calobject_warp(mrcal_problem_selections_t problem_selections, int Nobservations_board);

int mrcal_state_index_intrinsics(int icam_intrinsics,
                                 int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                 int Npoints, int Npoints_fixed, int Nobservations_board,
                                 mrcal_problem_selections_t problem_selections,
                                 const mrcal_lensmodel_t* lensmodel);
int mrcal_state_index_extrinsics(int icam_extrinsics,
                                 int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                 int Npoints, int Npoints_fixed, int Nobservations_board,
                                 mrcal_problem_selections_t problem_selections,
                                 const mrcal_lensmodel_t* lensmodel);
int mrcal_state_index_frames(int iframe,
                             int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                             int Npoints, int Npoints_fixed, int Nobservations_board,
                             mrcal_problem_selections_t problem_selections,
                             const mrcal_lensmodel_t* lensmodel);
int mrcal_state_index_points(int i_point,
                             int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                             int Npoints, int Npoints_fixed, int Nobservations_board,
                             mrcal_problem_selections_t problem_selections,
                             const mrcal_lensmodel_t* lensmodel);
int mrcal_state_index_calobject_warp(int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                     int Npoints, int Npoints_fixed, int Nobservations_board,
                                     mrcal_problem_selections_t problem_selections,
                                     const mrcal_lensmodel_t* lensmodel);

// replaces mrcal.h:792-853 (mrcal.c:395-735)
int mrcal_measurement_index_boards(int i_observation_board,
                                   int Nobservations_board, int Nobservations_point,
                                   int calibration_object_width_n, int calibration_object_height_n);
int mrcal_num_measurements_boards(int Nobservations_board,
                                  int calibration_object_width_n, int calibration_object_height_n);
int mrcal_measurement_index_points(int i_observation_point,
                                   int Nobservations_board, int Nobservations_point,
                                   int calibration_object_width_n, int calibration_object_height_n);
int mrcal_num_measurements_points(int Nobservations_point);
int mrcal_measurement_index_points_triangulated(int i_point_triangulated,
                                                int Nobservations_board, int Nobservations_point,
                                                const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                                                int Nobservations_point_triangulated,
                                                int calibration_object_width_n, int calibration_object_height_n);
int mrcal_num_measurements_points_triangulated_initial_Npoints(
        const mrcal_observation_point_triangulated_t* observations_point_triangulated,
        int Nobservations_point_triangulated, int Npoints);
int mrcal_num_measurements_points_triangulated(
        const mrcal_observation_point_triangulated_t* observations_point_triangulated,
        int Nobservations_point_triangulated);
int mrcal_measurement_index_regularization(
        const mrcal_observation_point_triangulated_t* observations_point_triangulated,
        int Nobservations_point_triangulated,
        int calibration_object_width_n, int calibration_object_height_n,
        int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
        int Npoints, int Npoints_fixed, int Nobservations_board, int Nobservations_point,
        mrcal_problem_selections_t problem_selections,
        const mrcal_lensmodel_t* lensmodel);
int mrcal_num_measurements_regularization(int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                          int Npoints, int Npoints_fixed, int Nobservations_board,
                                          mrcal_problem_selections_t problem_selections,
                                          const mrcal_lensmodel_t* lensmodel);
int mrcal_num_measurements(int Nobservations_board, int Nobservations_point,
                           const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                           int Nobservations_point_triangulated,
                           int calibration_object_width_n, int calibration_object_height_n,
                           int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                           int Npoints, int Npoints_fixed,
                           mrcal_problem_selections_t problem_selections,
                           const mrcal_lensmodel_t* lensmodel);
// replaces internal.h:99-114 (mrcal.c:743-882)
int _mrcal_num_j_nonzero(int Nobservations_board, int Nobservations_point,
                         const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                         int Nobservations_point_triangulated,
                         int calibration_object_width_n, int calibration_object_height_n,
                         int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                         int Npoints, int Npoints_fixed,
                         const mrcal_observation_board_t* observations_board,
                         const mrcal_observation_point_t* observations_point,
                         mrcal_problem_selections_t problem_selections,
                         const mrcal_lensmodel_t* lensmodel);

// replaces mrcal.h:389-431 (mrcal.c:3442-3506, 3690-3735). In place; b is one
// state vector of mrcal_num_states() doubles
void mrcal_pack_solver_state_vector(double* b,
                                    int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                    int Npoints, int Npoints_fixed, int Nobservations_board,
                                    mrcal_problem_selections_t problem_selections,
                                    const mrcal_lensmodel_t* lensmodel);
void mrcal_unpack_solver_state_vector(double* b,
                                      int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                                      int Npoints, int Npoints_fixed, int Nobservations_board,
                                      mrcal_problem_selections_t problem_selections,
                                      const mrcal_lensmodel_t* lensmodel);

// replaces mrcal.h (mrcal.c:3940-3976)
bool mrcal_corresponding_icam_extrinsics(int* icam_extrinsics,
                                         int icam_intrinsics,
                                         int Ncameras_intrinsics, int Ncameras_extrinsics,
                                         int Nobservations_board,
                                         const mrcal_observation_board_t* observations_board,
                                         int Nobservations_point,
                                         const mrcal_observation_point_t* observations_point);

////////////////////////////////////////////////////////////////////////////////
// Part 1d. The hot path (runs on the GPU; every buffer below is HOST memory
// owned by the caller, exactly as in the reference)
////////////////////////////////////////////////////////////////////////////////

// replaces mrcal.h:165-191: q = project(p), N points in camera coordinates. dq_dp (N,2,3) and
// dq_dintrinsics (N,2,Nintrinsics: dense, as mrcal.c:2866-2992 fills it) may be NULL
bool mrcal_project(mrcal_point2_t* q, mrcal_point3_t* dq_dp, double* dq_dintrinsics,
                   const mrcal_point3_t* p, int N,
                   const mrcal_lensmodel_t* lensmodel, const double* intrinsics);
// replaces mrcal.h:193-224: observation rays (not normalised) of N pixels. Models without a closed-form
// inverse are inverted iteratively, as in the reference (mrcal.c:3106-3270); a point that cannot be inverted
// comes back with NaN x,y. This is what turns mrcal.optimize()'s observations_point_triangulated pixels
// into the rays of mrcal_observation_point_triangulated_t (mrcal-pywrap.c:1383-1401)
bool mrcal_unproject(mrcal_point3_t* out, const mrcal_point2_t* q, int N,
                     const mrcal_lensmodel_t* lensmodel, const double* intrinsics);

// One evaluation of the cost function at the given (unpacked) seed:
//   b_packed <- packed state, x <- residuals, Jt <- CSR Jacobian dx/db_packed
// replaces mrcal.h:539-609 (mrcal.c:5972-6177). Buffer sizes are in BYTES and
// must match exactly. Jt may be NULL. Returns false (with a message on stderr)
// on any error, including "no usable CUDA device"
bool mrcal_optimizer_callback(double* b_packed, int buffer_size_b_packed,
                              double* x,        int buffer_size_x,
                              mrcal_b200_sparse_t* Jt,
                              const double*                 intrinsics,
                              const mrcal_pose_t*           rt_cam_ref,
                              const mrcal_pose_t*           rt_ref_frame,
                              const mrcal_point3_t*         points,
                              const mrcal_calobject_warp_t* calobject_warp,
                              int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                              int Npoints, int Npoints_fixed,
                              const mrcal_observation_board_t* observations_board,
                              const mrcal_observation_point_t* observations_point,
                              int Nobservations_board, int Nobservations_point,
                              const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                              int Nobservations_point_triangulated,
                              const mrcal_point3_t* observations_board_pool,
                              const mrcal_point3_t* observations_point_pool,
                              const mrcal_lensmodel_t* lensmodel,
                              const int* imagersizes,
                              mrcal_problem_selections_t       problem_selections,
                              const mrcal_problem_constants_t* problem_constants,
                              double calibration_object_spacing,
                              int calibration_object_width_n, int calibration_object_height_n,
                              bool verbose);

// The full solve. intrinsics, rt_cam_ref, rt_ref_frame, points, calobject_warp
// are a seed on input and the solution on output; observations_board_pool[].z
// is negated for newly-found outliers. b_packed_final / x_final may be NULL.
// replaces mrcal.h:453-521 (mrcal.c:6179-6624). On error
// stats.rms_reproj_error__pixels < 0. check_gradient is not supported (it is a
// libdogleg debugging facility, mrcal.c:6602-6605) and yields an error
mrcal_stats_t mrcal_optimize(double* b_packed_final, int buffer_size_b_packed_final,
                             double* x_final,        int buffer_size_x_final,
                             double*                 intrinsics,
                             mrcal_pose_t*           rt_cam_ref,
                             mrcal_pose_t*           rt_ref_frame,
                             mrcal_point3_t*         points,
                             mrcal_calobject_warp_t* calobject_warp,
                             int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                             int Npoints, int Npoints_fixed,
                             const mrcal_observation_board_t* observations_board,
                             const mrcal_observation_point_t* observations_point,
                             int Nobservations_board, int Nobservations_point,
                             const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                             int Nobservations_point_triangulated,
                             mrcal_point3_t* observations_board_pool,
                             mrcal_point3_t* observations_point_pool,
                             const mrcal_lensmodel_t* lensmodel,
                             const int* imagersizes,
                             mrcal_problem_selections_t       problem_selections,
                             const mrcal_problem_constants_t* problem_constants,
                             double calibration_object_spacing,
                             int calibration_object_width_n, int calibration_object_height_n,
                             bool verbose,
                             bool check_gradient);

////////////////////////////////////////////////////////////////////////////////
// Part 2. Extensions (no counterpart in the reference)
////////////////////////////////////////////////////////////////////////////////

// Version / build introspection. The string names the arch the kernels were
// compiled for ("sm_90a")
const char* mrcal_b200_version(void);
// Number of usable CUDA devices; 0 (never an error) when there is no GPU
int mrcal_b200_device_count(void);
// Message of the most recent failure in this thread ("" if none)
const char* mrcal_b200_last_error(void);

// Trust-region parameters. Defaults are libdogleg's, overridden the way
// mrcal_optimize() overrides them (mrcal.c:6289-6299)
typedef struct
{
    int    max_iterations;                   // 300
    double trustregion0;                     // 1e3
    double trustregion_decrease_factor;      // 0.1
    double trustregion_decrease_threshold;   // 0.25
    double trustregion_increase_factor;      // 2.0
    double trustregion_increase_threshold;   // 0.75
    double Jt_x_threshold;                   // 0
    double update_threshold;                 // 1e-7
    double trustregion_threshold;            // 0
} mrcal_b200_solver_parameters_t;
void mrcal_b200_default_solver_parameters(mrcal_b200_solver_parameters_t* parameters);

// Per-solve statistics beyond mrcal_stats_t
typedef struct
{
    int    Niterations;          // accepted trust-region steps
    int    Nevaluations;         // cost-function evaluations (residual+Jacobian kernels)
    int    Nfactorizations;      // Cholesky factorizations of the reduced system
    int    Nouter;               // outlier-rejection passes (>=1)
    int    Nreduced;             // order of the reduced (camera) system that was factored
    int    Nkernel_launches;     // launches of THIS library's kernels inside the solve
    int    Nsyncs;               // host waits on the device inside the solve (one per trust-region step)
    int    Ncollectives;         // NCCL all-reduce calls inside the solve (sharded solves)
    double norm2_x_initial, norm2_x_final;
    double ms_total;             // device time of the whole solve (CUDA events)
    double ms_evaluate;          // ... spent in residual/Jacobian kernels
    double ms_assemble;          // ... normal-equation assembly + Schur elimination
    double ms_factor;            // ... Cholesky
    double ms_solve;             // ... triangular solves + back-substitution
    double lambda_final;         // diagonal loading in use at the end (0 normally)
} mrcal_b200_solve_info_t;

// Device-resident problem. create() copies every input to the GPU once;
// optimize()/callback() then run without touching the host inputs again. This
// is what mrcal_optimize()/mrcal_optimizer_callback() are built from.
typedef struct mrcal_b200_problem mrcal_b200_problem_t;

// Arguments have the meaning they have in mrcal_optimize(). Returns NULL on error
mrcal_b200_problem_t*
mrcal_b200_problem_create(const double*                 intrinsics,
                          const mrcal_pose_t*           rt_cam_ref,
                          const mrcal_pose_t*           rt_ref_frame,
                          const mrcal_point3_t*         points,
                          const mrcal_calobject_warp_t* calobject_warp,
                          int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                          int Npoints, int Npoints_fixed,
                          const mrcal_observation_board_t* observations_board,
                          const mrcal_observation_point_t* observations_point,
                          int Nobservations_board, int Nobservations_point,
                          const mrcal_point3_t* observations_board_pool,
                          const mrcal_point3_t* observations_point_pool,
                          const mrcal_lensmodel_t* lensmodel,
                          const int* imagersizes,
                          mrcal_problem_selections_t problem_selections,
                          double calibration_object_spacing,
                          int calibration_object_width_n, int calibration_object_height_n);
// The same with triangulated-point observations (mrcal_optimize()'s observations_point_triangulated: rays in
// camera coordinates, sets closed by last_in_set; mrcal.c:5180-5653). Allowed only with the intrinsics locked
// and the extrinsics optimized, as in the reference (mrcal.c:6260-6275)
mrcal_b200_problem_t*
mrcal_b200_problem_create_triangulated(const double*                 intrinsics,
                          const mrcal_pose_t*           rt_cam_ref,
                          const mrcal_pose_t*           rt_ref_frame,
                          const mrcal_point3_t*         points,
                          const mrcal_calobject_warp_t* calobject_warp,
                          int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                          int Npoints, int Npoints_fixed,
                          const mrcal_observation_board_t* observations_board,
                          const mrcal_observation_point_t* observations_point,
                          int Nobservations_board, int Nobservations_point,
                          const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                          int Nobservations_point_triangulated,
                          const mrcal_point3_t* observations_board_pool,
                          const mrcal_point3_t* observations_point_pool,
                          const mrcal_lensmodel_t* lensmodel,
                          const int* imagersizes,
                          mrcal_problem_selections_t problem_selections,
                          double calibration_object_spacing,
                          int calibration_object_width_n, int calibration_object_height_n);
void mrcal_b200_problem_destroy(mrcal_b200_problem_t* problem);

int mrcal_b200_problem_num_states      (const mrcal_b200_problem_t* problem);
int mrcal_b200_problem_num_measurements(const mrcal_b200_problem_t* problem);
int mrcal_b200_problem_num_j_nonzero   (const mrcal_b200_problem_t* problem);

// Reset the device state to the seed given at create() (or to a new packed
// state, if b_packed != NULL) and restore the observation weights. Lets one
// handle run the same solve repeatedly
bool mrcal_b200_problem_reset(mrcal_b200_problem_t* problem, const double* b_packed);

// Re-upload the inputs a solve consumes (seed + observation pool) from host
// memory into an existing handle; the shapes must match create()
bool mrcal_b200_problem_upload(mrcal_b200_problem_t* problem,
                               const double* intrinsics, const mrcal_pose_t* rt_cam_ref,
                               const mrcal_pose_t* rt_ref_frame, const mrcal_point3_t* points,
                               const mrcal_calobject_warp_t* calobject_warp,
                               const mrcal_point3_t* observations_board_pool,
                               const mrcal_point3_t* observations_point_pool);

// Evaluate at the current device state. Any output may be NULL. Host buffers
bool mrcal_b200_problem_callback(mrcal_b200_problem_t* problem,
                                 double* b_packed, double* x,
                                 int32_t* Jrowptr, int32_t* Jcolidx, double* Jval);

// Run the trust-region solve on the device. parameters may be NULL (defaults).
// info may be NULL. Nothing is copied to the host except a few scalars per
// iteration
bool mrcal_b200_problem_optimize(mrcal_b200_problem_t* problem,
                                 const mrcal_b200_solver_parameters_t* parameters,
                                 mrcal_stats_t* stats, mrcal_b200_solve_info_t* info);

// Introspection (tests, debugging): the reduced normal equations at the current
// state, after the frame/point blocks have been eliminated. n_reduced <- number
// of shared unknowns; S_out [n_reduced][n_reduced] row-major, LOWER triangle
// valid; g_reduced [n_reduced]; g_full [Nstate] = J'x. Any output may be NULL
bool mrcal_b200_problem_reduced_system(mrcal_b200_problem_t* problem, double lambda, int* n_reduced,
                                       double* S_out, double* g_reduced, double* g_full);

// Copy results to the host: the packed state, the residuals, the unpacked
// solution and the (possibly outlier-marked) board observation pool. Any may be NULL
bool mrcal_b200_problem_download(mrcal_b200_problem_t* problem,
                                 double* b_packed, double* x,
                                 double* intrinsics, mrcal_pose_t* rt_cam_ref,
                                 mrcal_pose_t* rt_ref_frame, mrcal_point3_t* points,
                                 mrcal_calobject_warp_t* calobject_warp,
                                 mrcal_point3_t* observations_board_pool);

// Outlier flags of the triangulated-point observations as they stand on the device (outlier rejection
// adds to the flags the caller passed; the reference writes them into its input array,
// mrcal.c:4231-4232,4370-4371). flags: [N] ints, may be NULL. Returns the number of observations; <0 on error
int mrcal_b200_problem_triangulated_outliers(mrcal_b200_problem_t* problem, int* flags, int N);

/* K = drt_ref_refperturbed/db_packed (icam_intrinsics < 0) or drt_cam_camperturbed/db_packed (that camera), shape
   (6, Nstate) row-major, zero outside the extrinsics / frames / points / calobject_warp columns: what
   mrcal.drt_cross_reprojection__dbpacked() returns (mrcal-pywrap.c:2016-2110), computed as the reference's
   internal entry point of the same name with a leading underscore defines it (mrcal.h:611-660, uncertainty.c:798-1577) from the Jacobian at the
   problem's current state, which is evaluated on the device by this call. The reference's entry point takes a CHOLMOD
   matrix of J on the host; this one takes the device-resident problem (the Jacobian never leaves the GPU). Refuses what
   the reference refuses (uncertainty.c:944-989). */
bool mrcal_b200_problem_drt_cross_reprojection__dbpacked(mrcal_b200_problem_t* problem, int icam_intrinsics, double* K /* [6][Nstate] */);

// Timing hook for benchmarks: run N cost-function evaluations (residuals +
// Jacobian) at the current state back to back, return the mean device time per
// evaluation in milliseconds (CUDA events on the library's stream); <0 on error
double mrcal_b200_problem_time_callback(mrcal_b200_problem_t* problem, int N, bool with_jacobian);

// Multi-GPU: one process per GPU; the frames (and their observations) are
// sharded across ranks by the caller, the shared state is replicated and this
// library all-reduces the reduced normal equations with NCCL each iteration.
// Protocol: rank 0 calls get_unique_id() and broadcasts the 128 bytes by any
// means (e.g. torch.distributed); every rank then calls comm_init()
bool mrcal_b200_nccl_get_unique_id(void* id128);
bool mrcal_b200_nccl_comm_init(const void* id128, int rank, int nranks, int device);
void mrcal_b200_nccl_comm_destroy(void);
// Attach a created problem to the communicator. frame_offset/Nframes_global
// describe where this rank's frames sit in the global frame list
bool mrcal_b200_problem_set_sharding(mrcal_b200_problem_t* problem,
                                     int frame_offset, int Nframes_global,
                                     int point_offset, int Npoints_global);

// The factorization object: the 4th return value of mrcal.optimizer_callback()
// and mrcal.CHOLMOD_factorization(J). replaces mrcal-pywrap.c:110-649.
// J is CSR, shape (Nrows, Ncols); the object holds a Cholesky factorization of
// JtJ on the GPU
typedef struct mrcal_b200_factorization mrcal_b200_factorization_t;
mrcal_b200_factorization_t*
mrcal_b200_factorization_create(const int32_t* Jrowptr, const int32_t* Jcolidx, const double* Jval,
                                int Nrows, int Ncols);
void mrcal_b200_factorization_destroy(mrcal_b200_factorization_t* factorization);
// out[i,:] = solve(JtJ, bt[i,:]) for each of the Nrhs rows of bt; shape (Nrhs, Ncols),
// row-major. Corresponds to solve_xt_JtJ_bt(bt, sys='A') (mrcal-pywrap.c:425-578)
bool mrcal_b200_factorization_solve_xt_JtJ_bt(mrcal_b200_factorization_t* factorization,
                                              double* out, const double* bt, int Nrhs);
// The other systems of solve_xt_JtJ_bt(bt, sys=...) (mrcal-pywrap.c:467-493 -> cholmod_solve2). The
// factorization here is P JtJ P' = L D L' with P = I, D = I and L the Cholesky factor: A and LDLt solve the
// whole system, LD and L solve L x = b, DLt and Lt solve L' x = b, D, P and Pt copy. CHOLMOD's own P and D
// differ, the identities between the systems (what mrcal/model_analysis.py:837-841 relies on) hold
enum { MRCAL_B200_SYS_A = 0, MRCAL_B200_SYS_LDLt, MRCAL_B200_SYS_LD, MRCAL_B200_SYS_DLt, MRCAL_B200_SYS_L,
       MRCAL_B200_SYS_Lt, MRCAL_B200_SYS_D, MRCAL_B200_SYS_P, MRCAL_B200_SYS_Pt };
bool mrcal_b200_factorization_solve_sys(mrcal_b200_factorization_t* factorization,
                                        double* out, const double* bt, int Nrhs, int sys);
// Reciprocal condition-number estimate from the diagonal of the factor, as
// cholmod_rcond() defines it (mrcal-pywrap.c:580-593)
double mrcal_b200_factorization_rcond(mrcal_b200_factorization_t* factorization);
// The same object for the calibration problem the LAST mrcal_optimizer_callback() call evaluated, built from the
// problem's structure (per-frame/point blocks eliminated, dense factor of the reduced camera system only) instead of a
// dense Nstate x Nstate matrix: what mrcal-pywrap.c:1980-1988 does with the Jt it just filled. Takes over the device
// problem that call left behind. NULL if there is none or if JtJ is not positive definite (see mrcal_b200_last_error())
mrcal_b200_factorization_t* mrcal_b200_factorization_create_from_last_callback(void);

// A sparse Jacobian held on the GPU, for the consumers downstream of the solve (the reference's
// projection-uncertainty code, mrcal/model_analysis.py:716-870). J is CSR, shape (Nrows, Ncols), given as the
// reference gives it: p/i/x = indptr/indices/data of a scipy.sparse.csr_matrix = the arrays of the cholmod_sparse Jt.
typedef struct mrcal_b200_csr mrcal_b200_csr_t;
mrcal_b200_csr_t* mrcal_b200_csr_create(const int32_t* Jrowptr, const int32_t* Jcolidx, const double* Jval, int Nrows, int Ncols);
void mrcal_b200_csr_destroy(mrcal_b200_csr_t* J);
// out[Ncols] = Jt xt.  replaces _Jt_x, mrcal-genpywrap.py:640-731. Every output sums its column in row order, like
// the reference's loop: the result is bit-identical to the reference's
bool mrcal_b200_csr_Jt_x(mrcal_b200_csr_t* J, double* out, const double* xt);
// out[Nx][Nx] = A Jt J At over the Nleading_rows_J leading rows of J; A is (Nx, Ncols) row-major.
// replaces _A_Jt_J_At and _A_Jt_J_At__2, mrcal-genpywrap.py:477-638
bool mrcal_b200_csr_A_Jt_J_At(mrcal_b200_csr_t* J, double* out, const double* A, int Nx, int Nleading_rows_J);

#ifdef __cplusplus
}
#endif
