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

// replaces image.h:68-80 (the two image types stereo.h uses): w x h pixels, rows stride BYTES apart
typedef struct
{
    union { struct { int w, h; }; struct { int width, height; }; struct { int cols, rows; }; };
    int stride;
    uint16_t* data;
} mrcal_image_uint16_t;
typedef struct
{
    union { struct { int w, h; }; struct { int width, height; }; struct { int cols, rows; }; };
    int stride;
    double* data;
} mrcal_image_double_t;

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
/* The unprojection of N pixels with its gradients, as mrcal.unproject(normalize=, get_gradients=) returns it
   (mrcal/projections.py:112-397). dv_dq (N,3,2) and dv_dintrinsics (N,3,Nintrinsics; dense) may be NULL. With neither,
   v is mrcal_unproject()'s, or with normalize its unit vector (the zero vector where the unprojection failed). With
   either: the closed-form models (pinhole, stereographic, lonlat, latlon) give their closed-form ray and derivatives;
   the others give v = unproject_stereographic(project_stereographic(mrcal_unproject())) -- the same direction, a
   different magnitude where mrcal_unproject() flipped a point to the front -- with dv/dq = dv/du (dq/du)^-1 in its
   stereographic coordinates u, and dv/dintrinsics = -dv/dq dq/dintrinsics. normalize: unit rays and the gradients of
   the unit rays. A failed unprojection or a singular dq/du gives NaN. Refuses CAHVORE with E != 0. False +
   mrcal_b200_last_error() on refusal or failure */
bool mrcal_b200_unproject_with_gradients(mrcal_point3_t* v, double* dv_dq, double* dv_dintrinsics,
                                         const mrcal_point2_t* q, int N, const mrcal_lensmodel_t* lensmodel,
                                         const double* intrinsics, bool normalize);
/* mrcal_project(), or with MRCAL_B200_PROJECT_UNPROJECT mrcal_b200_unproject_with_gradients(), element-wise over a
   broadcast shape: each element of the ndim-dimensional shape `shape` projects its point `in` (3,) through its
   intrinsics row (Nintrinsics,), or unprojects its pixel `in` (2,). Every row has one lens model, `lensmodel`.
     flags: MRCAL_B200_PROJECT_GET_GRADIENTS   dout_din (2,3) or (3,2) and dout_dintrinsics (2 or 3,Nintrinsics; dense:
                                               the entries the projection does not touch are 0). Either may be NULL
            MRCAL_B200_PROJECT_UNPROJECT       unproject: out is the ray (3,)
            MRCAL_B200_PROJECT_NORMALIZE       (with UNPROJECT) unit rays, as mrcal_b200_unproject_with_gradients()
   The values, the NaN of a failed unprojection and the refusal of CAHVORE with E != 0 (in any row the call reads) are
   those of the single-intrinsics entries. Operand element at broadcast index (i_0 .. i_ndim-1) starts at
   in + sum_d i_d strides_in[d] (intrinsics + sum_d i_d strides_intrinsics[d]), in doubles; 0 where the operand is
   repeated along d, so no operand needs to be expanded, and is packed. Outputs are packed: output k of element e
   starts at out_k + e * (its size). ndim <= 8. False + mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_PROJECT_GET_GRADIENTS = 1, MRCAL_B200_PROJECT_UNPROJECT = 2, MRCAL_B200_PROJECT_NORMALIZE = 4 };
bool mrcal_b200_project(const mrcal_lensmodel_t* lensmodel, int flags, int ndim, const int64_t* shape,
                        const double* in, const int64_t* strides_in, const double* intrinsics,
                        const int64_t* strides_intrinsics, double* out, double* dout_din, double* dout_dintrinsics);
/* The same with every buffer on the device: the kernel is enqueued on stream (a cudaStream_t; NULL: the default
   stream) and the call returns without waiting for it, except when it unprojects with CAHVORE: then one flag per call
   comes back to the host to check every intrinsics row's E terms, and the call waits for the stream. shape and the
   strides stay on the host */
bool mrcal_b200_project_device(const mrcal_lensmodel_t* lensmodel, int flags, int ndim, const int64_t* shape,
                               const double* in, const int64_t* strides_in, const double* intrinsics,
                               const int64_t* strides_intrinsics, double* out, double* dout_din,
                               double* dout_dintrinsics, void* stream);
/* The angular resolution of a camera in degrees per pixel at N pixels, as mrcal.model_resolution__deg_pixel()
   computes it (mrcal/model_analysis.py:2152-2246): from the eigenvalues of M'M, M = dq/dv [u0 u1] at the unit ray v
   of each pixel, [u0 u1] an orthonormal basis of the plane perpendicular to v, the smaller one clamped at 1e-6. mode:
   one of MB200_RESOLUTION_*. One fused kernel. Refuses CAHVORE with E != 0. False + mrcal_b200_last_error() on refusal
   or failure */
enum { MB200_RESOLUTION_MEAN = 0, MB200_RESOLUTION_MIN = 1, MB200_RESOLUTION_MAX = 2, MB200_RESOLUTION_ECCENTRICITY = 3 };
bool mrcal_b200_model_resolution__deg_pixel(double* resolution, const mrcal_point2_t* q, int N,
                                            const mrcal_lensmodel_t* lensmodel, const double* intrinsics, int mode);

// Stereo (replaces stereo.h:15-173, stereo.c:19-972, 1242-1417). Host buffers in and out, as in the reference.
// The geometry is host code; the maps and the ranges are computed on the device, one thread per element.
//
// replaces stereo.h:15-31: the resolution of a rectified view (rectification model LATLON, LONLAT or PINHOLE).
// pixels_per_deg_* < 0 asks for that multiple of camera 0's resolution at (az0, el0), which takes one device
// projection; LATLON and LONLAT then fit a whole number of pixels into the field of view
bool mrcal_rectified_resolution(double* pixels_per_deg_az, double* pixels_per_deg_el,
                                const mrcal_lensmodel_t* lensmodel, const double* intrinsics,
                                const mrcal_point2_t* azel_fov_deg, const mrcal_point2_t* azel0_deg,
                                const double* R_cam0_rect0, const mrcal_lensmodel_type_t rectification_model_type);
// replaces stereo.h:33-80: the rectified system of a stereo pair: imager (Naz, Nel), fxycxy, rt_rect0_ref and the
// baseline. Rectification model LATLON or PINHOLE; central models only (CAHVORE with E = 0). Of the autodetections
// only az0's is supported
bool mrcal_rectified_system2(unsigned int* imagersize_rectified, double* fxycxy_rectified, double* rt_rect0_ref,
                             double* baseline, double* pixels_per_deg_az, double* pixels_per_deg_el,
                             mrcal_point2_t* azel_fov_deg, mrcal_point2_t* azel0_deg,
                             const double az_edge_margin_deg,
                             const mrcal_lensmodel_t* lensmodel0, const double* intrinsics0,
                             const double* rt_cam0_ref, const double* rt_cam1_ref,
                             const mrcal_lensmodel_type_t rectification_model_type,
                             bool az0_deg_autodetect, bool el0_deg_autodetect,
                             bool az_fov_deg_autodetect, bool el_fov_deg_autodetect);
// replaces stereo.h:82-117: the legacy form, az_edge_margin_deg = 10
bool mrcal_rectified_system(unsigned int* imagersize_rectified, double* fxycxy_rectified, double* rt_rect0_ref,
                            double* baseline, double* pixels_per_deg_az, double* pixels_per_deg_el,
                            mrcal_point2_t* azel_fov_deg, mrcal_point2_t* azel0_deg,
                            const mrcal_lensmodel_t* lensmodel0, const double* intrinsics0,
                            const double* rt_cam0_ref, const double* rt_cam1_ref,
                            const mrcal_lensmodel_type_t rectification_model_type,
                            bool az0_deg_autodetect, bool el0_deg_autodetect,
                            bool az_fov_deg_autodetect, bool el_fov_deg_autodetect);
// replaces stereo.h:119-135: rectification_maps (2, Nel, Naz, 2) float32: for each camera and rectified pixel, the
// pixel of that camera that sees the same ray
bool mrcal_rectification_maps(float* rectification_maps,
                              const mrcal_lensmodel_t* lensmodel0, const double* intrinsics0, const double* r_cam0_ref,
                              const mrcal_lensmodel_t* lensmodel1, const double* intrinsics1, const double* r_cam1_ref,
                              const mrcal_lensmodel_type_t rectification_model_type,
                              const double* fxycxy_rectified, const unsigned int* imagersize_rectified,
                              const double* r_rect0_ref);
// replaces stereo.h:137-152: range[N] of disparities at rectified pixels qrect0; 0 where d <= 0, d is outside
// [disparity_min, disparity_max] or the range is not finite
bool mrcal_stereo_range_sparse(double* range, const double* disparity, const mrcal_point2_t* qrect0, const int N,
                               const double disparity_min, const double disparity_max,
                               const mrcal_lensmodel_type_t rectification_model_type,
                               const double* fxycxy_rectified, const double baseline);
// replaces stereo.h:154-170: the same for a whole disparity image of scaled uint16 values
bool mrcal_stereo_range_dense(mrcal_image_double_t* range, const mrcal_image_uint16_t* disparity_scaled,
                              const uint16_t disparity_scale,
                              const uint16_t disparity_scaled_min, const uint16_t disparity_scaled_max,
                              const mrcal_lensmodel_type_t rectification_model_type,
                              const double* fxycxy_rectified, const double baseline);

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
// The same, with the board observations' blocks from the fused evaluation (the
// path mrcal_b200_problem_optimize() takes for splined models with the core
// locked) instead of the stored Jacobian. False if this problem does not take it
bool mrcal_b200_problem_reduced_system_fused(mrcal_b200_problem_t* problem, double lambda, int* n_reduced,
                                             double* S_out, double* g_reduced, double* g_full);
// Introspection: the two sums of the Cauchy step at the current state, out[0] = |g|^2 and
// out[1] = |J g|^2 with g = J'x, from the kernels a step of mrcal_b200_problem_optimize()
// runs: with fused, the board rows of J g from the fused evaluation's blocks and the other
// rows from their Jacobian rows (false if this problem does not take that path); without,
// every row from the stored Jacobian
bool mrcal_b200_problem_cauchy_denominator(mrcal_b200_problem_t* problem, bool fused, double* out);

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

/* Projection uncertainty, as mrcal.projection_uncertainty(what='covariance') computes it (mrcal/model_analysis.py:1192-1517):
   Var(q) [N][2][2] of the projections of the camera-frame points p_cam [N] by camera icam_intrinsics, propagated from
   the noise of the pixel observations through the solve, at the problem's current state. method: one of the enum
   below (the reference's 'mean-pcam', 'cross-reprojection-rrp-Jfp', 'cross-reprojection-ccp'). atinfinity: the
   points are directions; only the rotations propagate. observed_pixel_uncertainty <= 0: estimated from the residuals
   (model_analysis.py:491-556); the value used is returned in *sigma_used (may be NULL). Evaluation, factorization,
   the dF/db rows, the solves and the reductions all run on the device; only Var comes back. Refuses what the
   reference refuses, and sharded problems. False + mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_UNCERTAINTY_MEAN_PCAM = 0, MRCAL_B200_UNCERTAINTY_RRP_JFP, MRCAL_B200_UNCERTAINTY_CCP };
bool mrcal_b200_problem_projection_uncertainty(mrcal_b200_problem_t* problem, int icam_intrinsics, int method,
                                               bool atinfinity, const mrcal_point3_t* p_cam, int N,
                                               double observed_pixel_uncertainty, double* Var, double* sigma_used);

/* The same for several cameras from ONE evaluation and factorization of the problem: camera icam_intrinsics[c] gets
   N[c] points; p_cam and Var [sum N][2][2] hold every camera's points, camera after camera. Each camera's Var is what
   mrcal_b200_problem_projection_uncertainty() gives for it alone, bit for bit: the same kernels run in the same order.
   The observed-pixel uncertainty is estimated once (or given) and shared. False + mrcal_b200_last_error() if the
   method or any camera is refused, or on failure */
bool mrcal_b200_problem_projection_uncertainty_cameras(mrcal_b200_problem_t* problem, const int* icam_intrinsics,
                                                       const int* N, int Ncameras, int method, bool atinfinity,
                                                       const mrcal_point3_t* p_cam, double observed_pixel_uncertainty,
                                                       double* Var, double* sigma_used);

/* The observed-pixel uncertainty estimated from the residuals at the problem's current state
   (mrcal.model_analysis._observed_pixel_uncertainty_from_inputs(), model_analysis.py:491-556): the estimate, and the
   evaluation behind it, that mrcal_b200_problem_projection_uncertainty() makes, so *sigma is bit for bit the
   *sigma_used it returns. False + mrcal_b200_last_error() without board or point observations, or on failure */
bool mrcal_b200_problem_observed_pixel_uncertainty(mrcal_b200_problem_t* problem, double* sigma);

/* Residual statistics binned by imager cell, as mrcal.calibration._report_regional_statistics() computes them
   (mrcal/calibration.py:1720-1866), for the cameras icam_intrinsics [Ncameras] in one launch. q_cell_center
   [Ncameras][gridn_height][gridn_width][2]: each camera's cell centres (mrcal.sample_imager()); rcell [Ncameras][2]:
   each camera's cell half-size. A board corner counts in a cell when its observation is of that camera, its weight
   is > 0 and its observed pixel q has |q - centre| < rcell on both axes; its weighted x and y residuals both count.
   stats [Ncameras][gridn_height][gridn_width][3] = (mean, population stdev, count), (0, 0, count) where count <= 5.
   evaluate: evaluate the residuals at the problem's current state first; false: use those of the last evaluation
   (the last callback, solve or projection-uncertainty call). x [Nmeasurements] (may be NULL) receives the residuals
   used. Sums in a fixed order: two calls give the same bits. False + mrcal_b200_last_error() on refusal or failure */
bool mrcal_b200_problem_regional_statistics(mrcal_b200_problem_t* problem, const int* icam_intrinsics, int Ncameras,
                                            int gridn_width, int gridn_height, const double* q_cell_center,
                                            const double* rcell, bool evaluate, double* stats, double* x);

/* The transformation implied by two cameras' intrinsics, as mrcal.implied_Rt10__from_unprojections() fits it
   (mrcal/model_analysis.py:27-395): Rt10 [4][3] (R then t; t = 0 if atinfinity) minimizing the huber-robust sum over the
   points (m, i) in the focus region (|q0[i] - focus_center|^2 < focus_radius^2) of (w[m][i] th2)^2, th2 = 2 (1 -
   cos(angle between R p0[m][i] + t and v1[i])). p0 [M][N]: unit vectors if atinfinity, else points; v1 [N]: unit
   vectors; weights [M][N] or NULL for 1. Points with a non-finite p0, v1 or weight are ignored. One CTA on the device
   runs the whole fit. False + mrcal_b200_last_error() on refusal ("Focus region contained too few points": fewer than
   3) or failure */
bool mrcal_b200_implied_Rt10__from_unprojections(double* Rt10, const mrcal_point2_t* q0, int N, const mrcal_point3_t* p0,
                                                 int M, const mrcal_point3_t* v1, const double* weights, bool atinfinity,
                                                 const double* focus_center, double focus_radius);

/* The projection difference of Nmodels >= 2 camera models over a grid, as mrcal.projection_diff() computes it after
   its unprojection (mrcal/model_analysis.py:1520-1928). q0 [N]: the grid; v [Nmodels][N]: its unit rays unprojected
   by each model; distance [Nd], or NULL for infinity (Nd = 1); lensmodels [Nmodels] and their intrinsics, concatenated
   in model order. If fit_Rt10, Rt10 [Nmodels-1][4][3] is fitted for each pair (0, k) as
   mrcal_b200_implied_Rt10__from_unprojections() does, with p0 = v[0] * distance, v1 = v[k] and, if uncertainties
   [Nmodels][Nd][N] (worst-direction stdev of each model's projection of v[k] * distance) is given, the weights
   (1/(u_0 u_k))^2; all pairs in one launch. Otherwise Rt10 is read. Then q_k = project_k(R_k v[0] distance + t_k):
   with 2 models difflen [Nd][N] = |q_1 - q0| and diff [Nd][N][2] = q_1 - q0 (may be NULL); with more, difflen =
   sqrt(mean_k |q_k - q0|^2). Each grid-sized array crosses the bus once each way. False + mrcal_b200_last_error() on
   refusal or failure */
bool mrcal_b200_projection_diff(double* Rt10, double* difflen, double* diff,
                                const mrcal_point2_t* q0, int N, const mrcal_point3_t* v, int Nmodels,
                                const double* distance, int Nd,
                                const mrcal_lensmodel_t* lensmodels, const double* intrinsics,
                                const double* uncertainties, const double* focus_center, double focus_radius,
                                bool fit_Rt10);

/* The reprojection of pixels q [N] from camera 0 to camera 1 of Npairs (1 or 2) camera pairs, as mrcal.stereo_pair_diff()
   computes it (mrcal/model_analysis.py:1931-2103): q1_p = project_p1(R_p (distance unproject_p0(q, normalized)) + t_p)
   with Rt10 [Npairs][4][3] (R, then t). lensmodels [Npairs][2] and their intrinsics, concatenated in that order. out
   [N][2] is q1_0 for one pair and q1_1 - q1_0 for two; outlen [N] (may be NULL) is |out|. Refuses a camera 0 that is
   CAHVORE with E != 0. False + mrcal_b200_last_error() on refusal or failure */
bool mrcal_b200_stereo_pair_reproject(double* out, double* outlen, const mrcal_point2_t* q, int N, int Npairs,
                                      const mrcal_lensmodel_t* lensmodels, const double* intrinsics, const double* Rt10,
                                      double distance);

// The point cloud of disparities in rectified camera-0 coordinates, as mrcal.stereo_unproject() computes it
// (mrcal/stereo.py:1453-1607) in one pass on the device: p[k] = range[k] * normalize(unproject_rect(qrect0[k])),
// (0,0,0) where the range is 0. Exactly one source of ranges is given:
// - disparity_scaled: a whole image, as mrcal_stereo_range_dense() reads it; qrect0 is its pixel grid, p is (h, w)
// - disparity [N]: as mrcal_stereo_range_sparse() reads it, with disparity_min, disparity_max
// - ranges [N]: given
// With the last two, qrect0 [N], or NULL for the pixel grid of width W (N a multiple of W). range [N] receives the
// ranges (may be NULL). False + mrcal_b200_last_error() on refusal or failure
bool mrcal_b200_stereo_unproject(mrcal_point3_t* p, double* range,
                                 const mrcal_image_uint16_t* disparity_scaled, uint16_t disparity_scale,
                                 uint16_t disparity_scaled_min, uint16_t disparity_scaled_max,
                                 const double* disparity, const double* ranges, const mrcal_point2_t* qrect0,
                                 int N, int W, double disparity_min, double disparity_max,
                                 mrcal_lensmodel_type_t rectification_model_type,
                                 const double* fxycxy_rectified, double baseline);

/* The reprojection map between two camera models, as mrcal.image_transformation_map() computes it
   (mrcal/image_transforms.py:276-511): mapxy [H_to][W_to][2] (float32) is, for each pixel of model_to's imager, the
   pixel of model_from that sees the same point. Each pixel is unprojected through model_to, then
   - Rt_to_from [4][3] (R, then t) NULL: the cameras share their frame (intrinsics_only)
   - plane_n [3] given: A_from_to v, with A_to_from = plane_d R_to_from + t_to_from plane_n'
   - distance given: invert_Rt(Rt_to_from) applied to normalize(v) * (*distance)
   - otherwise (at infinity): R_to_from' v
   and projected through model_from in fp64. region [Nregion] (a closed polygon in model_from's pixels) or NULL: map
   points outside it, by the even-odd rule, and NaN points become (-1, -1). Two passes on the device, one thread per
   pixel. Refuses a CAHVORE model_to with E != 0. False + mrcal_b200_last_error() on refusal or failure */
bool mrcal_b200_image_transformation_map(float* mapxy, int W_to, int H_to,
                                         const mrcal_lensmodel_t* lensmodel_from, const double* intrinsics_from,
                                         const mrcal_lensmodel_t* lensmodel_to, const double* intrinsics_to,
                                         const double* Rt_to_from, const double* distance,
                                         const double* plane_n, double plane_d,
                                         const mrcal_point2_t* region, int Nregion);

/* Which of the points q [N] lie strictly inside the closed polygon region [Nregion], as
   mrcal.is_within_valid_intrinsics_region() (shapely's Polygon.contains()) decides it: mask[i] is false for a point
   on an edge or a vertex (an exact test for integer coordinates), for a NaN point, and for every point if Nregion is
   0; otherwise the even-odd rule decides. Any number of vertices. One thread per point on the device. False +
   mrcal_b200_last_error() on failure */
bool mrcal_b200_is_within_region(bool* mask, const mrcal_point2_t* q, int N, const mrcal_point2_t* region, int Nregion);

/* An image remapped through a map, as mrcal.transform_image() (cv2.remap()) computes it, pixel for pixel: out
   [H_out][W_out][channels] (packed) from image [H][W][channels] (rows image_stride bytes apart) and mapxy
   [H_out][W_out][2] (float32, packed). type: an MRCAL_B200_IMAGE_* element type; channels: 1 or 3; interpolation:
   MRCAL_B200_INTER_*; border_mode: MRCAL_B200_BORDER_* (OpenCV's values). border_value [channels]: the value of
   pixels outside the image under BORDER_CONSTANT. Under BORDER_TRANSPARENT those output pixels keep what out held.
   One thread per output pixel. False + mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_IMAGE_UINT8 = 0, MRCAL_B200_IMAGE_UINT16 = 1, MRCAL_B200_IMAGE_FLOAT = 2 };
enum { MRCAL_B200_INTER_NEAREST = 0, MRCAL_B200_INTER_LINEAR = 1 };
enum { MRCAL_B200_BORDER_CONSTANT = 0, MRCAL_B200_BORDER_TRANSPARENT = 5 };
bool mrcal_b200_transform_image(void* out, const void* image, int W, int H, int image_stride, int type, int channels,
                                const float* mapxy, int W_out, int H_out, int interpolation, int border_mode,
                                const double* border_value);
/* The same with every buffer on the device: the kernel is enqueued on stream (a cudaStream_t; NULL: the default
   stream) and the call returns without waiting for it. image, out and image_stride must be aligned to the element
   size, mapxy to 4 bytes (a float); a buffer that is not is refused */
bool mrcal_b200_transform_image_device(void* out, const void* image, int W, int H, int image_stride, int type,
                                       int channels, const float* mapxy, int W_out, int H_out, int interpolation,
                                       int border_mode, const double* border_value, void* stream);

/* Template matching for M features in one call, as mrcal.match_feature() computes it with cv2.matchTemplate(): the
   device part, after the host has decided which features can be matched. image0 [H0][W0] and image1 [H1][W1] (rows
   stride0, stride1 bytes apart) are both MRCAL_B200_IMAGE_UINT8 or both MRCAL_B200_IMAGE_FLOAT. Feature i is
   features[6i..6i+5] = (tx, ty, cx, cy, cw, ch): its template's top-left pixel in image 1 and its search cut of image
   1, cw x ch pixels at (cx, cy), inside image 1 and at least template_w x template_h; and Hinv[9i..9i+8], the float32
   inverse of its homography H10 (row-major). The template is image0 remapped (INTER_LINEAR, BORDER_CONSTANT 0) through
   apply_homography(Hinv, q1) of the template's pixels q1; its match output has (ch - template_h + 1) rows of
   (cw - template_w + 1) values of method (OpenCV's TM_* values, 0..5). out: M rows of 4 doubles (the sub-pixel
   optimum's x and y in match-output coordinates and its value, NaN unless the status is MRCAL_B200_MATCH_OK; the
   status), then M slots of slot_w * slot_h float32, each starting with its feature's packed match output. No output
   may exceed its slot. templates: NULL, or M * template_h * template_w elements of the image type. False +
   mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_MATCH_OK = 0, MRCAL_B200_MATCH_EDGE_PEAK = 1, MRCAL_B200_MATCH_OUTSIDE_IMAGE1 = 2,
       MRCAL_B200_MATCH_OUTSIDE_IMAGE0 = 3, MRCAL_B200_MATCH_SEARCH_TOO_SMALL = 4 };
bool mrcal_b200_match_feature(double* out, void* templates, const void* image0, int W0, int H0, int stride0,
                              const void* image1, int W1, int H1, int stride1, int type, const int* features,
                              const float* Hinv, int M, int template_w, int template_h, int slot_w, int slot_h,
                              int method);
/* The same with image0 and image1 on the device, aligned to their element: the work is enqueued on stream (a
   cudaStream_t; NULL: the default stream), and the call returns once out and templates (host memory) are written */
bool mrcal_b200_match_feature_device(double* out, void* templates, const void* image0, int W0, int H0, int stride0,
                                     const void* image1, int W1, int H1, int stride1, int type, const int* features,
                                     const float* Hinv, int M, int template_w, int template_h, int slot_w, int slot_h,
                                     int method, void* stream);

/* The pose utilities of mrcal.poseutils, element-wise over a broadcast shape: one operation `op`
   (MRCAL_B200_POSE_*) applied to every element of the ndim-dimensional shape `shape`. Each operation takes one or two
   inputs and gives a value and, with MRCAL_B200_POSE_GET_GRADIENTS, one or two gradients, in the reference's layouts
   (mrcal/poseutils.py):

     op                    inputs       value  gradients
     R_FROM_r              r            R      dR/dr (3,3,3)
     r_FROM_R              R            r      dr/dR (3,3,3)
     Rt_FROM_rt            rt           Rt     dR/dr (3,3,3)
     rt_FROM_Rt            Rt           rt     dr/dR (3,3,3)
     INVERT_R, INVERT_Rt   R, Rt        R, Rt
     INVERT_rt             rt           rt     drt_out/drt_in (6,6)
     COMPOSE_Rt            Rt0, Rt1     Rt                                         inverted0, inverted1
     COMPOSE_r             r0, r1       r      dr/dr0 (3,3), dr/dr1 (3,3)          inverted0, inverted1
     COMPOSE_rt            rt0, rt1     rt     drt/drt0 (6,6), drt/drt1 (6,6)      inverted0, inverted1
     COMPOSE_r_TINYr0      r1           dr/dr0 (3,3) at r0 = 0
     COMPOSE_r_TINYr1      r0           dr/dr1 (3,3) at r1 = 0
     COMPOSE_rt_TINYrt0    rt1          drt/drt0 (6,6) at rt0 = 0
     COMPOSE_rt_TINYrt1    rt0          drt/drt1 (6,6) at rt1 = 0
     ROTATE_POINT_r        r, x         x      dx/dr (3,3), dx/dx_in (3,3)         inverted (as inverted0)
     ROTATE_POINT_R        R, x         x      dx/dR (3,3,3), dx/dx_in (3,3)       inverted
     TRANSFORM_POINT_rt    rt, x        x      dx/drt (3,6), dx/dx_in (3,3)        inverted
     TRANSFORM_POINT_Rt    Rt, x        x      dx/dRt (3,4,3), dx/dx_in (3,3)      inverted
     SKEW_SYMMETRIC        a            (3,3)
     R_FROM_QUAT           q (w,x,y,z)  R
     QUAT_FROM_R           R            q
     QT_FROM_Rt, Rt_FROM_qt             qt (7,) <-> Rt
     R_ALIGNED_TO_VECTOR   v            R

   Gradients are taken with respect to the inputs as passed, inverted or not. Input k's element at broadcast index
   (i_0 .. i_ndim-1) starts at in_k + sum_d i_d strides_k[d] (in doubles; 0 where input k is repeated along d, so no
   input needs to be expanded) and is packed. Outputs are packed: output k of element e starts at out_k + e * (its
   size). NULL for an input or output the operation does not have. ndim <= 8. A NaN input gives NaN outputs. False +
   mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_POSE_R_FROM_r = 0, MRCAL_B200_POSE_r_FROM_R, MRCAL_B200_POSE_Rt_FROM_rt, MRCAL_B200_POSE_rt_FROM_Rt,
       MRCAL_B200_POSE_INVERT_R, MRCAL_B200_POSE_INVERT_Rt, MRCAL_B200_POSE_INVERT_rt, MRCAL_B200_POSE_COMPOSE_Rt,
       MRCAL_B200_POSE_COMPOSE_r, MRCAL_B200_POSE_COMPOSE_rt, MRCAL_B200_POSE_COMPOSE_r_TINYr0,
       MRCAL_B200_POSE_COMPOSE_r_TINYr1, MRCAL_B200_POSE_COMPOSE_rt_TINYrt0, MRCAL_B200_POSE_COMPOSE_rt_TINYrt1,
       MRCAL_B200_POSE_ROTATE_POINT_r, MRCAL_B200_POSE_ROTATE_POINT_R, MRCAL_B200_POSE_TRANSFORM_POINT_rt,
       MRCAL_B200_POSE_TRANSFORM_POINT_Rt, MRCAL_B200_POSE_SKEW_SYMMETRIC, MRCAL_B200_POSE_R_FROM_QUAT,
       MRCAL_B200_POSE_QUAT_FROM_R, MRCAL_B200_POSE_QT_FROM_Rt, MRCAL_B200_POSE_Rt_FROM_qt,
       MRCAL_B200_POSE_R_ALIGNED_TO_VECTOR, MRCAL_B200_POSE_NUM_OPS };
enum { MRCAL_B200_POSE_GET_GRADIENTS = 1, MRCAL_B200_POSE_INVERTED0 = 2, MRCAL_B200_POSE_INVERTED1 = 4 };
bool mrcal_b200_poseutils(int op, int flags, int ndim, const int64_t* shape, const double* in0, const int64_t* strides0,
                          const double* in1, const int64_t* strides1, double* out0, double* out1, double* out2);
/* The same with every buffer on the device: the kernel is enqueued on stream (a cudaStream_t; NULL: the default
   stream) and the call returns without waiting for it. shape and the strides stay on the host */
bool mrcal_b200_poseutils_device(int op, int flags, int ndim, const int64_t* shape, const double* in0,
                                 const int64_t* strides0, const double* in1, const int64_t* strides1, double* out0,
                                 double* out1, double* out2, void* stream);

/* The two-view triangulation routines of mrcal.triangulation, element-wise over a broadcast shape: one method
   (MRCAL_B200_TRIANGULATE_*) applied to every element of the ndim-dimensional shape `shape`, with the reference's
   inputs and output layouts (mrcal/triangulation.py, triangulation-genpywrap.py):

     method                        inputs                            value    gradients
     GEOMETRIC, LEECIVERA_L1,      v0, v1, t01 (camera-0 coords)     p (3,)   dp/dv0 (3,3), dp/dv1 (3,3), dp/dt01 (3,3)
     LEECIVERA_LINF, _MID2, _WMID2
     LINDSTROM                     v0, v1 (local), Rt01 (4,3)        p (3,)   dp/dv0 (3,3), dp/dv1 (3,3), dp/dRt01 (3,4,3)
     TRIANGULATED_ERROR            v0, v1, t01 (camera-0 coords)     err ()   derr/dv1 (3,), derr/dt01 (3,)

   In each gradient, entry [i, j] is dp_i/dx_j. TRIANGULATED_ERROR is the solver's measurement of a triangulated
   point (_mrcal_triangulated_error()); it has no gradient in v0 and no fourth output. Where a method fails (parallel
   or divergent rays, a point behind a camera) p is (0,0,0), as in the reference, and its gradients are written as
   zeros: the reference leaves them unwritten. Input k's element at broadcast index (i_0 .. i_ndim-1) starts at
   in_k + sum_d i_d strides_k[d] (in doubles; 0 where input k is repeated along d, so no input needs to be expanded)
   and is packed. Outputs are packed: output k of element e starts at out_k + e * (its size). NULL for an output
   the call does not have. ndim <= 8. False + mrcal_b200_last_error() on refusal or failure */
enum { MRCAL_B200_TRIANGULATE_GEOMETRIC = 0, MRCAL_B200_TRIANGULATE_LEECIVERA_L1, MRCAL_B200_TRIANGULATE_LEECIVERA_LINF,
       MRCAL_B200_TRIANGULATE_LEECIVERA_MID2, MRCAL_B200_TRIANGULATE_LEECIVERA_WMID2, MRCAL_B200_TRIANGULATE_LINDSTROM,
       MRCAL_B200_TRIANGULATE_TRIANGULATED_ERROR, MRCAL_B200_TRIANGULATE_NUM_METHODS };
enum { MRCAL_B200_TRIANGULATE_GET_GRADIENTS = 1 };
bool mrcal_b200_triangulate(int method, int flags, int ndim, const int64_t* shape, const double* v0,
                            const int64_t* strides0, const double* v1, const int64_t* strides1,
                            const double* t01_or_Rt01, const int64_t* strides2, double* out0, double* out1,
                            double* out2, double* out3);
/* The same with every buffer on the device: the kernel is enqueued on stream (a cudaStream_t; NULL: the default
   stream) and the call returns without waiting for it. shape and the strides stay on the host */
bool mrcal_b200_triangulate_device(int method, int flags, int ndim, const int64_t* shape, const double* v0,
                                   const int64_t* strides0, const double* v1, const int64_t* strides1,
                                   const double* t01_or_Rt01, const int64_t* strides2, double* out0, double* out1,
                                   double* out2, double* out3, void* stream);

/* The projections behind mrcal.synthesize_board_observations() (mrcal/synthetic_data.py:236-554) for one chunk of
   Nframes board poses: Rt_ref_boardref [Nframes][4][3] = Rt_from_rt(rt_ref_boardref [Nframes][6]); for every frame,
   camera and corner of board [Npoints][3] (the centered board), q [Nframes][Ncameras][Npoints][2] =
   project(transform_point_Rt(Rt_cam_ref[c], transform_point_Rt(Rt_ref_boardref[f], corner))), two transforms as
   the reference makes them; Nvisible [Nframes][Ncameras] counts the corners with 0 <= q <= imagersize - 1 on both
   axes. Camera c has the lens model lensmodels[c], its intrinsics packed one camera after the other in intrinsics,
   Rt_cam_ref [Ncameras][4][3] and imagersizes [Ncameras][2] (width, height). The random poses, the culling and the
   selection of frames are the caller's. False + mrcal_b200_last_error() on refusal or failure */
bool mrcal_b200_synthesize_board_observations(double* q, int* Nvisible, double* Rt_ref_boardref,
                                              const double* rt_ref_boardref, int Nframes, const double* board,
                                              int Npoints, int Ncameras, const mrcal_lensmodel_t* lensmodels,
                                              const double* intrinsics, const double* Rt_cam_ref,
                                              const int* imagersizes);
/* The camera-frame board corners and the perfect observations of a problem, as mrcal.hypothesis_board_corner_positions()
   (mrcal/utils.py:440-584) and mrcal.make_perfect_observations() (mrcal/synthetic_data.py:594-750) compute them. For
   each board observation o (indices in the Python order: iframe, icam_intrinsics, icam_extrinsics) and each corner of
   board [Npoints_board][3] (ref_calibration_object() of the problem), pcam_board [o][corner][3] =
   transform_point_Rt(compose_Rt(Rt_cam_ref, Rt_ref_frame), corner), Rt_cam_ref the identity for icam_extrinsics = -1,
   and q_board [o][corner][2] its projection through the camera's intrinsics [Ncameras_intrinsics][Nintrinsics]. For
   each point observation (i_point, icam_intrinsics, icam_extrinsics), q_point [o][2] = the projection of
   transform_point_Rt(Rt_cam_ref, points[i_point]). Any of the three outputs may be NULL, but point observations need
   q_point; lensmodel and intrinsics are needed only to project. False + mrcal_b200_last_error() on refusal (an index
   out of range) or failure */
bool mrcal_b200_problem_corners(double* pcam_board, double* q_board, double* q_point,
                                const int32_t* indices_frame_camintrinsics_camextrinsics, int Nobservations_board,
                                const double* board, int Npoints_board,
                                const int32_t* indices_point_camintrinsics_camextrinsics, int Nobservations_point,
                                const double* points, int Npoints, const double* rt_ref_frame, int Nframes,
                                const double* rt_cam_ref, int Ncameras_extrinsics, const mrcal_lensmodel_t* lensmodel,
                                const double* intrinsics, int Ncameras_intrinsics);

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
