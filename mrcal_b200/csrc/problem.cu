// The device-resident problem: creation (one H2D of everything), evaluation at
// the current state, and readback. Part 2 of include/mrcal_b200.h.
#include "device_math.cuh"
#include "problem_impl.h"

namespace mb200 {

bool spline_segments_per_u(double* out, const mrcal_lensmodel_t* lm);   // layout.cpp

int lens_kind_of(const mrcal_lensmodel_t* lm)
{
    switch(lm->type)
    {
    case MRCAL_LENSMODEL_PINHOLE:       return LENS_PINHOLE;
    case MRCAL_LENSMODEL_STEREOGRAPHIC: return LENS_STEREOGRAPHIC;
    case MRCAL_LENSMODEL_LONLAT:        return LENS_LONLAT;
    case MRCAL_LENSMODEL_LATLON:        return LENS_LATLON;
    case MRCAL_LENSMODEL_OPENCV4:       return LENS_OPENCV4;
    case MRCAL_LENSMODEL_OPENCV5:       return LENS_OPENCV5;
    case MRCAL_LENSMODEL_OPENCV8:       return LENS_OPENCV8;
    case MRCAL_LENSMODEL_OPENCV12:      return LENS_OPENCV12;
    case MRCAL_LENSMODEL_CAHVOR:        return LENS_CAHVOR;
    case MRCAL_LENSMODEL_CAHVORE:       return LENS_CAHVORE;
    case MRCAL_LENSMODEL_SPLINED_STEREOGRAPHIC:
        return lm->LENSMODEL_SPLINED_STEREOGRAPHIC__config.order == 3 ? LENS_SPLINED3 :
               lm->LENSMODEL_SPLINED_STEREOGRAPHIC__config.order == 2 ? LENS_SPLINED2 : -1;
    default: return -1;
    }
}

template <typename T>
static bool upload(T* dst, const T* src, size_t n, cudaStream_t s)
{
    if(n == 0) return true;
    MB200_CUDA_CHECK(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, s));
    return true;
}

static bool pack_seed_host(mrcal_b200_problem* P, std::vector<double>* b,
                           const double* intrinsics, const mrcal_pose_t* rt_cam_ref, const mrcal_pose_t* rt_ref_frame,
                           const mrcal_point3_t* points, const mrcal_calobject_warp_t* warp)
{
    // b = value/scale, block by block (mrcal.c:3377-3439)
    const Layout& L = P->L;
    b->assign(L.Nstate, 0.);
    std::vector<double> scale(L.Nstate);
    fill_state_scales(scale.data(), L);
    int i = 0;
    for(int c = 0; c < L.d.Ncam_i; c++)
    {
        if(L.Ncore_state) for(int k = 0; k < 4; k++) { (*b)[i] = intrinsics[c * L.Nintr + k] / scale[i]; i++; }
        for(int k = 0; k < L.Ndist_state; k++)       { (*b)[i] = intrinsics[c * L.Nintr + 4 + k] / scale[i]; i++; }
    }
    if(L.i_extr0 >= 0)
        for(int k = 0; k < 6 * L.d.Ncam_e; k++) { (*b)[i] = ((const double*)rt_cam_ref)[k] / scale[i]; i++; }
    if(L.i_frame0 >= 0)
        for(int k = 0; k < 6 * L.d.Nframes; k++) { (*b)[i] = ((const double*)rt_ref_frame)[k] / scale[i]; i++; }
    if(L.i_point0 >= 0)
        for(int k = 0; k < 3 * L.Npoints_variable; k++) { (*b)[i] = ((const double*)points)[k] / scale[i]; i++; }
    if(L.i_warp0 >= 0)
        for(int k = 0; k < 2; k++) { (*b)[i] = warp->values[k] / scale[i]; i++; }
    if(i != L.Nstate) { set_error("internal error: packed %d of %d state elements", i, L.Nstate); return false; }
    return true;
}

int device_sm_count()
{
    static int cached[kMaxDevices] = {};
    int dev = 0;
    if(cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) { cudaGetLastError(); return 0; }
    if(cached[dev] == 0 && cudaDeviceGetAttribute(&cached[dev], cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    {
        cudaGetLastError();
        cached[dev] = 0;
    }
    return cached[dev];
}

bool problem_evaluate(mrcal_b200_problem* P, int which, bool with_jacobian, bool with_rowptr)
{
    return launch_evaluate(P->dp, P->op[which], with_jacobian, with_rowptr ? P->d_rowptr : nullptr, P->stream, &P->launches);
}

}  // namespace mb200

using namespace mb200;

extern "C" const char* mrcal_b200_version(void) { return "mrcal_b200 0.1 (sm_90a)"; }
extern "C" const char* mrcal_b200_last_error(void) { return get_error(); }
extern "C" int mrcal_b200_device_count(void)
{
    int n = 0;
    if(cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" mrcal_b200_problem_t*
mrcal_b200_problem_create(const double* intrinsics, const mrcal_pose_t* rt_cam_ref, const mrcal_pose_t* rt_ref_frame,
                          const mrcal_point3_t* points, const mrcal_calobject_warp_t* calobject_warp,
                          int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                          int Npoints, int Npoints_fixed,
                          const mrcal_observation_board_t* observations_board,
                          const mrcal_observation_point_t* observations_point,
                          int Nobservations_board, int Nobservations_point,
                          const mrcal_point3_t* observations_board_pool,
                          const mrcal_point3_t* observations_point_pool,
                          const mrcal_lensmodel_t* lensmodel, const int* imagersizes,
                          mrcal_problem_selections_t sel,
                          double calibration_object_spacing,
                          int calibration_object_width_n, int calibration_object_height_n)
{
    return mrcal_b200_problem_create_triangulated(intrinsics, rt_cam_ref, rt_ref_frame, points, calobject_warp,
                                                  Ncameras_intrinsics, Ncameras_extrinsics, Nframes, Npoints, Npoints_fixed,
                                                  observations_board, observations_point, Nobservations_board, Nobservations_point,
                                                  nullptr, 0,
                                                  observations_board_pool, observations_point_pool, lensmodel, imagersizes, sel,
                                                  calibration_object_spacing, calibration_object_width_n, calibration_object_height_n);
}

extern "C" mrcal_b200_problem_t*
mrcal_b200_problem_create_triangulated(const double* intrinsics, const mrcal_pose_t* rt_cam_ref, const mrcal_pose_t* rt_ref_frame,
                          const mrcal_point3_t* points, const mrcal_calobject_warp_t* calobject_warp,
                          int Ncameras_intrinsics, int Ncameras_extrinsics, int Nframes,
                          int Npoints, int Npoints_fixed,
                          const mrcal_observation_board_t* observations_board,
                          const mrcal_observation_point_t* observations_point,
                          int Nobservations_board, int Nobservations_point,
                          const mrcal_observation_point_triangulated_t* observations_point_triangulated,
                          int Nobservations_point_triangulated,
                          const mrcal_point3_t* observations_board_pool,
                          const mrcal_point3_t* observations_point_pool,
                          const mrcal_lensmodel_t* lensmodel, const int* imagersizes,
                          mrcal_problem_selections_t sel,
                          double calibration_object_spacing,
                          int calibration_object_width_n, int calibration_object_height_n)
{
    if(mrcal_b200_device_count() <= 0)
    {
        set_error("no usable CUDA device: libmrcal_b200 has no CPU fallback");
        return nullptr;
    }
    if(Nobservations_board < 0) Nobservations_board = 0;
    if(Nobservations_point < 0) Nobservations_point = 0;
    if(Nobservations_board > 0)
    {
        if(sel.do_optimize_calobject_warp && calobject_warp == nullptr)
        {
            set_error("ERROR: We're optimizing the calibration object warp, so a buffer with a seed MUST be passed in.");
            return nullptr;
        }
        if(calibration_object_width_n < 1 || calibration_object_height_n < 1)
        {
            set_error("board observations given, but the calibration object has no corners");
            return nullptr;
        }
    }
    else
        sel.do_optimize_calobject_warp = false;

    const int kind = lens_kind_of(lensmodel);
    if(kind < 0)
    {
        char name[256] = "?";
        mrcal_lensmodel_name(name, sizeof(name), lensmodel);
        set_error("lens model %s has no CUDA implementation yet (supported: PINHOLE, STEREOGRAPHIC, LONLAT, LATLON, OPENCV4/5/8/12, CAHVOR, CAHVORE, SPLINED_STEREOGRAPHIC order 2,3)", name);
        return nullptr;
    }

    // triangulated points: pairs within each set of consecutive observations (mrcal.c:5197-5290)
    std::vector<int> tri_pairs, tri_cam_e, tri_outlier, tri_set_obs0, tri_set_m0;
    std::vector<double> tri_px;
    if(observations_point_triangulated == nullptr || Nobservations_point_triangulated < 0) Nobservations_point_triangulated = 0;
    if(Nobservations_point_triangulated > 0)
    {
        // the reference's rule (mrcal.c:6260-6275)
        if(sel.do_optimize_intrinsics_core || sel.do_optimize_intrinsics_distortions || !sel.do_optimize_extrinsics)
        {
            set_error("ERROR: We have triangulated points. At this time this is only allowed if we're NOT optimizing intrinsics AND if we ARE optimizing extrinsics.");
            return nullptr;
        }
        const int N = Nobservations_point_triangulated;
        if(!observations_point_triangulated[N - 1].last_in_set)
        { set_error("the last triangulated observation must close its set (last_in_set)"); return nullptr; }
        for(int i = 0; i < N; i++)
        {
            const auto& o = observations_point_triangulated[i];
            if(o.icam.intrinsics < 0 || o.icam.intrinsics >= Ncameras_intrinsics || o.icam.extrinsics >= Ncameras_extrinsics)
            { set_error("triangulated observation %d has out-of-range indices", i); return nullptr; }
            if(i == 0 || observations_point_triangulated[i - 1].last_in_set)
            {
                tri_set_obs0.push_back(i);
                tri_set_m0.push_back((int)(tri_pairs.size() / 2));
            }
            tri_cam_e.push_back(o.icam.extrinsics < 0 ? -1 : o.icam.extrinsics);
            tri_outlier.push_back(o.outlier ? 1 : 0);
            tri_px.push_back(o.px.x); tri_px.push_back(o.px.y); tri_px.push_back(o.px.z);
            if(o.last_in_set) continue;
            for(int i1 = i + 1; i1 < N; i1++)
            {
                tri_pairs.push_back(i); tri_pairs.push_back(i1);
                if(observations_point_triangulated[i1].last_in_set) break;
            }
        }
    }

    tri_set_obs0.push_back(Nobservations_point_triangulated);
    std::unique_ptr<mrcal_b200_problem> P(new mrcal_b200_problem());
    Dims d;
    d.Nmeas_tri = (int)(tri_pairs.size() / 2);
    d.Ncam_i = Ncameras_intrinsics; d.Ncam_e = Ncameras_extrinsics; d.Nframes = Nframes;
    d.Npoints = Npoints; d.Npoints_fixed = Npoints_fixed;
    d.Nobs_board = Nobservations_board; d.Nobs_point = Nobservations_point;
    d.W = Nobservations_board > 0 ? calibration_object_width_n : 0;
    d.H = Nobservations_board > 0 ? calibration_object_height_n : 0;
    if(!make_layout(&P->L, d, sel, lensmodel)) return nullptr;
    const Layout& L = P->L;
    if(L.Nstate <= 0) { set_error("Not optimizing any of our variables!"); return nullptr; }

    // index sanity: everything below is used unchecked on the device
    for(int i = 0; i < d.Nobs_board; i++)
    {
        const auto& o = observations_board[i];
        if(o.icam.intrinsics < 0 || o.icam.intrinsics >= d.Ncam_i || o.icam.extrinsics >= d.Ncam_e ||
           o.iframe < 0 || o.iframe >= d.Nframes)
        { set_error("board observation %d has out-of-range indices", i); return nullptr; }
    }
    for(int i = 0; i < d.Nobs_point; i++)
    {
        const auto& o = observations_point[i];
        if(o.icam.intrinsics < 0 || o.icam.intrinsics >= d.Ncam_i || o.icam.extrinsics >= d.Ncam_e ||
           o.i_point < 0 || o.i_point >= d.Npoints)
        { set_error("point observation %d has out-of-range indices", i); return nullptr; }
    }

    // Jacobian offsets of each observation (rows within one observation have equal width)
    P->h_board_j0.resize(d.Nobs_board + 1);
    P->h_point_j0.resize(d.Nobs_point + 1);
    P->h_obs_board.resize(3 * (size_t)d.Nobs_board);
    P->h_obs_point.resize(3 * (size_t)d.Nobs_point);
    long j = 0;
    for(int i = 0; i < d.Nobs_board; i++)
    {
        P->h_board_j0[i] = (int)j;
        const bool cam = L.sel.do_optimize_extrinsics && observations_board[i].icam.extrinsics >= 0;
        j += (long)2 * d.W * d.H * (L.nnz_row_intr + (cam ? 6 : 0) + L.nnz_row_board_geom);
        P->h_obs_board[3 * i + 0] = observations_board[i].icam.intrinsics;
        P->h_obs_board[3 * i + 1] = observations_board[i].icam.extrinsics < 0 ? -1 : observations_board[i].icam.extrinsics;
        P->h_obs_board[3 * i + 2] = observations_board[i].iframe;
    }
    P->h_board_j0[d.Nobs_board] = (int)j;
    for(int i = 0; i < d.Nobs_point; i++)
    {
        P->h_point_j0[i] = (int)j;
        const bool cam = L.sel.do_optimize_extrinsics && observations_point[i].icam.extrinsics >= 0;
        const bool pt  = L.sel.do_optimize_frames && observations_point[i].i_point < L.Npoints_variable;
        j += (long)2 * (L.nnz_row_intr + (cam ? 6 : 0) + (pt ? 3 : 0));
        P->h_obs_point[3 * i + 0] = observations_point[i].icam.intrinsics;
        P->h_obs_point[3 * i + 1] = observations_point[i].icam.extrinsics < 0 ? -1 : observations_point[i].icam.extrinsics;
        P->h_obs_point[3 * i + 2] = observations_point[i].i_point;
    }
    P->h_point_j0[d.Nobs_point] = (int)j;
    std::vector<int> tri_j0(d.Nmeas_tri + 1);
    for(int ip = 0; ip < d.Nmeas_tri; ip++)
    {
        tri_j0[ip] = (int)j;
        j += (tri_cam_e[tri_pairs[2 * ip]] >= 0 ? 6 : 0) + (tri_cam_e[tri_pairs[2 * ip + 1]] >= 0 ? 6 : 0);
    }
    tri_j0[d.Nmeas_tri] = (int)j;
    const int reg_j0 = (int)j;
    j += (long)(L.splined ? 2 : 1) * L.Nreg_dist + L.Nreg_center + 3 * L.Nreg_unity;
    if(j > 0x7fffffffL) { set_error("Jacobian has %ld nonzeros: too many for int32 indices", j); return nullptr; }
    P->nnz = (int)j;

    if(cudaGetDevice(&P->device) != cudaSuccess) { set_error("cudaGetDevice failed"); return nullptr; }
    if(cudaStreamCreateWithFlags(&P->stream, cudaStreamNonBlocking) != cudaSuccess)
    { set_error("cudaStreamCreate failed: %s", cudaGetErrorString(cudaGetLastError())); return nullptr; }

    DeviceArena& A = P->arena;
    DevProblem& dp = P->dp;
    memset(&dp, 0, sizeof(dp));
    const size_t nfeat = (size_t)d.Nobs_board * d.W * d.H;
    int *d_obs_board, *d_obs_point, *d_board_j0, *d_point_j0, *d_imagersizes;
    int *d_tri_pairs = nullptr, *d_tri_cam_e = nullptr, *d_tri_outlier = nullptr, *d_tri_j0 = nullptr;
    int *d_tri_set_obs0 = nullptr, *d_tri_set_m0 = nullptr;
    double* d_tri_px = nullptr;
    bool ok = A.alloc(&d_tri_pairs, tri_pairs.size()) && A.alloc(&d_tri_cam_e, tri_cam_e.size()) && A.alloc(&d_tri_outlier, tri_outlier.size()) &&
              A.alloc(&d_tri_j0, tri_j0.size()) && A.alloc(&d_tri_px, tri_px.size()) &&
              A.alloc(&d_tri_set_obs0, tri_set_obs0.size()) && A.alloc(&d_tri_set_m0, tri_set_m0.size()) &&
              A.alloc(&P->d_tri_outlier_seed, tri_outlier.size()) &&
              A.alloc(&P->d_seed_intr, (size_t)d.Ncam_i * L.Nintr) && A.alloc(&P->d_seed_rtcam, 6 * (size_t)d.Ncam_e) &&
              A.alloc(&P->d_seed_rtframe, 6 * (size_t)d.Nframes) && A.alloc(&P->d_seed_points, 3 * (size_t)d.Npoints) &&
              A.alloc(&P->d_seed_warp, 2, true) &&
              A.alloc(&P->d_pool_board, 3 * nfeat) && A.alloc(&P->d_pool_board_seed, 3 * nfeat) &&
              A.alloc(&P->d_pool_point, 3 * (size_t)d.Nobs_point) &&
              A.alloc(&P->d_scale, L.Nstate) && A.alloc(&P->d_rowptr, (size_t)L.Nmeas + 1) &&
              A.alloc(&d_obs_board, 3 * (size_t)d.Nobs_board) && A.alloc(&d_obs_point, 3 * (size_t)d.Nobs_point) &&
              A.alloc(&d_board_j0, (size_t)d.Nobs_board + 1) && A.alloc(&d_point_j0, (size_t)d.Nobs_point + 1) &&
              A.alloc(&d_imagersizes, 2 * (size_t)d.Ncam_i) &&
              A.alloc(&dp.u_intr, (size_t)d.Ncam_i * L.Nintr) && A.alloc(&dp.u_rtcam, 6 * (size_t)d.Ncam_e) &&
              A.alloc(&dp.u_rtframe, 6 * (size_t)d.Nframes) && A.alloc(&dp.u_points, 3 * (size_t)d.Npoints) &&
              A.alloc(&dp.u_warp, 2, true) && A.alloc(&dp.u_rot_frame, 36 * (size_t)d.Nframes) && A.alloc(&dp.u_rot_cam, 36 * (size_t)d.Ncam_e);
    for(int k = 0; k < 2 && ok; k++)
        ok = A.alloc(&P->op[k].p, L.Nstate, true) && A.alloc(&P->op[k].x, L.Nmeas, true) &&
             A.alloc(&P->op[k].Jval, P->nnz) && A.alloc(&P->op[k].Jcol, P->nnz) && A.alloc(&P->op[k].norm2, 1, true);
    if(!ok) return nullptr;

    cudaStream_t s = P->stream;
    std::vector<double> scale(L.Nstate);
    fill_state_scales(scale.data(), L);
    ok = upload(d_obs_board, P->h_obs_board.data(), P->h_obs_board.size(), s) &&
         upload(d_obs_point, P->h_obs_point.data(), P->h_obs_point.size(), s) &&
         upload(d_board_j0, P->h_board_j0.data(), P->h_board_j0.size(), s) &&
         upload(d_point_j0, P->h_point_j0.data(), P->h_point_j0.size(), s) &&
         upload(d_imagersizes, imagersizes, 2 * (size_t)d.Ncam_i, s) &&
         upload(P->d_scale, scale.data(), scale.size(), s) &&
         upload(d_tri_pairs, tri_pairs.data(), tri_pairs.size(), s) && upload(d_tri_cam_e, tri_cam_e.data(), tri_cam_e.size(), s) &&
         upload(d_tri_outlier, tri_outlier.data(), tri_outlier.size(), s) && upload(d_tri_j0, tri_j0.data(), tri_j0.size(), s) &&
         upload(d_tri_px, tri_px.data(), tri_px.size(), s) &&
         upload(d_tri_set_obs0, tri_set_obs0.data(), tri_set_obs0.size(), s) && upload(d_tri_set_m0, tri_set_m0.data(), tri_set_m0.size(), s) &&
         upload(P->d_tri_outlier_seed, tri_outlier.data(), tri_outlier.size(), s);
    if(!ok) return nullptr;
    if(cudaStreamSynchronize(s) != cudaSuccess) { set_error("upload failed"); return nullptr; }   // the staging vectors go out of scope

    dp.Ncam_i = d.Ncam_i; dp.Ncam_e = d.Ncam_e; dp.Nframes = d.Nframes; dp.Npoints = d.Npoints;
    dp.Npoints_variable = L.Npoints_variable; dp.Nobs_board = d.Nobs_board; dp.Nobs_point = d.Nobs_point;
    dp.W = d.W; dp.H = d.H;
    dp.Nintr = L.Nintr; dp.Ncore_state = L.Ncore_state; dp.Ndist_state = L.Ndist_state; dp.Nintr_state = L.Nintr_state;
    dp.i_intr0 = L.i_intr0 < 0 ? 0 : L.i_intr0; dp.i_extr0 = L.i_extr0; dp.i_frame0 = L.i_frame0;
    dp.i_point0 = L.i_point0; dp.i_warp0 = L.i_warp0; dp.Nstate = L.Nstate;
    dp.m_point0 = L.m_point0; dp.m_reg0 = L.m_reg0; dp.Nmeas = L.Nmeas;
    dp.lens_kind = kind; dp.Nx = L.Nx; dp.Ny = L.Ny;
    dp.segments_per_u = 0.;
    dp.lens_cfg = lensmodel->type == MRCAL_LENSMODEL_CAHVORE ? lensmodel->LENSMODEL_CAHVORE__config.linearity : 0.;
    if(L.splined && !spline_segments_per_u(&dp.segments_per_u, lensmodel)) return nullptr;
    dp.spacing = calibration_object_spacing;
    dp.opt_core = L.sel.do_optimize_intrinsics_core; dp.opt_dist = L.sel.do_optimize_intrinsics_distortions;
    dp.opt_extr = L.i_extr0 >= 0; dp.opt_frames = L.sel.do_optimize_frames; dp.opt_warp = L.i_warp0 >= 0;
    dp.have_warp = calobject_warp != nullptr;
    dp.reg = L.sel.do_apply_regularization; dp.reg_unity = L.Nreg_unity > 0; dp.reg_owner = true;
    dp.opencv8plus = lensmodel->type == MRCAL_LENSMODEL_OPENCV8 || lensmodel->type == MRCAL_LENSMODEL_OPENCV12;
    dp.nnz_row_intr = L.nnz_row_intr; dp.nnz_row_board_geom = L.nnz_row_board_geom;
    dp.in_intrinsics = P->d_seed_intr; dp.in_rt_cam = P->d_seed_rtcam; dp.in_rt_frame = P->d_seed_rtframe;
    dp.in_points = P->d_seed_points; dp.in_warp = P->d_seed_warp; dp.imagersizes = d_imagersizes;
    dp.obs_board = d_obs_board; dp.obs_board_pool = P->d_pool_board;
    dp.obs_point = d_obs_point; dp.obs_point_pool = P->d_pool_point;
    dp.board_j0 = d_board_j0; dp.point_j0 = d_point_j0; dp.reg_j0 = reg_j0;
    dp.m_tri0 = L.m_tri0; dp.Ntri = d.Nmeas_tri;
    dp.tri_px = d_tri_px; dp.tri_cam_e = d_tri_cam_e; dp.tri_outlier = d_tri_outlier; dp.tri_pairs = d_tri_pairs; dp.tri_j0 = d_tri_j0;
    dp.Ntri_sets = (int)tri_set_m0.size(); dp.tri_set_obs0 = d_tri_set_obs0; dp.tri_set_m0 = d_tri_set_m0;
    P->Nobs_tri = Nobservations_point_triangulated;
    // the extrinsics regularization needs the frames off/extrinsics on case to see u_rtcam: always unpacked

    P->Nframes_global = d.Nframes;
    P->Npoints_global = d.Npoints;
    if(!mrcal_b200_problem_upload(P.get(), intrinsics, rt_cam_ref, rt_ref_frame, points, calobject_warp,
                                  observations_board_pool, observations_point_pool))
        return nullptr;
    return P.release();
}

extern "C" bool mrcal_b200_problem_upload(mrcal_b200_problem_t* P,
                                          const double* intrinsics, const mrcal_pose_t* rt_cam_ref,
                                          const mrcal_pose_t* rt_ref_frame, const mrcal_point3_t* points,
                                          const mrcal_calobject_warp_t* calobject_warp,
                                          const mrcal_point3_t* observations_board_pool,
                                          const mrcal_point3_t* observations_point_pool)
{
    const Layout& L = P->L;
    const Dims& d = L.d;
    cudaStream_t s = P->stream;
    const size_t nfeat = (size_t)d.Nobs_board * d.W * d.H;
    std::vector<double> b;
    mrcal_calobject_warp_t zero_warp = {};
    if(!pack_seed_host(P, &b, intrinsics, rt_cam_ref, rt_ref_frame, points, calobject_warp ? calobject_warp : &zero_warp))
        return false;
    bool ok = upload(P->d_seed_intr, intrinsics, (size_t)d.Ncam_i * L.Nintr, s) &&
              upload(P->d_seed_rtcam, (const double*)rt_cam_ref, 6 * (size_t)d.Ncam_e, s) &&
              upload(P->d_seed_rtframe, (const double*)rt_ref_frame, 6 * (size_t)d.Nframes, s) &&
              upload(P->d_seed_points, (const double*)points, 3 * (size_t)d.Npoints, s) &&
              (calobject_warp == nullptr || upload(P->d_seed_warp, calobject_warp->values, 2, s)) &&
              upload(P->d_pool_board, (const double*)observations_board_pool, 3 * nfeat, s) &&
              upload(P->d_pool_board_seed, (const double*)observations_board_pool, 3 * nfeat, s) &&
              upload(P->d_pool_point, (const double*)observations_point_pool, 3 * (size_t)d.Nobs_point, s) &&
              upload(P->op[0].p, b.data(), b.size(), s);
    if(!ok) return false;
    P->cur = 0;
    // b lives on the host stack frame: finish the copy before returning
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" void mrcal_b200_problem_destroy(mrcal_b200_problem_t* P)
{
    if(P == nullptr) return;
    if(P->stream) { cudaStreamSynchronize(P->stream); }
    P->ws.reset();
    P->arena.release();
    if(P->stream) cudaStreamDestroy(P->stream);
    delete P;
}

extern "C" int mrcal_b200_problem_num_states(const mrcal_b200_problem_t* P)       { return P->L.Nstate; }
extern "C" int mrcal_b200_problem_num_measurements(const mrcal_b200_problem_t* P) { return P->L.Nmeas; }
extern "C" int mrcal_b200_problem_num_j_nonzero(const mrcal_b200_problem_t* P)    { return P->nnz; }

__global__ void pack_from_unpacked_kernel(DevProblem P, const double* __restrict__ scale,
                                          const double* intr, const double* rtcam, const double* rtframe,
                                          const double* points, const double* warp, double* __restrict__ b)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= P.Nstate) return;
    double v;
    if(P.i_warp0 >= 0 && i >= P.i_warp0)        v = warp[i - P.i_warp0];
    else if(P.i_point0 >= 0 && i >= P.i_point0) v = points[i - P.i_point0];
    else if(P.i_frame0 >= 0 && i >= P.i_frame0) v = rtframe[i - P.i_frame0];
    else if(P.i_extr0 >= 0 && i >= P.i_extr0)   v = rtcam[i - P.i_extr0];
    else
    {
        const int cam = i / P.Nintr_state, k = i - cam * P.Nintr_state;
        const int kk = k < P.Ncore_state ? k : 4 + (k - P.Ncore_state);
        v = intr[cam * P.Nintr + kk];
    }
    b[i] = v / scale[i];
}

extern "C" bool mrcal_b200_problem_reset(mrcal_b200_problem_t* P, const double* b_packed)
{
    const Layout& L = P->L;
    cudaStream_t s = P->stream;
    P->cur = 0;
    if(b_packed != nullptr)
        MB200_CUDA_CHECK(cudaMemcpyAsync(P->op[0].p, b_packed, L.Nstate * sizeof(double), cudaMemcpyHostToDevice, s));
    else
    {
        pack_from_unpacked_kernel<<<(L.Nstate + 255) / 256, 256, 0, s>>>(P->dp, P->d_scale, P->d_seed_intr, P->d_seed_rtcam,
                                                                        P->d_seed_rtframe, P->d_seed_points, P->d_seed_warp,
                                                                        P->op[0].p);
        P->launches++;
    }
    const size_t nfeat = (size_t)L.d.Nobs_board * L.d.W * L.d.H;
    if(nfeat)
        MB200_CUDA_CHECK(cudaMemcpyAsync(P->d_pool_board, P->d_pool_board_seed, 3 * nfeat * sizeof(double),
                                         cudaMemcpyDeviceToDevice, s));
    if(P->Nobs_tri > 0)
        MB200_CUDA_CHECK(cudaMemcpyAsync(P->dp.tri_outlier, P->d_tri_outlier_seed, (size_t)P->Nobs_tri * sizeof(int),
                                         cudaMemcpyDeviceToDevice, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" bool mrcal_b200_problem_callback(mrcal_b200_problem_t* P, double* b_packed, double* x,
                                            int32_t* Jrowptr, int32_t* Jcolidx, double* Jval)
{
    const bool want_j = Jrowptr != nullptr || Jcolidx != nullptr || Jval != nullptr;
    if(!problem_evaluate(P, P->cur, want_j, Jrowptr != nullptr)) return false;
    const EvalBuffers& e = P->op[P->cur];
    cudaStream_t s = P->stream;
    if(b_packed) MB200_CUDA_CHECK(cudaMemcpyAsync(b_packed, e.p, P->L.Nstate * sizeof(double), cudaMemcpyDeviceToHost, s));
    if(x)        MB200_CUDA_CHECK(cudaMemcpyAsync(x, e.x, P->L.Nmeas * sizeof(double), cudaMemcpyDeviceToHost, s));
    if(Jrowptr)  MB200_CUDA_CHECK(cudaMemcpyAsync(Jrowptr, P->d_rowptr, ((size_t)P->L.Nmeas + 1) * sizeof(int), cudaMemcpyDeviceToHost, s));
    if(Jcolidx)  MB200_CUDA_CHECK(cudaMemcpyAsync(Jcolidx, e.Jcol, (size_t)P->nnz * sizeof(int), cudaMemcpyDeviceToHost, s));
    if(Jval)     MB200_CUDA_CHECK(cudaMemcpyAsync(Jval, e.Jval, (size_t)P->nnz * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" bool mrcal_b200_problem_download(mrcal_b200_problem_t* P, double* b_packed, double* x,
                                            double* intrinsics, mrcal_pose_t* rt_cam_ref, mrcal_pose_t* rt_ref_frame,
                                            mrcal_point3_t* points, mrcal_calobject_warp_t* calobject_warp,
                                            mrcal_point3_t* observations_board_pool)
{
    const Layout& L = P->L;
    const Dims& d = L.d;
    cudaStream_t s = P->stream;
    const EvalBuffers& e = P->op[P->cur];
    // unpacked view of the accepted state (mrcal.c:3647-3688)
    if(!launch_unpack_state(P->dp, e.p, s, &P->launches)) return false;
#define D2H(dst, src, n) do { if((dst) != nullptr && (n) > 0) \
        MB200_CUDA_CHECK(cudaMemcpyAsync((void*)(dst), (src), (size_t)(n) * sizeof(double), cudaMemcpyDeviceToHost, s)); } while(0)
    D2H(b_packed, e.p, L.Nstate);
    D2H(x, e.x, L.Nmeas);
    D2H(intrinsics, P->dp.u_intr, (size_t)d.Ncam_i * L.Nintr);
    D2H(rt_cam_ref, P->dp.u_rtcam, 6 * (size_t)d.Ncam_e);
    D2H(rt_ref_frame, P->dp.u_rtframe, 6 * (size_t)d.Nframes);
    D2H(points, P->dp.u_points, 3 * (size_t)d.Npoints);
    if(L.i_warp0 >= 0) D2H(calobject_warp, P->dp.u_warp, 2);
    D2H(observations_board_pool, P->d_pool_board, 3 * (size_t)d.Nobs_board * d.W * d.H);
#undef D2H
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}

extern "C" int mrcal_b200_problem_triangulated_outliers(mrcal_b200_problem_t* P, int* flags, int N)
{
    if(flags == nullptr || N <= 0) return P->Nobs_tri;
    if(N > P->Nobs_tri) N = P->Nobs_tri;
    if(N > 0)
    {
        if(cudaMemcpyAsync(flags, P->dp.tri_outlier, (size_t)N * sizeof(int), cudaMemcpyDeviceToHost, P->stream) != cudaSuccess ||
           cudaStreamSynchronize(P->stream) != cudaSuccess)
        { set_error("triangulated_outliers: %s", cudaGetErrorString(cudaGetLastError())); return -1; }
    }
    return P->Nobs_tri;
}

extern "C" double mrcal_b200_problem_time_callback(mrcal_b200_problem_t* P, int N, bool with_jacobian)
{
    if(N < 1) N = 1;
    cudaEvent_t e0, e1;
    if(cudaEventCreate(&e0) != cudaSuccess || cudaEventCreate(&e1) != cudaSuccess) return -1.;
    if(!problem_evaluate(P, P->cur, with_jacobian, false)) return -1.;   // warm
    cudaStreamSynchronize(P->stream);
    cudaEventRecord(e0, P->stream);
    for(int i = 0; i < N; i++)
        if(!problem_evaluate(P, P->cur, with_jacobian, false)) return -1.;
    cudaEventRecord(e1, P->stream);
    if(cudaEventSynchronize(e1) != cudaSuccess) { set_error("time_callback: %s", cudaGetErrorString(cudaGetLastError())); return -1.; }
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    return (double)ms / N;
}
