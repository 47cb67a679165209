// Residual statistics binned by imager cell: the reference's mrcal.calibration._report_regional_statistics()
// (mrcal/calibration.py:1720-1866), which the valid-intrinsics region of each camera is built from, for a list of
// cameras in one launch, on the problem's own observation pool and residuals.
//
// A board corner of camera icam counts in a cell when its observation's icam_intrinsics is icam, its weight is > 0
// and its OBSERVED pixel q satisfies |q - c| < rcell strictly on both axes (c the cell's centre, rcell half the cell
// spacing); a corner that passes for two neighbouring cells counts in both. It adds its two weighted residuals
// (x and y pooled: a corner counts 2). A cell reports (mean, population stdev, count), or (0, 0, count) when
// count <= 5.
//
// One CTA per (camera, cell): it scans the corners of its camera's observations twice, once for the sum and once for
// the squared deviations from the mean (numpy's two-pass np.std()), each thread in a fixed stride and the warps
// combined in a fixed order (reduce.cuh). No atomics: two calls give the same bits. The scans are bounded by reading
// the camera's corners from L2 once per cell and pass; at a few hundred cells and a few hundred thousand corners that
// is well under a millisecond, next to the factorization the region also needs.
#include <vector>

#include "device_call.h"
#include "reduce.cuh"
#include "solver_internal.h"

namespace mb200 {
namespace {

constexpr int kStatsThreads = 256;

struct CornerScan
{
    const double* pool;      // [Nobs_board][ncorner][3] qx, qy, weight
    const double* x;         // the board residuals: [Nobs_board][ncorner][2]
    const int* obs_ptr;      // [Ncams + 1] each camera's run in obs
    const int* obs;          // the camera's board observations, increasing
    int ncorner;             // corners per board observation
};

// f(ex, ey) for every corner of camera c in the cell centred at (cx, cy), this thread's share, in index order
template <typename F>
__device__ __forceinline__ void for_corners_in_cell(const CornerScan& S, int c, double cx, double cy, double rx, double ry,
                                                    F&& f)
{
    const int o0 = S.obs_ptr[c];
    const long n = (long)(S.obs_ptr[c + 1] - o0) * S.ncorner;
    for(long it = threadIdx.x; it < n; it += kStatsThreads)
    {
        const int oi = (int)(it / S.ncorner), k = (int)(it - (long)oi * S.ncorner);
        const long corner = (long)S.obs[o0 + oi] * S.ncorner + k;
        const double* q = S.pool + 3 * corner;
        if(q[2] > 0. && fabs(q[0] - cx) < rx && fabs(q[1] - cy) < ry) f(S.x[2 * corner], S.x[2 * corner + 1]);
    }
}

// stats[c][cell] = (mean, stdev, count): grid (Ncells, Ncams)
__global__ void __launch_bounds__(kStatsThreads)
regional_statistics_kernel(CornerScan S, int Ncells, const double* __restrict__ centers /*[Ncams][Ncells][2]*/,
                           const double* __restrict__ rcell /*[Ncams][2]*/, double* __restrict__ stats)
{
    constexpr int NW = kStatsThreads / 32;
    __shared__ double part[2][NW];
    __shared__ double total[2];
    const int cell = blockIdx.x, c = blockIdx.y;
    const double cx = centers[2 * ((size_t)c * Ncells + cell)], cy = centers[2 * ((size_t)c * Ncells + cell) + 1];
    const double rx = rcell[2 * c], ry = rcell[2 * c + 1];

    double v[2] = {0., 0.};   // sum, count
    for_corners_in_cell(S, c, cx, cy, rx, ry, [&](double ex, double ey) { v[0] += ex; v[0] += ey; v[1] += 2.; });
    double t = block_sum_by_warps<2, NW>(v, part);
    if(threadIdx.x < 2) total[threadIdx.x] = t;
    __syncthreads();
    const double count = total[1], mean = total[0] / count;

    double d[1] = {0.};
    if(count > 5.)
        for_corners_in_cell(S, c, cx, cy, rx, ry, [&](double ex, double ey)
        {
            const double a = ex - mean, b = ey - mean;
            d[0] += a * a; d[0] += b * b;
        });
    t = block_sum_by_warps<1, NW>(d, part);
    if(threadIdx.x == 0)
    {
        double* out = stats + 3 * ((size_t)c * Ncells + cell);
        out[0] = count > 5. ? mean : 0.;
        out[1] = count > 5. ? sqrt(t / count) : 0.;
        out[2] = count;
    }
}

}  // namespace
}  // namespace mb200
using namespace mb200;

extern "C" bool mrcal_b200_problem_regional_statistics(mrcal_b200_problem_t* P, const int* icam_intrinsics, int Ncameras,
                                                       int gridn_width, int gridn_height, const double* q_cell_center,
                                                       const double* rcell, bool evaluate, double* stats, double* x)
{
    if(!have_device()) return false;
    if(P == nullptr) { set_error("regional_statistics: no problem"); return false; }
    if(P->sharded) { set_error("regional_statistics: not available for sharded problems"); return false; }
    if(Ncameras < 0 || gridn_width < 2 || gridn_height < 2)
    { set_error("regional_statistics: need Ncameras >= 0 and a grid of at least 2x2 cells; got %d cameras, %dx%d", Ncameras, gridn_width, gridn_height); return false; }
    const DevProblem& dp = P->dp;
    const int ncorner = dp.W * dp.H;
    // each camera's board observations, in their order
    std::vector<int> obs_ptr(1, 0), obs;
    for(int c = 0; c < Ncameras; c++)
    {
        if(icam_intrinsics[c] < 0 || icam_intrinsics[c] >= dp.Ncam_i)
        { set_error("icam_intrinsics = %d is out of range", icam_intrinsics[c]); return false; }
        for(size_t o = 0; o < P->h_obs_board.size() / 3; o++)
            if(P->h_obs_board[3 * o] == icam_intrinsics[c]) obs.push_back((int)o);
        obs_ptr.push_back((int)obs.size());
    }
    cudaStream_t s = P->stream;
    if(evaluate && !problem_evaluate(P, P->cur, false, false)) return false;
    const double* d_x = P->op[P->cur].x;
    const int Ncells = gridn_width * gridn_height;
    DeviceArena mem;   // freed after the stream has drained
    if(Ncameras > 0)
    {
        int *d_obs_ptr, *d_obs;
        double *d_centers, *d_rcell, *d_stats;
        if(!mem.alloc(&d_obs_ptr, obs_ptr.size()) || !mem.alloc(&d_obs, obs.size()) ||
           !mem.alloc(&d_centers, (size_t)2 * Ncameras * Ncells) || !mem.alloc(&d_rcell, (size_t)2 * Ncameras) ||
           !mem.alloc(&d_stats, (size_t)3 * Ncameras * Ncells))
            return false;
        MB200_CUDA_CHECK(cudaMemcpyAsync(d_obs_ptr, obs_ptr.data(), obs_ptr.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        if(!obs.empty()) MB200_CUDA_CHECK(cudaMemcpyAsync(d_obs, obs.data(), obs.size() * sizeof(int), cudaMemcpyHostToDevice, s));
        MB200_CUDA_CHECK(cudaMemcpyAsync(d_centers, q_cell_center, (size_t)2 * Ncameras * Ncells * sizeof(double), cudaMemcpyHostToDevice, s));
        MB200_CUDA_CHECK(cudaMemcpyAsync(d_rcell, rcell, (size_t)2 * Ncameras * sizeof(double), cudaMemcpyHostToDevice, s));
        const CornerScan S{P->d_pool_board, d_x + P->L.m_board0, d_obs_ptr, d_obs, ncorner};
        regional_statistics_kernel<<<dim3((unsigned)Ncells, (unsigned)Ncameras), kStatsThreads, 0, s>>>(S, Ncells, d_centers, d_rcell, d_stats);
        MB200_CUDA_CHECK(cudaGetLastError());
        P->launches++;
        MB200_CUDA_CHECK(cudaMemcpyAsync(stats, d_stats, (size_t)3 * Ncameras * Ncells * sizeof(double), cudaMemcpyDeviceToHost, s));
    }
    if(x) MB200_CUDA_CHECK(cudaMemcpyAsync(x, d_x, (size_t)P->L.Nmeas * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return true;
}
