// Outlier marking on the device: what the reference does in markOutliers()
// (mrcal.c:3978-4402) between the passes of mrcal_optimize()'s outer loop
// (mrcal.c:6430-6481).
//
//   var = sum of x^2 over the inlier measurements / their count (boards: two
//   per corner; triangulated points: one per pair of observations);
//   if any inlier measurement has x^2 > 25 var: negate the weight of every
//   board corner with x^2 > 16 var in either coordinate, and flag both
//   observations of every triangulated pair with x^2 > 16 var; the caller
//   solves again. Triangulated pairs whose rays diverge are flagged first.
//
// The board part is embarrassingly parallel (sums in a fixed order, so that the
// result does not depend on scheduling). The triangulated part is sequential
// BY DEFINITION within one point: flagging an observation changes how the later
// pairs of the same point are treated (mrcal.c:4171-4254,4357-4390), so one
// thread walks the pairs of one point in the reference's order; points are
// independent of each other. Sharded solves: the sums and the "found" flag are
// all-reduced, every rank marks its own frames.
#include "device_math.cuh"
#include "problem_impl.h"

namespace mb200 {

bool comm_active();
bool comm_allreduce_sum(double* d_buf, size_t count, cudaStream_t s);

constexpr double kOutlierK0 = 4.0, kOutlierK1 = 5.0;
// Fixed, not derived from the SM count: the number of partial sums sets the order of the additions, and so
// the bits of the result, which must not depend on the device. 592 blocks of 256 threads are resident at once
// on a 132-SM H100 (8 per SM), so the count costs no second wave
constexpr int kOutlierBlocks = 592;

// acc layout (doubles)
enum { OA_SUMSQ = 0, OA_NINL_B, OA_NOUT_B, OA_NINL_T, OA_NOUT_T, OA_FOUND, OA_NEW_B, OA_NEW_T, OA_N };

// per-block partial sums over the board corners: [b][3] = sum x^2 of inliers, inliers, outliers
__global__ void __launch_bounds__(256)
outlier_board_stats_kernel(const double* __restrict__ pool, const double* __restrict__ x, long Nfeat, double* __restrict__ part)
{
    __shared__ double sh[3][8];
    double s = 0., ni = 0., no = 0.;
    // contiguous chunk per block, strided by threads inside: the order of the additions is fixed
    const long per = (Nfeat + gridDim.x - 1) / gridDim.x;
    const long i0 = (long)blockIdx.x * per, i1 = min(Nfeat, i0 + per);
    for(long i = i0 + threadIdx.x; i < i1; i += blockDim.x)
    {
        if(pool[3 * i + 2] <= 0.0) { no += 1.; continue; }   // mrcal.c:4116
        const double dx = x[2 * i], dy = x[2 * i + 1];
        s += dx * dx + dy * dy;
        ni += 1.;
    }
#pragma unroll
    for(int o = 16; o > 0; o >>= 1)
    {
        s += __shfl_xor_sync(0xffffffffu, s, o);
        ni += __shfl_xor_sync(0xffffffffu, ni, o);
        no += __shfl_xor_sync(0xffffffffu, no, o);
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if(lane == 0) { sh[0][w] = s; sh[1][w] = ni; sh[2][w] = no; }
    __syncthreads();
    if(threadIdx.x < 3)
    {
        double t = 0.;
        for(int k = 0; k < 8; k++) t += sh[threadIdx.x][k];
        part[3 * blockIdx.x + threadIdx.x] = t;
    }
}

// Do the rays of a pair converge? The value part of mrcal_triangulate_leecivera_mid2()
// (triangulation.cc:576-706): the cheirality test, then "the midpoint is not exactly 0"
__device__ bool tri_is_convergent(const double v0[3], const double v1[3], const double t01[3])
{
    auto cross_norm2 = [](const double* a, const double* b)
    {
        const double c0 = a[1] * b[2] - a[2] * b[1], c1 = a[2] * b[0] - a[0] * b[2], c2 = a[0] * b[1] - a[1] * b[0];
        return c0 * c0 + c1 * c1 + c2 * c2;
    };
    const double p_norm2_recip = 1. / cross_norm2(v0, v1);
    const double l0 = sqrt(cross_norm2(v1, t01) * p_norm2_recip);
    const double l1 = sqrt(cross_norm2(v0, t01) * p_norm2_recip);
    double w0 = 0., w1 = 0., w01 = 0.;
    for(int i = 0; i < 3; i++)
    {
        const double xn  = ( l1 * v1[i] + t01[i]) - l0 * v0[i];
        const double x0  = ( l1 * v1[i] + t01[i]) + l0 * v0[i];
        const double x1  = (-l1 * v1[i] + t01[i]) - l0 * v0[i];
        const double x01 = (-l1 * v1[i] + t01[i]) + l0 * v0[i];
        w0  += x0 * x0 - xn * xn;
        w1  += x1 * x1 - xn * xn;
        w01 += x01 * x01 - xn * xn;
    }
    if(!(w0 > 0. && w1 > 0. && w01 > 0.)) return false;
    double m[3];
    for(int i = 0; i < 3; i++) m[i] = (v0[i] * l0 + t01[i] + v1[i] * l1) / 2.0;
    return !(m[0] == 0.0 && m[1] == 0.0 && m[2] == 0.0);
}

// One thread per triangulated point (= set of consecutive observations). phase 0: flag divergent pairs,
// then the statistics (mrcal.c:4132-4256). phase 1: does an inlier pair exceed k1 sigma (mrcal.c:4290-4311)?
// phase 2: flag the pairs beyond k0 sigma (mrcal.c:4357-4390).
// set_part: [set][4] = sum x^2, inlier pairs, outlier pairs, flag
__global__ void __launch_bounds__(128)
outlier_tri_kernel(DevProblem P, int phase, const double* __restrict__ x, const double* __restrict__ acc,
                   double* __restrict__ set_part)
{
    const int is = blockIdx.x * blockDim.x + threadIdx.x;
    if(is >= P.Ntri_sets) return;
    const int o0 = P.tri_set_obs0[is], o1 = P.tri_set_obs0[is + 1];
    int m = P.tri_set_m0[is];
    const double* xt = x + P.m_tri0;
    double var = 0.;
    if(phase > 0) var = acc[OA_SUMSQ] / (2. * acc[OA_NINL_B] + acc[OA_NINL_T]);
    double s = 0., ni = 0., no = 0., flag = 0.;
    for(int i0 = o0; i0 < o1 - 1; i0++)
    {
        double v0_ref[3], t_r0[3] = {0., 0., 0.};
        const int e0 = P.tri_cam_e[i0];
        const double* v0 = &P.tri_px[3 * i0];
        if(phase == 0)
        {
            if(e0 >= 0)
            {
                double R0[9];
                const double* rt0 = &P.in_rt_cam[6 * e0];
                rodrigues(R0, nullptr, rt0);
                for(int c = 0; c < 3; c++)
                {
                    v0_ref[c] = R0[c] * v0[0] + R0[3 + c] * v0[1] + R0[6 + c] * v0[2];
                    t_r0[c] = -(R0[c] * rt0[3] + R0[3 + c] * rt0[4] + R0[6 + c] * rt0[5]);
                }
            }
            else
                for(int c = 0; c < 3; c++) v0_ref[c] = v0[c];
        }
        for(int i1 = i0 + 1; i1 < o1; i1++, m++)
        {
            if(phase == 0)
            {
                if(!(P.tri_outlier[i0] || P.tri_outlier[i1]))
                {
                    const int e1 = P.tri_cam_e[i1];
                    double v0_cam1[3], t_10[3];
                    if(e1 >= 0)
                    {
                        double R1[9];
                        const double* rt1 = &P.in_rt_cam[6 * e1];
                        rodrigues(R1, nullptr, rt1);
                        mat3_vec(v0_cam1, R1, v0_ref);
                        mat3_vec(t_10, R1, t_r0);
                        t_10[0] += rt1[3]; t_10[1] += rt1[4]; t_10[2] += rt1[5];
                    }
                    else
                        for(int c = 0; c < 3; c++) { v0_cam1[c] = v0_ref[c]; t_10[c] = t_r0[c]; }
                    if(!tri_is_convergent(&P.tri_px[3 * i1], v0_cam1, t_10))
                    {
                        // which of the two is broken is unknown: both are flagged
                        P.tri_outlier[i0] = 1;
                        P.tri_outlier[i1] = 1;
                        flag = 1.;
                    }
                }
                if(P.tri_outlier[i0] || P.tri_outlier[i1]) no += 1.;
                else { s += xt[m] * xt[m]; ni += 1.; }
            }
            else if(phase == 1)
            {
                if(!P.tri_outlier[i0] && !P.tri_outlier[i1] && xt[m] * xt[m] > kOutlierK1 * kOutlierK1 * var) flag = 1.;
            }
            else
            {
                if(!P.tri_outlier[i0] && !P.tri_outlier[i1] && xt[m] * xt[m] > kOutlierK0 * kOutlierK0 * var)
                {
                    P.tri_outlier[i0] = 1;
                    P.tri_outlier[i1] = 1;
                    no += 1.;
                }
            }
        }
    }
    set_part[4 * is + 0] = s; set_part[4 * is + 1] = ni; set_part[4 * is + 2] = no; set_part[4 * is + 3] = flag;
}

// one block: partial sums -> acc, in index order
__global__ void __launch_bounds__(256)
outlier_reduce_kernel(int mode, const double* __restrict__ part, int nblocks, const double* __restrict__ set_part, int nsets,
                      double* __restrict__ acc)
{
    // The sums are short (<= 592 and <= #points entries): one thread adds them in order. Deterministic by construction
    if(threadIdx.x != 0) return;
    if(mode == 0)
    {
        double s = 0., ni = 0., no = 0.;
        for(int b = 0; b < nblocks; b++) { s += part[3 * b]; ni += part[3 * b + 1]; no += part[3 * b + 2]; }
        double st = 0., nit = 0., notr = 0., fl = 0.;
        for(int k = 0; k < nsets; k++) { st += set_part[4 * k]; nit += set_part[4 * k + 1]; notr += set_part[4 * k + 2]; fl += set_part[4 * k + 3]; }
        acc[OA_SUMSQ] = s + st; acc[OA_NINL_B] = ni; acc[OA_NOUT_B] = no; acc[OA_NINL_T] = nit; acc[OA_NOUT_T] = notr;
        acc[OA_FOUND] = fl > 0. ? 1. : 0.;
        acc[OA_NEW_B] = 0.; acc[OA_NEW_T] = 0.;
    }
    else if(mode == 1)
    {
        double fl = 0.;
        for(int b = 0; b < nblocks; b++) fl += part[3 * b];
        for(int k = 0; k < nsets; k++) fl += set_part[4 * k + 3];
        if(fl > 0.) acc[OA_FOUND] = 1.;
    }
    else
    {
        double nb = 0., nt = 0.;
        for(int b = 0; b < nblocks; b++) nb += part[3 * b];
        for(int k = 0; k < nsets; k++) nt += set_part[4 * k + 2];
        acc[OA_NEW_B] = nb; acc[OA_NEW_T] = nt;
    }
}

// does any inlier corner exceed k1 sigma? part[3 b] = count found by block b
__global__ void __launch_bounds__(256)
outlier_board_find_kernel(const double* __restrict__ pool, const double* __restrict__ x, long Nfeat,
                          const double* __restrict__ acc, double* __restrict__ part)
{
    __shared__ int any;
    if(threadIdx.x == 0) any = 0;
    __syncthreads();
    const double var = acc[OA_SUMSQ] / (2. * acc[OA_NINL_B] + acc[OA_NINL_T]);
    const double lim = kOutlierK1 * kOutlierK1 * var;
    bool f = false;
    for(long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < Nfeat; i += (long)gridDim.x * blockDim.x)
    {
        if(pool[3 * i + 2] <= 0.0) continue;
        const double dx = x[2 * i], dy = x[2 * i + 1];
        if(dx * dx > lim || dy * dy > lim) f = true;
    }
    if(f) any = 1;   // benign race: every writer stores 1
    __syncthreads();
    if(threadIdx.x == 0) part[3 * blockIdx.x] = any ? 1. : 0.;
}

// One block per board observation: negate the weight of every inlier corner beyond k0 sigma.
// new_part[3 o] = newly marked; few_inliers[o] = inliers before marking if < 3, else -1 (for the host's warning)
__global__ void __launch_bounds__(128)
outlier_board_mark_kernel(double* __restrict__ pool, const double* __restrict__ x, int WH, const double* __restrict__ acc,
                          double* __restrict__ new_part, int* __restrict__ few_inliers)
{
    __shared__ int s_in, s_new;
    if(threadIdx.x == 0) { s_in = 0; s_new = 0; }
    __syncthreads();
    const double var = acc[OA_SUMSQ] / (2. * acc[OA_NINL_B] + acc[OA_NINL_T]);
    const double lim = kOutlierK0 * kOutlierK0 * var;
    const long base = (long)blockIdx.x * WH;
    int nin = 0, nnew = 0;
    for(int k = threadIdx.x; k < WH; k += blockDim.x)
    {
        const long i = base + k;
        if(pool[3 * i + 2] <= 0.0) continue;
        nin++;
        const double dx = x[2 * i], dy = x[2 * i + 1];
        if(dx * dx > lim || dy * dy > lim) { pool[3 * i + 2] *= -1.0; nnew++; }
    }
    atomicAdd(&s_in, nin);     // integer: order-independent
    atomicAdd(&s_new, nnew);
    __syncthreads();
    if(threadIdx.x == 0)
    {
        new_part[3 * blockIdx.x] = (double)s_new;
        few_inliers[blockIdx.x] = s_in < 3 ? s_in : -1;   // mrcal.c:4347 counts the inliers BEFORE this pass's marking
    }
}

struct OutlierWorkspace
{
    DeviceArena arena;
    double* part = nullptr;       // [max(kOutlierBlocks, Nobs_board)][3]
    double* set_part = nullptr;   // [Nsets][4]
    double* acc = nullptr;        // [OA_N]
    int*    few = nullptr;        // [Nobs_board]
    double* h_acc = nullptr;      // pinned
    std::vector<int> h_few;
    ~OutlierWorkspace() { if(h_acc) cudaFreeHost(h_acc); }
};
void outlier_workspace_delete(OutlierWorkspace* w) { delete w; }

// One call of the reference's markOutliers() at the accepted state (residuals P->op[P->cur].x).
// *found: new outliers were marked (solve again). Counts as the reference reports them.
bool outliers_mark(mrcal_b200_problem* P, bool* found, int* Noutliers_board, int* Noutliers_tri)
{
    const Layout& L = P->L;
    cudaStream_t s = P->stream;
    const long Nfeat = (long)L.d.Nobs_board * L.d.W * L.d.H;
    const int Nsets = P->dp.Ntri_sets;
    if(!P->ows)
    {
        std::unique_ptr<OutlierWorkspace, void (*)(OutlierWorkspace*)> w(new OutlierWorkspace(), outlier_workspace_delete);
        const size_t npart = (size_t)(L.d.Nobs_board > kOutlierBlocks ? L.d.Nobs_board : kOutlierBlocks);
        if(!w->arena.alloc(&w->part, 3 * npart, true) || !w->arena.alloc(&w->set_part, 4 * (size_t)(Nsets > 0 ? Nsets : 1), true) ||
           !w->arena.alloc(&w->acc, OA_N, true) || !w->arena.alloc(&w->few, (size_t)(L.d.Nobs_board > 0 ? L.d.Nobs_board : 1), true))
            return false;
        MB200_CUDA_CHECK(cudaMallocHost(&w->h_acc, OA_N * sizeof(double)));
        P->ows = std::move(w);
    }
    OutlierWorkspace* W = P->ows.get();
    const double* x = P->op[P->cur].x;
    const int nb = Nfeat > 0 ? kOutlierBlocks : 0;
    int* nl = &P->launches;

    // The divergent-ray test of the triangulated branch (mrcal.c:4143-4230) looks at rt_cam_ref AS THE CALLER GAVE IT:
    // mrcal_optimize() hands markOutliers() its own argument (mrcal.c:6472), which is only overwritten with the
    // solution after the outer loop. The seed poses, then, in every pass -- matched here (P.in_rt_cam)

    // ---- statistics (and the divergent-ray flags)
    if(nb) { outlier_board_stats_kernel<<<nb, 256, 0, s>>>(P->d_pool_board, x, Nfeat, W->part); (*nl)++; }
    if(Nsets) { outlier_tri_kernel<<<(Nsets + 127) / 128, 128, 0, s>>>(P->dp, 0, x, W->acc, W->set_part); (*nl)++; }
    outlier_reduce_kernel<<<1, 32, 0, s>>>(0, W->part, nb, W->set_part, Nsets, W->acc);
    (*nl)++;
    if(comm_active() && !comm_allreduce_sum(W->acc, OA_N, s)) return false;
    // ---- anything beyond k1 sigma?
    if(nb) { outlier_board_find_kernel<<<nb, 256, 0, s>>>(P->d_pool_board, x, Nfeat, W->acc, W->part); (*nl)++; }
    if(Nsets) { outlier_tri_kernel<<<(Nsets + 127) / 128, 128, 0, s>>>(P->dp, 1, x, W->acc, W->set_part); (*nl)++; }
    outlier_reduce_kernel<<<1, 32, 0, s>>>(1, W->part, nb, W->set_part, Nsets, W->acc);
    (*nl)++;
    if(comm_active() && !comm_allreduce_sum(W->acc + OA_FOUND, 1, s)) return false;
    MB200_CUDA_CHECK(cudaMemcpyAsync(W->h_acc, W->acc, OA_N * sizeof(double), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    *found = W->h_acc[OA_FOUND] > 0.;
    if(getenv("MRCAL_B200_DEBUG_OUTLIERS"))
    {
        fprintf(stderr, "mrcal_b200 outliers: sets %d, acc", Nsets);
        for(int i = 0; i < OA_N; i++) fprintf(stderr, " %.6g", W->h_acc[i]);
        fprintf(stderr, "\n");
    }
    *Noutliers_board = (int)W->h_acc[OA_NOUT_B];
    *Noutliers_tri = (int)W->h_acc[OA_NOUT_T];
    if(Nsets > 0)
        fprintf(stderr, "mrcal_b200: I started with %d triangulated outliers\n", *Noutliers_tri);
    if(!*found) return true;

    // ---- mark everything beyond k0 sigma
    if(L.d.Nobs_board > 0)
    {
        outlier_board_mark_kernel<<<L.d.Nobs_board, 128, 0, s>>>(P->d_pool_board, x, L.d.W * L.d.H, W->acc, W->part, W->few);
        (*nl)++;
    }
    if(Nsets) { outlier_tri_kernel<<<(Nsets + 127) / 128, 128, 0, s>>>(P->dp, 2, x, W->acc, W->set_part); (*nl)++; }
    outlier_reduce_kernel<<<1, 32, 0, s>>>(2, W->part, L.d.Nobs_board, W->set_part, Nsets, W->acc);
    (*nl)++;
    if(comm_active() && !comm_allreduce_sum(W->acc + OA_NEW_B, 2, s)) return false;
    W->h_few.resize(L.d.Nobs_board);
    MB200_CUDA_CHECK(cudaMemcpyAsync(W->h_acc, W->acc, OA_N * sizeof(double), cudaMemcpyDeviceToHost, s));
    if(L.d.Nobs_board > 0)
        MB200_CUDA_CHECK(cudaMemcpyAsync(W->h_few.data(), W->few, (size_t)L.d.Nobs_board * sizeof(int), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    *Noutliers_board += (int)W->h_acc[OA_NEW_B];
    *Noutliers_tri += (int)W->h_acc[OA_NEW_T];
    const int WH = L.d.W * L.d.H;
    for(int o = 0; o < L.d.Nobs_board; o++)
        if(W->h_few[o] >= 0)
            fprintf(stderr, "mrcal_b200: WARNING: Board observation %d (icam_intrinsics=%d, icam_extrinsics=%d, iframe=%d) had almost "
                            "all of its points thrown out as outliers: only %d/%d remain. The normal equations are about to "
                            "become singular. Something is wrong with this observation\n",
                    o, P->h_obs_board[3 * o], P->h_obs_board[3 * o + 1], P->h_obs_board[3 * o + 2] + P->frame_offset, W->h_few[o], WH);
    return true;
}

}  // namespace mb200
