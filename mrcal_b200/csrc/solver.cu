// The trust-region loop: Powell's dogleg, as the reference runs it through
// libdogleg's dogleg_optimize2() (call site mrcal.c:6435; parameters
// mrcal.c:6289-6299), and the outlier-rejection outer loop around it
// (mrcal.c:6430-6481, markOutliers mrcal.c:3978-4402).
//
// libdogleg is not part of the reference tree; the step logic below restates
// its published algorithm (the same restatement, in numpy, is the parity oracle:
// oracle/dogleg_np.py). What differs is where the work happens: the state, the
// residuals, the Jacobian strips, the reduced normal equations and their factor
// never leave the GPU; the host only sees a handful of scalars per iteration
// and takes the accept/reject decisions.
#include <algorithm>
#include <cmath>

#include "comm.h"
#include "reduce.cuh"
#include "solver_internal.h"

namespace mb200 {

static void delete_ws(SolverWorkspace* w) { delete w; }
static bool build_workspace(mrcal_b200_problem* P);

////////////////////////////////////////////////////////////////////////////////
// small vector kernels
////////////////////////////////////////////////////////////////////////////////
// out[0] += (J v).x ; out[1] += |J v|^2. Eight lanes per row (rows are 2..32 entries wide), four rows per warp
// in flight: the kernel streams J once and wants as many loads outstanding as it can get
__global__ void __launch_bounds__(256)
jv_kernel(const int* __restrict__ rowptr, const int* __restrict__ col, const double* __restrict__ val,
          const double* __restrict__ v, const double* __restrict__ x, int row_begin, int Nrows, double* __restrict__ out)
{
    __shared__ double red0[8], red1[8];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, sub = lane & 7;
    const int nwarps = (gridDim.x * blockDim.x) >> 5;
    double s0 = 0., s1 = 0.;
    // (the loop bound is per WARP, so that all 32 lanes reach the shuffles together)
    for(int row0 = row_begin + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 4; row0 < Nrows; row0 += nwarps * 4)
    {
        const int row = row0 + (lane >> 3);
        const bool live = row < Nrows;
        const int j0 = live ? rowptr[row] : 0, j1 = live ? rowptr[row + 1] : 0;
        double acc = 0.;
#pragma unroll 4
        for(int j = j0 + sub; j < j1; j += 8) acc += val[j] * v[col[j]];
        acc += __shfl_xor_sync(0xffffffffu, acc, 4);
        acc += __shfl_xor_sync(0xffffffffu, acc, 2);
        acc += __shfl_xor_sync(0xffffffffu, acc, 1);
        if(sub == 0 && live) { s0 += acc * x[row]; s1 += acc * acc; }
    }
#pragma unroll
    for(int o = 16; o >= 8; o >>= 1) { s0 += __shfl_xor_sync(0xffffffffu, s0, o); s1 += __shfl_xor_sync(0xffffffffu, s1, o); }
    if(lane == 0) { red0[wib] = s0; red1[wib] = s1; }
    __syncthreads();
    if(threadIdx.x == 0)
    {
        double a = 0., b = 0.;
        for(int i = 0; i < (int)(blockDim.x >> 5); i++) { a += red0[i]; b += red1[i]; }
        atomicAdd(&out[0], a);
        atomicAdd(&out[1], b);
    }
}

// Block k in {0,1,2} reduces range k of the state vector: [0,e0) shared head, [e0,e1) eliminated
// (the only part that differs between ranks when the frames are sharded), [e1,n) shared tail.
// out[3j+0] = a.a, out[3j+1] = b.b, out[3j+2] = a.b  (b may be null); j: see below
__global__ void __launch_bounds__(1024)
dots_kernel(const double* __restrict__ a, const double* __restrict__ b, int e0, int e1, int n, double* __restrict__ out)
{
    __shared__ double r[3][32];
    const int i0 = blockIdx.x == 0 ? 0 : (blockIdx.x == 1 ? e0 : e1);
    const int i1 = blockIdx.x == 0 ? e0 : (blockIdx.x == 1 ? e1 : n);
    // slots: head 0..2, tail 3..5, eliminated 6..8 -- the per-rank partial sums (eliminated range) come last, next to
    // the row sums the caller keeps behind them, so that ONE cross-rank reduction covers both
    out += blockIdx.x == 0 ? 0 : (blockIdx.x == 1 ? 6 : 3);
    double s[3] = {0., 0., 0.};
    for(int i = i0 + threadIdx.x; i < i1; i += blockDim.x)
    {
        const double x = a[i], y = b ? b[i] : 0.;
        s[0] += x * x; s[1] += y * y; s[2] += x * y;
    }
    const double t = block_sum_by_warps(s, r, (int)(blockDim.x >> 5));
    if(threadIdx.x < 3) out[threadIdx.x] = t;
}

// number of board corners with weight < 0 (mrcal.c:6420-6425). Integer atomics: order-independent
__global__ void count_negative_kernel(const double* __restrict__ pool, long n, int* __restrict__ out)
{
    int c = 0;
    for(long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x)
        if(pool[3 * i + 2] < 0.0) c++;
    c = warp_sum(c);
    if((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

////////////////////////////////////////////////////////////////////////////////
// workspace
////////////////////////////////////////////////////////////////////////////////
bool solver_build_workspace(mrcal_b200_problem* P) { return build_workspace(P); }
static bool build_workspace(mrcal_b200_problem* P)
{
    if(P->ws) return true;
    const Layout& L = P->L;
    std::unique_ptr<SolverWorkspace, void (*)(SolverWorkspace*)> ws(new SolverWorkspace(), delete_ws);
    NormalBuffers& N = ws->N;
    DeviceArena& A = ws->arena;

    if(!normal_buffers_create(&N, P, A)) return false;
    const bool ok = A.alloc(&ws->invL, (size_t)N.ldS_max * kCholBlock) && A.alloc(&ws->rhs, N.ldS_max, true) &&
                    A.alloc(&ws->step_gn, L.Nstate, true) && A.alloc(&ws->step, L.Nstate, true) && A.alloc(&ws->scal, 64, true) &&
                    A.alloc(&ws->ictl, 8, true);
    if(!ok) return false;
    MB200_CUDA_CHECK(cudaMallocHost(&ws->h_scal, 64 * sizeof(double)));
    MB200_CUDA_CHECK(cudaMallocHost(&ws->h_info, 16 * sizeof(int)));
    N.h_stat = ws->h_info + 4;
    ws->h_ictl = ws->h_info + 8;
    MB200_CUDA_CHECK(cudaHostGetDevicePointer((void**)&ws->h_scal_dev, ws->h_scal, 0));
    MB200_CUDA_CHECK(cudaHostGetDevicePointer((void**)&ws->h_info_dev, ws->h_info, 0));
    if(!chol_scratch_create(&ws->chol, N.ldS_max)) return false;
    P->ws = std::move(ws);
    return true;
}

static bool count_negative_weights(mrcal_b200_problem* P, int* count)
{
    SolverWorkspace* ws = P->ws.get();
    const Layout& L = P->L;
    const long n = (long)L.d.Nobs_board * L.d.W * L.d.H;
    int* d_cnt = ws->N.stat + 2;
    MB200_CUDA_CHECK(cudaMemsetAsync(d_cnt, 0, sizeof(int), P->stream));
    count_negative_kernel<<<2 * std::max(1, device_sm_count()), 256, 0, P->stream>>>(P->d_pool_board, n, d_cnt);
    P->launches++;
    MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_info + 2, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, P->stream));
    MB200_CUDA_CHECK(cudaStreamSynchronize(P->stream));
    *count = ws->h_info[2];
    if(comm_active())
    {
        ws->h_scal[31] = (double)*count;
        MB200_CUDA_CHECK(cudaMemcpyAsync(ws->scal + 31, ws->h_scal + 31, sizeof(double), cudaMemcpyHostToDevice, P->stream));
        if(!comm_allreduce_sum(ws->scal + 31, 1, P->stream)) return false;
        MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_scal + 31, ws->scal + 31, sizeof(double), cudaMemcpyDeviceToHost, P->stream));
        MB200_CUDA_CHECK(cudaStreamSynchronize(P->stream));
        *count = (int)ws->h_scal[31];
    }
    return true;
}

////////////////////////////////////////////////////////////////////////////////
// one dogleg solve from the current state (the reference's dogleg_optimize2())
////////////////////////////////////////////////////////////////////////////////
struct PhaseTimer
{
    SolverWorkspace* ws; cudaStream_t s;
    std::vector<std::pair<int, int>> spans[4];   // evaluate, assemble, factor, solve
    size_t used = 0;
    int mark()
    {
        if(used == ws->ev.size()) { cudaEvent_t e; cudaEventCreate(&e); ws->ev.push_back(e); }
        cudaEventRecord(ws->ev[used], s);
        return (int)used++;
    }
    double total(int phase)
    {
        double t = 0.;
        for(auto& sp : spans[phase]) { float ms = 0.f; cudaEventElapsedTime(&ms, ws->ev[sp.first], ws->ev[sp.second]); t += ms; }
        return t;
    }
};

// ---- the step logic on the device. scal[] slots:
//   0..8   dots of g = J'x by range (shared head | eliminated | shared tail): a.a, -, -
//   9,10   x.(J g), |J g|^2
//   11..19 dots of (gn, g) by range: gn.gn, g.g, gn.g
//   22     |x|^2 at the trial point
//   32 cg  33 cn  34 update_lensq  35 edge  36 cauchy_lensq  37 gn_lensq  38 kc  39 expected improvement
// ictl[]: 0 need_gn (the Cauchy point is inside the trust region)  1 zero gradient
enum { SC_CG = 32, SC_CN, SC_UPDATE, SC_EDGE, SC_CAUCHY2, SC_GN2, SC_KC, SC_EXPECTED, SC_N = 48 };

// Sharded solves: the per-rank partial sums among the scalars -- [6..10] (eliminated part of |g|^2, the row sums of
// |J g|^2) and [17..19] (eliminated parts of the Gauss-Newton dots) -- through ONE reduction: gathered to [50..57],
// summed over the ranks there, scattered back
__global__ void stage_partials_kernel(double* __restrict__ scal, bool gather)
{
    const int i = threadIdx.x;
    if(blockIdx.x != 0 || i >= 8) return;
    const int slot = i < 5 ? 6 + i : 17 + (i - 5);
    if(gather) scal[50 + i] = scal[slot];
    else       scal[slot] = scal[50 + i];
}

__global__ void cauchy_decide_kernel(double* __restrict__ scal, int* __restrict__ ictl, double trustregion)
{
    if(threadIdx.x != 0 || blockIdx.x != 0) return;
    const double g2 = scal[0] + scal[3] + scal[6];
    const double Jg2 = scal[10];
    if(!(g2 > 0.) || !(Jg2 > 0.))
    {
        // zero gradient: nothing to do (libdogleg's Jt_x_threshold test)
        ictl[1] = 1; ictl[0] = 0;
        scal[SC_KC] = 0.; scal[SC_CAUCHY2] = 0.;
        return;
    }
    const double kc = g2 / Jg2;
    const double c2 = kc * kc * g2;
    scal[SC_KC] = kc;
    scal[SC_CAUCHY2] = c2;
    ictl[1] = 0;
    ictl[0] = c2 >= trustregion * trustregion ? 0 : 1;   // Cauchy point inside the trust region: go on to Gauss-Newton
}

// Cauchy step to the edge | Gauss-Newton step | dogleg to the edge (libdogleg's takeStepFrom()), and the improvement
// the quadratic model expects of the step s = cg g + cn gn:  |x|^2 - |x + J s|^2 = -2 x.(J s) - |J s|^2. libdogleg gets it
// from an explicit product J s; here it follows from scalars already on the device, because the Gauss-Newton step
// solves (JtJ + lambda I) gn = -g:   x.(J s) = g.s ;  (J g).(J gn) = -g.g - lambda g.gn ;  |J gn|^2 = -g.gn - lambda gn.gn
__global__ void select_step_kernel(double* __restrict__ scal, const int* __restrict__ ictl, double trustregion, double lambda)
{
    if(threadIdx.x != 0 || blockIdx.x != 0) return;
    const double kc = scal[SC_KC], a2 = scal[SC_CAUCHY2];
    const double tr2 = trustregion * trustregion;
    const double g2 = scal[0] + scal[3] + scal[6], Jg2 = scal[10];
    double gn2 = 0., g_dot_gn = 0.;
    double cg, cn, upd, edge;
    if(ictl[1]) { cg = 0.; cn = 0.; upd = 0.; edge = 0.; }
    else if(a2 >= tr2)
    {
        cg = -kc * trustregion / sqrt(a2); cn = 0.; upd = tr2; edge = 1.;
    }
    else
    {
        gn2 = scal[11] + scal[14] + scal[17];
        g_dot_gn = scal[13] + scal[16] + scal[19];
        scal[SC_GN2] = gn2;
        if(gn2 <= tr2) { cg = 0.; cn = 1.; upd = gn2; edge = 0.; }
        else
        {
            // a + k (b-a) on the boundary; a = Cauchy = -kc g, b = Gauss-Newton
            const double ab = -kc * g_dot_gn;
            const double l2 = a2 - 2. * ab + gn2;
            const double c = ab - a2;
            const double disc = c * c - l2 * (a2 - tr2);
            const double k = (-c + sqrt(disc > 0. ? disc : 0.)) / l2;
            cg = -kc * (1. - k); cn = k; upd = tr2; edge = 1.;
        }
    }
    scal[SC_CG] = cg; scal[SC_CN] = cn; scal[SC_UPDATE] = upd; scal[SC_EDGE] = edge;
    const double x_Js = cg * g2 + cn * g_dot_gn;
    const double Js2 = cg * cg * Jg2 + 2. * cg * cn * (-g2 - lambda * g_dot_gn) + cn * cn * (-g_dot_gn - lambda * gn2);
    scal[SC_EXPECTED] = -2. * x_Js - Js2;
}

// Everything the host looks at after a step, straight into its pinned mirrors in one launch (one stream operation
// instead of a device-to-device and four device-to-host copies): the scalars, with |x|^2 of the trial point in slot 22,
// the factorization codes, the sizes normal_prepare() found, the control flags. h_info: [0..1] info, [4..7] stat,
// [8..9] ictl (the layout of the SolverWorkspace mirrors)
__global__ void read_back_kernel(double* __restrict__ scal, const double* __restrict__ norm2, const int* __restrict__ info,
                                 const int* __restrict__ stat, const int* __restrict__ ictl, double* __restrict__ h_scal,
                                 int* __restrict__ h_info)
{
    const int i = threadIdx.x;
    const double n2 = *norm2;
    if(i < SC_N) h_scal[i] = i == 22 ? n2 : scal[i];
    if(i == 22) scal[22] = n2;
    if(i < 2) h_info[i] = info[i];
    if(i < 4) h_info[4 + i] = stat[i];
    if(i < 2) h_info[8 + i] = ictl[i];
}

// step = cg g + cn gn ; p_new = p + step, with cg, cn read on the device
__global__ void combine_step_dev_kernel(int n, const double* __restrict__ scal, const double* __restrict__ g, const double* __restrict__ gn,
                                        const double* __restrict__ p, double* __restrict__ step, double* __restrict__ p_new)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= n) return;
    const double cg = scal[SC_CG], cn = scal[SC_CN];
    const double sv = (cg != 0. ? cg * g[i] : 0.) + (cn != 0. ? cn * gn[i] : 0.);
    step[i] = sv;
    p_new[i] = p[i] + sv;
}

static bool dogleg_pass(mrcal_b200_problem* P, const mrcal_b200_solver_parameters_t& par, double* lambda,
                        mrcal_b200_solve_info_t* info, PhaseTimer* T, double* norm2_final)
{
    SolverWorkspace* ws = P->ws.get();
    NormalBuffers& N = ws->N;
    const Layout& L = P->L;
    cudaStream_t s = P->stream;
    const int Nstate = L.Nstate, Nmeas = L.Nmeas;
    int* nl = &P->launches;

    // evaluate the cost function at op[which] and, in the same breath, find out which shared unknowns its rows touch:
    // the size of the reduced system then reaches the host with the same read as everything else
    bool norm2_summed = false;
    auto evaluate = [&](int which) -> bool
    {
        const int a = T->mark();
        if(!normal_evaluate(P->dp, N, P->op[which], s, nl)) return false;
        T->spans[0].push_back({a, T->mark()});
        info->Nevaluations++;
        const int b = T->mark();
        // (sharded: the cost of this evaluation is summed over the ranks in the collective that unites the active sets.
        // Not sharded: the sizes reach the host with the step's scalars, in read_back)
        if(!normal_prepare(P->dp, N, P->op[which], s, nl, N.fused, P->op[which].norm2, &norm2_summed, comm_active())) return false;
        T->spans[1].push_back({b, T->mark()});
        return true;
    };
    auto assemble = [&](int which) -> bool
    {
        const int a = T->mark();
        // (the scalars of the Cauchy step that follows are cleared with the assembly's accumulators)
        if(!normal_finish(P->dp, N, P->op[which], P->d_rowptr, *lambda, s, nl, N.fused, ws->scal, 32)) return false;
        T->spans[1].push_back({a, T->mark()});
        return true;
    };
    // ONE device -> host read per iteration: the scalars (|x|^2 of the evaluation at op[which] in slot 22), the control
    // flags, the factorization codes, the sizes of the next reduced system
    auto read_back = [&](int which) -> bool
    {
        if(comm_active())
        {
            // (sharded: |x|^2 is summed over the ranks in place, in scal[22])
            MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_scal, ws->scal, SC_N * sizeof(double), cudaMemcpyDeviceToHost, s));
            MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_info, N.info, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
            MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_ictl, ws->ictl, 2 * sizeof(int), cudaMemcpyDeviceToHost, s));
        }
        else
        {
            read_back_kernel<<<1, 64, 0, s>>>(ws->scal, P->op[which].norm2, N.info, N.stat, ws->ictl, ws->h_scal_dev, ws->h_info_dev);
            (*nl)++;
            MB200_CUDA_CHECK(cudaGetLastError());
        }
        MB200_CUDA_CHECK(cudaStreamSynchronize(s));
        info->Nsyncs++;
        return normal_adopt_sizes(N, s);   // n_c, widest item: from the prepare() that ran last
    };
    // rows whose sums this rank contributes to cross-rank reductions: the regularization rows are
    // replicated on every rank but counted once
    const int Nrows_mine = P->dp.reg_owner ? Nmeas : P->dp.m_reg0;
    const int e0 = N.e0, e1 = N.e1;

    // evaluate + read back; if the fused kernel had to give up on an observation, once more through the stored-Jacobian path
    auto evaluate_and_read = [&](int which) -> bool
    {
        for(int attempt = 0; attempt < 2; attempt++)
        {
            if(!evaluate(which)) return false;
            if(comm_active())
            {
                MB200_CUDA_CHECK(cudaMemcpyAsync(ws->scal + 22, P->op[which].norm2, sizeof(double), cudaMemcpyDeviceToDevice, s));
                if(!norm2_summed && !comm_allreduce_sum(ws->scal + 22, 1, s)) return false;
            }
            if(!read_back(which)) return false;
            if(!(N.fused && N.h_stat[3] != 0)) return true;
            fprintf(stderr, "mrcal_b200: an observation touches more control points than the fused evaluation handles: "
                            "continuing with the stored-Jacobian path\n");
            N.fused = false;
            info->Nevaluations--;
            // (the blocks' places in the pool are computed per assembly on that path)
        }
        return true;
    };
    if(!evaluate_and_read(P->cur)) return false;
    double norm2_x = ws->h_scal[22];
    if(info->Nevaluations == 1) info->norm2_x_initial = norm2_x;

    double trustregion = par.trustregion0;
    bool have_system = false, have_cauchy = false, have_gn = false, sizes_are_cur = true;
    int stepCount = 0;
    bool done = false;

    while(!done && stepCount < par.max_iterations)
    {
        while(true)
        {
            const EvalBuffers& cur = P->op[P->cur];
            const EvalBuffers& nxt = P->op[1 - P->cur];
            if(!have_system)
            {
                if(!sizes_are_cur)
                {
                    // (only after a failed factorization: the column bookkeeping belongs to the trial point by now)
                    if(!evaluate_and_read(P->cur)) return false;
                    info->Nevaluations--;
                    sizes_are_cur = true;
                }
                if(!assemble(P->cur)) return false;
                have_system = true;
                have_cauchy = have_gn = false;
            }
            // ---- Cauchy step: -k g, k = |g|^2 / |J g|^2. Its sums need nothing of the factorization and the factorization
            // nothing of them: they run on a second stream, UNDER the factorization (whose spine leaves the machine mostly
            // idle). The price: whether the Cauchy point already leaves the trust region -- and the Gauss-Newton step is
            // unnecessary -- is only known afterwards, so every new operating point is factored; the rare unnecessary
            // factorization (the first few steps of a solve) costs less than those sums on the critical path of every step
            if(!have_cauchy)
            {
                // (scal[0..31] were cleared by the assembly, which always comes right before)
                cudaStream_t sc = N.s_side[0];
                MB200_CUDA_CHECK(cudaEventRecord(N.ev_fork, s));
                MB200_CUDA_CHECK(cudaStreamWaitEvent(sc, N.ev_fork, 0));
                dots_kernel<<<3, 1024, 0, sc>>>(N.g_full, nullptr, e0, e1, Nstate, ws->scal + 0);
                const int nsm = std::max(1, device_sm_count());
                if(N.fused)
                {
                    // |J g|^2: the board rows from the observations' blocks, the others from their stored rows
                    if(!launch_quadform_boards(P->dp, N, N.g_full, N.qf_part, ws->scal + 10, sc, nl)) return false;
                    if(Nrows_mine > P->dp.m_point0)
                        jv_kernel<<<nsm * 4, 256, 0, sc>>>(P->d_rowptr, cur.Jcol, cur.Jval, N.g_full, cur.x, P->dp.m_point0, Nrows_mine, ws->scal + 9);
                }
                else
                    jv_kernel<<<nsm * 16, 256, 0, sc>>>(P->d_rowptr, cur.Jcol, cur.Jval, N.g_full, cur.x, 0, Nrows_mine, ws->scal + 9);
                *nl += 2;
                MB200_CUDA_CHECK(cudaEventRecord(N.ev_join[0], sc));
                // eliminated-range dots and the row sums are per-rank partial sums. Sharded: they wait for the partial sums
                // of the Gauss-Newton dots and go through ONE reduction with them (below)
                have_cauchy = true;
            }
            // (have_gn: same operating point, smaller trust region: everything is there)
            bool factored_now = false;
            if(!have_gn)
            {
                // ---- Gauss-Newton step: factor the reduced system, solve, back-substitute
                const int a = T->mark();
                if(!chol_factor(N.S, N.ldS, N.n_c, ws->invL, N.info + 1, s, nl, &ws->chol)) return false;
                T->spans[2].push_back({a, T->mark()});
                const int b = T->mark();
                if(!normal_extract_y(N, ws->rhs, s, nl)) return false;
                if(N.n_c > 0 && !chol_solve_backward(N.S, N.ldS, ws->invL, ws->rhs, N.info + 1, s, nl, &ws->chol)) return false;
                if(!normal_expand_step(P->dp, N, P->op[P->cur], *lambda, ws->rhs, ws->step_gn, s, nl)) return false;
                dots_kernel<<<3, 1024, 0, s>>>(ws->step_gn, N.g_full, e0, e1, Nstate, ws->scal + 11);
                (*nl)++;
                MB200_CUDA_CHECK(cudaStreamWaitEvent(s, N.ev_join[0], 0));
                if(comm_active())
                {
                    stage_partials_kernel<<<1, 32, 0, s>>>(ws->scal, true);
                    if(!comm_allreduce_sum(ws->scal + 50, 8, s)) return false;
                    stage_partials_kernel<<<1, 32, 0, s>>>(ws->scal, false);
                    *nl += 2;
                }
                T->spans[3].push_back({b, T->mark()});
                factored_now = true;
            }
            cauchy_decide_kernel<<<1, 32, 0, s>>>(ws->scal, ws->ictl, trustregion);
            (*nl)++;
            // ---- take the step
            select_step_kernel<<<1, 32, 0, s>>>(ws->scal, ws->ictl, trustregion, *lambda);
            combine_step_dev_kernel<<<(Nstate + 255) / 256, 256, 0, s>>>(Nstate, ws->scal, N.g_full, ws->step_gn, cur.p, ws->step, nxt.p);
            *nl += 2;
            sizes_are_cur = false;
            if(!evaluate_and_read(1 - P->cur)) return false;

            const bool need_gn = ws->h_ictl[0] != 0, zero_grad = ws->h_ictl[1] != 0;
            if(zero_grad) { done = true; break; }
            if(factored_now && need_gn)
            {
                info->Nfactorizations++;
                const bool bad = ws->h_info[0] != 0 || ws->h_info[1] != 0;
                if(ws->h_info[1] == -9)
                {
                    set_error("the persistent factorization kernel gave up waiting for a tile (code -9): not a property of the matrix");
                    return false;
                }
                // (sharded: a frame block that is singular on ONE rank has been reported to every rank with the reduced system
                // itself, normal_schur.cu:unpack_extras_kernel, and the factorization is replicated)
                if(bad)
                {
                    // singular JtJ: add lambda I "from now on", as libdogleg does (1e-10, then x10), and do this operating point again
                    *lambda = (*lambda == 0.) ? 1e-10 : *lambda * 10.;
                    if(!std::isfinite(*lambda) || *lambda > 1e30) { set_error("the normal equations stay singular even with lambda=%g", *lambda); return false; }
                    fprintf(stderr, "mrcal_b200: singular JtJ (codes %d,%d). Adding %g I from now on\n", ws->h_info[0], ws->h_info[1], *lambda);
                    have_system = false;
                    continue;
                }
                have_gn = true;
            }
            const double update_lensq = ws->h_scal[SC_UPDATE];
            const bool edge = ws->h_scal[SC_EDGE] != 0.;
            if(update_lensq < par.update_threshold)
            {
                // libdogleg compares the SQUARED step length with update_threshold
                done = true;
                break;
            }
            // |x|^2 - |x + J step|^2, as the quadratic model has it
            const double expected = ws->h_scal[SC_EXPECTED];
            const double norm2_new = ws->h_scal[22];
            const double observed = norm2_x - norm2_new;
            const double rho = observed / expected;
            if(rho < par.trustregion_decrease_threshold)               trustregion *= par.trustregion_decrease_factor;
            else if(rho > par.trustregion_increase_threshold && edge)  trustregion *= par.trustregion_increase_factor;
            if(rho > 0.0)
            {
                P->cur = 1 - P->cur;
                norm2_x = norm2_new;
                have_system = false;
                sizes_are_cur = true;
                break;
            }
            // rejected: same operating point, smaller trust region
            if(trustregion < par.trustregion_threshold) { done = true; break; }
        }
        if(done) break;
        stepCount++;
        info->Niterations++;
    }
    *norm2_final = norm2_x;
    return true;
}

bool solver_run(mrcal_b200_problem* P, const mrcal_b200_solver_parameters_t* params,
                mrcal_stats_t* stats, mrcal_b200_solve_info_t* info_out)
{
    mrcal_b200_solver_parameters_t par;
    if(params) par = *params; else mrcal_b200_default_solver_parameters(&par);
    mrcal_b200_solve_info_t info = {};
    if(!build_workspace(P)) return false;
    SolverWorkspace* ws = P->ws.get();
    const Layout& L = P->L;
    cudaStream_t s = P->stream;
    const int launches0 = P->launches;
    const long collectives0 = comm_collective_count();

    // the CSR row pointers are analytic; jv_kernel and the regularization assembly read them
    if(!problem_evaluate(P, P->cur, false, true)) return false;

    PhaseTimer T{ws, s};
    const int t0 = T.mark();
    const size_t Nfeat = (size_t)L.d.Nobs_board * L.d.W * L.d.H;
    // stats as mrcal_optimize() initialises them (mrcal.c:6416-6425): board corners with weight < 0; the
    // triangulated count stays 0 unless markOutliers() runs
    int Noutliers = 0, Noutliers_tri = 0;
    if(Nfeat)
    {
        if(!count_negative_weights(P, &Noutliers)) return false;
    }
    double lambda = 0., norm2 = -1.;
    while(true)
    {
        info.Nouter++;
        // every pass is a fresh dogleg_optimize2() call in the reference (mrcal.c:6432-6439): lambda and the
        // trust region start over
        lambda = 0.;
        if(!dogleg_pass(P, par, &lambda, &info, &T, &norm2)) return false;
        if(!L.sel.do_apply_outlier_rejection) break;
        bool found = false;
        if(!outliers_mark(P, &found, &Noutliers, &Noutliers_tri)) return false;
        if(!found) break;
        fprintf(stderr, "mrcal_b200: Threw out some outliers. New count = %d/%d (%.1f%%). Going again\n",
                Noutliers, L.Nmeas_board, (double)(Noutliers * 100) / (double)L.Nmeas_board);
    }
    const int t1 = T.mark();
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ws->ev[t0], ws->ev[t1]);
    info.ms_total = ms;
    info.ms_evaluate = T.total(0);
    info.ms_assemble = T.total(1);
    info.ms_factor = T.total(2);
    info.ms_solve = T.total(3);
    info.Nreduced = ws->N.n_c;
    info.norm2_x_final = norm2;
    info.lambda_final = lambda;
    info.Nkernel_launches = P->launches - launches0;
    info.Ncollectives = (int)(comm_collective_count() - collectives0);
    if(stats)
    {
        // mrcal.c:6607-6612. Sharded: the measurement count of the whole problem (regularization counted once)
        double nmeas = (double)L.Nmeas;
        if(comm_active())
        {
            ws->h_scal[31] = (double)(P->dp.reg_owner ? L.Nmeas : P->dp.m_reg0);
            MB200_CUDA_CHECK(cudaMemcpyAsync(ws->scal + 31, ws->h_scal + 31, sizeof(double), cudaMemcpyHostToDevice, s));
            if(!comm_allreduce_sum(ws->scal + 31, 1, s)) return false;
            MB200_CUDA_CHECK(cudaMemcpyAsync(ws->h_scal + 31, ws->scal + 31, sizeof(double), cudaMemcpyDeviceToHost, s));
            MB200_CUDA_CHECK(cudaStreamSynchronize(s));
            nmeas = ws->h_scal[31];
        }
        stats->rms_reproj_error__pixels = sqrt(norm2 / nmeas);
        stats->Noutliers_board = Noutliers;
        stats->Noutliers_triangulated_point = Noutliers_tri;
    }
    if(info_out) *info_out = info;
    return true;
}

}  // namespace mb200
using namespace mb200;

extern "C" void mrcal_b200_default_solver_parameters(mrcal_b200_solver_parameters_t* p)
{
    // libdogleg's defaults with mrcal's overrides (mrcal.c:6289-6299)
    p->max_iterations = 300;
    p->trustregion0 = 1e3;
    p->trustregion_decrease_factor = 0.1;
    p->trustregion_decrease_threshold = 0.25;
    p->trustregion_increase_factor = 2.0;
    p->trustregion_increase_threshold = 0.75;
    p->Jt_x_threshold = 0.;
    p->update_threshold = 1e-7;
    p->trustregion_threshold = 0.;
}

// S, g', g_full of the assembly that just ran, to the host
static bool download_reduced_system(mrcal_b200_problem_t* P, double* S_out, double* g_reduced, double* g_full)
{
    NormalBuffers& N = P->ws->N;
    // the device holds the system over the active unknowns only; expand to reduced numbering here
    // (inactive rows/columns come out as zero: they are not part of the coupled system)
    std::vector<double> Sc((size_t)N.n_c * N.n_c), gc(N.n_c);
    std::vector<int> cinv(N.n_c);
    if(N.n_c > 0)
    {
        MB200_CUDA_CHECK(cudaMemcpy2DAsync(Sc.data(), (size_t)N.n_c * sizeof(double), N.S, (size_t)N.ldS * sizeof(double),
                                           (size_t)N.n_c * sizeof(double), N.n_c, cudaMemcpyDeviceToHost, P->stream));
        MB200_CUDA_CHECK(cudaMemcpyAsync(gc.data(), N.gs, (size_t)N.n_c * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
        MB200_CUDA_CHECK(cudaMemcpyAsync(cinv.data(), N.cinv, (size_t)N.n_c * sizeof(int), cudaMemcpyDeviceToHost, P->stream));
    }
    if(g_full)
        MB200_CUDA_CHECK(cudaMemcpyAsync(g_full, N.g_full, (size_t)P->L.Nstate * sizeof(double), cudaMemcpyDeviceToHost, P->stream));
    MB200_CUDA_CHECK(cudaStreamSynchronize(P->stream));
    if(S_out) memset(S_out, 0, (size_t)N.n_r * N.n_r * sizeof(double));
    if(g_reduced) memset(g_reduced, 0, (size_t)N.n_r * sizeof(double));
    for(int a = 0; a < N.n_c; a++)
    {
        if(g_reduced) g_reduced[cinv[a]] = gc[a];
        if(S_out) for(int b = 0; b <= a; b++) S_out[(size_t)cinv[a] * N.n_r + cinv[b]] = Sc[(size_t)a * N.n_c + b];
    }
    return true;
}

extern "C" bool mrcal_b200_problem_reduced_system(mrcal_b200_problem_t* P, double lambda, int* n_reduced,
                                                  double* S_out, double* g_reduced, double* g_full)
{
    if(!build_workspace(P)) return false;
    NormalBuffers& N = P->ws->N;
    if(n_reduced) *n_reduced = N.n_r;
    if(S_out == nullptr && g_reduced == nullptr && g_full == nullptr) return true;
    if(!problem_evaluate(P, P->cur, true, true)) return false;
    if(!normal_assemble(P->dp, N, P->op[P->cur], P->d_rowptr, lambda, P->stream, &P->launches)) return false;
    return download_reduced_system(P, S_out, g_reduced, g_full);
}

extern "C" bool mrcal_b200_problem_reduced_system_fused(mrcal_b200_problem_t* P, double lambda, int* n_reduced,
                                                        double* S_out, double* g_reduced, double* g_full)
{
    if(!build_workspace(P)) return false;
    NormalBuffers& N = P->ws->N;
    if(n_reduced) *n_reduced = N.n_r;
    if(!N.fused) { set_error("reduced_system_fused: this problem does not take the fused evaluation"); return false; }
    if(S_out == nullptr && g_reduced == nullptr && g_full == nullptr) return true;
    // what an optimize() step does: the boards' blocks from the fused evaluation, the other rows from their Jacobian
    cudaStream_t s = P->stream;
    int* nl = &P->launches;
    const EvalBuffers& o = P->op[P->cur];
    if(!normal_evaluate(P->dp, N, o, s, nl) || !normal_prepare(P->dp, N, o, s, nl, true)) return false;
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    if(!normal_adopt_sizes(N, s)) return false;
    if(N.h_stat[3] != 0)
    {
        set_error("reduced_system_fused: the fused evaluation's blocks do not fit this problem");
        return false;
    }
    if(!normal_finish(P->dp, N, o, P->d_rowptr, lambda, s, nl, true)) return false;
    return download_reduced_system(P, S_out, g_reduced, g_full);
}

extern "C" bool mrcal_b200_problem_optimize(mrcal_b200_problem_t* P, const mrcal_b200_solver_parameters_t* parameters,
                                            mrcal_stats_t* stats, mrcal_b200_solve_info_t* info)
{
    return solver_run(P, parameters, stats, info);
}
