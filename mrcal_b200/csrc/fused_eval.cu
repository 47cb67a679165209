// The cost function and the per-observation normal-equation blocks in ONE pass, for the solver's own use: the
// board rows of the Jacobian are never written to memory.
//
// mrcal.optimize() needs, at every trust-region step, the residuals x and -- for the normal equations --
// only what J'J and J'x contribute per board observation: the Gram matrix of the observation's 2 W H rows over the
// shared unknowns they touch (A), its coupling to the observation's frame (B, D), and J'x over both (gs, gf).
// mrcal.optimizer_callback() still returns the reference's CSR Jacobian (eval.cu); this file is the path
// Problem.optimize() takes for the splined models with the core locked (the reference's own configuration for them,
// mrcal-calibrate-cameras:641-643; every BASELINE splined config).
//
// One CTA per board observation, one thread per corner:
//   1. project the corner (its point from observation.cuh): residuals, the B-spline basis (wx, wy) of its window,
//      and the 14 "geometric" entries of each of its two rows (camera r,t | frame r,t | warp)
//   2. the knots the observation touches form a patch of the control-point grid; the x row of a corner touches the
//      x surface with values  w b fx, the y row the y surface with  w b fy,  b = wx (x) wy THE SAME for both rows.
//      So with  Dk[corner][knot] = w b  (one matrix, not two half-empty ones):
//          knot x knot     fx^2 Dk'Dk on the x surface, fy^2 Dk'Dk on the y surface, 0 across
//          knot x geometry fx Dk'Gx, fy Dk'Gy ;  knot x residual  fx Dk'ex, fy Dk'ey
//      two dense products Dk'[Dk | Gx Gy ex ey] on the fp64 tensor pipe (DMMA 8x8x4) -- a quarter of the flops of
//      the Gram matrix over the full row width that normal.cu's kernel computes from the stored Jacobian
//   3. geometry x geometry (14 x 14) and J'x over the geometry: plain FMAs
//   4. the blocks go out in the layout normal_schur.cu consumes: A in the compact layout (normal.h, kCompactSlot: fx^2,
//      fy^2, M = Dk'Dk once, the geometry rows, -J'x once), and B, D, gf
//
// Replaces, for this path: the board loop of optimizer_callback() (mrcal.c:4604-4900), libdogleg's Jt*x and what
// CHOLMOD's A*A' does with those rows.
#include "normal_items.cuh"
#include "observation.cuh"

namespace mb200 {

namespace {

constexpr int FLDK = 68;    // row stride of Dk [K][<=64 knots]: 4 (mod 16), conflict-free DMMA fragment loads
constexpr int FLDG = 36;    // row stride of G  [K][32]
constexpr int FMAXK = kCompactMaxKnots;   // most knots of one observation's patch that are touched
constexpr int FMAXPATCH = 400;   // bounding box of the patch (knots)
constexpr int FMAXCORNERS = 128; // one thread per corner

// the dynamic shared memory of fused_boards_kernel for K (= W*H rounded up to 4) rows: Dk, G, C, GG and gv (below).
// 125 088 bytes at K = 128: one CTA per SM above 112 corners (two fit up to K = 112)
constexpr size_t fused_smem_bytes(int K) { return ((size_t)K * (FLDK + FLDG) + FMAXK * 33 + 14 * 14 + 14 + 2) * sizeof(double); }

}  // namespace

// G columns: 0..5 x-row camera (r,t) | 6..11 x-row frame (r,t) | 12,13 x-row warp | 14..27 the same of the y row | 28 ex | 29 ey
template <int RUN>
__global__ void __launch_bounds__(128, 2)
fused_boards_kernel(DevProblem P, NormalBuffers N, double* __restrict__ x, double* __restrict__ norm_part, int K)
{
    extern __shared__ __align__(16) double dsm[];
    double* Dk = dsm;                        // [K][FLDK]
    double* Gs = Dk + (size_t)K * FLDK;      // [K][FLDG]
    double* Cs = Gs + (size_t)K * FLDG;      // [FMAXK][33]  Dk'[Gx Gy ex ey]
    double* GG = Cs + FMAXK * 33;            // [14][14] + gv[14]
    __shared__ ObsPoses G;
    __shared__ short s_kidx[FMAXPATCH];
    __shared__ unsigned char s_touched[FMAXPATCH];
    __shared__ int s_win[128];               // per corner: window origin (wy0 << 16 | wx0)
    __shared__ int s_box[4], s_scan[128], s_bad;
    __shared__ double s_red[4];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int iobs = blockIdx.x;
    const int icam_i = P.obs_board[3 * iobs + 0], icam_e = P.obs_board[3 * iobs + 1], iframe = P.obs_board[3 * iobs + 2];
    const bool cam_identity = icam_e < 0;
    const bool emit_cam = P.opt_extr && !cam_identity;
    const int NWH = P.W * P.H;

    load_obs_poses(G, P, iframe, icam_e, tid);
    if(tid == 0) { s_box[0] = 1 << 30; s_box[1] = -1; s_box[2] = 1 << 30; s_box[3] = -1; s_bad = 0; }
    for(int e = tid; e < K * FLDK; e += 128) Dk[e] = 0.;
    for(int e = tid; e < K * FLDG; e += 128) Gs[e] = 0.;
    for(int e = tid; e < FMAXPATCH; e += 128) s_touched[e] = 0;
    __syncthreads();

    const double* __restrict__ intr = &P.u_intr[(size_t)icam_i * P.Nintr];
    const double wx2 = P.u_warp[0], wy2 = P.u_warp[1];

    // ---- 1. the corner
    double bw[RUN * RUN];      // w wx wy of the window
    double sumsq = 0.;
    int wx0 = 0, wy0 = 0;
    const bool have = tid < NWH;
    if(have)
    {
        const int ipt = tid;
        const int cx = ipt % P.W, cy = ipt / P.W;
        double pt[3], dz[2], v[3], p[3];
        board_corner(pt, dz, v, p, P, G, cam_identity, cx, cy, wx2, wy2);

        double q[2], dq_dp[2][3], wxb[4], wyb[4], upd[2];
        int ivar0;
        project_splined<RUN>(q, dq_dp, wxb, wyb, &ivar0, upd, p, intr, P.Nx, P.Ny, P.segments_per_u);
        const int k0 = (ivar0 - 4) >> 1;
        wy0 = k0 / P.Nx; wx0 = k0 - wy0 * P.Nx;
        s_win[tid] = (wy0 << 16) | wx0;
        atomicMin(&s_box[0], wx0); atomicMax(&s_box[1], wx0);
        atomicMin(&s_box[2], wy0); atomicMax(&s_box[3], wy0);

        const size_t ifeat = (size_t)iobs * NWH + ipt;
        const double qx_obs = P.obs_board_pool[3 * ifeat + 0], qy_obs = P.obs_board_pool[3 * ifeat + 1];
        const double wgt = P.obs_board_pool[3 * ifeat + 2];
        const bool outlier = !(wgt >= 0.0);   // mrcal.c:4695
        const double w = outlier ? 0. : wgt;
        const double e0 = outlier ? 0. : (q[0] - qx_obs) * wgt;
        const double e1 = outlier ? 0. : (q[1] - qy_obs) * wgt;
        x[2 * ifeat + 0] = e0;
        x[2 * ifeat + 1] = e1;
        sumsq = e0 * e0 + e1 * e1;
#pragma unroll
        for(int iy = 0; iy < RUN; iy++)
#pragma unroll
            for(int ix = 0; ix < RUN; ix++) bw[iy * RUN + ix] = w * wxb[ix] * wyb[iy];

        // the geometric entries of the two rows (eval.cu computes the same)
        double G2[2][3];
        if(cam_identity) { for(int k = 0; k < 2; k++) { G2[k][0] = dq_dp[k][0]; G2[k][1] = dq_dp[k][1]; G2[k][2] = dq_dp[k][2]; } }
        else
        {
#pragma unroll
            for(int k = 0; k < 2; k++)
#pragma unroll
                for(int j = 0; j < 3; j++) G2[k][j] = dq_dp[k][0] * G.Rc[j] + dq_dp[k][1] * G.Rc[3 + j] + dq_dp[k][2] * G.Rc[6 + j];
        }
        double* g = Gs + (size_t)tid * FLDG;
#pragma unroll
        for(int k = 0; k < 3; k++)
        {
            double dv[3];
            mat3_vec(dv, &G.dRf[9 * k], pt);
            g[6 + k]      = (G2[0][0] * dv[0] + G2[0][1] * dv[1] + G2[0][2] * dv[2]) * w * kScaleRotFrame;
            g[14 + 6 + k] = (G2[1][0] * dv[0] + G2[1][1] * dv[1] + G2[1][2] * dv[2]) * w * kScaleRotFrame;
            g[9 + k]      = G2[0][k] * w * kScaleTransFrame;
            g[14 + 9 + k] = G2[1][k] * w * kScaleTransFrame;
        }
        if(emit_cam)
        {
#pragma unroll
            for(int k = 0; k < 3; k++)
            {
                double dp[3];
                mat3_vec(dp, &G.dRc[9 * k], v);
                g[k]          = (dq_dp[0][0] * dp[0] + dq_dp[0][1] * dp[1] + dq_dp[0][2] * dp[2]) * w * kScaleRotCam;
                g[14 + k]     = (dq_dp[1][0] * dp[0] + dq_dp[1][1] * dp[1] + dq_dp[1][2] * dp[2]) * w * kScaleRotCam;
                g[3 + k]      = dq_dp[0][k] * w * kScaleTransCam;
                g[14 + 3 + k] = dq_dp[1][k] * w * kScaleTransCam;
            }
        }
        if(P.opt_warp)
        {
#pragma unroll
            for(int k = 0; k < 2; k++)
            {
                const double dq_dz = G2[k][0] * G.Rf[2] + G2[k][1] * G.Rf[5] + G2[k][2] * G.Rf[8];
                g[14 * k + 12] = dq_dz * dz[0] * w * kScaleWarp;
                g[14 * k + 13] = dq_dz * dz[1] * w * kScaleWarp;
            }
        }
        g[28] = e0; g[29] = e1;
    }
    // |x|^2 of this observation: one partial per CTA, summed in a fixed order later
    sumsq = warp_sum(sumsq);
    if(lane == 0) s_red[warp] = sumsq;
    __syncthreads();
    if(tid == 0) norm_part[iobs] = (s_red[0] + s_red[1]) + (s_red[2] + s_red[3]);

    // ---- 2. the patch of control points this observation touches
    const int bx0 = s_box[0], by0 = s_box[2];
    const int pw = s_box[1] - bx0 + RUN, ph = s_box[3] - by0 + RUN;
    const int npk = pw * ph;
    if(npk > FMAXPATCH)
    {
        if(tid == 0) N.stat[3] = 1;   // the host takes the other path for this evaluation
        return;
    }
    if(have)
    {
#pragma unroll
        for(int iy = 0; iy < RUN; iy++)
#pragma unroll
            for(int ix = 0; ix < RUN; ix++) s_touched[(wy0 - by0 + iy) * pw + (wx0 - bx0 + ix)] = 1;
    }
    __syncthreads();
    int nk;
    {
        // rank of each touched knot among the touched, in grid (= state) order
        const int per = (npk + 127) / 128;
        const int lo = tid * per, hi = min(lo + per, npk);
        int cnt = 0;
        for(int i = lo; i < hi; i++) cnt += s_touched[i];
        int base = block_exclusive_scan<int, 128>(cnt, s_scan, nk);
        for(int i = lo; i < hi; i++) s_kidx[i] = s_touched[i] ? (short)(base++) : (short)-1;
        __syncthreads();
    }
    const int ncam = emit_cam ? 6 : 0, nwarp = P.opt_warp ? 2 : 0;
    const int nsh = 2 * nk + ncam + nwarp;
    if(nk > FMAXK || nsh + 2 > N.capA)
    {
        if(tid == 0) N.stat[3] = 1;
        return;
    }
    // ---- the item's column list (reduced numbering = state numbering for the intrinsics), the active marks
    const int w_item = iobs;
    {
        const int cbase = P.i_intr0 + icam_i * P.Nintr_state + P.Ncore_state;
        int* cols = N.wi_cols + (size_t)w_item * N.cap;
        for(int i = tid; i < npk; i += 128)
        {
            const int k = s_kidx[i];
            if(k < 0) continue;
            const int ly = i / pw, lx = i - ly * pw;
            const int c0 = cbase + 2 * ((by0 + ly) * P.Nx + bx0 + lx);
            cols[2 * k] = c0; cols[2 * k + 1] = c0 + 1;
            N.active[c0] = 1; N.active[c0 + 1] = 1;
        }
        if(tid < ncam)  { const int r = N.reduced_index(P.i_extr0 + 6 * icam_e + tid); cols[2 * nk + tid] = r; N.active[r] = 1; }
        if(tid < nwarp) { const int r = N.reduced_index(P.i_warp0 + tid); cols[2 * nk + ncam + tid] = r; N.active[r] = 1; }
        if(tid == 0)
        {
            N.wi_nsh[w_item] = nsh;
            N.wi_lda[w_item] = ~nk;   // the compact layout, at this observation's fixed slot
            N.wi_Aoff[w_item] = (long long)w_item * kCompactSlot;
            atomicMax(&N.stat[1], nsh + 6);
        }
    }
    // ---- Dk
    if(have)
    {
        double* d = Dk + (size_t)tid * FLDK;
#pragma unroll
        for(int iy = 0; iy < RUN; iy++)
#pragma unroll
            for(int ix = 0; ix < RUN; ix++) d[s_kidx[(wy0 - by0 + iy) * pw + (wx0 - bx0 + ix)]] = bw[iy * RUN + ix];
    }
    __syncthreads();

    // ---- 3. Dk'[Dk | G] on the tensor pipe. Tiles of 8x8 outputs: T(T+1)/2 of the symmetric part + 4 T of the rest,
    // dealt round-robin to the 4 warps, 4 at a time per warp (independent accumulator chains)
    const int T = (nk + 7) >> 3;
    const int nsym = T * (T + 1) / 2, ntiles = nsym + 4 * T;
    const int g = lane >> 2, t = lane & 3;
    const int ksteps = K >> 2;
    const double fx = intr[0], fy = intr[1];
    double* Aw = N.wi_A + (size_t)w_item * kCompactSlot;
    if(tid == 0) { Aw[0] = fx * fx; Aw[1] = fy * fy; }
    for(int q0 = warp; q0 < ntiles; q0 += 16)
    {
        int ti[4], tj[4];
        bool sym[4], live[4];
        const double *pa[4], *pb[4];
        int ldb[4];
#pragma unroll
        for(int u = 0; u < 4; u++)
        {
            const int q = q0 + 4 * u;
            live[u] = q < ntiles;
            const int qq = live[u] ? q : 0;
            sym[u] = qq < nsym;
            if(sym[u])
            {
                tri_row_col(qq, ti[u], tj[u]);
                pb[u] = Dk + 8 * tj[u] + g + (size_t)t * FLDK; ldb[u] = FLDK;
            }
            else
            {
                const int r = qq - nsym;
                ti[u] = r >> 2; tj[u] = r & 3;
                pb[u] = Gs + 8 * tj[u] + g + (size_t)t * FLDG; ldb[u] = FLDG;
            }
            pa[u] = Dk + 8 * ti[u] + g + (size_t)t * FLDK;
        }
        double acc[4][2] = {{0., 0.}, {0., 0.}, {0., 0.}, {0., 0.}};
        for(int ks = 0; ks < ksteps; ks++)
#pragma unroll
            for(int u = 0; u < 4; u++)
                dmma(acc[u][0], acc[u][1], pa[u][(size_t)ks * 4 * FLDK], pb[u][(size_t)ks * 4 * ldb[u]]);
#pragma unroll
        for(int u = 0; u < 4; u++)
        {
            if(!live[u]) continue;
            const int k1 = 8 * ti[u] + g;
            if(sym[u])
            {
                // M[k1][k2], k2 = 8 tj + 2t + h, lower triangle: once (the readers scale it by fx^2 and fy^2)
#pragma unroll
                for(int h = 0; h < 2; h++)
                {
                    const int k2 = 8 * tj[u] + 2 * t + h;
                    if(k1 >= nk || k2 > k1) continue;
                    Aw[2 + k1 * (k1 + 1) / 2 + k2] = acc[u][h];
                }
            }
            else if(k1 < FMAXK)
            {
                Cs[k1 * 33 + 8 * tj[u] + 2 * t] = acc[u][0];
                Cs[k1 * 33 + 8 * tj[u] + 2 * t + 1] = acc[u][1];
            }
        }
    }
    // ---- geometry x geometry and J'x over the geometry: entry (i >= j) of the 14 x 14 block, then the 14 gradients
    if(tid < 105 + 14)
    {
        int i, j;
        if(tid < 105) tri_row_col(tid, i, j);
        else { i = tid - 105; j = -1; }
        double s = 0.;
        for(int k = 0; k < NWH; k++)
        {
            const double* gk = Gs + (size_t)k * FLDG;
            if(j >= 0) s += gk[i] * gk[j] + gk[14 + i] * gk[14 + j];
            else       s += gk[i] * gk[28] + gk[14 + i] * gk[29];
        }
        if(j >= 0) { GG[i * 14 + j] = s; GG[j * 14 + i] = s; }
        else GG[196 + i] = s;
    }
    __syncthreads();

    // ---- 4. the rest of the item's blocks. Local geometry column l (after the 2 nk knot columns) -> G column
    auto gcol = [&](int l) { return l < ncam ? l : 12 + (l - ncam); };
    const int ngeo = ncam + nwarp;
    double* Ag = Aw + compact_geo0(nk);
    // geometry rows of A: [geom l][knot (k,s)] = f_s C[k][gcol(l) + 14 s];  [geom l][geom l2 <= l] = GG
    for(int e = tid; e < ngeo * (2 * nk + ngeo); e += 128)
    {
        const int l = e / (2 * nk + ngeo), c = e - l * (2 * nk + ngeo);
        double v;
        if(c < 2 * nk) { const int k = c >> 1, sfc = c & 1; v = (sfc ? fy : fx) * Cs[k * 33 + gcol(l) + 14 * sfc]; }
        else
        {
            const int l2 = c - 2 * nk;
            if(l2 > l) continue;
            v = GG[gcol(l) * 14 + gcol(l2)];
        }
        Ag[(size_t)l * nsh + c] = v;
    }
    // -J'x over the shared columns
    for(int c = tid; c < nsh; c += 128)
    {
        double v;
        if(c < 2 * nk) { const int k = c >> 1, sfc = c & 1; v = (sfc ? fy : fx) * Cs[k * 33 + 28 + sfc]; }
        else v = GG[196 + gcol(c - 2 * nk)];
        Ag[(size_t)ngeo * nsh + c] = -v;
    }
    // the frame: B [6][cap], D, gf
    {
        double* B = N.wi_B + (size_t)w_item * 6 * N.cap;
        for(int e = tid; e < 6 * nsh; e += 128)
        {
            const int p = e / nsh, c = e - p * nsh;
            double v;
            if(c < 2 * nk) { const int k = c >> 1, sfc = c & 1; v = (sfc ? fy : fx) * Cs[k * 33 + 6 + p + 14 * sfc]; }
            else v = GG[(6 + p) * 14 + gcol(c - 2 * nk)];
            B[(size_t)p * N.cap + c] = v;
        }
        if(tid < 36) N.wi_D[(size_t)w_item * 36 + tid] = GG[(6 + tid / 6) * 14 + 6 + tid % 6];
        if(tid >= 64 && tid < 70) N.wi_gf[(size_t)w_item * 6 + tid - 64] = GG[196 + 6 + tid - 64];
    }
}

// |J g|^2 over the board rows from the blocks: g_w' [A B'; B D] g_w per observation. part[w] = that. One CTA per item, one
// entry of the lower triangle of A per thread and step (all loads independent); the per-thread sums are added in a fixed tree.
// A is in the compact layout (normal.h); each entry is formed as the full layout holds it, the zeros across the two
// surfaces included
__global__ void __launch_bounds__(128)
quadform_items_kernel(DevProblem P, NormalBuffers N, const double* __restrict__ g_full, int Nitems, double* __restrict__ part)
{
    __shared__ double s_g[168];
    __shared__ double s_red[128];
    const int w = blockIdx.x, tid = threadIdx.x;
    const int nsh = N.wi_nsh[w], nk = ~N.wi_lda[w];
    const double* A = N.wi_A + N.wi_Aoff[w];
    const double* Ag = A + compact_geo0(nk);
    const double fx2 = A[0], fy2 = A[1];
    const int* cols = N.wi_cols + (size_t)w * N.cap;
    const int iframe = P.obs_board[3 * w + 2];
    for(int i = tid; i < nsh; i += 128) s_g[i] = g_full[N.state_index(cols[i])];
    __syncthreads();
    double q = 0.;
    // shared x shared (A symmetric, lower stored): sum over i >= j of (2 - [i == j]) g_i A_ij g_j
    const int nent = nsh * (nsh + 1) / 2;
    for(int e = tid; e < nent; e += 128)
    {
        int i, j;
        tri_row_col(e, i, j);
        double a;
        if(i >= 2 * nk)     a = Ag[(size_t)(i - 2 * nk) * nsh + j];
        else if((i ^ j) & 1) a = 0.;
        else                a = __dmul_rn(i & 1 ? fy2 : fx2, A[2 + (i >> 1) * ((i >> 1) + 1) / 2 + (j >> 1)]);
        const double v = a * s_g[i] * s_g[j];
        q += i == j ? v : 2. * v;
    }
    // frame: 2 g_f' B g_s + g_f' D g_f
    if(P.opt_frames)
    {
        const double* B = N.wi_B + (size_t)w * 6 * N.cap;
        double gf[6];
        for(int p = 0; p < 6; p++) gf[p] = g_full[P.i_frame0 + 6 * iframe + p];
        for(int i = tid; i < nsh; i += 128)
        {
            double sv = 0.;
            for(int p = 0; p < 6; p++) sv += gf[p] * B[(size_t)p * N.cap + i];
            q += 2. * s_g[i] * sv;
        }
        if(tid == 0)
        {
            const double* D = N.wi_D + (size_t)w * 36;
            for(int p = 0; p < 6; p++)
                for(int rr = 0; rr < 6; rr++) q += gf[p] * D[p * 6 + rr] * gf[rr];
        }
    }
    tree_sum<128>(s_red, q);
    if(tid == 0) part[w] = s_red[0];
}

// The board observations of the evaluation at `out`: x, |x|^2, and the per-item blocks. The caller has cleared
// N.active / N.stat for this evaluation and has unpacked the state (launch_unpack_state)
bool launch_fused_boards(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& out, double* norm_part, cudaStream_t s, int* nlaunch)
{
    constexpr size_t smem_max = fused_smem_bytes(FMAXCORNERS);
    if(!set_max_dynamic_smem<fused_boards_kernel<4>>((int)smem_max) || !set_max_dynamic_smem<fused_boards_kernel<3>>((int)smem_max)) return false;
    const int NWH = dp.W * dp.H;
    if(NWH > FMAXCORNERS) { set_error("internal error: the fused path needs W*H <= %d", FMAXCORNERS); return false; }
    const int K = (NWH + 3) & ~3;
    const size_t smem = fused_smem_bytes(K);
    if(dp.lens_kind == LENS_SPLINED3) fused_boards_kernel<4><<<dp.Nobs_board, 128, smem, s>>>(dp, N, out.x, norm_part, K);
    else                              fused_boards_kernel<3><<<dp.Nobs_board, 128, smem, s>>>(dp, N, out.x, norm_part, K);
    sum_partials_kernel<256><<<1, 256, 0, s>>>(norm_part, dp.Nobs_board, out.norm2);
    *nlaunch += 2;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

bool launch_quadform_boards(const DevProblem& dp, const NormalBuffers& N, const double* g_full, double* part, double* out, cudaStream_t s, int* nlaunch)
{
    if(dp.Nobs_board <= 0) return true;
    quadform_items_kernel<<<dp.Nobs_board, 128, 0, s>>>(dp, N, g_full, dp.Nobs_board, part);
    sum_partials_kernel<256><<<1, 256, 0, s>>>(part, dp.Nobs_board, out);
    *nlaunch += 2;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace mb200
