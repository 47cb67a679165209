// The reduced normal equations from the per-item blocks that normal.cu leaves: the Gram matrix of each work item (a
// board or point observation) over the shared unknowns it touches (wi_A), and the blocks B, D, gf that couple it to its
// eliminated group (a frame or a point). Here
//
//     S = sum_items A_w  -  sum_groups Y_g' Y_g ,      Y_g = inv(L_Dg) B_g ,  D_g = L_Dg L_Dg'
//
// is formed by OWNER-COMPUTES: one CTA per 64x64 tile of the lower triangle of S adds up everything that lands in its
// tile, in a fixed order, and writes the tile once. No fp64 atomics, so the result -- and with it the iteration count of
// a solve -- is the same from run to run, as the reference's is.
//
//   groups_panels_kernel          one CTA per group: D, its Cholesky factor, Y_g written as dense
//                                 6x64 panels per 64-column block the group reaches (zeros where it does
//                                 not), -inv(L_D) gf as the column that forms the right-hand side
//   tile_plan / tile_slots        what each tile sums, and over how many CTAs
//   schur_tiles_kernel            one CTA per tile. Phase A: the items' Gram blocks, each warp owning the
//                                 tile rows = its number (mod 8); a compact block (a fused board observation,
//                                 normal.h) brings a knot row's own surface only. Phase S: the panels of the groups that
//                                 reach both block r and block c, stacked along K, through DMMA 8x8x4;
//                                 operands staged with cp.async, double buffered.
//   [sharded solves]              the tiles summed over the ranks
//   reg_blocks_kernel             the regularization rows: one thread per knot (or per unknown), the
//                                 single owner of the entries it adds to
//   tri_rows_kernel               the triangulated-point rows: one CTA per entry of the extrinsics block
//                                 and of the gradient rows, walking the pairs of the entry's camera
//   finish_rhs_kernel             g' and the shared part of J'x out of the two gradient rows
//   backsub_panels_kernel         after the solve: the eliminated unknowns
//
// The right-hand side travels as row n_c of S (forward substitution for free), the plain gradient J'x of the shared
// unknowns as row n_c+1.
//
// Replaces what the reference gets from libdogleg's Jt*x and CHOLMOD's A*A' + factorization of the full
// sparse JtJ (call site mrcal.c:6435).
#include "comm.h"
#include "normal_items.cuh"

namespace mb200 {

namespace {

constexpr int TB = 64;          // tile
constexpr int TLD = 68;         // row stride of tiles and panels in shared memory (conflict-free DMMA fragment loads)
constexpr int kChunkItems = 64; // phase A: items staged per chunk
constexpr int kChunkGroups = 6; // phase S: groups per K chunk (36 rows); two CTAs of ~88 KB per SM

}  // namespace

// 6x6 (or 3x3) Cholesky factor and its inverse, in registers of one thread. False if not positive definite
__device__ bool chol6_inverse(double* Linv, const double* D, int n)
{
    double L[6][6] = {};
    for(int j = 0; j < n; j++)
    {
        double s = D[j * 6 + j];
        for(int k = 0; k < j; k++) s -= L[j][k] * L[j][k];
        if(!(s > 0.)) return false;
        L[j][j] = sqrt(s);
        for(int i = j + 1; i < n; i++)
        {
            double t = D[i * 6 + j];
            for(int k = 0; k < j; k++) t -= L[i][k] * L[j][k];
            L[i][j] = t / L[j][j];
        }
    }
    for(int i = 0; i < 36; i++) Linv[i] = 0.;
    for(int c = 0; c < n; c++)
    {
        Linv[c * 6 + c] = 1. / L[c][c];
        for(int i = c + 1; i < n; i++)
        {
            double t = 0.;
            for(int k = c; k < i; k++) t += L[i][k] * Linv[k * 6 + c];
            Linv[i * 6 + c] = -t / L[i][i];
        }
    }
    return true;
}

// One CTA per elimination group
__global__ void __launch_bounds__(256)
groups_panels_kernel(NormalBuffers N, double lambda, int n_c, int nblk)
{
    __shared__ double s_D[36], s_gf[6], s_Linv[36], s_h[6];
    extern __shared__ unsigned s_blk[];   // [bwords] the blocks the group reaches
    const int grp = blockIdx.x, tid = threadIdx.x;
    const int i0 = N.grp_ptr[grp], i1 = N.grp_ptr[grp + 1];
    const int nelim = grp < N.Nframe_groups ? 6 : 3;
    if(tid < 36)
    {
        double v = 0.;
        for(int i = i0; i < i1; i++) v += N.wi_D[(size_t)N.grp_items[i] * 36 + tid];
        const int p = tid / 6, q = tid % 6;
        if(p == q && p < nelim) v += lambda;
        s_D[tid] = v;
    }
    if(tid >= 64 && tid < 70)
    {
        double v = 0.;
        for(int i = i0; i < i1; i++) v += N.wi_gf[(size_t)N.grp_items[i] * 6 + (tid - 64)];
        s_gf[tid - 64] = v;
    }
    for(int i = tid; i < N.bwords; i += 256) s_blk[i] = 0u;
    __syncthreads();
    if(tid == 0)
    {
        double Linv[36];
        // a group nobody observes (or all of whose observations are outliers) has D = 0: the reference would hand
        // CHOLMOD a singular matrix here (mrcal.c:4826-4833); report it
        if(!chol6_inverse(Linv, s_D, nelim))
        {
            atomicCAS(N.info, 0, 1000000000 + grp);
            for(int i = 0; i < 36; i++) Linv[i] = 0.;
        }
        const int e0 = N.e0 + group_col0(N, grp);
        for(int p = 0; p < 6; p++)
        {
            double t = 0.;
            for(int q = 0; q <= p; q++) t += Linv[p * 6 + q] * s_gf[q];
            s_h[p] = t;
            N.grp_h[(size_t)grp * 6 + p] = t;
            if(p < nelim) N.g_full[e0 + p] = s_gf[p];    // the eliminated part of the full gradient
        }
        for(int i = 0; i < 36; i++) { s_Linv[i] = Linv[i]; N.grp_Linv[(size_t)grp * 36 + i] = Linv[i]; }
    }
    // the blocks this group reaches (the block of column n_c always: the right-hand side)
    for(int i = i0; i < i1; i++)
    {
        const int w = N.grp_items[i];
        const int nsh = N.wi_nsh[w];
        const unsigned short* cc = N.wi_ccol + (size_t)w * N.capA;
        for(int l = tid; l < nsh; l += 256) { const int b = cc[l] >> 6; atomicOr(&s_blk[b >> 5], 1u << (b & 31)); }
    }
    if(tid == 0) { const int b = n_c >> 6; atomicOr(&s_blk[b >> 5], 1u << (b & 31)); }
    __syncthreads();
    double* Yg = N.Ypan + (size_t)grp * N.nblk_max * kYpanel;
    for(int b = 0; b < nblk; b++)
    {
        if(!((s_blk[b >> 5] >> (b & 31)) & 1u)) continue;   // uniform
        for(int e = tid; e < kYpanel; e += 256) Yg[(size_t)b * kYpanel + e] = 0.;
        if(tid == 0) atomicOr(&N.grp_present[(size_t)b * N.gwords + (grp >> 5)], 1u << (grp & 31));
    }
    for(int i = tid; i < N.bwords; i += 256) N.grp_blkmask[(size_t)grp * N.bwords + i] = s_blk[i];
    __syncthreads();
    // Y = inv(L) B, item after item: items of one group may share columns (the board warp; the intrinsics of a
    // camera seen twice), and the order of the additions is part of the result
    for(int i = i0; i < i1; i++)
    {
        const int w = N.grp_items[i];
        const int nsh = N.wi_nsh[w];
        const unsigned short* cc = N.wi_ccol + (size_t)w * N.capA;
        const double* B = N.wi_B + (size_t)w * 6 * N.cap;
        for(int l = tid; l < nsh; l += 256)
        {
            const int c = cc[l];
            double* y = Yg + (size_t)(c >> 6) * kYpanel + (c & 63);
            double bq[6];
#pragma unroll
            for(int q = 0; q < 6; q++) bq[q] = q < nelim ? B[(size_t)q * N.cap + l] : 0.;
#pragma unroll
            for(int p = 0; p < 6; p++)
            {
                double t = 0.;
#pragma unroll
                for(int q = 0; q < 6; q++) if(q <= p) t += s_Linv[p * 6 + q] * bq[q];
                if(p < nelim) y[p * kYld] += t;
            }
        }
        __syncthreads();
    }
    if(tid < 6) Yg[(size_t)(n_c >> 6) * kYpanel + tid * kYld + (n_c & 63)] = -s_h[tid];
}

struct alignas(16) TileCommon
{
    int wl[2048];      // items (or groups) that reach both blocks of the tile
    int scan[256];
    int count;
    int pad[3];        // what follows in shared memory is accessed 16 bytes at a time (bulk copies, double2)
    unsigned long long bar[2];   // mbarriers of the two panel buffers of phase S
};
static_assert(sizeof(TileCommon) % 16 == 0, "the tile and the staging buffers behind TileCommon need 16-byte alignment");
struct alignas(16) TileSmemA
{
    double tile[TB * TLD];
    int    meta[kChunkItems][4];           // a0 | na<<16,  b0 | nb<<16,  lda (< 0: compact layout, ~nk),  nsh
    long long base[kChunkItems];
    double f2[kChunkItems][2];             // compact layout: fx*fx, fy*fy
    unsigned char rl[kChunkItems][TB + 4]; // tile row of each local row
    unsigned char cl[kChunkItems][TB + 4]; // tile column of each local column
};
struct alignas(16) TileSmemS
{
    double R[2][6 * kChunkGroups][TLD];
    double C[2][6 * kChunkGroups][TLD];
};
constexpr size_t kTileSmemBody = sizeof(TileSmemA) > sizeof(TileSmemS) ? sizeof(TileSmemA) : sizeof(TileSmemS);
constexpr size_t kTileSmem = sizeof(TileCommon) + kTileSmemBody;

// worklist of the set bits of (rowA[w] & rowB[w]), w in [w0, w1), at most 64 words: ids -> sm.wl, count -> sm.count.
// (the first two warps hold a word per lane; their scan goes through shuffles)
__device__ __forceinline__ void build_worklist(TileCommon& sm, const unsigned* rowA, const unsigned* rowB, int w0, int w1)
{
    const int tid = threadIdx.x, lane = tid & 31;
    unsigned m = 0;
    int cnt = 0, inc = 0;
    if(tid < 64)
    {
        if(tid < w1 - w0) m = rowA[w0 + tid] & rowB[w0 + tid];
        cnt = __popc(m);
        inc = cnt;
#pragma unroll
        for(int o = 1; o < 32; o <<= 1)
        {
            const int v = __shfl_up_sync(0xffffffffu, inc, o);
            if(lane >= o) inc += v;
        }
        if(lane == 31) sm.scan[tid >> 5] = inc;
    }
    __syncthreads();
    if(tid < 64)
    {
        int pos = inc - cnt + (tid >= 32 ? sm.scan[0] : 0);
        while(m) { const int b = __ffs(m) - 1; m &= m - 1; sm.wl[pos++] = 32 * (w0 + tid) + b; }
    }
    if(tid == 0) sm.count = sm.scan[0] + sm.scan[1];
    __syncthreads();
}
constexpr int kPackedExtras = 8;      // doubles behind the packed tiles (sharded solves)
constexpr int kMaxParts = 64;         // a tile's contributors may be split over this many CTAs
constexpr int kCtasPerTile = 4;       // the grid: this many CTAs per tile on average (kernel_ctas()); parts are cut to fit
// (at least kMaxParts: the one tile of a small system, which every observation reaches, may be split as far as a tile can be)
__host__ __device__ inline int kernel_ctas(int ntiles) { return kCtasPerTile * ntiles > kMaxParts ? kCtasPerTile * ntiles : kMaxParts; }

// What each tile has to sum, and over how many CTAs: plan[itile] = (items, groups, parts, -), then the numbers of items
// and of groups in each stretch of 64 bitmap words (kPlanStretches + kPlanGroupStretches ints; a tile CTA walks past the
// stretches that hold nothing of its share without looking at the bitmaps). One warp per tile
constexpr int kPlanStretches = 32, kPlanGroupStretches = 8;
constexpr int kPlanInts = 4 + kPlanStretches + kPlanGroupStretches;
__global__ void __launch_bounds__(256)
tile_plan_kernel(NormalBuffers N, int nblk, int ns_per_item, int ns_per_group, int ns_per_part, bool can_split, int* __restrict__ plan)
{
    const int itile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if(itile >= nblk * (nblk + 1) / 2) return;
    int r, c;
    tri_row_col(itile, r, c);
    const unsigned* wiA = N.wi_present + (size_t)r * N.wwords;
    const unsigned* wiB = N.wi_present + (size_t)c * N.wwords;
    int n_items = 0, n_groups = 0;
    int* mine = plan + (size_t)itile * kPlanInts;
    for(int st = 0; 64 * st < N.wwords; st++)
    {
        int cnt = 0;
        for(int w = 64 * st + lane; w < min(64 * st + 64, N.wwords); w += 32) cnt += __popc(wiA[w] & wiB[w]);
        cnt = warp_sum(cnt);
        if(lane == 0 && st < kPlanStretches) mine[4 + st] = cnt;
        n_items += cnt;
    }
    if(N.Ngroups > 0)
    {
        const unsigned* grA = N.grp_present + (size_t)r * N.gwords;
        const unsigned* grB = N.grp_present + (size_t)c * N.gwords;
        for(int st = 0; 64 * st < N.gwords; st++)
        {
            int cnt = 0;
            for(int w = 64 * st + lane; w < min(64 * st + 64, N.gwords); w += 32) cnt += __popc(grA[w] & grB[w]);
            cnt = warp_sum(cnt);
            if(lane == 0 && st < kPlanGroupStretches) mine[4 + kPlanStretches + st] = cnt;
            n_groups += cnt;
        }
    }
    // what the tile costs one CTA (a cost model: ns_per_item per item of phase A, ns_per_group per group of phase S), cut
    // into parts of ns_per_part each: the kernel ends when its longest CTA does
    const long cost = (long)n_items * ns_per_item + (long)n_groups * ns_per_group;
    int parts = (int)((cost + ns_per_part - 1) / ns_per_part);
    parts = min(kMaxParts, max(1, parts));
    if(!can_split) parts = 1;
    if(lane == 0) { mine[0] = n_items; mine[1] = n_groups; mine[2] = parts; mine[3] = 0; }
}

// The CTAs of schur_tiles_kernel: cta[k] = (tile << 8) | part, the tiles in the kernel's order (late block rows first: they
// carry the most work), the parts of a tile next to each other: slot k of the partial-sum scratch belongs to CTA k, so a
// tile's partial sums are contiguous. The grid holds kernel_ctas(ntiles) CTAs: every tile gets one, the parts beyond
// that as long as there is room. plan[tile][2] <- the parts it got, plan[tile][3] <- its first slot; cta[nctas_max] <- the
// number of CTAs with work. One CTA of 1024 threads
__global__ void __launch_bounds__(1024)
tile_slots_kernel(int ntiles, int* __restrict__ plan, int* __restrict__ cta)
{
    __shared__ int s_scan[1024];
    __shared__ int s_carry, s_room;
    const int tid = threadIdx.x;
    const int nctas_max = kernel_ctas(ntiles);
    if(tid == 0) { s_carry = 0; s_room = nctas_max - ntiles; }
    // if the tiles wish for more extra parts than there is room for, every wish is scaled down alike
    long wish = 0;
    for(int k = tid; k < ntiles; k += 1024) wish += plan[(size_t)k * kPlanInts + 2] - 1;
    tree_sum<1024>(s_scan, (int)wish);
    const long wish_total = s_scan[0];
    __syncthreads();
    for(int k0 = 0; k0 < ntiles; k0 += 1024)
    {
        const int k = k0 + tid;                        // position in launch order
        const int itile = ntiles - 1 - k;
        int extra = k < ntiles ? plan[(size_t)itile * kPlanInts + 2] - 1 : 0;
        if(wish_total > nctas_max - ntiles) extra = (int)((long)extra * (nctas_max - ntiles) / wish_total);
        // the extra parts, granted in launch order while there is room
        int wished;                                    // by the tiles of the chunk
        const int before = block_exclusive_scan<int, 1024>(extra, s_scan, wished);   // by the tiles ahead of this one
        const int room = s_room;
        const int granted = max(0, min(extra, room - before));
        // slots: the tiles ahead took (their 1 + granted): granted_before = min(before, room)
        const int slot0 = s_carry + tid + min(before, room);
        if(k < ntiles)
        {
            plan[(size_t)itile * kPlanInts + 2] = 1 + granted;
            plan[(size_t)itile * kPlanInts + 3] = slot0;
            for(int p = 0; p <= granted; p++) cta[slot0 + p] = (itile << 8) | p;
        }
        __syncthreads();
        if(tid == 1023)
        {
            const int used = min(wished, room);
            s_carry += min(1024, ntiles - k0) + used;
            s_room = room - used;
        }
        __syncthreads();
    }
    if(tid == 0) cta[nctas_max] = s_carry;
}

// One CTA per (64x64 tile of the lower triangle of S, part). A tile that many items / groups reach -- the block row of
// the extrinsics, the board warp and the right-hand side reaches all of them -- is split: each part sums its share of
// the contributors (contiguous ranges of the worklists) into a partial tile; the part that finishes LAST adds the
// partial tiles up in part order. Which part is last varies; what it computes does not.
__global__ void __launch_bounds__(256, 2)
schur_tiles_kernel(NormalBuffers N, double lambda, int n_c, int nblk, bool add_lambda, double* __restrict__ packed,
                   double* __restrict__ part_scratch, int* __restrict__ part_arrive, const int* __restrict__ plan,
                   const int* __restrict__ cta)
{
    extern __shared__ __align__(16) unsigned char dsm_raw[];
    TileCommon& sc = *reinterpret_cast<TileCommon*>(dsm_raw);
    TileSmemA& sa = *reinterpret_cast<TileSmemA*>(dsm_raw + sizeof(TileCommon));
    TileSmemS& ss = *reinterpret_cast<TileSmemS*>(dsm_raw + sizeof(TileCommon));
    __shared__ int s_last;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int ntiles_all = nblk * (nblk + 1) / 2;
    if((int)blockIdx.x >= cta[kernel_ctas(ntiles_all)]) return;
    const int itile = cta[blockIdx.x] >> 8, part = cta[blockIdx.x] & 255;
    const int* pl = plan + (size_t)itile * kPlanInts;
    const int n_items = pl[0], n_groups = pl[1], parts = pl[2], slot0 = pl[3];
    int r, c;
    tri_row_col(itile, r, c);
    const bool diag = r == c;
    const unsigned* wiA = N.wi_present + (size_t)r * N.wwords;
    const unsigned* wiB = N.wi_present + (size_t)c * N.wwords;
    const unsigned* grA = N.grp_present + (size_t)r * N.gwords;
    const unsigned* grB = N.grp_present + (size_t)c * N.gwords;
    if(tid == 0)
    {
        mbar_init(&sc.bar[0], 1);
        mbar_init(&sc.bar[1], 1);
        fence_mbar_init();
    }
    const int item_lo = (int)((long)n_items * part / parts), item_hi = (int)((long)n_items * (part + 1) / parts);
    const int grp_lo = (int)((long)n_groups * part / parts), grp_hi = (int)((long)n_groups * (part + 1) / parts);

    ////////////////////////////// phase A: the items' Gram blocks
    for(int e = tid; e < TB * TLD; e += 256) sa.tile[e] = 0.;
    __syncthreads();
    int seen = 0;
    for(int w0 = 0; w0 < N.wwords && seen < item_hi; w0 += 64)
    {
        // a stretch that holds nothing of this part's share: past it without a look at the bitmaps
        if((w0 >> 6) < kPlanStretches)
        {
            const int cnt = pl[4 + (w0 >> 6)];
            if(cnt == 0 || seen + cnt <= item_lo) { seen += cnt; continue; }
        }
        build_worklist(sc, wiA, wiB, w0, min(w0 + 64, N.wwords));
        const int nwl = sc.count;
        // my share of this stretch of the worklist
        const int lo = max(item_lo - seen, 0), hi = min(item_hi - seen, nwl);
        seen += nwl;
        for(int ch = lo; ch < hi; ch += kChunkItems)
        {
            const int nch = min(kChunkItems, hi - ch);
            // ---- stage: where the item's rows and columns of this tile sit
            if(tid < nch)
            {
                const int w = sc.wl[ch + tid];
                const unsigned short* seg = N.wi_segoff + (size_t)w * (N.nblk_max + 1);
                const int nsh = N.wi_nsh[w];
                const int a0 = seg[r], a1 = seg[r + 1];
                int b0 = seg[c], b1 = seg[c + 1];
                if(b1 > nsh) b1 = nsh;              // the gradient rows are rows only
                if(b0 > b1) b0 = b1;
                sa.meta[tid][0] = a0 | ((a1 - a0) << 16);
                sa.meta[tid][1] = b0 | ((b1 - b0) << 16);
                const int lda = N.wi_lda[w];
                const long long base = N.wi_Aoff[w];
                sa.meta[tid][2] = lda;
                sa.meta[tid][3] = nsh;
                sa.base[tid] = base;
                if(lda < 0) { sa.f2[tid][0] = __ldg(N.wi_A + base); sa.f2[tid][1] = __ldg(N.wi_A + base + 1); }
            }
            __syncthreads();
            for(int e = tid; e < nch * 2 * TB; e += 256)
            {
                const int i = e / (2 * TB), k = e - i * (2 * TB);
                const int w = sc.wl[ch + i];
                const unsigned short* cc = N.wi_ccol + (size_t)w * N.capA;
                if(k < TB)
                {
                    const int a0 = sa.meta[i][0] & 0xffff, na = sa.meta[i][0] >> 16;
                    if(k < na) sa.rl[i][k] = (unsigned char)(cc[a0 + k] - TB * r);
                }
                else
                {
                    const int kk = k - TB;
                    const int b0 = sa.meta[i][1] & 0xffff, nb = sa.meta[i][1] >> 16;
                    if(kk < nb) sa.cl[i][kk] = (unsigned char)(cc[b0 + kk] - TB * c);
                }
            }
            __syncthreads();
            // ---- accumulate. Warp `warp` owns the tile rows = warp (mod 8): no two warps ever touch the same entry, and
            // every entry sees its nonzero contributions in item order. A "task" is one owned row of one item (<= 64 values,
            // two per lane). A knot row of a compact block holds its surface's columns only: lane j takes knot k2 =
            // ceil((b0 - s) / 2) + j of surface s and adds f_s^2 M[k1][k2] at column 2 k2 + s; the zeros across the
            // surfaces are not added (those entries of S start at +0 and receive only zeros). Rows of consecutive tile rows
            // go to different warps, so the few rows an item brings to a tile are spread over the warps. Tasks are taken 4
            // at a time so that their loads are in flight together
            {
                int ti = -1;
                unsigned cur0 = 0, cur1 = 0;
                bool exhausted = false;
                while(!exhausted || cur0 || cur1)
                {
                    // every task is decoded ONCE: where its values are (an element offset into the pool), where they go
                    // in the tile, which of the lane's two columns exist, the factor of a knot row. The kernel is bound by
                    // the instructions it issues here, not by the latency of the loads: 4 tasks in flight are enough
                    constexpr int NT = 4;
                    unsigned src[NT];
                    int dst0[NT], dst1[NT];
                    double scl[NT];
                    unsigned have = 0;   // bit 2u: column `lane` of task u exists, bit 2u+1: column lane+32
                    int cnt = 0;
#pragma unroll
                    for(int u = 0; u < NT; u++)
                    {
                        int item = -1, lrow = 0;
                        while(!exhausted && cur0 == 0 && cur1 == 0)
                        {
                            ti++;
                            if(ti >= nch) { exhausted = true; break; }
                            const int na = sa.meta[ti][0] >> 16, nb = sa.meta[ti][1] >> 16;
                            if(na == 0 || nb == 0) continue;
                            cur0 = __ballot_sync(0xffffffffu, lane < na && (sa.rl[ti][lane] & 7) == warp);
                            cur1 = __ballot_sync(0xffffffffu, lane + 32 < na && (sa.rl[ti][lane + 32] & 7) == warp);
                        }
                        if(cur0) { item = ti; lrow = __ffs(cur0) - 1; cur0 &= cur0 - 1; cnt++; }
                        else if(cur1) { item = ti; lrow = 32 + __ffs(cur1) - 1; cur1 &= cur1 - 1; cnt++; }
                        src[u] = 0u; dst0[u] = dst1[u] = 0; scl[u] = 1.;
                        if(item >= 0)
                        {
                            const int a = (sa.meta[item][0] & 0xffff) + lrow;
                            const int b0 = sa.meta[item][1] & 0xffff, nb = sa.meta[item][1] >> 16;
                            const int lda = sa.meta[item][2];
                            const int nk = lda < 0 ? ~lda : 0;
                            const int trow = (int)sa.rl[item][lrow] * TLD;
                            if(lda >= 0 || a >= 2 * nk)
                            {
                                // a row as stored: the full layout, or a geometry / gradient row of a compact block (nsh wide;
                                // the two gradient rows are one stored row)
                                const int nsh = sa.meta[item][3];
                                const long long row = lda >= 0 ? (long long)a * lda : compact_geo0(nk) + (long long)(min(a, nsh) - 2 * nk) * nsh;
                                // lower triangle of the item's block: local column <= local row (always true off the diagonal tiles)
                                const bool p0 = lane < nb && b0 + lane <= a, p1 = lane + 32 < nb && b0 + lane + 32 <= a;
                                have |= (p0 ? 1u : 0u) << (2 * u) | (p1 ? 2u : 0u) << (2 * u);
                                src[u] = (unsigned)(sa.base[item] + row + b0 + lane);
                                dst0[u] = trow + (p0 ? sa.cl[item][lane] : 0);
                                dst1[u] = trow + (p1 ? sa.cl[item][lane + 32] : 0);
                            }
                            else
                            {
                                const int k1 = a >> 1, sfc = a & 1;
                                const int k2 = ((b0 + 1 - sfc) >> 1) + lane, col = 2 * k2 + sfc - b0;
                                const bool p = k2 <= k1 && col < nb;
                                have |= (p ? 1u : 0u) << (2 * u);
                                src[u] = (unsigned)(sa.base[item] + 2 + k1 * (k1 + 1) / 2 + k2);
                                dst0[u] = trow + (p ? sa.cl[item][col] : 0);
                                scl[u] = sa.f2[item][sfc];
                            }
                        }
                    }
                    if(cnt == 0) break;
                    double v0[NT], v1[NT];
#pragma unroll
                    for(int u = 0; u < NT; u++)
                    {
                        v0[u] = (have >> (2 * u)) & 1u ? __ldg(N.wi_A + src[u]) : 0.;
                        v1[u] = (have >> (2 * u + 1)) & 1u ? __ldg(N.wi_A + src[u] + 32) : 0.;
                    }
#pragma unroll
                    for(int u = 0; u < NT; u++)
                    {
                        // (the product is rounded on its own, as the full layout's entries were: no contraction into the sum)
                        if((have >> (2 * u)) & 1u) sa.tile[dst0[u]] += __dmul_rn(scl[u], v0[u]);
                        if((have >> (2 * u + 1)) & 1u) sa.tile[dst1[u]] += v1[u];
                        // two items may bring the same tile entry to DIFFERENT lanes of this warp: the additions of one task
                        // are done (and visible to the warp) before those of the next
                        __syncwarp();
                    }
                }
            }
            __syncthreads();
        }
    }

    ////////////////////////////// phase S: minus the groups' Y'Y, through the tensor pipe
    // accumulators start at -tile and collect +Y'Y: the tile is -acc. 8 warps as 4 x 2, warp tile 16 x 32
    const int wm = warp >> 1, wn = warp & 1, g = lane >> 2, t = lane & 3;
    double acc[2][4][2];
#pragma unroll
    for(int a = 0; a < 2; a++)
#pragma unroll
        for(int b = 0; b < 4; b++)
        {
            const double2 v = *reinterpret_cast<const double2*>(&sa.tile[(wm * 16 + a * 8 + g) * TLD + wn * 32 + b * 8 + 2 * t]);
            acc[a][b][0] = -v.x;
            acc[a][b][1] = -v.y;
        }
    __syncthreads();
    seen = 0;
    unsigned bar_phase = 0;   // bit b: the parity the next wait on buffer b looks for
    for(int w0 = 0; w0 < N.gwords && N.Ngroups > 0 && seen < grp_hi; w0 += 64)
    {
        if((w0 >> 6) < kPlanGroupStretches)
        {
            const int cnt = pl[4 + kPlanStretches + (w0 >> 6)];
            if(cnt == 0 || seen + cnt <= grp_lo) { seen += cnt; continue; }
        }
        build_worklist(sc, grA, grB, w0, min(w0 + 64, N.gwords));
        const int nwl_all = sc.count;
        const int lo = max(grp_lo - seen, 0), hi = min(grp_hi - seen, nwl_all);
        seen += nwl_all;
        const int nwl = hi - lo;
        if(nwl <= 0) continue;
        const int nchunks = (nwl + kChunkGroups - 1) / kChunkGroups;
        // what the generic proxy wrote to this memory (phase A, the zero rows of an earlier stretch) comes before what
        // the bulk copies write
        fence_proxy_async();
        __syncthreads();
        // rows 6 i .. 6 i + 5 of the K panel <- group i of the chunk: ONE bulk copy (TMA) per group and side -- the panels
        // are contiguous in Ypan and carry the row padding of the shared-memory layout; a bulk copy has a fixed cost in the
        // copy engine, whatever its size -- issued by one thread each, all counted on the buffer's
        // mbarrier. No thread spends instructions on moving the data
        static_assert(kYld == TLD, "the panels of Ypan are copied as they are");
        const int sides = diag ? 1 : 2;
        auto stage = [&](int chunk, int buf)
        {
            const int ng = min(kChunkGroups, nwl - chunk * kChunkGroups);
            if(tid == 0) mbar_arrive_expect_tx(&sc.bar[buf], (unsigned)(sides * ng * kYpanel * sizeof(double)));
            if(tid < sides * ng)
            {
                const int side = tid >= ng ? 1 : 0, gi = tid - side * ng;
                const int grp = sc.wl[lo + chunk * kChunkGroups + gi];
                const double* src = N.Ypan + ((size_t)grp * N.nblk_max + (side == 0 ? r : c)) * kYpanel;
                bulk_load(side == 0 ? &ss.R[buf][6 * gi][0] : &ss.C[buf][6 * gi][0], src, (unsigned)(kYpanel * sizeof(double)), &sc.bar[buf]);
            }
        };
        stage(0, 0);
        for(int ch = 0; ch < nchunks; ch++)
        {
            const int buf = ch & 1;
            if(ch + 1 < nchunks) stage(ch + 1, buf ^ 1);   // (that buffer was read last in iteration ch-1, which ended with a barrier)
            mbar_wait(&sc.bar[buf], (bar_phase >> buf) & 1u);
            bar_phase ^= 1u << buf;
            const int ng = min(kChunkGroups, nwl - ch * kChunkGroups);
            const int ksteps = (6 * ng + 3) >> 2;
            if(6 * ng < 4 * ksteps)
            {
                // the K rows up to the next multiple of 4: zeros (only ever in the last chunk of a stretch)
                const int npad = 4 * ksteps - 6 * ng;
                for(int e = tid; e < sides * npad * TB; e += 256)
                {
                    const int side = e / (npad * TB), rem = e - side * (npad * TB);
                    const int row = 6 * ng + rem / TB, col = rem & (TB - 1);
                    (side == 0 ? ss.R[buf][row] : ss.C[buf][row])[col] = 0.;
                }
                __syncthreads();
            }
            const double* Rb = &ss.R[buf][0][0];
            const double* Cb = diag ? Rb : &ss.C[buf][0][0];
            for(int ks = 0; ks < ksteps; ks++)
            {
                double af[2], bf[4];
#pragma unroll
                for(int a = 0; a < 2; a++) af[a] = Rb[(ks * 4 + t) * TLD + wm * 16 + a * 8 + g];
#pragma unroll
                for(int b = 0; b < 4; b++) bf[b] = Cb[(ks * 4 + t) * TLD + wn * 32 + b * 8 + g];
#pragma unroll
                for(int a = 0; a < 2; a++)
#pragma unroll
                    for(int b = 0; b < 4; b++) dmma(acc[a][b][0], acc[a][b][1], af[a], bf[b]);
            }
            __syncthreads();   // this buffer is staged again two chunks from now
        }
    }

    ////////////////////////////// a split tile: leave the partial sum; the last part to arrive adds them up in part order
    if(parts > 1)
    {
        double* mine = part_scratch + (size_t)(slot0 + part) * (TB * TB);
#pragma unroll
        for(int a = 0; a < 2; a++)
#pragma unroll
            for(int b = 0; b < 4; b++)
                *reinterpret_cast<double2*>(&mine[(wm * 16 + a * 8 + g) * TB + wn * 32 + b * 8 + 2 * t]) = make_double2(acc[a][b][0], acc[a][b][1]);
        __threadfence();
        __syncthreads();
        if(tid == 0) s_last = atomicAdd(&part_arrive[itile], 1) == parts - 1;
        __syncthreads();
        if(!s_last) return;
        __threadfence();
#pragma unroll
        for(int a = 0; a < 2; a++)
#pragma unroll
            for(int b = 0; b < 4; b++) acc[a][b][0] = acc[a][b][1] = 0.;
        for(int p = 0; p < parts; p++)
        {
            const double* src = part_scratch + (size_t)(slot0 + p) * (TB * TB);
#pragma unroll
            for(int a = 0; a < 2; a++)
#pragma unroll
                for(int b = 0; b < 4; b++)
                {
                    const double2 v = __ldcg(reinterpret_cast<const double2*>(&src[(wm * 16 + a * 8 + g) * TB + wn * 32 + b * 8 + 2 * t]));
                    acc[a][b][0] += v.x;
                    acc[a][b][1] += v.y;
                }
        }
    }

    ////////////////////////////// sharded solve: the raw tile goes to the tile-packed buffer (lower-triangle tiles only, each
    // contiguous) that is all-reduced; unpack_tiles_kernel finishes the job on the sum
    if(packed != nullptr)
    {
        double* dstt = packed + (size_t)itile * (TB * TB);
#pragma unroll
        for(int a = 0; a < 2; a++)
#pragma unroll
            for(int b = 0; b < 4; b++)
                *reinterpret_cast<double2*>(&dstt[(wm * 16 + a * 8 + g) * TB + wn * 32 + b * 8 + 2 * t]) = make_double2(-acc[a][b][0], -acc[a][b][1]);
        return;
    }
    ////////////////////////////// write the tile. Rows >= n_c: the right-hand side (row n_c), the plain gradient (row n_c+1), padding
#pragma unroll
    for(int a = 0; a < 2; a++)
#pragma unroll
        for(int b = 0; b < 4; b++)
        {
            const int i = TB * r + wm * 16 + a * 8 + g;
            const int j0 = TB * c + wn * 32 + b * 8 + 2 * t;
            double out[2];
#pragma unroll
            for(int h = 0; h < 2; h++)
            {
                const int j = j0 + h;
                const double v = -acc[a][b][h];
                if(i < n_c)           out[h] = v + ((i == j && add_lambda) ? lambda : 0.);
                else if(i <= n_c + 1) out[h] = j < n_c ? v : (i == j ? 1. : 0.);
                else                  out[h] = i == j ? 1. : 0.;
            }
            double* dst = &N.S[(size_t)i * N.ldS + j0];
            if(j0 + 1 <= i) *reinterpret_cast<double2*>(dst) = make_double2(out[0], out[1]);
            else if(j0 <= i) dst[0] = out[0];
        }
}

// Sharded solves: what every rank has to know about the others' frame blocks rides behind the tiles in the same
// all-reduce: extras[0] = this rank has a singular elimination block
__global__ void pack_extras_kernel(NormalBuffers N, double* __restrict__ extras)
{
    if(threadIdx.x == 0 && blockIdx.x == 0) extras[0] = N.info[0] != 0 ? 1. : 0.;
}
__global__ void unpack_extras_kernel(NormalBuffers N, const double* __restrict__ extras)
{
    // a block that is singular on ONE rank sends every rank down the same path
    if(threadIdx.x == 0 && blockIdx.x == 0 && extras[0] != 0. && N.info[0] == 0) N.info[0] = 2000000000;
}

// tile-packed (summed over the ranks) -> the lower triangle of S, with the diagonal loading and the padding rows
__global__ void __launch_bounds__(256)
unpack_tiles_kernel(NormalBuffers N, const double* __restrict__ packed, double lambda, int n_c, int nblk)
{
    int r, c;
    tri_row_col((int)blockIdx.x, r, c);
    const double* src = packed + (size_t)blockIdx.x * (TB * TB);
    for(int e = threadIdx.x; e < TB * TB; e += 256)
    {
        const int i = TB * r + e / TB, j = TB * c + (e & (TB - 1));
        if(j > i) continue;
        const double v = src[e];
        double out;
        if(i < n_c)           out = v + (i == j ? lambda : 0.);
        else if(i <= n_c + 1) out = j < n_c ? v : (i == j ? 1. : 0.);
        else                  out = i == j ? 1. : 0.;
        N.S[(size_t)i * N.ldS + j] = out;
    }
}

// The regularization rows (mrcal.c:5655-5955): each touches 1..3 shared unknowns, and the rows of one spline knot
// (radial, tangential) touch the same two. One thread per knot / per unknown: the single owner of what it adds to.
// Blocks whose unknowns no observation touches stay out of S (inactive_step_kernel solves them in closed form);
// their gradient still goes to g_full.
// every_rank: the sharded path adds these AFTER the cross-rank reduction, on every rank alike
__global__ void reg_blocks_kernel(DevProblem P, NormalBuffers N, int n_c, const double* __restrict__ x,
                                  const double* __restrict__ Jval, const int* __restrict__ Jcol, bool every_rank)
{
    if(!P.reg_owner && !every_rank) return;
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if(t >= reg_block_count(P, N.splined)) return;
    const RegBlock b = reg_block(P, N.splined, t);
    const int m0 = b.m0, nrows = b.nrows, j0 = b.j0, ncol = b.ncol;

    int col[3], ci[3];
    double gk[3] = {0., 0., 0.}, H[3][3] = {};
    bool all_active = true;
    for(int k = 0; k < ncol; k++)
    {
        col[k] = Jcol[j0 + k];
        ci[k] = N.cidx[N.reduced_index(col[k])];
        if(ci[k] < 0) all_active = false;
    }
    for(int rr = 0; rr < nrows; rr++)
    {
        const double xm = x[m0 + rr];
        double v[3];
        for(int k = 0; k < ncol; k++) { v[k] = Jval[j0 + rr * ncol + k]; gk[k] += v[k] * xm; }
        for(int k = 0; k < ncol; k++)
            for(int l = 0; l <= k; l++) H[k][l] += v[k] * v[l];
    }
    if(!all_active)
    {
        for(int k = 0; k < ncol; k++) N.g_full[col[k]] = gk[k];
        return;
    }
    for(int k = 0; k < ncol; k++)
    {
        N.S[(size_t)n_c * N.ldS + ci[k]] -= gk[k];
        N.S[(size_t)(n_c + 1) * N.ldS + ci[k]] -= gk[k];
        for(int l = 0; l <= k; l++)
        {
            const int hi = ci[k] > ci[l] ? ci[k] : ci[l], lo = ci[k] > ci[l] ? ci[l] : ci[k];
            N.S[(size_t)hi * N.ldS + lo] += H[k][l];
        }
    }
}

// The triangulated-point rows (mrcal.c:5180-5653) touch the extrinsics of the two cameras of a pair only. One CTA per
// entry of the extrinsics x extrinsics block of S (t < nx (nx+1) / 2, lower triangle) and of the two gradient rows (the
// nx CTAs behind): its threads take the pairs that see the entry's first camera (tri_cam_rows, in order) in turn, each
// adds what a row brings to the entry -- the product of the row's values on the two columns (a pair of observations of
// the same camera names each column twice: the values are summed) -- and the threads' sums are added in a fixed tree.
// Every column is in the coupled system: mark_tri_active_kernel made it so
__global__ void __launch_bounds__(256)
tri_rows_kernel(DevProblem P, NormalBuffers N, int n_c, const double* __restrict__ x, const double* __restrict__ Jval,
                const int* __restrict__ Jcol, const int* __restrict__ rowptr)
{
    __shared__ double s_part[8];
    const int nx = 6 * P.Ncam_e;
    const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const int ntri = nx * (nx + 1) / 2;
    int ka, kb = -1;   // kb < 0: the gradient entry of column ka
    if(t < ntri) tri_row_col(t, ka, kb);
    else ka = t - ntri;
    const int ca = P.i_extr0 + ka, cb = P.i_extr0 + (kb >= 0 ? kb : 0);
    const int ia = N.cidx[N.reduced_index(ca)], ib = N.cidx[N.reduced_index(cb)];
    if(ia < 0 || (kb >= 0 && ib < 0)) return;   // (CTA-uniform)
    const int e = ka / 6;
    double sum = 0.;
    for(int k = P.tri_cam_ptr[e] + tid; k < P.tri_cam_ptr[e + 1]; k += 256)
    {
        const int m = P.m_tri0 + P.tri_cam_rows[k];
        double va = 0., vb = 0.;
        for(int j = rowptr[m]; j < rowptr[m + 1]; j++)
        {
            const int c = Jcol[j];
            if(c == ca) va += Jval[j];
            if(c == cb) vb += Jval[j];
        }
        sum += kb >= 0 ? va * vb : va * x[m];
    }
    sum = warp_sum(sum);
    if(lane == 0) s_part[tid >> 5] = sum;
    __syncthreads();
    if(tid != 0) return;
    sum = ((s_part[0] + s_part[1]) + (s_part[2] + s_part[3])) + ((s_part[4] + s_part[5]) + (s_part[6] + s_part[7]));
    if(kb >= 0) N.S[(size_t)ia * N.ldS + ib] += sum;
    else
    {
        N.S[(size_t)n_c * N.ldS + ia] -= sum;
        N.S[(size_t)(n_c + 1) * N.ldS + ia] -= sum;
    }
}

// gs = g' and the shared part of J'x out of rows n_c, n_c+1 of S; row n_c+1 becomes plain padding
__global__ void finish_rhs_kernel(NormalBuffers N, int n_c)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= n_c) return;
    N.gs[c] = -N.S[(size_t)n_c * N.ldS + c];
    N.g_full[N.state_index(N.cinv[c])] = -N.S[(size_t)(n_c + 1) * N.ldS + c];
    N.S[(size_t)(n_c + 1) * N.ldS + c] = 0.;
}

// df_g = -inv(L_D)' (h + Y ds): one CTA of 4 warps per group; warp w takes the blocks w, w+4, ... the group reaches, the
// four partial sums are added in warp order. sol: the compact solution
__global__ void __launch_bounds__(128)
backsub_panels_kernel(NormalBuffers N, const double* __restrict__ sol, double* __restrict__ step_full, int nblk)
{
    __shared__ double s_part[4][6];
    const int grp = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int nelim = grp < N.Nframe_groups ? 6 : 3;
    const double* Yg = N.Ypan + (size_t)grp * N.nblk_max * kYpanel;
    const unsigned* mask = N.grp_blkmask + (size_t)grp * N.bwords;
    double tsum[6] = {0., 0., 0., 0., 0., 0.};
    int seen = 0;   // present blocks so far: the k-th present block goes to warp k mod 4 (an even share whatever the pattern)
    for(int b = 0; b < nblk; b++)
    {
        if(!((mask[b >> 5] >> (b & 31)) & 1u)) continue;
        if(((seen++) & 3) != warp) continue;
        const double d0 = sol[TB * b + lane], d1 = sol[TB * b + 32 + lane];
#pragma unroll
        for(int p = 0; p < 6; p++)
            tsum[p] += Yg[(size_t)b * kYpanel + p * kYld + lane] * d0 + Yg[(size_t)b * kYpanel + p * kYld + 32 + lane] * d1;
    }
    warp_sum(tsum);
    if(lane == 0)
#pragma unroll
        for(int p = 0; p < 6; p++) s_part[warp][p] = tsum[p];
    __syncthreads();
    if(threadIdx.x < nelim)
    {
        const int l = threadIdx.x;
        double v = 0.;
        for(int p = l; p < 6; p++)
            v += N.grp_Linv[(size_t)grp * 36 + p * 6 + l] * (N.grp_h[(size_t)grp * 6 + p] + (((s_part[0][p] + s_part[1][p]) + s_part[2][p]) + s_part[3][p]));
        step_full[N.e0 + group_col0(N, grp) + l] = -v;
    }
}

static int env_int(const char* name, int dflt)
{
    const char* v = getenv(name);
    const int x = v ? atoi(v) : 0;
    return x > 0 ? x : dflt;
}

// groups -> tiles -> [cross-rank sum of the lower-triangle tiles] -> regularization -> triangulated points -> g', J'x.
// Expects cleared: the presence bitmaps of the groups and the tiles' arrival counters (normal_finish())
bool normal_schur_sum(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                      double lambda, cudaStream_t s, int* nlaunch)
{
    if(!set_max_dynamic_smem<schur_tiles_kernel>((int)kTileSmem)) return false;
    const int nblk = N.ldS / TB;
    const int ntiles = nblk * (nblk + 1) / 2;
    if(N.Ngroups > 0)
    {
        groups_panels_kernel<<<N.Ngroups, 256, (size_t)N.bwords * sizeof(unsigned), s>>>(N, lambda, N.n_c, nblk);
        (*nlaunch)++;
    }
    const bool sharded = comm_active();
    if(sharded && N.S_packed == nullptr) { set_error("internal error: sharded solve without the packed tile buffer"); return false; }
    // part_arrive: [ntiles] arrival counters | the plan | the CTA list (+ its length)
    const int ntiles_max = N.nblk_max * (N.nblk_max + 1) / 2;
    int* plan = N.part_arrive + ntiles_max;
    int* cta = plan + (size_t)kPlanInts * ntiles_max;
    static const int ns_per_item = env_int("MRCAL_B200_TILE_NS_PER_ITEM", 1000), ns_per_group = env_int("MRCAL_B200_TILE_NS_PER_GROUP", 270),
                     ns_per_part = env_int("MRCAL_B200_TILE_NS_PER_PART", 40000);
    tile_plan_kernel<<<(ntiles * 32 + 255) / 256, 256, 0, s>>>(N, nblk, ns_per_item, ns_per_group, ns_per_part, N.part_scratch != nullptr, plan);
    tile_slots_kernel<<<1, 1024, 0, s>>>(ntiles, plan, cta);
    schur_tiles_kernel<<<kernel_ctas(ntiles), 256, kTileSmem, s>>>(N, lambda, N.n_c, nblk, true, sharded ? N.S_packed : nullptr,
                                                                 N.part_scratch, N.part_arrive, plan, cta);
    (*nlaunch) += 3;
    if(sharded)
    {
        // THE collective of the algorithm: the reduced normal equations -- lower-triangle tiles only, with g' and the
        // gradient as rows n_c, n_c+1 of the same tiles -- summed over the frame shards
        double* extras = N.S_packed + (size_t)ntiles * TB * TB;
        pack_extras_kernel<<<1, 32, 0, s>>>(N, extras);
        if(!comm_allreduce_sum(N.S_packed, (size_t)ntiles * TB * TB + kPackedExtras, s)) return false;
        unpack_extras_kernel<<<1, 32, 0, s>>>(N, extras);
        unpack_tiles_kernel<<<ntiles, 256, 0, s>>>(N, N.S_packed, lambda, N.n_c, nblk);
        (*nlaunch) += 3;
    }
    const int Nreg_blocks = reg_block_count(dp, N.splined);
    if(Nreg_blocks > 0)
    {
        reg_blocks_kernel<<<(Nreg_blocks + 127) / 128, 128, 0, s>>>(dp, N, N.n_c, op.x, op.Jval, op.Jcol, sharded);
        (*nlaunch)++;
    }
    if(dp.Ntri > 0 && dp.opt_extr)
    {
        const int nx = 6 * dp.Ncam_e;
        tri_rows_kernel<<<nx * (nx + 1) / 2 + nx, 256, 0, s>>>(dp, N, N.n_c, op.x, op.Jval, op.Jcol, d_rowptr);
        (*nlaunch)++;
    }
    if(N.n_c > 0)
    {
        finish_rhs_kernel<<<(N.n_c + 255) / 256, 256, 0, s>>>(N, N.n_c);
        (*nlaunch)++;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// what the buffers of the tiles need for a system of up to nblk_max 64-column blocks
NormalSchurSizes normal_schur_sizes(int nblk_max)
{
    const int nt = nblk_max * (nblk_max + 1) / 2;
    NormalSchurSizes z;
    z.part_scratch_doubles = (size_t)kernel_ctas(nt) * TB * TB;   // the partial tiles of the split tiles
    z.part_arrive_ints = nt + kPlanInts * nt + kernel_ctas(nt) + 1;   // arrival counters, the plan, the CTA list and its length
    z.packed_doubles = (size_t)nt * TB * TB + kPackedExtras;
    return z;
}

bool normal_schur_backsub(const NormalBuffers& N, const double* sol_compact, double* step_full, cudaStream_t s, int* nlaunch)
{
    if(N.Ngroups == 0) return true;
    backsub_panels_kernel<<<N.Ngroups, 128, 0, s>>>(N, sol_compact, step_full, N.ldS / TB);
    (*nlaunch)++;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace mb200
