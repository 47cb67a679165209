// Kernel family 2a: the normal equations. From the Jacobian strips written by
// eval.cu, form JtJ in its block-diagonal + arrowhead structure, eliminate the
// per-frame (6x6) and per-point (3x3) blocks (Schur complement), and leave the
// small dense reduced system S, g' of the shared unknowns (all intrinsics, all
// extrinsics, the board warp) for chol.cu:
//
//     [ A  B ] [ds]     [gs]        S  = A  - sum_j B_j D_j^-1 B_j'
//     [ B' D ] [df] = - [gf]        g' = gs - sum_j B_j D_j^-1 gf_j
//                                   df_j = -D_j^-1 (gf_j + B_j' ds)
//
// This replaces what the reference gets from libdogleg/CHOLMOD (Jt*x, the
// symbolic+numeric factorization of the whole sparse JtJ; call site
// mrcal.c:6435). The unit of work is the OBSERVATION: one CTA per board
// observation (or point observation) builds the Gram matrix of that
// observation's rows over the few columns they touch, in shared memory, and
// only the reduced result goes to global memory. For splined models the touched
// knot columns are data-dependent (mrcal.c:2171-2185), so each CTA discovers
// its own local column set every time.
#include "normal_items.cuh"
#include "chol.h"

namespace mb200 {

bool comm_active();
bool comm_allreduce_sum(double* d_buf, size_t count, cudaStream_t s);
bool comm_allreduce_max_int(int* d_buf, size_t count, cudaStream_t s);

// COMPACTION. Only the shared unknowns that some observation row touches are coupled to anything.
// For the wide splined models most knots are never hit by a board corner and appear only in their
// own 2x2 regularization block (at BASELINE config 3: 1266 of 4820 shared unknowns are coupled), so
// each assembly first marks the touched ("active") shared unknowns, numbers them compactly, and S is
// built and factored over those alone; the untouched ones are solved from their regularization rows
// directly (inactive_step_kernel). The reference gets the same saving from CHOLMOD's sparse
// factorization.
// Pass 1, one CTA per work item: which shared columns does the item touch? Writes the item's column
// list (reduced numbering, increasing) and marks those unknowns active.
__global__ void __launch_bounds__(256)
item_columns_kernel(DevProblem P, NormalBuffers N, const int* __restrict__ Jcol, int w0)
{
    extern __shared__ __align__(16) double dsm[];
    __shared__ int s_scan[256];
    const int w = blockIdx.x + w0, tid = threadIdx.x;
    const ItemDesc d = describe_item(P, w, N.Nframe_groups);
    const int ncam = d.cam0 >= 0 ? 6 : 0, nwarp = d.warp0 >= 0 ? 2 : 0;
    short* lmap = reinterpret_cast<short*>(dsm);   // [clen]
    for(int i = tid; i < d.clen; i += 256) lmap[i] = 0;
    __syncthreads();
    if(d.nI > 0)
        for(int e = tid; e < d.rows * d.nI; e += 256)
        {
            const int r = e / d.nI, k = e - r * d.nI;
            const int c = Jcol[(size_t)d.j0 + (size_t)r * d.nnz_row + k] - d.cbase;
            lmap[c] = 1;
            // the two surfaces of a spline knot stay together: their regularization rows couple them
            if(N.splined && c >= P.Ncore_state) lmap[P.Ncore_state + ((c - P.Ncore_state) ^ 1)] = 1;
        }
    __syncthreads();
    // exclusive scan over clen flags, 256 threads each owning a contiguous chunk
    const int per = (d.clen + 255) / 256;
    const int lo = tid * per, hi = min(lo + per, d.clen);
    int cnt = 0;
    for(int i = lo; i < hi; i++) cnt += lmap[i];
    s_scan[tid] = cnt;
    __syncthreads();
    for(int o = 1; o < 256; o <<= 1)
    {
        const int v = tid >= o ? s_scan[tid - o] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    int base = s_scan[tid] - cnt;
    int* cols = N.wi_cols + (size_t)w * N.cap;
    for(int i = lo; i < hi; i++)
        if(lmap[i])
        {
            const int r = N.reduced_index(d.cbase + i);
            cols[base++] = r;
            N.active[r] = 1;
        }
    const int nloc = s_scan[255];
    if(tid < ncam)  { const int r = N.reduced_index(d.cam0 + tid);  cols[nloc + tid] = r;        N.active[r] = 1; }
    if(tid < nwarp) { const int r = N.reduced_index(d.warp0 + tid); cols[nloc + ncam + tid] = r; N.active[r] = 1; }
    if(tid == 0)
    {
        const int nsh = nloc + ncam + nwarp;
        N.wi_nsh[w] = nsh;
        atomicMax(&N.stat[1], nsh + d.nelim);
    }
}

// unknowns named by a regularization row that is not a per-unknown (or per-knot) block must be in the
// coupled system: today that is the unity_cam01 row (3 columns)
__global__ void mark_reg_active_kernel(DevProblem P, NormalBuffers N)
{
    if(P.reg_unity && threadIdx.x < 3) N.active[N.reduced_index(P.i_extr0 + 3 + threadIdx.x)] = 1;
}

// ... and so must the extrinsics of every camera that observes a triangulated point
__global__ void mark_tri_active_kernel(DevProblem P, NormalBuffers N)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= 2 * P.Ntri) return;
    const int e = P.tri_cam_e[P.tri_pairs[i]];
    if(e >= 0)
        for(int k = 0; k < 6; k++) N.active[N.reduced_index(P.i_extr0 + 6 * e + k)] = 1;
}

// compact numbering of the active shared unknowns: one CTA
__global__ void __launch_bounds__(1024)
compact_scan_kernel(NormalBuffers N)
{
    __shared__ int s_scan[1024];
    const int tid = threadIdx.x;
    const int per = (N.n_r + 1023) / 1024;
    const int lo = tid * per, hi = min(lo + per, N.n_r);
    int cnt = 0;
    for(int i = lo; i < hi; i++) cnt += N.active[i] ? 1 : 0;
    s_scan[tid] = cnt;
    __syncthreads();
    for(int o = 1; o < 1024; o <<= 1)
    {
        const int v = tid >= o ? s_scan[tid - o] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    int base = s_scan[tid] - cnt;
    for(int i = lo; i < hi; i++)
    {
        if(N.active[i]) { N.cidx[i] = base; N.cinv[base] = i; base++; }
        else            N.cidx[i] = -1;
    }
    if(tid == 1023) N.stat[0] = s_scan[1023];
}

// Pass 2, one CTA per work item: the Gram matrix of the item's rows over its local columns. The tensor-pipe kernel below
// takes the items up to kDmmaMaxCols local columns; this one the wider ones (splined observations that touch many knots).
// Like that kernel, it leaves the shared x shared block and -J'x in the item's own block of the pool and B, D, gf in the
// item's slots; normal_det.cu sums the blocks into S in a fixed order
__global__ void __launch_bounds__(256, 1)
assemble_items_kernel(DevProblem P, NormalBuffers N, int gram_cap, const double* __restrict__ x,
                      const double* __restrict__ Jval, const int* __restrict__ Jcol, int w0)
{
    extern __shared__ __align__(16) double dsm[];
    __shared__ short s_lidx[2][RCH][kMaxRowNnz];
    __shared__ double s_val[2][RCH][kMaxRowNnz];
    __shared__ double s_xr[2][RCH];
    __shared__ unsigned char s_pa[kMaxRowNnz * (kMaxRowNnz + 1) / 2], s_pb[kMaxRowNnz * (kMaxRowNnz + 1) / 2];

    const int w = blockIdx.x + w0, tid = threadIdx.x;
    const ItemDesc d = describe_item(P, w, N.Nframe_groups);
    const int ncam = d.cam0 >= 0 ? 6 : 0, nwarp = d.warp0 >= 0 ? 2 : 0;
    const int nsh = N.wi_nsh[w], nloc = nsh - ncam - nwarp, ntot = nsh + d.nelim;
    // Gram matrix does not fit: shared x shared is summed in the item's block of the pool, which only this CTA touches
    const bool big = ntot > gram_cap;
    double* Aw = N.wi_A + N.wi_Aoff[w];
    const int lda = N.wi_lda[w];

    // shared-memory carve-up: lmap [clen] shorts | gram | gvec [ntot]
    short* lmap = reinterpret_cast<short*>(dsm);
    const int lmap_doubles = (d.clen * (int)sizeof(short) + 7) / 8;
    double* gram = dsm + lmap_doubles;
    const int ngram = big ? d.nelim * ntot : ntot * (ntot + 1) / 2;
    double* gvec = gram + ngram;   // [ntot] J'x of this item

    const int* cols = N.wi_cols + (size_t)w * N.cap;
    for(int i = tid; i < d.clen; i += 256) lmap[i] = -1;
    for(int e = tid; e < kMaxRowNnz * (kMaxRowNnz + 1) / 2; e += 256)
    {
        // decode pair index e -> (a >= b)
        int a = (int)((sqrtf(8.f * e + 1.f) - 1.f) * 0.5f);
        while(a * (a + 1) / 2 > e) a--;
        while((a + 1) * (a + 2) / 2 <= e) a++;
        s_pa[e] = (unsigned char)a;
        s_pb[e] = (unsigned char)(e - a * (a + 1) / 2);
    }
    for(int i = tid; i < ngram + ntot; i += 256) gram[i] = 0.;
    if(big) for(int i = tid; i < nsh * lda; i += 256) Aw[i] = 0.;
    __syncthreads();
    // intrinsics columns sit before the eliminated range: reduced == state index
    for(int l = tid; l < nloc; l += 256) lmap[cols[l] - d.cbase] = (short)l;
    __syncthreads();

    // Rows are consumed in chunks of RCH: while one chunk is being accumulated, the (column, value)
    // pairs of the next are already in flight from global memory into registers, so the per-row
    // critical path has no global-memory latency in it
    const int npairs = d.nnz_row * (d.nnz_row + 1) / 2;
    const int per_chunk = RCH * d.nnz_row;
    const int nchunks = (d.rows + RCH - 1) / RCH;
    int    pf_col[3];
    double pf_val[3];
    auto prefetch = [&](int chunk)
    {
#pragma unroll
        for(int q = 0; q < 3; q++)
        {
            const int e = tid + q * 256;
            const int rr = e / d.nnz_row, k = e - rr * d.nnz_row;
            const int r = chunk * RCH + rr;
            pf_col[q] = 0; pf_val[q] = 0.;
            if(e < per_chunk && r < d.rows)
            {
                const size_t j = (size_t)d.j0 + (size_t)r * d.nnz_row + k;
                if(k < d.nI) pf_col[q] = Jcol[j];
                pf_val[q] = Jval[j];
            }
        }
    };
    auto commit = [&](int chunk, int buf)
    {
#pragma unroll
        for(int q = 0; q < 3; q++)
        {
            const int e = tid + q * 256;
            if(e >= per_chunk) continue;
            const int rr = e / d.nnz_row, k = e - rr * d.nnz_row;
            int l;
            if(k < d.nI)                          l = chunk * RCH + rr < d.rows ? lmap[pf_col[q] - d.cbase] : 0;
            else if(k < d.nI + ncam)              l = nloc + (k - d.nI);
            else if(k < d.nI + ncam + d.nelim)    l = nsh + (k - d.nI - ncam);
            else                                  l = nloc + ncam + (k - d.nI - ncam - d.nelim);
            s_lidx[buf][rr][k] = (short)l;
            s_val[buf][rr][k] = pf_val[q];
        }
        if(tid < RCH) s_xr[buf][tid] = chunk * RCH + tid < d.rows ? x[d.m0 + chunk * RCH + tid] : 0.;
    };
    prefetch(0);
    for(int c = 0; c < nchunks; c++)
    {
        const int buf = c & 1;
        commit(c, buf);
        __syncthreads();
        if(c + 1 < nchunks) prefetch(c + 1);
        const int nrows_here = min(RCH, d.rows - c * RCH);
        for(int rr = 0; rr < nrows_here; rr++)
        {
            const short*  lidx = s_lidx[buf][rr];
            const double* val  = s_val[buf][rr];
            for(int e = tid; e < npairs; e += 256)
            {
                const int a = s_pa[e], b = s_pb[e];
                const double v = val[a] * val[b];
                if(v == 0.) continue;
                int la = lidx[a], lb = lidx[b];
                if(la < lb) { const int t = la; la = lb; lb = t; }
                if(!big) gram[tri(la, lb)] += v;
                else if(la >= nsh) gram[(la - nsh) * ntot + lb] += v;            // eliminated x anything
                else Aw[(size_t)la * lda + lb] += v;                              // shared x shared
            }
            if(tid >= 224 && tid < 224 + d.nnz_row) gvec[lidx[tid - 224]] += val[tid - 224] * s_xr[buf][rr];
            // two different rows can hit the same Gram entry from different threads: one barrier per row.
            // (Within a row, distinct (a,b) hit distinct entries.)
            __syncthreads();
        }
    }

    // ---- write out
    // shared x shared -> the item's block (every entry of the lower triangle, zeros included)
    if(!big)
        for(int e = tid; e < nsh * (nsh + 1) / 2; e += 256)
        {
            int a = (int)((sqrt(8. * e + 1.) - 1.) * 0.5);
            while(a * (a + 1) / 2 > e) a--;
            while((a + 1) * (a + 2) / 2 <= e) a++;
            Aw[(size_t)a * lda + (e - a * (a + 1) / 2)] = gram[e];
        }
    // rows nsh and nsh+1 of the block: -J'x over the shared columns, as the tensor-pipe kernel leaves them
    for(int l = tid; l < nsh; l += 256)
    {
        Aw[(size_t)nsh * lda + l] = -gvec[l];
        Aw[(size_t)(nsh + 1) * lda + l] = -gvec[l];
    }
    // eliminated block of this item: B (nelim x nsh), D (nelim x nelim), gf (nelim)
    if(d.nelim > 0)
    {
        double* B = N.wi_B + (size_t)w * 6 * N.cap;
        for(int e = tid; e < d.nelim * nsh; e += 256)
        {
            const int p = e / nsh, l = e - p * nsh;
            B[(size_t)p * N.cap + l] = big ? gram[p * ntot + l] : gram[tri(nsh + p, l)];
        }
        if(tid < 36)
        {
            const int p = tid / 6, q = tid % 6;
            double v = 0.;
            if(p < d.nelim && q < d.nelim)
            {
                const int hi = p > q ? p : q, lo = p > q ? q : p;
                v = big ? gram[hi * ntot + nsh + lo] : gram[tri(nsh + hi, nsh + lo)];
            }
            N.wi_D[(size_t)w * 36 + tid] = v;
        }
        if(tid < 6) N.wi_gf[(size_t)w * 6 + tid] = tid < d.nelim ? gvec[nsh + tid] : 0.;
    }
}

// Pass 2 on the fp64 tensor pipe. The Gram matrix of one observation is a dense contraction:
//   G = D' D,   D = [ rows of the item over its ntot local columns | x ]   (200 x ~75, ~40 % dense)
// so it goes through DMMA.8x8x4. D is built 32 rows at a time in shared memory (scatter of the
// 30 nonzeros of each row), every warp owns a fixed set of 8x8 tiles of the lower triangle of G
// and keeps them in registers for the whole item; the x column makes J'x the last row of G.
// 3 barriers per 32 rows instead of one per row, ~10x fewer shared-memory transactions than
// the scalar kernel above (which takes the items with more than kDmmaMaxCols local columns).
constexpr int kDmmaMaxCols = 160;                       // ntot + 1, padded to 8
constexpr int DCH = 32;                                 // rows per chunk
// Three instantiations by item width, so that the common narrow items do not pay the register
// footprint (hence the occupancy) of the widest: tiles per warp for T = ncols/8 <= 10, 16, 20
constexpr int kDmmaClassT[3]     = {10, 16, 20};
constexpr int kDmmaClassTiles[3] = {7, 17, 27};


template <int kDmmaMaxTiles, int TMIN, int TMAX>
__global__ void __launch_bounds__(256)
assemble_items_dmma_kernel(DevProblem P, NormalBuffers N, int ldD, const double* __restrict__ x,
                           const double* __restrict__ Jval, const int* __restrict__ Jcol, int w0)
{
    extern __shared__ __align__(16) double dsm[];
    __shared__ unsigned char s_ti[kDmmaMaxTiles * 8], s_tj[kDmmaMaxTiles * 8];
    {
        // this instantiation handles the items whose tile count T is in (TMIN, TMAX]
        const int T_ = (N.wi_nsh[blockIdx.x + w0] + describe_item(P, blockIdx.x + w0, N.Nframe_groups).nelim + 1 + 7) >> 3;
        if(T_ <= TMIN || T_ > TMAX) return;
    }

    const int w = blockIdx.x + w0, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, t = lane & 3;
    const ItemDesc d = describe_item(P, w, N.Nframe_groups);
    const int ncam = d.cam0 >= 0 ? 6 : 0, nwarp = d.warp0 >= 0 ? 2 : 0;
    const int nsh = N.wi_nsh[w], nloc = nsh - ncam - nwarp, ntot = nsh + d.nelim;
    const int ncols = ntot + 1;                         // + the x column
    const int T = (ncols + 7) >> 3, ntiles = T * (T + 1) / 2;

    // shared-memory carve-up: lmap [clen] shorts | D [DCH][ldD]
    short* lmap = reinterpret_cast<short*>(dsm);
    const int lmap_doubles = (d.clen * (int)sizeof(short) + 7) / 8;
    double* D = dsm + lmap_doubles;

    const int* cols = N.wi_cols + (size_t)w * N.cap;
    for(int i = tid; i < d.clen; i += 256) lmap[i] = -1;
    for(int i = tid; i < DCH * ldD; i += 256) D[i] = 0.;
    for(int q = tid; q < ntiles; q += 256)
    {
        // tile q -> (ti >= tj); warp q%8 owns it as its (q/8)-th tile
        int ti = (int)((sqrtf(8.f * q + 1.f) - 1.f) * 0.5f);
        while(ti * (ti + 1) / 2 > q) ti--;
        while((ti + 1) * (ti + 2) / 2 <= q) ti++;
        s_ti[q] = (unsigned char)ti;
        s_tj[q] = (unsigned char)(q - ti * (ti + 1) / 2);
    }
    __syncthreads();
    for(int l = tid; l < nloc; l += 256) lmap[cols[l] - d.cbase] = (short)l;
    __syncthreads();

    double acc[kDmmaMaxTiles][2];
#pragma unroll
    for(int i = 0; i < kDmmaMaxTiles; i++) acc[i][0] = acc[i][1] = 0.;
    const int my_ntiles = (ntiles - warp + 7) / 8;      // tiles warp, warp+8, ...

    const int per_chunk = DCH * d.nnz_row;
    const int nchunks = (d.rows + DCH - 1) / DCH;
    int    pf_col[4];
    double pf_val[4];
    double pf_x = 0.;
    // entry q of this thread is entry (rr, k) of every chunk: the index arithmetic is loop invariant
    int my_rr[4], my_k[4], my_l[4];
#pragma unroll
    for(int q = 0; q < 4; q++)
    {
        const int e = tid + q * 256;
        my_rr[q] = e < per_chunk ? e / d.nnz_row : -1;
        my_k[q] = e < per_chunk ? e - my_rr[q] * d.nnz_row : 0;
        const int k = my_k[q];
        if(k < d.nI)                          my_l[q] = -1;                                   // per-row lookup
        else if(k < d.nI + ncam)              my_l[q] = nloc + (k - d.nI);
        else if(k < d.nI + ncam + d.nelim)    my_l[q] = nsh + (k - d.nI - ncam);
        else                                  my_l[q] = nloc + ncam + (k - d.nI - ncam - d.nelim);
    }
    auto prefetch = [&](int chunk)
    {
#pragma unroll
        for(int q = 0; q < 4; q++)
        {
            const int r = chunk * DCH + my_rr[q];
            pf_col[q] = 0; pf_val[q] = 0.;
            if(my_rr[q] >= 0 && r < d.rows)
            {
                const size_t j = (size_t)d.j0 + (size_t)r * d.nnz_row + my_k[q];
                if(my_k[q] < d.nI) pf_col[q] = Jcol[j];
                pf_val[q] = Jval[j];
            }
        }
        if(tid < DCH) pf_x = chunk * DCH + tid < d.rows ? x[d.m0 + chunk * DCH + tid] : 0.;
    };
    // where entry q of this thread lands in D (or -1)
    auto slot = [&](int chunk, int q) -> int
    {
        if(my_rr[q] < 0 || chunk * DCH + my_rr[q] >= d.rows) return -1;
        const int l = my_l[q] >= 0 ? my_l[q] : (int)lmap[pf_col[q] - d.cbase];
        return my_rr[q] * ldD + l;
    };
    prefetch(0);
    for(int c = 0; c < nchunks; c++)
    {
        int where[4];
#pragma unroll
        for(int q = 0; q < 4; q++)
        {
            where[q] = slot(c, q);
            if(where[q] >= 0) D[where[q]] = pf_val[q];
        }
        if(tid < DCH) D[tid * ldD + ntot] = pf_x;
        __syncthreads();
        if(c + 1 < nchunks) prefetch(c + 1);
        // tiles in groups of 4: the operand pointers are formed once per tile, and the 4 accumulator
        // chains are independent, so the DMMAs of a group issue back to back
#pragma unroll
        for(int i0 = 0; i0 < kDmmaMaxTiles; i0 += 4)
        {
            if(i0 >= my_ntiles) continue;   // warp-uniform
            const double* Da[4];
            const double* Db[4];
#pragma unroll
            for(int u = 0; u < 4; u++)
            {
                // past the warp's last tile: aim at tile 0 (harmless work into an accumulator that is never read)
                const int q = (i0 + u < my_ntiles && i0 + u < kDmmaMaxTiles) ? warp + 8 * (i0 + u) : 0;
                Da[u] = D + 8 * s_ti[q] + g + t * ldD;     // A operand: element (row g of the tile, k = t) = D[k][8 ti + g]
                Db[u] = D + 8 * s_tj[q] + g + t * ldD;     // B operand: element (k = t, col g)            = D[k][8 tj + g]
            }
#pragma unroll
            for(int ks = 0; ks < DCH / 4; ks++)
#pragma unroll
                for(int u = 0; u < 4; u++)
                    if(i0 + u < kDmmaMaxTiles)
                        dmma884(acc[i0 + u][0], acc[i0 + u][1], Da[u][ks * 4 * ldD], Db[u][ks * 4 * ldD]);
        }
        __syncthreads();
        // un-scatter: cheaper than clearing the whole chunk
#pragma unroll
        for(int q = 0; q < 4; q++) if(where[q] >= 0) D[where[q]] = 0.;
        if(tid < DCH) D[tid * ldD + ntot] = 0.;
        // (the next chunk's scatter touches other or the same entries of D only after the barrier below,
        //  which is the one at the top of the next iteration's MMA; a thread zeroes only what it wrote)
        __syncthreads();
    }

    // ---- write out from the accumulators. Lane holds G[8 ti + g][8 tj + 2t + {0,1}]
    double* B = N.wi_B + (size_t)w * 6 * N.cap;
    // the shared x shared block and the gradient go to this item's own block of the pool (every entry of the lower
    // triangle exactly once, zeros included); normal_det.cu sums the blocks into S in a fixed order
    double* Aw = N.wi_A + N.wi_Aoff[w];
    const int lda = N.wi_lda[w];
#pragma unroll
    for(int i = 0; i < kDmmaMaxTiles; i++)
    {
        if(i >= my_ntiles) continue;
        const int q = warp + 8 * i;
        const int row = 8 * s_ti[q] + g;
#pragma unroll
        for(int h = 0; h < 2; h++)
        {
            const int col = 8 * s_tj[q] + 2 * t + h;
            const double v = acc[i][h];
            // lower triangle (incl. diagonal) of the (ntot+1)^2 Gram matrix; the (x,x) corner is |x|^2: unused
            if(row > ntot || col > row || col >= ntot) continue;
            if(row < nsh) Aw[(size_t)row * lda + col] = v;                                      // shared x shared
            else if(row < ntot)
            {
                const int p = row - nsh;
                if(col < nsh) B[(size_t)p * N.cap + col] = v;                                  // eliminated x shared
                else
                {
                    const int qq = col - nsh;                                                   // eliminated x eliminated
                    N.wi_D[(size_t)w * 36 + p * 6 + qq] = v;
                    N.wi_D[(size_t)w * 36 + qq * 6 + p] = v;
                }
            }
            else   // row == ntot: the x row = J'x
            {
                if(col < nsh)
                {
                    // rows nsh and nsh+1 of the block: -J'x (the right-hand side rides through the factorization as
                    // row n_c of S; row n_c+1 collects the plain gradient)
                    Aw[(size_t)nsh * lda + col] = -v;
                    Aw[(size_t)(nsh + 1) * lda + col] = -v;
                }
                else N.wi_gf[(size_t)w * 6 + (col - nsh)] = v;
            }
        }
    }
    // unused corners of the 6x6 / 6-vector for 3-unknown (point) groups and for no elimination at all
    if(d.nelim > 0 && d.nelim < 6)
    {
        if(tid < 36) { const int p = tid / 6, qq = tid % 6; if(p >= d.nelim || qq >= d.nelim) N.wi_D[(size_t)w * 36 + tid] = 0.; }
        if(tid >= 64 && tid < 70 && tid - 64 >= d.nelim) N.wi_gf[(size_t)w * 6 + tid - 64] = 0.;
    }
}

// Gauss-Newton step of the INACTIVE shared unknowns: each is coupled only to its regularization
// block (a spline knot's two surfaces: 2x2; anything else: 1x1), solved here in closed form.
// One thread per shared unknown
__global__ void inactive_step_kernel(DevProblem P, NormalBuffers N, double lambda, const double* __restrict__ x,
                                     const double* __restrict__ Jval, double* __restrict__ step_full)
{
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if(r >= N.n_r || N.cidx[r] >= 0) return;
    const int c = N.state_index(r);
    double step = 0.;
    const int n_intr = P.Ncam_i * P.Nintr_state;
    if(P.reg && c < n_intr)
    {
        const int cam = c / P.Nintr_state, k = c - cam * P.Nintr_state;
        const int Ndist_rows = P.opt_dist ? P.Ncam_i * (P.Nintr - 4) : 0;
        if(k >= P.Ncore_state)
        {
            const int j = k - P.Ncore_state;
            if(N.splined)
            {
                // rows (radial, tangential) of this knot; entries [d/dx, d/dy] each (eval.cu)
                const int knot = j >> 1, which = j & 1;
                const int t0 = cam * (P.Nintr - 4) + 2 * knot;
                const double* e0 = &Jval[(size_t)P.reg_j0 + 2 * (size_t)t0];
                const double* e1 = e0 + 2;
                const double x0 = x[P.m_reg0 + t0], x1 = x[P.m_reg0 + t0 + 1];
                const double Hxx = e0[0] * e0[0] + e1[0] * e1[0] + lambda;
                const double Hyy = e0[1] * e0[1] + e1[1] * e1[1] + lambda;
                const double Hxy = e0[0] * e0[1] + e1[0] * e1[1];
                const double gx = e0[0] * x0 + e1[0] * x1, gy = e0[1] * x0 + e1[1] * x1;
                const double det = Hxx * Hyy - Hxy * Hxy;
                if(det > 0.) step = which == 0 ? -(Hyy * gx - Hxy * gy) / det : -(Hxx * gy - Hxy * gx) / det;
            }
            else
            {
                const int t = cam * (P.Nintr - 4) + j;
                const double e = Jval[(size_t)P.reg_j0 + t];
                const double H = e * e + lambda;
                if(H > 0.) step = -e * x[P.m_reg0 + t] / H;
            }
        }
        else if(k >= 2)
        {
            const int t = Ndist_rows + 2 * cam + (k - 2);
            const double e = Jval[(size_t)P.reg_j0 + (size_t)(N.splined ? 2 : 1) * Ndist_rows + 2 * cam + (k - 2)];
            const double H = e * e + lambda;
            if(H > 0.) step = -e * x[P.m_reg0 + t] / H;
        }
    }
    step_full[c] = step;
}

// One-time, per-device kernel attributes
static bool configure_kernels()
{
    static bool configured[kMaxDevices] = {};
    int dev = 0;
    MB200_CUDA_CHECK(cudaGetDevice(&dev));
    if(dev < 0 || dev >= kMaxDevices) { set_error("device index %d out of range", dev); return false; }
    if(configured[dev]) return true;
    MB200_CUDA_CHECK(cudaFuncSetAttribute(assemble_items_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    MB200_CUDA_CHECK(cudaFuncSetAttribute((assemble_items_dmma_kernel<kDmmaClassTiles[0], 0, kDmmaClassT[0]>), cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    MB200_CUDA_CHECK(cudaFuncSetAttribute((assemble_items_dmma_kernel<kDmmaClassTiles[1], kDmmaClassT[0], kDmmaClassT[1]>), cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    MB200_CUDA_CHECK(cudaFuncSetAttribute((assemble_items_dmma_kernel<kDmmaClassTiles[2], kDmmaClassT[1], kDmmaClassT[2]>), cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
    configured[dev] = true;
    return true;
}

static bool launch_gram_dmma(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, int Nwi, int max_ntot,
                             size_t lmap_bytes, cudaStream_t s, int* nlaunch, int w0)
{
    Nwi -= w0;
    if(Nwi <= 0) return true;
    // the tensor-pipe kernel: D chunk [32][ldD], ldD = 4 (mod 16) for conflict-free fragment loads
    const int ncols_pad = ((max_ntot + 1 + 7) / 8) * 8;
    const int Tmax = ncols_pad / 8;
    auto ld_for = [](int T) { int ld = 8 * T; while(ld % 16 != 4) ld++; return ld; };
    auto smem_for = [&](int T) { return lmap_bytes + (size_t)DCH * ld_for(T) * sizeof(double); };
    // The size classes touch disjoint items: they run side by side on forked streams (owned by the workspace),
    // so that the CTAs of one fill the tails of the other
    const bool c1 = Tmax > kDmmaClassT[0], c2 = Tmax > kDmmaClassT[1];
    if(c1 || c2)
    {
        MB200_CUDA_CHECK(cudaEventRecord(N.ev_fork, s));
        if(c1) MB200_CUDA_CHECK(cudaStreamWaitEvent(N.s_side[0], N.ev_fork, 0));
        if(c2) MB200_CUDA_CHECK(cudaStreamWaitEvent(N.s_side[1], N.ev_fork, 0));
    }
    {
        const int T0 = Tmax < kDmmaClassT[0] ? Tmax : kDmmaClassT[0];
        assemble_items_dmma_kernel<kDmmaClassTiles[0], 0, kDmmaClassT[0]><<<Nwi, 256, smem_for(T0), s>>>(dp, N, ld_for(T0), op.x, op.Jval, op.Jcol, w0);
        (*nlaunch)++;
    }
    if(c1)
    {
        const int T1 = Tmax < kDmmaClassT[1] ? Tmax : kDmmaClassT[1];
        assemble_items_dmma_kernel<kDmmaClassTiles[1], kDmmaClassT[0], kDmmaClassT[1]><<<Nwi, 256, smem_for(T1), N.s_side[0]>>>(dp, N, ld_for(T1), op.x, op.Jval, op.Jcol, w0);
        MB200_CUDA_CHECK(cudaEventRecord(N.ev_join[0], N.s_side[0]));
        MB200_CUDA_CHECK(cudaStreamWaitEvent(s, N.ev_join[0], 0));
        (*nlaunch)++;
    }
    if(c2)
    {
        assemble_items_dmma_kernel<kDmmaClassTiles[2], kDmmaClassT[1], kDmmaClassT[2]><<<Nwi, 256, smem_for(Tmax), N.s_side[1]>>>(dp, N, ld_for(Tmax), op.x, op.Jval, op.Jcol, w0);
        MB200_CUDA_CHECK(cudaEventRecord(N.ev_join[1], N.s_side[1]));
        MB200_CUDA_CHECK(cudaStreamWaitEvent(s, N.ev_join[1], 0));
        (*nlaunch)++;
    }
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// Pass 1 of the assembly: which shared unknowns do the rows at `op` touch; their compact numbering; where each
// item's block goes. Ends with an ASYNCHRONOUS copy of (n_c, widest item) to the host: the caller synchronises
// the stream when it suits it (the solver does so once per trust-region step, with everything else it reads)
// and then calls normal_adopt_sizes()
// rider: a device scalar that is a per-rank partial sum (the cost of this evaluation). Sharded solves sum it over the
// ranks in the SAME collective that unites the active sets: the marks travel as 0/1 doubles, the scalar behind them.
// *rider_summed says whether that happened
__global__ void marks_stage_kernel(const int* __restrict__ active, int n_r, const double* __restrict__ rider, double* __restrict__ stage)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i < n_r) stage[i] = active[i] != 0 ? 1. : 0.;
    else if(i == n_r) stage[i] = rider != nullptr ? *rider : 0.;
}
__global__ void marks_unstage_kernel(int* __restrict__ active, int n_r, double* __restrict__ rider, const double* __restrict__ stage)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i < n_r) active[i] = stage[i] > 0. ? 1 : 0;
    else if(i == n_r && rider != nullptr) *rider = stage[i];
}

bool normal_prepare(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, cudaStream_t s, int* nlaunch, bool boards_done,
                    double* rider, bool* rider_summed, bool copy_sizes)
{
    if(rider_summed) *rider_summed = false;
    if(!configure_kernels()) return false;
    const size_t lmap_bytes = ((size_t)dp.Nintr_state * sizeof(short) + 7) / 8 * 8;
    // (the scalar Gram kernel's shared memory for the widest item the model allows: its eliminated rows and J'x)
    if(lmap_bytes + (size_t)(7 * (N.cap + 6) + 2) * sizeof(double) > 200 * 1024)
    {
        set_error("lens model with %d intrinsics per camera is too large for the assembly kernels", dp.Nintr_state);
        return false;
    }
    const int Nwi = dp.Nobs_board + dp.Nobs_point;
    // boards_done: the fused evaluation (fused_eval.cu) has already listed the board observations' columns and marked
    // them, into buffers the caller cleared before it ran
    if(!boards_done && !normal_clear_marks(N, s)) return false;
    const int w0 = boards_done ? dp.Nobs_board : 0;
    if(Nwi - w0 > 0) { item_columns_kernel<<<Nwi - w0, 256, lmap_bytes, s>>>(dp, N, op.Jcol, w0); (*nlaunch)++; }
    if(dp.reg_unity) { mark_reg_active_kernel<<<1, 32, 0, s>>>(dp, N); (*nlaunch)++; }
    if(dp.Ntri > 0) { mark_tri_active_kernel<<<(2 * dp.Ntri + 127) / 128, 128, 0, s>>>(dp, N); (*nlaunch)++; }
    // sharded solve: every rank must number the union of the active sets identically
    if(comm_active() && N.n_r > 0)
    {
        if(N.S_packed != nullptr)
        {
            // (the packed-tile buffer is idle between assemblies)
            marks_stage_kernel<<<(N.n_r + 1 + 255) / 256, 256, 0, s>>>(N.active, N.n_r, rider, N.S_packed);
            if(!comm_allreduce_sum(N.S_packed, (size_t)N.n_r + 1, s)) return false;
            marks_unstage_kernel<<<(N.n_r + 1 + 255) / 256, 256, 0, s>>>(N.active, N.n_r, rider, N.S_packed);
            (*nlaunch) += 2;
            if(rider_summed) *rider_summed = rider != nullptr;
        }
        else if(!comm_allreduce_max_int(N.active, (size_t)N.n_r, s)) return false;
    }
    compact_scan_kernel<<<1, 1024, 0, s>>>(N);
    (*nlaunch)++;
    // (the fused evaluation placed the board observations' blocks at their fixed slots)
    if(!normal_det_item_offsets(dp, N, w0, s, nlaunch)) return false;
    if(copy_sizes) MB200_CUDA_CHECK(cudaMemcpyAsync(N.h_stat, N.stat, 4 * sizeof(int), cudaMemcpyDeviceToHost, s));
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

void normal_marks_to_clear(const NormalBuffers& N, WordFill* f)
{
    f->add(N.active, (size_t)(N.n_r > 0 ? N.n_r : 1) * sizeof(int));
    f->add(N.stat, 4 * sizeof(int));
}

bool normal_clear_marks(NormalBuffers& N, cudaStream_t s)
{
    WordFill f;
    normal_marks_to_clear(N, &f);
    return fill_words(f, s);
}

// After the stream was synchronised: take over what normal_prepare() found. If the items' blocks outgrew the pool (wide
// splined observations on the stored-Jacobian path), it grows here and the items are placed again before the assembly
bool normal_adopt_sizes(NormalBuffers& N, cudaStream_t s)
{
    N.n_c = N.h_stat[0];
    N.max_ntot = N.h_stat[1];
    // wi_ccol holds compact indices up to n_c + 1 in 16 bits
    if(N.n_c > 65533) { set_error("the reduced system has %d coupled unknowns: at most 65533 are supported", N.n_c); return false; }
    if(N.h_stat[2] != 0)
    {
        long long need = 0;
        MB200_CUDA_CHECK(cudaMemcpyAsync(&need, N.pool_need, sizeof(long long), cudaMemcpyDeviceToHost, s));
        MB200_CUDA_CHECK(cudaStreamSynchronize(s));
        // (schur_tiles_kernel addresses the pool with 32-bit element offsets)
        if(need >= (1ll << 32)) { set_error("the observations' normal-equation blocks need %lld doubles: at most 2^32 are supported", need); return false; }
        double* pool = nullptr;
        MB200_CUDA_CHECK(cudaMalloc(&pool, (size_t)need * sizeof(double)));
        // the fused evaluation's fixed slots at the front of the pool stay where they are
        if(N.fused && (cudaMemcpyAsync(pool, N.wi_A, (size_t)N.A_pool * sizeof(double), cudaMemcpyDeviceToDevice, s) != cudaSuccess ||
                       cudaStreamSynchronize(s) != cudaSuccess))
        {
            cudaFree(pool);
            set_error("growing the pool of the observations' blocks: %s", cudaGetErrorString(cudaGetLastError()));
            return false;
        }
        MB200_CUDA_CHECK(cudaFree(N.wi_A));
        N.wi_A = pool;
        N.A_pool = need;
        N.replace_items = true;
    }
    // padding rows: one carries the right-hand side through the factorization, the second the plain gradient
    N.ldS = chol_padded(N.n_c + 2);
    if(N.ldS > N.ldS_max) N.ldS = N.ldS_max;
    return true;
}

bool normal_assemble(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                     double lambda, cudaStream_t s, int* nlaunch)
{
    if(!normal_prepare(dp, N, op, s, nlaunch, false)) return false;
    MB200_CUDA_CHECK(cudaStreamSynchronize(s));
    return normal_adopt_sizes(N, s) && normal_finish(dp, N, op, d_rowptr, lambda, s, nlaunch, false);
}

// Pass 2: Gram matrices, Schur elimination, regularization, right-hand side: S, g', J'x
bool normal_finish(const DevProblem& dp, NormalBuffers& N, const EvalBuffers& op, const int* d_rowptr,
                   double lambda, cudaStream_t s, int* nlaunch, bool boards_done, double* also_clear, int also_clear_n)
{
    const size_t lmap_bytes = ((size_t)dp.Nintr_state * sizeof(short) + 7) / 8 * 8;
    const int Nwi = dp.Nobs_board + dp.Nobs_point;
    // (boards_done: the fused evaluation left the board observations' blocks; only the point observations remain)
    const int w0 = boards_done ? dp.Nobs_board : 0;
    const int max_ntot = N.max_ntot;
    if(N.replace_items)
    {
        if(!normal_det_item_offsets(dp, N, w0, s, nlaunch)) return false;
        N.replace_items = false;
    }
    // every accumulator and counter of the assembly (and the caller's scalars) zeroed in one launch
    WordFill clear;
    clear.add(N.g_full, (size_t)dp.Nstate * sizeof(double));
    clear.add(N.info, sizeof(int));
    if(also_clear) clear.add(also_clear, (size_t)also_clear_n * sizeof(double));
    normal_det_to_clear(N, &clear);
    if(!fill_words(clear, s)) return false;

    if(!normal_det_item_prepare(dp, N, s, nlaunch)) return false;
    if(((max_ntot + 1 + 7) / 8) * 8 <= kDmmaMaxCols)
    {
        if(!launch_gram_dmma(dp, N, op, Nwi, max_ntot, lmap_bytes, s, nlaunch, w0)) return false;
    }
    else if(Nwi > w0)
    {
        const int gram_cap = max_ntot < kGramMax ? max_ntot : kGramMax;
        size_t gram_doubles = (size_t)gram_cap * (gram_cap + 1) / 2 + gram_cap;
        if(max_ntot > kGramMax && (size_t)7 * max_ntot > gram_doubles) gram_doubles = (size_t)7 * max_ntot;
        assemble_items_kernel<<<Nwi - w0, 256, lmap_bytes + (gram_doubles + 2) * sizeof(double), s>>>(dp, N, gram_cap, op.x, op.Jval, op.Jcol, w0);
        (*nlaunch)++;
    }
    if(!normal_det_finish(dp, N, op, d_rowptr, lambda, s, nlaunch)) return false;
    if(!normal_det_rhs(N, s, nlaunch)) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// y (the forward-substituted right-hand side) out of row n_c of the factor; padding 0
__global__ void extract_y_kernel(NormalBuffers N, double* __restrict__ rhs)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c < N.ldS) rhs[c] = c < N.n_c ? N.S[(size_t)N.n_c * N.ldS + c] : 0.;
}
bool normal_extract_y(const NormalBuffers& N, double* rhs, cudaStream_t s, int* nlaunch)
{
    extract_y_kernel<<<(N.ldS + 255) / 256, 256, 0, s>>>(N, rhs);
    (*nlaunch)++;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

// compact solution -> the shared part of the full-length step
__global__ void scatter_compact_kernel(NormalBuffers N, const double* __restrict__ sol, double* __restrict__ step_full)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if(c >= N.n_c) return;
    const int r = N.cinv[c];
    step_full[N.state_index(r)] = sol[c];
}

// the full-length Gauss-Newton step from the compact solution `sol`
bool normal_expand_step(const DevProblem& dp, const NormalBuffers& N, const EvalBuffers& op, double lambda,
                        const double* sol, double* step_full, cudaStream_t s, int* nlaunch)
{
    if(N.n_c > 0) { scatter_compact_kernel<<<(N.n_c + 255) / 256, 256, 0, s>>>(N, sol, step_full); (*nlaunch)++; }
    if(N.n_r > N.n_c)
    {
        inactive_step_kernel<<<(N.n_r + 255) / 256, 256, 0, s>>>(dp, N, lambda, op.x, op.Jval, step_full);
        (*nlaunch)++;
    }
    if(!normal_det_backsub(N, sol, step_full, s, nlaunch)) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

}  // namespace mb200
