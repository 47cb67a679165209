// Template matching for many features in one call: the device half of match_feature() (reference: mrcal/stereo.py:
// 1609-2091, which calls cv2.remap(), cv2.matchTemplate() and np.linalg.lstsq() once per feature).
//
// The host decides everything that can fail before a launch (mrcal_b200/stereo.py): which features have a template
// inside both images and a search cut at least as large as the template. It passes only those, each as its template's
// top-left pixel in image 1, its clipped search cut and the float32 inverse of its homography. Then:
//   1. template_maps_kernel: every feature's map apply_homography(inv(H10), q1_grid) in float32, one (M*th, tw, 2) map,
//      and one call of the remap launcher (image_transforms.cu) with transform_image()'s defaults makes the templates;
//   2. template_sums_kernel: each template's sum and sum of squares, one thread per feature;
//   3. match_kernel: one CTA per feature (grid x) x tile of output rows (grid y), the six cv2.matchTemplate() methods from the window
//      sums. The template and the rows of the cut the tile reads are staged in shared memory when they fit; otherwise
//      the kernel reads both through L2;
//   4. match_optimum_kernel: one warp per feature, numpy's argmax/argmin, the edge test and the 3x3 quadratic fit.
//
// Exactness (DESIGN.md section 4.10): uint8 sums are exact integers; float32 products are exact in fp64 and summed in
// one fixed order, row-major over the template, by one thread. Every later step is a fixed fp64 expression with no
// contraction, rounded once to float32. So the output does not depend on the launch shape.
#include <cuda_runtime.h>
#include <cfloat>
#include <cmath>
#include <cstdint>

#include "common.h"
#include "device_call.h"
#include "problem.h"
#include "remap.h"

namespace mb200 {
namespace {

// OpenCV's TemplateMatchModes
enum { TM_SQDIFF = 0, TM_SQDIFF_NORMED = 1, TM_CCORR = 2, TM_CCORR_NORMED = 3, TM_CCOEFF = 4, TM_CCOEFF_NORMED = 5 };

// one feature, as the host passes it: the template's top-left pixel in image 1 and the search cut of image 1
struct MatchFeature
{
    int tx, ty;   // q1_template_min
    int cx, cy;   // q1_min, clipped to image 1
    int cw, ch;   // the cut's size, >= the template's
};

// one feature's result: the sub-pixel optimum in match-output coordinates, its value, and a status
struct MatchResult
{
    double at[2], value, status;
};

// a template's sums: exact integers for uint8, fp64 in row-major order for float32
struct TemplateSums
{
    long long s, s2;
    double fs, fs2;
};

constexpr int kThreads = 256;
// the most dynamic shared memory the staged path uses; a tile that needs more reads through L2
constexpr int kStagedBytes = 96 * 1024;
// the positions a CTA aims to cover, about two per thread
constexpr int kPositionsPerCta = 2 * kThreads;
// OpenCV's 10 * FLT_EPSILON, formed in float as its templmatch.cpp forms it
constexpr double kTenFltEps = (double)(10.f * FLT_EPSILON);

////////////////////////////////////////////////////////////////////////////////
// 1. the templates' maps
////////////////////////////////////////////////////////////////////////////////

// map[k] = apply_homography(Hinv_i, (tx + u, ty + v)) in float32, ((H00 x + H01 y) + H02) / ((H20 x + H21 y) + H22),
// rounded operation by operation: the reference's float32 body. Pixel k is (u, v) of feature i's (th, tw) template
__global__ void template_maps_kernel(const MatchFeature* __restrict__ f, const float* __restrict__ Hinv, int tw, int th,
                                     long Npix, float* __restrict__ map)
{
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= Npix) return;
    const int per = tw * th;
    const int i = (int)(k / per), r = (int)(k - (long)i * per);
    const int v = r / tw, u = r - v * tw;
    const float* H = Hinv + 9 * i;
    const float x = (float)(f[i].tx + u), y = (float)(f[i].ty + v);
    float xyz[3];
    for(int j = 0; j < 3; j++)
        xyz[j] = __fadd_rn(__fadd_rn(__fmul_rn(H[3 * j], x), __fmul_rn(H[3 * j + 1], y)), H[3 * j + 2]);
    map[2 * k] = __fdiv_rn(xyz[0], xyz[2]);
    map[2 * k + 1] = __fdiv_rn(xyz[1], xyz[2]);
}

////////////////////////////////////////////////////////////////////////////////
// 2. the templates' sums
////////////////////////////////////////////////////////////////////////////////

template <typename T>
__global__ void template_sums_kernel(const T* __restrict__ templ, int n, int M, TemplateSums* __restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if(i >= M) return;
    const T* t = templ + (size_t)i * n;
    TemplateSums r{0, 0, 0., 0.};
    for(int e = 0; e < n; e++)
    {
        if constexpr(std::is_same<T, uint8_t>::value)
        {
            r.s += t[e];
            r.s2 += (int)t[e] * (int)t[e];
        }
        else
        {
            const double x = (double)t[e];
            r.fs = __dadd_rn(r.fs, x);
            r.fs2 = __dadd_rn(r.fs2, __dmul_rn(x, x));
        }
    }
    out[i] = r;
}

////////////////////////////////////////////////////////////////////////////////
// 3. the match output
////////////////////////////////////////////////////////////////////////////////

// OpenCV's rule for the normalised methods (templmatch.cpp, common_matchTemplate()): t = sqrt(max(diff2, 0)) * tnorm,
// or 0 where the window's energy is within rounding of nothing; then num / t, or +-1 just above t, or 0 (1 for
// SQDIFF_NORMED) beyond. Comparisons are written so that NaN falls through as OpenCV's does
__device__ __forceinline__ double normed(double num, double diff2, double wsum2, double tnorm, bool sqdiff)
{
    diff2 = diff2 < 0. ? 0. : diff2;
    const double thr = fmin(0.5, __dmul_rn(kTenFltEps, wsum2));
    const double t = diff2 <= thr ? 0. : __dmul_rn(__dsqrt_rn(diff2), tnorm);
    const double a = fabs(num);
    if(a < t) return __ddiv_rn(num, t);
    if(a < __dmul_rn(t, 1.125)) return num > 0. ? 1. : -1.;
    return sqdiff ? 1. : 0.;
}

// The quantities every method is formed from, in fp64: sq the SQDIFF numerator, cc the cross-correlation, co the
// CCOEFF numerator (n STI - ST SI) / n, eT and eI the template's and the window's centred energies (n S2 - S^2) / n,
// and the plain energies ST2, SI2
struct MatchTerms
{
    double sq, cc, co, eT, eI, ST2, SI2;
};

__device__ __forceinline__ float match_value(int method, const MatchTerms& m, double nd)
{
    double r;
    switch(method)
    {
    case TM_SQDIFF: r = m.sq; break;
    case TM_SQDIFF_NORMED: r = normed(m.sq, m.SI2, m.SI2, __dsqrt_rn(m.ST2), true); break;
    case TM_CCORR: r = m.cc; break;
    case TM_CCORR_NORMED: r = normed(m.cc, m.SI2, m.SI2, __dsqrt_rn(m.ST2), false); break;
    case TM_CCOEFF: r = m.co; break;
    default:
        // a flat template (variance below DBL_EPSILON) matches everywhere with 1, as in OpenCV
        r = __ddiv_rn(m.eT, nd) < DBL_EPSILON ? 1. : normed(m.co, m.eI, m.SI2, __dsqrt_rn(m.eT), false);
    }
    return __double2float_rn(r);
}

// exact integers, one fp64 rounding each where they are converted; the products fit int64 for templates of up to 2^23
// pixels (the C entry refuses larger)
__device__ __forceinline__ MatchTerms terms_u8(long long n, long long ST, long long ST2, long long SI, long long SI2,
                                               long long STI)
{
    const double nd = (double)n;
    MatchTerms m;
    m.sq = (double)(SI2 - 2 * STI + ST2);
    m.cc = (double)STI;
    m.co = __ddiv_rn((double)(n * STI - ST * SI), nd);
    m.eT = __ddiv_rn((double)(n * ST2 - ST * ST), nd);
    m.eI = __ddiv_rn((double)(n * SI2 - SI * SI), nd);
    m.ST2 = (double)ST2;
    m.SI2 = (double)SI2;
    return m;
}

__device__ __forceinline__ MatchTerms terms_f32(double nd, double ST, double ST2, double SI, double SI2, double STI)
{
    MatchTerms m;
    const double sq = __dadd_rn(__dsub_rn(SI2, __dmul_rn(2., STI)), ST2);
    m.sq = sq < 0. ? 0. : sq;
    m.cc = STI;
    m.co = __ddiv_rn(__dsub_rn(__dmul_rn(nd, STI), __dmul_rn(ST, SI)), nd);
    m.eT = __ddiv_rn(__dsub_rn(__dmul_rn(nd, ST2), __dmul_rn(ST, ST)), nd);
    m.eI = __ddiv_rn(__dsub_rn(__dmul_rn(nd, SI2), __dmul_rn(SI, SI)), nd);
    m.ST2 = ST2;
    m.SI2 = SI2;
    return m;
}

// Output rows [y0, y0 + TR) of feature blockIdx.x (y0 = blockIdx.y TR), one thread per position in turn. The feature is
// on x, whose limit is 2^31 - 1, so a batch of any size is one launch; the row tiles (at most 32767) are on y. out: the feature's slot, its
// (oh, ow) output packed at its start. img1: image 1, rows stride1 elements apart. staged: the template and the cut's
// rows the tile reads go through shared memory first (the host checked they fit)
template <typename T>
__global__ void __launch_bounds__(kThreads) match_kernel(const T* __restrict__ img1, size_t stride1,
                                                         const T* __restrict__ templ, const MatchFeature* __restrict__ feat,
                                                         const TemplateSums* __restrict__ tsums, int tw, int th,
                                                         int method, int TR, bool staged, long slot,
                                                         float* __restrict__ out)
{
    extern __shared__ __align__(16) uint8_t smem[];
    const int i = blockIdx.x;
    const MatchFeature f = feat[i];
    const int ow = f.cw - tw + 1, oh = f.ch - th + 1;
    const int y0 = blockIdx.y * TR;
    if(y0 >= oh) return;
    const int rows = min(TR, oh - y0);
    const int n = tw * th;

    const T* t = templ + (size_t)i * n;
    size_t tpitch = tw;
    const T* w = img1 + (size_t)(f.cy + y0) * stride1 + f.cx;
    size_t wpitch = stride1;
    if(staged)
    {
        T* st = (T*)smem;
        T* sw = (T*)(smem + ((n * sizeof(T) + 15) & ~(size_t)15));
        for(int e = threadIdx.x; e < n; e += blockDim.x) st[e] = t[e];
        const int nw = (rows + th - 1) * f.cw;
        for(int e = threadIdx.x; e < nw; e += blockDim.x)
        {
            const int r = e / f.cw, c = e - r * f.cw;
            sw[e] = w[(size_t)r * stride1 + c];
        }
        __syncthreads();
        t = st;
        w = sw;
        wpitch = f.cw;
    }

    const TemplateSums ts = tsums[i];
    float* o = out + (size_t)i * slot + (size_t)y0 * ow;
    for(int p = threadIdx.x; p < rows * ow; p += blockDim.x)
    {
        const int yy = p / ow, xx = p - yy * ow;
        const T* wp = w + (size_t)yy * wpitch + xx;
        MatchTerms m;
        if constexpr(std::is_same<T, uint8_t>::value)
        {
            // a row's sums fit int32 (255^2 * 32767 < 2^31); rows add up in int64
            long long SI = 0, SI2 = 0, STI = 0;
            for(int v = 0; v < th; v++)
            {
                const T* a = wp + (size_t)v * wpitch;
                const T* b = t + (size_t)v * tpitch;
                int si = 0, si2 = 0, sti = 0;
                for(int u = 0; u < tw; u++)
                {
                    const int x = a[u], y = b[u];
                    si += x;
                    si2 += x * x;
                    sti += x * y;
                }
                SI += si;
                SI2 += si2;
                STI += sti;
            }
            m = terms_u8(n, ts.s, ts.s2, SI, SI2, STI);
        }
        else
        {
            // each product is exact in fp64; the sums run row-major over the template, one element at a time
            double SI = 0., SI2 = 0., STI = 0.;
            for(int v = 0; v < th; v++)
            {
                const T* a = wp + (size_t)v * wpitch;
                const T* b = t + (size_t)v * tpitch;
                for(int u = 0; u < tw; u++)
                {
                    const double x = (double)a[u], y = (double)b[u];
                    SI = __dadd_rn(SI, x);
                    SI2 = __dadd_rn(SI2, __dmul_rn(x, x));
                    STI = __dadd_rn(STI, __dmul_rn(y, x));
                }
            }
            m = terms_f32((double)n, ts.fs, ts.fs2, SI, SI2, STI);
        }
        o[p] = match_value(method, m, (double)n);
    }
}

////////////////////////////////////////////////////////////////////////////////
// 4. the optimum and the sub-pixel fit
////////////////////////////////////////////////////////////////////////////////

// numpy's argmax (argmin with lowest): the first NaN if there is one, else the first position of the extreme value.
// This is a total order on (value, index), so any reduction tree finds the same winner
__device__ __forceinline__ bool better(float a, int ia, float b, int ib, bool lowest)
{
    const bool na = isnan(a), nb = isnan(b);
    if(na != nb) return na;
    if(!na && a != b) return lowest ? a < b : a > b;
    return ia < ib;
}

// the pseudo-inverse of the reference's 9x6 design matrix (columns 1, x, y, x^2, xy, y^2 over the 3x3 neighbourhood,
// x fastest): coefficient k is (sum_j kFitNum[k][j] z_j) / kFitDen[k]
__constant__ signed char kFitNum[6][9] = {
    {-1, 2, -1, 2, 5, 2, -1, 2, -1},
    {-1, 0, 1, -1, 0, 1, -1, 0, 1},
    {-1, -1, -1, 0, 0, 0, 1, 1, 1},
    {1, -2, 1, 1, -2, 1, 1, -2, 1},
    {1, 0, -1, 0, 0, 0, -1, 0, 1},
    {1, 1, 1, -2, -2, -2, 1, 1, 1},
};
__constant__ double kFitDen[6] = {9., 6., 6., 6., 4., 6.};

__global__ void match_optimum_kernel(const MatchFeature* __restrict__ feat, int M, int tw, int th, int method,
                                     long slot, const float* __restrict__ out, MatchResult* __restrict__ res)
{
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if(i >= M) return;
    const MatchFeature f = feat[i];
    const int ow = f.cw - tw + 1, oh = f.ch - th + 1, np = ow * oh;
    const float* o = out + (size_t)i * slot;
    const bool lowest = method == TM_SQDIFF || method == TM_SQDIFF_NORMED;
    float bv = o[0];
    int bi = 0;
    for(int p = lane; p < np; p += 32)
        if(better(o[p], p, bv, bi, lowest)) { bv = o[p]; bi = p; }
    for(int d = 16; d > 0; d >>= 1)
    {
        const float v = __shfl_xor_sync(0xffffffffu, bv, d);
        const int j = __shfl_xor_sync(0xffffffffu, bi, d);
        if(better(v, j, bv, bi, lowest)) { bv = v; bi = j; }
    }
    if(lane) return;

    const int qy = bi / ow, qx = bi - qy * ow;
    MatchResult r{{NAN, NAN}, NAN, (double)MRCAL_B200_MATCH_OK};
    if(qx <= 0 || qy <= 0 || qx >= ow - 1 || qy >= oh - 1)
    {
        r.status = MRCAL_B200_MATCH_EDGE_PEAK;
        res[i] = r;
        return;
    }
    double z[9];
    for(int j = 0; j < 9; j++) z[j] = (double)o[(qy - 1 + j / 3) * ow + qx - 1 + j % 3];
    double c[6];
    for(int k = 0; k < 6; k++)
    {
        // the terms left to right, the first nonzero one first; each product is exact
        double acc = 0.;
        bool first = true;
        for(int j = 0; j < 9; j++)
        {
            const int a = kFitNum[k][j];
            if(a == 0) continue;
            const double term = __dmul_rn((double)a, z[j]);
            acc = first ? term : __dadd_rn(acc, term);
            first = false;
        }
        c[k] = __ddiv_rn(acc, kFitDen[k]);
    }
    const double c00 = c[0], c10 = c[1], c01 = c[2], c20 = c[3], c11 = c[4], c02 = c[5];
    // as the reference writes them (stereo.py:2016-2020), left to right
    const double det = __dsub_rn(__dmul_rn(__dmul_rn(4., c20), c02), __dmul_rn(c11, c11));
    const double x = __ddiv_rn(-__dsub_rn(__dmul_rn(__dmul_rn(2., c10), c02), __dmul_rn(c01, c11)), det);
    const double y = __ddiv_rn(-__dsub_rn(__dmul_rn(__dmul_rn(2., c01), c20), __dmul_rn(c10, c11)), det);
    double value = __dadd_rn(c00, __dmul_rn(c10, x));
    value = __dadd_rn(value, __dmul_rn(c01, y));
    value = __dadd_rn(value, __dmul_rn(__dmul_rn(c20, x), x));
    value = __dadd_rn(value, __dmul_rn(__dmul_rn(c11, x), y));
    value = __dadd_rn(value, __dmul_rn(__dmul_rn(c02, y), y));
    r.at[0] = __dadd_rn((double)qx, x);
    r.at[1] = __dadd_rn((double)qy, y);
    r.value = value;
    res[i] = r;
}

////////////////////////////////////////////////////////////////////////////////
// the launches
////////////////////////////////////////////////////////////////////////////////

size_t element_size(int type) { return type == MRCAL_B200_IMAGE_UINT8 ? 1 : 4; }

bool arguments_ok(int W0, int H0, int stride0, int W1, int H1, int stride1, int type, const int* features, int M,
                  int tw, int th, int slot_w, int slot_h, int method)
{
    if(type != MRCAL_B200_IMAGE_UINT8 && type != MRCAL_B200_IMAGE_FLOAT)
    { set_error("match_feature() supports uint8 and float32 images only, as cv2.matchTemplate() does; got element type %d", type); return false; }
    if(method < TM_SQDIFF || method > TM_CCOEFF_NORMED)
    { set_error("match_feature(): method must be one of the TM_* values 0..5; got %d", method); return false; }
    const size_t es = element_size(type);
    if(W0 <= 0 || H0 <= 0 || W1 <= 0 || H1 <= 0 || W0 > 32767 || H0 > 32767 || W1 > 32767 || H1 > 32767)
    { set_error("match_feature(): the images must be between 1x1 and 32767x32767 pixels; got %dx%d and %dx%d", W0, H0, W1, H1); return false; }
    if(stride0 < (long)W0 * (long)es || stride1 < (long)W1 * (long)es || stride0 % es || stride1 % es)
    { set_error("match_feature(): an image's row stride is shorter than a row or not a multiple of its element"); return false; }
    if(M < 0 || tw <= 0 || th <= 0 || (long)tw * th > (1L << 23))
    { set_error("match_feature(): M = %d must be >= 0 and the template (%dx%d) between 1 and 2^23 pixels", M, tw, th); return false; }
    if(slot_w <= 0 || slot_h <= 0)
    { set_error("match_feature(): the output slot must be at least 1x1; got %dx%d", slot_w, slot_h); return false; }
    for(int i = 0; i < M; i++)
    {
        const int* f = features + 6 * i;
        const bool ok = f[2] >= 0 && f[3] >= 0 && f[4] >= tw && f[5] >= th && (long)f[2] + f[4] <= W1 &&
                        (long)f[3] + f[5] <= H1 && f[4] - tw + 1 <= slot_w && f[5] - th + 1 <= slot_h;
        if(!ok)
        {
            set_error("match_feature(): feature %d's search cut (%d,%d) %dx%d is outside image 1, smaller than the "
                      "template or larger than the output slot", i, f[2], f[3], f[4], f[5]);
            return false;
        }
    }
    return true;
}

// Everything after the images are on the device: two uploads, the kernels, the downloads into out (and templates)
template <typename T>
bool match_run(const T* img0, size_t stride0, int W0, int H0, const T* img1, size_t stride1, int W1, int H1, int type,
               const int* features, const float* Hinv, int M, int tw, int th, int slot_w, int slot_h, int method,
               double* out, void* templates, DeviceCall& D)
{
    const long slot = (long)slot_w * slot_h;
    const int n = tw * th;
    // the templates are one (M*th, tw) image
    if((long)M * th > INT32_MAX)
    { set_error("match_feature(): %d templates of %d rows are too many for one call", M, th); return false; }
    const size_t res_bytes = (size_t)M * sizeof(MatchResult), out_bytes = res_bytes + (size_t)M * slot * sizeof(float);
    MatchFeature* d_feat;
    float *d_Hinv, *d_map;
    T* d_templ;
    TemplateSums* d_tsums;
    uint8_t* d_out;
    static_assert(sizeof(MatchFeature) == 6 * sizeof(int), "MatchFeature is the host's 6 ints");
    if(!D.upload(&d_feat, (const MatchFeature*)features, (size_t)M) || !D.upload(&d_Hinv, Hinv, 9 * (size_t)M) ||
       !D.alloc(&d_map, 2 * (size_t)M * n) || !D.alloc(&d_templ, (size_t)M * n) || !D.alloc(&d_tsums, (size_t)M) ||
       !D.alloc(&d_out, out_bytes))
        return false;
    const cudaStream_t s = D.stream;
    MatchResult* d_res = (MatchResult*)d_out;
    float* d_match = (float*)(d_out + res_bytes);

    const long Npix = (long)M * n;
    template_maps_kernel<<<(unsigned)((Npix + 255) / 256), 256, 0, s>>>(d_feat, d_Hinv, tw, th, Npix, d_map);
    MB200_CUDA_CHECK(cudaGetLastError());
    // transform_image()'s defaults: INTER_LINEAR, BORDER_CONSTANT, 0
    const double zero[3] = {0., 0., 0.};
    if(!launch_remap(img0, stride0 * sizeof(T), W0, H0, d_map, tw, M * th, type, 1, MRCAL_B200_INTER_LINEAR,
                     MRCAL_B200_BORDER_CONSTANT, zero, d_templ, s))
        return false;
    template_sums_kernel<T><<<(M + 127) / 128, 128, 0, s>>>(d_templ, n, M, d_tsums);
    MB200_CUDA_CHECK(cudaGetLastError());

    // rows per tile: about kPositionsPerCta positions, fewer if that is what it takes to stage them
    const int cw_max = min(tw + slot_w - 1, W1);
    int TR = max(1, min(slot_h, (kPositionsPerCta + slot_w - 1) / slot_w));
    auto staged_bytes = [&](int tr)
    { return (((size_t)n * sizeof(T) + 15) & ~(size_t)15) + (size_t)(tr + th - 1) * cw_max * sizeof(T); };
    if(staged_bytes(TR) > (size_t)kStagedBytes) TR = 1;
    const bool staged = staged_bytes(TR) <= (size_t)kStagedBytes;
    if(!set_max_dynamic_smem<match_kernel<T>>(kStagedBytes)) return false;
    const dim3 grid((unsigned)M, (unsigned)((slot_h + TR - 1) / TR));
    match_kernel<T><<<grid, kThreads, staged ? staged_bytes(TR) : 0, s>>>(img1, stride1, d_templ, d_feat, d_tsums, tw,
                                                                          th, method, TR, staged, slot, d_match);
    MB200_CUDA_CHECK(cudaGetLastError());
    match_optimum_kernel<<<(M + 3) / 4, 128, 0, s>>>(d_feat, M, tw, th, method, slot, d_match, d_res);
    MB200_CUDA_CHECK(cudaGetLastError());

    return D.download((uint8_t*)out, d_out, out_bytes) && (!templates || D.download((T*)templates, d_templ, (size_t)M * n)) &&
           D.finish();
}

bool match_dispatch(const void* img0, int stride0, int W0, int H0, const void* img1, int stride1, int W1, int H1,
                    int type, const int* features, const float* Hinv, int M, int tw, int th, int slot_w, int slot_h,
                    int method, double* out, void* templates, DeviceCall& D)
{
    if(type == MRCAL_B200_IMAGE_UINT8)
        return match_run<uint8_t>((const uint8_t*)img0, (size_t)stride0, W0, H0, (const uint8_t*)img1,
                                  (size_t)stride1, W1, H1, type, features, Hinv, M, tw, th, slot_w, slot_h, method,
                                  out, templates, D);
    return match_run<float>((const float*)img0, (size_t)stride0 / 4, W0, H0, (const float*)img1, (size_t)stride1 / 4,
                            W1, H1, type, features, Hinv, M, tw, th, slot_w, slot_h, method, out, templates, D);
}

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_match_feature(double* out, void* templates, const void* image0, int W0, int H0, int stride0,
                                         const void* image1, int W1, int H1, int stride1, int type,
                                         const int* features, const float* Hinv, int M, int template_w, int template_h,
                                         int slot_w, int slot_h, int method)
{
    if(!arguments_ok(W0, H0, stride0, W1, H1, stride1, type, features, M, template_w, template_h, slot_w, slot_h, method))
        return false;
    if(M == 0) return true;
    const size_t es = element_size(type), row0 = (size_t)W0 * es, row1 = (size_t)W1 * es;
    DeviceCall D;
    uint8_t *d0, *d1;
    if(!D.start() || !D.upload(&d0, image0, (size_t)stride0, row0, (size_t)H0) ||
       !D.upload(&d1, image1, (size_t)stride1, row1, (size_t)H1))
        return false;
    return match_dispatch(d0, (int)row0, W0, H0, d1, (int)row1, W1, H1, type, features, Hinv, M, template_w,
                          template_h, slot_w, slot_h, method, out, templates, D);
}

extern "C" bool mrcal_b200_match_feature_device(double* out, void* templates, const void* image0, int W0, int H0,
                                                int stride0, const void* image1, int W1, int H1, int stride1, int type,
                                                const int* features, const float* Hinv, int M, int template_w,
                                                int template_h, int slot_w, int slot_h, int method, void* stream)
{
    if(!arguments_ok(W0, H0, stride0, W1, H1, stride1, type, features, M, template_w, template_h, slot_w, slot_h, method))
        return false;
    const size_t es = element_size(type);
    if((uintptr_t)image0 % es || (uintptr_t)image1 % es)
    { set_error("match_feature(): the images must be aligned to their element size (%zu bytes)", es); return false; }
    if(M == 0) return true;
    DeviceCall D;
    return D.start((cudaStream_t)stream) &&
           match_dispatch(image0, stride0, W0, H0, image1, stride1, W1, H1, type, features, Hinv, M, template_w,
                          template_h, slot_w, slot_h, method, out, templates, D);
}
