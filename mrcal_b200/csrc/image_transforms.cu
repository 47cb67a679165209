// Image reprojection, as the reference's mrcal/image_transforms.py defines it: the map between two camera models
// (image_transformation_map(): unproject every target pixel, move the ray into the source camera, project) and its
// application to an image (transform_image(): cv2.remap()'s arithmetic, one thread per output pixel).
//
// The map is two passes so that the instantiations stay linear in the lens kinds: the unprojection pass is templated
// on the target model's kind and writes fp64 rays already in the source camera's frame; the projection pass is
// templated on the source model's kind, applies the valid-intrinsics mask and writes the float32 map.
#include <cuda_runtime.h>
#include <climits>
#include <cstdint>

#include "common.h"
#include "device_call.h"
#include "device_math.cuh"
#include "lens_dispatch.cuh"
#include "polygon.cuh"
#include "remap.h"
#include "unproject.cuh"

namespace mb200 {
namespace {

////////////////////////////////////////////////////////////////////////////////
// the map
////////////////////////////////////////////////////////////////////////////////

// p = M (normalize ? v / |v| * distance : v) + c: every mode of image_transformation_map() (image_transforms.py:
// 476-497). intrinsics_only: M = I; at infinity: M = R_to_from'; at a distance: M = R_to_from', c = -R_to_from' t;
// a plane: M = A_from_to
struct RayTransform
{
    double M[9], c[3];
    double distance;
    bool normalize;
};

// the largest valid-intrinsics region the projection pass holds in shared memory (48 KB of double2)
constexpr int kMaxRegion = 3072;

template <int KIND>
__global__ void reprojection_rays_kernel(LensArgs a, bool behind_ok, RayTransform T, int W, long Npix,
                                         double* __restrict__ ray)
{
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= Npix) return;
    const int i = (int)(k / W), j = (int)(k - (long)i * W);
    double v[3];
    unproject_any<KIND>(v, (double)j, (double)i, a, behind_ok);
    if(T.normalize)
    {
        const double mag = sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
        for(int r = 0; r < 3; r++) v[r] = v[r] / mag * T.distance;
    }
    for(int r = 0; r < 3; r++)
        ray[3 * k + r] = T.M[3 * r] * v[0] + T.M[3 * r + 1] * v[1] + T.M[3 * r + 2] * v[2] + T.c[r];
}

// map[k] = project_from(ray[k]) as a float32 pair; (-1, -1) outside the region, if one is given (Nregion > 0)
template <int KIND>
__global__ void reprojection_map_kernel(LensArgs a, const double* __restrict__ ray, long Npix,
                                        const double2* __restrict__ region, int Nregion, float2* __restrict__ map)
{
    extern __shared__ double2 poly[];
    for(int r = threadIdx.x; r < Nregion; r += blockDim.x) poly[r] = region[r];
    __syncthreads();
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= Npix) return;
    const double p[3] = {ray[3 * k], ray[3 * k + 1], ray[3 * k + 2]};
    double q[2], g[2][3];
    project_any<KIND>(q, g, p, a);
    if(Nregion > 0 && !inside_polygon(q[0], q[1], poly, Nregion)) { q[0] = -1.; q[1] = -1.; }
    map[k] = make_float2((float)q[0], (float)q[1]);
}

////////////////////////////////////////////////////////////////////////////////
// is_within_valid_intrinsics_region(): the strict test
////////////////////////////////////////////////////////////////////////////////

// vertices per shared-memory tile of the strict test (16 KB of double2)
constexpr int kRegionTile = 1024;

// mask[k]: q[k] lies strictly inside the region: on none of its edges, and inside by the even-odd rule. The vertices
// go through shared memory a tile at a time, slot 0 of a tile holding the vertex before the tile's first, so that a
// region of any size is accepted. The parity is the same whatever the order of the edges
__global__ void __launch_bounds__(256) within_region_kernel(const double2* __restrict__ q, long N,
                                                            const double2* __restrict__ region, int Nregion,
                                                            bool* __restrict__ mask)
{
    __shared__ double2 tile[kRegionTile + 1];
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    const double2 p = k < N ? q[k] : make_double2(NAN, NAN);
    bool in = false, edge = false;
    for(int t0 = 0; t0 < Nregion; t0 += kRegionTile)
    {
        const int n = min(kRegionTile, Nregion - t0);
        __syncthreads();
        for(int r = threadIdx.x; r <= n; r += blockDim.x)
            tile[r] = region[r > 0 ? t0 + r - 1 : (t0 > 0 ? t0 - 1 : Nregion - 1)];
        __syncthreads();
        for(int i = 1; i <= n; i++)
        {
            const double2 a = tile[i], b = tile[i - 1];
            edge = edge || on_segment(p.x, p.y, a, b);
            if(edge_crosses(p.x, p.y, a, b)) in = !in;
        }
    }
    if(k < N) mask[k] = in && !edge;
}

////////////////////////////////////////////////////////////////////////////////
// the remap: cv2.remap() with a CV_32FC2 map, restated
////////////////////////////////////////////////////////////////////////////////

// cvRound(float): round half to even; NaN, +-inf and anything outside int32 give INT_MIN, as the x86 conversion
// OpenCV uses does. The device's own conversions saturate and take NaN to 0, so those cases are explicit
__device__ __forceinline__ int cv_round(float v)
{
    return (v >= -2147483648.f && v < 2147483648.f) ? __float2int_rn(v) : INT_MIN;
}

__device__ __forceinline__ int saturate_short(int v) { return min(max(v, -32768), 32767); }

template <typename T> struct Cval { T v[3]; };

template <typename T>
__device__ __forceinline__ T cast_out(float s)
{
    if constexpr(std::is_same<T, float>::value) return s;
    else return (T)min(max(cv_round(s), 0), 65535);   // uint16_t: saturate_cast<ushort>(float)
}

// One output pixel of CN channels. src: rows of W*CN elements, stride bytes apart; dst and map are packed. With
// BORDER_TRANSPARENT the output pixel is left as it is where the map points outside the image. The map is read as two
// floats, not a float2: a caller's map (a tensor view, say) need only be 4-byte aligned
template <typename T, int CN, int INTER, int BORDER>
__global__ void remap_kernel(const T* __restrict__ src, size_t stride, int W, int H, const float* __restrict__ map,
                             long Npix, Cval<T> cval, T* __restrict__ dst)
{
    const long k = (long)blockIdx.x * blockDim.x + threadIdx.x;
    if(k >= Npix) return;
    const float2 m = make_float2(map[2 * k], map[2 * k + 1]);
    T* d = dst + k * CN;
    if constexpr(INTER == MRCAL_B200_INTER_NEAREST)
    {
        const int sx = saturate_short(cv_round(m.x)), sy = saturate_short(cv_round(m.y));
        if((unsigned)sx < (unsigned)W && (unsigned)sy < (unsigned)H)
        {
            const T* s = (const T*)((const char*)src + sy * stride) + sx * CN;
            for(int c = 0; c < CN; c++) d[c] = s[c];
        }
        else if(BORDER == MRCAL_B200_BORDER_CONSTANT)
            for(int c = 0; c < CN; c++) d[c] = cval.v[c];
        return;
    }
    else
    {
        // 5 fractional bits: X = cvRound(x * 32), the fraction X & 31, the integer part X >> 5 as int16
        const int X = cv_round(__fmul_rn(m.x, 32.f)), Y = cv_round(__fmul_rn(m.y, 32.f));
        const int fx = X & 31, fy = Y & 31;
        const int sx = saturate_short(X >> 5), sy = saturate_short(Y >> 5);
        int x1 = sx + 1, y1 = sy + 1;
        bool in00, in01, in10, in11;
        if constexpr(BORDER == MRCAL_B200_BORDER_CONSTANT)
        {
            if(sx >= W || x1 < 0 || sy >= H || y1 < 0)
            {
                for(int c = 0; c < CN; c++) d[c] = cval.v[c];
                return;
            }
            const bool ix0 = sx >= 0, ix1 = x1 < W, iy0 = sy >= 0, iy1 = y1 < H;
            in00 = ix0 && iy0; in01 = ix1 && iy0; in10 = ix0 && iy1; in11 = ix1 && iy1;
        }
        else
        {
            if((unsigned)sx >= (unsigned)W || (unsigned)sy >= (unsigned)H) return;
            x1 = min(x1, W - 1); y1 = min(y1, H - 1);
            in00 = in01 = in10 = in11 = true;
        }
        // the rows of the taps; a row outside the image is never read
        const T* r0 = (const T*)((const char*)src + max(sy, 0) * stride);
        const T* r1 = (const T*)((const char*)src + min(y1, H - 1) * stride);
        for(int c = 0; c < CN; c++)
        {
            const T t0 = in00 ? r0[sx * CN + c] : cval.v[c];
            const T t1 = in01 ? r0[x1 * CN + c] : cval.v[c];
            const T t2 = in10 ? r1[sx * CN + c] : cval.v[c];
            const T t3 = in11 ? r1[x1 * CN + c] : cval.v[c];
            if constexpr(std::is_same<T, uint8_t>::value)
            {
                // integer weights summing to 2^15, rounded back
                const int s = (int)t0 * ((32 - fy) * (32 - fx) * 32) + (int)t1 * ((32 - fy) * fx * 32) +
                              (int)t2 * (fy * (32 - fx) * 32) + (int)t3 * (fy * fx * 32);
                d[c] = (uint8_t)min((s + (1 << 14)) >> 15, 255);
            }
            else
            {
                // float32 weights, summed left to right without contraction
                const float a = (float)fx * 0.03125f, b = (float)fy * 0.03125f;
                const float w0 = __fmul_rn(1.f - b, 1.f - a), w1 = __fmul_rn(1.f - b, a);
                const float w2 = __fmul_rn(b, 1.f - a), w3 = __fmul_rn(b, a);
                const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn((float)t0, w0), __fmul_rn((float)t1, w1)),
                                                    __fmul_rn((float)t2, w2)),
                                          __fmul_rn((float)t3, w3));
                d[c] = cast_out<T>(s);
            }
        }
    }
}

template <typename T>
bool launch_remap_typed(const void* src, size_t stride, int W, int H, const float* map, long Npix, int channels, int interpolation,
                        int border, const double* border_value, void* dst, cudaStream_t s)
{
    // saturate_cast<T>(borderValue[c]) (imgwarp.cpp): round half to even and clamp for the integer types
    Cval<T> cval;
    for(int c = 0; c < 3; c++)
    {
        const double v = c < channels ? border_value[c] : 0.;
        if constexpr(std::is_same<T, float>::value) cval.v[c] = (float)v;
        else
        {
            const double hi = std::is_same<T, uint8_t>::value ? 255. : 65535.;
            cval.v[c] = (T)fmin(fmax(std::nearbyint(v), 0.), hi);
        }
    }
    const unsigned blocks = (unsigned)((Npix + 255) / 256);
    auto go = [&](auto cn, auto inter, auto bord)
    {
        remap_kernel<T, decltype(cn)::value, decltype(inter)::value, decltype(bord)::value><<<blocks, 256, 0, s>>>(
            (const T*)src, stride, W, H, map, Npix, cval, (T*)dst);
    };
    using I0 = std::integral_constant<int, MRCAL_B200_INTER_NEAREST>;
    using I1 = std::integral_constant<int, MRCAL_B200_INTER_LINEAR>;
    using BC = std::integral_constant<int, MRCAL_B200_BORDER_CONSTANT>;
    using BT = std::integral_constant<int, MRCAL_B200_BORDER_TRANSPARENT>;
    auto by_border = [&](auto cn, auto inter)
    {
        if(border == MRCAL_B200_BORDER_CONSTANT) go(cn, inter, BC{});
        else go(cn, inter, BT{});
    };
    auto by_inter = [&](auto cn)
    {
        if(interpolation == MRCAL_B200_INTER_NEAREST) by_border(cn, I0{});
        else by_border(cn, I1{});
    };
    if(channels == 1) by_inter(std::integral_constant<int, 1>{});
    else by_inter(std::integral_constant<int, 3>{});
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}

size_t element_size(int type) { return type == MRCAL_B200_IMAGE_UINT8 ? 1 : type == MRCAL_B200_IMAGE_UINT16 ? 2 : 4; }

bool remap_arguments_ok(int W, int H, int stride, int Wo, int Ho, int type, int channels, int interpolation, int border)
{
    if(type != MRCAL_B200_IMAGE_UINT8 && type != MRCAL_B200_IMAGE_UINT16 && type != MRCAL_B200_IMAGE_FLOAT)
    { set_error("transform_image() supports uint8, uint16 and float32 images only; got element type %d", type); return false; }
    if(channels != 1 && channels != 3)
    { set_error("transform_image() supports 1- and 3-channel images only; got %d channels", channels); return false; }
    if(interpolation != MRCAL_B200_INTER_NEAREST && interpolation != MRCAL_B200_INTER_LINEAR)
    { set_error("transform_image() supports INTER_NEAREST (0) and INTER_LINEAR (1) only; got %d", interpolation); return false; }
    if(border != MRCAL_B200_BORDER_CONSTANT && border != MRCAL_B200_BORDER_TRANSPARENT)
    { set_error("transform_image() supports BORDER_CONSTANT (0) and BORDER_TRANSPARENT (5) only; got %d", border); return false; }
    if(W <= 0 || H <= 0 || W > 32767 || H > 32767)
    { set_error("transform_image(): the image must be between 1x1 and 32767x32767 pixels; got %dx%d", W, H); return false; }
    if(Wo < 0 || Ho < 0) { set_error("transform_image(): the map has a negative size"); return false; }
    if(stride < (long)W * channels * (long)element_size(type))
    { set_error("transform_image(): the image's row stride (%d bytes) is shorter than a row", stride); return false; }
    return true;
}

}  // namespace

// The one launcher of both transform entry points and of match_feature()'s templates (remap.h): device pointers; the
// map and the output are packed
bool launch_remap(const void* src, size_t stride, int W, int H, const float* map, int Wo, int Ho, int type, int channels,
                  int interpolation, int border, const double* border_value, void* dst, cudaStream_t s)
{
    const long Npix = (long)Wo * Ho;
    if(Npix == 0) return true;
    switch(type)
    {
    case MRCAL_B200_IMAGE_UINT8:
        return launch_remap_typed<uint8_t>(src, stride, W, H, map, Npix, channels, interpolation, border, border_value, dst, s);
    case MRCAL_B200_IMAGE_UINT16:
        return launch_remap_typed<uint16_t>(src, stride, W, H, map, Npix, channels, interpolation, border, border_value, dst, s);
    default:
        return launch_remap_typed<float>(src, stride, W, H, map, Npix, channels, interpolation, border, border_value, dst, s);
    }
}

namespace {

// the inverse of the 3x3 A (row-major) by its adjugate; false if A is singular
bool invert3(double out[9], const double A[9])
{
    const double c00 = A[4] * A[8] - A[5] * A[7], c01 = A[5] * A[6] - A[3] * A[8], c02 = A[3] * A[7] - A[4] * A[6];
    const double det = A[0] * c00 + A[1] * c01 + A[2] * c02;
    if(!(fabs(det) > 0.) || !std::isfinite(det)) return false;
    const double adj[9] = {c00, A[2] * A[7] - A[1] * A[8], A[1] * A[5] - A[2] * A[4],
                           c01, A[0] * A[8] - A[2] * A[6], A[2] * A[3] - A[0] * A[5],
                           c02, A[1] * A[6] - A[0] * A[7], A[0] * A[4] - A[1] * A[3]};
    for(int i = 0; i < 9; i++) out[i] = adj[i] / det;
    return true;
}

}  // namespace
}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_image_transformation_map(float* mapxy, int W_to, int H_to,
                                                    const mrcal_lensmodel_t* lensmodel_from,
                                                    const double* intrinsics_from,
                                                    const mrcal_lensmodel_t* lensmodel_to, const double* intrinsics_to,
                                                    const double* Rt_to_from, const double* distance,
                                                    const double* plane_n, double plane_d,
                                                    const mrcal_point2_t* region, int Nregion)
{
    if(W_to <= 0 || H_to <= 0) { set_error("model_to's imager must be at least 1x1; got %dx%d", W_to, H_to); return false; }
    if(plane_n && (Rt_to_from == nullptr || distance))
    {
        set_error("A plane needs Rt_to_from, and excludes distance");
        return false;
    }
    if(distance && Rt_to_from == nullptr) { set_error("distance needs Rt_to_from"); return false; }
    if(region && (Nregion < 1 || Nregion > kMaxRegion))
    {
        set_error("The valid-intrinsics region must have between 1 and %d vertices; got %d", kMaxRegion, Nregion);
        return false;
    }
    HostLens from, to;
    if(!lens_setup(&from, lensmodel_from) || !lens_setup(&to, lensmodel_to) || !central_projection(to, intrinsics_to))
        return false;

    RayTransform T{};
    T.M[0] = T.M[4] = T.M[8] = 1.;
    if(Rt_to_from)
    {
        const double* R = Rt_to_from;   // (4,3): R, then t
        const double* t = Rt_to_from + 9;
        if(plane_n)
        {
            // A_to_from = plane_d R_to_from + t_to_from plane_n' (image_transforms.py:480-488)
            double A[9];
            for(int i = 0; i < 3; i++)
                for(int j = 0; j < 3; j++) A[3 * i + j] = plane_d * R[3 * i + j] + t[i] * plane_n[j];
            if(!invert3(T.M, A)) { set_error("The plane homography A_to_from is singular"); return false; }
        }
        else
        {
            for(int i = 0; i < 3; i++)
                for(int j = 0; j < 3; j++) T.M[3 * i + j] = R[3 * j + i];
            if(distance)
            {
                T.normalize = true;
                T.distance = *distance;
                for(int i = 0; i < 3; i++) T.c[i] = -(R[i] * t[0] + R[3 + i] * t[1] + R[6 + i] * t[2]);
            }
        }
    }
    DeviceCall D;
    if(!D.start()) return false;

    const long Npix = (long)W_to * H_to;
    double *d_intr_from, *d_intr_to, *d_ray, *d_region = nullptr;
    float2* d_map;
    if(!D.upload(&d_intr_from, intrinsics_from, (size_t)from.Nintr) || !D.upload(&d_intr_to, intrinsics_to, (size_t)to.Nintr) ||
       (region && !D.upload(&d_region, (const double*)region, 2 * (size_t)Nregion)) ||
       !D.alloc(&d_ray, 3 * (size_t)Npix) || !D.alloc(&d_map, (size_t)Npix))
        return false;
    from.a.intr = d_intr_from;
    to.a.intr = d_intr_to;
    const bool behind_ok = mrcal_lensmodel_metadata(lensmodel_to).can_project_behind_camera;
    const unsigned blocks = (unsigned)((Npix + 127) / 128);
    if(!dispatch_lens_kind(to.kind, [&](auto k)
    {
        reprojection_rays_kernel<decltype(k)::value><<<blocks, 128, 0, D.stream>>>(to.a, behind_ok, T, W_to, Npix, d_ray);
    })) return false;
    const int nreg = region ? Nregion : 0;
    if(!dispatch_lens_kind(from.kind, [&](auto k)
    {
        reprojection_map_kernel<decltype(k)::value><<<blocks, 128, nreg * sizeof(double2), D.stream>>>(
            from.a, d_ray, Npix, (const double2*)d_region, nreg, d_map);
    })) return false;
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download((float2*)mapxy, d_map, (size_t)Npix) && D.finish();
}

extern "C" bool mrcal_b200_is_within_region(bool* mask, const mrcal_point2_t* q, int N, const mrcal_point2_t* region,
                                            int Nregion)
{
    if(N < 0 || Nregion < 0) { set_error("is_within_region: N = %d and Nregion = %d must be >= 0", N, Nregion); return false; }
    if(N == 0) return true;
    DeviceCall D;
    double *d_q, *d_region;
    bool* d_mask;
    if(!D.start() || !D.upload(&d_q, (const double*)q, 2 * (size_t)N) ||
       !D.upload(&d_region, (const double*)region, 2 * (size_t)Nregion) || !D.alloc(&d_mask, (size_t)N))
        return false;
    within_region_kernel<<<(unsigned)((N + 255) / 256), 256, 0, D.stream>>>((const double2*)d_q, N, (const double2*)d_region,
                                                                            Nregion, d_mask);
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(mask, d_mask, (size_t)N) && D.finish();
}

extern "C" bool mrcal_b200_transform_image(void* out, const void* image, int W, int H, int image_stride, int type,
                                           int channels, const float* mapxy, int W_out, int H_out, int interpolation,
                                           int border_mode, const double* border_value)
{
    if(!remap_arguments_ok(W, H, image_stride, W_out, H_out, type, channels, interpolation, border_mode)) return false;
    DeviceCall D;
    if(!D.start()) return false;
    const size_t row = (size_t)W * channels * element_size(type);
    const long Npix = (long)W_out * H_out;
    if(Npix == 0) return true;
    const size_t out_bytes = Npix * channels * element_size(type);
    uint8_t *d_src, *d_dst;
    float* d_map;
    // a transparent border leaves pixels as they were: start from the caller's output
    const bool transparent = border_mode == MRCAL_B200_BORDER_TRANSPARENT;
    if(!D.upload(&d_src, image, (size_t)image_stride, row, (size_t)H) ||
       !(transparent ? D.upload(&d_dst, (const uint8_t*)out, out_bytes) : D.alloc(&d_dst, out_bytes)) ||
       !D.upload(&d_map, mapxy, 2 * (size_t)Npix))
        return false;
    return launch_remap(d_src, row, W, H, d_map, W_out, H_out, type, channels, interpolation, border_mode, border_value,
                        d_dst, D.stream) &&
           D.download((uint8_t*)out, d_dst, out_bytes) && D.finish();
}

extern "C" bool mrcal_b200_transform_image_device(void* out, const void* image, int W, int H, int image_stride,
                                                  int type, int channels, const float* mapxy, int W_out, int H_out,
                                                  int interpolation, int border_mode, const double* border_value,
                                                  void* stream)
{
    if(!remap_arguments_ok(W, H, image_stride, W_out, H_out, type, channels, interpolation, border_mode)) return false;
    // every access is of one element: each buffer and the row stride need that element's alignment, and no more
    const size_t es = element_size(type);
    if((uintptr_t)image % es || (uintptr_t)out % es || image_stride % es || (uintptr_t)mapxy % sizeof(float))
    {
        set_error("transform_image(): image, out and the row stride must be aligned to the element size (%zu bytes), "
                  "mapxy to 4 bytes", es);
        return false;
    }
    return launch_remap(image, (size_t)image_stride, W, H, mapxy, W_out, H_out, type, channels, interpolation, border_mode, border_value, out,
                        (cudaStream_t)stream);
}
