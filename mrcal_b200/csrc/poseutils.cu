// The pose utilities of mrcal.poseutils on the device: one element-wise kernel family, templated on the operation.
// Each thread takes one element of the broadcast shape: it decodes the element's offset into every operand (an
// operand repeated along a dimension has stride 0 there, so it is never expanded in memory), computes in fp64 registers
// (pose.cuh) and writes the value and any gradients, packed. All indexing is 64-bit.
#include "broadcast.cuh"
#include "pose.cuh"

namespace mb200 {

namespace {

enum { F_GRAD = MRCAL_B200_POSE_GET_GRADIENTS, F_INV0 = MRCAL_B200_POSE_INVERTED0, F_INV1 = MRCAL_B200_POSE_INVERTED1 };

// doubles per element of each operand; grad: whether the operation has gradients; ninv: how many inverted flags it takes
struct OpShape
{
    int in0, in1, out0, out1, out2;
    bool grad;
    int ninv;
};

__host__ __device__ constexpr OpShape op_shape(int op)
{
    switch(op)
    {
    case MRCAL_B200_POSE_R_FROM_r:              return {3, 0, 9, 27, 0, true, 0};
    case MRCAL_B200_POSE_r_FROM_R:              return {9, 0, 3, 27, 0, true, 0};
    case MRCAL_B200_POSE_Rt_FROM_rt:            return {6, 0, 12, 27, 0, true, 0};
    case MRCAL_B200_POSE_rt_FROM_Rt:            return {12, 0, 6, 27, 0, true, 0};
    case MRCAL_B200_POSE_INVERT_R:              return {9, 0, 9, 0, 0, false, 0};
    case MRCAL_B200_POSE_INVERT_Rt:             return {12, 0, 12, 0, 0, false, 0};
    case MRCAL_B200_POSE_INVERT_rt:             return {6, 0, 6, 36, 0, true, 0};
    case MRCAL_B200_POSE_COMPOSE_Rt:            return {12, 12, 12, 0, 0, false, 2};
    case MRCAL_B200_POSE_COMPOSE_r:             return {3, 3, 3, 9, 9, true, 2};
    case MRCAL_B200_POSE_COMPOSE_rt:            return {6, 6, 6, 36, 36, true, 2};
    case MRCAL_B200_POSE_COMPOSE_r_TINYr0:      return {3, 0, 9, 0, 0, false, 0};
    case MRCAL_B200_POSE_COMPOSE_r_TINYr1:      return {3, 0, 9, 0, 0, false, 0};
    case MRCAL_B200_POSE_COMPOSE_rt_TINYrt0:    return {6, 0, 36, 0, 0, false, 0};
    case MRCAL_B200_POSE_COMPOSE_rt_TINYrt1:    return {6, 0, 36, 0, 0, false, 0};
    case MRCAL_B200_POSE_ROTATE_POINT_r:        return {3, 3, 3, 9, 9, true, 1};
    case MRCAL_B200_POSE_ROTATE_POINT_R:        return {9, 3, 3, 27, 9, true, 1};
    case MRCAL_B200_POSE_TRANSFORM_POINT_rt:    return {6, 3, 3, 18, 9, true, 1};
    case MRCAL_B200_POSE_TRANSFORM_POINT_Rt:    return {12, 3, 3, 36, 9, true, 1};
    case MRCAL_B200_POSE_SKEW_SYMMETRIC:        return {3, 0, 9, 0, 0, false, 0};
    case MRCAL_B200_POSE_R_FROM_QUAT:           return {4, 0, 9, 0, 0, false, 0};
    case MRCAL_B200_POSE_QUAT_FROM_R:           return {9, 0, 4, 0, 0, false, 0};
    case MRCAL_B200_POSE_QT_FROM_Rt:            return {12, 0, 7, 0, 0, false, 0};
    case MRCAL_B200_POSE_Rt_FROM_qt:            return {7, 0, 12, 0, 0, false, 0};
    case MRCAL_B200_POSE_R_ALIGNED_TO_VECTOR:   return {3, 0, 9, 0, 0, false, 0};
    default:                                    return {0, 0, 0, 0, 0, false, 0};
    }
}

struct PoseArgs : Broadcast<2>
{
    double* out[3];                     // packed: element e's output k at out[k] + e * out_k
};

// compose_rt (mrcal_compose_rt_full, poseutils.c:745-1001, and _compose_rt_withgrad, poseutils-genpywrap.py): r by
// compose_r(), t by the reference's four cases. d0, d1: the (6,6) drt/drt0, drt/drt1, or nullptr
__device__ __forceinline__ void compose_rt(double out[6], double* d0, double* d1, const double rt0[6],
                                           const double rt1[6], bool inv0, bool inv1)
{
    const bool G = d0 != nullptr;
    double dr0[9], dr1[9], dt_r0[9], dt_x[9];
    compose_r(out, G ? dr0 : nullptr, dr1, rt0, rt1, inv0, inv1);
    double dp_r1[9], dp_t1[9], p[3];
    if(!inv1)
    {
        // t01 = rot(r0, t1) + t0, or if inverted0: rot(-r0, t1 - t0)
        for(int i = 0; i < 3; i++) p[i] = inv0 ? rt1[3 + i] - rt0[3 + i] : rt1[3 + i];
        rotate_point_r(&out[3], G ? dt_r0 : nullptr, dt_x, rt0, p, inv0);
        if(!inv0)
            for(int i = 0; i < 3; i++) out[3 + i] += rt0[3 + i];
    }
    else
    {
        // p = -rot(-r1, t1) (-t0 if inverted0); t01 = rot(r0, p) + t0, or if inverted0: rot(-r0, p)
        rotate_point_r(p, G ? dp_r1 : nullptr, dp_t1, rt1, &rt1[3], true);
        for(int i = 0; i < 3; i++) p[i] = inv0 ? -p[i] - rt0[3 + i] : -p[i];
        rotate_point_r(&out[3], G ? dt_r0 : nullptr, dt_x, rt0, p, inv0);
        if(!inv0)
            for(int i = 0; i < 3; i++) out[3 + i] += rt0[3 + i];
    }
    if(!G) return;
    for(int i = 0; i < 3; i++)
        for(int j = 0; j < 3; j++)
        {
            double dt_t0, dt_r1, dt_t1;
            if(!inv1)
            {
                dt_t1 = dt_x[3 * i + j];
                dt_t0 = inv0 ? -dt_t1 : (i == j ? 1. : 0.);
                dt_r1 = 0.;
            }
            else
            {
                // dt/dp dp/dr1, dt/dp dp/dt1 with dp/d(r1,t1) = -drot/d(r1,t1)
                dt_r1 = -(dt_x[3 * i] * dp_r1[j] + dt_x[3 * i + 1] * dp_r1[3 + j] + dt_x[3 * i + 2] * dp_r1[6 + j]);
                dt_t1 = -(dt_x[3 * i] * dp_t1[j] + dt_x[3 * i + 1] * dp_t1[3 + j] + dt_x[3 * i + 2] * dp_t1[6 + j]);
                dt_t0 = inv0 ? -dt_x[3 * i + j] : (i == j ? 1. : 0.);
            }
            d0[6 * i + j] = dr0[3 * i + j];
            d0[6 * i + 3 + j] = 0.;
            d0[6 * (3 + i) + j] = dt_r0[3 * i + j];
            d0[6 * (3 + i) + 3 + j] = dt_t0;
            d1[6 * i + j] = dr1[3 * i + j];
            d1[6 * i + 3 + j] = 0.;
            d1[6 * (3 + i) + j] = dt_r1;
            d1[6 * (3 + i) + 3 + j] = dt_t1;
        }
}

// y0 = the value, y1, y2 = the gradients (with G) of operation OP on the inputs x0, x1
template <int OP, bool G>
__device__ __forceinline__ void pose_op(double* y0, double* y1, double* y2, const double* x0, const double* x1, int flags)
{
    const bool inv0 = flags & F_INV0, inv1 = flags & F_INV1;
    if constexpr(OP == MRCAL_B200_POSE_R_FROM_r)
        R_from_r(y0, G ? y1 : nullptr, x0);
    else if constexpr(OP == MRCAL_B200_POSE_r_FROM_R)
        r_from_R(y0, G ? y1 : nullptr, x0);
    else if constexpr(OP == MRCAL_B200_POSE_Rt_FROM_rt)
    {
        R_from_r(y0, G ? y1 : nullptr, x0);
        for(int i = 0; i < 3; i++) y0[9 + i] = x0[3 + i];
    }
    else if constexpr(OP == MRCAL_B200_POSE_rt_FROM_Rt)
    {
        r_from_R(y0, G ? y1 : nullptr, x0);
        for(int i = 0; i < 3; i++) y0[3 + i] = x0[9 + i];
    }
    else if constexpr(OP == MRCAL_B200_POSE_INVERT_R)
        invert_R(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_INVERT_Rt)
        invert_Rt(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_INVERT_rt)
    {
        // r' = -r, t' = -rot(-r, t) (mrcal_invert_rt_full, poseutils.c:557-597)
        double Jr[9], Jx[9];
        for(int i = 0; i < 3; i++) y0[i] = -x0[i];
        rotate_point_r(&y0[3], G ? Jr : nullptr, Jx, y0, &x0[3], false);
        for(int i = 0; i < 3; i++) y0[3 + i] = -y0[3 + i];
        if constexpr(G)
            for(int i = 0; i < 3; i++)
                for(int j = 0; j < 3; j++)
                {
                    y1[6 * i + j] = i == j ? -1. : 0.;
                    y1[6 * i + 3 + j] = 0.;
                    y1[6 * (3 + i) + j] = Jr[3 * i + j];
                    y1[6 * (3 + i) + 3 + j] = -Jx[3 * i + j];
                }
    }
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_Rt)
        compose_Rt(y0, x0, x1, inv0, inv1);
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_r)
        compose_r(y0, G ? y1 : nullptr, y2, x0, x1, inv0, inv1);
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_rt)
        compose_rt(y0, G ? y1 : nullptr, y2, x0, x1, inv0, inv1);
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_r_TINYr0)
        compose_r_tinyr0_gradient(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_r_TINYr1)
        compose_r_tinyr1_gradient(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_rt_TINYrt0)
    {
        // [dr/dr0 0; -skew(t1) I] (compose_rt_tinyrt0_gradientrt0, mrcal/poseutils.py)
        double D[9];
        compose_r_tinyr0_gradient(D, x0);
        const double* t = &x0[3];
        const double mS[9] = {0., t[2], -t[1], -t[2], 0., t[0], t[1], -t[0], 0.};
        for(int i = 0; i < 3; i++)
            for(int j = 0; j < 3; j++)
            {
                y0[6 * i + j] = D[3 * i + j];
                y0[6 * i + 3 + j] = 0.;
                y0[6 * (3 + i) + j] = mS[3 * i + j];
                y0[6 * (3 + i) + 3 + j] = i == j ? 1. : 0.;
            }
    }
    else if constexpr(OP == MRCAL_B200_POSE_COMPOSE_rt_TINYrt1)
    {
        // drt01/drt1 of compose_rt(rt0, 0), as compose_rt_tinyrt1_gradientrt1 (mrcal/poseutils.py) computes it
        const double zero[6] = {};
        double rt01[6], d0[36];
        compose_rt(rt01, d0, y0, x0, zero, false, false);
    }
    else if constexpr(OP == MRCAL_B200_POSE_ROTATE_POINT_r)
        rotate_point_r(y0, G ? y1 : nullptr, y2, x0, x1, inv0);
    else if constexpr(OP == MRCAL_B200_POSE_ROTATE_POINT_R || OP == MRCAL_B200_POSE_TRANSFORM_POINT_Rt)
    {
        // R x + t, or R'(x - t) if inverted (mrcal_rotate_point_R_full, mrcal_transform_point_Rt_full,
        // poseutils.c:271-424); dx/dR: x (or x - t) in row i (column i if inverted) of dx_i/dR
        constexpr bool T = OP == MRCAL_B200_POSE_TRANSFORM_POINT_Rt;
        double p[3];
        for(int i = 0; i < 3; i++) p[i] = T && inv0 ? x1[i] - x0[9 + i] : x1[i];
        for(int i = 0; i < 3; i++)
            y0[i] = Rij(x0, inv0, i, 0) * p[0] + Rij(x0, inv0, i, 1) * p[1] + Rij(x0, inv0, i, 2) * p[2] +
                    (T && !inv0 ? x0[9 + i] : 0.);
        if constexpr(G)
        {
            constexpr int W = T ? 12 : 9;   // doubles per row i of the gradient in R (or Rt)
            for(int i = 0; i < 3; i++)
                for(int jk = 0; jk < W; jk++)
                {
                    const int j = jk / 3, k = jk % 3;
                    double v;
                    if(j == 3) v = inv0 ? -x0[3 * k + i] : (i == k ? 1. : 0.);
                    else v = inv0 ? (k == i ? p[j] : 0.) : (j == i ? p[k] : 0.);
                    y1[W * i + jk] = v;
                }
            for(int i = 0; i < 3; i++)
                for(int j = 0; j < 3; j++) y2[3 * i + j] = Rij(x0, inv0, i, j);
        }
    }
    else if constexpr(OP == MRCAL_B200_POSE_TRANSFORM_POINT_rt)
    {
        // rot(r, x) + t, or rot(-r, x - t) if inverted (mrcal_transform_point_rt_full,
        // poseutils-uses-autodiff.cc:158-277)
        double p[3], Jr[9];
        for(int i = 0; i < 3; i++) p[i] = inv0 ? x1[i] - x0[3 + i] : x1[i];
        rotate_point_r(y0, G ? Jr : nullptr, y2, x0, p, inv0);
        if(!inv0)
            for(int i = 0; i < 3; i++) y0[i] += x0[3 + i];
        if constexpr(G)
            for(int i = 0; i < 3; i++)
                for(int j = 0; j < 3; j++)
                {
                    y1[6 * i + j] = Jr[3 * i + j];
                    y1[6 * i + 3 + j] = inv0 ? -y2[3 * i + j] : (i == j ? 1. : 0.);
                }
    }
    else if constexpr(OP == MRCAL_B200_POSE_SKEW_SYMMETRIC)
        skew_symmetric(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_R_FROM_QUAT)
        R_from_quat(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_QUAT_FROM_R)
        quat_from_R(y0, x0);
    else if constexpr(OP == MRCAL_B200_POSE_QT_FROM_Rt)
    {
        quat_from_R(y0, x0);
        for(int i = 0; i < 3; i++) y0[4 + i] = x0[9 + i];
    }
    else if constexpr(OP == MRCAL_B200_POSE_Rt_FROM_qt)
    {
        R_from_quat(y0, x0);
        for(int i = 0; i < 3; i++) y0[9 + i] = x0[4 + i];
    }
    else if constexpr(OP == MRCAL_B200_POSE_R_ALIGNED_TO_VECTOR)
        R_aligned_to_vector(y0, x0);
}

template <int OP, bool G> __global__ void __launch_bounds__(256) poseutils_kernel(const PoseArgs a)
{
    constexpr OpShape S = op_shape(OP);
    const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if(e >= a.N) return;
    int64_t o[2];
    broadcast_offsets(a, e, o);
    const int64_t o0 = o[0], o1 = o[1];

    double x0[S.in0], x1[S.in1 > 0 ? S.in1 : 1];
#pragma unroll
    for(int i = 0; i < S.in0; i++) x0[i] = __ldg(&a.in[0][o0 + i]);
#pragma unroll
    for(int i = 0; i < S.in1; i++) x1[i] = __ldg(&a.in[1][o1 + i]);
    constexpr int W1 = G ? S.out1 : 0, W2 = G ? S.out2 : 0;
    double y0[S.out0], y1[W1 > 0 ? W1 : 1], y2[W2 > 0 ? W2 : 1];
    pose_op<OP, G>(y0, y1, y2, x0, x1, a.flags);
    double* p0 = a.out[0] + e * S.out0;
#pragma unroll
    for(int i = 0; i < S.out0; i++) p0[i] = y0[i];
    if constexpr(G)
    {
        double* p1 = a.out[1] + e * W1;
#pragma unroll
        for(int i = 0; i < W1; i++) p1[i] = y1[i];
        double* p2 = a.out[2] + e * W2;
#pragma unroll
        for(int i = 0; i < W2; i++) p2[i] = y2[i];
    }
}

template <int OP> void launch_op(const PoseArgs& a, cudaStream_t stream)
{
    const unsigned blocks = (unsigned)((a.N + 255) / 256);
    if constexpr(op_shape(OP).grad)
        if(a.flags & F_GRAD)
        {
            poseutils_kernel<OP, true><<<blocks, 256, 0, stream>>>(a);
            return;
        }
    poseutils_kernel<OP, false><<<blocks, 256, 0, stream>>>(a);
}

template <int OP = 0> void dispatch(int op, const PoseArgs& a, cudaStream_t stream)
{
    if constexpr(OP < MRCAL_B200_POSE_NUM_OPS)
    {
        if(op == OP) launch_op<OP>(a, stream);
        else dispatch<OP + 1>(op, a, stream);
    }
}

// The checks both flavours make, and the broadcast frame of the launch. Pointers are not filled in
bool prepare(PoseArgs& a, int op, int flags, int ndim, const int64_t* shape, const int64_t* strides0,
             const int64_t* strides1)
{
    if(op < 0 || op >= MRCAL_B200_POSE_NUM_OPS)
    {
        set_error("poseutils: unknown operation %d", op);
        return false;
    }
    const OpShape S = op_shape(op);
    if(flags & ~(F_GRAD | F_INV0 | F_INV1) || ((flags & F_GRAD) && !S.grad) || ((flags & F_INV0) && S.ninv < 1) ||
       ((flags & F_INV1) && S.ninv < 2))
    {
        set_error("poseutils: operation %d does not take flags 0x%x", op, flags);
        return false;
    }
    const int64_t* const st[2] = {strides0, strides1};
    const int width[2] = {S.in0, S.in1};
    a = PoseArgs{};
    return broadcast_prepare<2>(a, "poseutils", flags, ndim, shape, st, width);
}

}  // namespace

}  // namespace mb200

using namespace mb200;

extern "C" bool mrcal_b200_poseutils(int op, int flags, int ndim, const int64_t* shape, const double* in0,
                                     const int64_t* strides0, const double* in1, const int64_t* strides1,
                                     double* out0, double* out1, double* out2)
{
    PoseArgs a;
    if(!prepare(a, op, flags, ndim, shape, strides0, strides1)) return false;
    if(a.N == 0) return true;
    const OpShape S = op_shape(op);
    const bool G = flags & F_GRAD;
    const size_t n0 = a.N * S.out0, n1 = G ? a.N * S.out1 : 0, n2 = G ? a.N * S.out2 : 0;
    DeviceCall D;
    const double *d_in0 = nullptr, *d_in1 = nullptr;
    double *d_out0, *d_out1 = nullptr, *d_out2 = nullptr;
    if(!D.start() || !D.upload((double**)&d_in0, in0, broadcast_extent(a, 0, S.in0)) ||
       (S.in1 && !D.upload((double**)&d_in1, in1, broadcast_extent(a, 1, S.in1))) || !D.alloc(&d_out0, n0) ||
       (n1 && !D.alloc(&d_out1, n1)) || (n2 && !D.alloc(&d_out2, n2)))
        return false;
    a.in[0] = d_in0;
    a.in[1] = d_in1;
    a.out[0] = d_out0;
    a.out[1] = d_out1;
    a.out[2] = d_out2;
    dispatch(op, a, D.stream);
    MB200_CUDA_CHECK(cudaGetLastError());
    return D.download(out0, d_out0, n0) && (!n1 || D.download(out1, d_out1, n1)) &&
           (!n2 || D.download(out2, d_out2, n2)) && D.finish();
}

extern "C" bool mrcal_b200_poseutils_device(int op, int flags, int ndim, const int64_t* shape, const double* in0,
                                            const int64_t* strides0, const double* in1, const int64_t* strides1,
                                            double* out0, double* out1, double* out2, void* stream)
{
    PoseArgs a;
    if(!prepare(a, op, flags, ndim, shape, strides0, strides1)) return false;
    if(a.N == 0) return true;
    if(!have_device()) return false;
    a.in[0] = in0;
    a.in[1] = in1;
    a.out[0] = out0;
    a.out[1] = out1;
    a.out[2] = out2;
    dispatch(op, a, (cudaStream_t)stream);
    MB200_CUDA_CHECK(cudaGetLastError());
    return true;
}
