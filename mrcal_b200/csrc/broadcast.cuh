// The broadcast frame of the element-wise kernels (poseutils.cu, triangulation.cu, project.cu): one thread per element
// of a broadcast shape, K operands read through per-dimension strides (0 where an operand is repeated, so it is never
// expanded in memory), every index 64-bit.
#pragma once
#include <cstdint>

#include "device_call.h"

namespace mb200 {

constexpr int MAX_DIMS = 8;

template <int K> struct Broadcast
{
    int64_t N;                          // elements of the broadcast shape
    int ndim, flags;                    // flags: the operation's own, passed through to the kernel
    int64_t shape[MAX_DIMS];
    const double* in[K];                // the operands
    int64_t stride[K][MAX_DIMS];        // in doubles, per broadcast dimension; 0 where the operand is repeated
};

// o[k]: the offset of operand k's element e
template <int K>
__host__ __device__ __forceinline__ void broadcast_offsets(const Broadcast<K>& a, int64_t e, int64_t o[K])
{
    int64_t rem = e;
    for(int k = 0; k < K; k++) o[k] = 0;
    for(int d = a.ndim - 1; d > 0; d--)
    {
        const int64_t n = a.shape[d], c = rem % n;
        rem /= n;
        for(int k = 0; k < K; k++) o[k] += c * a.stride[k][d];
    }
    for(int k = 0; k < K; k++) o[k] += rem * a.stride[k][0];
}

// The shape checks every element-wise call makes, and the frame of its launch: the broadcast shape with its unit
// dimensions dropped and, where every operand allows it, neighbouring dimensions merged. Pointers are not filled
// in. strides[k] is read only where width[k] > 0 (operand k exists); who prefixes the error messages
template <int K>
bool broadcast_prepare(Broadcast<K>& a, const char* who, int flags, int ndim, const int64_t* shape,
                       const int64_t* const strides[K], const int width[K])
{
    if(ndim < 0 || ndim > MAX_DIMS)
    {
        set_error("%s: at most %d broadcast dimensions are supported; got %d", who, MAX_DIMS, ndim);
        return false;
    }
    a = Broadcast<K>{};
    a.flags = flags;
    a.N = 1;
    for(int d = 0; d < ndim; d++)
    {
        bool negative = shape[d] < 0;
        for(int k = 0; k < K; k++) negative |= width[k] > 0 && strides[k][d] < 0;
        if(negative)
        {
            set_error("%s: negative size or stride in broadcast dimension %d", who, d);
            return false;
        }
        a.N *= shape[d];
        if(shape[d] == 1) continue;
        const int n = a.ndim;
        int64_t s[K];
        bool continues = n > 0;
        for(int k = 0; k < K; k++)
        {
            s[k] = width[k] > 0 ? strides[k][d] : 0;
            // dimension d continues the previous one if each operand steps over it as over one of its elements
            continues = continues && a.stride[k][n - 1] == s[k] * shape[d];
        }
        if(continues)
        {
            a.shape[n - 1] *= shape[d];
            for(int k = 0; k < K; k++) a.stride[k][n - 1] = s[k];
            continue;
        }
        a.shape[n] = shape[d];
        for(int k = 0; k < K; k++) a.stride[k][n] = s[k];
        a.ndim++;
    }
    if(a.ndim == 0)
    {
        a.ndim = 1;
        a.shape[0] = 1;
    }
    return true;
}

// The rows of operand k that a broadcast reads, each once: a frame over a's dimensions where k is not repeated, its
// operand 0 being a's operand k
template <int K> Broadcast<1> broadcast_rows(const Broadcast<K>& a, int k)
{
    Broadcast<1> r{};
    r.N = 1;
    r.in[0] = a.in[k];
    for(int d = 0; d < a.ndim; d++)
        if(a.stride[k][d] != 0 && a.shape[d] != 1)
        {
            r.shape[r.ndim] = a.shape[d];
            r.stride[0][r.ndim] = a.stride[k][d];
            r.N *= a.shape[d];
            r.ndim++;
        }
    if(r.ndim == 0)
    {
        r.ndim = 1;
        r.shape[0] = 1;
    }
    return r;
}

// doubles operand k spans: its last element's offset plus one element
template <int K> size_t broadcast_extent(const Broadcast<K>& a, int k, int width)
{
    int64_t last = 0;
    for(int d = 0; d < a.ndim; d++) last += (a.shape[d] - 1) * a.stride[k][d];
    return (size_t)(last + width);
}

}  // namespace mb200
