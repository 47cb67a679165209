// Internal: point-in-polygon tests on the device, for the valid-intrinsics regions of camera models.
//
// A region is a closed polygon P[0..N) of imager pixels; edge i joins P[i] and P[i-1] (P[N-1] for i = 0). Two tests
// share the even-odd crossing rule written here once: inside_polygon() for image_transformation_map(), which follows
// matplotlib's contains_points() and is silent about points on an edge, and the strict test of
// is_within_valid_intrinsics_region(), which follows shapely's Polygon.contains(): a point on an edge or a vertex is
// outside.
#pragma once
#include <cuda_runtime.h>

namespace mb200 {

// Does the edge a-b cross the ray from (x, y) towards +x? A NaN point crosses nothing
__device__ __forceinline__ bool edge_crosses(double x, double y, double2 a, double2 b)
{
    return (a.y > y) != (b.y > y) && x < (b.x - a.x) * (y - a.y) / (b.y - a.y) + a.x;
}

// even-odd crossing number of the closed polygon P[N] around (x, y). A NaN point crosses nothing: outside
__device__ __forceinline__ bool inside_polygon(double x, double y, const double2* P, int N)
{
    bool c = false;
    for(int i = 0, j = N - 1; i < N; j = i++)
        if(edge_crosses(x, y, P[i], P[j])) c = !c;
    return c;
}

// Is (x, y) on the segment a-b (its end points included)? The cross product is rounded once per operation, with no
// fused multiply-add, so that a host restatement in plain double arithmetic gives the same answer; it is exact when
// the coordinates are integers below 2^26, as region vertices and pixel grids are
__device__ __forceinline__ bool on_segment(double x, double y, double2 a, double2 b)
{
    if(!(x >= fmin(a.x, b.x) && x <= fmax(a.x, b.x) && y >= fmin(a.y, b.y) && y <= fmax(a.y, b.y))) return false;
    return __dsub_rn(__dmul_rn(__dsub_rn(b.x, a.x), __dsub_rn(y, a.y)), __dmul_rn(__dsub_rn(b.y, a.y), __dsub_rn(x, a.x))) == 0.;
}

}  // namespace mb200
