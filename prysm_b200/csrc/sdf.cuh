// Signed distance to a polygon, shared by the geometry kernels and the segmented-aperture rasteriser.
#pragma once
#include <cuda_runtime.h>

namespace pb {

// prysm/geometry.py:419-463 in fp64: distance to the nearest edge segment, negative inside by even-odd crossing
// parity (either winding, convex or not).  numpy's per-operation rounding without FMA contraction, so that a
// sample on an edge line keeps the sign the reference gives it.  v: (x, y) per vertex, no repeated closing vertex.
__device__ __forceinline__ double polygon_distance(const double* v, int nv, double x, double y) {
    double d2 = INFINITY;
    bool inside = false;
    for (int i = 0; i < nv; ++i) {
        const int j = i + 1 == nv ? 0 : i + 1;
        const double x0 = v[2 * i], y0 = v[2 * i + 1], x1 = v[2 * j], y1 = v[2 * j + 1];
        const double ex = x1 - x0, ey = y1 - y0, wx = x - x0, wy = y - y0;
        double t = __ddiv_rn(__dadd_rn(__dmul_rn(wx, ex), __dmul_rn(wy, ey)), __dadd_rn(__dmul_rn(ex, ex), __dmul_rn(ey, ey)));
        t = fmin(fmax(t, 0.0), 1.0);
        const double px = __dsub_rn(wx, __dmul_rn(t, ex)), py = __dsub_rn(wy, __dmul_rn(t, ey));
        d2 = fmin(d2, __dadd_rn(__dmul_rn(px, px), __dmul_rn(py, py)));
        if ((y0 > y) != (y1 > y) && ((__dmul_rn(wx, ey) < __dmul_rn(ex, wy)) == (y1 > y0))) inside = !inside;
    }
    const double d = sqrt(d2);
    return inside ? -d : d;
}

}  // namespace pb
