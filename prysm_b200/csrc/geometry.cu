// Signed-distance pupil geometry (prysm/geometry.py:37-93, 182-248, 375-463, 550-726): polygons of any winding and
// convexity (even-odd parity), regular polygons, spider vanes, rectangles (plain and with corner fillets), annuli and
// offset circles, plus the union / intersect / subtract combinators.  Every distance is computed in fp64 from the
// stored coordinates and rounded once to the output dtype (or compared with 0 for the bool masks).  Shape parameters
// travel in kernel-parameter space, so a launch reads no table from memory and is CUDA-graph capturable.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "sdf.cuh"

namespace pb {

namespace {

struct SdfShape {
    int kind, nv;
    double p[8];
    double v[2 * PB_SDF_MAX_VERTICES];     // polygon: (x, y) per vertex; spider: (cos, sin) per vane
};

__device__ __forceinline__ double box_distance(double qx, double qy) {
    return hypot(fmax(qx, 0.0), fmax(qy, 0.0)) + fmin(fmax(qx, qy), 0.0);
}

__device__ double shape_distance(const SdfShape& s, double x, double y) {
    switch (s.kind) {
    case PB_SDF_POLYGON:
        return polygon_distance(s.v, s.nv, x, y);
    case PB_SDF_SPIDER: {                      // p: half width, centre x, centre y
        x -= s.p[1];
        y -= s.p[2];
        double d = INFINITY;
        for (int i = 0; i < s.nv; ++i) {
            const double c = s.v[2 * i], sn = s.v[2 * i + 1];
            const double along = x * c - y * sn, across = x * sn + y * c;
            d = fmin(d, hypot(fmin(along, 0.0), across) - s.p[0]);
        }
        return d;
    }
    case PB_SDF_RECTANGLE: {                   // p: half width, half height, mode (0 none, 1 swap, 2 rotate), cos, sin
        double xr = x, yr = y;
        if (s.p[2] == 1.0) { xr = y; yr = x; }
        else if (s.p[2] == 2.0) { xr = x * s.p[3] - y * s.p[4]; yr = x * s.p[4] + y * s.p[3]; }
        return box_distance(fabs(xr) - s.p[0], fabs(yr) - s.p[1]);
    }
    case PB_SDF_FILLET_RECTANGLE: {            // p: half width, half height, fillet radius, cx, cy, rotate, cos, sin
        double xr = x, yr = y;
        if (s.p[5] != 0.0) { xr = x * s.p[6] - y * s.p[7]; yr = x * s.p[7] + y * s.p[6]; }
        xr -= s.p[3];
        yr -= s.p[4];
        return box_distance(fabs(xr) - (s.p[0] - s.p[2]), fabs(yr) - (s.p[1] - s.p[2])) - s.p[2];
    }
    case PB_SDF_ANNULUS:                       // x is r; p: inner radius, outer radius
        return fabs(x - (s.p[0] + s.p[1]) / 2) - (s.p[1] - s.p[0]) / 2;
    default:                                   // PB_SDF_OFFSET_CIRCLE, p: radius, cx, cy
        return hypot(x - s.p[1], y - s.p[2]) - s.p[0];
    }
}

// out[iy, ix] = sdf(x, y) (R) or sdf <= 0 (u8).  separable: x is a row of nx values, y a column of ny values
template <typename R>
__global__ void __launch_bounds__(256) sdf_kernel(const R* __restrict__ x, const R* __restrict__ y, int separable, int ny,
                                                  int nx, const __grid_constant__ SdfShape s, int mask, void* __restrict__ out) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        double xv, yv;
        if (separable) {
            const int iy = (int)(i / nx);
            xv = (double)x[i - (long long)iy * nx];
            yv = y ? (double)y[iy] : 0.0;
        } else {
            xv = (double)x[i];
            yv = y ? (double)y[i] : 0.0;
        }
        const double d = shape_distance(s, xv, yv);
        if (mask) reinterpret_cast<unsigned char*>(out)[i] = d <= 0.0 ? 1 : 0;
        else reinterpret_cast<R*>(out)[i] = (R)d;
    }
}

// union: min(a, b); intersect: max(a, b); subtract: max(a, -b).  A NaN in either operand gives NaN, as numpy's
// minimum / maximum do, whatever the argument order.
template <typename R>
__global__ void sdf_combine_kernel(int op, const R* __restrict__ a, const R* __restrict__ b, long long n, R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const R u = a[i], v = op == PB_SDF_SUBTRACT ? -b[i] : b[i];
        R r;
        if (u != u) r = u;
        else if (v != v) r = v;
        else r = op == PB_SDF_UNION ? (v < u ? v : u) : (v > u ? v : u);
        out[i] = r;
    }
}

}  // namespace

}  // namespace pb

using namespace pb;

extern "C" int pb_sdf(pb_handle_t hh, int dtype, int kind, const void* x, const void* y, int separable, int ny, int nx,
                      const double* params_host, int nparams, const double* verts_host, int nverts, int mask, void* out,
                      void* stream) {
    PB_ENTER_REAL(hh);
    if (kind < PB_SDF_POLYGON || kind > PB_SDF_OFFSET_CIRCLE) return fail(h, PB_ERR_INVALID, "unknown shape kind");
    if (ny < 0 || nx < 0 || nparams < 0 || nparams > 8 || nverts < 0 || (nparams && !params_host) || (nverts && !verts_host))
        return fail(h, PB_ERR_INVALID, "bad shape arguments");
    if (nverts > PB_SDF_MAX_VERTICES) return fail(h, PB_ERR_UNSUPPORTED, "more than 128 polygon vertices or spider vanes");
    if ((kind == PB_SDF_POLYGON || kind == PB_SDF_SPIDER) && nverts < 1)
        return fail(h, PB_ERR_INVALID, "a polygon needs vertices and a spider vanes");
    if ((long long)ny * nx == 0) return PB_OK;
    if (!x || !out || (kind != PB_SDF_ANNULUS && !y)) return fail(h, PB_ERR_INVALID, "null pointer");
    SdfShape s{};
    s.kind = kind;
    s.nv = nverts;
    for (int i = 0; i < nparams; ++i) s.p[i] = params_host[i];
    for (int i = 0; i < 2 * nverts; ++i) s.v[i] = verts_host[i];
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    const void* yy = kind == PB_SDF_ANNULUS ? nullptr : y;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        sdf_kernel<R><<<g, 256, 0, st>>>((const R*)x, (const R*)yy, separable, ny, nx, s, mask, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_sdf_combine(pb_handle_t hh, int dtype, int op, const void* a, const void* b, long long count, void* out,
                              void* stream) {
    PB_ENTER_REAL(hh);
    if (op < PB_SDF_UNION || op > PB_SDF_SUBTRACT) return fail(h, PB_ERR_INVALID, "unknown combine op");
    if (count <= 0) return PB_OK;
    if (!a || !b || !out) return fail(h, PB_ERR_INVALID, "null pointer");
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        sdf_combine_kernel<R><<<g, 256, 0, st>>>(op, (const R*)a, (const R*)b, count, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
