// Deformable mirror (prysm/x/dm.py) and the cubic-spline warp it needs (prysm/coordinates.py:644-672, which is
// scipy.ndimage.map_coordinates(img, (y, x)) at order 3, mode='constant', cval=0, prefilter=True).
//
// Spline prefilter.  scipy's spline_filter runs, per axis and in float64 whatever the input dtype, the causal /
// anticausal pair of the one cubic pole z = sqrt(3) - 2 with gain 6, initialised for a mirror-extended line (for
// mode='constant' the coefficients are those of mode='mirror').  Both initialisations are exact for the mirror
// extension, so the coefficients are the infinite convolution of the mirror-extended line with
//     G z^|k|,   G = -6 z / (1 - z^2) = sqrt(3),
// and, by partial fractions, c = G (c+ + c- - s), with c+ the causal recursion c+[i] = s[i] + z c+[i-1] and c- the
// anticausal c-[i] = s[i] + z c-[i+1], both run on the input itself.  |z|^32 < 5e-19, so each thread runs both
// recursions over a chunk of kChunk samples, warmed up over kWarm samples of the mirror-extended line beyond each
// end of its chunk from a zero state: every line length (1 included) takes the same code, and lines are cut into
// independent chunks instead of being walked serially.
//
// Interpolation.  An output sample at (row r, col c) is 0 unless both lie in [0, n-1] (a coordinate exactly on the
// last sample interpolates); otherwise it is the 4 x 4 sum of the coefficients from floor(.) - 1 on, weighted by the
// cubic B-spline, with tap indices outside the array mirrored (index -1 reads 1, index n reads n - 2).  The weights
// and the sum are float64; the result is rounded to the output dtype once, as scipy does.  Coordinates come from
// two arrays (coordinates.warp) or from a 3 x 3 homography evaluated in fp64 at each output pixel (the DM: no
// coordinate arrays in memory).
#include "common.cuh"

namespace pb {

namespace {

constexpr int kChunk = 64;     // outputs per thread along a line
constexpr int kWarm = 32;      // warm-up samples beyond each end of a chunk: |z|^32 < 5e-19

struct Mat3 { double m[9]; };

__device__ __forceinline__ int mirror_index(int i, int n) {
    if (n == 1) return 0;
    const int p = 2 * (n - 1);
    i %= p;
    if (i < 0) i += p;
    return i < n ? i : p - i;
}

template <typename R>
__device__ __forceinline__ double load_real(const void* base, bool is_complex, long long idx) {
    if (is_complex) return (double)reinterpret_cast<const cplx<R>*>(base)[idx].x;
    return (double)reinterpret_cast<const R*>(base)[idx];
}

// One axis of the prefilter.  Lines are `nline` apart by `line_stride` elements, samples along a line by `step`.
// Threads take consecutive lines first, so the axis-0 pass (lines = columns, step = nx) reads and writes coalesced
// rows; the axis-1 pass walks each row within one thread.  in: T (real), complex<T> (real part) or double.
template <typename T, int kIn>   // kIn: 0 real T, 1 complex<T>, 2 double
__global__ void __launch_bounds__(128) spline_axis_kernel(const void* __restrict__ in, int n, int nline, long long step,
                                                          long long line_stride, double* __restrict__ out) {
    const long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x;
    const int nchunk = (n + kChunk - 1) / kChunk;
    if (t >= (long long)nline * nchunk) return;
    const int line = (int)(t % nline), chunk = (int)(t / nline);
    const long long base = (long long)line * line_stride;
    const int s0 = chunk * kChunk, s1 = min(n, s0 + kChunk);
    const double z = 1.7320508075688772 - 2.0;       // sqrt(3) - 2
    const double G = -6.0 * z / (1.0 - z * z);
    const bool interior = s0 - kWarm >= 0 && s1 - 1 + kWarm < n;    // no sample of the chunk's window is mirrored
    auto at = [&](int i) -> double {
        const long long idx = base + (long long)(interior ? i : mirror_index(i, n)) * step;
        if (kIn == 2) return reinterpret_cast<const double*>(in)[idx];
        return load_real<T>(in, kIn == 1, idx);
    };
    double acc = 0.0;
    for (int i = s0 - kWarm; i < s0; ++i) acc = at(i) + z * acc;
    for (int i = s0; i < s1; ++i) {
        acc = at(i) + z * acc;
        out[base + (long long)i * step] = acc;                        // c+ for now
    }
    acc = 0.0;
    for (int i = s1 - 1 + kWarm; i >= s1; --i) acc = at(i) + z * acc;
    for (int i = s1 - 1; i >= s0; --i) {
        const double s = at(i);
        acc = s + z * acc;
        const long long o = base + (long long)i * step;
        out[o] = G * (out[o] + acc - s);
    }
}

__device__ __forceinline__ void bspline3_weights(double t, double w[4]) {
    const double u = 1.0 - t, t2 = t * t, t3 = t2 * t;
    w[0] = u * u * u / 6.0;
    w[1] = (4.0 - 6.0 * t2 + 3.0 * t3) / 6.0;
    w[2] = (1.0 + 3.0 * t + 3.0 * t2 - 3.0 * t3) / 6.0;
    w[3] = t3 / 6.0;
}

// out[q] = scale * spline(coef)(row, col); coordinates from (xc, yc) arrays of type C, or the homography M applied to
// the output pixel (x, y, 1) when xc is NULL.
template <typename R, typename C>
__global__ void __launch_bounds__(256) spline_interp_kernel(const double* __restrict__ coef, int ny, int nx,
                                                            const C* __restrict__ xc, const C* __restrict__ yc, Mat3 M,
                                                            int oy, int ox, double scale, R* __restrict__ out) {
    const long long total = (long long)oy * ox;
    PB_GRID_STRIDE(q, total) {
        double cx, cy;
        if (xc) {
            cx = (double)xc[q];
            cy = (double)yc[q];
        } else {
            const double px = (double)(q % ox), py = (double)(q / ox);
            const double xp = M.m[0] * px + M.m[1] * py + M.m[2];
            const double yp = M.m[3] * px + M.m[4] * py + M.m[5];
            const double w = M.m[6] * px + M.m[7] * py + M.m[8];
            cx = xp / w;
            cy = yp / w;
        }
        double v = 0.0;
        if (cx >= 0.0 && cx <= (double)(nx - 1) && cy >= 0.0 && cy <= (double)(ny - 1)) {
            const double fx = floor(cx), fy = floor(cy);
            double wx[4], wy[4];
            bspline3_weights(cx - fx, wx);
            bspline3_weights(cy - fy, wy);
            const int x0 = (int)fx - 1, y0 = (int)fy - 1;
            int ix[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) ix[j] = mirror_index(x0 + j, nx);
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const double* row = coef + (long long)mirror_index(y0 + i, ny) * nx;
                double r = 0.0;
#pragma unroll
                for (int j = 0; j < 4; ++j) r += wx[j] * row[ix[j]];
                v += wy[i] * r;
            }
        }
        out[q] = (R)(scale * v);
    }
}

// poke[y, x] = act[(y - y0)/sy, (x - x0)/sx] on the lattice, 0 elsewhere: every sample written, no memset
template <typename R>
__global__ void dm_scatter_kernel(const R* __restrict__ act, int nay, int nax, int ny, int nx, int y0, int sy, int x0,
                                  int sx, R* __restrict__ poke) {
    const long long total = (long long)ny * nx;
    PB_GRID_STRIDE(q, total) {
        const int y = (int)(q / nx), x = (int)(q - (long long)y * nx);
        const int dy = y - y0, dx = x - x0;
        R v = R(0);
        if (dy >= 0 && dx >= 0 && dy % sy == 0 && dx % sx == 0) {
            const int ay = dy / sy, ax = dx / sx;
            if (ay < nay && ax < nax) v = act[(long long)ay * nax + ax];
        }
        poke[q] = v;
    }
}

// act[ay, ax] = real(in[y0 + ay*sy, x0 + ax*sx])
template <typename R>
__global__ void dm_gather_kernel(const void* __restrict__ in, bool cplx_in, int nx, int nay, int nax, int y0, int sy,
                                 int x0, int sx, R* __restrict__ act) {
    const long long total = (long long)nay * nax;
    PB_GRID_STRIDE(q, total) {
        const int ay = (int)(q / nax), ax = (int)(q - (long long)ay * nax);
        const long long idx = (long long)(y0 + ay * sy) * nx + (x0 + ax * sx);
        act[q] = (R)load_real<R>(in, cplx_in, idx);
    }
}

// both axes of the prefilter into `coef` (ny, nx) fp64, through `tmp` (ny, nx) fp64
template <typename R>
int spline_prefilter(Handle* h, const void* in, bool cplx_in, int ny, int nx, double* tmp, double* coef, cudaStream_t st) {
    // axis 1 (along rows) first, from the caller's array into tmp; then axis 0 (down columns) into coef
    const long long t1 = (long long)ny * ((nx + kChunk - 1) / kChunk);
    const int g1 = (int)((t1 + 127) / 128);
    if (cplx_in) spline_axis_kernel<R, 1><<<g1, 128, 0, st>>>(in, nx, ny, 1, nx, tmp);
    else spline_axis_kernel<R, 0><<<g1, 128, 0, st>>>(in, nx, ny, 1, nx, tmp);
    PB_LAUNCH_CHECK(h);
    const long long t0 = (long long)nx * ((ny + kChunk - 1) / kChunk);
    const int g0 = (int)((t0 + 127) / 128);
    spline_axis_kernel<R, 2><<<g0, 128, 0, st>>>(tmp, ny, nx, nx, 1, coef);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

}  // namespace

}  // namespace pb

using namespace pb;

extern "C" int pb_spline_prefilter(pb_handle_t hh, int dtype, const void* in, int in_complex, int ny, int nx, double* coef,
                                   void* stream) {
    PB_ENTER_REAL(hh);
    if (!in || !coef || ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "bad prefilter arguments");
    void* tmp = nullptr;
    PB_TRY(ensure_scratch(h, 1, (size_t)ny * nx * sizeof(double), &tmp));
    int rc = PB_OK;
    with_real(dtype, [&](auto r) {
        rc = spline_prefilter<decltype(r)>(h, in, in_complex != 0, ny, nx, (double*)tmp, coef, st);
    });
    return rc;
}

extern "C" int pb_warp(pb_handle_t hh, int dtype, const void* in, int in_complex, int ny, int nx, const void* xc,
                       const void* yc, int coord_dtype, const double* matrix_host, int oy, int ox, double scale, void* out,
                       void* stream) {
    PB_ENTER_REAL(hh);
    if (!in || !out || ny < 1 || nx < 1 || oy < 0 || ox < 0) return fail(h, PB_ERR_INVALID, "bad warp arguments");
    if ((xc == nullptr) != (yc == nullptr)) return fail(h, PB_ERR_INVALID, "give both coordinate arrays or neither");
    if (!xc && !matrix_host) return fail(h, PB_ERR_INVALID, "warp needs coordinate arrays or a projection matrix");
    if (coord_dtype != PB_C64 && coord_dtype != PB_C128) return fail(h, PB_ERR_INVALID, "bad coordinate dtype");
    if ((long long)oy * ox == 0) return PB_OK;
    void *coef = nullptr, *tmp = nullptr;
    PB_TRY(ensure_scratch(h, 0, (size_t)ny * nx * sizeof(double), &coef));
    PB_TRY(ensure_scratch(h, 1, (size_t)ny * nx * sizeof(double), &tmp));
    Mat3 M{};
    if (!xc) for (int i = 0; i < 9; ++i) M.m[i] = matrix_host[i];
    const int g = grid_for((long long)oy * ox, 256, h->sm_count);
    int rc = PB_OK;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        rc = spline_prefilter<R>(h, in, in_complex != 0, ny, nx, (double*)tmp, (double*)coef, st);
        if (rc != PB_OK) return;
        with_real(coord_dtype, [&](auto c) {
            using C = decltype(c);
            spline_interp_kernel<R, C><<<g, 256, 0, st>>>((const double*)coef, ny, nx, (const C*)xc, (const C*)yc, M, oy, ox,
                                                          scale, (R*)out);
        });
    });
    PB_TRY(rc);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_dm_scatter(pb_handle_t hh, int dtype, const void* act, int nay, int nax, int ny, int nx, int y0, int sy,
                             int x0, int sx, void* poke, void* stream) {
    PB_ENTER_REAL(hh);
    if (!act || !poke || nay < 1 || nax < 1 || ny < 1 || nx < 1 || sy < 1 || sx < 1 || y0 < 0 || x0 < 0 ||
        y0 + (long long)(nay - 1) * sy >= ny || x0 + (long long)(nax - 1) * sx >= nx)
        return fail(h, PB_ERR_INVALID, "actuator lattice does not fit the poke grid");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        dm_scatter_kernel<R><<<g, 256, 0, st>>>((const R*)act, nay, nax, ny, nx, y0, sy, x0, sx, (R*)poke);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_dm_gather(pb_handle_t hh, int dtype, const void* in, int in_complex, int ny, int nx, int nay, int nax, int y0,
                            int sy, int x0, int sx, void* act, void* stream) {
    PB_ENTER_REAL(hh);
    if (!in || !act || nay < 1 || nax < 1 || ny < 1 || nx < 1 || sy < 1 || sx < 1 || y0 < 0 || x0 < 0 ||
        y0 + (long long)(nay - 1) * sy >= ny || x0 + (long long)(nax - 1) * sx >= nx)
        return fail(h, PB_ERR_INVALID, "actuator lattice does not fit the array");
    const int g = grid_for((long long)nay * nax, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        dm_gather_kernel<R><<<g, 256, 0, st>>>(in, in_complex != 0, nx, nay, nax, y0, sy, x0, sx, (R*)act);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
