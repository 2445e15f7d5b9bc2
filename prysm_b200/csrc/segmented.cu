// Segmented apertures (prysm/segmented.py:133-368): one launch rasterises every hexagonal segment, one launch
// composes the per-segment modal OPD, and two launches give its adjoint with respect to the coefficients.
//
// Geometry of the work.  Segment s owns a window (y0, x0, h, w) of the (ny, nx) grid and h*w samples in each packed
// per-segment buffer (coverage, local x, local y) starting at moff; its modal basis (nmodes, h, w) starts at boff in
// the packed basis buffer, shared by every segment with the same local grid.  The host lists, per output tile of
// PB_SEGMENT_TILE_Y x PB_SEGMENT_TILE_X samples, the segments whose windows meet the tile, in segment order (CSR).
// A block owns one tile: windows may overlap (a gap narrower than a sample), but each output sample is written by
// one thread, which walks that list in order with an fp64 accumulator.  No atomics: every call and every graph
// replay gives the same bits.
#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "sdf.cuh"

namespace pb {

namespace {

constexpr int kTY = PB_SEGMENT_TILE_Y, kTX = PB_SEGMENT_TILE_X, kThreads = 256;
constexpr int kRows = kTY * kTX / kThreads;      // output rows per thread, kThreads / kTX apart
constexpr int kMaxSides = 8;
constexpr int kModeBlock = 8;                    // modes reduced together by the adjoint

struct Win { int y0, x0, h, w; long long moff, boff; };

__device__ __forceinline__ Win load_win(const long long* __restrict__ seg, int s) {
    const long long* e = seg + (long long)s * PB_SEGMENT_FIELDS;
    return Win{(int)e[0], (int)e[1], (int)e[2], (int)e[3], e[4], e[5]};
}

// coverage = clip(0.5 - polygon_sdf/dx, 0, 1) (segmented.py:321-322, 361-362; geometry.py:11-34) of every segment
// window sample, its local coordinates (x - cx, y - cy; segmented.py:359), and amp = the max over the segments that
// cover a sample, 0 elsewhere (segmented.py:316, 324, 364).  geo: per segment nv (x, y) vertices, then (cx, cy).
template <typename R>
__global__ void __launch_bounds__(kThreads) hex_raster_kernel(const R* __restrict__ x, const R* __restrict__ y, int ny, int nx,
                                                              int tiles_x, const int* __restrict__ tile_ptr,
                                                              const int* __restrict__ tile_seg, const long long* __restrict__ seg,
                                                              const double* __restrict__ geo, int nv, double dx,
                                                              R* __restrict__ cover, R* __restrict__ lx, R* __restrict__ ly,
                                                              R* __restrict__ amp) {
    const int tile = blockIdx.x;
    const int col = (tile % tiles_x) * kTX + threadIdx.x % kTX;
    const int row0 = (tile / tiles_x) * kTY + threadIdx.x / kTX;
    double a[kRows];
#pragma unroll
    for (int j = 0; j < kRows; ++j) a[j] = 0.0;
    __shared__ double v[2 * kMaxSides + 2];     // the segment's vertices, then its centre
    for (int e = tile_ptr[tile]; e < tile_ptr[tile + 1]; ++e) {
        const int s = tile_seg[e];
        __syncthreads();                        // the previous segment's vertices are no longer read
        if (threadIdx.x < 2 * nv + 2) v[threadIdx.x] = geo[(long long)s * (2 * nv + 2) + threadIdx.x];
        __syncthreads();
        const Win win = load_win(seg, s);
        const double cx = v[2 * nv], cy = v[2 * nv + 1];
        const int lc = col - win.x0;
        if (lc < 0 || lc >= win.w) continue;
#pragma unroll
        for (int j = 0; j < kRows; ++j) {
            const int row = row0 + j * (kThreads / kTX), lr = row - win.y0;
            if (lr < 0 || lr >= win.h) continue;
            const long long p = (long long)row * nx + col, q = win.moff + (long long)lr * win.w + lc;
            const double xv = (double)x[p], yv = (double)y[p];
            const double c = fmin(fmax(0.5 - polygon_distance(v, nv, xv, yv) / dx, 0.0), 1.0);
            const R cr = (R)c;
            cover[q] = cr;
            lx[q] = (R)(xv - cx);
            ly[q] = (R)(yv - cy);
            a[j] = fmax(a[j], (double)cr);
        }
    }
    if (col >= nx) return;
#pragma unroll
    for (int j = 0; j < kRows; ++j) {
        const int row = row0 + j * (kThreads / kTX);
        if (row < ny) amp[(long long)row * nx + col] = (R)a[j];
    }
}

// out += sum over the tile's segments s < ncoef, in order, of mask_s * sum_k c[s, k] * base_{s,k}, accumulated in
// fp64 and rounded once (segmented.py:278-285; zip truncation: only the first ncoef segments)
template <typename R>
__global__ void __launch_bounds__(kThreads) segment_compose_kernel(int ny, int nx, int tiles_x, const int* __restrict__ tile_ptr,
                                                                   const int* __restrict__ tile_seg,
                                                                   const long long* __restrict__ seg, const R* __restrict__ masks,
                                                                   const R* __restrict__ bases, int nmodes,
                                                                   const double* __restrict__ coefs, long long cstride,
                                                                   int ncoef, R* __restrict__ out) {
    const int tile = blockIdx.x;
    const int e0 = tile_ptr[tile], e1 = tile_ptr[tile + 1];
    if (e0 == e1 || tile_seg[e0] >= ncoef) return;
    const int col = (tile % tiles_x) * kTX + threadIdx.x % kTX;
    const int row0 = (tile / tiles_x) * kTY + threadIdx.x / kTX;
    double acc[kRows];
#pragma unroll
    for (int j = 0; j < kRows; ++j) acc[j] = 0.0;
    for (int e = e0; e < e1; ++e) {
        const int s = tile_seg[e];
        if (s >= ncoef) break;                  // lists are in segment order
        const Win win = load_win(seg, s);
        const int lc = col - win.x0;
        if (lc < 0 || lc >= win.w) continue;
        const long long hw = (long long)win.h * win.w;
        const double* c = coefs + (long long)s * cstride;
#pragma unroll
        for (int j = 0; j < kRows; ++j) {
            const int lr = row0 + j * (kThreads / kTX) - win.y0;
            if (lr < 0 || lr >= win.h) continue;
            const long long q = (long long)lr * win.w + lc;
            const double m = (double)masks[win.moff + q];
            if (m == 0.0) continue;             // adds 0 in the reference
            const R* b = bases + win.boff + q;
            double v = 0.0;
            for (int k = 0; k < nmodes; ++k) v += c[k] * (double)b[k * hw];
            acc[j] += m * v;
        }
    }
    if (col >= nx) return;
#pragma unroll
    for (int j = 0; j < kRows; ++j) {
        const int row = row0 + j * (kThreads / kTX);
        if (row < ny) {
            const long long p = (long long)row * nx + col;
            out[p] = (R)((double)out[p] + acc[j]);
        }
    }
}

// level 1 of the adjoint: partial[s, b, k] = sum over chunk b of segment s's window of g * mask_s * base_{s,k}
template <typename R>
__global__ void __launch_bounds__(kThreads) segment_adjoint_partial_kernel(int nx, const long long* __restrict__ seg,
                                                                           const R* __restrict__ masks, const R* __restrict__ bases,
                                                                           int nmodes, const R* __restrict__ g, int nchunk,
                                                                           double* __restrict__ partial) {
    __shared__ double red[kThreads / 32][kModeBlock];
    const int s = blockIdx.y, b = blockIdx.x;
    const Win win = load_win(seg, s);
    const long long hw = (long long)win.h * win.w;
    const long long q0 = (long long)b * PB_SEGMENT_CHUNK, q1 = std::min(hw, q0 + PB_SEGMENT_CHUNK);
    for (int k0 = 0; k0 < nmodes; k0 += kModeBlock) {
        double acc[kModeBlock];
#pragma unroll
        for (int kk = 0; kk < kModeBlock; ++kk) acc[kk] = 0.0;
        for (long long q = q0 + threadIdx.x; q < q1; q += kThreads) {
            const int lr = (int)(q / win.w), lc = (int)(q - (long long)lr * win.w);
            const double gm = (double)g[(long long)(win.y0 + lr) * nx + win.x0 + lc] * (double)masks[win.moff + q];
            if (gm == 0.0) continue;
            const R* bp = bases + win.boff + q;
#pragma unroll
            for (int kk = 0; kk < kModeBlock; ++kk)
                if (k0 + kk < nmodes) acc[kk] += gm * (double)bp[(long long)(k0 + kk) * hw];
        }
        warp_partials<kThreads>(acc, OpAdd{}, red);
        if (threadIdx.x < kModeBlock && k0 + threadIdx.x < nmodes) {
            double v = 0.0;
            for (int w = 0; w < kThreads / 32; ++w) v += red[w][threadIdx.x];
            partial[((long long)s * nchunk + b) * nmodes + k0 + threadIdx.x] = v;
        }
        __syncthreads();
    }
}

// level 2: out[s, k] = sum over b, in order, of partial[s, b, k], rounded once
template <typename R>
__global__ void segment_adjoint_final_kernel(int nseg, int nmodes, int nchunk, const double* __restrict__ partial,
                                             R* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nseg * nmodes) return;
    const int s = i / nmodes, k = i - s * nmodes;
    double v = 0.0;
    for (int b = 0; b < nchunk; ++b) v += partial[((long long)s * nchunk + b) * nmodes + k];
    out[i] = (R)v;
}

}  // namespace

}  // namespace pb

using namespace pb;

static inline int tile_count(int ny, int nx, int tiles_y, int tiles_x) {
    return (tiles_y == (ny + kTY - 1) / kTY && tiles_x == (nx + kTX - 1) / kTX) ? tiles_y * tiles_x : -1;
}

extern "C" int pb_hex_segments(pb_handle_t hh, int dtype, const void* x, const void* y, int ny, int nx, int tiles_y, int tiles_x,
                               const int* tile_ptr, const int* tile_seg, const long long* seg, const double* geo, int nverts,
                               double dx, void* cover, void* local_x, void* local_y, void* amp, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || nverts < 3 || nverts > kMaxSides || !(dx > 0.0))
        return fail(h, PB_ERR_INVALID, "bad segment raster arguments");
    const int nt = tile_count(ny, nx, tiles_y, tiles_x);
    if (nt < 0) return fail(h, PB_ERR_INVALID, "tile grid does not match the array");
    if (!x || !y || !tile_ptr || !tile_seg || !seg || !geo || !cover || !local_x || !local_y || !amp)
        return fail(h, PB_ERR_INVALID, "null pointer");
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        hex_raster_kernel<R><<<nt, kThreads, 0, st>>>((const R*)x, (const R*)y, ny, nx, tiles_x, tile_ptr, tile_seg, seg, geo, nverts,
                                                      dx, (R*)cover, (R*)local_x, (R*)local_y, (R*)amp);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_segment_compose(pb_handle_t hh, int dtype, int ny, int nx, int tiles_y, int tiles_x, const int* tile_ptr,
                                  const int* tile_seg, const long long* seg, const void* masks, const void* bases, int nmodes,
                                  const double* coefs, long long coef_stride, int ncoef, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || nmodes < 0 || ncoef < 0 || coef_stride < nmodes) return fail(h, PB_ERR_INVALID, "bad compose arguments");
    const int nt = tile_count(ny, nx, tiles_y, tiles_x);
    if (nt < 0) return fail(h, PB_ERR_INVALID, "tile grid does not match the array");
    if (!tile_ptr || !tile_seg || !seg || !masks || !out || (nmodes > 0 && ncoef > 0 && (!bases || !coefs)))
        return fail(h, PB_ERR_INVALID, "null pointer");
    if (ncoef == 0 || nmodes == 0) return PB_OK;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        segment_compose_kernel<R><<<nt, kThreads, 0, st>>>(ny, nx, tiles_x, tile_ptr, tile_seg, seg, (const R*)masks, (const R*)bases,
                                                           nmodes, coefs, coef_stride, ncoef, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_segment_compose_adjoint(pb_handle_t hh, int dtype, int ny, int nx, int nseg, const long long* seg,
                                          const void* masks, const void* bases, int nmodes, const void* opdbar, int nchunk,
                                          void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || nseg < 0 || nmodes < 0 || nchunk < 1 || nseg > 65535)
        return fail(h, PB_ERR_INVALID, "bad compose adjoint arguments");
    if ((long long)nseg * nmodes == 0) return PB_OK;
    if (!seg || !masks || !bases || !opdbar || !out) return fail(h, PB_ERR_INVALID, "null pointer");
    double* partial = nullptr;
    PB_TRY(ensure_scratch(h, FOLD_SLOT, (size_t)nseg * nchunk * nmodes * sizeof(double), (void**)&partial));
    const dim3 grid(nchunk, nseg);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        segment_adjoint_partial_kernel<R><<<grid, kThreads, 0, st>>>(nx, seg, (const R*)masks, (const R*)bases, nmodes,
                                                                     (const R*)opdbar, nchunk, partial);
    });
    PB_LAUNCH_CHECK(h);
    const int n = nseg * nmodes, g = (n + 255) / 256;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        segment_adjoint_final_kernel<R><<<g, 256, 0, st>>>(nseg, nmodes, nchunk, partial, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
