// Shack-Hartmann sensing (prysm/x/shack_hartmann.py): the lenslet-array phase screen, per-subaperture spot centroids
// and the modal reconstructor's batched GEMV.
//
// The screen reproduces the reference's loop over lenslets bit for bit at fp64: every sample sums the phase of the
// lenslets whose window covers it and whose aperture mask admits it, in the reference's order (lenslet row outer,
// column inner), with no fused multiply-add, and forms the exponential in the same pass.  The windows are separable,
// so the host hands over, per grid column and per grid row, the contiguous range of lenslets whose window covers it.
//
// The centroid and reconstruction passes accumulate in fp64 with fixed-order reductions and no atomics, so repeated
// calls are bit-identical; nothing synchronises with the host, so every call can be captured in a CUDA graph.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace pb {

namespace {

constexpr int kThreads = 256;
constexpr int kCentroidVec = 4;                    // grid columns per thread of a centroid CTA when rows allow it
constexpr size_t kCentroidSmemMax = 48 * 1024;     // dynamic shared memory of a centroid CTA without opt-in

// ---- pb_lenslet_screen ---------------------------------------------------------------------------------------------
struct ApertureParams { double v[4]; };            // half-width, half-height, angle (rad), lenslet r^2

__device__ inline bool lenslet_admits(int kind, const ApertureParams& p, double lx, double ly, double rsq) {
    switch (kind) {
        case PB_LENSLET_RECT:                       // angle 0: rectangle_sdf <= 0  <=>  |lx| <= w and |ly| <= h
            return fabs(lx) <= p.v[0] && fabs(ly) <= p.v[1];
        case PB_LENSLET_RECT_SWAP:                  // angle 90: the reference swaps x and y
            return fabs(ly) <= p.v[0] && fabs(lx) <= p.v[1];
        case PB_LENSLET_RECT_ROTATED: {             // cart_to_polar, p += angle, polar_to_cart
            const double r = hypot(lx, ly);
            const double t = __dadd_rn(atan2(ly, lx), p.v[2]);
            double s, c;
            sincos(t, &s, &c);
            return fabs(__dmul_rn(r, c)) <= p.v[0] && fabs(__dmul_rn(r, s)) <= p.v[1];
        }
        default:                                    // circle(pitch^2 / 4, r=rsq): rsq - lenslet_rsq <= 0
            return rsq <= p.v[3];
    }
}

// One thread per sample.  cand_x: per grid column, the first and one-past-last lenslet column whose window covers it;
// cand_y likewise per grid row.  The accumulator has the storage type R and is rounded after every addition, as the
// reference's `total_phase[win] += phase` is.
template <typename R>
__global__ void __launch_bounds__(kThreads) lenslet_screen_kernel(
        const R* __restrict__ x, const R* __restrict__ y, int H, int W, const double* __restrict__ xc,
        const double* __restrict__ yc, const int2* __restrict__ cand_x, const int2* __restrict__ cand_y, int kind,
        ApertureParams p, double two_efl, double kphase, cplx<R>* __restrict__ out) {
    const long long n = (long long)H * W;
    for (long long s = blockIdx.x * (long long)kThreads + threadIdx.x; s < n; s += (long long)gridDim.x * kThreads) {
        const int r = (int)(s / W), c = (int)(s - (long long)r * W);
        const double xv = (double)x[s], yv = (double)y[s];
        const int2 cx = cand_x[c], cy = cand_y[r];
        R acc = 0;
        for (int j = cy.x; j < cy.y; ++j) {
            const double ly = __dsub_rn(yv, yc[j]);
            const double ly2 = __dmul_rn(ly, ly);
            for (int i = cx.x; i < cx.y; ++i) {
                const double lx = __dsub_rn(xv, xc[i]);
                const double rsq = __dadd_rn(__dmul_rn(lx, lx), ly2);
                if (lenslet_admits(kind, p, lx, ly, rsq)) acc = (R)__dadd_rn((double)acc, __ddiv_rn(rsq, two_efl));
            }
        }
        double sn, cs;
        sincos(__dmul_rn(kphase, (double)acc), &sn, &cs);
        out[s] = mk<R>((R)cs, (R)sn);
    }
}

// ---- pb_subaperture_centroids --------------------------------------------------------------------------------------
// One CTA per (lenslet row j, frame f).  It reads the rows of j's band whole: thread t takes grid columns
// c0 + V t .. c0 + V t + V - 1 of each chunk of V kThreads columns, loads them as one vector per row and sums down the
// band, so a warp's load of one row is 32 V contiguous elements (V = 4: 256 bytes of uint16, 512 of float32).  The
// column sums go through shared memory to the lenslet columns, each of which one thread sums in column order, carrying
// its sums from one chunk to the next.  With a threshold a first sweep finds each subaperture's maximum (order-free)
// before the weighted sums.  The sums of a column and of a lenslet do not depend on V, so every V gives the same bits.
// V = 1 serves rows whose length is not a multiple of 4, frames whose start or stride is not aligned to a vector, and
// rows of more than 614 lenslets: the shared memory holds 5 ncols + 3 kThreads V doubles, at most 48 KB, so V = 4 takes
// ncols <= 614 and V = 1 ncols <= 1075; more lenslet columns are refused.
//
// dtab (fp64): x of each grid column [W], y of each grid row [H], lenslet centres xc [ncols], yc [nrows].
// itab (int32): owner lenslet column of each grid column or -1 [W], owned grid-column range of each lenslet column
// [ncols] lo then [ncols] hi, owned grid-row range of each lenslet row [nrows] lo then [nrows] hi.
template <typename T, int V> struct alignas(sizeof(T) * V) Vec { T v[V]; };

template <typename T, typename O, int V>
__global__ void __launch_bounds__(kThreads) centroid_kernel(
        const T* __restrict__ frames, int H, int W, long long fstride, int ncols, int nrows,
        const double* __restrict__ dtab, const int* __restrict__ itab, double threshold, double scale,
        O* __restrict__ disp, O* __restrict__ flux) {
    constexpr int CC = kThreads * V;               // grid columns per chunk
    extern __shared__ double sm[];
    double* acc = sm;                              // [4][ncols]: sum w, sum w x, sum w y, sum I
    double* lmax = acc + 4 * ncols;                // [ncols]
    double* cw = lmax + ncols;                     // [CC] per chunk column: sum w, sum w y, sum I (or max)
    double* cwy = cw + CC;
    double* cI = cwy + CC;
    const int j = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
    const double* xv = dtab;
    const double* yv = xv + W;
    const double* xc = yv + H;
    const double* yc = xc + ncols;
    const int* owner = itab;
    const int* col_lo = owner + W;
    const int* col_hi = col_lo + ncols;
    const int r0 = itab[W + 2 * ncols + j], r1 = itab[W + 2 * ncols + nrows + j];
    const T* F = frames + (long long)f * fstride;

    for (int i = tid; i < ncols; i += kThreads) {
        acc[i] = acc[ncols + i] = acc[2 * ncols + i] = acc[3 * ncols + i] = 0.0;
        lmax[i] = -INFINITY;
    }
    // the lenslet columns that own part of chunk [c0, c0 + CC): lenslet i is summed by thread i % kThreads
    auto reduce_chunk = [&](int c0, bool max_only) {
        __syncthreads();
        for (int i = tid; i < ncols; i += kThreads) {
            const int lo = max(col_lo[i], c0), hi = min(col_hi[i], c0 + CC);
            if (lo >= hi) continue;
            if (max_only) {
                double m = lmax[i];
                for (int c = lo; c < hi; ++c) m = fmax(m, cw[c - c0]);
                lmax[i] = m;
            } else {
                double sw = acc[i], swx = acc[ncols + i], swy = acc[2 * ncols + i], sI = acc[3 * ncols + i];
                for (int c = lo; c < hi; ++c) {
                    const double w = cw[c - c0];
                    sw += w;
                    swx += w * xv[c];
                    swy += cwy[c - c0];
                    sI += cI[c - c0];
                }
                acc[i] = sw; acc[ncols + i] = swx; acc[2 * ncols + i] = swy; acc[3 * ncols + i] = sI;
            }
        }
        __syncthreads();
    };
    // W is a multiple of V, so a thread's V columns are all inside the row or all past it
    auto load = [&](int r, int cb) { return *reinterpret_cast<const Vec<T, V>*>(F + (long long)r * W + cb); };
    if (threshold != 0.0) {
        for (int c0 = 0; c0 < W; c0 += CC) {
            const int cb = c0 + tid * V;
            double m[V];
            bool own[V];
#pragma unroll
            for (int k = 0; k < V; ++k) {
                m[k] = -INFINITY;
                own[k] = cb < W && owner[cb + k] >= 0;
            }
            if (cb < W) {
#pragma unroll 4
                for (int r = r0; r < r1; ++r) {
                    const Vec<T, V> q = load(r, cb);
#pragma unroll
                    for (int k = 0; k < V; ++k)
                        if (own[k]) m[k] = fmax(m[k], (double)q.v[k]);
                }
            }
#pragma unroll
            for (int k = 0; k < V; ++k) cw[tid * V + k] = m[k];
            reduce_chunk(c0, true);
        }
    }
    for (int c0 = 0; c0 < W; c0 += CC) {
        const int cb = c0 + tid * V;
        double sw[V], swy[V], sI[V], t[V];
        bool own[V];
#pragma unroll
        for (int k = 0; k < V; ++k) {
            sw[k] = swy[k] = sI[k] = 0.0;
            const int o = cb < W ? owner[cb + k] : -1;
            own[k] = o >= 0;
            t[k] = own[k] && threshold != 0.0 ? threshold * lmax[o] : 0.0;
        }
        if (cb < W) {
#pragma unroll 4
            for (int r = r0; r < r1; ++r) {
                const Vec<T, V> q = load(r, cb);
                const double yr = yv[r];
#pragma unroll
                for (int k = 0; k < V; ++k) {
                    if (!own[k]) continue;
                    const double v = (double)q.v[k];
                    const double d = v - t[k];
                    const double w = d > 0.0 ? d : (d != d ? d : 0.0);     // numpy's maximum(I - t, 0): NaN propagates
                    sI[k] += v;
                    sw[k] += w;
                    swy[k] += w * yr;
                }
            }
        }
#pragma unroll
        for (int k = 0; k < V; ++k) {
            cw[tid * V + k] = sw[k];
            cwy[tid * V + k] = swy[k];
            cI[tid * V + k] = sI[k];
        }
        reduce_chunk(c0, false);
    }
    const long long plane = (long long)nrows * ncols;
    for (int i = tid; i < ncols; i += kThreads) {
        const double sw = acc[i];
        const long long o = (long long)j * ncols + i;
        const bool empty = sw == 0.0;
        disp[(2 * f) * plane + o] = (O)(empty ? NAN : (acc[ncols + i] / sw - xc[i]) * scale);
        disp[(2 * f + 1) * plane + o] = (O)(empty ? NAN : (acc[2 * ncols + i] / sw - yc[j]) * scale);
        flux[f * plane + o] = (O)acc[3 * ncols + i];
    }
}

// ---- pb_sh_reconstruct ---------------------------------------------------------------------------------------------
// One CTA per (mode k, frame f): a strided fp64 dot product over the M valid slopes, then a fixed-shape tree.
template <typename S>
__global__ void __launch_bounds__(kThreads) reconstruct_kernel(
        const S* __restrict__ slopes, long long fstride, const int* __restrict__ idx, const double* __restrict__ ref,
        const double* __restrict__ R, int K, int M, S* __restrict__ out) {
    __shared__ double part[kThreads];
    const int k = blockIdx.x, f = blockIdx.y, tid = threadIdx.x;
    const S* s = slopes + (long long)f * fstride;
    const double* row = R + (long long)k * M;
    double a = 0.0;
    for (int m = tid; m < M; m += kThreads) {
        double v = (double)s[idx[m]];
        if (ref) v -= ref[m];
        a += row[m] * v;
    }
    a = tree_sum<kThreads>(a, part);
    if (tid == 0) out[(long long)f * K + k] = (S)a;
}

}  // namespace

}  // namespace pb

using namespace pb;

extern "C" int pb_lenslet_screen(pb_handle_t hh, int dtype, const void* x, const void* y, int H, int W, int ncols,
                                 int nrows, const double* centres, const int* cand, int kind, const double* params_host,
                                 double two_efl, double kphase, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (H < 0 || W < 0 || ncols < 0 || nrows < 0 || kind < PB_LENSLET_RECT || kind > PB_LENSLET_CIRCLE)
        return fail(h, PB_ERR_INVALID, "bad lenslet screen arguments");
    if ((long long)H * W == 0) return PB_OK;
    if (!x || !y || !cand || !out || !params_host || (ncols * nrows > 0 && !centres))
        return fail(h, PB_ERR_INVALID, "null pointer");
    ApertureParams p{};
    std::copy(params_host, params_host + 4, p.v);
    const int2* cx = reinterpret_cast<const int2*>(cand);
    const int2* cy = cx + W;
    const int grid = grid_for((long long)H * W, kThreads, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        lenslet_screen_kernel<R><<<grid, kThreads, 0, st>>>((const R*)x, (const R*)y, H, W, centres, centres + ncols, cx, cy, kind,
                                                            p, two_efl, kphase, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_subaperture_centroids(pb_handle_t hh, int frame_type, const void* frames, int nframes, int H, int W,
                                        long long frame_stride, int ncols, int nrows, const double* dtab,
                                        const int* itab, double threshold, double scale, int out_type, void* disp,
                                        void* flux, void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool type_ok = frame_type == PB_ELEM_F32 || frame_type == PB_ELEM_F64 || frame_type == PB_ELEM_U16 ||
                         frame_type == PB_ELEM_I32;
    if (!type_ok || nframes < 0 || H < 0 || W < 0 || ncols < 0 || nrows < 0 || frame_stride < (long long)H * W ||
        !std::isfinite(threshold) || !std::isfinite(scale))
        return fail(h, PB_ERR_INVALID, "bad centroid arguments");
    if (out_type != (frame_type == PB_ELEM_F64 ? PB_ELEM_F64 : PB_ELEM_F32))
        return fail(h, PB_ERR_INVALID, "centroids are float64 for float64 frames and float32 otherwise");
    if (nframes == 0 || ncols == 0 || nrows == 0) return PB_OK;
    if (nrows > 65535) return fail(h, PB_ERR_UNSUPPORTED, "more than 65535 lenslet rows");
    if (nframes > 65535) return fail(h, PB_ERR_UNSUPPORTED, "more than 65535 frames in one call");
    if (!frames || !dtab || !itab || !disp || !flux) return fail(h, PB_ERR_INVALID, "null pointer");
    const size_t fsz = elem_size(frame_type), vbytes = fsz * kCentroidVec;
    auto smem_for = [&](int v) { return (5 * (size_t)ncols + 3 * (size_t)kThreads * v) * sizeof(double); };
    const bool vec = W % kCentroidVec == 0 && reinterpret_cast<uintptr_t>(frames) % vbytes == 0 &&
                     (frame_stride * fsz) % vbytes == 0 && smem_for(kCentroidVec) <= kCentroidSmemMax;
    const size_t smem = smem_for(vec ? kCentroidVec : 1);
    if (smem > kCentroidSmemMax) return fail(h, PB_ERR_UNSUPPORTED, "too many lenslet columns");
    const dim3 grid(nrows, nframes);
    with_elem(frame_type, [&](auto t) {
        using T = decltype(t);
        if constexpr (is_one_of<T, float, double, uint16_t, int32_t>) {
            using O = std::conditional_t<std::is_same<T, double>::value, double, float>;
            if (vec)
                centroid_kernel<T, O, kCentroidVec><<<grid, kThreads, smem, st>>>(
                    (const T*)frames, H, W, frame_stride, ncols, nrows, dtab, itab, threshold, scale, (O*)disp, (O*)flux);
            else
                centroid_kernel<T, O, 1><<<grid, kThreads, smem, st>>>(
                    (const T*)frames, H, W, frame_stride, ncols, nrows, dtab, itab, threshold, scale, (O*)disp, (O*)flux);
        }
    });
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_CENTROID, vec ? kCentroidVec : 1, frame_type)]++;
    return PB_OK;
}

extern "C" int pb_sh_reconstruct(pb_handle_t hh, int dtype, const void* slopes, int nframes, long long frame_stride,
                                 const int* idx, const double* ref, const double* R, int K, int M, void* out,
                                 void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (dtype != PB_ELEM_F32 && dtype != PB_ELEM_F64) return fail(h, PB_ERR_INVALID, "slopes must be float32 or float64");
    if (nframes < 0 || K < 0 || M < 0 || frame_stride < 0) return fail(h, PB_ERR_INVALID, "bad reconstruct sizes");
    if (nframes == 0 || K == 0) return PB_OK;
    if (nframes > 65535) return fail(h, PB_ERR_UNSUPPORTED, "more than 65535 frames in one call");
    if (!slopes || !out || (M > 0 && (!idx || !R))) return fail(h, PB_ERR_INVALID, "null pointer");
    const dim3 grid(K, nframes);
    with_elem(dtype, [&](auto t) {
        using T = decltype(t);
        if constexpr (std::is_floating_point<T>::value)
            reconstruct_kernel<T><<<grid, kThreads, 0, st>>>((const T*)slopes, frame_stride, idx, ref, R, K, M, (T*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
