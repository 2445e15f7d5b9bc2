// Interferometric metrology (prysm/interferogram.py, prysm/util.py mean / pv / rms / Sa / std and
// prysm/polynomials/fitting.py lstsq): NaN-aware statistics, the masked Gram reduction of a least-squares fit, the PSD
// prologue and epilogue around pb_fft2, the band-limited trapezoid, the radial filter, the gradient, the finite
// bounding box and the masked writes of the Interferogram methods.
//
// Every reduction accumulates in fp64 and combines its blocks with the grid fold of common.cuh (DESIGN.md §4.4), so
// repeated calls give the same bits.
#include <math_constants.h>

#include "common.cuh"

namespace pb {

constexpr int MET_THREADS = 256;
constexpr int MET_TILE = 32;                 // pixels per shared-memory tile of the Gram kernel
constexpr int MET_TILE_LD = MET_TILE + 1;    // its row stride: threads with consecutive (i, j) read different banks
constexpr int MET_GRAM_PER_THREAD = (PB_GRAM_MAX_K + 1) * (PB_GRAM_MAX_K + 2) / 2 / MET_THREADS + 1;

// ---- statistics -------------------------------------------------------------------------------------------------
// pass 1: count, sum, min, max, sum of squares of the finite values, NaN count -> res[0..5]; res[6] = mean
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) stats_pass1_kernel(const T* __restrict__ x, long long n, double* part,
                                                                  unsigned* counter, double* res) {
    double v[4] = {0.0, 0.0, 0.0, 0.0};   // count, sum, sumsq, nan count
    double mn = CUDART_INF, mx = -CUDART_INF;
    PB_GRID_STRIDE(i, n) {
        const double a = (double)x[i];
        if (isfinite(a)) {
            v[0] += 1.0; v[1] += a; v[2] = fma(a, a, v[2]);
            mn = fmin(mn, a); mx = fmax(mx, a);
        } else if (isnan(a)) {
            v[3] += 1.0;
        }
    }
    block_reduce<MET_THREADS>(v, OpAdd{});
    mn = block_reduce<MET_THREADS>(mn, OpMin{});
    mx = block_reduce<MET_THREADS>(mx, OpMax{});
    if (threadIdx.x == 0) {
        double* p = part + (size_t)blockIdx.x * 6;
        p[0] = v[0]; p[1] = v[1]; p[2] = mn; p[3] = mx; p[4] = v[2]; p[5] = v[3];
    }
    if (!arrive_last(counter)) return;
    double r[6];
    r[0] = fold_partials<MET_THREADS, 6>(part, 0, OpAdd{}, 0.0);
    r[1] = fold_partials<MET_THREADS, 6>(part, 1, OpAdd{}, 0.0);
    r[2] = fold_partials<MET_THREADS, 6>(part, 2, OpMin{}, CUDART_INF);
    r[3] = fold_partials<MET_THREADS, 6>(part, 3, OpMax{}, -CUDART_INF);
    r[4] = fold_partials<MET_THREADS, 6>(part, 4, OpAdd{}, 0.0);
    r[5] = fold_partials<MET_THREADS, 6>(part, 5, OpAdd{}, 0.0);
    if (threadIdx.x == 0) {
        for (int k = 0; k < 6; ++k) res[k] = r[k];
        res[6] = r[1] / r[0];
        *counter = 0;
    }
}

// pass 2: sum |x - mean| and sum (x - mean)^2 over the finite values, mean read from res[6] -> res[7], res[8]
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) stats_pass2_kernel(const T* __restrict__ x, long long n, double* part,
                                                                  unsigned* counter, double* res) {
    const double m = res[6];
    double v[2] = {0.0, 0.0};
    PB_GRID_STRIDE(i, n) {
        const double a = (double)x[i];
        if (isfinite(a)) {
            const double d = a - m;
            v[0] += fabs(d); v[1] = fma(d, d, v[1]);
        }
    }
    block_reduce<MET_THREADS>(v, OpAdd{});
    if (threadIdx.x == 0) { part[(size_t)blockIdx.x * 2] = v[0]; part[(size_t)blockIdx.x * 2 + 1] = v[1]; }
    if (!arrive_last(counter)) return;
    const double s0 = fold_partials<MET_THREADS, 2>(part, 0, OpAdd{}, 0.0);
    const double s1 = fold_partials<MET_THREADS, 2>(part, 1, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { res[7] = s0; res[8] = s1; *counter = 0; }
}

// ---- masked Gram reduction -------------------------------------------------------------------------------------
struct GramModes { const void* p[PB_GRAM_MAX_K]; };

// the (i, j) of packed upper-triangle index o of a (k x k) matrix, row-major
__device__ inline void tri_ij(int o, int k, int& i, int& j) {
    i = 0;
    while (o >= k - i) { o -= k - i; ++i; }
    j = i + o;
}

// column K of the augmented matrix is the data; a pixel whose data is not finite contributes nothing.  A NULL mode is
// the constant 1.  out (packed upper triangle of the (K+1) x (K+1) matrix [A d]^T [A d], fp64).
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) gram_kernel(GramModes modes, int K, const T* __restrict__ d, long long n,
                                                           double* part, unsigned* counter, double* out) {
    extern __shared__ double tile[];          // (K + 1) x MET_TILE, rows MET_TILE_LD apart
    const int K1 = K + 1, P = K1 * (K1 + 1) / 2;
    int oi[MET_GRAM_PER_THREAD], oj[MET_GRAM_PER_THREAD];
    double acc[MET_GRAM_PER_THREAD];
#pragma unroll
    for (int q = 0; q < MET_GRAM_PER_THREAD; ++q) {
        const int o = threadIdx.x + q * MET_THREADS;
        oi[q] = oj[q] = 0;
        if (o < P) tri_ij(o, K1, oi[q], oj[q]);
        acc[q] = 0.0;
    }
    const long long ntiles = (n + MET_TILE - 1) / MET_TILE;
    for (long long t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const long long p0 = t * MET_TILE;
        __syncthreads();
        for (int e = threadIdx.x; e < K1 * MET_TILE; e += MET_THREADS) {
            const int k = e / MET_TILE, p = e % MET_TILE;
            const long long i = p0 + p;
            double v = 0.0;
            if (i < n) {
                const double dv = (double)d[i];
                if (isfinite(dv)) v = k == K ? dv : (modes.p[k] ? (double)((const T*)modes.p[k])[i] : 1.0);
            }
            tile[k * MET_TILE_LD + p] = v;
        }
        __syncthreads();
#pragma unroll
        for (int q = 0; q < MET_GRAM_PER_THREAD; ++q) {
            if (threadIdx.x + q * MET_THREADS < P) {
                const double* a = tile + oi[q] * MET_TILE_LD;
                const double* b = tile + oj[q] * MET_TILE_LD;
                double s = acc[q];
#pragma unroll 8
                for (int p = 0; p < MET_TILE; ++p) s = fma(a[p], b[p], s);
                acc[q] = s;
            }
        }
    }
#pragma unroll
    for (int q = 0; q < MET_GRAM_PER_THREAD; ++q) {
        const int o = threadIdx.x + q * MET_THREADS;
        if (o < P) part[(size_t)blockIdx.x * P + o] = acc[q];
    }
    if (!arrive_last(counter)) return;
    for (int o = threadIdx.x; o < P; o += MET_THREADS) {
        double s = 0.0;
        for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(part + (size_t)b * P + o);
        out[o] = s;
    }
    if (threadIdx.x == 0) *counter = 0;
}

// ---- PSD ----------------------------------------------------------------------------------------------------------
// the four corner rectangles of the automatic window choice: (y0, y1, x0, x1) each
struct PbRect4 { int v[16]; };

// flag[c] = 1 when every sample of corner rectangle c is == 0 (a NaN is not); one block per corner
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) corners_kernel(const T* __restrict__ x, int nx, PbRect4 rect, int* flag) {
    const int* r = rect.v + 4 * blockIdx.x;
    const int h = r[1] - r[0], w = r[3] - r[2];
    double nz = 0.0;
    for (long long e = threadIdx.x; e < (long long)h * w; e += MET_THREADS) {
        const T v = x[(long long)(r[0] + e / w) * nx + r[2] + e % w];
        if (!(v == T(0))) nz = 1.0;
    }
    nz = block_reduce<MET_THREADS>(nz, OpMax{});
    if (threadIdx.x == 0) flag[blockIdx.x] = nz == 0.0;
}

__device__ inline double hanning(int k, int n) {
    if (n == 1) return 1.0;
    return 0.5 + 0.5 * cos(__ddiv_rn(__dmul_rn(CUDART_PI, (double)(2 * k + 1 - n)), (double)(n - 1)));
}

// w at (i, j): Welch from r = hypot(x, y) on the fftrange * dx grid, the Hann outer product, or a user array.  With
// PB_WIN_AUTO the corner flags pick Welch when all four corners are zero, else Hann.
template <typename T>
__device__ inline double window_at(int kind, const int* flag, const T* user, int i, int j, int ny, int nx, double dx,
                                   double alpha, double rmax) {
    if (kind == PB_WIN_AUTO) kind = (flag[0] && flag[1] && flag[2] && flag[3]) ? PB_WIN_WELCH : PB_WIN_HANN;
    if (kind == PB_WIN_USER) return (double)user[(long long)i * nx + j];
    if (kind == PB_WIN_HANN) return __dmul_rn(hanning(i, ny), hanning(j, nx));
    const double xx = __dmul_rn((double)(j - nx / 2), dx), yy = __dmul_rn((double)(i - ny / 2), dx);
    return __dadd_rn(1.0, -pow(fabs(__ddiv_rn(hypot(xx, yy), rmax)), alpha));
}

// shifted[k] = fftshift(height * w)[k] (real, T) and/or window[k] = w[k] (T); S2 = sum w^2 -> res[0]
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) psd_prologue_kernel(const T* __restrict__ height, int ny, int nx, int kind,
                                                                   const T* __restrict__ user, double dx, double alpha,
                                                                   double rmax, int* flag, T* shifted, T* window,
                                                                   double* part, unsigned* counter, double* res) {
    const long long n = (long long)ny * nx;
    double s2 = 0.0;
    PB_GRID_STRIDE(e, n) {
        const int i = (int)(e / nx), j = (int)(e % nx);
        const double w = window_at(kind, flag, user, i, j, ny, nx, dx, alpha, rmax);
        s2 = fma(w, w, s2);
        if (window) window[e] = (T)w;
        if (shifted) {
            const int si = (i + ny / 2) % ny, sj = (j + nx / 2) % nx;     // fftshift: out[si] = in[i]
            shifted[(long long)si * nx + sj] = (T)((double)height[e] * w);
        }
    }
    s2 = block_reduce<MET_THREADS>(s2, OpAdd{});
    if (threadIdx.x == 0) part[blockIdx.x] = s2;
    if (!arrive_last(counter)) return;
    const double s = fold_partials<MET_THREADS, 1>(part, 0, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { res[0] = s; *counter = 0; }
}

// psd[k] = |F[ifftshift k]|^2 / (S2 fs^2), S2 read from s2
template <typename R>
__global__ void __launch_bounds__(MET_THREADS) psd_epilogue_kernel(const cplx<R>* __restrict__ F, int ny, int nx,
                                                                   const double* s2, double fs, R* psd) {
    const double coef = s2[0] * fs * fs;
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        const int i = (int)(e / nx), j = (int)(e % nx);
        const int si = (i + ny / 2) % ny, sj = (j + nx / 2) % nx;       // ifftshift: out[i] = in[si]
        const cplx<R> v = F[(long long)si * nx + sj];
        const double a = hypot((double)v.x, (double)v.y);
        psd[e] = (R)(__dmul_rn(a, a) / coef);
    }
}

// ---- band-limited trapezoid ---------------------------------------------------------------------------------------
// hypot(x, y) rounded as a correctly rounded hypot rounds it (numpy's np.hypot on the host): x^2 + y^2 in double-double,
// then one Newton correction of its square root.  The band edges compare r with limits such as r.max() itself, so
// CUDA's hypot, good to 2 ulp, would move samples across them.
__device__ inline double hypot_cr(double x, double y) {
    const double xx = __dmul_rn(x, x), ex = fma(x, x, -xx);
    const double yy = __dmul_rn(y, y), ey = fma(y, y, -yy);
    const double s = __dadd_rn(xx, yy), bb = __dadd_rn(s, -xx);
    const double lo = __dadd_rn(__dadd_rn(__dadd_rn(xx, -__dadd_rn(s, -bb)), __dadd_rn(yy, -bb)), __dadd_rn(ex, ey));
    const double r = sqrt(s);
    if (r == 0.0) return 0.0;
    return __dadd_rn(r, __dadd_rn(fma(-r, r, s), lo) / (2.0 * r));
}

__device__ inline double trapz_w(int i, int n) { return n < 2 ? 0.0 : ((i == 0 || i == n - 1) ? 0.5 : 1.0); }

// res[0] = sum_ij wy_i wx_j psd_ij over flow <= r_ij <= fhigh, r from the array r or hypot(fx[j], fy[i]);
// twod = 0: one trapezoid along the ny axis (nx == 1)
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) band_trapz_kernel(const T* __restrict__ psd, const T* __restrict__ r,
                                                                 const double* fx, const double* fy, int ny, int nx,
                                                                 int twod, double flow, double fhigh, double* part,
                                                                 unsigned* counter, double* res) {
    double s = 0.0;
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        const int i = (int)(e / nx), j = (int)(e % nx);
        const double rr = r ? (double)r[e] : hypot_cr(fx[j], fy[i]);
        if (rr < flow || rr > fhigh) continue;
        const double w = trapz_w(i, ny) * (twod ? trapz_w(j, nx) : 1.0);
        if (w != 0.0) s = fma(w, (double)psd[e], s);
    }
    s = block_reduce<MET_THREADS>(s, OpAdd{});
    if (threadIdx.x == 0) part[blockIdx.x] = s;
    if (!arrive_last(counter)) return;
    const double t = fold_partials<MET_THREADS, 1>(part, 0, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { res[0] = t; *counter = 0; }
}

// ---- radial filter ------------------------------------------------------------------------------------------------
__device__ inline double met_jinc(double u) { return (u < 1e-8 && u > -1e-8) ? 0.5 : j1(u) / u; }

// hann2d(ny, nx): cos(pi / min(ny, nx) * hypot(n, m))^2, 0 beyond min // 2
__device__ inline double hann2d_at(int i, int j, int ny, int nx) {
    const int nm = min(ny, nx);
    const double nn = hypot((double)(j - nx / 2), (double)(i - ny / 2));
    if (nn > (double)(nm / 2)) return 0.0;
    const double c = cos(__dmul_rn(__ddiv_rn(CUDART_PI, (double)nm), nn));
    return __dmul_rn(c, c);
}

// ideal_lpf_iir2d(r, dx, fcn) = jinc(r pi fcn / dx) fcn^2 pi / 2
__device__ inline double lpf_at(double r, double dx, double fcn) {
    const double c = __ddiv_rn(__dmul_rn(CUDART_PI, fcn), dx);
    return __dmul_rn(met_jinc(__dmul_rn(r, c)), __dmul_rn(__dmul_rn(fcn, fcn), CUDART_PI) / 2.0);
}

// out0 (and out1 with fcn1) = the product of the factors `parts` asks for (PB_FILT_W hann2d, PB_FILT_H the ideal
// low-pass response at r); a missing factor is 1
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) filter_h_kernel(const T* __restrict__ r, int ny, int nx, int parts, double dx,
                                                               double fcn0, double fcn1, T* out0, T* out1) {
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        const int i = (int)(e / nx), j = (int)(e % nx);
        const double w = (parts & PB_FILT_W) ? hann2d_at(i, j, ny, nx) : 1.0;
        if (parts & PB_FILT_H) {
            const double rr = (double)r[e];
            out0[e] = (T)(parts & PB_FILT_W ? __dmul_rn(w, lpf_at(rr, dx, fcn0)) : lpf_at(rr, dx, fcn0));
            if (out1) out1[e] = (T)(parts & PB_FILT_W ? __dmul_rn(w, lpf_at(rr, dx, fcn1)) : lpf_at(rr, dx, fcn1));
        } else {
            out0[e] = (T)w;
        }
    }
}

// H from |Hl| (and |Hh|) by typ; D *= H in place, or with D NULL H into Hout
template <typename R>
__global__ void __launch_bounds__(MET_THREADS) filter_apply_kernel(cplx<R>* D, const cplx<R>* __restrict__ Hl,
                                                                   const cplx<R>* __restrict__ Hh, long long n, int typ,
                                                                   R* Hout) {
    PB_GRID_STRIDE(e, n) {
        const R l = hypot(Hl[e].x, Hl[e].y);
        R H;
        if (typ == PB_FILT_LOWPASS) H = l;
        else if (typ == PB_FILT_HIGHPASS) H = R(1) - l;
        else {
            const R hh = R(1) - hypot(Hh[e].x, Hh[e].y);
            H = typ == PB_FILT_BANDPASS ? R(1) - (hh + l) : hh + l;
        }
        if (D) { D[e].x *= H; D[e].y *= H; }
        else Hout[e] = H;
    }
}

// ---- gradient ---------------------------------------------------------------------------------------------------
// np.gradient(f, dx): central differences inside, one-sided first order on the edges; gx along rows, gy along columns
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) gradient_kernel(const T* __restrict__ f, int ny, int nx, double dx, T* gx,
                                                               T* gy, T* gr) {
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        const int i = (int)(e / nx), j = (int)(e % nx);
        double a, b;
        if (j == 0) a = ((double)f[e + 1] - (double)f[e]) / dx;
        else if (j == nx - 1) a = ((double)f[e] - (double)f[e - 1]) / dx;
        else a = ((double)f[e + 1] - (double)f[e - 1]) / (2.0 * dx);
        if (i == 0) b = ((double)f[e + nx] - (double)f[e]) / dx;
        else if (i == ny - 1) b = ((double)f[e] - (double)f[e - nx]) / dx;
        else b = ((double)f[e + nx] - (double)f[e - nx]) / (2.0 * dx);
        const T ta = (T)a, tb = (T)b;
        gx[e] = ta; gy[e] = tb;
        gr[e] = (T)hypot((double)ta, (double)tb);
    }
}

// ---- finite bounding box -----------------------------------------------------------------------------------------
// box (4 ints, zero on entry): max (ny - i), max (i + 1), max (nx - j), max (j + 1) over finite samples
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) finite_bounds_kernel(const T* __restrict__ x, int ny, int nx, int* box) {
    int b[4] = {0, 0, 0, 0};
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        if (!isfinite((double)x[e])) continue;
        const int i = (int)(e / nx), j = (int)(e % nx);
        b[0] = max(b[0], ny - i); b[1] = max(b[1], i + 1); b[2] = max(b[2], nx - j); b[3] = max(b[3], j + 1);
    }
    for (int k = 0; k < 4; ++k) {
        int v = b[k];
        for (int o = 16; o; o >>= 1) v = max(v, __shfl_down_sync(0xffffffffu, v, o));
        if ((threadIdx.x & 31) == 0 && v) atomicMax(box + k, v);
    }
}

// ---- masked writes ----------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(MET_THREADS) pointwise_kernel(int op, const T* __restrict__ x, const T* __restrict__ u,
                                                                const T* __restrict__ v, const uint8_t* __restrict__ m,
                                                                int ny, int nx, double a, double b, T* out) {
    const T nan = (T)CUDART_NAN;
    PB_GRID_STRIDE(e, (long long)ny * nx) {
        switch (op) {
            case PB_PW_FILL: out[e] = isnan((double)x[e]) ? (T)a : x[e]; break;
            case PB_PW_KEEP: out[e] = m[e] ? x[e] : nan; break;
            case PB_PW_CLIP: out[e] = fabs((double)x[e]) > a ? nan : x[e]; break;
            case PB_PW_RADIUS: out[e] = (double)u[e] / a > 1.0 ? nan : x[e]; break;
            case PB_PW_SUB: {
                const double p = __dadd_rn(__dmul_rn(a, u ? (double)u[e] : 1.0), v ? __dmul_rn(b, (double)v[e]) : 0.0);
                out[e] = (T)__dadd_rn((double)x[e], -p);
                break;
            }
            case PB_PW_RHO2: {
                const int i = (int)(e / nx), j = (int)(e % nx);
                // np.linspace(-1, 1, n): j * step - 1, the last sample exactly 1; a, b = the x and y steps 2 / (n - 1)
                const double xx = nx == 1 ? -1.0 : (j == nx - 1 ? 1.0 : __dadd_rn(__dmul_rn((double)j, a), -1.0));
                const double yy = ny == 1 ? -1.0 : (i == ny - 1 ? 1.0 : __dadd_rn(__dmul_rn((double)i, b), -1.0));
                const double rho = sqrt(__dadd_rn(__dmul_rn(xx, xx), __dmul_rn(yy, yy)));
                out[e] = (T)__dmul_rn(rho, rho);
                break;
            }
            case PB_PW_REAL: out[e] = x[2 * e]; break;
            case PB_PW_AXPBY:
                out[e] = (T)__dadd_rn(__dmul_rn(a, (double)u[e]), v ? __dmul_rn(b, (double)v[e]) : 0.0);
                break;
            case PB_PW_DIV: out[e] = (T)((double)x[e] / a); break;
            case PB_PW_WELCH: out[e] = (T)__dadd_rn(1.0, -pow(fabs((double)x[e] / a), b)); break;
        }
    }
}

}  // namespace pb

using namespace pb;

extern "C" int pb_nan_stats(pb_handle_t hh, int dtype, const void* x, long long n, double* res, void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !res || n < 0) return fail(h, PB_ERR_INVALID, "pb_nan_stats: null array or negative count");
    const int blocks = fold_blocks(n, h->sm_count);
    double* part; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, blocks, 6, st, &part, &counter));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        stats_pass1_kernel<R><<<blocks, MET_THREADS, 0, st>>>((const R*)x, n, part, counter, res);
        stats_pass2_kernel<R><<<blocks, MET_THREADS, 0, st>>>((const R*)x, n, part, counter, res);
    });
    PB_LAUNCH_CHECK(h);
    h->launches++;
    return PB_OK;
}

extern "C" int pb_masked_gram(pb_handle_t hh, int dtype, const void* const* modes, int k, const void* data, long long n,
                              double* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (k < 1 || k > PB_GRAM_MAX_K)
        return fail(h, PB_ERR_INVALID, "pb_masked_gram: k must be in [1, " + std::to_string(PB_GRAM_MAX_K) + "]");
    if (!modes || !data || !out || n < 1) return fail(h, PB_ERR_INVALID, "pb_masked_gram: null array or empty data");
    GramModes gm{};
    for (int q = 0; q < k; ++q) gm.p[q] = modes[q];
    const int P = (k + 1) * (k + 2) / 2;
    const int blocks = std::max(1, std::min<int>((int)((n + MET_TILE - 1) / MET_TILE), 2 * h->sm_count));
    double* part; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, blocks, P, st, &part, &counter));
    const size_t smem = (size_t)(k + 1) * MET_TILE_LD * sizeof(double);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        gram_kernel<R><<<blocks, MET_THREADS, smem, st>>>(gm, k, (const R*)data, n, part, counter, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_psd_prologue(pb_handle_t hh, int dtype, const void* height, int ny, int nx, int kind, const void* user,
                               double dx, double alpha, double rmax, const int* corners, void* shifted, void* window,
                               double* s2, int* flags, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || kind < PB_WIN_AUTO || kind > PB_WIN_USER || (kind == PB_WIN_USER && !user) ||
        (shifted && !height) || !s2 || !flags || (kind == PB_WIN_AUTO && !corners))
        return fail(h, PB_ERR_INVALID, "pb_psd_prologue: bad shape, window kind or missing array");
    const long long n = (long long)ny * nx;
    const int blocks = fold_blocks(n, h->sm_count);
    double* part; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, blocks, 1, st, &part, &counter));
    PbRect4 rect{};
    if (corners)
        for (int q = 0; q < 16; ++q) rect.v[q] = corners[q];
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        if (kind == PB_WIN_AUTO) {
            corners_kernel<R><<<4, MET_THREADS, 0, st>>>((const R*)height, nx, rect, flags);
            h->launches++;
        }
        psd_prologue_kernel<R><<<blocks, MET_THREADS, 0, st>>>((const R*)height, ny, nx, kind, (const R*)user, dx, alpha,
                                                               rmax, flags, (R*)shifted, (R*)window, part, counter, s2);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_psd_epilogue(pb_handle_t hh, int dtype, const void* F, int ny, int nx, const double* s2, double fs,
                               void* psd, void* stream) {
    PB_ENTER_REAL(hh);
    if (!F || !psd || !s2 || ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "pb_psd_epilogue: null array or bad shape");
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        psd_epilogue_kernel<R><<<grid_for((long long)ny * nx, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            (const cplx<R>*)F, ny, nx, s2, fs, (R*)psd);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_band_trapz(pb_handle_t hh, int dtype, const void* psd, const void* r, const double* fx,
                             const double* fy, int ny, int nx, int twod, double flow, double fhigh, double* res,
                             void* stream) {
    PB_ENTER_REAL(hh);
    if (!psd || !res || ny < 1 || nx < 1 || (!r && (!fx || !fy)))
        return fail(h, PB_ERR_INVALID, "pb_band_trapz: null array or bad shape");
    const long long n = (long long)ny * nx;
    const int blocks = fold_blocks(n, h->sm_count);
    double* part; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, blocks, 1, st, &part, &counter));
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        band_trapz_kernel<R><<<blocks, MET_THREADS, 0, st>>>((const R*)psd, (const R*)r, fx, fy, ny, nx, twod, flow, fhigh,
                                                             part, counter, res);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_filter_h(pb_handle_t hh, int dtype, const void* r, int ny, int nx, int parts, double dx, double fcn0,
                           double fcn1, void* out0, void* out1, void* stream) {
    PB_ENTER_REAL(hh);
    if (!out0 || ny < 1 || nx < 1 || !(parts & (PB_FILT_W | PB_FILT_H)) || ((parts & PB_FILT_H) && !r))
        return fail(h, PB_ERR_INVALID, "pb_filter_h: null array, bad shape or no factor");
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        filter_h_kernel<R><<<grid_for((long long)ny * nx, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            (const R*)r, ny, nx, parts, dx, fcn0, fcn1, (R*)out0, (R*)out1);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_filter_apply(pb_handle_t hh, int dtype, void* D, const void* Hl, const void* Hh, long long n, int typ,
                               void* Hout, void* stream) {
    PB_ENTER_REAL(hh);
    if (typ < PB_FILT_LOWPASS || typ > PB_FILT_BANDREJECT || !Hl || (typ >= PB_FILT_BANDPASS && !Hh) || (!D && !Hout))
        return fail(h, PB_ERR_INVALID, "pb_filter_apply: bad filter type or missing array");
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        filter_apply_kernel<R><<<grid_for(n, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            (cplx<R>*)D, (const cplx<R>*)Hl, (const cplx<R>*)Hh, n, typ, (R*)Hout);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_gradient2d(pb_handle_t hh, int dtype, const void* f, int ny, int nx, double dx, void* gx, void* gy,
                             void* gr, void* stream) {
    PB_ENTER_REAL(hh);
    if (!f || !gx || !gy || !gr || ny < 2 || nx < 2)
        return fail(h, PB_ERR_INVALID, "pb_gradient2d: null array or fewer than 2 samples along an axis");
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        gradient_kernel<R><<<grid_for((long long)ny * nx, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            (const R*)f, ny, nx, dx, (R*)gx, (R*)gy, (R*)gr);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_finite_bounds(pb_handle_t hh, int dtype, const void* x, int ny, int nx, int* box, void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !box || ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "pb_finite_bounds: null array or bad shape");
    void* w = nullptr;
    PB_TRY(ensure_scratch(h, 2, 4 * sizeof(int), &w));
    PB_CUDA(h, cudaMemsetAsync(w, 0, 4 * sizeof(int), st));
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        finite_bounds_kernel<R><<<grid_for((long long)ny * nx, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            (const R*)x, ny, nx, (int*)w);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaMemcpyAsync(box, w, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_metro_pointwise(pb_handle_t hh, int dtype, int op, const void* x, const void* u, const void* v,
                                  const void* m, int ny, int nx, double a, double b, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    const bool needs_x = op != PB_PW_RHO2 && op != PB_PW_AXPBY;
    if (op < PB_PW_FILL || op > PB_PW_WELCH || !out || ny < 1 || nx < 1 || (needs_x && !x) || (op == PB_PW_KEEP && !m) ||
        ((op == PB_PW_RADIUS || op == PB_PW_AXPBY) && !u))
        return fail(h, PB_ERR_INVALID, "pb_metro_pointwise: bad op or missing array");
    with_real(dtype, [&](auto rr) {
        using R = decltype(rr);
        pointwise_kernel<R><<<grid_for((long long)ny * nx, MET_THREADS, h->sm_count), MET_THREADS, 0, st>>>(
            op, (const R*)x, (const R*)u, (const R*)v, (const uint8_t*)m, ny, nx, a, b, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
