// PSF / MTF analysis (prysm/_richdata.py RichData.exact_* and Slices.az*, prysm/coordinates.py uniform_cart_to_polar,
// prysm/psf.py estimate_size and the Airy functions, prysm/otf.py diffraction_limited_mtf and
// analytical_encircled_energy_circular_aperture).
//
// Every entry point that samples data does it through interp_at, scipy's RegularGridInterpolator(method='linear') on
// sorted fp64 axes: the interval is the largest i with axis[i] <= p clipped to [0, n - 2], the weights are fp64, the
// four corners are summed in scipy's order with no fused multiply-add, so a NaN at any corner (even one of weight 0)
// gives NaN, and a point outside the axes gives `fill`.  The polar lattice of uniform_cart_to_polar is
// rho_j = linspace(0, rmax, nx), phi_i = linspace(0, 2 pi, ny), (x, y) = rho (cos phi, sin phi), fill 0; the
// azimuthal statistics and the crossings walk it without writing it to global memory.
#include <math_constants.h>

#include "common.cuh"

namespace pb {

constexpr int AN_THREADS = 256;
constexpr double AN_TWO_PI = 6.283185307179586;   // 2 * np.pi

template <typename T> struct acc_of { using type = double; };
template <> struct acc_of<float2> { using type = double2; };
template <> struct acc_of<double2> { using type = double2; };

template <typename T> __device__ inline typename acc_of<T>::type load_acc(const T* p) {
    if constexpr (std::is_same<T, float2>::value || std::is_same<T, double2>::value) {
        const T v = *p; return make_double2((double)v.x, (double)v.y);
    } else {
        return (double)*p;
    }
}
__device__ inline double acc_fma(double s, double v, double w0, double w1) { return __dadd_rn(s, __dmul_rn(__dmul_rn(v, w0), w1)); }
__device__ inline double2 acc_fma(double2 s, double2 v, double w0, double w1) {
    return make_double2(acc_fma(s.x, v.x, w0, w1), acc_fma(s.y, v.y, w0, w1));
}
template <typename A> __device__ inline A acc_fill(double f);
template <> __device__ inline double acc_fill<double>(double f) { return f; }
template <> __device__ inline double2 acc_fill<double2>(double f) { return make_double2(f, 0.0); }

template <typename T, typename A> __device__ inline void store_acc(T* p, A v) {
    if constexpr (std::is_same<T, float2>::value) *p = make_float2((float)v.x, (float)v.y);
    else if constexpr (std::is_same<T, double2>::value) *p = v;
    else *p = (T)v;
}

// sampled data: (ny, nx) with rows ld elements apart, x axis (nx) and y axis (ny) fp64 ascending.  An axis of one
// sample is allowed (a single row or column): its weight is 0 and both corners are that sample.
struct Grid {
    const double* x; const double* y; int nx, ny; long long ld;
};

// largest i with ax[i] <= p, clipped to [0, n - 2]
__device__ inline int interval(const double* __restrict__ ax, int n, double p) {
    if (n < 2 || !(ax[0] <= p)) return 0;
    int lo = 0, hi = n - 1;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (ax[mid] <= p) lo = mid; else hi = mid;
    }
    if (ax[hi] <= p) lo = hi;
    return min(lo, n - 2);
}

template <typename T>
__device__ inline typename acc_of<T>::type interp_at(const T* __restrict__ d, const Grid& g, double px, double py,
                                                     double fill) {
    using A = typename acc_of<T>::type;
    if (isnan(px) || isnan(py)) return acc_fill<A>(CUDART_NAN);
    if (!(py >= g.y[0] && py <= g.y[g.ny - 1] && px >= g.x[0] && px <= g.x[g.nx - 1])) return acc_fill<A>(fill);
    const int iy = interval(g.y, g.ny, py), ix = interval(g.x, g.nx, px);
    const int jy = g.ny > 1 ? iy + 1 : iy, jx = g.nx > 1 ? ix + 1 : ix;
    const double ty = g.ny > 1 ? __ddiv_rn(__dsub_rn(py, g.y[iy]), __dsub_rn(g.y[jy], g.y[iy])) : 0.0;
    const double tx = g.nx > 1 ? __ddiv_rn(__dsub_rn(px, g.x[ix]), __dsub_rn(g.x[jx], g.x[ix])) : 0.0;
    const double uy = __dsub_rn(1.0, ty), ux = __dsub_rn(1.0, tx);
    const T* r0 = d + (long long)iy * g.ld;
    const T* r1 = d + (long long)jy * g.ld;
    A s = acc_fill<A>(0.0);
    s = acc_fma(s, load_acc(r0 + ix), uy, ux);
    s = acc_fma(s, load_acc(r0 + jx), uy, tx);
    s = acc_fma(s, load_acc(r1 + ix), ty, ux);
    s = acc_fma(s, load_acc(r1 + jx), ty, tx);
    return s;
}

// element k of numpy.linspace(0, stop, n): k * (stop / (n - 1)), the last one stop itself
__device__ inline double linspace0(double stop, int n, int k) {
    if (n < 2) return 0.0;
    return k == n - 1 ? stop : __dmul_rn((double)k, __ddiv_rn(stop, (double)(n - 1)));
}

// the lattice point (rho_j, phi_i) of uniform_cart_to_polar, sampled
template <typename T>
__device__ inline typename acc_of<T>::type lattice_at(const T* __restrict__ d, const Grid& g, double rmax, int i, int j) {
    const double rho = linspace0(rmax, g.nx, j), phi = linspace0(AN_TWO_PI, g.ny, i);
    double s, c;
    sincos(phi, &s, &c);
    return interp_at(d, g, __dmul_rn(rho, c), __dmul_rn(rho, s), 0.0);
}

template <typename T>
__global__ void interp_points_kernel(const T* __restrict__ d, Grid g, const double* __restrict__ px,
                                     const double* __restrict__ py, long long count, double fill, T* __restrict__ out) {
    PB_GRID_STRIDE(k, count) store_acc(out + k, interp_at(d, g, px[k], py[k], fill));
}

template <typename T>
__global__ void interp_polar_kernel(const T* __restrict__ d, Grid g, double rmax, T* __restrict__ out) {
    const long long n = (long long)g.ny * g.nx;
    PB_GRID_STRIDE(k, n) {
        const int i = (int)(k / g.nx), j = (int)(k - (long long)i * g.nx);
        store_acc(out + k, lattice_at(d, g, rmax, i, j));
    }
}

// order-preserving key of a double; NaN above everything
__device__ inline unsigned long long order_key(double v) {
    if (isnan(v)) return ~0ull;
    const unsigned long long b = (unsigned long long)__double_as_longlong(v);
    return (b >> 63) ? ~b : (b | (1ull << 63));
}
__device__ inline double key_value(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~(1ull << 63)) : ~k));
}

// the rank-th smallest (0-based) of s[0, n) by an 8-bit radix select; every thread gets it
__device__ double select_rank(const double* s, int n, int rank, unsigned* hist, unsigned long long* shk, int* shr) {
    unsigned long long prefix = 0, mask = 0;
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long k = order_key(s[i]);
            if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1u);   // integer counts: order-free
        }
        __syncthreads();
        if (threadIdx.x < 32) {
            const int lane = threadIdx.x;
            unsigned part = 0;
            for (int b = 0; b < 8; ++b) part += hist[lane * 8 + b];
            unsigned incl = part;
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned w = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += w;
            }
            const unsigned excl = incl - part;
            const bool here = excl <= (unsigned)rank && (unsigned)rank < incl;
            if (here) {
                unsigned c = excl;
                int b = 0;
                for (; b < 8; ++b) {
                    const unsigned hb = hist[lane * 8 + b];
                    if ((unsigned)rank < c + hb) break;
                    c += hb;
                }
                *shk = prefix | ((unsigned long long)(lane * 8 + b) << shift);
                *shr = rank - (int)c;
            }
        }
        __syncthreads();
        prefix = *shk;
        rank = *shr;
        mask |= 255ull << shift;
        __syncthreads();
    }
    return key_value(prefix);
}

// one block per rho column j: the ny samples of the column are interpolated into shared memory once, then every
// statistic the mask asks for is reduced from there in a fixed order
template <typename R>
__global__ void __launch_bounds__(AN_THREADS) azimuthal_stats_kernel(const R* __restrict__ d, Grid g, double rmax,
                                                                     int stats, R* __restrict__ out) {
    extern __shared__ double s[];
    __shared__ unsigned hist[256];
    __shared__ unsigned long long shk;
    __shared__ int shr;
    const int j = blockIdx.x, n = g.ny;
    double cnt = 0, sum = 0, mn = CUDART_INF, mx = -CUDART_INF;
    for (int i = threadIdx.x; i < n; i += AN_THREADS) {
        const double v = lattice_at(d, g, rmax, i, j);
        s[i] = v;
        if (!isnan(v)) { cnt += 1; sum += v; mn = fmin(mn, v); mx = fmax(mx, v); }
    }
    cnt = block_reduce<AN_THREADS>(cnt, OpAdd{});
    sum = block_reduce<AN_THREADS>(sum, OpAdd{});
    const double mean = cnt > 0 ? sum / cnt : CUDART_NAN;
    const long long col = j;
    const long long nxo = g.nx;
    if (stats & PB_AZ_MIN) { mn = block_reduce<AN_THREADS>(mn, OpMin{}); if (threadIdx.x == 0) out[3 * nxo + col] = (R)(cnt > 0 ? mn : CUDART_NAN); }
    if (stats & PB_AZ_MAX) { mx = block_reduce<AN_THREADS>(mx, OpMax{}); if (threadIdx.x == 0) out[4 * nxo + col] = (R)(cnt > 0 ? mx : CUDART_NAN); }
    if (stats & PB_AZ_VAR) {
        double ss = 0;
        for (int i = threadIdx.x; i < n; i += AN_THREADS) {
            const double v = s[i];
            if (!isnan(v)) { const double e = v - mean; ss += e * e; }
        }
        ss = block_reduce<AN_THREADS>(ss, OpAdd{});
        if (threadIdx.x == 0) out[2 * nxo + col] = (R)(cnt > 0 ? ss / cnt : CUDART_NAN);
    }
    if (threadIdx.x == 0) {
        if (stats & PB_AZ_COUNT) out[col] = (R)cnt;
        if (stats & PB_AZ_MEAN) out[nxo + col] = (R)mean;
    }
    if (stats & PB_AZ_MEDIAN) {
        const int c = (int)cnt;
        double med = CUDART_NAN;
        if (c > 0) {
            const double hi = select_rank(s, n, c / 2, hist, &shk, &shr);
            med = (c & 1) ? hi : (select_rank(s, n, c / 2 - 1, hist, &shk, &shr) + hi) / 2;
        }
        if (threadIdx.x == 0) out[5 * nxo + col] = (R)med;
    }
}

// ---- estimate_size ------------------------------------------------------------------------------------------------
// rowmax[i] = max over the phi row i of the lattice, NaN if any sample is NaN
template <typename R>
__global__ void __launch_bounds__(AN_THREADS) lattice_rowmax_kernel(const R* __restrict__ d, Grid g, double rmax,
                                                                    double* __restrict__ rowmax) {
    const int i = blockIdx.x;
    double m = -CUDART_INF;
    for (int j = threadIdx.x; j < g.nx; j += AN_THREADS) m = OpMaxNan{}(m, lattice_at(d, g, rmax, i, j));
    m = block_reduce<AN_THREADS>(m, OpMaxNan{});
    if (threadIdx.x == 0) rowmax[i] = m;
}

// t = metric (absolute) or metric * max(rowmax) (relative), into *t
__global__ void __launch_bounds__(AN_THREADS) crossing_level_kernel(const double* __restrict__ rowmax, int n, double metric,
                                                                    int relative, double* __restrict__ t) {
    double m = -CUDART_INF;
    for (int i = threadIdx.x; i < n; i += AN_THREADS) m = OpMaxNan{}(m, rowmax[i]);
    m = block_reduce<AN_THREADS>(m, OpMaxNan{});
    if (threadIdx.x == 0) *t = relative ? __dmul_rn(metric, m) : metric;
}

// one block per phi row: the first (last = 0) or last crossing of the level along rho, as a radius; +inf if the row
// never crosses.  A crossing next to a NaN sample is a crossing with a NaN radius, as in the reference's loop.
// Thread k scans the contiguous samples [k L, (k + 1) L] (the shared end sample is interpolated twice).
template <typename R>
__global__ void __launch_bounds__(AN_THREADS) crossing_kernel(const R* __restrict__ d, Grid g, double rmax,
                                                              const double* __restrict__ level, int last,
                                                              double* __restrict__ radius) {
    __shared__ int shj;
    const int i = blockIdx.x, n = g.nx;
    const double t = *level;
    const int L = (n - 1 + AN_THREADS - 1) / AN_THREADS;
    const int j0 = threadIdx.x * L, j1 = min(j0 + L, n - 1);
    int found = -1;
    double y0 = 0, y1 = 0;
    if (j0 < j1) {
        double a = lattice_at(d, g, rmax, i, j0);
        for (int j = j0; j < j1; ++j) {
            const double b = lattice_at(d, g, rmax, i, j + 1);
            if ((a > t) != (b > t)) {
                found = j; y0 = a; y1 = b;
                if (!last) break;
            }
            a = b;
        }
    }
    if (threadIdx.x == 0) shj = last ? -1 : INT_MAX;
    __syncthreads();
    if (found >= 0) { if (last) atomicMax(&shj, found); else atomicMin(&shj, found); }   // integer: order-free
    __syncthreads();
    const int jj = shj;
    if (threadIdx.x == 0 && (jj < 0 || jj == INT_MAX)) radius[i] = CUDART_INF;
    if (found >= 0 && found == jj) {
        const double frac = y1 == y0 ? 0.0 : __ddiv_rn(__dsub_rn(t, y0), __dsub_rn(y1, y0));
        const double r0 = linspace0(rmax, n, jj), r1 = linspace0(rmax, n, jj + 1);
        radius[i] = __dadd_rn(r0, __dmul_rn(frac, __dsub_rn(r1, r0)));
    }
}

// res[0] = number of rows that cross, res[1] = the mean of their radii (fixed order); a NaN radius makes it NaN, as
// np.mean does
__global__ void __launch_bounds__(AN_THREADS) crossing_mean_kernel(const double* __restrict__ radius, int n,
                                                                   double* __restrict__ res) {
    double c = 0, s = 0;
    for (int i = threadIdx.x; i < n; i += AN_THREADS) {
        const double r = radius[i];
        if (r != CUDART_INF) { c += 1; s += r; }
    }
    c = block_reduce<AN_THREADS>(c, OpAdd{});
    s = block_reduce<AN_THREADS>(s, OpAdd{});
    if (threadIdx.x == 0) { res[0] = c; res[1] = c > 0 ? s / c : CUDART_NAN; }
}

// ---- analytic radial functions --------------------------------------------------------------------------------------
__device__ inline double jinc(double u) { return (u < 1e-8 && u > -1e-8) ? 0.5 : j1(u) / u; }
__device__ inline double difflim_core(double s) {
    return __dmul_rn(2.0 / M_PI, __dsub_rn(acos(s), __dmul_rn(s, sqrt(__dsub_rn(1.0, __dmul_rn(s, s))))));
}

template <typename Ti, typename To>
__global__ void analytic_radial_kernel(int kind, const Ti* __restrict__ x, long long count, double a, double b,
                                       To* __restrict__ out) {
    PB_GRID_STRIDE(k, count) {
        const double v = (double)x[k];
        double r;
        switch (kind) {
            case PB_AR_AIRYDISK:
            case PB_AR_AIRYDISK_EFIELD: {   // unit_r * pi / wavelength / fno
                const double e = 2.0 * jinc(__ddiv_rn(__ddiv_rn(__dmul_rn(v, M_PI), a), b));
                r = kind == PB_AR_AIRYDISK ? __dmul_rn(e, e) : e;
                break;
            }
            case PB_AR_AIRYDISK_FT: {       // |r| / (1 / (wavelength fno)), clamped at 1
                const double s = __ddiv_rn(fabs(v), __ddiv_rn(1.0, __dmul_rn(a, b)));
                r = difflim_core(fmin(s, 1.0));
                break;
            }
            case PB_AR_DIFFLIM_MTF: {       // |f / (1 / (wavelength / 1000 fno))|, clamped at 1
                const double s = fabs(__ddiv_rn(v, __ddiv_rn(1.0, __dmul_rn(__ddiv_rn(a, 1000.0), b))));
                r = difflim_core(fmin(s, 1.0));
                break;
            }
            case PB_AR_DIFFLIM_NORMALIZED: r = difflim_core(fmin(v, 1.0)); break;
            default: {                      // PB_AR_EE_CIRCULAR: points * pi / fno / wavelength
                const double p = __ddiv_rn(__ddiv_rn(__dmul_rn(v, M_PI), b), a);
                const double j0v = j0(p), j1v = j1(p);
                r = __dsub_rn(__dsub_rn(1.0, __dmul_rn(j0v, j0v)), __dmul_rn(j1v, j1v));
                break;
            }
        }
        out[k] = (To)r;
    }
}

static bool grid_ok(const double* xax, const double* yax, int ny, int nx) { return xax && yax && ny >= 1 && nx >= 1; }

}  // namespace pb

using namespace pb;

extern "C" int pb_interp2d_linear(pb_handle_t hh, int type, const void* data, int ny, int nx, long long ld,
                                  const double* xax, const double* yax, int mode, const double* px, const double* py,
                                  long long count, double rmax, double fill, void* out, void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (!data || !out || !grid_ok(xax, yax, ny, nx) || ld < nx) return fail(h, PB_ERR_INVALID, "bad interpolation grid");
    if (mode == PB_INTERP_POINTS) {
        if (count < 0 || (count > 0 && (!px || !py))) return fail(h, PB_ERR_INVALID, "bad interpolation points");
        if (count == 0) return PB_OK;
    } else if (mode == PB_INTERP_POLAR) {
        count = (long long)ny * nx;
    } else {
        return fail(h, PB_ERR_INVALID, "mode must be PB_INTERP_POINTS or PB_INTERP_POLAR");
    }
    const Grid g{xax, yax, nx, ny, ld};
    const int blocks = grid_for(count, AN_THREADS, h->sm_count);
    bool typed = false;
    with_elem(type, [&](auto t) {
        using T = decltype(t);
        if constexpr (is_one_of<T, float, double, float2, double2>) {
            typed = true;
            if (mode == PB_INTERP_POINTS)
                interp_points_kernel<T><<<blocks, AN_THREADS, 0, st>>>((const T*)data, g, px, py, count, fill, (T*)out);
            else
                interp_polar_kernel<T><<<blocks, AN_THREADS, 0, st>>>((const T*)data, g, rmax, (T*)out);
        }
    });
    if (!typed) return fail(h, PB_ERR_INVALID, "data must be PB_ELEM_F32, F64, C64 or C128");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_azimuthal_stats(pb_handle_t hh, int type, const void* data, int ny, int nx, const double* xax,
                                  const double* yax, double rmax, int stats, void* out, void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (!data || !out || !grid_ok(xax, yax, ny, nx)) return fail(h, PB_ERR_INVALID, "bad azimuthal-statistics grid");
    if (type != PB_ELEM_F32 && type != PB_ELEM_F64) return fail(h, PB_ERR_INVALID, "data must be PB_ELEM_F32 or F64");
    if (ny > PB_AZ_MAX_NY)
        return fail(h, PB_ERR_INVALID, "azimuthal statistics hold a column on chip: at most " +
                                           std::to_string(PB_AZ_MAX_NY) + " phi samples (rows), got " + std::to_string(ny));
    if (stats & ~PB_AZ_ALL) return fail(h, PB_ERR_INVALID, "unknown statistic bits");
    if (!stats) return PB_OK;
    const Grid g{xax, yax, nx, ny, (long long)nx};
    const size_t smem = (size_t)ny * sizeof(double);
    int rc = PB_OK;
    with_elem(type, [&](auto t) {
        using T = decltype(t);
        if constexpr (is_one_of<T, float, double>) {
            const void* fn = (const void*)azimuthal_stats_kernel<T>;
            if (attr_needed(h, fn)) {
                cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                     PB_AZ_MAX_NY * (int)sizeof(double));
                if (e != cudaSuccess) { rc = fail(h, PB_ERR_CUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(e)); return; }
            }
            azimuthal_stats_kernel<T><<<nx, AN_THREADS, smem, st>>>((const T*)data, g, rmax, stats, (T*)out);
        }
    });
    PB_TRY(rc);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_polar_crossings(pb_handle_t hh, int type, const void* data, int ny, int nx, const double* xax,
                                  const double* yax, double rmax, double metric, int relative, int last, double* result,
                                  void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if (!data || !result || !grid_ok(xax, yax, ny, nx)) return fail(h, PB_ERR_INVALID, "bad crossing grid");
    if (type != PB_ELEM_F32 && type != PB_ELEM_F64) return fail(h, PB_ERR_INVALID, "data must be PB_ELEM_F32 or F64");
    if (nx < 2) { result[0] = 0; result[1] = std::nan(""); return PB_OK; }   // no pair of samples: nothing crosses
    // scratch: rowmax [ny], radius [ny], level, count and mean
    void* w = nullptr;
    PB_TRY(ensure_scratch(h, 2, (2 * (size_t)ny + 3) * sizeof(double), &w));
    double* rowmax = (double*)w;
    double* radius = rowmax + ny;
    double* level = radius + ny;
    double* res = level + 1;
    const Grid g{xax, yax, nx, ny, (long long)nx};
    with_elem(type, [&](auto t) {
        using T = decltype(t);
        if constexpr (is_one_of<T, float, double>) {
            if (relative) lattice_rowmax_kernel<T><<<ny, AN_THREADS, 0, st>>>((const T*)data, g, rmax, rowmax);
            crossing_level_kernel<<<1, AN_THREADS, 0, st>>>(rowmax, relative ? ny : 0, metric, relative, level);
            crossing_kernel<T><<<ny, AN_THREADS, 0, st>>>((const T*)data, g, rmax, level, last, radius);
            crossing_mean_kernel<<<1, AN_THREADS, 0, st>>>(radius, ny, res);
        }
    });
    PB_LAUNCH_CHECK(h);
    h->launches += relative ? 3 : 2;
    PB_CUDA(h, cudaMemcpyAsync(result, res, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_analytic_radial(pb_handle_t hh, int in_type, int out_type, int kind, const void* x, long long count,
                                  double a, double b, void* out, void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    if ((!x || !out) && count > 0) return fail(h, PB_ERR_INVALID, "null pointer");
    if (kind < PB_AR_AIRYDISK || kind > PB_AR_EE_CIRCULAR) return fail(h, PB_ERR_INVALID, "unknown analytic kind");
    if ((in_type != PB_ELEM_F32 && in_type != PB_ELEM_F64) || (out_type != PB_ELEM_F32 && out_type != PB_ELEM_F64))
        return fail(h, PB_ERR_INVALID, "input and output must be PB_ELEM_F32 or F64");
    if (count <= 0) return PB_OK;
    const int blocks = grid_for(count, AN_THREADS, h->sm_count);
    with_elem(in_type, [&](auto ti) {
        using Ti = decltype(ti);
        if constexpr (is_one_of<Ti, float, double>) {
            with_elem(out_type, [&](auto to) {
                using To = decltype(to);
                if constexpr (is_one_of<To, float, double>)
                    analytic_radial_kernel<Ti, To><<<blocks, AN_THREADS, 0, st>>>(kind, (const Ti*)x, count, a, b, (To*)out);
            });
        }
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
