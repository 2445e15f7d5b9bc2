// Image sensors (prysm/detector.py, prysm/bayer.py): a detector exposure with counter-based shot and read noise, the
// lookup-table gather, the pixel footprint, and the Bayer colour-filter-array operations.
//
// Random numbers: Philox4x32-10 with a 64-bit key.  The counter of a draw is (pixel low 32 bits, pixel high 32 bits,
// frame, draw index); shot noise uses draw indices from 0 upwards (PTRS may retry), read noise from 2^31, so the value of
// one (key, pixel, frame) never depends on the launch shape, on `frames`, or on how many retries a neighbour needed.
// Each Philox call yields two 53-bit uniforms in [0, 1).
//
// Shot noise is exact Poisson: inversion for 0 < lam < 10, Hoermann's PTRS transformed rejection for lam >= 10 (the
// sampler numpy's legacy `poisson` uses), 0 for lam = 0; the slow acceptance test is evaluated in fp64.
#include "common.cuh"

namespace pb {

namespace {

constexpr int kSensorThreads = 256;

// ---- Philox4x32-10 -------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
    constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(M0, c.x), lo0 = M0 * c.x;
        const uint32_t hi1 = __umulhi(M1, c.z), lo1 = M1 * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += W0;
        k.y += W1;
    }
    return c;
}

__device__ __forceinline__ double u53(uint32_t a, uint32_t b) {
    return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) * (1.0 / 9007199254740992.0);
}

// the uniforms of one (pixel, frame) stream, two per Philox call
struct Uniforms {
    uint4 ctr;
    uint2 key;
    double spare;
    bool have = false;
    __device__ Uniforms(uint2 k, unsigned long long pixel, uint32_t frame, uint32_t first_draw)
        : ctr(make_uint4((uint32_t)pixel, (uint32_t)(pixel >> 32), frame, first_draw)), key(k) {}
    __device__ __forceinline__ double next() {
        if (have) { have = false; return spare; }
        const uint4 r = philox4x32_10(ctr, key);
        ctr.w++;
        spare = u53(r.z, r.w);
        have = true;
        return u53(r.x, r.y);
    }
};

// log Gamma(x) by Stirling's series with upward shift below 7 (the form numpy's random_loggam uses)
__device__ double loggam(double x) {
    constexpr double a[10] = {8.333333333333333e-02, -2.777777777777778e-03, 7.936507936507937e-04,
                              -5.952380952380952e-04, 8.417508417508418e-04, -1.917526917526918e-03,
                              6.410256410256410e-03, -2.955065359477124e-02, 1.796443723688307e-01,
                              -1.39243221690590e+00};
    if (x == 1.0 || x == 2.0) return 0.0;
    double x0 = x;
    int n = 0;
    if (x <= 7.0) { n = (int)(7.0 - x); x0 = x + n; }
    const double x2 = 1.0 / (x0 * x0);
    double gl0 = a[9];
    for (int k = 8; k >= 0; --k) gl0 = gl0 * x2 + a[k];
    double gl = gl0 / x0 + 0.5 * log(2.0 * M_PI) + (x0 - 0.5) * log(x0) - x0;
    for (int k = 0; k < n; ++k) { gl -= log(x0 - 1.0); x0 -= 1.0; }
    return gl;
}

// per-pixel constants of the sampler, computed once and reused for every frame
struct PoissonPlan {
    double lam, enlam, slam, loglam, b, a, invalpha, log_invalpha, vr;
    __device__ explicit PoissonPlan(double l) : lam(l) {
        if (lam >= 10.0) {
            slam = sqrt(lam);
            loglam = log(lam);
            b = 0.931 + 2.53 * slam;
            a = -0.059 + 0.02483 * b;
            invalpha = 1.1239 + 1.1328 / (b - 3.4);
            log_invalpha = log(invalpha);
            vr = 0.9277 - 3.6224 / (b - 2.0);
        } else {
            enlam = exp(-lam);
        }
    }
    __device__ double sample(Uniforms& u) const {
        if (lam == 0.0) return 0.0;
        if (lam < 10.0) {           // inversion: one uniform, at most a few dozen terms
            const double U = u.next();
            double p = enlam, F = p, k = 0.0;
            while (U > F && k < 1000.0) {
                k += 1.0;
                p *= lam / k;
                F += p;
            }
            return k;
        }
        for (;;) {                  // PTRS
            const double U = u.next() - 0.5, V = u.next();
            const double us = 0.5 - fabs(U);
            const double k = floor((2.0 * a / us + b) * U + lam + 0.43);
            if (us >= 0.07 && V <= vr) return k;
            if (k < 0.0 || (us < 0.013 && V > us)) continue;
            if (log(V) + log_invalpha - log(a / (us * us) + b) <= -lam + k * loglam - loggam(k + 1.0)) return k;
        }
    }
};

struct ExposeParams {
    long long n, nx;                     // pixels; the image is viewed as (n / nx, nx)
    long long prnu_sr, prnu_sc, dcnu_sr, dcnu_sc;
    int frames;
    double t, dark, read_sigma, bias, fwc, scaling, cap;
    long long lut_len;
    uint2 key;
};

// flags[0] bit 0: a lam < 0 or NaN; bit 1: a lam above numpy's POISSON_LAM_MAX; bit 2: a code outside the LUT.
// flags[1]: the largest such code.
template <typename R, typename Code, typename Out>
__global__ void __launch_bounds__(kSensorThreads) expose_kernel(const R* __restrict__ aerial, const R* __restrict__ prnu,
                                                                const R* __restrict__ dcnu, const Out* __restrict__ lut,
                                                                ExposeParams p, Out* __restrict__ out,
                                                                unsigned int* __restrict__ flags) {
    // np.iinfo('l').max - sqrt(np.iinfo('l').max) * 10, in fp64 as numpy forms it
    const double lam_max = 9223372036854775807.0 - sqrt(9223372036854775807.0) * 10.0;
    PB_GRID_STRIDE(i, p.n) {
        // electrons = aerial * t [* prnu] + dark [* dcnu], every step rounded in R as numpy does
        R e = mul_rn(aerial[i], (R)p.t);
        R d = (R)p.dark;
        if (prnu || dcnu) {
            const long long r = i / p.nx, c = i - r * p.nx;
            if (prnu) e = mul_rn(e, prnu[r * p.prnu_sr + c * p.prnu_sc]);
            if (dcnu) d = mul_rn(d, dcnu[r * p.dcnu_sr + c * p.dcnu_sc]);
        }
        double lam = (double)add_rn(e, d);
        if (!(lam >= 0.0)) { atomicOr(flags, 1u); lam = 0.0; }
        else if (lam > lam_max) { atomicOr(flags, 2u); lam = 0.0; }
        const PoissonPlan plan(lam);
        for (int f = 0; f < p.frames; ++f) {
            Uniforms shot(p.key, (unsigned long long)i, (uint32_t)f, 0u);
            double x = plan.sample(shot);
            if (p.read_sigma != 0.0) {
                Uniforms rd(p.key, (unsigned long long)i, (uint32_t)f, 0x80000000u);
                const double u1 = 1.0 - rd.next(), u2 = rd.next();           // u1 in (0, 1]
                x = x + p.read_sigma * (sqrt(-2.0 * log(u1)) * cospi(2.0 * u2));
            }
            x = x + p.bias;
            if (x > p.fwc) x = p.fwc;
            x = x * p.scaling;
            if (x < 0.0) x = 0.0;
            if (x > p.cap) x = p.cap;
            const Code code = (Code)x;
            Out v;
            if (lut) {
                if ((long long)code >= p.lut_len) {
                    atomicOr(flags, 4u);
                    atomicMax(flags + 1, (unsigned int)code);
                    v = lut[p.lut_len - 1];
                } else {
                    v = lut[code];
                }
            } else {
                v = (Out)code;
            }
            out[(long long)f * p.n + i] = v;
        }
    }
}

// np.take(lut, codes) for unsigned codes; a code >= lut_len sets flags[0] bit 2 and raises flags[1] to it
template <typename Code, typename Out>
__global__ void lut_kernel(const Code* __restrict__ codes, long long n, const Out* __restrict__ lut, long long lut_len,
                           int check, Out* __restrict__ out, unsigned int* __restrict__ flags) {
    PB_GRID_STRIDE(i, n) {
        long long c = (long long)codes[i];
        if (check && c >= lut_len) {
            atomicOr(flags, 4u);
            atomicMax(flags + 1, (unsigned int)c);
            c = lut_len - 1;
        }
        out[i] = lut[c];
    }
}

// (x <= wx) & (x >= -wx) & (y <= wy) & (y >= -wy) over an (n / nx, nx) view; x and y are read through row / column
// strides so that broadcast operands are never materialised
template <typename R>
__global__ void pixel_kernel(const R* __restrict__ x, long long xsr, long long xsc, const R* __restrict__ y, long long ysr,
                             long long ysc, long long n, long long nx, double wx, double wy, uint8_t* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const long long r = i / nx, c = i - r * nx;
        const double xv = (double)x[r * xsr + c * xsc], yv = (double)y[r * ysr + c * ysc];
        out[i] = (xv <= wx) & (xv >= -wx) & (yv <= wy) & (yv >= -wy);
    }
}

// ---- Bayer ---------------------------------------------------------------------------------------------------------
// CFA site of (row, col): 0 top-left, 1 top-right, 2 bottom-left, 3 bottom-right of each 2x2 cell
__device__ __forceinline__ int cfa_site(long long y, long long x) { return (int)(((y & 1) << 1) | (x & 1)); }

struct Planes4 { const void* p[4]; long long ld[4]; };

// out (M, N) with row pitch out_ld: the value of site s comes from plane s, at (y, x) (composite) or (y/2, x/2)
// (recomposite).  A copy of elements of sizeof(T) bytes, so any dtype of that size.
template <typename T>
__global__ void interleave_kernel(Planes4 src, int half, long long M, long long N, T* __restrict__ out, long long out_ld) {
    const long long n = M * N;
    PB_GRID_STRIDE(i, n) {
        const long long y = i / N, x = i - y * N;
        const int s = cfa_site(y, x);
        const long long sy = half ? y >> 1 : y, sx = half ? x >> 1 : x;
        out[y * out_ld + x] = static_cast<const T*>(src.p[s])[sy * src.ld[s] + sx];
    }
}

// (m/2, n/2, 3) = (R, (G1 + G2) / 2, B) with the green sum in the input type (numpy's uint16 + uint16 wraps)
template <typename In, typename Out>
__global__ void deinterlace_kernel(const In* __restrict__ img, long long m2, long long n2, long long ld, int r_site,
                                   int b_site, Out* __restrict__ out) {
    const long long n = m2 * n2;
    PB_GRID_STRIDE(i, n) {
        const long long y = i / n2, x = i - y * n2;
        const In* c = img + 2 * y * ld + 2 * x;
        const In v[4] = {c[0], c[1], c[ld], c[ld + 1]};
        const In gsum = (In)(v[1] + v[2]);
        out[3 * i + 0] = (Out)v[r_site];
        out[3 * i + 1] = (Out)gsum / (Out)2;
        out[3 * i + 2] = (Out)v[b_site];
    }
}

// white balance: the gain of element i is gains[site] (mosaic, kind 0) or gains[i % 3] (rgb, kind 1)
struct Gains4 { double g[4]; double sat[4]; };
constexpr int kWbMaxBlocks = 1024;     // blocks of the white-balance launches; the ratio kernel folds their plane maxima

__device__ __forceinline__ int wb_plane(int kind, long long i, long long nx) {
    if (kind == 1) return (int)(i % 3);
    const long long y = i / nx;
    return cfa_site(y, i - y * nx);
}

// per-block maxima of each plane -> partial[block * 4 + plane]
template <typename T>
__global__ void wb_plane_max_kernel(const T* __restrict__ a, long long n, long long nx, int kind,
                                    double* __restrict__ partial) {
    double mx[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    PB_GRID_STRIDE(i, n) {
        const int pl = wb_plane(kind, i, nx);
        mx[pl] = fmax(mx[pl], (double)a[i]);
    }
    __shared__ double sh[4][kSensorThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
    for (int pl = 0; pl < 4; ++pl) {
        double v = mx[pl];
        for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
        if (lane == 0) sh[pl][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x < 4) {
        double v = -INFINITY;
        for (int w = 0; w < kSensorThreads / 32; ++w) v = fmax(v, sh[threadIdx.x][w]);
        partial[blockIdx.x * 4 + threadIdx.x] = v;
    }
}

// ratio = max(1, max_p(max_p * gain_p / sat_p)) over the planes in use, as the reference's descaling loop
__global__ void __launch_bounds__(kSensorThreads) wb_ratio_kernel(const double* __restrict__ partial, int nblocks,
                                                                  int nplanes, Gains4 g, double* __restrict__ ratio) {
    __shared__ double sh[4][kSensorThreads / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (int pl = 0; pl < 4; ++pl) {
        double v = -INFINITY;
        for (int b = threadIdx.x; b < nblocks; b += kSensorThreads) v = fmax(v, partial[b * 4 + pl]);
        for (int o = 16; o; o >>= 1) v = fmax(v, __shfl_down_sync(0xffffffffu, v, o));
        if (lane == 0) sh[pl][wid] = v;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double r = 1.0;
        for (int pl = 0; pl < nplanes; ++pl) {
            double mx = -INFINITY;
            for (int w = 0; w < kSensorThreads / 32; ++w) mx = fmax(mx, sh[pl][w]);
            const double rat = mx * g.g[pl] / g.sat[pl];
            if (rat > 1.0 && rat > r) r = rat;
        }
        *ratio = r;
    }
}

template <typename T>
__global__ void wb_scale_kernel(T* __restrict__ a, long long n, long long nx, int kind, Gains4 g,
                                const double* __restrict__ ratio) {
    T gain[4];
    const double r = ratio ? *ratio : 1.0;
#pragma unroll
    for (int pl = 0; pl < 4; ++pl) gain[pl] = (T)(ratio ? g.g[pl] / r : g.g[pl]);
    PB_GRID_STRIDE(i, n)
        a[i] = a[i] * gain[wb_plane(kind, i, nx)];
}

// ---- Malvar-He-Cutler demosaic (Malvar, He & Cutler, ICASSP 2004, fig. 2), one pass -----------------------------------
// Each block stages a (TY + 4) x (TX + 4) tile with a 2-sample halo, mirrored at the image edges as scipy.ndimage's
// mode='reflect' (d c b a | a b c d | d c b a, for any side length >= 1).  Each output pixel evaluates only the two
// 5x5 filters its CFA site needs, accumulating in fp64.  The filters are symmetric under a 180-degree rotation, so
// correlation and convolution agree.
constexpr int kMalvarTX = 32, kMalvarTY = 16, kMalvarRows = 4;   // block 32 x 4, four output rows per thread

__device__ __forceinline__ long long reflect_index(long long i, long long n) {
    const long long p = 2 * n;
    long long j = i % p;
    if (j < 0) j += p;
    return j < n ? j : p - 1 - j;
}

// taps of the five filters, times 8 (the reference divides by 8): G at R/B; R at G in an R row (c1); R at G in a B row
// (c2); R at B (c3).  Indexed [dy + 2][dx + 2].
__device__ constexpr float kMalvarTaps[4][5][5] = {
    {{0, 0, -1, 0, 0}, {0, 0, 2, 0, 0}, {-1, 2, 4, 2, -1}, {0, 0, 2, 0, 0}, {0, 0, -1, 0, 0}},
    {{0, 0, 0.5f, 0, 0}, {0, -1, 0, -1, 0}, {-1, 4, 5, 4, -1}, {0, -1, 0, -1, 0}, {0, 0, 0.5f, 0, 0}},
    {{0, 0, -1, 0, 0}, {0, -1, 4, -1, 0}, {0.5f, 0, 5, 0, 0.5f}, {0, -1, 4, -1, 0}, {0, 0, -1, 0, 0}},
    {{0, 0, -1.5f, 0, 0}, {0, 2, 0, 2, 0}, {-1.5f, 0, 6, 0, -1.5f}, {0, 2, 0, 2, 0}, {0, 0, -1.5f, 0, 0}},
};

// the filter is a template argument so that the taps fold into the instructions and the zero taps vanish
template <int W, typename S>
__device__ __forceinline__ double malvar_filter(const S (*tile)[kMalvarTX + 4], int ty, int tx) {
    double acc = 0.0;
#pragma unroll
    for (int dy = 0; dy < 5; ++dy)
#pragma unroll
        for (int dx = 0; dx < 5; ++dx) {
            const float w = kMalvarTaps[W][dy][dx];
            if (w != 0.0f) acc += (double)w * (double)tile[ty + dy][tx + dx];
        }
    return acc * 0.125;
}

// S: the staging type (float holds uint8 / uint16 / float32 exactly; double for float64)
template <typename In, typename S, typename Out>
__global__ void __launch_bounds__(kMalvarTX * kMalvarRows) malvar_kernel(const In* __restrict__ img, long long m, long long n,
                                                                         long long ld, int bggr, Out* __restrict__ out) {
    __shared__ S tile[kMalvarTY + 4][kMalvarTX + 4];
    const long long y0 = (long long)blockIdx.y * kMalvarTY, x0 = (long long)blockIdx.x * kMalvarTX;
    const int tid = threadIdx.y * kMalvarTX + threadIdx.x;
    for (int k = tid; k < (kMalvarTY + 4) * (kMalvarTX + 4); k += kMalvarTX * kMalvarRows) {
        const int ty = k / (kMalvarTX + 4), tx = k - ty * (kMalvarTX + 4);
        const long long gy = reflect_index(y0 + ty - 2, m), gx = reflect_index(x0 + tx - 2, n);
        tile[ty][tx] = (S)img[gy * ld + gx];
    }
    __syncthreads();
    const int tx = threadIdx.x;
    const long long x = x0 + tx;
    if (x >= n) return;
    for (int rr = 0; rr < kMalvarTY / kMalvarRows; ++rr) {
        const int ty = threadIdx.y + rr * kMalvarRows;
        const long long y = y0 + ty;
        if (y >= m) break;
        const double c = (double)tile[ty + 2][tx + 2];
        // site 0 holds R (rggb) or B (bggr); site 3 the other; 1 and 2 are greens
        const int s = cfa_site(y, x);
        double own = c, g, other_a, other_b;   // own colour at sites 0 / 3; the two chromas at 1 / 2
        double rv, gv, bv;
        if (s == 0 || s == 3) {
            g = malvar_filter<0>(tile, ty, tx);
            other_a = malvar_filter<3>(tile, ty, tx);
            // s == 0: first colour = c, second = c3; s == 3: the reverse
            const double first = s == 0 ? own : other_a, second = s == 0 ? other_a : own;
            rv = bggr ? second : first;
            bv = bggr ? first : second;
            gv = g;
        } else {
            other_a = malvar_filter<1>(tile, ty, tx);   // c1
            other_b = malvar_filter<2>(tile, ty, tx);   // c2
            // rggb: R = c1 at top-right, c2 at bottom-left; B the other way round.  bggr swaps R and B.
            const double first = s == 1 ? other_a : other_b, second = s == 1 ? other_b : other_a;
            rv = bggr ? second : first;
            bv = bggr ? first : second;
            gv = c;
        }
        Out* o = out + 3 * (y * n + x);
        o[0] = (Out)rv;
        o[1] = (Out)gv;
        o[2] = (Out)bv;
    }
}

// assemble_superresolved: (m, n, 3) = (Re rp, (Re g2p + g1) / 2, Re bp)
template <typename R>
__global__ void assemble_kernel(const cplx<R>* __restrict__ rp, const cplx<R>* __restrict__ g2p, const cplx<R>* __restrict__ bp,
                                const R* __restrict__ g1, long long n, R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        out[3 * i + 0] = rp[i].x;
        out[3 * i + 1] = (g2p[i].x + g1[i]) / R(2);
        out[3 * i + 2] = bp[i].x;
    }
}

}  // namespace

}  // namespace pb

using namespace pb;

namespace {

// element size -> an unsigned container of that size (the LUT and interleave kernels only move bytes)
template <typename F>
bool with_bytes(int bytes, F&& f) {
    switch (bytes) {
        case 1: f(uint8_t{}); return true;
        case 2: f(uint16_t{}); return true;
        case 4: f(uint32_t{}); return true;
        case 8: f((unsigned long long)0); return true;
        default: return false;
    }
}

}  // namespace

extern "C" int pb_expose(pb_handle_t hh, int dtype, const void* aerial, long long n, long long nx, const void* prnu,
                         long long prnu_sr, long long prnu_sc, const void* dcnu, long long dcnu_sr, long long dcnu_sc,
                         const double* params_host, int frames, long long key, int code_bytes, const void* lut,
                         long long lut_len, int out_bytes, void* out, void* flags, void* stream) {
    PB_ENTER(hh);
    if (!aerial || !out || !flags || !params_host || n < 1 || nx < 1 || n % nx || frames < 1)
        return fail(h, PB_ERR_INVALID, "bad expose arguments");
    if (lut ? lut_len < 1 : out_bytes != code_bytes) return fail(h, PB_ERR_INVALID, "bad expose lookup table");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    ExposeParams p;
    p.n = n; p.nx = nx;
    p.prnu_sr = prnu_sr; p.prnu_sc = prnu_sc; p.dcnu_sr = dcnu_sr; p.dcnu_sc = dcnu_sc;
    p.frames = frames;
    p.t = params_host[0]; p.dark = params_host[1]; p.read_sigma = params_host[2]; p.bias = params_host[3];
    p.fwc = params_host[4]; p.scaling = params_host[5]; p.cap = params_host[6];
    p.lut_len = lut_len;
    p.key = make_uint2((uint32_t)key, (uint32_t)(key >> 32));
    const int g = grid_for(n, kSensorThreads, h->sm_count);
    bool ok = false;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        auto launch = [&](auto code, auto o) {
            using Code = decltype(code);
            using Out = decltype(o);
            expose_kernel<R, Code, Out><<<g, kSensorThreads, 0, st>>>((const R*)aerial, (const R*)prnu, (const R*)dcnu,
                                                                       (const Out*)lut, p, (Out*)out, (unsigned int*)flags);
            ok = true;
        };
        with_bytes(code_bytes, [&](auto code) {
            if constexpr (sizeof(code) <= 4) {
                if (!lut) launch(code, code);
                else with_bytes(out_bytes, [&](auto o) { launch(code, o); });
            }
        });
    });
    if (!ok) return fail(h, PB_ERR_INVALID, "expose: dtype must be PB_C64 / PB_C128, codes of 1, 2 or 4 bytes");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_apply_lut(pb_handle_t hh, int code_bytes, const void* codes, long long n, const void* lut,
                            long long lut_len, int out_bytes, int check, void* out, void* flags, void* stream) {
    PB_ENTER(hh);
    if (!codes || !lut || !out || (check && !flags) || lut_len < 1 || n < 0) return fail(h, PB_ERR_INVALID, "bad lut arguments");
    if (n == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int g = grid_for(n, kSensorThreads, h->sm_count);
    bool ok = false;
    with_bytes(code_bytes, [&](auto code) {
        using Code = decltype(code);
        if constexpr (sizeof(Code) <= 4) {
            with_bytes(out_bytes, [&](auto o) {
                using Out = decltype(o);
                lut_kernel<Code, Out><<<g, kSensorThreads, 0, st>>>((const Code*)codes, n, (const Out*)lut, lut_len,
                                                                   check, (Out*)out, (unsigned int*)flags);
                ok = true;
            });
        }
    });
    if (!ok) return fail(h, PB_ERR_INVALID, "apply_lut: codes of 1, 2 or 4 bytes, table entries of 1, 2, 4 or 8 bytes");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_pixel(pb_handle_t hh, int dtype, const void* x, long long xsr, long long xsc, const void* y,
                        long long ysr, long long ysc, long long n, long long nx, double wx, double wy, void* out,
                        void* stream) {
    PB_ENTER(hh);
    if (!x || !y || !out || n < 0 || nx < 1 || n % nx) return fail(h, PB_ERR_INVALID, "bad pixel arguments");
    if (n == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int g = grid_for(n, kSensorThreads, h->sm_count);
    if (!with_real(dtype, [&](auto r) {
            using R = decltype(r);
            pixel_kernel<R><<<g, kSensorThreads, 0, st>>>((const R*)x, xsr, xsc, (const R*)y, ysr, ysc, n, nx, wx, wy,
                                                          (uint8_t*)out);
        }))
        return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_bayer_interleave(pb_handle_t hh, int elem_bytes, const void* const* planes_host, const long long* ld_host,
                                   int half, long long M, long long N, void* out, long long out_ld, void* stream) {
    PB_ENTER(hh);
    if (!planes_host || !ld_host || !out || M < 0 || N < 0 || out_ld < N) return fail(h, PB_ERR_INVALID, "bad interleave arguments");
    Planes4 src;
    for (int s = 0; s < 4; ++s) {
        src.p[s] = planes_host[s];
        src.ld[s] = ld_host[s];
        // a site that occurs in the output needs its plane
        const bool used = (s < 2 || M > 1) && ((s & 1) == 0 || N > 1);
        if (used && !src.p[s]) return fail(h, PB_ERR_INVALID, "null plane");
    }
    if (M * N == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int g = grid_for(M * N, kSensorThreads, h->sm_count);
    if (!with_bytes(elem_bytes, [&](auto e) {
            using T = decltype(e);
            interleave_kernel<T><<<g, kSensorThreads, 0, st>>>(src, half, M, N, (T*)out, out_ld);
        }))
        return fail(h, PB_ERR_INVALID, "elements of 1, 2, 4 or 8 bytes");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_demosaic_deinterlace(pb_handle_t hh, int in_type, const void* img, long long m, long long n, long long ld,
                                       int bggr, int out_type, void* out, void* stream) {
    PB_ENTER(hh);
    if (!img || !out || m < 0 || n < 0 || (m % 2) || (n % 2) || ld < n) return fail(h, PB_ERR_INVALID, "bad deinterlace arguments");
    const long long m2 = m / 2, n2 = n / 2;
    if (m2 * n2 == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int g = grid_for(m2 * n2, kSensorThreads, h->sm_count);
    const int r_site = bggr ? 3 : 0, b_site = bggr ? 0 : 3;
    bool ok = false;
    with_elem(in_type, [&](auto i) {
        using In = decltype(i);
        with_elem(out_type, [&](auto o) {
            using Out = decltype(o);
            if constexpr (is_one_of<In, float, double, uint8_t, uint16_t, uint32_t> && std::is_floating_point<Out>::value) {
                deinterlace_kernel<In, Out><<<g, kSensorThreads, 0, st>>>((const In*)img, m2, n2, ld, r_site, b_site, (Out*)out);
                ok = true;
            }
        });
    });
    if (!ok) return fail(h, PB_ERR_INVALID, "deinterlace: unsupported input type or a non-float output type");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_white_balance(pb_handle_t hh, int dtype, void* a, long long n, long long nx, int kind,
                                const double* gains_host, const double* sat_host, void* stream) {
    PB_ENTER(hh);
    if (!a || !gains_host || n < 0 || nx < 1 || kind < 0 || kind > 1)
        return fail(h, PB_ERR_INVALID, "bad white-balance arguments");
    if (n == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Gains4 g4;
    const int nplanes = kind == 1 ? 3 : 4;
    for (int pl = 0; pl < 4; ++pl) {
        g4.g[pl] = pl < nplanes ? gains_host[pl] : 1.0;
        g4.sat[pl] = sat_host && pl < nplanes ? sat_host[pl] : 1.0;
    }
    const int g = std::min(grid_for(n, kSensorThreads, h->sm_count), kWbMaxBlocks);
    double *partial = nullptr, *ratio = nullptr;
    if (sat_host) {
        PB_TRY(ensure_scratch(h, FOLD_SLOT, (size_t)(4 * g + 1) * sizeof(double), (void**)&partial));
        ratio = partial + 4 * g;
    }
    if (!with_real(dtype, [&](auto r) {
            using T = decltype(r);
            if (sat_host) {
                wb_plane_max_kernel<T><<<g, kSensorThreads, 0, st>>>((const T*)a, n, nx, kind, partial);
                wb_ratio_kernel<<<1, kSensorThreads, 0, st>>>(partial, g, nplanes, g4, ratio);
            }
            wb_scale_kernel<T><<<g, kSensorThreads, 0, st>>>((T*)a, n, nx, kind, g4, ratio);
        }))
        return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_demosaic_malvar(pb_handle_t hh, int in_type, const void* img, long long m, long long n, long long ld,
                                  int bggr, int out_type, void* out, void* stream) {
    PB_ENTER(hh);
    if (!img || !out || m < 1 || n < 1 || ld < n) return fail(h, PB_ERR_INVALID, "bad demosaic arguments");
    if ((m + kMalvarTY - 1) / kMalvarTY > 65535) return fail(h, PB_ERR_INVALID, "demosaic: too many rows");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const dim3 grid((unsigned)((n + kMalvarTX - 1) / kMalvarTX), (unsigned)((m + kMalvarTY - 1) / kMalvarTY));
    const dim3 block(kMalvarTX, kMalvarRows);
    bool ok = false;
    with_elem(in_type, [&](auto i) {
        using In = decltype(i);
        if constexpr (is_one_of<In, float, double, uint8_t, uint16_t>) {
            using S = typename std::conditional<std::is_same<In, double>::value, double, float>::type;
            if (out_type == PB_ELEM_F32 && !std::is_same<In, double>::value) {
                malvar_kernel<In, S, float><<<grid, block, 0, st>>>((const In*)img, m, n, ld, bggr, (float*)out);
                ok = true;
            } else if (out_type == PB_ELEM_F64) {
                malvar_kernel<In, S, double><<<grid, block, 0, st>>>((const In*)img, m, n, ld, bggr, (double*)out);
                ok = true;
            }
        }
    });
    if (!ok) return fail(h, PB_ERR_INVALID, "demosaic: unsupported input / output types");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_bayer_assemble(pb_handle_t hh, int dtype, const void* rp, const void* g2p, const void* bp, const void* g1,
                                 long long n, void* out, void* stream) {
    PB_ENTER(hh);
    if (!rp || !g2p || !bp || !g1 || !out || n < 0) return fail(h, PB_ERR_INVALID, "bad assemble arguments");
    if (n == 0) return PB_OK;
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int g = grid_for(n, kSensorThreads, h->sm_count);
    if (!with_real(dtype, [&](auto r) {
            using R = decltype(r);
            assemble_kernel<R><<<g, kSensorThreads, 0, st>>>((const cplx<R>*)rp, (const cplx<R>*)g2p, (const cplx<R>*)bp,
                                                             (const R*)g1, n, (R*)out);
        }))
        return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
