// Streaming elementwise kernels and small reductions on the path (all HBM-bound):
// phase-screen synthesis, |.|^2 (+ weighted accumulate), separable multiplies, weighted mode
// sum, OTF normalisation, first moments, angular-spectrum factor vectors, MDFT bases.
#include "common.cuh"
#include "czt.cuh"

namespace pb {

// out[i] = amp * exp(2 pi i kturns opd) over the n elements of a dense array of rows of nx; opd and amp are read with
// row pitch ld (elements)
template <typename R>
__global__ void phase_screen_kernel(const void* amp, int amp_kind, const R* __restrict__ opd, double kturns,
                                    long long n, long long nx, long long ld, cplx<R>* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const long long s = ld == nx ? i : i / nx * ld + i % nx;
        R a = R(1);
        if (amp_kind == PB_AMP_REAL) a = reinterpret_cast<const R*>(amp)[s];
        else if (amp_kind == PB_AMP_U8) a = reinterpret_cast<const unsigned char*>(amp)[s] ? R(1) : R(0);
        cplx<R> e = mk<R>(R(0), R(0));
        if (a != R(0)) {
            e = expi_turns(kturns * (double)opd[s], R(0));
            e.x *= a; e.y *= a;
        }
        out[i] = e;
    }
}

int launch_phase_screen(Handle* h, int dtype, const void* amp, int amp_kind, const void* opd, double kturns, long long count,
                        long long nx, long long ld, void* out, cudaStream_t st) {
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        phase_screen_kernel<R><<<g, 256, 0, st>>>(amp, amp_kind, (const R*)opd, kturns, count, nx, ld, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

template <typename R>
__global__ void intensity_kernel(const cplx<R>* __restrict__ in, long long n, R weight, int accumulate,
                                 R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        cplx<R> v = in[i];
        R I = v.x * v.x + v.y * v.y;
        if (accumulate) out[i] += weight * I; else out[i] = weight * I;
    }
}

template <typename R>
__global__ void mul_outer_kernel(const cplx<R>* __restrict__ in, long long in_ld, int ny, int nx,
                                 const cplx<R>* __restrict__ vy, int conj_y, const cplx<R>* __restrict__ vx,
                                 int conj_x, R scale, cplx<R>* __restrict__ out, long long out_ld) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        cplx<R> v = in[y * in_ld + x];
        if (vy) { cplx<R> m = vy[y]; v = conj_y ? cmulc(v, m) : cmul(v, m); }
        if (vx) { cplx<R> m = vx[x]; v = conj_x ? cmulc(v, m) : cmul(v, m); }
        v.x *= scale; v.y *= scale;
        out[y * out_ld + x] = v;
    }
}

// Complex division in fp64, rounded once to R by the caller: x * w with w = conj(y) / |y|^2.  For float operands the
// fp64 |y|^2 neither overflows nor goes subnormal anywhere in the float range (in R = float it overflows above
// |y| ~ 1.8e19 and loses bits below ~1e-19); for double operands it holds for 1e-154 < |y| < 1e154 (DESIGN.md §4.4).
// One fp64 reciprocal per divisor: no slower than the two float divisions it replaces.
template <typename R>
__device__ inline double2 crecip_fp64(cplx<R> y) {
    const double yx = y.x, yy = y.y, inv = 1.0 / (yx * yx + yy * yy);
    return make_double2(yx * inv, -yy * inv);
}

template <typename R>
__device__ inline double2 cmul_fp64(cplx<R> x, double2 w) {
    return make_double2((double)x.x * w.x - (double)x.y * w.y, (double)x.x * w.y + (double)x.y * w.x);
}

// out = a (op) b, or with b == nullptr a (op) scalar; reverse swaps the operands.  op: 0 mul, 1 div, 2 add, 3 sub
template <typename R>
__global__ void binary_kernel(int op, const cplx<R>* __restrict__ a, const cplx<R>* __restrict__ b, cplx<R> sc,
                              int reverse, long long n, cplx<R>* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        cplx<R> x = a[i], y = b ? b[i] : sc;
        if (reverse) { cplx<R> t = x; x = y; y = t; }
        cplx<R> r;
        if (op == 0) r = cmul(x, y);
        else if (op == 1) { const double2 q = cmul_fp64<R>(x, crecip_fp64<R>(y)); r = mk<R>((R)q.x, (R)q.y); }
        else if (op == 2) r = cadd(x, y);
        else r = csub(x, y);
        out[i] = r;
    }
}

#define PB_MAX_MODES 64
template <typename R> struct ModeWeights { R w[PB_MAX_MODES]; };

template <typename R>
__global__ void weighted_sum_kernel(const R* __restrict__ modes, int k, long long n, ModeWeights<R> w, int accumulate,
                                    R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        R acc = accumulate ? out[i] : R(0);
        for (int m = 0; m < k; ++m) acc += w.w[m] * modes[(long long)m * n + i];
        out[i] = acc;
    }
}

template <typename R>
__global__ void otf_normalize_kernel(const cplx<R>* __restrict__ D, long long n, long long centre, int which,
                                     R* __restrict__ mtf, R* __restrict__ ptf, cplx<R>* __restrict__ otf) {
    const double2 w = crecip_fp64<R>(D[centre]);
    PB_GRID_STRIDE(i, n) {
        const double2 qd = cmul_fp64<R>(D[i], w);
        const cplx<R> q = mk<R>((R)qd.x, (R)qd.y);      // the quotient, rounded once to R
        if (which & 1) mtf[i] = hypot(q.x, q.y);
        if (which & 2) ptf[i] = atan2(q.y, q.x);
        if (which & 4) otf[i] = q;
    }
}

template <typename R>
__global__ void moments_kernel(const R* __restrict__ d, int ny, int nx, double* __restrict__ part, unsigned* __restrict__ counter,
                               double* __restrict__ sums) {
    double s[3] = {0, 0, 0};     // sum v, sum v y, sum v x
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        const double v = (double)d[i];
        s[0] += v; s[1] += v * y; s[2] += v * x;
    }
    block_reduce<256>(s, OpAdd{});
    if (threadIdx.x == 0) { double* p = part + blockIdx.x * 3; p[0] = s[0]; p[1] = s[1]; p[2] = s[2]; }
    if (!arrive_last(counter)) return;
    s[0] = fold_partials<256, 3>(part, 0, OpAdd{}, 0.0);
    s[1] = fold_partials<256, 3>(part, 1, OpAdd{}, 0.0);
    s[2] = fold_partials<256, 3>(part, 2, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { sums[0] = s[0]; sums[1] = s[1]; sums[2] = s[2]; }
}

// Baliga & Cohn encircled energy: r * sum( MTF * J1(2 pi r nu) / nu ) * dnu^2 on the fftrange*df grid, nu(0) -> 1e-16
// (prysm/otf.py:319-414).  One folded reduction per radius (grid row blockIdx.y), fp64 Bessel and accumulation.
template <typename R>
__global__ void encircled_energy_kernel(const R* __restrict__ mtf, int ny, int nx, double df, const double* __restrict__ radii,
                                        double* __restrict__ part, unsigned* __restrict__ counters, double* __restrict__ out) {
    const double r = radii[blockIdx.y];
    const long long n = (long long)ny * nx;
    double acc = 0.0;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        const double fy = (double)(y - ny / 2) * df, fx = (double)(x - nx / 2) * df;
        double nu = hypot(fx, fy);
        if (nu == 0.0) nu = 1e-16;
        acc += (double)mtf[i] * j1(6.283185307179586476925 * r * nu) / nu;
    }
    acc = block_reduce<256>(acc, OpAdd{});
    if (threadIdx.x == 0) part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = acc;
    if (!arrive_last(counters)) return;
    acc = fold_partials<256, 1>(part, 0, OpAdd{}, 0.0);
    if (threadIdx.x == 0) out[blockIdx.y] = acc * r * df * df;
}

// Bluestein pieces of one CZT axis built on the device from scalars (prysm/fttools.py:372-389, 277-281):
//   b[n]    = exp(sign*i*pi*alpha*n^2),            n = -(N/2) .. ;      N entries
//   post[m] = exp(sign*i*pi*alpha*(m+shift)^2) * exp(sign*2*pi*i*xc*f[m]),  f[m] = f0 + m*df;   M entries
//   h[d]    = exp(-sign*i*pi*alpha*(d+shift)^2),   d = m0-n_last .. m_last-n0, zero-extended to K entries
// all phases in fp64 turns, reduced before the sincos.
template <typename R>
__global__ void czt_plan_kernel(int N, int M, int K, double shift, double alpha, int sign, double xc, double f0, double df,
                                cplx<R>* __restrict__ b, cplx<R>* __restrict__ post, cplx<R>* __restrict__ hk) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const double half = 0.5 * sign * alpha;
    if (i < N) {
        const double n = (double)(i - N / 2);
        b[i] = expi_turns(half * n * n, R(0));
    }
    if (i < M) {
        const double q = (double)(i - M / 2) + shift;
        post[i] = expi_turns(half * q * q + sign * xc * (f0 + i * df), R(0));
    }
    if (i < K) {
        const int nd = N + M - 1;
        cplx<R> v = mk<R>(R(0), R(0));
        if (i < nd) {
            const double d = (double)(i + (-(M / 2)) - (-(N / 2) + N - 1)) + shift;   // m0 - n_last + i + shift
            v = expi_turns(-half * d * d, R(0));
        }
        hk[i] = v;
    }
}

// Hadj[k] = conj(H[k]) * exp(-2*pi*i*(N-1)*k/K): the adjoint's embedding at offset N-1 as a spectral phase
template <typename R>
__global__ void czt_hadj_kernel(int N, int K, const cplx<R>* __restrict__ H, cplx<R>* __restrict__ Hadj) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= K) return;
    const long long r = ((long long)(N - 1) * k) % K;
    const cplx<R> ph = expi_turns(-(double)r / (double)K, R(0));
    Hadj[k] = cmul(cconj(H[k]), ph);
}

// exp(-i*pi*wvl_mm*z*k^2), k = fftfreq(n, dx).  The phase is formed in fp64 for both dtypes
// (the reference rounds k to float32 first when precision=32, costing it ~1e-4 rad at C5 sizes).
template <typename R>
__global__ void as_vector_kernel(int n, double wvl_mm, double dx, double z, cplx<R>* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int fi = i < (n + 1) / 2 ? i : i - n;      // numpy fftfreq ordering
    const double kf = (double)fi / ((double)n * dx);
    const double k2 = kf * kf;                        // kept in fp64: the complex64 path then tracks the fp64 reference
    out[i] = expi_turns(-0.5 * wvl_mm * z * k2, R(0));  // -pi*w*z*k^2 rad = -(w*z*k^2)/2 turns
}

template <typename R>
__global__ void mdft_basis_kernel(const double* __restrict__ f, int m, const double* __restrict__ x, int n, int sign,
                                  cplx<R>* __restrict__ E) {
    const long long tot = (long long)m * n;
    PB_GRID_STRIDE(i, tot) {
        const int j = (int)(i / n), l = (int)(i - (long long)j * n);
        E[i] = expi_turns(sign * f[j] * x[l], R(0));
    }
}

}  // namespace pb

using namespace pb;

extern "C" int pb_phase_screen(pb_handle_t hh, int dtype, const void* amp, int amp_kind, const void* opd,
                               double kscale, long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (count <= 0) return PB_OK;
    return launch_phase_screen(h, dtype, amp, amp_kind, opd, kscale / (2.0 * M_PI), count, count, count, out, st);
}

extern "C" int pb_intensity(pb_handle_t hh, int dtype, const void* in, long long count, double weight, int accumulate,
                            void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        intensity_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)in, count, (R)weight, accumulate, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_binary(pb_handle_t hh, int dtype, int op, const void* a, const void* b, double s_re, double s_im,
                         int reverse, long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (op < 0 || op > 3 || !a || !out) return fail(h, PB_ERR_INVALID, "bad binary-op arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        binary_kernel<R><<<g, 256, 0, st>>>(op, (const cplx<R>*)a, (const cplx<R>*)b, mk<R>((R)s_re, (R)s_im), reverse, count, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_mul_outer(pb_handle_t hh, int dtype, const void* in, long long in_ld, int ny, int nx, const void* vy,
                            int conj_y, const void* vx, int conj_x, double scale, void* out, long long out_ld,
                            void* stream) {
    PB_ENTER_REAL(hh);
    if (ny <= 0 || nx <= 0) return PB_OK;
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        mul_outer_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)in, in_ld, ny, nx, (const cplx<R>*)vy, conj_y, (const cplx<R>*)vx,
                                               conj_x, (R)scale, (cplx<R>*)out, out_ld);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_weighted_sum(pb_handle_t hh, int dtype, const void* modes, int k, long long count,
                               const double* weights_host, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (k < 1 || count <= 0 || !weights_host) return fail(h, PB_ERR_INVALID, "bad mode count / weights");
    const int g = grid_for(count, 256, h->sm_count);
    for (int k0 = 0; k0 < k; k0 += PB_MAX_MODES) {
        const int kk = std::min(PB_MAX_MODES, k - k0);
        with_real(dtype, [&](auto r) {
            using R = decltype(r);
            ModeWeights<R> w;
            for (int i = 0; i < kk; ++i) w.w[i] = (R)weights_host[k0 + i];
            weighted_sum_kernel<R><<<g, 256, 0, st>>>((const R*)modes + (long long)k0 * count, kk, count, w, k0 > 0, (R*)out);
        });
        PB_LAUNCH_CHECK(h);
    }
    return PB_OK;
}

extern "C" int pb_otf_normalize(pb_handle_t hh, int dtype, const void* D, int ny, int nx, int which, void* mtf,
                                void* ptf, void* otf, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "bad shape");
    const long long n = (long long)ny * nx, centre = (long long)(ny / 2) * nx + nx / 2;
    const int g = grid_for(n, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        otf_normalize_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)D, n, centre, which, (R*)mtf, (R*)ptf, (cplx<R>*)otf);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_moments(pb_handle_t hh, int dtype, const void* data, int ny, int nx, double* sums_host,
                          void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || !sums_host) return fail(h, PB_ERR_INVALID, "bad shape");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    double *part, *sums; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, g, 3, st, &part, &counter));
    PB_TRY(ensure_scratch(h, 2, 3 * sizeof(double), (void**)&sums));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        moments_kernel<R><<<g, 256, 0, st>>>((const R*)data, ny, nx, part, counter, sums);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaMemcpyAsync(sums_host, sums, 3 * sizeof(double), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_encircled_energy(pb_handle_t hh, int dtype, const void* mtf, int ny, int nx, double df,
                                   const double* radii_mm_host, int nr, double* out_host, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || nr < 1 || !mtf || !radii_mm_host || !out_host) return fail(h, PB_ERR_INVALID, "bad encircled-energy arguments");
    void* d = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)2 * nr * sizeof(double), &d));
    double* dr = (double*)d;
    double* dout = dr + nr;
    PB_CUDA(h, cudaMemcpyAsync(dr, radii_mm_host, nr * sizeof(double), cudaMemcpyHostToDevice, st));
    const int gx = fold_blocks((long long)ny * nx, h->sm_count);
    double* part; unsigned* counters;
    PB_TRY(fold_scratch(h, nr, gx, 1, st, &part, &counters));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        encircled_energy_kernel<R><<<dim3(gx, nr), 256, 0, st>>>((const R*)mtf, ny, nx, df, dr, part, counters, dout);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaMemcpyAsync(out_host, dout, nr * sizeof(double), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

int pb::czt_plan_impl(Handle* h, pb_handle_t hh, int dtype, int N, int M, int K, double shift, double alpha, int sign, double xc,
                      double f0, double df, void* b, void* post, void* H, void* Hadj, void* hk, void* stream) {
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int n = std::max(K, std::max(N, M));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        czt_plan_kernel<R><<<(n + 255) / 256, 256, 0, st>>>(N, M, K, shift, alpha, sign, xc, f0, df, (cplx<R>*)b, (cplx<R>*)post,
                                                           (cplx<R>*)hk);
    });
    PB_LAUNCH_CHECK(h);
    PB_TRY(pb_fft1(hh, dtype, hk, 1, K, K, 1, K, -1, 1.0, H, K, stream));   // H = FFT_K(h)
    if (Hadj) {
        with_real(dtype, [&](auto r) {
            using R = decltype(r);
            czt_hadj_kernel<R><<<(K + 255) / 256, 256, 0, st>>>(N, K, (const cplx<R>*)H, (cplx<R>*)Hadj);
        });
        PB_LAUNCH_CHECK(h);
    }
    return PB_OK;
}

extern "C" int pb_czt_plan(pb_handle_t hh, int dtype, int N, int M, int K, double shift, double alpha, int sign, double xc,
                           double f0, double df, void* b, void* post, void* H, void* Hadj, void* stream) {
    PB_ENTER_REAL(hh);
    (void)st;
    if (N < 1 || M < 1 || K < N + M - 1 || (sign != 1 && sign != -1) || !b || !post || !H || !Hadj)
        return fail(h, PB_ERR_INVALID, "bad czt plan arguments");
    void* hk = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)K * csize(dtype), &hk));
    return czt_plan_impl(h, hh, dtype, N, M, K, shift, alpha, sign, xc, f0, df, b, post, H, Hadj, hk, stream);
}

extern "C" int pb_angular_spectrum_vectors(pb_handle_t hh, int dtype, int ky, int kx, double wvl_um, double dx_mm,
                                           double z_mm, void* ty, void* tx, void* stream) {
    PB_ENTER_REAL(hh);
    if (ky < 1 || kx < 1) return fail(h, PB_ERR_INVALID, "bad shape");
    const double w = wvl_um / 1e3;
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        as_vector_kernel<R><<<(ky + 255) / 256, 256, 0, st>>>(ky, w, dx_mm, z_mm, (cplx<R>*)ty);
        as_vector_kernel<R><<<(kx + 255) / 256, 256, 0, st>>>(kx, w, dx_mm, z_mm, (cplx<R>*)tx);
    });
    PB_LAUNCH_CHECK(h);
    h->launches++;
    return PB_OK;
}

extern "C" int pb_mdft_basis(pb_handle_t hh, int dtype, const double* f_host, int m, const double* x_host, int n,
                             int sign, void* E, void* stream) {
    PB_ENTER_REAL(hh);
    if (m < 1 || n < 1 || !f_host || !x_host || (sign != 1 && sign != -1)) return fail(h, PB_ERR_INVALID, "bad basis arguments");
    void* d = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)(m + n) * sizeof(double), &d));
    double* df = (double*)d;
    double* dxv = df + m;
    // pageable host memory: the copies return after staging, so the caller's arrays may be freed
    PB_CUDA(h, cudaMemcpyAsync(df, f_host, m * sizeof(double), cudaMemcpyHostToDevice, st));
    PB_CUDA(h, cudaMemcpyAsync(dxv, x_host, n * sizeof(double), cudaMemcpyHostToDevice, st));
    const int g = grid_for((long long)m * n, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        mdft_basis_kernel<R><<<g, 256, 0, st>>>(df, m, dxv, n, sign, (cplx<R>*)E);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
