// Wavefront sensing (prysm/x/fibers.py, sri.py, pdi.py, psi.py): LP mode fields, the fused mode-coupling reduction,
// the interferometers' combine and grating passes, and the PSI accumulation.
//
// Every kernel computes in fp64 and rounds each stored value once.  No atomics, no host synchronisation: the
// coupling reduction writes per-chunk partials and a second launch sums them in a fixed order, so its result does
// not depend on scheduling and every call can be captured in a CUDA graph.  Per-launch tables (mode plans, mode
// pointers, PSI weights and frame pointers) travel in kernel-parameter space.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace pb {

namespace {

constexpr int kThreads = 256;
constexpr int kLpMax = 64;                 // mode plans per pb_lp_modes launch
constexpr int kOvGroup = 8;                // modes per stage-1 block: E is read once per eight modes
constexpr int kOvMax = 256;                // mode pointers per pb_overlap launch
constexpr int kPsiMax = 64;                // frames of pb_psi
constexpr double kEulerGamma = 0.57721566490153286061;

// ---- Bessel functions ----------------------------------------------------------------------------------------------
// J_l(x), x >= 0.  Orders 0 and 1 are CUDA's j0 / j1.  Above: forward recurrence from them where x > l (stable
// there), Miller's backward recurrence below, normalised by J0 + 2 (J2 + J4 + ...) = 1 and rescaled against overflow.
// (CUDA's jn returns NaN at x = 0 and carries ~1e-14 absolute error at moderate x.)  Below x = 1e-20 the leading term
// of the series, (x/2)^l / l!, is J_l to a relative 1e-40; Miller's rescaling by 1e-100 per step cannot keep up there
// once j * 2 / x passes 1e100, so the recurrence would overflow to NaN.
__device__ double bessel_j(int l, double x) {
    if (l == 0) return j0(x);
    if (l == 1) return j1(x);
    if (x < 1e-20) {
        double t = 1.0;
        for (int k = 1; k <= l; ++k) t *= 0.5 * x / k;
        return t;
    }
    const double tox = 2.0 / x;
    if (x > l) {
        double bjm = j0(x), bj = j1(x);
        for (int j = 1; j < l; ++j) {
            const double bjp = j * tox * bj - bjm;
            bjm = bj;
            bj = bjp;
        }
        return bj;
    }
    const int m = 2 * ((l + 24 + (int)sqrt(400.0 * l)) / 2);
    double bjp = 0.0, bj = 1.0, sum = 0.0, ans = 0.0;
    bool even = false;
    for (int j = m; j > 0; --j) {
        const double bjm = j * tox * bj - bjp;
        bjp = bj;
        bj = bjm;
        if (fabs(bj) > 1e100) {
            bj *= 1e-100;
            bjp *= 1e-100;
            ans *= 1e-100;
            sum *= 1e-100;
        }
        if (even) sum += bj;
        even = !even;
        if (j == l) ans = bjp;
    }
    return ans / (2.0 * sum - bj);
}

// e^x K0(x) and e^x K1(x), x > 0.  x <= 2: the ascending series (A&S 9.6.13 and 9.6.11 at n = 1) around I0 and I1;
// above: Steed's evaluation of Temme's continued fraction for K at order 0 (Temme, J. Comput. Phys. 19, 324 (1975)),
// which yields the scaled values directly.
__device__ void bessel_k01_scaled(double x, double& k0, double& k1) {
    if (x <= 2.0) {
        const double q = 0.25 * x * x, lg = log(0.5 * x);
        double t0 = 1.0, t1 = 1.0;                      // q^k / (k!)^2,  q^k / (k! (k+1)!)
        double hk = 0.0, ps = 1.0 - 2.0 * kEulerGamma;  // harmonic number H_k,  psi(k+1) + psi(k+2)
        double s0 = 0.0, s1 = ps;
        for (int k = 1; k < 20; ++k) {
            t0 *= q / ((double)k * k);
            t1 *= q / ((double)k * (k + 1));
            hk += 1.0 / k;
            ps += 1.0 / k + 1.0 / (k + 1);
            s0 += hk * t0;
            s1 += ps * t1;
        }
        const double e = exp(x);
        k0 = (s0 - (lg + kEulerGamma) * cyl_bessel_i0(x)) * e;
        k1 = (1.0 / x + lg * cyl_bessel_i1(x) - 0.25 * x * s1) * e;
        return;
    }
    double b = 2.0 * (1.0 + x), d = 1.0 / b, h = d, delh = d, q1 = 0.0, q2 = 1.0;
    const double a1 = 0.25;
    double q = a1, c = a1, a = -a1, s = 1.0 + q * delh;
    for (int i = 1; i < 1000; ++i) {
        a -= 2.0 * i;
        c = -a * c / (i + 1.0);
        const double qn = (q1 - b * q2) / a;
        q1 = q2;
        q2 = qn;
        q += c * qn;
        b += 2.0;
        d = 1.0 / (b + a * d);
        delh = (b * d - 1.0) * delh;
        h += delh;
        const double ds = q * delh;
        s += ds;
        if (fabs(ds) < 1e-17 * fabs(s)) break;
    }
    k0 = sqrt(3.14159265358979323846 / (2.0 * x)) / s;
    k1 = k0 * (x + 0.5 - a1 * h) / x;
}

// e^x K_l(x): upward recurrence K_{n+1} = K_{n-1} + (2n / x) K_n, stable for K
__device__ double bessel_k_scaled(int l, double x) {
    double k0, k1;
    bessel_k01_scaled(x, k0, k1);
    if (l == 0) return k0;
    for (int n = 1; n < l; ++n) {
        const double k2 = k0 + (2.0 * n / x) * k1;
        k0 = k1;
        k1 = k2;
    }
    return k1;
}

// ---- pb_lp_modes ---------------------------------------------------------------------------------------------------
struct LpMode { double U, W; int l, ld, rule, az; };
struct LpPlan { LpMode m[kLpMax]; };

template <typename R>
__global__ void __launch_bounds__(kThreads) lp_modes_kernel(const R* __restrict__ r, const R* __restrict__ t, long long n,
                                                            double a, LpPlan plan, R* __restrict__ out) {
    const LpMode m = plan.m[blockIdx.y];
    const double jd = bessel_j(m.ld, m.U), kd = bessel_k_scaled(m.ld, m.W);
    R* o = out + (long long)blockIdx.y * n;
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const double ri = (double)r[i];
        double rho;
        bool core;
        if (m.rule == PB_LP_RULE_LP) {          // fibers.py:371-373
            rho = ri / a;
            core = ri <= a;
        } else {                                // fibers.py:447-448
            rho = ri * (1.0 / a);
            core = rho < 1.0;
        }
        double v = core ? bessel_j(m.l, m.U * rho) / jd
                        : bessel_k_scaled(m.l, m.W * rho) / kd * exp(m.W * (1.0 - rho));
        if (m.az == PB_LP_COS) v *= cos(m.l * (double)t[i]);
        else if (m.az == PB_LP_SIN) v *= sin(m.l * (double)t[i]);
        o[i] = (R)v;
    }
}

// ---- pb_overlap ----------------------------------------------------------------------------------------------------
struct ModeTable { const void* p[kOvMax]; };

// stage 1: block (chunk, group) sums sum conj(M_p) E, sum |M_p|^2 of its eight modes over PB_OVERLAP_CHUNK pixels;
// the blocks of the first group of the first launch also sum |E|^2
template <typename R, bool MC>
__global__ void __launch_bounds__(kThreads) overlap_partial_kernel(const cplx<R>* __restrict__ E, long long n, int nmodes,
                                                                   int mode0, int nchunk, ModeTable tab, int need_ip,
                                                                   int need_ie, double* __restrict__ part,
                                                                   double* __restrict__ part_e) {
    constexpr int NV = kOvGroup * 3 + 1;
    __shared__ double sh[kThreads / 32][NV];
    const int chunk = blockIdx.x, g0 = blockIdx.y * kOvGroup, ng = min(kOvGroup, nmodes - g0);
    const bool do_e = need_ie && mode0 == 0 && blockIdx.y == 0;
    double acc[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) acc[k] = 0.0;
    const long long lo = (long long)chunk * PB_OVERLAP_CHUNK, hi = min(n, lo + PB_OVERLAP_CHUNK);
    for (long long i = lo + threadIdx.x; i < hi; i += kThreads) {
        const cplx<R> e = E[i];
        const double er = e.x, ei = e.y;
        if (do_e) acc[NV - 1] += er * er + ei * ei;
#pragma unroll
        for (int k = 0; k < kOvGroup; ++k) {
            if (k < ng) {
                double mr, mi = 0.0;
                if constexpr (MC) {
                    const cplx<R> m = reinterpret_cast<const cplx<R>*>(tab.p[g0 + k])[i];
                    mr = m.x;
                    mi = m.y;
                } else {
                    mr = reinterpret_cast<const R*>(tab.p[g0 + k])[i];
                }
                acc[3 * k] += mr * er + mi * ei;        // re conj(m) e
                acc[3 * k + 1] += mr * ei - mi * er;    // im conj(m) e
                if (need_ip) acc[3 * k + 2] += mr * mr + mi * mi;
            }
        }
    }
    warp_partials<kThreads>(acc, OpAdd{}, sh);
    const int v = threadIdx.x;
    if (v < NV) {
        double s = 0.0;
        for (int w = 0; w < kThreads / 32; ++w) s += sh[w][v];      // fixed order
        if (v == NV - 1) {
            if (do_e) part_e[chunk] = s;
        } else if (v / 3 < ng) {
            part[((long long)(mode0 + g0 + v / 3) * nchunk + chunk) * 3 + v % 3] = s;
        }
    }
}

// stage 2: block p sums the chunk partials of mode p in a fixed order and writes eta_p (and c for p = 0)
template <typename R>
__global__ void __launch_bounds__(kThreads) overlap_finish_kernel(const double* __restrict__ part,
                                                                  const double* __restrict__ part_e, int nchunk,
                                                                  const double* __restrict__ ip_in,
                                                                  const double* __restrict__ ie_in, R* __restrict__ eta,
                                                                  R* __restrict__ c_out) {
    __shared__ double sh[kThreads / 32][4];
    const int p = blockIdx.x;
    double s[4] = {0.0, 0.0, 0.0, 0.0};
    for (int k = threadIdx.x; k < nchunk; k += kThreads) {
        const double* q = part + ((long long)p * nchunk + k) * 3;
        s[0] += q[0];
        s[1] += q[1];
        if (!ip_in) s[2] += q[2];
        if (!ie_in) s[3] += part_e[k];
    }
    warp_partials<kThreads>(s, OpAdd{}, sh);
    if (threadIdx.x == 0) {
        double t[4] = {0.0, 0.0, 0.0, 0.0};
        for (int w = 0; w < kThreads / 32; ++w)
            for (int k = 0; k < 4; ++k) t[k] += sh[w][k];
        // eta = q^2 with q = |sum conj(M) E| / sqrt(I_p I_E) <= 1: formed without squaring a sum, so fields far from
        // unit magnitude (|E| ~ 1e150 or 1e-150 in fp64) neither overflow nor underflow
        const double ip = ip_in ? ip_in[p] : t[2], ie = ie_in ? ie_in[0] : t[3];
        const double q = hypot(t[0], t[1]) / sqrt(ip) / sqrt(ie);
        eta[p] = (R)(q * q);
        if (c_out && p == 0) c_out[0] = (R)(sqrt(ie) * q);
    }
}

// ---- pb_wfs_combine ------------------------------------------------------------------------------------------------
template <typename R, bool REAL_OUT>
__global__ void __launch_bounds__(kThreads) combine_kernel(long long n, const cplx<R>* __restrict__ a,
                                                           const cplx<R>* __restrict__ b, double ar, double ai, double br,
                                                           double bi, const R* __restrict__ as, const R* __restrict__ bs,
                                                           void* __restrict__ out) {
    if (as) { const double f = (double)*as; ar *= f; ai *= f; }
    if (bs) { const double f = (double)*bs; br *= f; bi *= f; }
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const cplx<R> x = a[i];
        double re = ar * x.x - ai * x.y, im = ar * x.y + ai * x.x;
        if (b) {
            const cplx<R> y = b[i];
            re += br * y.x - bi * y.y;
            im += br * y.y + bi * y.x;
        }
        if constexpr (REAL_OUT) reinterpret_cast<R*>(out)[i] = (R)(re * re + im * im);
        else reinterpret_cast<cplx<R>*>(out)[i] = mk<R>((R)re, (R)im);
    }
}

// ---- pb_grating ----------------------------------------------------------------------------------------------------
struct GratingParams { double v[6]; };

template <typename R>
__global__ void __launch_bounds__(kThreads) grating_kernel(int kind, long long n, const R* __restrict__ x, double shift,
                                                           GratingParams p, const cplx<R>* __restrict__ E,
                                                           void* __restrict__ out) {
    for (long long i = blockIdx.x * (long long)kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
        const double xv = (double)x[i] + shift;
        double g;
        if (kind == PB_GRATING_SIN_AMP) {                // pdi.py:132-145; v = prefix
            g = 1.0 - (sin(p.v[0] * xv) + 1.0) / 2.0 * 0.1;
        } else {                                         // pdi.py:37-51; v = period, edge, hi, lo, mid, eps
            const double period = p.v[0];
            double xw = fmod(xv, period);                // np.mod: the remainder takes the sign of the divisor
            if (xw != 0.0) {
                if ((period < 0.0) != (xw < 0.0)) xw += period;
            } else {
                xw = copysign(0.0, period);
            }
            g = xw < p.v[1] ? p.v[2] : p.v[3];
            if (fabs(xw) < p.v[5]) g = p.v[4];
        }
        if (E) {
            const cplx<R> e = E[i];
            reinterpret_cast<cplx<R>*>(out)[i] = mk<R>((R)(e.x * g), (R)(e.y * g));
        } else {
            reinterpret_cast<R*>(out)[i] = (R)g;
        }
    }
}

// ---- pb_psi --------------------------------------------------------------------------------------------------------
struct PsiPlan { double s[kPsiMax]; double c[kPsiMax]; const void* f[kPsiMax]; };

template <typename T, int V> struct alignas(sizeof(T) * V) Vec { T v[V]; };

// V pixels per thread, read as one 16-byte access per frame when V > 1; ACC is long long (integer frames, integer
// weights: exact) or double
template <typename T, int V, typename ACC, typename NT, typename PT>
__global__ void __launch_bounds__(kThreads) psi_kernel(int nf, long long groups, PsiPlan plan, NT* __restrict__ num,
                                                       NT* __restrict__ den, PT* __restrict__ phase) {
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < groups; g += (long long)gridDim.x * kThreads) {
        ACC s[V], c[V];
#pragma unroll
        for (int j = 0; j < V; ++j) s[j] = c[j] = 0;
        for (int k = 0; k < nf; ++k) {
            const Vec<T, V> f = reinterpret_cast<const Vec<T, V>*>(plan.f[k])[g];
            const ACC ws = (ACC)plan.s[k], wc = (ACC)plan.c[k];
#pragma unroll
            for (int j = 0; j < V; ++j) {
                s[j] += ws * (ACC)f.v[j];
                c[j] += wc * (ACC)f.v[j];
            }
        }
#pragma unroll
        for (int j = 0; j < V; ++j) {
            const long long i = g * V + j;
            if (num) num[i] = (NT)s[j];
            if (den) den[i] = (NT)c[j];
            if (phase) phase[i] = (PT)atan2((double)s[j], (double)c[j]);
        }
    }
}

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

}  // namespace pb

using namespace pb;

extern "C" int pb_lp_modes(pb_handle_t hh, int dtype, const void* r, const void* t, long long n, double a, int nmodes,
                           const double* plan_host, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0 || nmodes < 0 || !(a > 0)) return fail(h, PB_ERR_INVALID, "bad LP mode arguments");
    if (n == 0 || nmodes == 0) return PB_OK;
    if (!r || !out || !plan_host) return fail(h, PB_ERR_INVALID, "null pointer");
    std::vector<LpMode> modes(nmodes);
    for (int p = 0; p < nmodes; ++p) {
        const double* q = plan_host + 6 * p;
        LpMode& m = modes[p];
        m.l = (int)q[0];
        m.ld = (int)q[1];
        m.U = q[2];
        m.W = q[3];
        m.rule = (int)q[4];
        m.az = (int)q[5];
        if (m.l < 0 || m.ld < 0 || (m.rule != PB_LP_RULE_LP && m.rule != PB_LP_RULE_SMF) || m.az < PB_LP_NONE ||
            m.az > PB_LP_SIN)
            return fail(h, PB_ERR_INVALID, "bad LP mode plan entry");
        if (m.az != PB_LP_NONE && !t) return fail(h, PB_ERR_INVALID, "an azimuthal mode needs the angle grid");
    }
    const int gx = grid_for(n, kThreads, h->sm_count);
    for (int p0 = 0; p0 < nmodes; p0 += kLpMax) {
        LpPlan plan{};
        const int np = std::min(kLpMax, nmodes - p0);
        std::copy(modes.begin() + p0, modes.begin() + p0 + np, plan.m);
        const dim3 grid(gx, np);
        with_real(dtype, [&](auto real) {
            using R = decltype(real);
            lp_modes_kernel<R><<<grid, kThreads, 0, st>>>((const R*)r, (const R*)t, n, a, plan, (R*)out + (long long)p0 * n);
        });
        PB_LAUNCH_CHECK(h);
    }
    return PB_OK;
}

extern "C" int pb_overlap(pb_handle_t hh, int dtype, const void* E, long long n, int nmodes, const void* modes,
                          const void* const* mode_ptrs_host, int modes_complex, const double* ip_dev,
                          const double* ie_dev, void* eta, void* c_out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n <= 0 || nmodes <= 0) return fail(h, PB_ERR_INVALID, "bad overlap sizes");
    if (!E || !eta || (!modes && !mode_ptrs_host)) return fail(h, PB_ERR_INVALID, "null pointer");
    const long long nchunk_ll = (n + PB_OVERLAP_CHUNK - 1) / PB_OVERLAP_CHUNK;
    if (nchunk_ll > (1LL << 30)) return fail(h, PB_ERR_UNSUPPORTED, "field too large for the chunked reduction");
    const int nchunk = (int)nchunk_ll;
    double* part = nullptr;
    PB_TRY(ensure_scratch(h, FOLD_SLOT, (size_t)nchunk * (3 * nmodes + 1) * sizeof(double), (void**)&part));
    double* part_e = part + (long long)nmodes * nchunk * 3;
    const size_t esz = rsize(dtype) * (modes_complex ? 2 : 1);
    for (int p0 = 0; p0 < nmodes; p0 += kOvMax) {
        ModeTable tab{};
        const int np = std::min(kOvMax, nmodes - p0);
        for (int k = 0; k < np; ++k) {
            tab.p[k] = modes ? static_cast<const char*>(modes) + (size_t)(p0 + k) * n * esz : mode_ptrs_host[p0 + k];
            if (!tab.p[k]) return fail(h, PB_ERR_INVALID, "null mode pointer");
        }
        const dim3 grid(nchunk, (np + kOvGroup - 1) / kOvGroup);
        auto go = [&](auto r, auto mc) {
            using R = decltype(r);
            overlap_partial_kernel<R, decltype(mc)::value><<<grid, kThreads, 0, st>>>(
                reinterpret_cast<const cplx<R>*>(E), n, np, p0, nchunk, tab, ip_dev == nullptr, ie_dev == nullptr, part,
                part_e);
        };
        with_real(dtype, [&](auto r) {
            if (modes_complex) go(r, std::true_type()); else go(r, std::false_type());
        });
        PB_LAUNCH_CHECK(h);
    }
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        overlap_finish_kernel<R><<<nmodes, kThreads, 0, st>>>(part, part_e, nchunk, ip_dev, ie_dev, (R*)eta, (R*)c_out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_wfs_combine(pb_handle_t hh, int dtype, long long n, const void* a, const void* b,
                              const double* coefs_host, const void* alpha_scale, const void* beta_scale, int real_out,
                              void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0) return fail(h, PB_ERR_INVALID, "negative pixel count");
    if (n == 0) return PB_OK;
    if (!a || !out || !coefs_host) return fail(h, PB_ERR_INVALID, "null pointer");
    const double* k = coefs_host;
    const int grid = grid_for(n, kThreads, h->sm_count);
    auto go = [&](auto r, auto ro) {
        using R = decltype(r);
        combine_kernel<R, decltype(ro)::value><<<grid, kThreads, 0, st>>>(
            n, reinterpret_cast<const cplx<R>*>(a), reinterpret_cast<const cplx<R>*>(b), k[0], k[1], k[2], k[3],
            reinterpret_cast<const R*>(alpha_scale), reinterpret_cast<const R*>(beta_scale), out);
    };
    with_real(dtype, [&](auto r) {
        if (real_out) go(r, std::true_type()); else go(r, std::false_type());
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_grating(pb_handle_t hh, int dtype, int kind, long long n, const void* x, double shift,
                          const double* params_host, int nparams, const void* E, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0 || (kind != PB_GRATING_SIN_AMP && kind != PB_GRATING_RECTANGLE) ||
        nparams != (kind == PB_GRATING_SIN_AMP ? 1 : 6))
        return fail(h, PB_ERR_INVALID, "bad grating arguments");
    if (n == 0) return PB_OK;
    if (!x || !out || !params_host) return fail(h, PB_ERR_INVALID, "null pointer");
    GratingParams p{};
    std::copy(params_host, params_host + nparams, p.v);
    const int grid = grid_for(n, kThreads, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        grating_kernel<R><<<grid, kThreads, 0, st>>>(kind, n, (const R*)x, shift, p, (const cplx<R>*)E, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_psi(pb_handle_t hh, int frame_type, int nframes, const void* const* frames_host, const void* stack,
                      long long frame_stride, long long n, const double* s_host, const double* c_host, int num_type,
                      void* num, void* den, int phase_type, void* phase, void* stream) {
    PB_ENTER(hh);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const bool int_frames = frame_type == PB_ELEM_U16 || frame_type == PB_ELEM_I32;
    if ((frame_type != PB_ELEM_F32 && frame_type != PB_ELEM_F64 && !int_frames) || nframes < 1 || nframes > kPsiMax || n < 0)
        return fail(h, PB_ERR_INVALID, "bad PSI arguments");
    // output types follow numpy: float frames keep their type; integer frames give int64 (integer weights) or
    // float64 sums and a float64 phase
    const bool types_ok = int_frames ? ((num_type == PB_ELEM_I64 || num_type == PB_ELEM_F64) && phase_type == PB_ELEM_F64)
                                     : (num_type == frame_type && phase_type == frame_type);
    if (!types_ok) return fail(h, PB_ERR_INVALID, "PSI output types do not follow the frame type");
    if (n == 0) return PB_OK;
    if (!s_host || !c_host || (!frames_host && !stack) || (!num && !den && !phase))
        return fail(h, PB_ERR_INVALID, "null pointer");
    const size_t fsz = elem_size(frame_type);
    PsiPlan plan{};
    bool vec = true;
    for (int k = 0; k < nframes; ++k) {
        plan.s[k] = s_host[k];
        plan.c[k] = c_host[k];
        plan.f[k] = frames_host ? frames_host[k] : static_cast<const char*>(stack) + (size_t)k * frame_stride * fsz;
        if (!plan.f[k]) return fail(h, PB_ERR_INVALID, "null frame pointer");
        vec = vec && aligned16(plan.f[k]);
        if (num_type == PB_ELEM_I64 && (plan.s[k] != rint(plan.s[k]) || plan.c[k] != rint(plan.c[k])))
            return fail(h, PB_ERR_INVALID, "int64 PSI sums need integer weights");
    }
    vec = vec && n % (long long)(16 / fsz) == 0 && aligned16(num) && aligned16(den) && aligned16(phase);
    auto go = [&](auto t, auto v, auto acc, auto nt, auto pt) {
        using T = decltype(t);
        constexpr int V = decltype(v)::value;
        using NT = decltype(nt);
        using PT = decltype(pt);
        const long long groups = n / V;
        psi_kernel<T, V, decltype(acc), NT, PT><<<grid_for(groups, kThreads, h->sm_count), kThreads, 0, st>>>(
            nframes, groups, plan, (NT*)num, (NT*)den, (PT*)phase);
        h->route_launches[route_code(PB_ROUTE_PSI, V, std::is_same<decltype(acc), long long>::value)]++;
    };
    auto dispatch = [&](auto t, auto vv) {
        using T = decltype(t);
        if constexpr (std::is_floating_point<T>::value) {
            go(t, vv, double(), T(), T());
        } else {
            if (num_type == PB_ELEM_I64) go(t, vv, (long long)0, (long long)0, double());
            else go(t, vv, double(), double(), double());
        }
    };
    with_elem(frame_type, [&](auto t) {
        using T = decltype(t);
        if constexpr (is_one_of<T, float, double, uint16_t, int32_t>) {
            if (vec) dispatch(t, std::integral_constant<int, 16 / sizeof(T)>());
            else dispatch(t, std::integral_constant<int, 1>());
        }
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
