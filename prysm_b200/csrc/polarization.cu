// Jones calculus (prysm/x/polarization.py): four streaming per-pixel passes over element-planar arrays.
//
// Layout.  A Jones array of n pixels is four contiguous planes of n complex samples, plane 2*i + j holding J[..., i, j];
// a Mueller or Kronecker array is sixteen planes, plane 4*r + c.  Every kernel reads and writes whole planes with
// consecutive threads on consecutive pixels.  At complex64 a thread owns two adjacent pixels, so each plane access is
// one 16-byte load or store (complex128 is 16 bytes per pixel already); a misaligned plane or an odd pixel count at
// complex64 runs the same code one pixel per thread.  All arithmetic is fp64 and each stored value is rounded once.
// No atomics, no shared memory, no host synchronisation: every call can be captured in a CUDA graph.
#include <algorithm>
#include <cmath>

#include "common.cuh"

namespace pb {

namespace {

constexpr int kThreads = 256;

struct Z { double re, im; };
__device__ __forceinline__ Z zmul(Z a, Z b) { return {a.re * b.re - a.im * b.im, a.re * b.im + a.im * b.re}; }
__device__ __forceinline__ Z zadd(Z a, Z b) { return {a.re + b.re, a.im + b.im}; }
__device__ __forceinline__ Z zsub(Z a, Z b) { return {a.re - b.re, a.im - b.im}; }
__device__ __forceinline__ Z zconj(Z a) { return {a.re, -a.im}; }
__device__ __forceinline__ Z zscale(Z a, double s) { return {a.re * s, a.im * s}; }

// V pixels of one complex plane, moved as one 16-byte access when V == 2 (complex64) or V == 1 at complex128
template <typename R, int V> struct Px { Z v[V]; };

template <typename R, int V>
__device__ __forceinline__ Px<R, V> ld(const cplx<R>* __restrict__ p, long long g) {
    Px<R, V> r;
    if constexpr (V == 2) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(p) + g);
        r.v[0] = {t.x, t.y};
        r.v[1] = {t.z, t.w};
    } else {
        const cplx<R> t = p[g];
        r.v[0] = {(double)t.x, (double)t.y};
    }
    return r;
}

template <typename R, int V>
__device__ __forceinline__ void st(cplx<R>* __restrict__ p, long long g, const Z (&v)[V]) {
    if constexpr (V == 2) {
        reinterpret_cast<float4*>(p)[g] = make_float4((float)v[0].re, (float)v[0].im, (float)v[1].re, (float)v[1].im);
    } else {
        p[g] = mk<R>((R)v[0].re, (R)v[0].im);
    }
}

template <typename R, int V>
__device__ __forceinline__ void st_real(R* __restrict__ p, long long g, const double (&v)[V]) {
    if constexpr (V == 2) reinterpret_cast<float2*>(p)[g] = make_float2((float)v[0], (float)v[1]);
    else p[g] = (R)v[0];
}

__device__ __forceinline__ double ld_real(const void* p, int type, long long i) {
    return type == PB_ELEM_F32 ? (double)reinterpret_cast<const float*>(p)[i] : reinterpret_cast<const double*>(p)[i];
}

template <typename R> __device__ __forceinline__ double ld_plain(const R* __restrict__ p, long long i) { return (double)p[i]; }

// ---- pb_jones_planar ---------------------------------------------------------------------------------------------
// strided (rows, cols, 2, 2) of any real or complex type -> 4 planes; one thread per V pixels
template <typename T, bool CPLX, typename R, int V>
__global__ void __launch_bounds__(kThreads) jones_planar_kernel(const T* __restrict__ src, long long cols, long long s_row,
                                                                long long s_col, long long s_i, long long s_j, long long groups,
                                                                long long n, cplx<R>* __restrict__ out) {
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < groups; g += (long long)gridDim.x * kThreads) {
        Z e[4][V];
#pragma unroll
        for (int s = 0; s < V; ++s) {
            const long long p = g * V + s, r = p / cols, c = p - r * cols;
            const T* base = src + (r * s_row + c * s_col) * (CPLX ? 2 : 1);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const long long o = ((k >> 1) * s_i + (k & 1) * s_j) * (CPLX ? 2 : 1);
                e[k][s] = CPLX ? Z{(double)base[o], (double)base[o + 1]} : Z{(double)base[o], 0.0};
            }
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) st<R, V>(out + k * n, g, e[k]);
    }
}

// ---- pb_jones_product --------------------------------------------------------------------------------------------
struct JonesConsts { double v[16]; };   // A's four complex values, then B's

template <typename R, int V>
__device__ __forceinline__ void load_operand(int kind, const void* p, int op, const double* c, long long n, long long g,
                                             Z (&e)[4][V]) {
    if (kind == PB_JONES_CONST) {
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int s = 0; s < V; ++s) e[k][s] = {c[2 * k], c[2 * k + 1]};
    } else if (kind == PB_JONES_PLANES) {
        const cplx<R>* q = reinterpret_cast<const cplx<R>*>(p);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const Px<R, V> t = ld<R, V>(q + k * n, g);
#pragma unroll
            for (int s = 0; s < V; ++s) e[k][s] = t.v[s];
        }
    } else {
        Z t[V];
        if (kind == PB_JONES_SCALAR) {
            const Px<R, V> u = ld<R, V>(reinterpret_cast<const cplx<R>*>(p), g);
#pragma unroll
            for (int s = 0; s < V; ++s) t[s] = u.v[s];
        } else {
#pragma unroll
            for (int s = 0; s < V; ++s) t[s] = {ld_plain(reinterpret_cast<const R*>(p), g * V + s), 0.0};
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int s = 0; s < V; ++s) e[k][s] = t[s];
    }
    if (op == PB_JONES_OP_H) {
#pragma unroll
        for (int s = 0; s < V; ++s) {
            const Z a01 = e[1][s];
            e[0][s] = zconj(e[0][s]);
            e[1][s] = zconj(e[2][s]);
            e[2][s] = zconj(a01);
            e[3][s] = zconj(e[3][s]);
        }
    }
}

template <typename R, int V>
__global__ void __launch_bounds__(kThreads) jones_product_kernel(int mode, long long groups, long long n, int a_kind,
                                                                 const void* a, int a_op, int b_kind, const void* b, int b_op,
                                                                 JonesConsts k, cplx<R>* __restrict__ out) {
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < groups; g += (long long)gridDim.x * kThreads) {
        Z A[4][V], B[4][V], O[4][V];
        load_operand<R, V>(a_kind, a, a_op, k.v, n, g, A);
        load_operand<R, V>(b_kind, b, b_op, k.v + 8, n, g, B);
#pragma unroll
        for (int s = 0; s < V; ++s) {
            if (mode == PB_JONES_MATMUL) {
                O[0][s] = zadd(zmul(A[0][s], B[0][s]), zmul(A[1][s], B[2][s]));
                O[1][s] = zadd(zmul(A[0][s], B[1][s]), zmul(A[1][s], B[3][s]));
                O[2][s] = zadd(zmul(A[2][s], B[0][s]), zmul(A[3][s], B[2][s]));
                O[3][s] = zadd(zmul(A[2][s], B[1][s]), zmul(A[3][s], B[3][s]));
            } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) O[e][s] = zmul(A[e][s], B[e][s]);
            }
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) st<R, V>(out + e * n, g, O[e]);
    }
}

// ---- pb_jones_elements -------------------------------------------------------------------------------------------
struct JonesParams { double v[8]; };

// R(-t) @ M @ R(t) with R(t) = [[cos t, sin t], [-sin t, cos t]] (polarization.py:133-160, 195, 230, 344)
__device__ __forceinline__ void rotate_about(double t, Z (&m)[4]) {
    double s, c;
    sincos(t, &s, &c);
    // M @ R(t)
    const Z a0 = zsub(zscale(m[0], c), zscale(m[1], s)), a1 = zadd(zscale(m[0], s), zscale(m[1], c));
    const Z a2 = zsub(zscale(m[2], c), zscale(m[3], s)), a3 = zadd(zscale(m[2], s), zscale(m[3], c));
    // R(-t) @ (M @ R(t)), R(-t) = [[c, -s], [s, c]]
    m[0] = zsub(zscale(a0, c), zscale(a2, s));
    m[1] = zsub(zscale(a1, c), zscale(a3, s));
    m[2] = zadd(zscale(a0, s), zscale(a2, c));
    m[3] = zadd(zscale(a1, s), zscale(a3, c));
}

template <typename R, int V>
__global__ void __launch_bounds__(kThreads) jones_elements_kernel(int kind, long long groups, long long n, const void* plane,
                                                                  int plane_type, JonesParams p, cplx<R>* __restrict__ out) {
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < groups; g += (long long)gridDim.x * kThreads) {
        Z O[4][V];
#pragma unroll
        for (int s = 0; s < V; ++s) {
            Z m[4];
            if (kind == PB_JONES_FILL) {
#pragma unroll
                for (int e = 0; e < 4; ++e) m[e] = {p.v[2 * e], p.v[2 * e + 1]};
            } else if (kind == PB_JONES_ROTATION) {      // params: theta, scale of the plane
                const double t = plane ? ld_real(plane, plane_type, g * V + s) * p.v[1] : p.v[0];
                double sn, cs;
                sincos(t, &sn, &cs);
                m[0] = {cs, 0.0}; m[1] = {sn, 0.0}; m[2] = {-sn, 0.0}; m[3] = {cs, 0.0};
            } else if (kind == PB_JONES_RETARDER || kind == PB_JONES_DIATTENUATOR) {    // params: theta, retardance | alpha
                const double q = plane ? ld_real(plane, plane_type, g * V + s) : p.v[1];
                Z d = {q, 0.0};
                if (kind == PB_JONES_RETARDER) sincos(q, &d.im, &d.re);
                m[0] = {1.0, 0.0}; m[1] = {0.0, 0.0}; m[2] = {0.0, 0.0}; m[3] = d;
                rotate_about(p.v[0], m);
            } else {                                       // PB_JONES_VVR; params: charge, retardance, rotate
                const double t = ld_real(plane, plane_type, g * V + s) * p.v[0];
                double sn, cs, sr, cr;
                sincos(t, &sn, &cs);
                sincos(p.v[1] / 2, &sr, &cr);
                // jsinr * [[cos, sin], [sin, -cos]] + [[-i cos(ret/2), 0], [0, 0]]: the reference writes the
                // constant term to [0, 0] twice and never to [1, 1] (polarization.py:339-340)
                m[0] = {cs * sr, -cr}; m[1] = {sn * sr, 0.0}; m[2] = {sn * sr, 0.0}; m[3] = {-cs * sr, 0.0};
                rotate_about(p.v[2], m);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) O[e][s] = m[e];
        }
#pragma unroll
        for (int e = 0; e < 4; ++e) st<R, V>(out + e * n, g, O[e]);
    }
}

// ---- pb_jones_reduce ---------------------------------------------------------------------------------------------
// Rows of U = [[1, 0, 0, 1], [1, 0, 0, -1], [0, 1, 1, 0], [0, i, -i, 0]] / sqrt(2) (polarization.py:395-399) applied
// to v, and v applied to the columns of U^H (U is unitary, so U^-1 = U^H).  The 1/sqrt(2) of both is the 1/2 below.
__device__ __forceinline__ Z u_row(int r, const Z (&v)[4]) {
    switch (r) {
        case 0: return zadd(v[0], v[3]);
        case 1: return zsub(v[0], v[3]);
        case 2: return zadd(v[1], v[2]);
        default: { const Z d = zsub(v[1], v[2]); return {-d.im, d.re}; }          // i (v1 - v2)
    }
}
__device__ __forceinline__ Z uh_col(int c, const Z (&v)[4]) {
    switch (c) {
        case 0: return zadd(v[0], v[3]);
        case 1: return zsub(v[0], v[3]);
        case 2: return zadd(v[1], v[2]);
        default: { const Z d = zsub(v[1], v[2]); return {d.im, -d.re}; }          // -i (v1 - v2)
    }
}

template <typename R, int V>
__global__ void __launch_bounds__(kThreads) jones_reduce_kernel(int kind, long long groups, long long n,
                                                                const cplx<R>* __restrict__ a, const cplx<R>* __restrict__ b,
                                                                void* __restrict__ out) {
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < groups; g += (long long)gridDim.x * kThreads) {
        Z A[4][V];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const Px<R, V> t = ld<R, V>(a + e * n, g);
#pragma unroll
            for (int s = 0; s < V; ++s) A[e][s] = t.v[s];
        }
        if (kind == PB_JONES_PAULI) {     // polarization.py:470-473
            cplx<R>* o = reinterpret_cast<cplx<R>*>(out);
            Z c[4][V];
#pragma unroll
            for (int s = 0; s < V; ++s) {
                c[0][s] = zscale(zadd(A[0][s], A[3][s]), 0.5);
                c[1][s] = zscale(zsub(A[0][s], A[3][s]), 0.5);
                c[2][s] = zscale(zadd(A[1][s], A[2][s]), 0.5);
                const Z d = zsub(A[1][s], A[2][s]);
                c[3][s] = zscale(Z{-d.im, d.re}, 0.5);
            }
#pragma unroll
            for (int e = 0; e < 4; ++e) st<R, V>(o + e * n, g, c[e]);
        } else if (kind == PB_JONES_KRON) {   // out[2i+j, 2k+l] = a[i, k] * b[j, l] (polarization.py:375-376)
            cplx<R>* o = reinterpret_cast<cplx<R>*>(out);
            Z B[4][V];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const Px<R, V> t = ld<R, V>(b + e * n, g);
#pragma unroll
                for (int s = 0; s < V; ++s) B[e][s] = t.v[s];
            }
#pragma unroll
            for (int row = 0; row < 4; ++row)
#pragma unroll
                for (int col = 0; col < 4; ++col) {
                    Z v[V];
#pragma unroll
                    for (int s = 0; s < V; ++s)
                        v[s] = zmul(A[(row >> 1) * 2 + (col >> 1)][s], B[(row & 1) * 2 + (col & 1)][s]);
                    st<R, V>(o + (row * 4 + col) * n, g, v);
                }
        } else {                               // Mueller: real(U kron(conj J, J) U^-1) (polarization.py:395-407)
            R* o = reinterpret_cast<R*>(out);
            Z T[4][4][V];                       // T[r][m] = (U K)[r, m]
#pragma unroll
            for (int s = 0; s < V; ++s)
#pragma unroll
                for (int col = 0; col < 4; ++col) {
                    Z kc[4];                    // column col of K: K[2i+j, 2k+l] = conj(J[i, k]) J[j, l]
#pragma unroll
                    for (int row = 0; row < 4; ++row)
                        kc[row] = zmul(zconj(A[(row >> 1) * 2 + (col >> 1)][s]), A[(row & 1) * 2 + (col & 1)][s]);
#pragma unroll
                    for (int r = 0; r < 4; ++r) T[r][col][s] = u_row(r, kc);
                }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    double v[V];
#pragma unroll
                    for (int s = 0; s < V; ++s) {
                        const Z row[4] = {T[r][0][s], T[r][1][s], T[r][2][s], T[r][3][s]};
                        v[s] = 0.5 * uh_col(c, row).re;
                    }
                    st_real<R, V>(o + (r * 4 + c) * n, g, v);
                }
        }
    }
}

// complex64 planes move two pixels per 16-byte access when every plane base is 16-byte aligned and n is even
inline bool pairs_ok(long long n, std::initializer_list<const void*> ptrs) {
    if (n % 2) return false;
    for (const void* p : ptrs)
        if (p && (reinterpret_cast<uintptr_t>(p) & 15)) return false;
    return true;
}

}  // namespace

}  // namespace pb

using namespace pb;


// launch f(R, V, groups) for n pixels: V = 2 at complex64 when the planes allow it, else 1
template <typename F>
static int jones_launch(Handle* h, int dtype, bool pairs, long long n, F&& f) {
    if (dtype == PB_C64 && pairs) f(float(), std::integral_constant<int, 2>(), n / 2);
    else with_real(dtype, [&](auto r) { f(r, std::integral_constant<int, 1>(), n); });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_jones_planar(pb_handle_t hh, int dtype, const void* src, int src_type, long long rows, long long cols,
                               long long s_row, long long s_col, long long s_i, long long s_j, void* out, void* stream) {
    const long long n = rows < 0 || cols < 0 ? -1 : rows * cols;
    PB_ENTER_REAL(hh);
    if (n < 0) return fail(h, PB_ERR_INVALID, "negative pixel count");
    if (src_type < PB_ELEM_F32 || src_type > PB_ELEM_C128) return fail(h, PB_ERR_INVALID, "bad Jones source type");
    if (n == 0) return PB_OK;
    if (!src || !out) return fail(h, PB_ERR_INVALID, "null pointer");
    return jones_launch(h, dtype, pairs_ok(n, {out}), n, [&](auto r, auto v, long long groups) {
        using R = decltype(r);
        constexpr int V = decltype(v)::value;
        const int g = grid_for(groups, kThreads, h->sm_count);
        with_elem(src_type, [&](auto t) {
            using T = decltype(t);
            if constexpr (is_one_of<T, float, double, float2, double2>) {
                // a complex source is read as interleaved scalars
                using S = std::conditional_t<is_one_of<T, float, float2>, float, double>;
                jones_planar_kernel<S, is_one_of<T, float2, double2>, R, V><<<g, kThreads, 0, st>>>(
                    (const S*)src, cols, s_row, s_col, s_i, s_j, groups, n, reinterpret_cast<cplx<R>*>(out));
            }
        });
    });
}

extern "C" int pb_jones_product(pb_handle_t hh, int dtype, int mode, long long n, int a_kind, const void* a, int a_op,
                                int b_kind, const void* b, int b_op, const double* consts_host, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0) return fail(h, PB_ERR_INVALID, "negative pixel count");
    auto kind_ok = [](int k) { return k >= PB_JONES_CONST && k <= PB_JONES_SCALAR_REAL; };
    auto op_ok = [](int o) { return o == PB_JONES_OP_N || o == PB_JONES_OP_H; };
    if ((mode != PB_JONES_MATMUL && mode != PB_JONES_HADAMARD) || !kind_ok(a_kind) || !kind_ok(b_kind) || !op_ok(a_op) ||
        !op_ok(b_op))
        return fail(h, PB_ERR_INVALID, "bad Jones product arguments");
    if (n == 0) return PB_OK;
    const bool konst = a_kind == PB_JONES_CONST || b_kind == PB_JONES_CONST;
    if (!out || (a_kind != PB_JONES_CONST && !a) || (b_kind != PB_JONES_CONST && !b) || (konst && !consts_host))
        return fail(h, PB_ERR_INVALID, "null pointer");
    JonesConsts k{};
    if (konst) std::copy(consts_host, consts_host + 16, k.v);
    // a real scalar plane is read one sample at a time: only the complex operands decide the pairing
    const bool pairs = pairs_ok(n, {out, a_kind == PB_JONES_SCALAR_REAL ? nullptr : a,
                                    b_kind == PB_JONES_SCALAR_REAL ? nullptr : b});
    return jones_launch(h, dtype, pairs, n, [&](auto r, auto v, long long groups) {
        using R = decltype(r);
        const int g = grid_for(groups, kThreads, h->sm_count);
        jones_product_kernel<R, decltype(v)::value><<<g, kThreads, 0, st>>>(mode, groups, n, a_kind, a, a_op, b_kind, b, b_op, k,
                                                                           reinterpret_cast<cplx<R>*>(out));
    });
}

extern "C" int pb_jones_elements(pb_handle_t hh, int dtype, int kind, long long n, const void* plane, int plane_type,
                                 const double* params_host, int nparams, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0) return fail(h, PB_ERR_INVALID, "negative pixel count");
    static const int need[] = {8, 2, 2, 2, 3};
    if (kind < PB_JONES_FILL || kind > PB_JONES_VVR || nparams < need[kind] || nparams > 8 ||
        (plane && plane_type != PB_ELEM_F32 && plane_type != PB_ELEM_F64) || (kind == PB_JONES_FILL && plane))
        return fail(h, PB_ERR_INVALID, "bad Jones element arguments");
    if (n == 0) return PB_OK;
    if (!out || !params_host || (kind == PB_JONES_VVR && !plane)) return fail(h, PB_ERR_INVALID, "null pointer");
    JonesParams p{};
    std::copy(params_host, params_host + nparams, p.v);
    return jones_launch(h, dtype, pairs_ok(n, {out}), n, [&](auto r, auto v, long long groups) {
        using R = decltype(r);
        const int g = grid_for(groups, kThreads, h->sm_count);
        jones_elements_kernel<R, decltype(v)::value><<<g, kThreads, 0, st>>>(kind, groups, n, plane, plane_type, p,
                                                                            reinterpret_cast<cplx<R>*>(out));
    });
}

extern "C" int pb_jones_reduce(pb_handle_t hh, int dtype, int kind, long long n, const void* a, const void* b, void* out,
                               void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 0) return fail(h, PB_ERR_INVALID, "negative pixel count");
    if (kind < PB_JONES_MUELLER || kind > PB_JONES_PAULI) return fail(h, PB_ERR_INVALID, "bad Jones reduction");
    if (n == 0) return PB_OK;
    if (!a || !out || (kind == PB_JONES_KRON && !b)) return fail(h, PB_ERR_INVALID, "null pointer");
    // the Mueller planes are real: two float32 pixels are 8 bytes, so their base needs only 8-byte alignment
    const bool pairs = pairs_ok(n, {a, kind == PB_JONES_KRON ? b : nullptr, kind == PB_JONES_MUELLER ? nullptr : out}) &&
                       (reinterpret_cast<uintptr_t>(out) & 7) == 0;
    return jones_launch(h, dtype, pairs, n, [&](auto r, auto v, long long groups) {
        using R = decltype(r);
        const int g = grid_for(groups, kThreads, h->sm_count);
        jones_reduce_kernel<R, decltype(v)::value><<<g, kThreads, 0, st>>>(
            kind, groups, n, reinterpret_cast<const cplx<R>*>(a), reinterpret_cast<const cplx<R>*>(b), out);
    });
}
