// The one-variable orthogonal families on the device (prysm/polynomials/{jacobi,cheby,legendre,hermite,laguerre,
// dickson}.py), the Jacobi Clenshaw and radial sums, and the two-variable XY-monomial and Chebyshev tensor sums
// (xy.py, cheby.py).
//
// Every 1-D family is one three-term recurrence P_k = (A_k x + B_k) P_{k-1} - C_k P_{k-2} with two seeds, so one
// kernel serves them all (pb_jacobi_seq included).  The plan, in kernel-parameter space, holds the per-order
// (A, B, C) in fp64, the family's seed kind (the Jacobi form of P_1 or a plain a x + b, so that Chebyshev-1's
// P_1 = x keeps every bit of x near 0), and per order the range of output planes that take it, each with a scale
// and a track (value or derivative).  Each thread runs the recurrence once in fp64 registers, carrying dP/dx when
// a plane asks for it, and rounds each output once to the storage dtype.  Derivatives the reference forms by
// shifting the order (Jacobi, Hermite, Laguerre) are value planes of the shifted recurrence with a per-plane scale.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace pb {

#define PB_POLY_PLANES 1024        // output planes per 1-D call
#define PB_XY_PLANES 1024          // output planes per XY-monomial call
#define PB_TSUM_COEFS 1024         // (max m + 1) (max n + 1) of a tensor-product sum

enum { SEED_JACOBI = 0, SEED_LINEAR = 1 };

struct P1Step { double A, B, C, wv, wd; short e0, e1, pad0, pad1; };
struct P1Plan {
    int seed, nmax;
    double p0, s1a, s1b, dp1;      // P_0; P_1 = s1a + s1b (x - 1)/2 (SEED_JACOBI) or s1a x + s1b; dP_1/dx
    P1Step s[PB_POLY_NMAX + 1];    // order k: (A, B, C) of the step that makes P_k (k >= 2), sum weights, planes [e0, e1)
    int ent[PB_POLY_PLANES];       // plane << 1 | (1: the derivative track)
    double scale[PB_POLY_PLANES];
};
static_assert(sizeof(P1Plan) <= 32764, "the 1-D plan must fit the kernel parameter space");

// MODE 0: planes of P_n(a) or dP_n/dx (out0, (planes, n));  MODE 1: the radial sum z = sum w P(u), u = 2 (a^2 + b^2) / R^2
// - 1, into out0, and with DER dz/dx, dz/dy into out1, out2 (jacobi_radial_sum(_der_xy))
template <typename R, int MODE, bool DER>
__global__ void poly1d_kernel(const R* __restrict__ a, const R* __restrict__ b, long long n, const __grid_constant__ P1Plan pl,
                              double rsq, double inv_rsq, R* __restrict__ out0, R* __restrict__ out1, R* __restrict__ out2) {
    PB_GRID_STRIDE(i, n) {
        double xv, xa = 0.0, yb = 0.0;
        if (MODE == 0) xv = a[i];
        else {
            xa = a[i]; yb = b[i];
            const double q = xa * xa + yb * yb;
            xv = DER ? 2.0 * q * inv_rsq - 1.0 : 2.0 * q / rsq - 1.0;      // as jacobi.py:382 and :401 write it
        }
        double Pm2 = pl.p0, Pm1 = pl.seed == SEED_JACOBI ? pl.s1a + pl.s1b * ((xv - 1.0) / 2.0) : pl.s1a * xv + pl.s1b;
        double dPm2 = 0.0, dPm1 = pl.dp1;
        double z = 0.0, dz = 0.0;
        for (int k = 0; k <= pl.nmax; ++k) {
            const P1Step& st = pl.s[k];
            double P, dP = 0.0;
            if (k == 0) P = Pm2;
            else if (k == 1) { P = Pm1; dP = dPm1; }
            else {
                const double lin = st.A * xv + st.B;
                P = lin * Pm1 - st.C * Pm2;
                if (DER) { dP = st.A * Pm1 + lin * dPm1 - st.C * dPm2; dPm2 = dPm1; dPm1 = dP; }
                Pm2 = Pm1; Pm1 = P;
            }
            if (MODE == 0) {
                for (int e = st.e0; e < st.e1; ++e) {
                    const int code = pl.ent[e];
                    out0[(long long)(code >> 1) * n + i] = (R)(pl.scale[e] * ((code & 1) ? dP : P));
                }
            } else {
                z += st.wv * P;
                if (DER) dz += st.wd * dP;
            }
        }
        if (MODE == 1) {
            out0[i] = (R)z;
            if (DER) {
                out1[i] = (R)(dz * (4.0 * xa * inv_rsq));
                out2[i] = (R)(dz * (4.0 * yb * inv_rsq));
            }
        }
    }
}

// Clenshaw's backward recurrence for sum_n s_n P_n^(alpha,beta)(x) and its first j derivatives (prysm/polynomials/
// _clenshaw.py), per sample in registers: n descends in the outer loop, the derivative order jj in the inner one.
// alpha_jj[n] = (jj ? jj A_n alpha_{jj-1}[n+1] : s_n) + (A_n x + B_n) alpha_jj[n+1] - C_{n+1} alpha_jj[n+2], and 0 for
// n > M - jj.  table: every plane (jj, n) of out (j+1, N, count);  otherwise alpha_0[0] alone into out (count).
struct ClenPlan {
    int N, M, j, table;
    double s[PB_POLY_NMAX + 1], A[PB_POLY_NMAX + 1], B[PB_POLY_NMAX + 1];
    double C1[PB_POLY_NMAX + 1];   // C1[n] = C_{n+1}
};
static_assert(sizeof(ClenPlan) <= 32764, "the Clenshaw plan must fit the kernel parameter space");

template <typename R>
__global__ void clenshaw_kernel(const R* __restrict__ x, long long n, const __grid_constant__ ClenPlan pl, R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const double xv = x[i];
        double a1[PB_CLENSHAW_JMAX + 1], a2[PB_CLENSHAW_JMAX + 1];
#pragma unroll
        for (int jj = 0; jj <= PB_CLENSHAW_JMAX; ++jj) { a1[jj] = 0.0; a2[jj] = 0.0; }
        for (int k = pl.N - 1; k >= 0; --k) {
            const double lin = pl.A[k] * xv + pl.B[k];
#pragma unroll
            for (int jj = PB_CLENSHAW_JMAX; jj >= 0; --jj) {
                if (jj > pl.j) continue;
                double v = 0.0;
                if (k <= pl.M - jj) {
                    const double head = jj == 0 ? pl.s[k] : (jj * pl.A[k]) * a1[jj > 0 ? jj - 1 : 0];
                    v = head + lin * a1[jj] - pl.C1[k] * a2[jj];
                }
                a2[jj] = a1[jj]; a1[jj] = v;
                if (pl.table) out[((long long)jj * pl.N + k) * n + i] = (R)v;
                else if (jj == 0 && k == 0) out[i] = (R)v;
            }
        }
    }
}

// XY monomials x^m y^n and their d/dx, d/dy, d^2/dxdy as the reference forms them (xy.py:194-215): the powers by
// cumulative products, a derivative as k * z^(k-1), the plane as the product of the x and y terms.  sep: the grid is
// separable, x indexed by column (i % nx) and y by row (i / nx); otherwise x and y are elementwise.
struct XYPlan {
    int sep, nplanes;
    long long nx;
    short m[PB_XY_PLANES], nn[PB_XY_PLANES];
    unsigned char kind[PB_XY_PLANES];          // bit 0: d/dx, bit 1: d/dy
};
static_assert(sizeof(XYPlan) <= 32764, "the XY plan must fit the kernel parameter space");

__device__ inline double mono_term(double z, int k, bool der) {
    if (der) {
        if (k == 0) return 0.0;
        if (k == 1) return 1.0;
        double c = z;
        for (int q = 2; q < k; ++q) c *= z;
        return (double)k * c;
    }
    if (k == 0) return 1.0;
    double c = z;
    for (int q = 1; q < k; ++q) c *= z;
    return c;
}

template <typename R>
__global__ void xy_kernel(const R* __restrict__ x, const R* __restrict__ y, long long n, const __grid_constant__ XYPlan pl,
                          R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const long long iy = pl.sep ? i / pl.nx : i, ix = pl.sep ? i - iy * pl.nx : i;
        const double xv = x[ix], yv = y[iy];
        for (int p = 0; p < pl.nplanes; ++p) {
            const int kd = pl.kind[p];
            out[(long long)p * n + i] = (R)(mono_term(xv, pl.m[p], kd & 1) * mono_term(yv, pl.nn[p], kd & 2));
        }
    }
}

// Tensor-product sums z = sum c[q][p] P_p(x) P_q(y), P the monomials (BASIS 0) or Chebyshev-1 (BASIS 1), with DER
// dz/dx / sx and dz/dy / sy, in one pass: per row q the y term and its derivative by recurrence, per column p the x
// term and its derivative by the differentiated recurrence.  The dense (maxn + 1) x (maxm + 1) coefficients are in
// parameter space.
struct TSumPlan {
    int basis, maxm, maxn, sep;
    long long nx;
    double sx, sy;
    double c[PB_TSUM_COEFS];
};
static_assert(sizeof(TSumPlan) <= 32764, "the tensor-sum plan must fit the kernel parameter space");

template <typename R, bool DER>
__global__ void tsum_kernel(const R* __restrict__ x, const R* __restrict__ y, long long n, const __grid_constant__ TSumPlan pl,
                            R* __restrict__ z, R* __restrict__ dzdx, R* __restrict__ dzdy) {
    PB_GRID_STRIDE(i, n) {
        const long long iy = pl.sep ? i / pl.nx : i, ix = pl.sep ? i - iy * pl.nx : i;
        const double xv = x[ix], yv = y[iy];
        const double ca = pl.basis ? 2.0 : 1.0, cc = pl.basis ? 1.0 : 0.0;       // P_k = ca z P_{k-1} - cc P_{k-2}
        double zs = 0.0, zx = 0.0, zy = 0.0;
        double Q = 1.0, Qm = 0.0, dQ = 0.0, dQm = 0.0;
        for (int q = 0, row = 0; q <= pl.maxn; ++q, row += pl.maxm + 1) {
            if (q == 1) { Qm = Q; Q = yv; dQm = dQ; dQ = 1.0; }
            else if (q >= 2) {
                const double Qn = ca * yv * Q - cc * Qm, dQn = ca * Q + ca * yv * dQ - cc * dQm;
                Qm = Q; Q = Qn; dQm = dQ; dQ = dQn;
            }
            double P = 1.0, Pm = 0.0, dP = 0.0, dPm = 0.0, rv = 0.0, rd = 0.0;
            for (int p = 0; p <= pl.maxm; ++p) {
                if (p == 1) { Pm = P; P = xv; dPm = dP; dP = 1.0; }
                else if (p >= 2) {
                    const double Pn = ca * xv * P - cc * Pm, dPn = ca * P + ca * xv * dP - cc * dPm;
                    Pm = P; P = Pn; dPm = dP; dP = dPn;
                }
                rv += pl.c[row + p] * P;
                if (DER) rd += pl.c[row + p] * dP;
            }
            zs += Q * rv;
            if (DER) { zx += Q * rd; zy += dQ * rv; }
        }
        z[i] = (R)zs;
        if (DER) { dzdx[i] = (R)(zx / pl.sx); dzdy[i] = (R)(zy / pl.sy); }
    }
}

// ---- plans, on the host in fp64 ------------------------------------------------------------------------------------
struct Family { int seed; double p0, s1a, s1b, dp1; };

static Family family_seeds(int fam, double alpha, double beta) {
    switch (fam) {
        case PB_POLY_JACOBI: return {SEED_JACOBI, 1.0, alpha + 1, alpha + beta + 2, 0.5 * (alpha + beta + 2)};
        case PB_POLY_CHEBY1: return {SEED_LINEAR, 1.0, 1.0, 0.0, 1.0};
        case PB_POLY_CHEBY2: return {SEED_LINEAR, 1.0, 2.0, 0.0, 2.0};
        case PB_POLY_CHEBY3: return {SEED_LINEAR, 1.0, 2.0, -1.0, 2.0};
        case PB_POLY_CHEBY4: return {SEED_LINEAR, 1.0, 2.0, 1.0, 2.0};
        case PB_POLY_LEGENDRE: return {SEED_LINEAR, 1.0, 1.0, 0.0, 1.0};
        case PB_POLY_HERMITE_HE: return {SEED_LINEAR, 1.0, 1.0, 0.0, 1.0};
        case PB_POLY_HERMITE_H: return {SEED_LINEAR, 1.0, 2.0, 0.0, 2.0};
        case PB_POLY_LAGUERRE: return {SEED_LINEAR, 1.0, -1.0, alpha + 1, -1.0};
        case PB_POLY_DICKSON1: return {SEED_LINEAR, 2.0, 1.0, 0.0, 1.0};
        default: return {SEED_LINEAR, 1.0, 1.0, 0.0, 1.0};          // PB_POLY_DICKSON2
    }
}

// (A, B, C) of the step that makes P_k, k >= 2
static void family_abc(int fam, int k, double alpha, double beta, double* abc) {
    const double kk = k;
    switch (fam) {
        case PB_POLY_JACOBI: jacobi_abc(k - 1, alpha, beta, abc); return;
        case PB_POLY_CHEBY1: case PB_POLY_CHEBY2: case PB_POLY_CHEBY3: case PB_POLY_CHEBY4:
            abc[0] = 2.0; abc[1] = 0.0; abc[2] = 1.0; return;
        case PB_POLY_LEGENDRE: abc[0] = (2 * kk - 1) / kk; abc[1] = 0.0; abc[2] = (kk - 1) / kk; return;
        case PB_POLY_HERMITE_HE: abc[0] = 1.0; abc[1] = 0.0; abc[2] = kk - 1; return;
        case PB_POLY_HERMITE_H: abc[0] = 2.0; abc[1] = 0.0; abc[2] = 2 * (kk - 1); return;
        case PB_POLY_LAGUERRE: abc[0] = -1.0 / kk; abc[1] = (alpha + 2 * kk - 1) / kk; abc[2] = (alpha + kk - 1) / kk; return;
        default: abc[0] = 1.0; abc[1] = 0.0; abc[2] = alpha; return;                              // Dickson
    }
}

struct P1Term { int order, plane, der; double scale, wv, wd; };

static void build_p1plan(int fam, double alpha, double beta, std::vector<P1Term>& terms, P1Plan& pl) {
    std::stable_sort(terms.begin(), terms.end(), [](const P1Term& a, const P1Term& b) { return a.order < b.order; });
    const Family f = family_seeds(fam, alpha, beta);
    pl.seed = f.seed; pl.p0 = f.p0; pl.s1a = f.s1a; pl.s1b = f.s1b; pl.dp1 = f.dp1;
    pl.nmax = 0;
    for (const P1Term& t : terms) pl.nmax = std::max(pl.nmax, t.order);
    size_t q = 0;
    int nent = 0;
    for (int k = 0; k <= pl.nmax; ++k) {
        P1Step& st = pl.s[k];
        double abc[3] = {0.0, 0.0, 0.0};
        if (k >= 2) family_abc(fam, k, alpha, beta, abc);
        st.A = abc[0]; st.B = abc[1]; st.C = abc[2]; st.wv = 0.0; st.wd = 0.0;
        st.e0 = st.e1 = (short)nent; st.pad0 = st.pad1 = 0;
        for (; q < terms.size() && terms[q].order == k; ++q) {
            const P1Term& t = terms[q];
            st.wv += t.wv; st.wd += t.wd;
            if (t.plane >= 0) {
                pl.ent[nent] = t.plane << 1 | t.der;
                pl.scale[nent] = t.scale;
                st.e1 = (short)++nent;
            }
        }
    }
}

template <int MODE, bool DER>
static void launch_p1(int dtype, int g, cudaStream_t st, const void* a, const void* b, long long count, const P1Plan& pl,
                      double rsq, double inv_rsq, void* o0, void* o1, void* o2) {
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        poly1d_kernel<R, MODE, DER><<<g, 256, 0, st>>>((const R*)a, (const R*)b, count, pl, rsq, inv_rsq, (R*)o0, (R*)o1,
                                                       (R*)o2);
    });
}

static int run_p1_seq(Handle* h, int dtype, int fam, double alpha, double beta, const void* x, long long count,
                      std::vector<P1Term>& terms, bool der, void* out, cudaStream_t st) {
    P1Plan pl;
    build_p1plan(fam, alpha, beta, terms, pl);
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    if (der) launch_p1<0, true>(dtype, g, st, x, nullptr, count, pl, 1.0, 1.0, out, nullptr, nullptr);
    else launch_p1<0, false>(dtype, g, st, x, nullptr, count, pl, 1.0, 1.0, out, nullptr, nullptr);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_jacobi_seq(pb_handle_t hh, int dtype, const void* x, long long count, int nmax, double alpha, double beta,
                             const int* slots_host, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !out || !slots_host || nmax < 0) return fail(h, PB_ERR_INVALID, "bad jacobi arguments");
    if (nmax > PB_POLY_NMAX) return fail(h, PB_ERR_UNSUPPORTED, "jacobi order above 120");
    if (count <= 0) return PB_OK;
    std::vector<P1Term> terms;
    for (int j = 0; j <= nmax; ++j)
        if (slots_host[j] >= 0) terms.push_back({j, slots_host[j], 0, 1.0, 0.0, 0.0});
    if (terms.size() > PB_POLY_PLANES) return fail(h, PB_ERR_UNSUPPORTED, "more than 1024 jacobi planes");
    terms.push_back({nmax, -1, 0, 0.0, 0.0, 0.0});           // the recurrence runs to nmax as it always has
    return run_p1_seq(h, dtype, PB_POLY_JACOBI, alpha, beta, x, count, terms, false, out, st);
}

extern "C" int pb_poly_seq(pb_handle_t hh, int dtype, int family, int kind, double alpha, double beta, const void* x,
                           long long count, int k, const int* n_host, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (family < PB_POLY_JACOBI || family > PB_POLY_DICKSON2 || kind < PB_POLY_VALUE || kind > PB_POLY_VALUE_DER)
        return fail(h, PB_ERR_INVALID, "poly: bad family or kind");
    if (!x || !out || k < 1 || !n_host) return fail(h, PB_ERR_INVALID, "bad poly arguments");
    if ((long long)k * (kind == PB_POLY_VALUE_DER ? 2 : 1) > PB_POLY_PLANES) return fail(h, PB_ERR_UNSUPPORTED, "poly: more than 1024 planes");
    for (int q = 0; q < k; ++q) {
        if (n_host[q] < 0) return fail(h, PB_ERR_INVALID, "poly: order n must be >= 0");
        if (n_host[q] > PB_POLY_NMAX) return fail(h, PB_ERR_UNSUPPORTED, "poly: order above 120");
    }
    // the derivative by order shift, as the reference forms it: Jacobi 0.5 (n + a + b + 1) P_{n-1}^(a+1, b+1),
    // Hermite kind n P_{n-1}, Laguerre -L_{n-1}^(a+1); an order-0 plane is 0 P_0
    const bool shifted = kind == PB_POLY_DER && (family == PB_POLY_JACOBI || family == PB_POLY_HERMITE_HE ||
                                                 family == PB_POLY_HERMITE_H || family == PB_POLY_LAGUERRE);
    std::vector<P1Term> terms;
    double a = alpha, b = beta;
    if (shifted) {
        if (family == PB_POLY_JACOBI) { a = alpha + 1; b = beta + 1; }
        if (family == PB_POLY_LAGUERRE) a = alpha + 1;
        for (int q = 0; q < k; ++q) {
            const int nq = n_host[q];
            double sc;
            if (family == PB_POLY_JACOBI) sc = 0.5 * (nq + alpha + beta + 1);
            else if (family == PB_POLY_LAGUERRE) sc = -1.0;
            else sc = (family == PB_POLY_HERMITE_H ? 2.0 : 1.0) * nq;
            terms.push_back({nq > 0 ? nq - 1 : 0, q, 0, nq > 0 ? sc : 0.0, 0.0, 0.0});
        }
        return run_p1_seq(h, dtype, family, a, b, x, count, terms, false, out, st);
    }
    for (int q = 0; q < k; ++q) {
        if (kind != PB_POLY_DER) terms.push_back({n_host[q], q, 0, 1.0, 0.0, 0.0});
        if (kind != PB_POLY_VALUE) terms.push_back({n_host[q], kind == PB_POLY_DER ? q : k + q, 1, 1.0, 0.0, 0.0});
    }
    return run_p1_seq(h, dtype, family, a, b, x, count, terms, kind != PB_POLY_VALUE, out, st);
}

extern "C" int pb_jacobi_radial_sum(pb_handle_t hh, int dtype, double alpha, double beta, const void* x, const void* y,
                                    long long count, int k, const int* n_host, const double* coefs_host, double radius,
                                    void* z, void* dzdx, void* dzdy, void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !y || !z || k < 0 || (k > 0 && (!n_host || !coefs_host)) || (!dzdx != !dzdy))
        return fail(h, PB_ERR_INVALID, "bad jacobi radial sum arguments");
    std::vector<P1Term> terms;
    for (int q = 0; q < k; ++q) {
        if (n_host[q] < 0) return fail(h, PB_ERR_INVALID, "poly: order n must be >= 0");
        if (n_host[q] > PB_POLY_NMAX) return fail(h, PB_ERR_UNSUPPORTED, "poly: order above 120");
        if (coefs_host[q] == 0.0) continue;                          // jacobi.py:386 skips zero weights
        terms.push_back({n_host[q], -1, 0, 0.0, coefs_host[q], coefs_host[q]});
    }
    P1Plan pl;
    build_p1plan(PB_POLY_JACOBI, alpha, beta, terms, pl);
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    const double rsq = radius * radius, inv_rsq = 1.0 / rsq;
    if (dzdx) launch_p1<1, true>(dtype, g, st, x, y, count, pl, rsq, inv_rsq, z, dzdx, dzdy);
    else launch_p1<1, false>(dtype, g, st, x, y, count, pl, rsq, inv_rsq, z, nullptr, nullptr);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_jacobi_clenshaw(pb_handle_t hh, int dtype, double alpha, double beta, const void* x, long long count,
                                  int len, const double* s_host, int j, int table, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !out || len < 1 || !s_host || j < 0) return fail(h, PB_ERR_INVALID, "bad clenshaw arguments");
    if (j > PB_CLENSHAW_JMAX) return fail(h, PB_ERR_UNSUPPORTED, "clenshaw: derivative order above 8");
    if (len > PB_POLY_NMAX + 1) return fail(h, PB_ERR_UNSUPPORTED, "clenshaw: more than 121 coefficients");
    ClenPlan pl;
    pl.M = len - 1; pl.N = std::max(len, 2); pl.j = j; pl.table = table ? 1 : 0;
    for (int nn = 0; nn < pl.N; ++nn) {
        double abc[3], abc1[3];
        jacobi_abc(nn, alpha, beta, abc);
        jacobi_abc(nn + 1, alpha, beta, abc1);
        pl.s[nn] = nn < len ? s_host[nn] : 0.0;
        pl.A[nn] = abc[0]; pl.B[nn] = abc[1]; pl.C1[nn] = abc1[2];
    }
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        clenshaw_kernel<R><<<g, 256, 0, st>>>((const R*)x, count, pl, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_xy_seq(pb_handle_t hh, int dtype, const void* x, const void* y, long long count, long long nx,
                         int separable, int k, const int* m_host, const int* n_host, const int* kind_host, void* out,
                         void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !y || !out || k < 1 || !m_host || !n_host || !kind_host || (separable && nx < 1))
        return fail(h, PB_ERR_INVALID, "bad xy arguments");
    if (k > PB_XY_PLANES) return fail(h, PB_ERR_UNSUPPORTED, "xy: more than 1024 planes");
    XYPlan pl;
    pl.sep = separable ? 1 : 0; pl.nplanes = k; pl.nx = separable ? nx : 1;
    for (int q = 0; q < k; ++q) {
        if (m_host[q] < 0 || n_host[q] < 0 || kind_host[q] < 0 || kind_host[q] > 3) return fail(h, PB_ERR_INVALID, "xy: orders must be >= 0");
        if (m_host[q] > 32767 || n_host[q] > 32767) return fail(h, PB_ERR_UNSUPPORTED, "xy: order above 32767");
        pl.m[q] = (short)m_host[q]; pl.nn[q] = (short)n_host[q]; pl.kind[q] = (unsigned char)kind_host[q];
    }
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        xy_kernel<R><<<g, 256, 0, st>>>((const R*)x, (const R*)y, count, pl, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_tensor_sum(pb_handle_t hh, int dtype, int basis, const void* x, const void* y, long long count, long long nx,
                             int separable, int k, const int* m_host, const int* n_host, const double* coefs_host,
                             double x_norm, double y_norm, void* z, void* dzdx, void* dzdy, void* stream) {
    PB_ENTER_REAL(hh);
    if (basis < PB_TSUM_MONOMIAL || basis > PB_TSUM_CHEBY1 || !x || !y || !z || k < 0 ||
        (k > 0 && (!m_host || !n_host || !coefs_host)) || (!dzdx != !dzdy) || (separable && nx < 1))
        return fail(h, PB_ERR_INVALID, "bad tensor sum arguments");
    int maxm = 0, maxn = 0;
    for (int q = 0; q < k; ++q) {
        if (m_host[q] < 0 || n_host[q] < 0) return fail(h, PB_ERR_INVALID, "tensor sum: orders must be >= 0");
        if (m_host[q] > PB_TSUM_COEFS || n_host[q] > PB_TSUM_COEFS) return fail(h, PB_ERR_UNSUPPORTED, "tensor sum: more than 1024 coefficients");
        maxm = std::max(maxm, m_host[q]); maxn = std::max(maxn, n_host[q]);
    }
    if ((long long)(maxm + 1) * (maxn + 1) > PB_TSUM_COEFS)
        return fail(h, PB_ERR_UNSUPPORTED, "tensor sum: (max m + 1)(max n + 1) above 1024");
    TSumPlan pl;
    pl.basis = basis; pl.maxm = maxm; pl.maxn = maxn; pl.sep = separable ? 1 : 0; pl.nx = separable ? nx : 1;
    pl.sx = x_norm; pl.sy = y_norm;
    std::fill(pl.c, pl.c + PB_TSUM_COEFS, 0.0);
    for (int q = 0; q < k; ++q) pl.c[n_host[q] * (maxm + 1) + m_host[q]] += coefs_host[q];
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        if (dzdx) tsum_kernel<R, true><<<g, 256, 0, st>>>((const R*)x, (const R*)y, count, pl, (R*)z, (R*)dzdx, (R*)dzdy);
        else tsum_kernel<R, false><<<g, 256, 0, st>>>((const R*)x, (const R*)y, count, pl, (R*)z, nullptr, nullptr);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
