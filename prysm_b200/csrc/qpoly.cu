// Forbes polynomials on the device: Q-bfs (slope-orthogonal asphere, oe-18-19-19700), Q-con (sag-orthogonal asphere,
// oe-18-13-13851) and the 2D-Q freeform basis (oe-20-3-2483) -- values, radial / polar / Cartesian derivatives, and
// coefficient-weighted sag and slope sums (prysm/polynomials/qpoly.py).
//
// One kernel, one thread per sample.  A plan in kernel-parameter space lists one group per recurrence (the Q-bfs or
// Q-con recurrence, or the 2D-Q recurrence of one |m|), and per order n of a group one step with the recurrence
// coefficients, the sum weights and the range of output planes that take this order.  Each thread runs every group's
// recurrence once in fp64 registers, carrying the value and its derivative with respect to the recurrence variable,
// and either writes the requested planes (MODE 0) or accumulates the weighted sums (MODE 1: forward recurrence with
// the weights applied as each order is made, the basis never stored).  The tables are made on the host in fp64.
#include <algorithm>
#include <cmath>
#include <limits>
#include <vector>

#include "common.cuh"

namespace pb {

#define PB_QPOLY_STEPS 256        // recurrence steps per call: the sum over groups of (highest n + 1)
#define PB_QPOLY_ENTRIES 1024     // output planes per basis call

enum { QG_BFS = 0, QG_CON = 1, QG_2D = 2 };

struct QGroup { short kind, am, nmax, first; };
// j >= 2 (and the 2D-Q seeds): P_j = (c0 + c1 v) P_{j-1} - C P_{j-2};  Q_j = (P_j - g Q_{j-1} - h Q_{j-2}) * invf
// v is u = r^2 (Q-bfs, 2D-Q) or 2u - 1 (Q-con).  2D-Q step 0 keeps Q_0 = 1/(2 f_0) in c0.
struct QStep {
    double c0, c1, C, g, h, invf;
    double wc, ws;                // MODE 1: weight of the cosine (or m = 0) and of the sine term of this order
    short e0, e1, pad0, pad1;     // MODE 0: output entries [e0, e1) of this order
};
struct QPlan {
    int ngroups, pad;
    QGroup g[PB_QPOLY_NMAX + 1];
    QStep s[PB_QPOLY_STEPS];
    short ent[PB_QPOLY_ENTRIES];  // 2 k + (1 for a sine term): output plane k
};
static_assert(sizeof(QPlan) <= 32764, "the qpoly plan must fit the kernel parameter space");

#define PB_Q_INV_SQRT19 0.22941573387056177   // 1 / sqrt(19)

// KIND 0: values (a = r or x of Q-bfs / Q-con, b = t);  1: d/dr (and d/dt of 2D-Q);  2: d/dx, d/dy (a = x, b = y)
// MODE 0: the basis, planes of out0 (and out1);  MODE 1: z -> out0, dz/dr -> out1, dz/dt -> out2 (each optional)
template <typename R, int KIND, int MODE>
__global__ void qpoly_kernel(const R* __restrict__ a, const R* __restrict__ b, long long n, const __grid_constant__ QPlan pl,
                             R* __restrict__ out0, R* __restrict__ out1, R* __restrict__ out2) {
    constexpr bool DER = KIND != 0;
    PB_GRID_STRIDE(i, n) {
        double r = 0.0, x = 0.0, y = 0.0, u, tv = 0.0;
        if (KIND == 2) {
            x = a[i]; y = b[i];
            u = x * x + y * y;
        } else {
            r = a[i];
            u = r * r;
            if (b) tv = b[i];
        }
        double rm = 1.0, rm1 = 1.0;                          // r^am, r^(am-1)
        double hc = 1.0, hs = 0.0, hc1 = 1.0, hs1 = 0.0;     // Re/Im (x + iy)^am and ^(am-1)
        int am_now = 0;
        double z = 0.0, zr = 0.0, zt = 0.0;
        for (int gi = 0; gi < pl.ngroups; ++gi) {
            const QGroup g = pl.g[gi];
            double c = 1.0, s = 0.0;
            if (g.kind == QG_2D) {
                for (; am_now < g.am; ++am_now) {
                    if (KIND == 2) {
                        hc1 = hc; hs1 = hs;
                        const double t0 = x * hc - y * hs;
                        hs = x * hs + y * hc;
                        hc = t0;
                    } else {
                        rm1 = rm;
                        rm = rm * r;
                    }
                }
                if (KIND != 2) sincos((double)g.am * tv, &s, &c);
            }
            const double v = g.kind == QG_CON ? 2.0 * u - 1.0 : u;
            double Pm1 = 0.0, Pm2 = 0.0, Qm1 = 0.0, Qm2 = 0.0, dPm1 = 0.0, dPm2 = 0.0, dQm1 = 0.0, dQm2 = 0.0;
            double Sa = 0.0, Sb = 0.0, dSa = 0.0, dSb = 0.0;
            for (int j = 0; j <= g.nmax; ++j) {
                const QStep& st = pl.s[g.first + j];
                double P, Q, dP = 0.0, dQ = 0.0;
                if (j == 0) {
                    P = g.kind == QG_BFS ? 2.0 : (g.kind == QG_CON ? 1.0 : 0.5);
                    Q = g.kind == QG_2D ? st.c0 : 1.0;
                } else if (j == 1 && g.kind == QG_BFS) {
                    P = 6.0 - 8.0 * u;
                    Q = PB_Q_INV_SQRT19 * (13.0 - 16.0 * u);
                    if (DER) { dP = -8.0; dQ = -16.0 * PB_Q_INV_SQRT19; }
                } else if (j == 1 && g.kind == QG_CON) {
                    P = st.c1 * v + st.c0;
                    Q = P;
                    if (DER) { dP = st.c1; dQ = dP; }
                } else {
                    if (j == 1) {                                 // 2D-Q seed P_1
                        if (g.am == 1) { P = 1.0 - u / 2.0; dP = -0.5; }
                        else { P = ((double)g.am - 0.5) + (1.0 - (double)g.am) * u; dP = 1.0 - (double)g.am; }
                    } else if (g.kind == QG_2D && g.am == 1 && j == 2) {
                        P = (3.0 - u * (12.0 - 8.0 * u)) / 6.0;
                        dP = (-12.0 + 16.0 * u) / 6.0;
                    } else if (g.kind == QG_2D && g.am == 1 && j == 3) {
                        P = (5.0 - u * (60.0 - u * (120.0 - 64.0 * u))) / 10.0;
                        dP = (-60.0 + u * (240.0 - 192.0 * u)) / 10.0;
                    } else {
                        const double lin = g.kind == QG_CON ? st.c1 * v + st.c0 : st.c0 + st.c1 * v;
                        P = lin * Pm1 - st.C * Pm2;
                        if (DER) dP = st.c1 * Pm1 + lin * dPm1 - st.C * dPm2;
                    }
                    Q = (P - st.g * Qm1 - st.h * Qm2) * st.invf;
                    if (DER) dQ = (dP - st.g * dQm1 - st.h * dQm2) * st.invf;
                }
                Pm2 = Pm1; Pm1 = P; Qm2 = Qm1; Qm1 = Q;
                if (DER) { dPm2 = dPm1; dPm1 = dP; dQm2 = dQm1; dQm1 = dQ; }
                if (MODE == 1) {
                    Sa += st.wc * Q; Sb += st.ws * Q;
                    if (DER) { dSa += st.wc * dQ; dSb += st.ws * dQ; }
                }
                for (int e = MODE == 0 ? st.e0 : 0; e < (MODE == 0 ? st.e1 : 0); ++e) {
                    const int code = pl.ent[e];
                    const long long o = (long long)(code >> 1) * n + i;
                    const bool sine = code & 1;
                    double v0, v1 = 0.0;
                    if (g.kind == QG_BFS) {
                        const double env = u * (1.0 - u);
                        if (KIND == 0) v0 = Q * env;
                        else if (KIND == 1) v0 = (2.0 * r - 4.0 * r * u) * Q + env * (2.0 * r) * dQ;
                        else {
                            const double common = (1.0 - 2.0 * u) * Q + env * dQ;
                            v0 = 2.0 * x * common; v1 = 2.0 * y * common;
                        }
                    } else if (g.kind == QG_CON) {
                        const double r3 = r * r * r;
                        v0 = KIND == 0 ? P * (u * u) : 4.0 * r3 * P + 4.0 * (r3 * r * r) * dP;
                    } else {
                        const double am = g.am;
                        if (KIND == 0) v0 = Q * ((sine ? s : c) * rm);
                        else if (KIND == 1) {
                            v0 = (sine ? s : c) * (am * rm1 * Q + 2.0 * rm * r * dQ);
                            v1 = (sine ? am * c : -am * s) * (rm * Q);
                        } else {
                            const double H = sine ? hs : hc;
                            const double dHdx = am * (sine ? hs1 : hc1), dHdy = sine ? am * hc1 : -am * hs1;
                            v0 = 2.0 * x * dQ * H + Q * dHdx;
                            v1 = 2.0 * y * dQ * H + Q * dHdy;
                        }
                    }
                    out0[o] = (R)v0;
                    if (KIND != 0 && out1) out1[o] = (R)v1;
                }
            }
            if (MODE == 1) {
                if (g.kind == QG_BFS) {
                    const double env = u * (1.0 - u);
                    z += env * Sa;
                    if (DER) zr += (2.0 * r - 4.0 * r * u) * Sa + env * (2.0 * r) * dSa;
                } else if (g.kind == QG_CON) {
                    const double r3 = r * r * r;
                    z += (u * u) * Sa;
                    if (DER) zr += 4.0 * r3 * Sa + 4.0 * (r3 * r * r) * dSa;
                } else {
                    const double am = g.am;
                    z += rm * (c * Sa + s * Sb);
                    if (DER) {
                        zr += rm1 * (c * (2.0 * u * dSa + am * Sa) + s * (2.0 * u * dSb + am * Sb));
                        zt += am * rm * (c * Sb - s * Sa);
                    }
                }
            }
        }
        if (MODE == 1) {
            if (out0) out0[i] = (R)z;
            if (DER && out1) out1[i] = (R)zr;
            if (DER && out2) out2[i] = (R)zt;
        }
    }
}

// ---- the tables, in fp64 on the host -------------------------------------------------------------------------------
// Q-bfs (oe-18-19-19700 A.14-A.16): f(0) = 2, f(1) = sqrt(19)/2, g(0) = -1/2,
//   h(k) = -(k+2)(k+1) / (2 f(k)),  g(k) = -(1 + g(k-1) h(k-1)) / f(k),  f(k) = sqrt(k(k+1) + 3 - g(k-1)^2 - h(k-2)^2)
static void qbfs_tables(int nmax, std::vector<double>& f, std::vector<double>& g, std::vector<double>& h) {
    f.assign(nmax + 1, 0.0); g.assign(nmax + 1, 0.0); h.assign(nmax + 1, 0.0);
    for (int k = 0; k <= nmax; ++k) {
        if (k == 0) f[k] = 2.0;
        else if (k == 1) f[k] = std::sqrt(19.0) / 2.0;
        else f[k] = std::sqrt((double)(k * (k + 1) + 3) - g[k - 1] * g[k - 1] - h[k - 2] * h[k - 2]);
        h[k] = -(double)(k + 2) * (double)(k + 1) / (2.0 * f[k]);
        g[k] = k == 0 ? -0.5 : -(1.0 + g[k - 1] * h[k - 1]) / f[k];
    }
}

// Jacobi (alpha = 0, beta = 4) recurrence of Q-con: P_{k+1} = (A x + B) P_k - C P_{k-1}
static void qcon_abc(int k, double* abc) {
    const double n = k;
    abc[0] = (2 * n + 5) * (n + 3) / ((n + 1) * (n + 5));
    abc[1] = -4 * (2 * n + 5) / ((n + 1) * (n + 5) * (n + 2));
    abc[2] = n * (n + 4) * (n + 3) / ((n + 1) * (n + 5) * (n + 2));
}

static double nan_or(double num, double den) {
    return den == 0.0 ? std::numeric_limits<double>::quiet_NaN() : num / den;
}

// 2D-Q (oe-20-3-2483 A.3): P_n = (A + B u) P_{n-1} - C P_{n-2} with A, B, C of (n - 1, m); NaN where D = 0
static void q2d_abc(int ni, int m, double* abc) {
    const double n = ni, mm = m;
    const double D = (4 * n * n - 1) * (mm + n - 2) * (mm + 2 * n - 3);
    abc[0] = nan_or((2 * n - 1) * (mm + 2 * n - 2) * (4 * n * (mm + n - 2) + (mm - 3) * (2 * mm - 1)), D);
    abc[1] = nan_or(-2 * (2 * n - 1) * (mm + 2 * n - 3) * (mm + 2 * n - 2) * (mm + 2 * n - 1), D);
    abc[2] = nan_or(n * (2 * n - 3) * (mm + 2 * n - 1) * (2 * mm + 2 * n - 3), D);
}

// gamma(n, m) of prysm.mathops (oe-20-3-2483 A.15 and A.13), m >= 2, n >= 1
static double q2d_gamma(int n, int m) {
    double v = 3.0 / 8.0;                                   // gamma(1, 2)
    for (int mm = 3; mm <= m; ++mm) v *= (2.0 * (mm - 1) + 1.0) / (2.0 * (mm - 2));
    for (int k = 2; k <= n; ++k) v *= (double)k * (2.0 * m + 2.0 * (k - 1) - 1.0) / ((m + (k - 1) - 2.0) * (2.0 * (k - 1) + 1.0));
    return v;
}

// (2m - 1)!! / (2^(m+1) (m - 1)!) and m^2 (2m - 3)!! / (2^(m+1) (m - 1)!) as products of ratios
static double q2d_G0(int m) {
    double v = 0.25;                                        // m = 1: 1!! / (4 * 0!)
    for (int k = 2; k <= m; ++k) v *= (2.0 * k - 1.0) / (2.0 * (k - 1));
    return v;
}

static double q2d_F0(int m) {
    if (m == 1) return 0.25;
    double v = 1.0 / 8.0;                                   // (2m-3)!! / (2^(m+1) (m-1)!) at m = 2: 1 / 8
    for (int k = 3; k <= m; ++k) v *= (2.0 * k - 3.0) / (2.0 * (k - 1));
    return (double)m * m * v;
}

static double q2d_G(int n, int m) {
    if (n == 0) return q2d_G0(m);
    if (m == 1) {
        const double nn = n;
        return -((2 * nn * nn - 1) * (nn * nn - 1)) / (8 * (4 * nn * nn - 1)) - (n == 1 ? 1.0 / 24.0 : 0.0);
    }
    const double nn = n, mm = m;
    const double num = (2 * nn * (mm + nn - 1) - mm) * ((nn + 1) * (2 * mm + 2 * nn - 1));
    const double den = ((mm + 2 * nn - 2) * (mm + 2 * nn - 1)) * ((mm + 2 * nn) * (2 * nn + 1));
    return -num / den * q2d_gamma(n, m);
}

static double q2d_F(int n, int m) {
    if (n == 0) return q2d_F0(m);
    const double nn = n, mm = m;
    if (m == 1) return (4 * (nn - 1) * (nn - 1) * nn * nn + 1) / (8 * (2 * nn - 1) * (2 * nn - 1)) + (n == 1 ? 11.0 / 32.0 : 0.0);
    const double chi = mm + nn - 2;
    const double num = 2 * nn * chi * (3 - 5 * mm + 4 * nn * chi) + mm * mm * (3 - mm + 4 * nn * chi);
    const double den = ((mm + 2 * nn - 3) * (mm + 2 * nn - 2)) * ((mm + 2 * nn - 1) * (2 * nn - 1));
    return num / den * q2d_gamma(n, m);
}

// f(n, m) = sqrt(F(n, m) - g(n-1, m)^2), f(0, m) = sqrt(F(0, m)), g(n, m) = G(n, m) / f(n, m)
static void q2d_fg(int nmax, int m, std::vector<double>& f, std::vector<double>& g) {
    f.assign(nmax + 1, 0.0); g.assign(nmax + 1, 0.0);
    for (int k = 0; k <= nmax; ++k) {
        f[k] = k == 0 ? std::sqrt(q2d_F(0, m)) : std::sqrt(q2d_F(k, m) - g[k - 1] * g[k - 1]);
        g[k] = q2d_G(k, m) / f[k];
    }
}

struct QTerm { int kind, am, n, sine, k; double w; };

// Groups in ascending (kind, |m|) order; one step per order 0..nmax of each group.  MODE 0 terms carry their output
// plane k (entries sorted by order), MODE 1 terms their weight.
static int build_qplan(Handle* h, std::vector<QTerm>& terms, int mode, QPlan& pl) {
    std::stable_sort(terms.begin(), terms.end(), [](const QTerm& a, const QTerm& b) {
        if (a.kind != b.kind) return a.kind < b.kind;
        if (a.am != b.am) return a.am < b.am;
        return a.n < b.n;
    });
    pl.ngroups = 0; pl.pad = 0;
    int nsteps = 0, nent = 0;
    size_t pos = 0;
    while (pos < terms.size()) {
        size_t end = pos;
        int nmax = 0;
        while (end < terms.size() && terms[end].kind == terms[pos].kind && terms[end].am == terms[pos].am) {
            nmax = std::max(nmax, terms[end].n);
            ++end;
        }
        if (nsteps + nmax + 1 > PB_QPOLY_STEPS)
            return fail(h, PB_ERR_UNSUPPORTED, "qpoly: more than 256 recurrence steps (the sum over |m| of the highest n + 1)");
        const int kind = terms[pos].kind, am = terms[pos].am;
        QGroup& g = pl.g[pl.ngroups++];
        g.kind = (short)kind; g.am = (short)am; g.nmax = (short)nmax; g.first = (short)nsteps;
        std::vector<double> f, gg, hh;
        if (kind == QG_BFS) qbfs_tables(nmax, f, gg, hh);
        else if (kind == QG_2D) q2d_fg(nmax, am, f, gg);
        for (int j = 0; j <= nmax; ++j) {
            QStep& st = pl.s[nsteps + j];
            st = QStep{0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 0, 0};
            if (kind == QG_BFS) {
                st.c0 = 2.0; st.c1 = -4.0; st.C = 1.0;
                if (j >= 2) { st.g = gg[j - 1]; st.h = hh[j - 2]; st.invf = 1.0 / f[j]; }
            } else if (kind == QG_CON) {
                double abc[3];
                qcon_abc(j - 1 < 0 ? 0 : j - 1, abc);
                st.c0 = abc[1]; st.c1 = abc[0]; st.C = abc[2];   // lin = A (2u - 1) + B
            } else {
                if (j == 0) st.c0 = 1.0 / (2.0 * f[0]);
                else {
                    st.g = gg[j - 1]; st.invf = 1.0 / f[j];
                    if (j >= 2 && !(am == 1 && j <= 3)) {
                        double abc[3];
                        q2d_abc(j - 1, am, abc);
                        st.c0 = abc[0]; st.c1 = abc[1]; st.C = abc[2];
                    }
                }
            }
            st.e0 = st.e1 = (short)nent;
            for (size_t q = pos; q < end; ++q) {
                const QTerm& t = terms[q];
                if (t.n != j) continue;
                if (mode == 0) { pl.ent[nent++] = (short)(2 * t.k + t.sine); st.e1 = (short)nent; }
                else (t.sine ? st.ws : st.wc) += t.w;
            }
        }
        nsteps += nmax + 1;
        pos = end;
    }
    return PB_OK;
}

static int build_qterms(Handle* h, int family, int k, const int* n_host, const int* m_host, const double* w,
                        std::vector<QTerm>& terms) {
    terms.clear();
    for (int q = 0; q < k; ++q) {
        const int n = n_host[q], m = family == QG_2D && m_host ? m_host[q] : 0, am = m < 0 ? -m : m;
        if (n < 0) return fail(h, PB_ERR_INVALID, "qpoly: radial order n must be >= 0");
        if (n > PB_QPOLY_NMAX || am > PB_QPOLY_NMAX) return fail(h, PB_ERR_UNSUPPORTED, "qpoly: n and |m| must be <= 64");
        if (w && w[q] == 0.0) continue;                     // a zero coefficient adds nothing: trailing zeros trim
        const int kind = family == QG_2D ? (am == 0 ? QG_BFS : QG_2D) : family;
        terms.push_back({kind, am, n, m < 0 ? 1 : 0, q, w ? w[q] : 0.0});
    }
    return PB_OK;
}

template <int KIND, int MODE>
static void launch_q(int dtype, int g, cudaStream_t st, const void* a, const void* b, long long count, const QPlan& pl,
                     void* o0, void* o1, void* o2) {
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        qpoly_kernel<R, KIND, MODE><<<g, 256, 0, st>>>((const R*)a, (const R*)b, count, pl, (R*)o0, (R*)o1, (R*)o2);
    });
}

}  // namespace pb

using namespace pb;

extern "C" int pb_qpoly_seq(pb_handle_t hh, int dtype, int family, int kind, const void* a, const void* b, long long count,
                            int k, const int* n_host, const int* m_host, void* out0, void* out1, void* stream) {
    PB_ENTER_REAL(hh);
    if (family < PB_QPOLY_BFS || family > PB_QPOLY_2D || kind < PB_QPOLY_VALUE || kind > PB_QPOLY_DER_XY)
        return fail(h, PB_ERR_INVALID, "qpoly: bad family or kind");
    if (family != PB_QPOLY_2D && kind == PB_QPOLY_DER_XY) return fail(h, PB_ERR_INVALID, "qpoly: Cartesian derivatives are 2D-Q only");
    if (!a || !out0 || k < 1 || !n_host || (family == PB_QPOLY_2D && !m_host)) return fail(h, PB_ERR_INVALID, "bad qpoly arguments");
    if (family == PB_QPOLY_2D && (!b || (kind != PB_QPOLY_VALUE && !out1))) return fail(h, PB_ERR_INVALID, "bad qpoly arguments");
    if (k > PB_QPOLY_ENTRIES) return fail(h, PB_ERR_UNSUPPORTED, "qpoly: more than 1024 modes");
    std::vector<QTerm> terms;
    PB_TRY(build_qterms(h, family, k, n_host, m_host, nullptr, terms));
    QPlan pl;
    PB_TRY(build_qplan(h, terms, 0, pl));
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    const void* bb = family == PB_QPOLY_2D ? b : nullptr;
    if (kind == PB_QPOLY_VALUE) launch_q<0, 0>(dtype, g, st, a, bb, count, pl, out0, nullptr, nullptr);
    else if (kind == PB_QPOLY_DER) launch_q<1, 0>(dtype, g, st, a, bb, count, pl, out0, out1, nullptr);
    else launch_q<2, 0>(dtype, g, st, a, b, count, pl, out0, out1, nullptr);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_qpoly_sum(pb_handle_t hh, int dtype, int family, const void* u, const void* t, long long count, int k,
                            const int* n_host, const int* m_host, const double* coefs_host, void* z, void* dzdr, void* dzdt,
                            void* stream) {
    PB_ENTER_REAL(hh);
    if (family < PB_QPOLY_BFS || family > PB_QPOLY_2D) return fail(h, PB_ERR_INVALID, "qpoly: bad family");
    if (!u || k < 0 || (k > 0 && (!n_host || !coefs_host || (family == PB_QPOLY_2D && !m_host))))
        return fail(h, PB_ERR_INVALID, "bad qpoly sum arguments");
    if (family == PB_QPOLY_2D && !t) return fail(h, PB_ERR_INVALID, "qpoly: 2D-Q sums need t");
    if (!z && !dzdr && !dzdt) return fail(h, PB_ERR_INVALID, "qpoly: no output");
    std::vector<QTerm> terms;
    PB_TRY(build_qterms(h, family, k, n_host, m_host, coefs_host, terms));
    QPlan pl;
    PB_TRY(build_qplan(h, terms, 1, pl));
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    const void* tt = family == PB_QPOLY_2D ? t : nullptr;
    if (dzdr || dzdt) launch_q<1, 1>(dtype, g, st, u, tt, count, pl, z, dzdr, dzdt);
    else launch_q<0, 1>(dtype, g, st, u, tt, count, pl, z, nullptr, nullptr);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_qpoly_tables(int family, int m, int nmax, double* out) {
    if (!out || nmax < 0 || nmax > PB_QPOLY_NMAX || family < PB_QPOLY_BFS || family > PB_QPOLY_2D) return PB_ERR_INVALID;
    if (family == PB_QPOLY_2D && (m < 1 || m > PB_QPOLY_NMAX)) return PB_ERR_INVALID;
    std::vector<double> f, g, hv;
    if (family == PB_QPOLY_BFS) qbfs_tables(nmax, f, g, hv);
    else if (family == PB_QPOLY_2D) q2d_fg(nmax, m, f, g);
    for (int n = 0; n <= nmax; ++n) {
        double* row = out + 7 * n;
        std::fill(row, row + 7, 0.0);
        if (family == PB_QPOLY_BFS) { row[0] = f[n]; row[1] = g[n]; row[2] = hv[n]; }
        else if (family == PB_QPOLY_CON) qcon_abc(n, row);
        else {
            q2d_abc(n, m, row);
            row[3] = q2d_G(n, m); row[4] = q2d_F(n, m); row[5] = g[n]; row[6] = f[n];
        }
    }
    return PB_OK;
}
