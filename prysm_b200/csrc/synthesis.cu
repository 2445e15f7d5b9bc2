// Pupil synthesis on the device -- the step before the path (SURVEY.md 8(f) rank 3): coordinate grids, circular
// masks (binary / one-sample grey edge), Zernike sequences, their polar and Cartesian derivatives and
// coefficient-weighted Zernike sums with and without slopes (the Jacobi sequences are in orthopoly.cu).  All streaming, HBM-bound on their outputs; the recurrences run in fp64
// registers whatever the storage precision (the reference runs them in config precision, prysm/polynomials/
// jacobi.py:147-175, zernike.py:74-181) and are driven by a plan passed in kernel-parameter space, so a launch
// reads no table from memory and is CUDA-graph capturable.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace pb {

// x = (ix - nx/2)*dx, y = (iy - ny/2)*dx in working precision (prysm/coordinates.py:344-378); r, t from them
template <typename R>
__global__ void xy_grid_kernel(int ny, int nx, double dx, R* __restrict__ x, R* __restrict__ y, R* __restrict__ r, R* __restrict__ t) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int iy = (int)(i / nx), ix = (int)(i - (long long)iy * nx);
        const R xv = mul_rn((R)(ix - nx / 2), (R)dx), yv = mul_rn((R)(iy - ny / 2), (R)dx);
        if (x) x[i] = xv;
        if (y) y[i] = yv;
        if (r) r[i] = (R)hypot((double)xv, (double)yv);
        if (t) t[i] = (R)atan2((double)yv, (double)xv);
    }
}

template <typename R>
__global__ void cart_to_polar_kernel(const R* __restrict__ x, const R* __restrict__ y, long long n, R* __restrict__ r, R* __restrict__ t) {
    PB_GRID_STRIDE(i, n) {
        const double xv = x[i], yv = y[i];
        if (r) r[i] = (R)hypot(xv, yv);
        if (t) t[i] = (R)atan2(yv, xv);
    }
}

// aa_dx <= 0: out(u8) = (r - radius <= 0)            (geometry.circle, prysm/geometry.py:337-372)
// aa_dx  > 0: out(R)  = clip(0.5 - (r - radius)/aa_dx, 0, 1)   (antialias(circle_sdf), geometry.py:11-34)
template <typename R>
__global__ void circle_kernel(const R* __restrict__ r, long long n, R radius, R aa_dx, void* out) {
    PB_GRID_STRIDE(i, n) {
        const R d = r[i] - radius;
        if (aa_dx > R(0)) {
            const R c = R(0.5) - d / aa_dx;
            reinterpret_cast<R*>(out)[i] = c < R(0) ? R(0) : (c > R(1) ? R(1) : c);
        } else {
            reinterpret_cast<unsigned char*>(out)[i] = d <= R(0) ? 1 : 0;
        }
    }
}

// Zernike plan: one group per |m| (ascending); per Jacobi order j of a group one step holding the recurrence
// coefficients that make P_j and the weights of the (at most one) cosine and sine mode of that (|m|, j).
// m = 0 modes are "cosine" modes of the |m| = 0 group (cos 0 = r^0 = 1).  Every index is warp-uniform, so the
// plan is read through the constant bank with uniform loads.
#define PB_ZERN_GROUPS 24
#define PB_ZERN_STEPS 72
struct ZernGroup { short am, njmax, first, pad; };
struct ZernStep { double A, B, C, wc, ws; };     // P_j = (A x + B) P_{j-1} - C P_{j-2};  value = P_j r^|m| (wc cos + ws sin)
struct ZernPlan {
    int ngroups;
    ZernGroup g[PB_ZERN_GROUPS];
    short kc[PB_ZERN_STEPS], ks[PB_ZERN_STEPS];  // output slots of the cosine / sine mode of a step (MODE 0), -1 = absent
    ZernStep s[PB_ZERN_STEPS];
};

// MODE 0: out[k][i] = w * Z_k   (zernike_nm_seq);  MODE 1: out[i] (+)= sum w * Z_k  (zernike_sum, w = c*norm)
// MODE 2 (POLAR): out[k][0|1][i] = w dZ_k/dr, w dZ_k/dt  (zernike_nm_der_seq)
// MODE 3: out[k][0|1][i] = w dZ_k/dx, w dZ_k/dy  (zernike_nm_der_xy_seq)
// MODE 4: out[0|1|2][i] (+)= W, dW/dx, dW/dy of W = sum w Z_k  (zernike_sum_der_xy)
// MODES 1 and 4 split over several plans carry the partial sums from launch to launch in the fp64 `stage` (the output
// itself for fp64 storage, so neither `stage` nor `out` is __restrict__) and round to R once, in the `last` launch.
// POLAR: inputs are (r, t); otherwise Cartesian (x, y) with r = hypot, cos t = x/r, sin t = y/r.  The derivative modes
// carry dP_j/dx2 beside P_j (seed (|m| + 2)/2, the differentiated recurrence); MODE 2 forms r^|m|, r^(|m|-1) and
// cos / sin(|m| t) per group, MODES 3 and 4 C_k, S_k = Re, Im (x + iy)^k for k = |m| and |m| - 1, finite at the origin.
template <typename R, int MODE, bool POLAR>
__global__ void zernike_kernel(const R* __restrict__ a, const R* __restrict__ b, long long n, const __grid_constant__ ZernPlan pl,
                               int accumulate, int last, double* stage, R* out) {
    constexpr bool DER = MODE >= 2, XY = MODE >= 3;
    PB_GRID_STRIDE(i, n) {
        double r = 0.0, c1 = 1.0, s1 = 0.0, xv = 0.0, yv = 0.0, tv = 0.0;
        if constexpr (XY) {
            xv = a[i]; yv = b[i];
        } else if constexpr (MODE == 2) {
            r = a[i]; tv = b[i];
        } else if (POLAR) {
            r = a[i];
            sincos((double)b[i], &s1, &c1);
        } else {
            const double xv = a[i], yv = b[i];
            r = hypot(xv, yv);
            c1 = r > 0.0 ? xv / r : 1.0;
            s1 = r > 0.0 ? yv / r : 0.0;
        }
        const double x2 = XY ? 2.0 * (xv * xv + yv * yv) - 1.0 : 2.0 * (r * r) - 1.0, hx = (x2 - 1.0) / 2.0;
        double rc = 1.0, rs = 0.0;                // r^am cos(am t), r^am sin(am t), advanced group to group
        const double rc1 = r * c1, rs1 = r * s1;
        double hc1 = 1.0, hs1 = 0.0;              // MODE 3, 4: (rc, rs) = Re, Im (x + iy)^am, (hc1, hs1) of ^(am - 1)
        double rm = 1.0, rm1 = 1.0, cs = 1.0, sn = 0.0;   // MODE 2: r^am, r^(am - 1), cos(am t), sin(am t)
        int am_now = 0;
        double acc = 0.0, accx = 0.0, accy = 0.0;
        for (int gi = 0; gi < pl.ngroups; ++gi) {
            const ZernGroup g = pl.g[gi];
            for (; am_now < g.am; ++am_now) {     // (r e^{it})^am by repeated complex multiplication
                if constexpr (XY) {
                    hc1 = rc; hs1 = rs;
                    const double t0 = xv * rc - yv * rs;
                    rs = xv * rs + yv * rc;
                    rc = t0;
                } else if constexpr (MODE == 2) {
                    rm1 = rm; rm = rm * r;
                } else {
                    const double t0 = rc * rc1 - rs * rs1;
                    rs = rs * rc1 + rc * rs1;
                    rc = t0;
                }
            }
            if constexpr (MODE == 2) sincos((double)g.am * tv, &sn, &cs);
            const double am = g.am;
            double Pm2 = 1.0, Pm1 = 1.0 + ((double)g.am + 2.0) * hx, P = 1.0;
            double dPm2 = 0.0, dPm1 = ((double)g.am + 2.0) / 2.0, dP = 0.0;
            double Sa = 0.0, Sb = 0.0, dSa = 0.0, dSb = 0.0;
            for (int j = 0; j <= g.njmax; ++j) {
                const int si = g.first + j;
                if (j == 1) { P = Pm1; dP = dPm1; }
                else if (j >= 2) {
                    if constexpr (DER) {
                        const double lin = pl.s[si].A * x2 + pl.s[si].B;
                        P = lin * Pm1 - pl.s[si].C * Pm2;
                        dP = pl.s[si].A * Pm1 + lin * dPm1 - pl.s[si].C * dPm2;
                        dPm2 = dPm1; dPm1 = dP;
                    } else {
                        P = (pl.s[si].A * x2 + pl.s[si].B) * Pm1 - pl.s[si].C * Pm2;
                    }
                    Pm2 = Pm1; Pm1 = P;
                }
                if constexpr (MODE == 1) {
                    acc += P * (pl.s[si].wc * rc + pl.s[si].ws * rs);
                } else if constexpr (MODE == 4) {
                    Sa += pl.s[si].wc * P; Sb += pl.s[si].ws * P;
                    dSa += pl.s[si].wc * dP; dSb += pl.s[si].ws * dP;
                } else {
                    const int kc = pl.kc[si], ks = pl.ks[si];
                    if constexpr (MODE == 0) {
                        if (kc >= 0) out[(long long)kc * n + i] = (R)(pl.s[si].wc * P * rc);
                        if (ks >= 0) out[(long long)ks * n + i] = (R)(pl.s[si].ws * P * rs);
                    } else if constexpr (MODE == 2) {
                        const double radial = g.am == 0 ? (4.0 * r) * dP : am * rm1 * P + rm * ((4.0 * r) * dP);
                        if (kc >= 0) {
                            out[(long long)(2 * kc) * n + i] = (R)(pl.s[si].wc * (radial * cs));
                            out[(long long)(2 * kc + 1) * n + i] = (R)(g.am == 0 ? 0.0 : pl.s[si].wc * (-am * sn * rm * P));
                        }
                        if (ks >= 0) {
                            out[(long long)(2 * ks) * n + i] = (R)(pl.s[si].ws * (radial * sn));
                            out[(long long)(2 * ks + 1) * n + i] = (R)(pl.s[si].ws * (am * cs * rm * P));
                        }
                    } else {
                        const double ddx = 4.0 * xv * dP, ddy = 4.0 * yv * dP;
                        if (kc >= 0) {
                            out[(long long)(2 * kc) * n + i] = (R)(pl.s[si].wc * (ddx * rc + am * P * hc1));
                            out[(long long)(2 * kc + 1) * n + i] = (R)(pl.s[si].wc * (ddy * rc - am * P * hs1));
                        }
                        if (ks >= 0) {
                            out[(long long)(2 * ks) * n + i] = (R)(pl.s[si].ws * (ddx * rs + am * P * hs1));
                            out[(long long)(2 * ks + 1) * n + i] = (R)(pl.s[si].ws * (ddy * rs + am * P * hc1));
                        }
                    }
                }
            }
            if constexpr (MODE == 4) {
                const double dH = dSa * rc + dSb * rs;
                acc += Sa * rc + Sb * rs;
                accx += 4.0 * xv * dH + am * (Sa * hc1 + Sb * hs1);
                accy += 4.0 * yv * dH + am * (Sb * hc1 - Sa * hs1);
            }
        }
        if constexpr (MODE == 1) {
            if (accumulate) acc += stage[i];
            if (last) out[i] = (R)acc;
            else stage[i] = acc;
        }
        if constexpr (MODE == 4) {
            if (accumulate) {
                acc += stage[i]; accx += stage[n + i]; accy += stage[2 * n + i];
            }
            if (last) { out[i] = (R)acc; out[n + i] = (R)accx; out[2 * n + i] = (R)accy; }
            else { stage[i] = acc; stage[n + i] = accx; stage[2 * n + i] = accy; }
        }
    }
}

// DLMF 18.9 coefficients as the reference writes them (prysm/polynomials/jacobi.py:13-39)
void jacobi_abc(int n, double alpha, double beta, double* abc) {
    const double apb = alpha + beta;
    if (n == 0 && (apb == 0.0 || apb == -1.0)) {
        abc[0] = 0.5 * (alpha + beta) + 1.0; abc[1] = 0.5 * (alpha - beta); abc[2] = 1.0;
        return;
    }
    abc[0] = ((2 * n + alpha + beta + 1) * (2 * n + alpha + beta + 2)) / (2 * (n + 1) * (n + alpha + beta + 1));
    abc[1] = ((alpha * alpha - beta * beta) * (2 * n + alpha + beta + 1)) / (2 * (n + 1) * (n + alpha + beta + 1) * (2 * n + alpha + beta));
    abc[2] = ((n + alpha) * (n + beta) * (2 * n + alpha + beta + 2)) / ((n + 1) * (n + alpha + beta + 1) * (2 * n + alpha + beta));
}

struct HostTerm { int am, nj, trig, k; double scale; };   // trig 1: cosine (and m = 0), 2: sine

// Fills a plan with as many whole |m| groups as fit; duplicate (n, m) pairs beyond the first stay in `terms` for a
// later plan (a step holds one cosine and one sine weight).
static int next_plan(std::vector<HostTerm>& terms, ZernPlan& pl) {
    pl.ngroups = 0;
    int nsteps = 0;
    std::vector<HostTerm> rest;
    size_t pos = 0;
    bool full = false;
    while (pos < terms.size()) {
        size_t end = pos;
        int njmax = 0;
        while (end < terms.size() && terms[end].am == terms[pos].am) { njmax = std::max(njmax, terms[end].nj); ++end; }
        if (njmax + 1 > PB_ZERN_STEPS) return PB_ERR_UNSUPPORTED;
        if (full || pl.ngroups == PB_ZERN_GROUPS || nsteps + njmax + 1 > PB_ZERN_STEPS) {
            full = true;
            rest.insert(rest.end(), terms.begin() + pos, terms.begin() + end);
            pos = end;
            continue;
        }
        ZernGroup& g = pl.g[pl.ngroups++];
        g.am = (short)terms[pos].am; g.njmax = (short)njmax; g.first = (short)nsteps; g.pad = 0;
        for (int j = 0; j <= njmax; ++j) {
            ZernStep& st = pl.s[nsteps + j];
            double abc[3] = {0.0, 0.0, 0.0};
            if (j >= 2) jacobi_abc(j - 1, 0.0, (double)g.am, abc);
            st.A = abc[0]; st.B = abc[1]; st.C = abc[2]; st.wc = 0.0; st.ws = 0.0;
            pl.kc[nsteps + j] = -1; pl.ks[nsteps + j] = -1;
        }
        for (size_t q = pos; q < end; ++q) {
            const HostTerm& t = terms[q];
            const int si = nsteps + t.nj;
            short& slot = t.trig == 2 ? pl.ks[si] : pl.kc[si];
            if (slot >= 0) { rest.push_back(t); continue; }       // a repeated (n, m): next plan
            slot = (short)t.k;
            (t.trig == 2 ? pl.s[si].ws : pl.s[si].wc) = t.scale;
        }
        nsteps += njmax + 1;
        pos = end;
    }
    terms.swap(rest);
    return PB_OK;
}

static int build_terms(Handle* h, int k, const int* n_host, const int* m_host, const double* coefs, int norm,
                       std::vector<HostTerm>& terms) {
    terms.clear();
    for (int q = 0; q < k; ++q) {
        const int n = n_host[q], m = m_host[q], am = m < 0 ? -m : m;
        if (n < 0 || am > n || ((n - am) & 1)) return fail(h, PB_ERR_INVALID, "zernike (n, m): need n >= |m| and n - |m| even");
        if (coefs && coefs[q] == 0.0) continue;                              // zernike.py:178-179 skips zero weights
        double sc = coefs ? coefs[q] : 1.0;
        if (norm) sc *= std::sqrt((2.0 * (n + 1)) / (m == 0 ? 2.0 : 1.0));   // zernike_norm, zernike.py:25-27
        terms.push_back({am, (n - am) / 2, m < 0 ? 2 : 1, q, sc});
    }
    std::stable_sort(terms.begin(), terms.end(), [](const HostTerm& a, const HostTerm& b) {
        return a.am != b.am ? a.am < b.am : a.nj < b.nj;
    });
    return PB_OK;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_xy_grid(pb_handle_t hh, int dtype, int ny, int nx, double dx, void* x, void* y, void* r, void* t, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "bad grid shape");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto real) {
        using R = decltype(real);
        xy_grid_kernel<R><<<g, 256, 0, st>>>(ny, nx, dx, (R*)x, (R*)y, (R*)r, (R*)t);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_cart_to_polar(pb_handle_t hh, int dtype, const void* x, const void* y, long long count, void* r, void* t,
                                void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !y) return fail(h, PB_ERR_INVALID, "null coordinates");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto real) {
        using R = decltype(real);
        cart_to_polar_kernel<R><<<g, 256, 0, st>>>((const R*)x, (const R*)y, count, (R*)r, (R*)t);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_circle(pb_handle_t hh, int dtype, const void* r, long long count, double radius, double aa_dx, void* out,
                         void* stream) {
    PB_ENTER_REAL(hh);
    if (!r || !out) return fail(h, PB_ERR_INVALID, "null pointer");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto real) {
        using R = decltype(real);
        circle_kernel<R><<<g, 256, 0, st>>>((const R*)r, count, (R)radius, (R)aa_dx, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

// a radial order no plan can hold is refused before the first of several launches
static int zernike_fits(Handle* h, const std::vector<HostTerm>& terms) {
    for (const HostTerm& t : terms)
        if (t.nj + 1 > PB_ZERN_STEPS) return fail(h, PB_ERR_UNSUPPORTED, "zernike: (n - |m|)/2 above 71");
    return PB_OK;
}

template <int MODE>
static int run_zernike(Handle* h, int dtype, int polar, const void* a, const void* b, long long count,
                       std::vector<HostTerm>& terms, void* out, cudaStream_t st) {
    const int g = grid_for(count, 256, h->sm_count);
    int launches = 0;
    if ((MODE == 1 || MODE == 4) && terms.empty()) {      // all weights zero: the sum (and its slopes) is zero
        PB_CUDA(h, cudaMemsetAsync(out, 0, (size_t)count * rsize(dtype) * (MODE == 4 ? 3 : 1), st));
        return PB_OK;
    }
    double* stage = nullptr;
    while (!terms.empty()) {
        ZernPlan pl;
        PB_TRY(next_plan(terms, pl));
        const int acc = launches > 0, last = terms.empty();
        if ((MODE == 1 || MODE == 4) && !last && !stage) {
            // the partial sums of a split call stay in fp64 until the last launch rounds them once
            if (dtype == PB_C128) stage = (double*)out;
            else {
                void* p = nullptr;
                PB_TRY(ensure_scratch(h, 2, (size_t)count * sizeof(double) * (MODE == 4 ? 3 : 1), &p));
                stage = (double*)p;
            }
        }
        with_real(dtype, [&](auto r) {
            using R = decltype(r);
            if (polar) zernike_kernel<R, MODE, true><<<g, 256, 0, st>>>((const R*)a, (const R*)b, count, pl, acc, last, stage, (R*)out);
            else zernike_kernel<R, MODE, false><<<g, 256, 0, st>>>((const R*)a, (const R*)b, count, pl, acc, last, stage, (R*)out);
        });
        PB_LAUNCH_CHECK(h);
        ++launches;
    }
    return PB_OK;
}

extern "C" int pb_zernike_seq(pb_handle_t hh, int dtype, int polar, const void* a, const void* b, long long count, int k,
                              const int* n_host, const int* m_host, int norm, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !b || !out || k < 1 || !n_host || !m_host) return fail(h, PB_ERR_INVALID, "bad zernike arguments");
    if (k > 32767) return fail(h, PB_ERR_UNSUPPORTED, "more than 32767 modes");
    if (count <= 0) return PB_OK;
    std::vector<HostTerm> terms;
    PB_TRY(build_terms(h, k, n_host, m_host, nullptr, norm, terms));
    PB_TRY(zernike_fits(h, terms));
    return run_zernike<0>(h, dtype, polar, a, b, count, terms, out, st);
}

extern "C" int pb_zernike_sum(pb_handle_t hh, int dtype, int polar, const void* a, const void* b, long long count, int k,
                              const int* n_host, const int* m_host, const double* coefs_host, int norm, void* out,
                              void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !b || !out || k < 0 || (k > 0 && (!n_host || !m_host || !coefs_host))) return fail(h, PB_ERR_INVALID, "bad zernike arguments");
    if (count <= 0) return PB_OK;
    std::vector<HostTerm> terms;
    PB_TRY(build_terms(h, k, n_host, m_host, coefs_host, norm, terms));
    PB_TRY(zernike_fits(h, terms));
    return run_zernike<1>(h, dtype, polar, a, b, count, terms, out, st);
}

extern "C" int pb_zernike_der(pb_handle_t hh, int dtype, int cartesian, const void* a, const void* b, long long count, int k,
                              const int* n_host, const int* m_host, int norm, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !b || !out || k < 1 || !n_host || !m_host) return fail(h, PB_ERR_INVALID, "bad zernike arguments");
    if (k > 16383) return fail(h, PB_ERR_UNSUPPORTED, "more than 16383 modes");
    std::vector<HostTerm> terms;
    PB_TRY(build_terms(h, k, n_host, m_host, nullptr, norm, terms));
    PB_TRY(zernike_fits(h, terms));
    if (count <= 0) return PB_OK;
    if (cartesian) return run_zernike<3>(h, dtype, 0, a, b, count, terms, out, st);
    return run_zernike<2>(h, dtype, 1, a, b, count, terms, out, st);
}

extern "C" int pb_zernike_sum_der_xy(pb_handle_t hh, int dtype, const void* x, const void* y, long long count, int k,
                                     const int* n_host, const int* m_host, const double* coefs_host, int norm, void* out,
                                     void* stream) {
    PB_ENTER_REAL(hh);
    if (!x || !y || !out || k < 0 || (k > 0 && (!n_host || !m_host || !coefs_host))) return fail(h, PB_ERR_INVALID, "bad zernike arguments");
    std::vector<HostTerm> terms, merged;
    PB_TRY(build_terms(h, k, n_host, m_host, coefs_host, norm, terms));
    // duplicate (n, m) pairs add their weights, in input order, as zernike.py:574-584 does
    for (const HostTerm& t : terms) {
        auto same = [&](const HostTerm& u) { return u.am == t.am && u.nj == t.nj && u.trig == t.trig; };
        auto it = std::find_if(merged.begin(), merged.end(), same);
        if (it == merged.end()) merged.push_back({t.am, t.nj, t.trig, t.k, 0.0 + t.scale});
        else it->scale += t.scale;
    }
    PB_TRY(zernike_fits(h, merged));
    if (count <= 0) return PB_OK;
    return run_zernike<4>(h, dtype, 0, x, y, count, merged, out, st);
}
