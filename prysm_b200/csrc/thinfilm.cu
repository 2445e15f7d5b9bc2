// Thin-film stacks on the device: the characteristic-matrix chain of prysm/thinfilm.py (multilayer_stack_rt) and of
// prysm/x/coatings (stack.py: r, t, boundary fields, R / T / per-layer A; diff.py: thickness and index gradients), and
// the field at arbitrary depth.
//
// One thread per sample (wavelength, angle, pixel).  The forward pass is one sweep from the substrate to the ambient
// side, v_N = [1, eta_sub], v_k = M_k v_{k+1}, (B, C) = v_0, the suffix products of the reference applied to a vector;
// the boundary fields are f_k = t v_k.  The gradient reads f_k back and runs the reverse sweep
// vbar_{k+1} += M_k^H vbar_k, Mbar_k = vbar_k v_{k+1}^H: v_{k+1} is never recovered from v_k by inverting M_k, which
// through an absorbing or evanescent layer would amplify the rounding error by about exp(2 |Im beta|).
// Every operand is fp64 and all arithmetic is fp64 in registers; the outputs are rounded once to the storage type.
#include <climits>
#include <cmath>

#include "common.cuh"

namespace pb {

#define PB_TF_THREADS 256

struct TfOut { void* p[PB_TF_NOUT]; };

struct TfOps {
    long long shape[PB_TF_DIMS];                 // collapsed calculation shape, padded with 1 in front
    long long st[PB_TF_NOPS][PB_TF_DIMS + 1];    // per operand: calculation strides, then the layer stride
    const void* p[PB_TF_NOPS];
    double theta_scale;          // radians per unit of the angle operand
    int nlayers, pol;
};

// complex helpers with numpy's rules, so that signed zeros on the branch cut of the square root come out as the
// reference's do: Smith's division (numpy's complex divide) and the C99 principal square root
__device__ inline double2 tf_div(double2 a, double2 b) {
    if (fabs(b.x) >= fabs(b.y)) {
        const double rat = b.y / b.x, scl = 1.0 / (b.x + b.y * rat);
        return make_double2((a.x + a.y * rat) * scl, (a.y - a.x * rat) * scl);
    }
    const double rat = b.x / b.y, scl = 1.0 / (b.y + b.x * rat);
    return make_double2((a.x * rat + a.y) * scl, (a.y * rat - a.x) * scl);
}

__device__ inline double2 tf_sqrt(double2 z) {
    if (z.x == 0.0 && z.y == 0.0) return make_double2(0.0, z.y);
    const double t = sqrt((fabs(z.x) + hypot(z.x, z.y)) * 0.5);
    if (z.x >= 0.0) return make_double2(t, z.y / (2.0 * t));
    return make_double2(fabs(z.y) / (2.0 * t), copysign(t, z.y));
}

// _cos_snell (thinfilm.py:75-80): sqrt(1 - sint^2) on the principal branch, negated for a real sint > 1
__device__ inline double2 tf_cos_snell(double2 n0, double2 n, double sin0) {
    const double2 q = tf_div(n0, n);
    const double2 s = make_double2(q.x * sin0 - q.y * 0.0, q.x * 0.0 + q.y * sin0);
    const double2 s2 = cmul(s, s);
    double2 c = tf_sqrt(make_double2(1.0 - s2.x, 0.0 - s2.y));
    if (s.y == 0.0 && s.x > 1.0) c = make_double2(-c.x, -c.y);
    return c;
}

// tilted admittance: n / cos (p) or n cos (s)
__device__ inline double2 tf_admittance(double2 n, double2 cost, int pol) {
    return pol == PB_TF_POL_P ? tf_div(n, cost) : cmul(n, cost);
}

// sin and cos of a complex argument
__device__ inline void tf_sincos(double2 b, double2* sb, double2* cb) {
    // sincospi has no slow-path argument reduction (a call that costs registers); b.x / pi adds one rounding,
    // a phase error of |b.x| * 1e-16
    double s, c;
    sincospi(b.x * M_1_PI, &s, &c);
    // cosh and sinh of |Im b| from one expm1 (sinh stays accurate for small |Im b|, and e^|Im b| never cancels), the
    // sign restored after: cosh is even and sinh odd.  Im b < 0 is an evanescent layer under total internal reflection.
    const double em1 = expm1(fabs(b.y)), e = 1.0 + em1;
    const double ch = 0.5 * (e + 1.0 / e), sh = copysign(0.5 * em1 * (1.0 + 1.0 / e), b.y);
    *sb = make_double2(s * ch, c * sh);
    *cb = make_double2(c * ch, -s * sh);
}

struct TfSample {
    long long off_n, off_d;      // offsets of the per-layer operands at layer 0
    double wvl, sin0, cos0;
    double2 n0, nsub;
};

__device__ inline TfSample tf_sample(const TfOps& op, long long i) {
    long long idx[PB_TF_DIMS];
    for (int j = PB_TF_DIMS - 1; j >= 0; --j) {
        idx[j] = i % op.shape[j];
        i /= op.shape[j];
    }
    long long off[PB_TF_NOPS];
    for (int q = 0; q < PB_TF_NOPS; ++q) {
        off[q] = 0;
        for (int j = 0; j < PB_TF_DIMS; ++j) off[q] += idx[j] * op.st[q][j];
    }
    TfSample s;
    s.off_n = off[PB_TF_IN_N];
    s.off_d = off[PB_TF_IN_D];
    s.wvl = ((const double*)op.p[PB_TF_IN_WVL])[off[PB_TF_IN_WVL]];
    sincos(((const double*)op.p[PB_TF_IN_THETA])[off[PB_TF_IN_THETA]] * op.theta_scale, &s.sin0, &s.cos0);
    s.n0 = ((const double2*)op.p[PB_TF_IN_N0])[off[PB_TF_IN_N0]];
    s.nsub = ((const double2*)op.p[PB_TF_IN_NSUB])[off[PB_TF_IN_NSUB]];
    return s;
}

// the substrate's tilted admittance
__device__ __forceinline__ double2 tf_eta_sub(const TfSample& s, int pol) {
    return tf_admittance(s.nsub, tf_cos_snell(s.n0, s.nsub, s.sin0), pol);
}

// layer k of a sample: index, cos theta_k, phase thickness beta, admittance eta and thickness
struct TfLayer { double2 n, cost, beta, eta; double d; };

// the phase thickness 2 pi n d cos / wvl of a layer of index n and thickness d
__device__ __forceinline__ double2 tf_beta(double2 n, double2 cost, double d, double wvl) {
    return cscale(cmul(cscale(n, 2.0 * M_PI * d), cost), 1.0 / wvl);
}

__device__ inline TfLayer tf_layer(const TfOps& op, const TfSample& s, int k, int pol) {
    TfLayer L;
    L.n = ((const double2*)op.p[PB_TF_IN_N])[s.off_n + (long long)k * op.st[PB_TF_IN_N][PB_TF_DIMS]];
    L.d = ((const double*)op.p[PB_TF_IN_D])[s.off_d + (long long)k * op.st[PB_TF_IN_D][PB_TF_DIMS]];
    L.cost = tf_cos_snell(s.n0, L.n, s.sin0);
    L.beta = tf_beta(L.n, L.cost, L.d, s.wvl);
    L.eta = tf_admittance(L.n, L.cost, pol);
    return L;
}

__device__ inline TfLayer tf_layer(const TfOps& op, const TfSample& s, int k) { return tf_layer(op, s, k, op.pol); }

// v <- M v with M = [[cos b, -i sin b / eta], [-i eta sin b, cos b]]
__device__ inline void tf_apply(double2 sb, double2 cb, double2 eta, double2& v0, double2& v1) {
    const double2 mis = make_double2(sb.y, -sb.x);               // -i sin b
    const double2 a = cadd(cmul(cb, v0), cmul(tf_div(mis, eta), v1));
    const double2 b = cadd(cmul(cmul(mis, eta), v0), cmul(cb, v1));
    v0 = a; v1 = b;
}

// vbar <- M^H vbar, the same M
__device__ __forceinline__ void tf_apply_adjoint(double2 sb, double2 cb, double2 eta, double2& vb0, double2& vb1) {
    const double2 mis = make_double2(sb.y, -sb.x);
    const double2 M01 = tf_div(mis, eta), M10 = cmul(mis, eta);
    const double2 nb0 = cadd(cmulc(vb0, cb), cmulc(vb1, M10));
    const double2 nb1 = cadd(cmulc(vb0, M01), cmulc(vb1, cb));
    vb0 = nb0; vb1 = nb1;
}

// the forward sweep from v = v_N on the substrate side, v_k = M_k v_{k+1}, to v = v_0 = (B, C); visit(k, v0, v1) sees
// every boundary k = N, ..., 0
template <typename Visit>
__device__ __forceinline__ void tf_sweep(const TfOps& op, const TfSample& s, int pol, double2& v0, double2& v1,
                                         Visit&& visit) {
    visit(op.nlayers, v0, v1);
    for (int k = op.nlayers - 1; k >= 0; --k) {
        const TfLayer L = tf_layer(op, s, k, pol);
        double2 sb, cb;
        tf_sincos(L.beta, &sb, &cb);
        tf_apply(sb, cb, L.eta, v0, v1);
        visit(k, v0, v1);
    }
}

__device__ inline double tf_abs2(double2 a) { return a.x * a.x + a.y * a.y; }

// fp64 staging of the field outputs before they are scaled by t: |v_k| grows like e^|Im beta| through an absorbing or
// evanescent layer and geometrically through a long high-contrast stack, which would overflow float32.  For fp64
// outputs the stage is the output itself.
struct TfStage { double2* E; double2* H; double* Esq; double* A; };

template <typename R, int MODE>
__global__ void stack_eval_kernel(const TfOps op, long long count, TfOut o, TfStage sg) {
    const int N = op.nlayers;
    const bool fields = sg.E || sg.H || sg.Esq || sg.A;
    PB_GRID_STRIDE(i, count) {
        const TfSample s = tf_sample(op, i);
        const double2 nsub = s.nsub;
        const double2 cos_sub = tf_cos_snell(s.n0, nsub, s.sin0);
        const double2 eta_sub = tf_admittance(nsub, cos_sub, op.pol);
        double2 v0, v1;
        if (MODE == PB_TF_THINFILM && op.pol == PB_TF_POL_P) { v0 = cos_sub; v1 = nsub; }
        else { v0 = make_double2(1.0, 0.0); v1 = MODE == PB_TF_THINFILM ? cmul(nsub, cos_sub) : eta_sub; }
        // v_k, |v_k,E|^2 and the flux differences are staged in fp64 and scaled by t or |t|^2 once v_0 (hence t)
        // is known
        double g_below = 0.0;
        tf_sweep(op, s, op.pol, v0, v1, [&](int k, double2 e, double2 h) {
            if (!fields) return;
            const long long ok = (long long)k * count + i;
            if (sg.E) sg.E[ok] = e;
            if (sg.H) sg.H[ok] = h;
            if (sg.Esq) sg.Esq[ok] = tf_abs2(e);
            const double g = cmulc(e, h).x;
            if (sg.A && k < N) sg.A[ok] = g - g_below;
            g_below = g;
        });
        double2 r, t;
        if (MODE == PB_TF_THINFILM) {
            // multilayer_stack_rt (thinfilm.py:295-311): term1 = 1 / (2 n0 cos0)
            const double2 term1 = tf_div(make_double2(1.0, 0.0), cscale(s.n0, 2.0 * s.cos0));
            const double2 a = op.pol == PB_TF_POL_P ? s.n0 : cscale(s.n0, s.cos0);
            const double2 q1 = op.pol == PB_TF_POL_P ? cscale(v1, s.cos0) : v1;
            const double2 aq = cmul(a, v0);
            const double2 A00 = cmul(term1, cadd(aq, q1)), A10 = cmul(term1, csub(aq, q1));
            r = tf_div(A10, A00);
            t = tf_div(make_double2(1.0, 0.0), A00);
        } else {
            const double2 eta0 = tf_admittance(s.n0, make_double2(s.cos0, 0.0), op.pol);
            const double2 eb = cmul(eta0, v0);
            const double2 den = cadd(eb, v1);
            r = tf_div(csub(eb, v1), den);
            t = tf_div(cscale(eta0, 2.0), den);
            if (o.p[PB_TF_OUT_ETA0]) ((cplx<R>*)o.p[PB_TF_OUT_ETA0])[i] = mk<R>((R)eta0.x, (R)eta0.y);
            if (o.p[PB_TF_OUT_ETASUB]) ((cplx<R>*)o.p[PB_TF_OUT_ETASUB])[i] = mk<R>((R)eta_sub.x, (R)eta_sub.y);
            if (o.p[PB_TF_OUT_TRANS]) ((R*)o.p[PB_TF_OUT_TRANS])[i] = (R)(eta_sub.x / eta0.x * tf_abs2(t));
            if (fields) {
                const double t2 = tf_abs2(t), fscale = t2 / eta0.x;
                cplx<R>* const Eo = (cplx<R>*)o.p[PB_TF_OUT_E];
                cplx<R>* const Ho = (cplx<R>*)o.p[PB_TF_OUT_H];
                R* const Esq = (R*)o.p[PB_TF_OUT_ESQ];
                R* const Ab = (R*)o.p[PB_TF_OUT_ABS];
                for (int k = 0; k <= N; ++k) {
                    const long long ok = (long long)k * count + i;
                    if (Eo) { const double2 v = cmul(t, sg.E[ok]); Eo[ok] = mk<R>((R)v.x, (R)v.y); }
                    if (Ho) { const double2 v = cmul(t, sg.H[ok]); Ho[ok] = mk<R>((R)v.x, (R)v.y); }
                    if (Esq) Esq[ok] = (R)(sg.Esq[ok] * t2);
                    if (Ab && k < N) Ab[ok] = (R)(sg.A[ok] * fscale);
                }
            }
        }
        if (o.p[PB_TF_OUT_R]) ((cplx<R>*)o.p[PB_TF_OUT_R])[i] = mk<R>((R)r.x, (R)r.y);
        if (o.p[PB_TF_OUT_T]) ((cplx<R>*)o.p[PB_TF_OUT_T])[i] = mk<R>((R)t.x, (R)t.y);
        if (o.p[PB_TF_OUT_REFL]) ((R*)o.p[PB_TF_OUT_REFL])[i] = (R)tf_abs2(r);
    }
}

// cotangent (Ebar, Hbar) = (H cf + 2 ce E, E cf) of a boundary field (E, H) (diff.py:204-224), from the coefficients
// of its flux Re(E conj H) (cf) and of |E|^2 (ce)
__device__ __forceinline__ void tf_field_cot(double cf, double ce, double2 E, double2 H, double2& Eb, double2& Hb) {
    Eb = cadd(cscale(H, cf), cscale(E, 2.0 * ce));
    Hb = cscale(E, cf);
}

// cotangent of boundary field k from the field seeds: flux_k = Re(E_k conj H_k) / Re(eta0) enters A_k with +1 and
// A_{k-1} with -1
__device__ inline void tf_field_bar(const double* dA, const double* dEsq, int N, long long count, long long i, int k,
                                    double inv_re0, double2 E, double2 H, double2& Eb, double2& Hb) {
    double fb = 0.0;
    if (dA) {
        if (k < N) fb += dA[(long long)k * count + i];
        if (k > 0) fb -= dA[(long long)(k - 1) * count + i];
    }
    fb *= inv_re0;
    tf_field_cot(fb, dEsq ? dEsq[(long long)k * count + i] : 0.0, E, H, Eb, Hb);
}

// vbar_0 = (Bbar, Cbar) from the amplitude cotangents rb, tb through the holomorphic partials of r and t in
// (B, C) = v_0 (diff.py:162-188); den = eta0 B + C
__device__ __forceinline__ void tf_seed(double2 r, double2 t, double2 eta0, double2 den, double2 rb, double2 tb,
                                        double2& vb0, double2& vb1) {
    const double2 inv_den = tf_div(make_double2(1.0, 0.0), den);
    const double2 dr_dB = cmul(cmul(eta0, make_double2(1.0 - r.x, -r.y)), inv_den);
    const double2 dr_dC = cmul(make_double2(-1.0 - r.x, -r.y), inv_den);
    const double2 dt_dB = cmul(make_double2(-(t.x * eta0.x - t.y * eta0.y), -(t.x * eta0.y + t.y * eta0.x)), inv_den);
    const double2 dt_dC = cmul(make_double2(-t.x, -t.y), inv_den);
    vb0 = cadd(cmulc(rb, dr_dB), cmulc(tb, dt_dB));
    vb1 = cadd(cmulc(rb, dr_dC), cmulc(tb, dt_dC));
}

// the thickness and index terms of one layer
struct TfGrad { double th, ix; };

// one layer of the reverse sweep: Mbar_k = vbar_k v_{k+1}^H through char_matrix_vjp (diff.py:22-60), the terms
// `kinds` asks for (0 otherwise), then vbar <- M_k^H vbar.  n0sq_sin2 = n0^2 sin^2 theta0.
__device__ __forceinline__ TfGrad tf_reverse_step(const TfLayer& L, double2 sb, double2 cb, double2 w0, double2 w1,
                                                  int kinds, double2 n0sq_sin2, double wvl, int pol, double2& vb0,
                                                  double2& vb1) {
    const double2 m00 = cmulc(vb0, w0), m01 = cmulc(vb0, w1), m10 = cmulc(vb1, w0), m11 = cmulc(vb1, w1);
    // c = sum conj(dM) * Mbar
    const double2 ieta = tf_div(make_double2(1.0, 0.0), L.eta);
    const double2 icb = make_double2(cb.y, -cb.x);                 // -i cos b
    const double2 dB01 = cmul(icb, ieta), dB10 = cmul(icb, L.eta);
    const double2 cbeta = csub(cadd(cmulc(m01, dB01), cmulc(m10, dB10)), cadd(cmulc(m00, sb), cmulc(m11, sb)));
    const double2 isb = make_double2(-sb.y, sb.x);                 // i sin b
    const double2 dE01 = cmul(isb, cmul(ieta, ieta)), dE10 = make_double2(-isb.x, -isb.y);
    const double2 ceta = cadd(cmulc(m01, dE01), cmulc(m10, dE10));
    TfGrad g{0.0, 0.0};
    if (kinds & PB_TF_GRAD_THICKNESS) {
        // dbeta/dd = 2 pi n cos / wvl (diff.py:110, 307)
        const double2 dbdd = cscale(cmul(L.n, L.cost), 2.0 * M_PI / wvl);
        g.th = cmulc(dbdd, cbeta).x;
    }
    if (kinds & PB_TF_GRAD_INDEX) {
        // diff.py:328-339: dcos/dn = n0^2 sin0^2 / (n^3 cos)
        const double2 n2 = cmul(L.n, L.n);
        const double2 dcdn = tf_div(n0sq_sin2, cmul(cmul(n2, L.n), L.cost));
        const double2 ndc = cmul(L.n, dcdn);
        const double2 dbdn = cscale(cadd(L.cost, ndc), 2.0 * M_PI * L.d / wvl);
        const double2 dedn = pol == PB_TF_POL_P
            ? csub(tf_div(make_double2(1.0, 0.0), L.cost), tf_div(ndc, cmul(L.cost, L.cost)))
            : cadd(L.cost, ndc);
        g.ix = cmulc(dbdn, cbeta).x + cmulc(dedn, ceta).x;
    }
    tf_apply_adjoint(sb, cb, L.eta, vb0, vb1);
    return g;
}

// lane 0 adds the warp's sum of v to its own slot p, written on the warp's first visit: no atomics, a fixed order
__device__ __forceinline__ void tf_warp_add(double v, bool act, int lane, bool first, double* p) {
    v = warp_reduce(act ? v : 0.0, OpAdd{});
    if (lane == 0) *p = first ? v : *p + v;
}

// One warp-uniform pass per 32 samples.  The sweeping kernels sum each contribution over the warp into the warp's
// slot of a partial row (row * W + warp), and tf_reduce_kernel sums the rows.  The rows are only those asked for:
// the thickness rows, then the index rows, N each.
__global__ void __launch_bounds__(PB_TF_THREADS, 2) stack_grad_kernel(const TfOps op, long long count, int kinds,
                                                                    const double2* __restrict__ E, const double2* __restrict__ H,
                                                                    const double* __restrict__ dR, const double* __restrict__ dT,
                                                                    const double* __restrict__ dA, const double* __restrict__ dEsq,
                                                                    double* __restrict__ partial) {
    const int N = op.nlayers;
    const long long W = (long long)gridDim.x * (blockDim.x / 32);
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const bool fseed = dA || dEsq;
    const int ix0 = kinds & PB_TF_GRAD_THICKNESS ? N : 0;           // the first index row
    for (long long base = warp * 32; base < count; base += W * 32) {
        const bool first = base == warp * 32;
        const bool act = base + lane < count;
        const long long i = act ? base + lane : count - 1;
        const TfSample s = tf_sample(op, i);
        const double2 eta_sub = tf_eta_sub(s, op.pol);
        const double2 eta0 = tf_admittance(s.n0, make_double2(s.cos0, 0.0), op.pol);
        const double inv_re0 = 1.0 / eta0.x;
        const double2 t = E[(long long)N * count + i];                  // f_N = t [1, eta_sub]
        const double2 inv_t = tf_div(make_double2(1.0, 0.0), t);
        const double2 B = cmul(E[i], inv_t), C = cmul(H[i], inv_t);
        const double2 eb = cmul(eta0, B);
        const double2 den = cadd(eb, C);
        const double2 r = tf_div(csub(eb, C), den);
        // amplitude cotangents (diff.py:191-201)
        double2 rb = make_double2(0.0, 0.0), tb = make_double2(0.0, 0.0);
        if (dR) rb = cscale(r, 2.0 * dR[i]);
        if (dT) tb = cscale(t, 2.0 * (eta_sub.x * inv_re0) * dT[i]);
        // f_k = t v_k: tbar += sum_k v_k^H fbar_k
        if (fseed) {
            for (int k = 0; k <= N; ++k) {
                const long long ok = (long long)k * count + i;
                const double2 e = E[ok], hh = H[ok];
                double2 eb2, hb2;
                tf_field_bar(dA, dEsq, N, count, i, k, inv_re0, e, hh, eb2, hb2);
                tb = cadd(tb, cadd(cmulc(eb2, cmul(e, inv_t)), cmulc(hb2, cmul(hh, inv_t))));
            }
        }
        double2 vb0, vb1;
        tf_seed(r, t, eta0, den, rb, tb, vb0, vb1);
        const double2 ct = cconj(t);
        if (fseed) {
            double2 eb2, hb2;
            tf_field_bar(dA, dEsq, N, count, i, 0, inv_re0, E[i], H[i], eb2, hb2);
            vb0 = cadd(vb0, cmul(ct, eb2));
            vb1 = cadd(vb1, cmul(ct, hb2));
        }
        const double2 n0sq_sin2 = cscale(cmul(s.n0, s.n0), s.sin0 * s.sin0);
        for (int k = 0; k < N; ++k) {
            const TfLayer L = tf_layer(op, s, k);
            double2 sb, cb;
            tf_sincos(L.beta, &sb, &cb);
            const long long o1 = (long long)(k + 1) * count + i;
            const double2 e1 = E[o1], h1 = H[o1];
            const TfGrad g = tf_reverse_step(L, sb, cb, cmul(e1, inv_t), cmul(h1, inv_t), kinds, n0sq_sin2, s.wvl,
                                             op.pol, vb0, vb1);
            // vbar_{k+1} += conj(t) fbar_{k+1}
            if (fseed) {
                double2 eb2, hb2;
                tf_field_bar(dA, dEsq, N, count, i, k + 1, inv_re0, e1, h1, eb2, hb2);
                vb0 = cadd(vb0, cmul(ct, eb2));
                vb1 = cadd(vb1, cmul(ct, hb2));
            }
            if (kinds & PB_TF_GRAD_THICKNESS) tf_warp_add(g.th, act, lane, first, partial + (long long)k * W + warp);
            if (kinds & PB_TF_GRAD_INDEX) tf_warp_add(g.ix, act, lane, first, partial + (long long)(ix0 + k) * W + warp);
        }
    }
}

// dst[row] = sum over the first nw warps of partial row `row`, in a fixed order, one block per row; with value, the last
// row goes to *value in fp64 instead.  With accumulate the sums are added to what dst and value hold.
template <typename R>
__global__ void __launch_bounds__(PB_TF_THREADS) tf_reduce_kernel(const double* __restrict__ partial, long long W,
                                                                   long long nw, int accumulate, R* __restrict__ dst,
                                                                   double* __restrict__ value) {
    __shared__ double sh[PB_TF_THREADS];
    const int row = blockIdx.x;
    const double* p = partial + (long long)row * W;
    double a = 0.0;
    for (long long w = threadIdx.x; w < nw; w += blockDim.x) a += p[w];
    a = tree_sum<PB_TF_THREADS>(a, sh);
    if (threadIdx.x) return;
    if (value && row == gridDim.x - 1) *value = accumulate ? *value + a : a;
    else dst[row] = accumulate ? dst[row] + (R)a : (R)a;
}

// stack.py:252-301: searchsorted(Z, z, 'right') - 1 clipped to [0, N - 1], then the partial layer below z applied to
// the field at the layer's substrate-side boundary
template <typename R>
__global__ void __launch_bounds__(PB_TF_THREADS) field_at_depth_kernel(const double* __restrict__ z, long long nz,
                                                                        const double* __restrict__ zb, int N,
                                                                        const double2* __restrict__ nl, double2 n0,
                                                                        double wvl, double sin0, int pol,
                                                                        const double2* __restrict__ Eb,
                                                                        const double2* __restrict__ Hb,
                                                                        cplx<R>* __restrict__ Eo, cplx<R>* __restrict__ Ho) {
    PB_GRID_STRIDE(i, nz) {
        const double zi = z[i];
        int lo = 0, hi = N + 1;                       // first boundary with zb > zi
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (zb[mid] <= zi) lo = mid + 1;
            else hi = mid;
        }
        const int li = min(max(lo - 1, 0), N - 1);
        const double2 n = nl[li];
        const double2 cost = tf_cos_snell(n0, n, sin0);
        const double2 eta = tf_admittance(n, cost, pol);
        const double2 beta = cscale(cmul(cscale(n, 2.0 * M_PI * (zb[li + 1] - zi)), cost), 1.0 / wvl);
        double2 sb, cb;
        tf_sincos(beta, &sb, &cb);
        double2 v0 = Eb[li + 1], v1 = Hb[li + 1];
        tf_apply(sb, cb, eta, v0, v1);
        Eo[i] = mk<R>((R)v0.x, (R)v0.y);
        Ho[i] = mk<R>((R)v1.x, (R)v1.y);
    }
}


// ---- coating design (prysm/x/coatings merit.py, needle.py) ------------------------------------------------------
// One thread per sample runs, per polarisation, the forward sweep into a stage in the handle's scratch (v_k of every
// boundary, unscaled), forms q and its seed in registers, and runs the reverse sweep of stack_grad_kernel with the
// seed applied where the term puts it: no field or seed array goes through HBM.  The warp partials are summed in a
// fixed order by a second launch.

// both polarisations in one thread take about 164 registers: 3 blocks of 128 threads per SM, 12 warps, against 8 for
// 256-thread blocks at that size
constexpr int cm_threads(int npol) { return npol == 2 ? 128 : PB_TF_THREADS; }

struct CmTerm {
    int quantity, npol, b0, b1, nb;
    const int* blist;              // nb boundaries, then nb "last listing" flags
    const double* tgt;
    const double* wgt;
    long long st_tgt[PB_TF_DIMS], st_wgt[PB_TF_DIMS];
    long long cpad;                // stage pitch: count rounded up to whole warps
};

struct NeedleStrides { long long st[PB_TF_DIMS]; };

// offset of sample i in a per-sample operand of strides st.  Target, weight and the needle index take this
// decomposition of their own rather than travelling in TfOps through tf_sample's: that way the needle kernel keeps 118
// registers, against 122 when their offsets come from tf_sample (and 120 with the needle index in CmTerm).
__device__ inline long long cm_offset(const TfOps& op, const long long* st, long long i) {
    long long off = 0;
    for (int j = PB_TF_DIMS - 1; j >= 0; --j) {
        off += (i % op.shape[j]) * st[j];
        i /= op.shape[j];
    }
    return off;
}

// forward sweep of one polarisation into the stage V0 / V1 (boundary k at row k); returns r, t and the admittances
struct CmFwd { double2 r, t, eta0; double t2; };

// r and t from (B, C) = v_0; the reverse sweep recomputes them from the stage, with the same operations
__device__ inline CmFwd cm_rt(const TfSample& s, int pol, double2 v0, double2 v1) {
    CmFwd f;
    f.eta0 = tf_admittance(s.n0, make_double2(s.cos0, 0.0), pol);
    const double2 eb = cmul(f.eta0, v0);
    const double2 den = cadd(eb, v1);
    f.r = tf_div(csub(eb, v1), den);
    f.t = tf_div(cscale(f.eta0, 2.0), den);
    f.t2 = tf_abs2(f.t);
    return f;
}

__device__ inline CmFwd cm_forward(const TfOps& op, const TfSample& s, int pol, double2* V0, double2* V1,
                                   long long pitch, long long is) {
    double2 v0 = make_double2(1.0, 0.0), v1 = tf_eta_sub(s, pol);
    tf_sweep(op, s, pol, v0, v1, [&](int k, double2 e, double2 h) {
        V0[(long long)k * pitch + is] = e;
        V1[(long long)k * pitch + is] = h;
    });
    return cm_rt(s, pol, v0, v1);
}

// q of one polarisation; for the peak, *arg is the list position of the first maximum (NaN counts as the maximum)
__device__ inline double cm_quantity(const CmTerm& tm, const TfSample& s, int pol, const CmFwd& f, const double2* V0,
                                     const double2* V1, long long pitch, long long is, int* arg) {
    switch (tm.quantity) {
    case PB_CM_Q_R: return tf_abs2(f.r);
    case PB_CM_Q_T: return tf_eta_sub(s, pol).x / f.eta0.x * f.t2;
    case PB_CM_Q_ABS: {
        const long long o = (long long)tm.b0 * pitch + is;
        const double g0 = cmulc(V0[o], V1[o]).x, g1 = cmulc(V0[o + pitch], V1[o + pitch]).x;
        return f.t2 * g0 / f.eta0.x - f.t2 * g1 / f.eta0.x;
    }
    case PB_CM_Q_ESQ: return f.t2 * tf_abs2(V0[(long long)tm.b0 * pitch + is]);
    case PB_CM_Q_PEAK: {
        double best = 0.0;
        for (int j = 0; j < tm.nb; ++j) {
            const double e = f.t2 * tf_abs2(V0[(long long)tm.blist[j] * pitch + is]);
            if (j == 0 || (!isnan(best) && (e > best || isnan(e)))) { best = e; *arg = j; }
        }
        return best;
    }
    default:
        return 0.5 * (f.t2 * tf_abs2(V0[(long long)tm.b0 * pitch + is]) + f.t2 * tf_abs2(V0[(long long)tm.b1 * pitch + is]));
    }
}

// the field seed of boundary k (diff.py:204-224): fbar = (H cf + 2 ce E, E cf) with E = t v0, H = t v1
struct CmSeed { int ka, kb; double cfa, cea, cfb, ceb; };

__device__ inline void cm_field_bar(const CmSeed& sd, int k, double2 E, double2 H, double2& Eb, double2& Hb) {
    double cf = 0.0, ce = 0.0;
    if (k == sd.ka) { cf += sd.cfa; ce += sd.cea; }
    if (k == sd.kb) { cf += sd.cfb; ce += sd.ceb; }
    tf_field_cot(cf, ce, E, H, Eb, Hb);
}

// the reverse-sweep start of one polarisation: vbar_0 from the amplitude and field seeds of dq, and the field seeds
__device__ inline void cm_seed(const CmTerm& tm, const TfSample& s, int pol, const CmFwd& f, double dq, int arg,
                               const double2* V0, const double2* V1, long long pitch, long long is, CmSeed& sd,
                               double2& vb0, double2& vb1) {
    const double inv_re0 = 1.0 / f.eta0.x;
    sd.ka = sd.kb = -1;
    sd.cfa = sd.cea = sd.cfb = sd.ceb = 0.0;
    double2 rb = make_double2(0.0, 0.0), tb = make_double2(0.0, 0.0);
    if (tm.quantity == PB_CM_Q_R) rb = cscale(f.r, 2.0 * dq);
    else if (tm.quantity == PB_CM_Q_T) tb = cscale(f.t, 2.0 * (tf_eta_sub(s, pol).x * inv_re0) * dq);
    else if (tm.quantity == PB_CM_Q_ABS) {
        sd.ka = tm.b0; sd.cfa = dq * inv_re0;
        sd.kb = tm.b0 + 1; sd.cfb = -dq * inv_re0;
    } else if (tm.quantity == PB_CM_Q_ESQ) {
        sd.ka = tm.b0; sd.cea = dq;
    } else if (tm.quantity == PB_CM_Q_PEAK) {
        if (tm.blist[tm.nb + arg]) { sd.ka = tm.blist[arg]; sd.cea = dq; }
    } else {
        sd.ka = tm.b0; sd.cea = 0.5 * dq;
        sd.kb = tm.b1; sd.ceb = 0.5 * dq;
    }
    // f_k = t v_k: tbar += v_k^H fbar_k at the seeded boundaries
    for (int w = 0; w < 2; ++w) {
        const int k = w == 0 ? sd.ka : (sd.kb == sd.ka ? -1 : sd.kb);
        if (k < 0) continue;
        const double2 v0 = V0[(long long)k * pitch + is], v1 = V1[(long long)k * pitch + is];
        double2 eb2, hb2;
        cm_field_bar(sd, k, cmul(f.t, v0), cmul(f.t, v1), eb2, hb2);
        tb = cadd(tb, cadd(cmulc(eb2, v0), cmulc(hb2, v1)));
    }
    tf_seed(f.r, f.t, f.eta0, cadd(cmul(f.eta0, V0[is]), V1[is]), rb, tb, vb0, vb1);
    if (sd.ka == 0 || sd.kb == 0) {
        double2 eb2, hb2;
        cm_field_bar(sd, 0, cmul(f.t, V0[is]), cmul(f.t, V1[is]), eb2, hb2);
        const double2 ct = cconj(f.t);
        vb0 = cadd(vb0, cmul(ct, eb2));
        vb1 = cadd(vb1, cmul(ct, hb2));
    }
}

// a / x for a real x, as numpy divides a complex array by a real one
__device__ inline double2 cm_over(double2 a, double x) { return make_double2(a.x / x, a.y / x); }

// partial rows: the gradient rows, then the value row
template <int NPOL>
__global__ void __launch_bounds__(cm_threads(NPOL), NPOL == 2 ? 3 : 2) coating_merit_kernel(const TfOps op, const CmTerm tm, long long count,
                                                                       int flags, double2* __restrict__ V0,
                                                                       double2* __restrict__ V1, double* __restrict__ partial,
                                                                       void* __restrict__ resid, bool resid_f32) {
    const int N = op.nlayers;
    const long long W = (long long)gridDim.x * (blockDim.x / 32);
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const int kinds = (flags >> 2) & 3;
    const int ix0 = kinds & PB_TF_GRAD_THICKNESS ? N : 0;           // the first index row
    const long long vrow = ix0 + (kinds & PB_TF_GRAD_INDEX ? N : 0);
    const long long pitch = tm.cpad;
    for (long long base = warp * 32; base < count; base += W * 32) {
        const bool first = base == warp * 32;
        const bool act = base + lane < count;
        const long long i = act ? base + lane : count - 1;
        const long long is = base + lane;                      // this lane's own stage column
        const TfSample s = tf_sample(op, i);
        const double tg = tm.tgt[cm_offset(op, tm.st_tgt, i)], w = tm.wgt[cm_offset(op, tm.st_wgt, i)];
        // the peak's list position per polarisation, 16 bits each (loops that are not unrolled keep it in a register)
        unsigned args = 0;
        double q = 0.0;
#pragma unroll 1
        for (int p = 0; p < NPOL; ++p) {
            const int pol = NPOL == 2 ? p : op.pol;
            double2* v0 = V0 + (long long)p * (N + 1) * pitch;
            double2* v1 = V1 + (long long)p * (N + 1) * pitch;
            const CmFwd f = cm_forward(op, s, pol, v0, v1, pitch, is);
            int a = 0;
            q += cm_quantity(tm, s, pol, f, v0, v1, pitch, is, &a);
            args |= (unsigned)a << (16 * p);
        }
        q = q / NPOL;
        const double d = q - tg;
        if (flags & PB_CM_OUT_RESIDUALS && act) {
            const double res = sqrt(w) * d;
            if (resid_f32) ((float*)resid)[i] = (float)res;
            else ((double*)resid)[i] = res;
        }
        if (flags & PB_CM_OUT_VALUE) tf_warp_add(w * (d * d), act, lane, first, partial + vrow * W + warp);
        if (!kinds) continue;
        const double dq = 2.0 * w * d / NPOL;
#pragma unroll 1
        for (int p = 0; p < NPOL; ++p) {
            const int pol = NPOL == 2 ? p : op.pol;
            const double2* v0 = V0 + (long long)p * (N + 1) * pitch;
            const double2* v1 = V1 + (long long)p * (N + 1) * pitch;
            const CmFwd f = cm_rt(s, pol, v0[is], v1[is]);
            CmSeed sd;
            double2 vb0, vb1;
            cm_seed(tm, s, pol, f, dq, (int)(args >> (16 * p) & 0xffffu), v0, v1, pitch, is, sd, vb0, vb1);
            const double2 ct = cconj(f.t);
            const double2 n0sq_sin2 = cscale(cmul(s.n0, s.n0), s.sin0 * s.sin0);
            for (int k = 0; k < N; ++k) {
                const TfLayer L = tf_layer(op, s, k, pol);
                double2 sb, cb;
                tf_sincos(L.beta, &sb, &cb);
                const long long o1 = (long long)(k + 1) * pitch + is;
                const double2 w0 = v0[o1], w1 = v1[o1];                         // v_{k+1}
                const TfGrad g = tf_reverse_step(L, sb, cb, w0, w1, kinds, n0sq_sin2, s.wvl, pol, vb0, vb1);
                // vbar_{k+1} += conj(t) fbar_{k+1}
                if (k + 1 == sd.ka || k + 1 == sd.kb) {
                    double2 eb2, hb2;
                    cm_field_bar(sd, k + 1, cmul(f.t, w0), cmul(f.t, w1), eb2, hb2);
                    vb0 = cadd(vb0, cmul(ct, eb2));
                    vb1 = cadd(vb1, cmul(ct, hb2));
                }
                if (kinds & PB_TF_GRAD_THICKNESS)
                    tf_warp_add(g.th, act, lane, first && p == 0, partial + (long long)k * W + warp);
                if (kinds & PB_TF_GRAD_INDEX)
                    tf_warp_add(g.ix, act, lane, first && p == 0, partial + (long long)(ix0 + k) * W + warp);
            }
        }
    }
}

// P(z) of an R or T term (needle.py:18-91).  The assembled-matrix cotangent of diff.py's _rt_assembly_cotangent is
// c_M = u w^H with u = (Bbar, Cbar) and w = (1, eta_sub), so Re tr(c_M^H L_j X R_{j+1}) = Re(vbar_j^H X v_{j+1}) with
// X = M_top G M_bot: each (sample, depth) costs two characteristic matrices applied to a 2-vector.
template <int NPOL>
__global__ void __launch_bounds__(cm_threads(NPOL), NPOL == 2 ? 3 : 2) needle_kernel(const TfOps op, const CmTerm tm, const double2* __restrict__ nn,
                                                                const NeedleStrides st_nn, long long count,
                                                                const double* __restrict__ zpart, long long nz,
                                                                const int* __restrict__ zlist,
                                                                double2* __restrict__ V0, double2* __restrict__ V1,
                                                                double* __restrict__ partial) {
    const int N = op.nlayers;
    const long long W = (long long)gridDim.x * (blockDim.x / 32);
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    const long long pitch = tm.cpad;
    const int* order = zlist + N + 1;
    for (long long base = warp * 32; base < count; base += W * 32) {
        const bool first = base == warp * 32;
        const bool act = base + lane < count;
        const long long i = act ? base + lane : count - 1;
        const long long is = base + lane;
        const TfSample s = tf_sample(op, i);
        const double tg = tm.tgt[cm_offset(op, tm.st_tgt, i)], w = tm.wgt[cm_offset(op, tm.st_wgt, i)];
        const double2 n = nn[cm_offset(op, st_nn.st, i)];
        double q = 0.0;
        int arg = 0;
#pragma unroll 1
        for (int p = 0; p < NPOL; ++p) {
            const int pol = NPOL == 2 ? p : op.pol;
            const CmFwd f = cm_forward(op, s, pol, V0 + (long long)p * (N + 1) * pitch,
                                       V1 + (long long)p * (N + 1) * pitch, pitch, is);
            q += cm_quantity(tm, s, pol, f, nullptr, nullptr, pitch, is, &arg);
        }
        q = q / NPOL;
        const double dq = 2.0 * w * (q - tg) / NPOL;
        const double2 cosn = tf_cos_snell(s.n0, n, s.sin0);
#pragma unroll 1
        for (int p = 0; p < NPOL; ++p) {
            const int pol = NPOL == 2 ? p : op.pol;
            const double2* v0 = V0 + (long long)p * (N + 1) * pitch;
            const double2* v1 = V1 + (long long)p * (N + 1) * pitch;
            CmSeed sd;
            double2 vb0, vb1;
            cm_seed(tm, s, pol, cm_rt(s, pol, v0[is], v1[is]), dq, 0, v0, v1, pitch, is, sd, vb0, vb1);
            // the needle generator G = dbeta/dd [[0, -i / eta_n], [-i eta_n, 0]]
            const double2 eta_n = tf_admittance(n, cosn, pol);
            const double2 gdn = cm_over(cmul(cscale(n, 2.0 * M_PI), cosn), s.wvl);
            const double2 g01 = cmul(gdn, tf_div(make_double2(0.0, -1.0), eta_n));
            const double2 g10 = cmul(gdn, cmul(make_double2(0.0, -1.0), eta_n));
            for (int k = 0; k < N; ++k) {
                const TfLayer L = tf_layer(op, s, k, pol);
                const long long o1 = (long long)(k + 1) * pitch + is;
                const double2 w0 = v0[o1], w1 = v1[o1];                         // v_{k+1}
                const double2 dbdd = cm_over(cmul(cscale(L.n, 2.0 * M_PI), L.cost), s.wvl);
                for (int j = zlist[k]; j < zlist[k + 1]; ++j) {
                    const int zi = order[j];
                    // M_bot (the part of layer k below z), G, then M_top
                    double2 x0 = w0, x1 = w1, sb, cb;
                    tf_sincos(cscale(dbdd, zpart[nz + zi]), &sb, &cb);
                    tf_apply(sb, cb, L.eta, x0, x1);
                    const double2 y0 = cmul(g01, x1), y1 = cmul(g10, x0);
                    x0 = y0; x1 = y1;
                    tf_sincos(cscale(dbdd, zpart[zi]), &sb, &cb);
                    tf_apply(sb, cb, L.eta, x0, x1);
                    tf_warp_add(cmulc(x0, vb0).x + cmulc(x1, vb1).x, act, lane, first && p == 0,
                                partial + (long long)zi * W + warp);
                }
                double2 sb, cb;
                tf_sincos(L.beta, &sb, &cb);
                tf_apply_adjoint(sb, cb, L.eta, vb0, vb1);
            }
        }
    }
}

// ---- optical monitoring (prysm/x/coatings monitoring.py) --------------------------------------------------------
// One CTA per as-built run deposits the layers from the substrate up: v = [1, eta_sub], and for k = N - 1, ..., 0 the
// threads stride over the thickness grid d_j, each forming the monitor signal of M_k(d_j) v; the CTA picks the
// termination thickness by the reference's rule with fixed-order block reductions and every thread advances
// v <- M_k(d_real) v with the same operations, so v stays uniform over the CTA.  The decisions read the grid in tiles of
// PB_MON_THREADS samples that overlap by two, so a thread sees samples i, i + 1 and i + 2 without a second evaluation.
#define PB_MON_THREADS 128
constexpr int MON_STEP = PB_MON_THREADS - 2;

template <typename T> __device__ inline T mon_sign(T x) { return x > T(0) ? T(1) : x < T(0) ? T(-1) : x == T(0) ? T(0) : x; }

// a distance as an argmin key: NaN counts as the smallest, as numpy's argmin takes the first NaN
__device__ inline double mon_key(double x) { return isnan(x) ? -1.0 : x; }

// numpy.linspace(start, stop, n)[i]: i step + start, step = (stop - start) / (n - 1), (i / (n - 1)) (stop - start) when
// the step is 0, i (stop - start) + start for n = 1; the last of n > 1 points is stop
__device__ inline double mon_grid(long long i, long long n, double start, double stop) {
    if (n > 1 && i == n - 1) return stop;
    const double delta = __dsub_rn(stop, start);
    if (n > 1) {
        const double div = (double)(n - 1), step = __ddiv_rn(delta, div);
        return __dadd_rn(step != 0.0 ? __dmul_rn((double)i, step) : __dmul_rn(__ddiv_rn((double)i, div), delta), start);
    }
    return __dadd_rn(__dmul_rn((double)i, delta), start);
}

// one tile of the grid: sample base + t of thread t in sd / ss; thread t owns sample base + t for t < MON_STEP
template <typename T, typename Pt>
__device__ inline void mon_tile(long long base, long long n, T* sd, T* ss, Pt& pt) {
    const long long i = base + threadIdx.x;
    __syncthreads();                 // the previous tile may still be read
    if (i < n) pt(i, sd[threadIdx.x], ss[threadIdx.x]);
    __syncthreads();
}

// level_cut (monitoring.py:111-146) of the n samples pt(i, d_i, sig_i) for one CTA: s = sig - level, a crossing between
// i and i + 1 wherever sign(s_i) != sign(s_i+1), at d_i + frac (d_i+1 - d_i) with frac = -s_i / (s_i+1 - s_i) (0 when
// they are equal); the crossing nearest target, the first on a tie; with none, the d of the first minimum of |s|.
// Arithmetic in T, one rounding per operation as numpy; n >= 1.  Every thread gets the result.
template <typename T, typename Pt>
__device__ T mon_level_cut(long long n, T level, T target, Pt&& pt) {
    __shared__ T sd[PB_MON_THREADS], ss[PB_MON_THREADS];
    __shared__ T res;
    const int t = threadIdx.x;
    double kc = INFINITY, kz = INFINITY;               // the thread's best keys: crossing, |s|
    long long ic = LLONG_MAX, iz = LLONG_MAX;
    T vc = T(0), vz = T(0);
    for (long long base = 0; base < n; base += MON_STEP) {
        mon_tile<T>(base, n, sd, ss, pt);
        const long long i = base + t;
        if (t >= MON_STEP || i >= n) continue;
        const T s0 = ss[t] - level, d0 = sd[t];
        const double z = mon_key((double)(s0 < T(0) ? -s0 : s0));
        if (iz == LLONG_MAX || z < kz) { kz = z; iz = i; vz = d0; }
        if (i + 1 >= n) continue;
        const T s1 = ss[t + 1] - level, d1 = sd[t + 1];
        if (mon_sign(s0) == mon_sign(s1)) continue;
        const T frac = s1 == s0 ? T(0) : -s0 / (s1 - s0);
        T c;
        if constexpr (sizeof(T) == 8) c = __dadd_rn(d0, __dmul_rn(frac, __dsub_rn(d1, d0)));
        else c = __fadd_rn(d0, __fmul_rn(frac, __fsub_rn(d1, d0)));
        const T dist = c - target;
        const double k = mon_key((double)(dist < T(0) ? -dist : dist));
        if (ic == LLONG_MAX || k < kc) { kc = k; ic = i; vc = c; }
    }
    // the smallest key, then the first index holding it (a thread without a candidate holds no index)
    double key[2] = {kc, kz};
    block_reduce<PB_MON_THREADS>(key, OpMin{});
    double idx[2] = {ic != LLONG_MAX && kc == key[0] ? (double)ic : INFINITY,
                     iz != LLONG_MAX && kz == key[1] ? (double)iz : INFINITY};
    block_reduce<PB_MON_THREADS>(idx, OpMin{});
    const bool crossed = idx[0] != INFINITY;
    if (crossed ? (double)ic == idx[0] : (double)iz == idx[1]) res = crossed ? vc : vz;
    __syncthreads();
    return res;
}

// turning_points (monitoring.py:88-108) of the n samples pt(i, d_i, sig_i) for one CTA: slope_i = sign(sig_i+1 - sig_i),
// a turning point at i + 1 wherever slope_i != slope_i+1, in T.  With out, every one is written to out in order and
// the count returned; otherwise the scan stops at the m-th (0-based), whose d goes to *found (every thread), and the
// count returned is m + 1, or the whole count (< m + 1) when there are fewer.
template <typename T, typename Pt>
__device__ long long mon_turning(long long n, long long m, T* out, T* found, Pt&& pt) {
    __shared__ T sd[PB_MON_THREADS], ss[PB_MON_THREADS];
    __shared__ int wc[PB_MON_THREADS / 32];
    __shared__ T res;
    const int t = threadIdx.x, lane = t & 31, w = t >> 5;
    long long count = 0;
    for (long long base = 0; base < n; base += MON_STEP) {
        mon_tile<T>(base, n, sd, ss, pt);
        const long long i = base + t;
        bool flag = false;
        if (t < MON_STEP && i + 2 < n)
            flag = mon_sign(ss[t + 1] - ss[t]) != mon_sign(ss[t + 2] - ss[t + 1]);
        const unsigned b = __ballot_sync(0xffffffffu, flag);
        if (lane == 0) wc[w] = __popc(b);
        __syncthreads();
        long long pos = count + __popc(b & ((1u << lane) - 1u));
        for (int j = 0; j < PB_MON_THREADS / 32; ++j) {
            if (j < w) pos += wc[j];
            count += wc[j];
        }
        if (flag) {
            if (out) out[pos] = sd[t + 1];
            else if (pos == m) res = sd[t + 1];
        }
        if (!out && count > m) {
            __syncthreads();
            *found = res;
            return m + 1;
        }
    }
    return count;
}

// the monitor signal of (B, C) = v (_signal_curve, monitoring.py:15-45): R = |r|^2, or T = Re eta_sub / Re eta0 |t|^2
__device__ inline double mon_signal(const TfSample& s, int pol, int mode, double2 eta_sub, double2 v0, double2 v1) {
    const CmFwd f = cm_rt(s, pol, v0, v1);
    return mode == PB_MON_R ? tf_abs2(f.r) : eta_sub.x / f.eta0.x * f.t2;
}

struct MonArgs {
    const double* err;             // (runs, N) signal (level) or thickness (turning) errors, or NULL
    const double* levels;          // (ncand, N) cutoff levels (level)
    long long per_cand, npts;
    double start, max_factor;
    int strategy, mode, turning_index;
};

// simulate_run (monitoring.py:168-233) of run blockIdx.x, at candidate blockIdx.x / per_cand: asbuilt (runs, N)
template <typename R>
__global__ void __launch_bounds__(PB_MON_THREADS) monitor_runs_kernel(const TfOps op, const MonArgs a,
                                                                      R* __restrict__ asbuilt) {
    const long long run = blockIdx.x;
    const long long c = run / a.per_cand;
    const int N = op.nlayers, pol = op.pol;
    const TfSample s = tf_sample(op, c);
    const double2 eta_sub = tf_eta_sub(s, pol);
    double2 v0 = make_double2(1.0, 0.0), v1 = eta_sub;
    for (int k = N - 1; k >= 0; --k) {
        const TfLayer L = tf_layer(op, s, k, pol);
        const double stop = __dmul_rn(a.max_factor, L.d);
        auto pt = [&](long long j, double& d, double& sig) {
            d = mon_grid(j, a.npts, a.start, stop);
            double2 sb, cb, w0 = v0, w1 = v1;
            tf_sincos(tf_beta(L.n, L.cost, d, s.wvl), &sb, &cb);
            tf_apply(sb, cb, L.eta, w0, w1);
            sig = mon_signal(s, pol, a.mode, eta_sub, w0, w1);
        };
        const double* e = a.err ? a.err + run * N + k : nullptr;
        double dr;
        if (a.strategy == PB_MON_TURNING) {
            double tp = 0.0;
            const long long m = a.turning_index - 1;
            dr = mon_turning<double>(a.npts, m, nullptr, &tp, pt) > m ? tp : L.d;
            if (e) dr = __dadd_rn(dr, *e);
        } else {
            double lv = a.levels[c * N + k];
            if (e) lv = __dadd_rn(lv, *e);
            dr = mon_level_cut<double>(a.npts, lv, L.d, pt);
        }
        dr = 0.0 > dr ? 0.0 : dr;                    // Python's max(d_real, 0.0)
        if (threadIdx.x == 0) asbuilt[run * N + k] = (R)dr;
        double2 sb, cb;
        tf_sincos(tf_beta(L.n, L.cost, dr, s.wvl), &sb, &cb);
        tf_apply(sb, cb, L.eta, v0, v1);
    }
}

// level_cut or turning_points of a given trace (d, sig of n samples) in one CTA: out[0] the cut, or out[0, count) the
// turning points and *count their number
template <typename T>
__global__ void __launch_bounds__(PB_MON_THREADS) monitor_cut_kernel(int strategy, const T* __restrict__ d,
                                                                     const T* __restrict__ sig, long long n, T level,
                                                                     T target, T* __restrict__ out,
                                                                     long long* __restrict__ count) {
    auto pt = [&](long long i, T& di, T& si) { di = d[i]; si = sig[i]; };
    if (strategy == PB_MON_TURNING) {
        const long long c = mon_turning<T>(n, 0, out, nullptr, pt);
        if (threadIdx.x == 0) *count = c;
    } else {
        const T v = mon_level_cut<T>(n, level, target, pt);
        if (threadIdx.x == 0) out[0] = v;
    }
}

// monitoring_error_sensitivity's J[c, w, k] = (Rr[c (N + 1) + 1 + k, w] - Rr[c (N + 1), w]) / eps of the realized
// reflectance Rr (runs, W), and choose_monitor_wavelength's score[c] = sqrt(sum J[c]^2) by the grid fold (DESIGN.md
// §4.4); grid row c
template <typename R>
__global__ void __launch_bounds__(256) monitor_jacobian_kernel(const double* __restrict__ Rr, int N, long long W,
                                                               double eps, R* __restrict__ J, R* __restrict__ score,
                                                               double* __restrict__ part, unsigned* __restrict__ counters) {
    const long long c = blockIdx.y, cnt = W * N;
    const double* R0 = Rr + c * (N + 1) * W;
    double acc = 0.0;
    PB_GRID_STRIDE(i, cnt) {
        const long long w = i / N, k = i % N;
        const double j = (R0[(k + 1) * W + w] - R0[w]) / eps;
        if (J) J[c * cnt + i] = (R)j;
        acc += j * j;
    }
    acc = block_reduce<256>(acc, OpAdd{});
    if (threadIdx.x == 0) part[blockIdx.y * gridDim.x + blockIdx.x] = acc;
    if (!arrive_last(counters)) return;
    const double ss = fold_partials<256, 1>(part, 0, OpAdd{}, 0.0);
    if (threadIdx.x == 0 && score) score[c] = (R)sqrt(ss);
}

// the n values of an outermost-first array of the C ABI right-aligned to PB_TF_DIMS dims, `fill` in front: the
// calculation shape (fill 1) or an operand's strides (fill 0)
static void tf_align(const long long* src, int n, long long fill, long long* dst) {
    for (int j = 0; j < PB_TF_DIMS; ++j) dst[j] = j >= PB_TF_DIMS - n ? src[j - (PB_TF_DIMS - n)] : fill;
}

static int tf_ops(Handle* h, int pol, int nlayers, int ndim, const long long* shape, const long long* strides,
                  const void* const* in, TfOps& op, long long& count) {
    if (pol != PB_TF_POL_S && pol != PB_TF_POL_P) return fail(h, PB_ERR_INVALID, "thinfilm: pol must be PB_TF_POL_S or P");
    if (nlayers < 0) return fail(h, PB_ERR_INVALID, "thinfilm: nlayers must be >= 0");
    if (ndim < 0 || ndim > PB_TF_DIMS) return fail(h, PB_ERR_INVALID, "thinfilm: the calculation shape has at most 4 dims");
    if ((ndim && !shape) || !strides || !in) return fail(h, PB_ERR_INVALID, "thinfilm: missing shape, strides or operands");
    tf_align(shape, ndim, 1, op.shape);
    count = 1;
    for (int j = 0; j < PB_TF_DIMS; ++j) {
        if (op.shape[j] < 0) return fail(h, PB_ERR_INVALID, "thinfilm: negative extent");
        count *= op.shape[j];
    }
    for (int q = 0; q < PB_TF_NOPS; ++q) {
        const bool layered = q == PB_TF_IN_N || q == PB_TF_IN_D;
        if (!in[q] && (!layered || nlayers > 0)) return fail(h, PB_ERR_INVALID, "thinfilm: missing operand");
        op.p[q] = in[q];
        tf_align(strides + 5 * q, ndim, 0, op.st[q]);
        op.st[q][PB_TF_DIMS] = layered ? strides[5 * q + PB_TF_DIMS] : 0;
    }
    op.nlayers = nlayers;
    op.pol = pol;
    op.theta_scale = 1.0;
    return PB_OK;
}

// the second launch of a sweeping kernel with W warp slots per row: tf_reduce_kernel over its `rows` partial rows
static int tf_reduce(Handle* h, cudaStream_t st, int dtype, const double* partial, long long W, long long count,
                     long long rows, int accumulate, void* dst, double* value) {
    const long long nw = std::min<long long>(W, (count + 31) / 32);     // warps that had at least one sample
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        tf_reduce_kernel<R><<<(unsigned)rows, PB_TF_THREADS, 0, st>>>(partial, W, nw, accumulate, (R*)dst, value);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_stack_eval(pb_handle_t hh, int dtype, int mode, int pol, int flags, int nlayers, int ndim,
                             const long long* shape, const long long* strides, const void* const* in, double theta_scale,
                             void* const* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (mode != PB_TF_THINFILM && mode != PB_TF_COATINGS) return fail(h, PB_ERR_INVALID, "thinfilm: bad mode");
    if (flags <= 0 || flags >= (1 << PB_TF_NOUT) || !out) return fail(h, PB_ERR_INVALID, "thinfilm: no output");
    if (mode == PB_TF_THINFILM && (flags & ~(1 << PB_TF_OUT_R | 1 << PB_TF_OUT_T)))
        return fail(h, PB_ERR_INVALID, "thinfilm: multilayer_stack_rt mode writes r and t only");
    if (mode == PB_TF_THINFILM && nlayers < 1) return fail(h, PB_ERR_INVALID, "thinfilm: at least one film layer");
    TfOps op;
    long long count;
    PB_TRY(tf_ops(h, pol, nlayers, ndim, shape, strides, in, op, count));
    op.theta_scale = theta_scale;
    TfOut o;
    for (int q = 0; q < PB_TF_NOUT; ++q) {
        o.p[q] = (flags >> q & 1) ? out[q] : nullptr;
        if ((flags >> q & 1) && !out[q]) return fail(h, PB_ERR_INVALID, "thinfilm: an output asked for is NULL");
    }
    if (count == 0) return PB_OK;
    TfStage sg{(double2*)o.p[PB_TF_OUT_E], (double2*)o.p[PB_TF_OUT_H], (double*)o.p[PB_TF_OUT_ESQ],
               (double*)o.p[PB_TF_OUT_ABS]};
    if (dtype == PB_C64 && (sg.E || sg.H || sg.Esq || sg.A)) {
        // float outputs: the stage lives in the handle's scratch, one fp64 array per field output
        const size_t nb = (size_t)(nlayers + 1) * count, na = (size_t)nlayers * count;
        const size_t bytes = (sg.E ? 16 * nb : 0) + (sg.H ? 16 * nb : 0) + (sg.Esq ? 8 * nb : 0) + (sg.A ? 8 * na : 0);
        void* base = nullptr;
        PB_TRY(ensure_scratch(h, 2, bytes, &base));
        char* p = (char*)base;
        if (sg.E) { sg.E = (double2*)p; p += 16 * nb; }
        if (sg.H) { sg.H = (double2*)p; p += 16 * nb; }
        if (sg.Esq) { sg.Esq = (double*)p; p += 8 * nb; }
        if (sg.A) sg.A = (double*)p;
    }
    const int g = grid_for(count, PB_TF_THREADS, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        if (mode == PB_TF_THINFILM) stack_eval_kernel<R, PB_TF_THINFILM><<<g, PB_TF_THREADS, 0, st>>>(op, count, o, sg);
        else stack_eval_kernel<R, PB_TF_COATINGS><<<g, PB_TF_THREADS, 0, st>>>(op, count, o, sg);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_stack_grad(pb_handle_t hh, int dtype, int pol, int kinds, int nlayers, int ndim, const long long* shape,
                             const long long* strides, const void* const* in, const void* E, const void* H,
                             const void* const* seeds, void* grad, void* stream) {
    PB_ENTER_REAL(hh);
    if (kinds < 1 || kinds > (PB_TF_GRAD_THICKNESS | PB_TF_GRAD_INDEX)) return fail(h, PB_ERR_INVALID, "thinfilm: bad gradient kind");
    if (!E || !H || !seeds || !grad) return fail(h, PB_ERR_INVALID, "thinfilm: missing fields, seeds or output");
    TfOps op;
    long long count;
    PB_TRY(tf_ops(h, pol, nlayers, ndim, shape, strides, in, op, count));
    if (nlayers == 0) return PB_OK;
    const int ng = (kinds & PB_TF_GRAD_THICKNESS ? 1 : 0) + (kinds & PB_TF_GRAD_INDEX ? 1 : 0);
    if (count == 0) {
        PB_CUDA(h, cudaMemsetAsync(grad, 0, (size_t)ng * nlayers * rsize(dtype), st));
        return PB_OK;
    }
    const int g = grid_for(count, PB_TF_THREADS, h->sm_count);
    const long long W = (long long)g * (PB_TF_THREADS / 32);
    void* partial = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)ng * nlayers * W * sizeof(double), &partial));
    stack_grad_kernel<<<g, PB_TF_THREADS, 0, st>>>(op, count, kinds, (const double2*)E, (const double2*)H,
                                                   (const double*)seeds[0], (const double*)seeds[1],
                                                   (const double*)seeds[2], (const double*)seeds[3], (double*)partial);
    PB_LAUNCH_CHECK(h);
    return tf_reduce(h, st, dtype, (const double*)partial, W, count, (long long)ng * nlayers, 0, grad, nullptr);
}

extern "C" int pb_field_at_depth(pb_handle_t hh, int dtype, int pol, int nlayers, const void* z, long long nz,
                                 const void* zb, const void* n, double n0_re, double n0_im, double wvl, double theta0,
                                 const void* E_b, const void* H_b, void* E, void* H, void* stream) {
    PB_ENTER_REAL(hh);
    if (pol != PB_TF_POL_S && pol != PB_TF_POL_P) return fail(h, PB_ERR_INVALID, "thinfilm: pol must be PB_TF_POL_S or P");
    if (nlayers < 1) return fail(h, PB_ERR_INVALID, "field_at_depth requires at least one layer");
    if (nz < 0 || !z || !zb || !n || !E_b || !H_b || !E || !H) return fail(h, PB_ERR_INVALID, "bad field_at_depth arguments");
    if (nz == 0) return PB_OK;
    const int g = grid_for(nz, PB_TF_THREADS, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        field_at_depth_kernel<R><<<g, PB_TF_THREADS, 0, st>>>((const double*)z, nz, (const double*)zb, nlayers,
                                                              (const double2*)n, make_double2(n0_re, n0_im), wvl,
                                                              sin(theta0), pol, (const double2*)E_b, (const double2*)H_b,
                                                              (cplx<R>*)E, (cplx<R>*)H);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

// the term of a pb_coating_merit / pb_needle call: the six thin-film operands through tf_ops, then target and weight
static int cm_setup(Handle* h, int quantity, int pol, int nlayers, int ndim, const long long* shape,
                    const long long* strides, const void* const* in, TfOps& op, CmTerm& tm, long long& count) {
    if (quantity < PB_CM_Q_R || quantity > PB_CM_Q_LAYER) return fail(h, PB_ERR_INVALID, "coating merit: bad quantity");
    if (pol != PB_TF_POL_S && pol != PB_TF_POL_P && pol != PB_CM_POL_AVG)
        return fail(h, PB_ERR_INVALID, "coating merit: pol must be PB_TF_POL_S, P or PB_CM_POL_AVG");
    if (!in || !strides) return fail(h, PB_ERR_INVALID, "coating merit: missing operands");
    PB_TRY(tf_ops(h, pol == PB_CM_POL_AVG ? PB_TF_POL_S : pol, nlayers, ndim, shape, strides, in, op, count));
    if (!in[PB_CM_IN_TARGET] || !in[PB_CM_IN_WEIGHT]) return fail(h, PB_ERR_INVALID, "coating merit: missing target or weight");
    tm.quantity = quantity;
    tm.npol = pol == PB_CM_POL_AVG ? 2 : 1;
    tm.tgt = (const double*)in[PB_CM_IN_TARGET];
    tm.wgt = (const double*)in[PB_CM_IN_WEIGHT];
    tf_align(strides + 5 * PB_CM_IN_TARGET, ndim, 0, tm.st_tgt);
    tf_align(strides + 5 * PB_CM_IN_WEIGHT, ndim, 0, tm.st_wgt);
    tm.cpad = (count + 31) / 32 * 32;
    tm.b0 = tm.b1 = tm.nb = 0;
    tm.blist = nullptr;
    return PB_OK;
}

// the handle's scratch as nrows * W fp64 warp partials, then the stage of npol * (nlayers + 1) boundary vectors
static int cm_scratch(Handle* h, const CmTerm& tm, int nlayers, long long nrows, long long W, double** partial,
                      double2** V0, double2** V1) {
    const size_t pbytes = ((size_t)nrows * W * sizeof(double) + 255) / 256 * 256;
    const size_t vn = (size_t)tm.npol * (nlayers + 1) * tm.cpad;
    void* base = nullptr;
    PB_TRY(ensure_scratch(h, 2, pbytes + 2 * vn * sizeof(double2), &base));
    *partial = (double*)base;
    *V0 = (double2*)((char*)base + pbytes);
    *V1 = *V0 + vn;
    return PB_OK;
}

extern "C" int pb_coating_merit(pb_handle_t hh, int dtype, int quantity, int pol, int flags, int nlayers, int ndim,
                                const long long* shape, const long long* strides, const void* const* in, int b0, int b1,
                                const void* blist, int nb, void* value, void* residuals, void* grad, void* stream) {
    PB_ENTER_REAL(hh);
    if (flags <= 0 || flags >= 2 * PB_CM_ACCUMULATE || !(flags & ~PB_CM_ACCUMULATE))
        return fail(h, PB_ERR_INVALID, "coating merit: no output");
    if ((flags & PB_CM_OUT_VALUE && !value) || (flags & PB_CM_OUT_RESIDUALS && !residuals) ||
        (flags & (PB_CM_OUT_GRAD_THICKNESS | PB_CM_OUT_GRAD_INDEX) && !grad))
        return fail(h, PB_ERR_INVALID, "coating merit: an output asked for is NULL");
    TfOps op;
    CmTerm tm;
    long long count;
    PB_TRY(cm_setup(h, quantity, pol, nlayers, ndim, shape, strides, in, op, tm, count));
    const int nbound = quantity == PB_CM_Q_ABS ? nlayers : nlayers + 1;
    if (quantity == PB_CM_Q_ABS || quantity == PB_CM_Q_ESQ || quantity == PB_CM_Q_LAYER) {
        if (b0 < 0 || b0 >= nbound || (quantity == PB_CM_Q_LAYER && (b1 < 0 || b1 >= nbound)))
            return fail(h, PB_ERR_INVALID, "coating merit: layer or boundary index out of range");
    }
    if (quantity == PB_CM_Q_PEAK && (nb < 1 || !blist)) return fail(h, PB_ERR_INVALID, "coating merit: no boundaries");
    tm.b0 = b0;
    tm.b1 = b1;
    tm.nb = quantity == PB_CM_Q_PEAK ? nb : 0;
    tm.blist = (const int*)blist;
    const int kinds = (flags >> 2) & 3;
    const bool acc = flags & PB_CM_ACCUMULATE;
    const int ng = (kinds & 1) + (kinds >> 1 & 1);
    if (count == 0) {
        if (!acc && (flags & PB_CM_OUT_VALUE)) PB_CUDA(h, cudaMemsetAsync(value, 0, sizeof(double), st));
        if (!acc && kinds && nlayers) PB_CUDA(h, cudaMemsetAsync(grad, 0, (size_t)ng * nlayers * rsize(dtype), st));
        return PB_OK;
    }
    const long long rows = (long long)ng * nlayers + (flags & PB_CM_OUT_VALUE ? 1 : 0);
    const int nt = cm_threads(tm.npol);
    const int g = grid_for(count, nt, h->sm_count);
    const long long W = (long long)g * (nt / 32);
    double* partial;
    double2 *V0, *V1;
    PB_TRY(cm_scratch(h, tm, nlayers, rows, W, &partial, &V0, &V1));
    if (tm.npol == 2) coating_merit_kernel<2><<<g, nt, 0, st>>>(op, tm, count, flags, V0, V1, partial, residuals,
                                                                dtype == PB_C64);
    else coating_merit_kernel<1><<<g, nt, 0, st>>>(op, tm, count, flags, V0, V1, partial, residuals, dtype == PB_C64);
    PB_LAUNCH_CHECK(h);
    if (!rows) return PB_OK;
    return tf_reduce(h, st, dtype, partial, W, count, rows, acc, grad, flags & PB_CM_OUT_VALUE ? (double*)value : nullptr);
}

extern "C" int pb_needle(pb_handle_t hh, int dtype, int quantity, int pol, int nlayers, int ndim, const long long* shape,
                         const long long* strides, const void* const* in, const void* zpart, long long nz,
                         const void* zlist, void* P, int accumulate, void* stream) {
    PB_ENTER_REAL(hh);
    if (quantity != PB_CM_Q_R && quantity != PB_CM_Q_T)
        return fail(h, PB_ERR_INVALID, "needle: the term must target R or T");
    if (nlayers < 1) return fail(h, PB_ERR_INVALID, "needle: at least one layer");
    if (nz < 0 || (nz && (!zpart || !zlist || !P))) return fail(h, PB_ERR_INVALID, "bad needle arguments");
    TfOps op;
    CmTerm tm;
    long long count;
    PB_TRY(cm_setup(h, quantity, pol, nlayers, ndim, shape, strides, in, op, tm, count));
    if (!in[PB_CM_IN_NEEDLE]) return fail(h, PB_ERR_INVALID, "needle: missing needle index");
    if (nz == 0) return PB_OK;
    if (count == 0) {
        if (!accumulate) PB_CUDA(h, cudaMemsetAsync(P, 0, (size_t)nz * rsize(dtype), st));
        return PB_OK;
    }
    const int nt = cm_threads(tm.npol);
    const int g = grid_for(count, nt, h->sm_count);
    const long long W = (long long)g * (nt / 32);
    double* partial;
    double2 *V0, *V1;
    PB_TRY(cm_scratch(h, tm, nlayers, nz, W, &partial, &V0, &V1));
    NeedleStrides ns;
    tf_align(strides + 5 * PB_CM_IN_NEEDLE, ndim, 0, ns.st);
    auto launch = [&](auto kern) {
        kern<<<g, nt, 0, st>>>(op, tm, (const double2*)in[PB_CM_IN_NEEDLE], ns, count, (const double*)zpart, nz,
                               (const int*)zlist, V0, V1, partial);
    };
    if (tm.npol == 2) launch(needle_kernel<2>);
    else launch(needle_kernel<1>);
    PB_LAUNCH_CHECK(h);
    return tf_reduce(h, st, dtype, partial, W, count, nz, accumulate, P, nullptr);
}

extern "C" int pb_monitor_runs(pb_handle_t hh, int dtype, int strategy, int mode, int pol, int nlayers, long long ncand,
                               const void* const* in, long long runs, long long per_cand, const void* err,
                               const void* levels, long long n_points, double start, double max_factor,
                               int turning_index, void* asbuilt, void* stream) {
    PB_ENTER_REAL(hh);
    if (strategy != PB_MON_LEVEL && strategy != PB_MON_TURNING) return fail(h, PB_ERR_INVALID, "monitor: bad strategy");
    if (mode != PB_MON_R && mode != PB_MON_T) return fail(h, PB_ERR_INVALID, "monitor: mode must be PB_MON_R or T");
    if (pol != PB_TF_POL_S && pol != PB_TF_POL_P) return fail(h, PB_ERR_INVALID, "monitor: pol must be PB_TF_POL_S or P");
    if (nlayers < 0 || ncand < 1 || runs < 0 || per_cand < 1 || runs > ncand * per_cand || runs > INT_MAX || n_points < 0)
        return fail(h, PB_ERR_INVALID, "monitor: bad layer, candidate, run or grid counts");
    if (runs && nlayers && (!in || !asbuilt || (strategy == PB_MON_LEVEL && (!levels || n_points < 1)) ||
                            (strategy == PB_MON_TURNING && turning_index < 1)))
        return fail(h, PB_ERR_INVALID, "monitor: missing operands, levels or output, an empty level grid, or a "
                                       "turning index below 1");
    if (!runs || !nlayers) return PB_OK;
    for (int q = 0; q < PB_TF_NOPS; ++q)
        if (!in[q]) return fail(h, PB_ERR_INVALID, "monitor: missing operand");
    // candidate c is sample c of a one-axis calculation shape; the nominal thicknesses are shared
    TfOps op{};
    for (int j = 0; j < PB_TF_DIMS; ++j) op.shape[j] = j == PB_TF_DIMS - 1 ? ncand : 1;
    for (int q = 0; q < PB_TF_NOPS; ++q) {
        op.p[q] = in[q];
        op.st[q][PB_TF_DIMS - 1] = q == PB_TF_IN_D ? 0 : 1;
    }
    op.st[PB_TF_IN_N][PB_TF_DIMS] = ncand;
    op.st[PB_TF_IN_D][PB_TF_DIMS] = 1;
    op.nlayers = nlayers;
    op.pol = pol;
    op.theta_scale = 1.0;
    const MonArgs a{(const double*)err, (const double*)levels, per_cand, n_points, start, max_factor, strategy, mode,
                    turning_index};
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        monitor_runs_kernel<R><<<(unsigned)runs, PB_MON_THREADS, 0, st>>>(op, a, (R*)asbuilt);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_monitor_cut(pb_handle_t hh, int dtype, int strategy, const void* d, const void* sig, long long n,
                              double level, double target, void* out, void* count, void* stream) {
    PB_ENTER_REAL(hh);
    if (strategy != PB_MON_LEVEL && strategy != PB_MON_TURNING) return fail(h, PB_ERR_INVALID, "monitor: bad strategy");
    if (n < 0 || (n && (!d || !sig || !out)) || (strategy == PB_MON_TURNING && !count))
        return fail(h, PB_ERR_INVALID, "monitor: bad trace arguments");
    if (strategy == PB_MON_LEVEL && n < 1) return fail(h, PB_ERR_INVALID, "monitor: level_cut of an empty trace");
    with_real(dtype, [&](auto r) {
        using T = decltype(r);
        monitor_cut_kernel<T><<<1, PB_MON_THREADS, 0, st>>>(strategy, (const T*)d, (const T*)sig, n, (T)level, (T)target,
                                                            (T*)out, (long long*)count);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_monitor_jacobian(pb_handle_t hh, int dtype, int ncand, int nlayers, long long nw, const void* Rr,
                                   double eps, void* J, void* score, void* stream) {
    PB_ENTER_REAL(hh);
    if (ncand < 0 || ncand > 65535 || nlayers < 0 || nw < 0 || (ncand && !Rr) || (!J && !score))
        return fail(h, PB_ERR_INVALID, "monitor: bad jacobian arguments");
    if (!ncand) return PB_OK;
    const long long cnt = nw * nlayers;
    if (!cnt) {
        if (score) PB_CUDA(h, cudaMemsetAsync(score, 0, (size_t)ncand * rsize(dtype), st));
        return PB_OK;
    }
    const int g = fold_blocks(cnt, h->sm_count);
    double* part;
    unsigned* counters;
    PB_TRY(fold_scratch(h, ncand, g, 1, st, &part, &counters));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        monitor_jacobian_kernel<R><<<dim3(g, ncand), 256, 0, st>>>((const double*)Rr, nlayers, nw, eps, (R*)J, (R*)score,
                                                                   part, counters);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
