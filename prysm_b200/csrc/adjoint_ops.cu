// Elementwise kernels and small reductions of the adjoint twins and the Lyot-coronagraph compositions
// (all HBM-bound streaming work; 16-48 algorithmic bytes per sample):
//   masked multiply  out (+)= scale * (a - b) * f(m) * w        coronagraph.py:12-99, 212-431, _kernels.py:30-38
//   field adjoints   from_amp_and_phase adjoints                  wavefront.py:172-242
//   weighted dot     sum w * a * conj(b)                          wavefront.py:244-280 (thin_lens_adjoint)
//   mode projection  sum modes[k] * bar                           polynomials/fitting.py:40-57
//   otf adjoint seed gradient at the k-space plane                otf.py:205-316
//   EE adjoint seed  MTF-plane gradient of the Baliga-Cohn sum    otf.py:417-471
//   vortex mask, multi-resolution hand-off window + grids         coronagraph.py:102-132, dft.py:155-294
#include "common.cuh"

namespace pb {

template <typename R>
__global__ void mask_multiply_kernel(const cplx<R>* __restrict__ a, const cplx<R>* __restrict__ b, const void* __restrict__ m,
                                     int m_kind, int flags, const R* __restrict__ w, R scale, long long n, void* out) {
    PB_GRID_STRIDE(i, n) {
        cplx<R> v = a[i];
        if (b) v = csub(v, b[i]);
        if (m) {
            cplx<R> f = m_kind == PB_MASK_COMPLEX ? reinterpret_cast<const cplx<R>*>(m)[i]
                                                  : mk<R>(reinterpret_cast<const R*>(m)[i], R(0));
            if (flags & PB_MASK_ONE_MINUS) { f.x = R(1) - f.x; f.y = -f.y; }
            if (flags & PB_MASK_CONJ) f.y = -f.y;
            v = cmul(v, f);
        }
        R s = scale;
        if (w) s *= w[i];
        v.x *= s; v.y *= s;
        if (flags & PB_MASK_REAL_OUT) {
            R* o = reinterpret_cast<R*>(out);
            o[i] = (flags & PB_MASK_ACCUMULATE) ? o[i] + v.x : v.x;
        } else {
            cplx<R>* o = reinterpret_cast<cplx<R>*>(out);
            if (flags & PB_MASK_ACCUMULATE) v = cadd(v, o[i]);
            o[i] = v;
        }
    }
}

// mode 0: out(complex) = i*k*imag(bar*conj(f));  1: out(real) = real(bar*conj(f))/|f| (0 where f = 0);
// mode 2: out(real) = real(bar*conj(S)), S = exp(i*k*opd)
template <typename R>
__global__ void field_adjoint_kernel(int mode, const cplx<R>* __restrict__ f, const cplx<R>* __restrict__ bar,
                                     const R* __restrict__ opd, double k, long long n, void* out) {
    const double kturns = k / (2.0 * M_PI);
    PB_GRID_STRIDE(i, n) {
        const cplx<R> g = bar[i];
        if (mode == 0) {
            const cplx<R> p = f[i];
            reinterpret_cast<cplx<R>*>(out)[i] = mk<R>(R(0), (R)k * (g.y * p.x - g.x * p.y));
        } else if (mode == 1) {
            const cplx<R> p = f[i];
            const R mod = hypot(p.x, p.y);
            reinterpret_cast<R*>(out)[i] = mod > R(0) ? (g.x * p.x + g.y * p.y) / mod : R(0);
        } else {
            const cplx<R> s = expi_turns(kturns * (double)opd[i], R(0));
            reinterpret_cast<R*>(out)[i] = g.x * s.x + g.y * s.y;
        }
    }
}

// which 0: re, 1: im, 2: angle, 3: abs
template <typename R>
__global__ void component_kernel(int which, const cplx<R>* __restrict__ in, long long n, R* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const cplx<R> v = in[i];
        out[i] = which == 0 ? v.x : which == 1 ? v.y : which == 2 ? (R)atan2(v.y, v.x) : (R)hypot(v.x, v.y);
    }
}

// sums[0..1] = sum w * a * conj(b)
template <typename R>
__global__ void dot_kernel(const cplx<R>* __restrict__ a, const cplx<R>* __restrict__ b, const R* __restrict__ w, long long n,
                           double* __restrict__ part, unsigned* __restrict__ counter, double* __restrict__ sums) {
    double re = 0, im = 0;
    PB_GRID_STRIDE(i, n) {
        const cplx<R> x = a[i], y = b[i];
        const double ww = w ? (double)w[i] : 1.0;
        re += ww * ((double)x.x * y.x + (double)x.y * y.y);
        im += ww * ((double)x.y * y.x - (double)x.x * y.y);
    }
    double v[2] = {re, im};
    block_reduce<256>(v, OpAdd{});
    if (threadIdx.x == 0) { part[blockIdx.x * 2] = v[0]; part[blockIdx.x * 2 + 1] = v[1]; }
    if (!arrive_last(counter)) return;
    v[0] = fold_partials<256, 2>(part, 0, OpAdd{}, 0.0);
    v[1] = fold_partials<256, 2>(part, 1, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { sums[0] = v[0]; sums[1] = v[1]; }
}

// sums[2k..2k+1] = sum modes[k][i] * bar[i]      (bar real or complex), mode k in grid row k
template <typename R>
__global__ void mode_projection_kernel(const R* __restrict__ modes, long long n, const void* __restrict__ bar, int bar_complex,
                                       double* __restrict__ part, unsigned* __restrict__ counters, double* __restrict__ sums) {
    const R* mode = modes + (long long)blockIdx.y * n;
    double re = 0, im = 0;
    PB_GRID_STRIDE(i, n) {
        const double mv = (double)mode[i];
        if (bar_complex) {
            const cplx<R> g = reinterpret_cast<const cplx<R>*>(bar)[i];
            re += mv * g.x; im += mv * g.y;
        } else {
            re += mv * reinterpret_cast<const R*>(bar)[i];
        }
    }
    double v[2] = {re, im};
    block_reduce<256>(v, OpAdd{});
    if (threadIdx.x == 0) {
        double* p = part + ((size_t)blockIdx.y * gridDim.x + blockIdx.x) * 2;
        p[0] = v[0]; p[1] = v[1];
    }
    if (!arrive_last(counters)) return;
    v[0] = fold_partials<256, 2>(part, 0, OpAdd{}, 0.0);
    v[1] = fold_partials<256, 2>(part, 1, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { sums[2 * blockIdx.y] = v[0]; sums[2 * blockIdx.y + 1] = v[1]; }
}

// which 1 (mtf): S = sum bar*|D|;  2 (ptf): S = sum bar;  4 (otf): S = sum conj(D)*bar
template <typename R>
__global__ void otf_adjoint_reduce_kernel(int which, const void* __restrict__ bar, const cplx<R>* __restrict__ D, long long n,
                                          double* __restrict__ part, unsigned* __restrict__ counter, double* __restrict__ sums) {
    double re = 0, im = 0;
    PB_GRID_STRIDE(i, n) {
        if (which == 4) {
            const cplx<R> g = reinterpret_cast<const cplx<R>*>(bar)[i], d = D[i];
            re += (double)d.x * g.x + (double)d.y * g.y;
            im += (double)d.x * g.y - (double)d.y * g.x;
        } else {
            const double g = (double)reinterpret_cast<const R*>(bar)[i];
            if (which == 1) { const cplx<R> d = D[i]; re += g * hypot((double)d.x, (double)d.y); }
            else re += g;
        }
    }
    double v[2] = {re, im};
    block_reduce<256>(v, OpAdd{});
    if (threadIdx.x == 0) { part[blockIdx.x * 2] = v[0]; part[blockIdx.x * 2 + 1] = v[1]; }
    if (!arrive_last(counter)) return;
    v[0] = fold_partials<256, 2>(part, 0, OpAdd{}, 0.0);
    v[1] = fold_partials<256, 2>(part, 1, OpAdd{}, 0.0);
    if (threadIdx.x == 0) { sums[0] = v[0]; sums[1] = v[1]; }
}

template <typename R>
__global__ void otf_adjoint_apply_kernel(int which, const void* __restrict__ bar, const cplx<R>* __restrict__ D, long long n,
                                         long long centre, const double* __restrict__ sums, cplx<R>* __restrict__ out) {
    const cplx<R> c = D[centre];
    const double Sre = sums[0], Sim = sums[1];
    const double cx = c.x, cy = c.y, cm2 = cx * cx + cy * cy;
    PB_GRID_STRIDE(i, n) {
        const cplx<R> d = D[i];
        double ore, oim;
        if (which == 1) {                       // bar * D/|D| / a ;  centre -= S*c/a^3
            const double g = (double)reinterpret_cast<const R*>(bar)[i];
            const double mag = hypot((double)d.x, (double)d.y), a = sqrt(cm2);
            ore = g * d.x / mag / a; oim = g * d.y / mag / a;
            if (i == centre) { const double a3 = a * a * a; ore -= Sre * cx / a3; oim -= Sre * cy / a3; }
        } else if (which == 2) {                // bar * i*D/|D|^2 ;  centre -= S*i*c/|c|^2
            const double g = (double)reinterpret_cast<const R*>(bar)[i];
            const double msq = (double)d.x * d.x + (double)d.y * d.y;
            ore = -g * d.y / msq; oim = g * d.x / msq;
            if (i == centre) { ore -= -Sre * cy / cm2; oim -= Sre * cx / cm2; }
        } else {                                // bar / conj(c) ;  centre -= S / conj(c)^2
            const cplx<R> g = reinterpret_cast<const cplx<R>*>(bar)[i];
            // 1/conj(c) = c/|c|^2
            ore = ((double)g.x * cx - (double)g.y * cy) / cm2;
            oim = ((double)g.x * cy + (double)g.y * cx) / cm2;
            if (i == centre) {
                // 1/conj(c)^2 = c^2/|c|^4
                const double c2re = cx * cx - cy * cy, c2im = 2 * cx * cy, den = cm2 * cm2;
                ore -= (Sre * c2re - Sim * c2im) / den;
                oim -= (Sre * c2im + Sim * c2re) / den;
            }
        }
        out[i] = mk<R>((R)ore, (R)oim);
    }
}

// mtf_bar[y,x] = sum_r eebar[r] * r * J1(2 pi r nu)/nu * df^2 on the fftrange*df grid (nu(0) -> 1e-16)
template <typename R>
__global__ void ee_adjoint_seed_kernel(int ny, int nx, double df, const double* __restrict__ radii, const double* __restrict__ eebar,
                                       int nr, R* __restrict__ out) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        double nu = hypot((double)(x - nx / 2) * df, (double)(y - ny / 2) * df);
        if (nu == 0.0) nu = 1e-16;
        double acc = 0.0;
        for (int r = 0; r < nr; ++r) acc += eebar[r] * radii[r] * (j1(6.283185307179586476925 * radii[r] * nu) / nu) * df * df;
        out[i] = (R)acc;
    }
}

template <typename R>
__global__ void vortex_kernel(int charge, const R* __restrict__ xf, const R* __restrict__ yf, long long n, cplx<R>* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const double th = atan2((double)yf[i], (double)xf[i]);
        out[i] = expi_turns((double)charge * th * 0.15915494309189533577, R(0));
    }
}

// Bilinear resampling of a complex map at col = (xf - cx)/dx + nx/2, row = (yf - cy)/dx + ny/2 with edge replication
// (scipy.ndimage.map_coordinates(order=1, mode='nearest')), `fill` outside [0, n-1] on either axis
// (prysm/propagation/coronagraph.py:192-207).
template <typename R>
__global__ void resample_bilinear_kernel(const cplx<R>* __restrict__ map, int ny, int nx, const R* __restrict__ xf,
                                         const R* __restrict__ yf, long long n, double cx, double cy, double dx,
                                         const cplx<R>* __restrict__ fill, cplx<R> fill_s, cplx<R>* __restrict__ out) {
    PB_GRID_STRIDE(i, n) {
        const double col = ((double)xf[i] - cx) / dx + (double)(nx / 2);
        const double row = ((double)yf[i] - cy) / dx + (double)(ny / 2);
        const bool inside = row >= 0.0 && row <= (double)(ny - 1) && col >= 0.0 && col <= (double)(nx - 1);
        if (!inside) { out[i] = fill ? fill[i] : fill_s; continue; }
        const double fr = floor(row), fc = floor(col);
        const int r0 = (int)fr, c0 = (int)fc;
        const int r1 = min(r0 + 1, ny - 1), c1 = min(c0 + 1, nx - 1);
        const double wr = row - fr, wc = col - fc;
        const cplx<R> a = map[(long long)r0 * nx + c0], b = map[(long long)r0 * nx + c1];
        const cplx<R> c = map[(long long)r1 * nx + c0], d = map[(long long)r1 * nx + c1];
        const double re = (1 - wr) * ((1 - wc) * a.x + wc * b.x) + wr * ((1 - wc) * c.x + wc * d.x);
        const double im = (1 - wr) * ((1 - wc) * a.y + wc * b.y) + wr * ((1 - wc) * c.y + wc * d.y);
        out[i] = mk<R>((R)re, (R)im);
    }
}

__device__ inline double smootherstep(double t) {
    t = fmin(fmax(t, 0.0), 1.0);
    return t * t * t * (t * (t * 6.0 - 15.0) + 10.0);
}

// grids xf = (ix - nx/2)*fdx + shift, yf likewise; window = taper(a0, b0) - taper(a1, b1) with taper = 1 - smootherstep((r-a)/(b-a));
// a0 < 0 -> outer taper == 1 (coarsest level), a1 < 0 -> inner taper == 0 (finest level)
template <typename R>
__global__ void radial_window_kernel(int ny, int nx, double fdx, double shift, double a0, double b0, double a1, double b1,
                                     R* __restrict__ win, R* __restrict__ xf, R* __restrict__ yf) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        // the reference builds the axes in config precision, then meshgrid/hypot in that precision
        const R xv = mul_add_rn((R)(x - nx / 2), (R)fdx, (R)shift), yv = mul_add_rn((R)(y - ny / 2), (R)fdx, (R)shift);
        if (xf) xf[i] = xv;
        if (yf) yf[i] = yv;
        if (win) {
            const double r = hypot((double)xv, (double)yv);
            const double here = a0 < 0 ? 1.0 : 1.0 - smootherstep((r - a0) / (b0 - a0));
            const double next = a1 < 0 ? 0.0 : 1.0 - smootherstep((r - a1) / (b1 - a1));
            win[i] = (R)(here - next);
        }
    }
}

}  // namespace pb

using namespace pb;

extern "C" int pb_mask_multiply(pb_handle_t hh, int dtype, const void* a, const void* b, const void* m, int m_kind, int flags,
                                const void* w, double scale, long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !out || (m && m_kind != PB_MASK_REAL && m_kind != PB_MASK_COMPLEX) || (flags & ~15))
        return fail(h, PB_ERR_INVALID, "bad masked-multiply arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        mask_multiply_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)a, (const cplx<R>*)b, m, m_kind, flags, (const R*)w, (R)scale, count, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_field_adjoint(pb_handle_t hh, int dtype, int mode, const void* field, const void* bar, const void* opd,
                                double kscale, long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (mode < 0 || mode > 2 || !bar || !out || (mode < 2 && !field) || (mode == 2 && !opd))
        return fail(h, PB_ERR_INVALID, "bad field-adjoint arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        field_adjoint_kernel<R><<<g, 256, 0, st>>>(mode, (const cplx<R>*)field, (const cplx<R>*)bar, (const R*)opd, kscale, count, out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_component(pb_handle_t hh, int dtype, int which, const void* in, long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (which < 0 || which > 3 || !in || !out) return fail(h, PB_ERR_INVALID, "bad component arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        component_kernel<R><<<g, 256, 0, st>>>(which, (const cplx<R>*)in, count, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_dot(pb_handle_t hh, int dtype, const void* a, const void* b, const void* w, long long count,
                      double* out_host, void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !b || !out_host || count < 0) return fail(h, PB_ERR_INVALID, "bad dot arguments");
    out_host[0] = out_host[1] = 0.0;
    if (count == 0) return PB_OK;
    const int g = fold_blocks(count, h->sm_count);
    double *part, *sums; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, g, 2, st, &part, &counter));
    PB_TRY(ensure_scratch(h, 2, 2 * sizeof(double), (void**)&sums));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        dot_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)a, (const cplx<R>*)b, (const R*)w, count, part, counter, sums);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaMemcpyAsync(out_host, sums, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_mode_projection(pb_handle_t hh, int dtype, const void* modes, int k, long long count, const void* bar,
                                  int bar_complex, double* out_host, void* stream) {
    PB_ENTER_REAL(hh);
    if (k < 1 || count <= 0 || !modes || !bar || !out_host) return fail(h, PB_ERR_INVALID, "bad mode-projection arguments");
    const int gx = (int)std::min<long long>((count + 255) / 256, std::max(1LL, (long long)h->sm_count * 4 / k));
    double *part, *sums; unsigned* counters;
    PB_TRY(fold_scratch(h, k, gx, 2, st, &part, &counters));
    PB_TRY(ensure_scratch(h, 2, (size_t)2 * k * sizeof(double), (void**)&sums));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        mode_projection_kernel<R><<<dim3(gx, k), 256, 0, st>>>((const R*)modes, count, bar, bar_complex, part, counters, sums);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaMemcpyAsync(out_host, sums, (size_t)2 * k * sizeof(double), cudaMemcpyDeviceToHost, st));
    PB_CUDA(h, cudaStreamSynchronize(st));
    return PB_OK;
}

extern "C" int pb_otf_adjoint_seed(pb_handle_t hh, int dtype, int which, const void* bar, const void* D, int ny, int nx,
                                   void* data_bar, void* stream) {
    PB_ENTER_REAL(hh);
    if ((which != 1 && which != 2 && which != 4) || !bar || !D || !data_bar || ny < 1 || nx < 1)
        return fail(h, PB_ERR_INVALID, "bad otf-adjoint arguments");
    const long long n = (long long)ny * nx, centre = (long long)(ny / 2) * nx + nx / 2;
    const int gr = fold_blocks(n, h->sm_count), g = grid_for(n, 256, h->sm_count);
    double *part, *sums; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, gr, 2, st, &part, &counter));
    PB_TRY(ensure_scratch(h, 2, 2 * sizeof(double), (void**)&sums));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        otf_adjoint_reduce_kernel<R><<<gr, 256, 0, st>>>(which, bar, (const cplx<R>*)D, n, part, counter, sums);
        otf_adjoint_apply_kernel<R><<<g, 256, 0, st>>>(which, bar, (const cplx<R>*)D, n, centre, sums, (cplx<R>*)data_bar);
    });
    PB_LAUNCH_CHECK(h);
    h->launches++;
    return PB_OK;
}

extern "C" int pb_encircled_energy_adjoint_seed(pb_handle_t hh, int dtype, int ny, int nx, double df, const double* radii_mm_host,
                                                const double* ee_bar_host, int nr, void* mtf_bar, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1 || nr < 1 || !radii_mm_host || !ee_bar_host || !mtf_bar) return fail(h, PB_ERR_INVALID, "bad encircled-energy adjoint arguments");
    void* d = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)2 * nr * sizeof(double), &d));
    double* dr = (double*)d;
    double* db = dr + nr;
    PB_CUDA(h, cudaMemcpyAsync(dr, radii_mm_host, nr * sizeof(double), cudaMemcpyHostToDevice, st));
    PB_CUDA(h, cudaMemcpyAsync(db, ee_bar_host, nr * sizeof(double), cudaMemcpyHostToDevice, st));
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        ee_adjoint_seed_kernel<R><<<g, 256, 0, st>>>(ny, nx, df, dr, db, nr, (R*)mtf_bar);
    });
    PB_LAUNCH_CHECK(h);
    PB_CUDA(h, cudaStreamSynchronize(st));   // the host arrays may go away after the call
    return PB_OK;
}

extern "C" int pb_vortex_phase(pb_handle_t hh, int dtype, int charge, const void* xf, const void* yf, long long count, void* out,
                               void* stream) {
    PB_ENTER_REAL(hh);
    if (!xf || !yf || !out) return fail(h, PB_ERR_INVALID, "bad vortex arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        vortex_kernel<R><<<g, 256, 0, st>>>(charge, (const R*)xf, (const R*)yf, count, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_resample_bilinear(pb_handle_t hh, int dtype, const void* map, int ny, int nx, const void* xf, const void* yf,
                                    long long count, double cx, double cy, double dx, const void* fill, double fill_re,
                                    double fill_im, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!map || !xf || !yf || !out || ny < 1 || nx < 1 || dx == 0.0) return fail(h, PB_ERR_INVALID, "bad resample arguments");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        resample_bilinear_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)map, ny, nx, (const R*)xf, (const R*)yf, count, cx, cy, dx,
                                                       (const cplx<R>*)fill, mk<R>((R)fill_re, (R)fill_im), (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_radial_window(pb_handle_t hh, int dtype, int ny, int nx, double fdx, double shift, double a0, double b0,
                                double a1, double b1, void* win, void* xf, void* yf, void* stream) {
    PB_ENTER_REAL(hh);
    if (ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "bad window shape");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        radial_window_kernel<R><<<g, 256, 0, st>>>(ny, nx, fdx, shift, a0, b0, a1, b1, (R*)win, (R*)xf, (R*)yf);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
