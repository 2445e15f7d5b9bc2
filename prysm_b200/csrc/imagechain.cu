// Image-chain consumers of the path's FFTs (SURVEY.md 8(f) rank 4, prysm/convolution.py:9-32): the two elementwise
// kernels that let a real-object x real-PSF convolution run as ONE forward and ONE inverse transform.
//   z = obj + i*psf  ->  Z = FFT2(z) = O + i*H with O, H Hermitian, so conj(Z[-k]) = O[k] - i*H[k] and
//   O[k]*H[k] = (Z[k]^2 - conj(Z[-k])^2) / (4i).
// Both stream; the product reads each spectrum sample twice (k and -k) through L2.
// Rounding: the transform's error is relative to |Z|, so a PSF of unit sum packed beside an object of sum 1e5 would
// lose log2(1e5) bits.  pb_balance_scale measures s = sqrt(sum obj^2 / sum psf^2) on the device; the pack kernel
// multiplies the imaginary part by s and the product kernel divides it back out -- no host round trip.
#include "common.cuh"

namespace pb {

template <typename R>
__global__ void pack_complex_kernel(const R* __restrict__ re, const R* __restrict__ im, const double* __restrict__ im_scale,
                                    long long n, cplx<R>* __restrict__ out) {
    const R s = im_scale ? (R)*im_scale : R(1);
    PB_GRID_STRIDE(i, n)
        out[i] = mk<R>(re[i], im ? s * im[i] : R(0));
}

// *scale = sqrt(sum a^2 / sum b^2), 1 when either sum is 0 or not finite
template <typename R>
__global__ void balance_kernel(const R* __restrict__ a, const R* __restrict__ b, long long n, double* __restrict__ part,
                               unsigned* __restrict__ counter, double* __restrict__ scale) {
    double s[2] = {0, 0};
    PB_GRID_STRIDE(i, n) {
        const double x = a[i], y = b[i];
        s[0] += x * x; s[1] += y * y;
    }
    block_reduce<256>(s, OpAdd{});
    if (threadIdx.x == 0) { part[blockIdx.x * 2] = s[0]; part[blockIdx.x * 2 + 1] = s[1]; }
    if (!arrive_last(counter)) return;
    const double sa = fold_partials<256, 2>(part, 0, OpAdd{}, 0.0);
    const double sb = fold_partials<256, 2>(part, 1, OpAdd{}, 0.0);
    if (threadIdx.x == 0) *scale = (sa > 0.0 && sb > 0.0 && isfinite(sa) && isfinite(sb)) ? sqrt(sa / sb) : 1.0;
}

template <typename R>
__global__ void packed_spectrum_product_kernel(const cplx<R>* __restrict__ Z, int ny, int nx, R scale,
                                               const double* __restrict__ im_scale, cplx<R>* __restrict__ out) {
    const long long n = (long long)ny * nx;
    if (im_scale) scale = (R)((double)scale / *im_scale);
    PB_GRID_STRIDE(i, n) {
        const int ky = (int)(i / nx), kx = (int)(i - (long long)ky * nx);
        const int my = ky ? ny - ky : 0, mx = kx ? nx - kx : 0;
        const cplx<R> a = Z[i], b = Z[(long long)my * nx + mx];
        // a^2 - conj(b)^2
        const R pre = (a.x * a.x - a.y * a.y) - (b.x * b.x - b.y * b.y);
        const R pim = 2 * a.x * a.y + 2 * b.x * b.y;
        // divide by 4i: (p)/(4i) = (pim - i*pre)/4
        out[i] = mk<R>(scale * R(0.25) * pim, -scale * R(0.25) * pre);
    }
}

// detector sampling (prysm/detector.py:151-338): block mean / sum over fy x fx samples, its adjoint (repeat), and the
// analytic pixel / OLPF transfer functions on separable frequency vectors
template <typename R>
__global__ void bindown_kernel(const R* __restrict__ in, int oy, int ox, int fy, int fx, R scale, R* __restrict__ out) {
    const long long n = (long long)oy * ox;
    const long long in_ld = (long long)ox * fx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / ox), x = (int)(i - (long long)y * ox);
        const R* p = in + (long long)y * fy * in_ld + (long long)x * fx;
        double acc = 0.0;
        for (int a = 0; a < fy; ++a)
            for (int b = 0; b < fx; ++b) acc += (double)p[a * in_ld + b];
        out[i] = (R)(acc * (double)scale);
    }
}

template <typename R>
__global__ void tile_kernel(const R* __restrict__ in, int ny, int nx, int fy, int fx, R scale, R* __restrict__ out) {
    const long long ox = (long long)nx * fx, n = (long long)ny * fy * ox;
    PB_GRID_STRIDE(i, n) {
        const long long y = i / ox, x = i - y * ox;
        out[i] = scale * in[(y / fy) * nx + x / fx];
    }
}

// kind 0: sinc(fx wx) sinc(fy wy) (pixel_ft);  1: cos(2 wx fx) cos(2 wy fy) (olpf_ft)
template <typename R>
__global__ void separable_tf_kernel(int kind, const R* __restrict__ fxv, const R* __restrict__ fyv, int ny, int nx, double wx,
                                    double wy, R* __restrict__ out) {
    const long long n = (long long)ny * nx;
    PB_GRID_STRIDE(i, n) {
        const int y = (int)(i / nx), x = (int)(i - (long long)y * nx);
        const double ax = (double)fxv[x] * wx, ay = (double)fyv[y] * wy;
        double v;
        if (kind == 0) v = (ax == 0.0 ? 1.0 : sinpi(ax) / (M_PI * ax)) * (ay == 0.0 ? 1.0 : sinpi(ay) / (M_PI * ay));
        else v = cos(2.0 * ax) * cos(2.0 * ay);
        out[i] = (R)v;
    }
}

}  // namespace pb

using namespace pb;

extern "C" int pb_pack_complex(pb_handle_t hh, int dtype, const void* re, const void* im, const double* im_scale_dev,
                               long long count, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!re || !out) return fail(h, PB_ERR_INVALID, "null pointer");
    if (count <= 0) return PB_OK;
    const int g = grid_for(count, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        pack_complex_kernel<R><<<g, 256, 0, st>>>((const R*)re, (const R*)im, im_scale_dev, count, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_balance_scale(pb_handle_t hh, int dtype, const void* a, const void* b, long long count, double* s_dev,
                                void* stream) {
    PB_ENTER_REAL(hh);
    if (!a || !b || !s_dev || count <= 0) return fail(h, PB_ERR_INVALID, "bad balance arguments");
    const int g = fold_blocks(count, h->sm_count);
    double* part; unsigned* counter;
    PB_TRY(fold_scratch(h, 1, g, 2, st, &part, &counter));
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        balance_kernel<R><<<g, 256, 0, st>>>((const R*)a, (const R*)b, count, part, counter, s_dev);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_packed_spectrum_product(pb_handle_t hh, int dtype, const void* Z, int ny, int nx, double scale,
                                          const double* im_scale_dev, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!Z || !out || ny < 1 || nx < 1 || Z == out) return fail(h, PB_ERR_INVALID, "bad spectrum-product arguments (out must not alias Z)");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        packed_spectrum_product_kernel<R><<<g, 256, 0, st>>>((const cplx<R>*)Z, ny, nx, (R)scale, im_scale_dev, (cplx<R>*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_bindown(pb_handle_t hh, int dtype, const void* in, int ny, int nx, int fy, int fx, int mean, void* out,
                          void* stream) {
    PB_ENTER_REAL(hh);
    if (!in || !out || fy < 1 || fx < 1 || ny < fy || nx < fx || ny % fy || nx % fx)
        return fail(h, PB_ERR_INVALID, "array shape must be a positive integer multiple of the binning factor");
    const int oy = ny / fy, ox = nx / fx;
    const double scale = mean ? 1.0 / ((double)fy * fx) : 1.0;
    const int g = grid_for((long long)oy * ox, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        bindown_kernel<R><<<g, 256, 0, st>>>((const R*)in, oy, ox, fy, fx, (R)scale, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_tile(pb_handle_t hh, int dtype, const void* in, int ny, int nx, int fy, int fx, double scale, void* out,
                       void* stream) {
    PB_ENTER_REAL(hh);
    if (!in || !out || fy < 1 || fx < 1 || ny < 1 || nx < 1) return fail(h, PB_ERR_INVALID, "bad tile arguments");
    const int g = grid_for((long long)ny * fy * nx * fx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        tile_kernel<R><<<g, 256, 0, st>>>((const R*)in, ny, nx, fy, fx, (R)scale, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" int pb_separable_tf(pb_handle_t hh, int dtype, int kind, const void* fx, const void* fy, int ny, int nx, double wx,
                               double wy, void* out, void* stream) {
    PB_ENTER_REAL(hh);
    if (!fx || !fy || !out || ny < 1 || nx < 1 || kind < 0 || kind > 1) return fail(h, PB_ERR_INVALID, "bad transfer-function arguments");
    const int g = grid_for((long long)ny * nx, 256, h->sm_count);
    with_real(dtype, [&](auto r) {
        using R = decltype(r);
        separable_tf_kernel<R><<<g, 256, 0, st>>>(kind, (const R*)fx, (const R*)fy, ny, nx, wx, wy, (R*)out);
    });
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}
