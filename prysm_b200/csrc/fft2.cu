// 2-D operators composed from axis passes: pb_fft2, pb_fft1, pb_angular_spectrum.
// Arbitrary (non power-of-two) lengths run Bluestein's algorithm on the same pass kernels.
#include <cmath>
#include <complex>

#include "axis_pass.cuh"
#include "fft_tuned.cuh"
#include "czt.cuh"

namespace pb {

static inline int ceil_half(int d) { return (d + 1) / 2; }  // ceil(d/2) for d >= 0

// ---------------------------------------------------------------------------------------
// host-side table builders
// ---------------------------------------------------------------------------------------

static void host_fft_pow2(std::vector<std::complex<double>>& a, int sign) {
    const int n = (int)a.size();
    for (int i = 1, j = 0; i < n; ++i) {
        int bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) std::swap(a[i], a[j]);
    }
    for (int len = 2; len <= n; len <<= 1) {
        for (int i = 0; i < n; i += len)
            for (int k = 0; k < len / 2; ++k) {
                const double ang = sign * 2.0 * M_PI * k / len;
                std::complex<double> w(cos(ang), sin(ang));
                auto u = a[i + k], v = a[i + k + len / 2] * w;
                a[i + k] = u + v;
                a[i + k + len / 2] = u - v;
            }
    }
}

int upload_table(Handle* h, const TwKey& key, const std::vector<std::complex<double>>& t, const void** out) {
    const size_t n = t.size();
    void* d = nullptr;
    PB_CUDA(h, cudaMalloc(&d, n * csize(key.dtype)));
    if (key.dtype == PB_C64) {
        std::vector<float2> f(n);
        for (size_t i = 0; i < n; ++i) f[i] = make_float2((float)t[i].real(), (float)t[i].imag());
        PB_CUDA(h, cudaMemcpy(d, f.data(), n * sizeof(float2), cudaMemcpyHostToDevice));
    } else {
        PB_CUDA(h, cudaMemcpy(d, t.data(), n * sizeof(double2), cudaMemcpyHostToDevice));
    }
    h->tables[key] = d;
    *out = d;
    return PB_OK;
}

int get_twiddles(Handle* h, int n, int dtype, const void** out) {
    return cached_table(h, {n, dtype, TW_ROOTS}, [n](auto& t) {
        t.resize(n);
        for (int k = 0; k < n; ++k) {
            // exact octant symmetry is not needed; long double keeps the table correctly rounded
            const long double ang = -2.0L * 3.14159265358979323846264338327950288L * k / n;
            t[k] = std::complex<double>((double)cosl(ang), (double)sinl(ang));
        }
    }, out);
}

static int bluestein_len(int n) { int m = 1; while (m < 2 * n - 1) m <<= 1; return m; }

// chirp c[j] = exp(dir*pi*i*j^2/n), j^2 reduced mod 2n exactly
static int get_chirp(Handle* h, int n, int dtype, int dir, const void** out) {
    return cached_table(h, {n, dtype, dir < 0 ? TW_CHIRP_FWD : TW_CHIRP_INV}, [n, dir](auto& t) {
        t.resize(n);
        for (int j = 0; j < n; ++j) {
            const long long r = ((long long)j * j) % (2LL * n);
            const long double ang = dir * 3.14159265358979323846264338327950288L * r / n;
            t[j] = std::complex<double>((double)cosl(ang), (double)sinl(ang));
        }
    }, out);
}

// spectrum of the Bluestein filter g[d mod M] = conj(c[|d|]), |d| < n
static int get_chirp_filter(Handle* h, int n, int dtype, int dir, const void** out) {
    return cached_table(h, {n, dtype, dir < 0 ? TW_FILTER_FWD : TW_FILTER_INV}, [n, dir](auto& g) {
        const int M = bluestein_len(n);
        g.assign(M, {0.0, 0.0});
        for (int d = 0; d < n; ++d) {
            const long long r = ((long long)d * d) % (2LL * n);
            const long double ang = -dir * 3.14159265358979323846264338327950288L * r / n;
            std::complex<double> v((double)cosl(ang), (double)sinl(ang));
            g[d] = v;
            if (d) g[M - d] = v;
        }
        host_fft_pow2(g, -1);
    }, out);
}

// ---------------------------------------------------------------------------------------
// one logical DFT pass of arbitrary length p.Llog (p.L is ignored on entry)
// ---------------------------------------------------------------------------------------
static int axis_dft(Handle* h, AxisPass p, cudaStream_t st) {
    const int n = p.Llog;
    // refused before any launch, in terms of the length the caller asked for (Bluestein runs at M ~ 2n)
    const int lmax = generic_max_len(h, p.dtype);
    if (n > lmax || (!is_pow2(n) && bluestein_len(n) > lmax)) {
        const char* name = p.dtype == PB_C64 ? "complex64" : "complex128";
        return fail(h, PB_ERR_UNSUPPORTED,
                    std::string(name) + " FFT of length " + std::to_string(n) + " does not fit one CTA's shared memory (" +
                        std::to_string(h->max_smem_optin) + " B): " + name + " takes any length up to " +
                        std::to_string(lmax / 2) + " and powers of two up to " + std::to_string(lmax));
    }
    if (is_pow2(n)) {
        p.L = n;
        return launch_axis_pass(h, p, st);
    }
    // Bluestein: X[k] = c[k] * IFFT_M( FFT_M(u*c) * G )[k]
    const int M = bluestein_len(n);
    const void *chirp = nullptr, *G = nullptr;
    PB_TRY(get_chirp(h, n, p.dtype, p.dir, &chirp));
    PB_TRY(get_chirp_filter(h, n, p.dtype, p.dir, &G));
    void* tmp = nullptr;
    PB_TRY(ensure_scratch(h, 2, (size_t)p.nb * M * csize(p.dtype), &tmp));

    AxisPass a = p;  // stage 1: chirp-modulated forward FFT_M times the filter spectrum
    a.L = M; a.Llog = n; a.Llog_out = M;
    a.pre_e2 = p.pre_e; a.pre_off2 = p.pre_off; a.pre_e2_conj = p.pre_e_conj;
    a.pre_e = chirp; a.pre_off = 0; a.pre_e_conj = 0;
    if (p.pre_e2) return fail(h, PB_ERR_UNSUPPORTED, "two pre-multipliers on a non power-of-two axis");
    a.dir = -1;
    a.out = tmp; a.n_out = M; a.crop_off = 0; a.rot_out = 0;
    a.obs = p.batch_contiguous ? 1 : M;
    a.oes = p.batch_contiguous ? p.nb : 1;
    a.post_e = G; a.post_off = 0; a.post_e_conj = 0;
    a.post_e2 = nullptr; a.post_b = nullptr; a.post_mat = nullptr;
    a.scale = 1.0; a.out_kind = PB_OUT_COMPLEX;
    PB_TRY(launch_axis_pass(h, a, st));

    AxisPass b = p;  // stage 2: inverse FFT_M, keep k < n, demodulate, user's epilogue
    b.L = M; b.Llog = M; b.Llog_out = n;
    b.in = tmp; b.in_kind = PB_IN_COMPLEX; b.amp = nullptr;
    b.ibs = a.obs; b.ies = a.oes;
    b.n_in = M; b.in_off = 0; b.rot_in = 0;
    b.pre_e = nullptr; b.pre_e2 = nullptr; b.pre_b = nullptr; b.pre_mat = nullptr;
    b.dir = +1;
    if (p.post_e2) return fail(h, PB_ERR_UNSUPPORTED, "two post-multipliers on a non power-of-two axis");
    b.post_e2 = p.post_e; b.post_off2 = p.post_off; b.post_e2_conj = p.post_e_conj;
    b.post_e = chirp; b.post_off = 0; b.post_e_conj = 0;
    b.scale = p.scale / M;
    return launch_axis_pass(h, b, st);
}

// ---------------------------------------------------------------------------------------
// pb_fft2
// ---------------------------------------------------------------------------------------
// one field (a.batch is ignored)
static int fft2_generic(Handle* h, const Fft2Args& a, cudaStream_t st) {
    void* tmp = nullptr;
    PB_TRY(ensure_scratch(h, 0, (size_t)a.ny * a.ox * csize(a.dtype), &tmp));
    AxisPass x;  // rows: only the ny populated rows are transformed (zero rows stay implicit)
    x.dtype = a.dtype;
    x.in = a.in; x.in_kind = a.in_kind; x.amp = a.amp; x.amp_kind = a.amp_kind; x.kturns = a.kturns();
    along(x, 1, a.ny, a.in_ld, a.ox);
    x.Llog = a.kx; x.n_in = a.nx; x.in_off = ceil_half(a.kx - a.nx); x.rot_in = a.shift_in ? a.kx / 2 : 0;
    x.dir = a.dir;
    x.out = tmp;
    x.n_out = a.ox; x.crop_off = ceil_half(a.kx - a.ox); x.rot_out = a.shift_out ? a.kx / 2 : 0;
    PB_TRY(axis_dft(h, x, st));

    AxisPass y;  // columns
    y.dtype = a.dtype;
    y.in = tmp;
    along(y, 0, a.ox, a.ox, a.out_ld);
    y.Llog = a.ky; y.n_in = a.ny; y.in_off = ceil_half(a.ky - a.ny); y.rot_in = a.shift_in ? a.ky / 2 : 0;
    y.dir = a.dir;
    y.out = a.out;
    y.n_out = a.oy; y.crop_off = ceil_half(a.ky - a.oy); y.rot_out = a.shift_out ? a.ky / 2 : 0;
    y.scale = a.scale; y.out_kind = a.out_kind; y.weight = a.weight;
    return axis_dft(h, y, st);
}

// pb_fft2 and pb_fft2_batch after their prologue (handle, dtype, batch >= 1): the fused focus pair where it covers the
// call, else one field at a time through the generic passes
static int fft2_run(Handle* h, const Fft2Args& a, cudaStream_t st) {
    if (a.ny < 1 || a.nx < 1 || a.ky < a.ny || a.kx < a.nx) return fail(h, PB_ERR_INVALID, "need 1 <= n <= k on both axes");
    if (a.oy < 1 || a.ox < 1 || a.oy > a.ky || a.ox > a.kx) return fail(h, PB_ERR_INVALID, "crop window must fit the transform");
    if (a.dir != -1 && a.dir != 1) return fail(h, PB_ERR_INVALID, "dir must be -1 or +1");
    if (!a.in || !a.out) return fail(h, PB_ERR_INVALID, "null array pointer");
    if (a.in_kind < 0 || a.in_kind > 2 || a.out_kind < 0 || a.out_kind > 2) return fail(h, PB_ERR_INVALID, "bad in/out kind");
    if (a.in_ld < a.nx || a.out_ld < a.ox) return fail(h, PB_ERR_INVALID, "row pitch smaller than the row");
    if (a.batch > 1 && (a.in_bs < (long long)(a.ny - 1) * a.in_ld + a.nx || a.out_bs < (long long)(a.oy - 1) * a.out_ld + a.ox))
        return fail(h, PB_ERR_INVALID, "batch stride smaller than one field");
    int rc = try_tuned_fft2_batch(h, a, st);
    if (rc != PB_ERR_UNSUPPORTED) return rc;
    for (int b = 0; b < a.batch; ++b) PB_TRY(fft2_generic(h, a.field(b), st));
    return PB_OK;
}

// pb_fft1 and pb_axis_dft after their prologue: one transform of length n along `axis` of an (ny, nx) plane
static int plane_axis_dft(Handle* h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int n, int dir,
                          double scale, const void* pre_e, int pre_e_conj, const void* pre_b, int pre_b_conj,
                          const void* post_e, int post_e_conj, const void* post_b, int post_b_conj, int out_off,
                          int n_out, void* out, long long out_ld, cudaStream_t st) {
    if (ny < 1 || nx < 1 || n < 1 || (axis != 0 && axis != 1)) return fail(h, PB_ERR_INVALID, "bad shape / axis");
    if (dir != -1 && dir != 1) return fail(h, PB_ERR_INVALID, "dir must be -1 or +1");
    if (out_off < 0 || n_out < 1 || out_off + n_out > n) return fail(h, PB_ERR_INVALID, "output window outside the transform");
    AxisPass p;
    p.dtype = dtype; p.in = in; p.dir = dir; p.scale = scale; p.out = out;
    p.Llog = n; p.n_out = n_out; p.crop_off = out_off;
    p.pre_e = pre_e; p.pre_e_conj = pre_e_conj; p.pre_b = pre_b; p.pre_b_conj = pre_b_conj;
    p.post_e = post_e; p.post_e_conj = post_e_conj; p.post_off = out_off; p.post_b = post_b; p.post_b_conj = post_b_conj;
    along(p, axis, axis == 1 ? ny : nx, in_ld, out_ld);
    p.n_in = std::min(axis == 1 ? nx : ny, n);
    return axis_dft(h, p, st);
}

}  // namespace pb

using namespace pb;

extern "C" int pb_fft2(pb_handle_t hh, int dtype, const void* in, int in_kind, const void* amp, int amp_kind,
                       double kscale, int ny, int nx, long long in_ld, int ky, int kx, int dir, double scale,
                       int shift_in, int shift_out, void* out, int out_kind, double weight, int oy, int ox,
                       long long out_ld, void* stream) {
    PB_ENTER_REAL(hh);
    return fft2_run(h, {dtype, in, in_kind, amp, amp_kind, kscale, 1, 0, 0, ny, nx, in_ld, ky, kx, dir, scale, shift_in,
                        shift_out, out, out_kind, weight, oy, ox, out_ld, 0}, st);
}

extern "C" int pb_fft2_batch(pb_handle_t hh, int dtype, const void* in, int in_kind, const void* amp, int amp_kind,
                             double kscale, int batch, long long in_bs, long long amp_bs, int ny, int nx, long long in_ld,
                             int ky, int kx, int dir, double scale, int shift_in, int shift_out, void* out, int out_kind,
                             double weight, int oy, int ox, long long out_ld, long long out_bs, void* stream) {
    PB_ENTER(hh);
    if (batch < 1) return fail(h, PB_ERR_INVALID, "batch must be >= 1");
    if (dtype != PB_C64 && dtype != PB_C128) return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    return fft2_run(h, {dtype, in, in_kind, amp, amp_kind, kscale, batch, in_bs, amp_bs, ny, nx, in_ld, ky, kx, dir, scale,
                        shift_in, shift_out, out, out_kind, weight, oy, ox, out_ld, out_bs},
                    reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int pb_fft1(pb_handle_t hh, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int n,
                       int dir, double scale, void* out, long long out_ld, void* stream) {
    PB_ENTER_REAL(hh);
    return plane_axis_dft(h, dtype, in, ny, nx, in_ld, axis, n, dir, scale, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0,
                          0, n, out, out_ld, st);
}

extern "C" int pb_axis_dft(pb_handle_t hh, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int n,
                           int dir, double scale, const void* pre_e, int pre_e_conj, const void* pre_b, int pre_b_conj,
                           const void* post_e, int post_e_conj, const void* post_b, int post_b_conj, int out_off,
                           int n_out, void* out, long long out_ld, void* stream) {
    PB_ENTER_REAL(hh);
    return plane_axis_dft(h, dtype, in, ny, nx, in_ld, axis, n, dir, scale, pre_e, pre_e_conj, pre_b, pre_b_conj, post_e,
                          post_e_conj, post_b, post_b_conj, out_off, n_out, out, out_ld, st);
}

int pb::czt_axis_impl(Handle* h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int K,
                         const void* pre_e, int pre_conj, const void* H, const void* post_e, int post_conj, int out_off,
                         int n_out, double scale, int out_kind, double weight, void* out, long long out_ld, cudaStream_t st) {
    if (ny < 1 || nx < 1 || K < 1 || (axis != 0 && axis != 1) || !H) return fail(h, PB_ERR_INVALID, "bad czt arguments");
    if (out_off < 0 || n_out < 1 || out_off + n_out > K) return fail(h, PB_ERR_INVALID, "output window outside the transform");
    if (!is_pow2(K)) return fail(h, PB_ERR_INVALID, "the Bluestein length K must be a power of two");
    const int nline = axis == 1 ? ny : nx, n_in = std::min(axis == 1 ? nx : ny, K);
    AxisPass f;  // fused: (in * pre) -> FFT_K -> * H -> IFFT_K -> window -> * post
    f.dtype = dtype; f.in = in; f.dir = -1; f.out = out; f.scale = scale / K;
    f.L = K; f.Llog = K; f.n_in = n_in; f.n_out = n_out; f.crop_off = out_off;
    f.pre_e = pre_e; f.pre_e_conj = pre_conj;
    f.post_e = H;
    f.post_e2 = post_e; f.post_e2_conj = post_conj;
    along(f, axis, nline, in_ld, out_ld);
    f.roundtrip = 1;
    f.out_kind = out_kind; f.weight = weight;
    int rc = try_tuned_axis_pass(h, f, st);
    if (rc != PB_ERR_UNSUPPORTED) return rc;
    // two passes through a (lines x K) scratch: K-element rows along axis 1, nline-element rows along axis 0
    void* tmp = nullptr;
    PB_TRY(ensure_scratch(h, 1, (size_t)nline * K * csize(dtype), &tmp));
    const long long tmp_ld = axis == 1 ? K : nline;
    AxisPass a = f;
    a.roundtrip = 0; a.post_e2 = nullptr; a.out = tmp; a.n_out = K; a.crop_off = 0; a.scale = 1.0;
    a.out_kind = PB_OUT_COMPLEX; a.weight = 1.0;
    along(a, axis, nline, in_ld, tmp_ld);
    PB_TRY(axis_dft(h, a, st));
    AxisPass b;
    b.dtype = dtype; b.in = tmp; b.dir = +1; b.out = out; b.scale = scale / K;
    b.Llog = K; b.n_in = K; b.n_out = n_out; b.crop_off = out_off;
    b.post_e = post_e; b.post_e_conj = post_conj; b.post_off = out_off;
    along(b, axis, nline, tmp_ld, out_ld);
    b.out_kind = out_kind; b.weight = weight;
    return axis_dft(h, b, st);
}

extern "C" int pb_czt_axis(pb_handle_t hh, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int K,
                           const void* pre_e, int pre_conj, const void* H, const void* post_e, int post_conj, int out_off,
                           int n_out, double scale, void* out, long long out_ld, void* stream) {
    PB_ENTER_REAL(hh);
    return czt_axis_impl(h, dtype, in, ny, nx, in_ld, axis, K, pre_e, pre_conj, H, post_e, post_conj, out_off, n_out, scale,
                         PB_OUT_COMPLEX, 1.0, out, out_ld, st);
}

extern "C" int pb_czt_axis_intensity(pb_handle_t hh, int dtype, const void* in, int ny, int nx, long long in_ld, int axis,
                                     int K, const void* pre_e, int pre_conj, const void* H, const void* post_e,
                                     int post_conj, int out_off, int n_out, double scale, int out_kind, double weight,
                                     void* out, long long out_ld, void* stream) {
    PB_ENTER(hh);
    if (out_kind != PB_OUT_INTENSITY && out_kind != PB_OUT_ACCUMULATE) return fail(h, PB_ERR_INVALID, "out_kind must be intensity or accumulate");
    if (dtype != PB_C64 && dtype != PB_C128) return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    return czt_axis_impl(h, dtype, in, ny, nx, in_ld, axis, K, pre_e, pre_conj, H, post_e, post_conj, out_off, n_out, scale,
                         out_kind, weight, out, out_ld, reinterpret_cast<cudaStream_t>(stream));
}

// dtype is checked by the entry points
static int angular_spectrum_impl(Handle* h, int dtype, const void* in, int ny, int nx, int ky, int kx, const void* ty,
                                 const void* tx, const void* tf, int conj_tf, const void* screen, int conj_screen, void* out,
                                 int oy, int ox, cudaStream_t st) {
    if (ny < 1 || nx < 1 || ky < ny || kx < nx || oy < 1 || ox < 1 || oy > ky || ox > kx)
        return fail(h, PB_ERR_INVALID, "bad shapes");
    if (!tf && (!ty || !tx)) return fail(h, PB_ERR_INVALID, "need tf or both ty and tx");

    const size_t cs = csize(dtype);
    void *t0 = nullptr, *t1 = nullptr;
    PB_TRY(ensure_scratch(h, 0, (size_t)ky * kx * cs, &t0));
    PB_TRY(ensure_scratch(h, 1, (size_t)ky * kx * cs, &t1));
    AxisPass p;  // rows forward (times the phase screen, if any): ny populated rows -> t0 (ny, kx)
    p.dtype = dtype; p.in = in;
    along(p, 1, ny, nx, kx);
    p.pre_mat = screen; p.pmi_bs = nx; p.pmi_es = 1; p.pre_mat_conj = conj_screen;
    p.Llog = kx; p.n_in = nx; p.in_off = ceil_half(kx - nx);
    p.dir = -1; p.out = t0; p.n_out = kx;
    PB_TRY(axis_dft(h, p, st));
    bool fused = false;
    if (!tf && dtype == PB_C64 && is_pow2(ky)) {  // separable TF: forward * TF * inverse along y in ONE tuned pass, if it is covered
        AxisPass f;  // -> t1 (oy, kx)
        f.dtype = dtype; f.in = t0;
        along(f, 0, kx, kx, kx);
        f.L = ky; f.Llog = ky; f.n_in = ny; f.in_off = ceil_half(ky - ny);
        f.dir = -1; f.out = t1; f.n_out = oy; f.crop_off = ceil_half(ky - oy);
        f.post_e = ty; f.post_e_conj = conj_tf; f.post_b = tx; f.post_b_conj = conj_tf;
        f.roundtrip = 1;
        const int frc = try_tuned_axis_pass(h, f, st);
        if (frc != PB_OK && frc != PB_ERR_UNSUPPORTED) return frc;
        fused = frc == PB_OK;
    }
    if (!fused) {
        AxisPass q;  // columns forward, times the transfer function -> t1 (ky, kx)
        q.dtype = dtype; q.in = t0;
        along(q, 0, kx, kx, kx);
        q.Llog = ky; q.n_in = ny; q.in_off = ceil_half(ky - ny);
        q.dir = -1; q.out = t1; q.n_out = ky;
        if (tf) { q.post_mat = tf; q.pm_bs = 1; q.pm_es = kx; q.pm_conj = conj_tf; }
        else { q.post_e = ty; q.post_e_conj = conj_tf; q.post_b = tx; q.post_b_conj = conj_tf; }
        PB_TRY(axis_dft(h, q, st));
        AxisPass r;  // columns inverse, keep the oy centred rows -> t0 (oy, kx)
        r.dtype = dtype; r.in = t1;
        along(r, 0, kx, kx, kx);
        r.Llog = ky; r.n_in = ky; r.dir = +1;
        r.out = t0; r.n_out = oy; r.crop_off = ceil_half(ky - oy);
        PB_TRY(axis_dft(h, r, st));
    }
    AxisPass s;  // rows inverse from the (oy, kx) result of the column passes, keep the ox centred columns, 1/(ky*kx)
    s.dtype = dtype; s.in = fused ? t1 : t0;
    along(s, 1, oy, kx, ox);
    s.Llog = kx; s.n_in = kx; s.dir = +1;
    s.out = out; s.n_out = ox; s.crop_off = ceil_half(kx - ox);
    s.scale = 1.0 / ((double)ky * (double)kx);
    return axis_dft(h, s, st);
}

extern "C" int pb_angular_spectrum(pb_handle_t hh, int dtype, const void* in, int ny, int nx, int ky, int kx,
                                   const void* ty, const void* tx, const void* tf, int conj_tf, void* out, int oy,
                                   int ox, void* stream) {
    PB_ENTER_REAL(hh);
    return angular_spectrum_impl(h, dtype, in, ny, nx, ky, kx, ty, tx, tf, conj_tf, nullptr, 0, out, oy, ox, st);
}

extern "C" int pb_angular_spectrum_screen(pb_handle_t hh, int dtype, const void* in, const void* screen, int conj_screen,
                                          int ny, int nx, int ky, int kx, const void* ty, const void* tx, const void* tf,
                                          int conj_tf, void* out, int oy, int ox, void* stream) {
    PB_ENTER(hh);
    if (!screen) return fail(h, PB_ERR_INVALID, "null screen");
    if (dtype != PB_C64 && dtype != PB_C128) return fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128");
    return angular_spectrum_impl(h, dtype, in, ny, nx, ky, kx, ty, tx, tf, conj_tf, screen, conj_screen, out, oy, ox,
                                 reinterpret_cast<cudaStream_t>(stream));
}
