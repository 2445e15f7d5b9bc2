// Generic shared-memory axis pass: any power-of-two length that fits one CTA's shared
// memory, complex64 or complex128, rows or columns.  Hot shapes are taken by the tuned
// register kernels in fft_tuned.cu before this one is reached.
#include "axis_pass.cuh"
#include "fft_tuned.cuh"

namespace pb {

template <typename R>
__device__ __forceinline__ cplx<R> load_input(const AxisPass& p, long long off) {
    using C = cplx<R>;
    if (p.in_kind == PB_IN_COMPLEX) return reinterpret_cast<const C*>(p.in)[off];
    if (p.in_kind == PB_IN_REAL) return mk<R>(reinterpret_cast<const R*>(p.in)[off], R(0));
    // amp * exp(2*pi*i * kturns * opd)
    R a = R(1);
    if (p.amp_kind == PB_AMP_REAL) a = reinterpret_cast<const R*>(p.amp)[off];
    else if (p.amp_kind == PB_AMP_U8) a = reinterpret_cast<const unsigned char*>(p.amp)[off] ? R(1) : R(0);
    if (a == R(0)) return mk<R>(R(0), R(0));
    C e = expi_turns(p.kturns * (double)reinterpret_cast<const R*>(p.in)[off], R(0));
    e.x *= a; e.y *= a;
    return e;
}

template <typename R>
__global__ void __launch_bounds__(512) axis_pass_kernel(const AxisPass p, const int T, const int log2L,
                                                         const cplx<R>* __restrict__ tw) {
    using C = cplx<R>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    C* s = reinterpret_cast<C*>(smem_raw);
    const int L = p.L;
    const int b0 = blockIdx.x * T;
    const int total = T * L;

    // ---- load (pad / rotate / synthesise / pre-multiply), bit-reversed into shared memory
    for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
        int bl, j;
        if (p.batch_contiguous) { bl = idx % T; j = idx / T; } else { j = idx & (L - 1); bl = idx >> log2L; }
        const int b = b0 + bl;
        C v = mk<R>(R(0), R(0));
        if (b < p.nb && j < p.Llog) {
            int pp = j + p.rot_in;
            if (pp >= p.Llog) pp -= p.Llog;
            const int li = pp - p.in_off;
            if (li >= 0 && li < p.n_in) {
                v = load_input<R>(p, (long long)b * p.ibs + (long long)li * p.ies);
                if (p.pre_mat) {
                    C m = reinterpret_cast<const C*>(p.pre_mat)[(long long)b * p.pmi_bs + (long long)li * p.pmi_es];
                    v = p.pre_mat_conj ? cmulc(v, m) : cmul(v, m);
                }
                if (p.pre_e) {
                    C m = reinterpret_cast<const C*>(p.pre_e)[j - p.pre_off];
                    v = p.pre_e_conj ? cmulc(v, m) : cmul(v, m);
                }
                if (p.pre_e2) {
                    C m = reinterpret_cast<const C*>(p.pre_e2)[j - p.pre_off2];
                    v = p.pre_e2_conj ? cmulc(v, m) : cmul(v, m);
                }
                if (p.pre_b) {
                    C m = reinterpret_cast<const C*>(p.pre_b)[b];
                    v = p.pre_b_conj ? cmulc(v, m) : cmul(v, m);
                }
            }
        }
        const int jr = log2L ? (int)(__brev((unsigned)j) >> (32 - log2L)) : 0;
        s[bl * L + jr] = v;
    }
    __syncthreads();

    // ---- in-place decimation-in-time: one radix-2 level if log2L is odd, then radix-4 levels
    const bool inv = p.dir > 0;
    int hh = 1;
    if (log2L & 1) {
        for (int g = threadIdx.x; g < total / 2; g += blockDim.x) {
            C a = s[2 * g], b = s[2 * g + 1];
            s[2 * g] = cadd(a, b);
            s[2 * g + 1] = csub(a, b);
        }
        hh = 2;
        __syncthreads();
    }
    for (; hh < L; hh <<= 2) {
        const int quarter = L >> 2;
        const int st2 = L / (2 * hh), st4 = L / (4 * hh);
        for (int g = threadIdx.x; g < T * quarter; g += blockDim.x) {
            const int bl = g / quarter, gi = g - bl * quarter;
            const int q = gi & (hh - 1), blk = gi / hh;
            C* x = s + bl * L + blk * 4 * hh + q;
            C w1 = tw[q * st2], w2 = tw[q * st4], w3 = tw[(q + hh) * st4];
            if (inv) { w1.y = -w1.y; w2.y = -w2.y; w3.y = -w3.y; }
            C A = x[0], B = x[hh], Cc = x[2 * hh], D = x[3 * hh];
            C t1 = cmul(w1, B), t2 = cmul(w1, D);
            C A1 = cadd(A, t1), B1 = csub(A, t1), C1 = cadd(Cc, t2), D1 = csub(Cc, t2);
            C t3 = cmul(w2, C1), t4 = cmul(w3, D1);
            x[0] = cadd(A1, t3);
            x[2 * hh] = csub(A1, t3);
            x[hh] = cadd(B1, t4);
            x[3 * hh] = csub(B1, t4);
        }
        __syncthreads();
    }

    // ---- store (rotate / crop / post-multiply / |.|^2)
    const R scale = (R)p.scale, weight = (R)p.weight;
    const int tot_out = T * p.n_out;
    const int Lout = p.Llog_out ? p.Llog_out : p.Llog;
    for (int idx = threadIdx.x; idx < tot_out; idx += blockDim.x) {
        int bl, q;
        if (p.batch_contiguous) { bl = idx % T; q = idx / T; } else { q = idx % p.n_out; bl = idx / p.n_out; }
        const int b = b0 + bl;
        if (b >= p.nb) continue;
        int k = q + p.crop_off - p.rot_out;
        if (k < 0) k += Lout;
        if (k >= Lout) k -= Lout;
        C v = s[bl * L + k];
        if (p.post_e) {
            C m = reinterpret_cast<const C*>(p.post_e)[k - p.post_off];
            v = p.post_e_conj ? cmulc(v, m) : cmul(v, m);
        }
        if (p.post_e2) {
            C m = reinterpret_cast<const C*>(p.post_e2)[k - p.post_off2];
            v = p.post_e2_conj ? cmulc(v, m) : cmul(v, m);
        }
        if (p.post_b) {
            C m = reinterpret_cast<const C*>(p.post_b)[b];
            v = p.post_b_conj ? cmulc(v, m) : cmul(v, m);
        }
        if (p.post_mat) {
            C m = reinterpret_cast<const C*>(p.post_mat)[(long long)b * p.pm_bs + (long long)q * p.pm_es];
            v = p.pm_conj ? cmulc(v, m) : cmul(v, m);
        }
        v.x *= scale; v.y *= scale;
        const long long o = (long long)b * p.obs + (long long)q * p.oes;
        if (p.out_kind == PB_OUT_COMPLEX) {
            reinterpret_cast<C*>(p.out)[o] = v;
        } else {
            const R I = v.x * v.x + v.y * v.y;
            R* dst = reinterpret_cast<R*>(p.out) + o;
            if (p.out_kind == PB_OUT_INTENSITY) *dst = I; else *dst += weight * I;
        }
    }
}

static int pow2ceil(int n) { int p = 1; while (p < n) p <<= 1; return p; }

int generic_max_len(const Handle* h, int dtype) {
    const long long cap = h->max_smem_optin, elem = csize(dtype);
    int L = 1;
    while ((long long)2 * L * elem <= cap) L <<= 1;
    return L;
}

template <typename R>
static int launch_generic(Handle* h, const AxisPass& p, cudaStream_t st) {
    const int L = p.L;
    const size_t elem = sizeof(cplx<R>);
    const size_t cap = (size_t)h->max_smem_optin;
    if ((size_t)L * elem > cap)
        return fail(h, PB_ERR_UNSUPPORTED, "FFT length " + std::to_string(L) + " exceeds one CTA's shared memory");
    int T;
    if (p.batch_contiguous) {
        T = 16;
        while (T > 1 && (size_t)T * L * elem > 65536) T >>= 1;
        const int t32 = (int)(32 / elem) ? (int)(32 / elem) : 1;
        if (T < t32 && (size_t)t32 * L * elem <= cap) T = t32;
    } else {
        T = 1;
        while ((long long)T * L < 2048) T <<= 1;
    }
    T = std::min(T, pow2ceil(p.nb));
    if (T < 1) T = 1;
    const size_t smem = (size_t)T * L * elem;
    int threads = (int)std::min<long long>(512, std::max<long long>(32, ((long long)T * L / 4 + 31) / 32 * 32));
    if (smem > 48 * 1024) {
        if (attr_needed(h, reinterpret_cast<const void*>(axis_pass_kernel<R>)))
            PB_CUDA(h, cudaFuncSetAttribute(axis_pass_kernel<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)cap));
    }
    const void* tw = nullptr;
    PB_TRY(get_twiddles(h, L, p.dtype, &tw));
    const int grid = (p.nb + T - 1) / T;
    axis_pass_kernel<R><<<grid, threads, smem, st>>>(p, T, ilog2(L), reinterpret_cast<const cplx<R>*>(tw));
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_AXIS_GENERIC, 0, 0)]++;  // every generic launch
    h->route_launches[route_code(PB_ROUTE_AXIS_GENERIC, L, p.dtype | p.batch_contiguous << 1)]++;
    return PB_OK;
}

int launch_axis_pass(Handle* h, const AxisPass& p, cudaStream_t st) {
    if (!is_pow2(p.L)) return fail(h, PB_ERR_INVALID, "axis pass needs a power-of-two length");
    if (p.nb <= 0 || p.n_out <= 0) return PB_OK;
    int rc = try_tuned_axis_pass(h, p, st);
    if (rc != PB_ERR_UNSUPPORTED) return rc;  // PB_OK or a real error
    if (p.dtype == PB_C64) return launch_generic<float>(h, p, st);
    return launch_generic<double>(h, p, st);
}

}  // namespace pb
