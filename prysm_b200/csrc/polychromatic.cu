// The wavelength loop of an incoherent (polychromatic) PSF as ONE native call.
//
// Reference recipe (docs/source/how-tos/Polychromatic Propagation.ipynb:86-98, prysm/polynomials/fitting.py:37): per
// wavelength  Wavefront.from_amp_and_phase -> prepare_executor(kind='czt') -> focus_dft -> .intensity, then the weighted
// sum.  Through Python that is ~7 library calls, ~10 kernel launches, two temporaries and an event per wavelength for
// a few hundred us of kernels: on a busy host the loop is launch-bound.
// Here the host loop runs inside the library: per unit the Bluestein plan (3 small launches, built from six scalars) is
// issued on the handle's helper stream ONE UNIT AHEAD, the main stream runs phase screen -> row pass -> column pass whose
// store adds weight * |.|^2 to the plane; field, intermediate and the two plan sets live in a caller-supplied work area.
#include "czt.cuh"

namespace pb {
namespace {

int ensure_side(Handle* h) {
    if (!h->side) PB_CUDA(h, cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
    for (auto& e : h->side_ev)
        if (!e) PB_CUDA(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    return PB_OK;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

}  // namespace
}  // namespace pb

using namespace pb;

extern "C" long long pb_polychromatic_czt_work_bytes(int dtype, int n, int m, int K) {
    if ((dtype != PB_C64 && dtype != PB_C128) || n < 1 || m < 1 || K < 1) return 0;
    const size_t cs = csize(dtype);
    return (long long)(align256((size_t)n * n * cs) + align256((size_t)n * m * cs) +
                       2 * (align256((size_t)n * cs) + align256((size_t)m * cs) + 2 * align256((size_t)K * cs)) + 256);
}

extern "C" int pb_polychromatic_czt(pb_handle_t hh, int dtype, const void* amp, int amp_kind, const void* opd, int n, int m,
                                    int K, int n_units, const double* units, void* work, void* plane, void* stream) {
    PB_ENTER_REAL(hh);
    if (n < 1 || m < 1 || K < n + m - 1 || !is_pow2(K) || n_units < 0 || !opd || !work || !plane || (n_units > 0 && !units))
        return fail(h, PB_ERR_INVALID, "bad polychromatic czt arguments");
    if ((uintptr_t)work & 255) return fail(h, PB_ERR_INVALID, "work must be 256-byte aligned");
    if (n_units == 0) return PB_OK;
    PB_TRY(ensure_side(h));
    cudaStream_t sd = h->side;
    cudaEvent_t ev_fork = h->side_ev[0];
    cudaEvent_t ev_plan[2] = {h->side_ev[1], h->side_ev[2]}, ev_used[2] = {h->side_ev[3], h->side_ev[4]};
    const size_t cs = csize(dtype);
    char* w = reinterpret_cast<char*>(work);
    void* field = w;             w += align256((size_t)n * n * cs);
    void* mid = w;               w += align256((size_t)n * m * cs);
    void *b[2], *post[2], *H[2], *hk[2];
    for (int j = 0; j < 2; ++j) {
        b[j] = w;    w += align256((size_t)n * cs);
        post[j] = w; w += align256((size_t)m * cs);
        H[j] = w;    w += align256((size_t)K * cs);
        hk[j] = w;   w += align256((size_t)K * cs);
    }
    // unit record: kscale (phase per unit of OPD), shift, alpha, xc, f0, df, norm, weight
    auto plan = [&](int i) -> int {   // on the helper stream, into buffer set i & 1
        const double* u = units + (size_t)i * 8;
        const int j = i & 1;
        if (i >= 2) PB_CUDA(h, cudaStreamWaitEvent(sd, ev_used[j], 0));   // unit i - 2 has finished reading that set
        PB_TRY(czt_plan_impl(h, hh, dtype, n, m, K, u[1], u[2], -1, u[3], u[4], u[5], b[j], post[j], H[j], nullptr, hk[j], sd));
        PB_CUDA(h, cudaEventRecord(ev_plan[j], sd));
        return PB_OK;
    };
    // fork: the helper stream starts after everything already queued on the caller's stream (the work area may be in use)
    PB_CUDA(h, cudaEventRecord(ev_fork, st));
    PB_CUDA(h, cudaStreamWaitEvent(sd, ev_fork, 0));
    PB_TRY(plan(0));
    const long long count = (long long)n * n;
    for (int i = 0; i < n_units; ++i) {
        const double* u = units + (size_t)i * 8;
        const int j = i & 1;
        if (i + 1 < n_units) PB_TRY(plan(i + 1));
        PB_TRY(pb_phase_screen(hh, dtype, amp, amp_kind, opd, u[0], count, field, stream));
        PB_CUDA(h, cudaStreamWaitEvent(st, ev_plan[j], 0));   // join: every plan is waited for before the call returns
        PB_TRY(czt_axis_impl(h, dtype, field, n, n, n, 1, K, b[j], 0, H[j], post[j], 0, n - 1, m, 1.0, PB_OUT_COMPLEX, 1.0,
                             mid, m, st));
        PB_TRY(czt_axis_impl(h, dtype, mid, n, m, m, 0, K, b[j], 0, H[j], post[j], 0, n - 1, m, u[6], PB_OUT_ACCUMULATE, u[7],
                             plane, m, st));
        PB_CUDA(h, cudaEventRecord(ev_used[j], st));
    }
    return PB_OK;
}
