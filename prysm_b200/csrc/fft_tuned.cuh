// Register-resident FFT kernels for the hot shapes (see fft_tuned.cu).  Each try_* returns
// PB_ERR_UNSUPPORTED *without touching the error string* when the shape is not one it covers;
// the caller then falls through to the generic shared-memory pass.
#pragma once
#include <cmath>
#include "axis_pass.cuh"

namespace pb {

// One pb_fft2 / pb_fft2_batch call, in the order of pb_fft2_batch's arguments: `batch` fields, field b at in + b in_bs,
// amp + b amp_bs and out + b out_bs (strides in elements; pb_fft2 is a batch of one with zero strides)
struct Fft2Args {
    int dtype;
    const void* in; int in_kind; const void* amp; int amp_kind; double kscale;
    int batch; long long in_bs, amp_bs;
    int ny, nx; long long in_ld;
    int ky, kx, dir; double scale; int shift_in, shift_out;
    void* out; int out_kind; double weight; int oy, ox; long long out_ld, out_bs;

    double kturns() const { return kscale / (2.0 * M_PI); }   // phase[turns] = kturns * opd (PB_IN_AMP_OPD)
    size_t in_elt() const { return in_kind == PB_IN_COMPLEX ? 2 * rsize(dtype) : rsize(dtype); }
    size_t out_elt() const { return out_kind == PB_OUT_COMPLEX ? 2 * rsize(dtype) : rsize(dtype); }
    // field b alone, as a batch of one
    Fft2Args field(int b) const {
        Fft2Args f = *this;
        f.batch = 1;
        f.in = reinterpret_cast<const char*>(in) + (size_t)b * in_bs * in_elt();
        if (amp) f.amp = reinterpret_cast<const char*>(amp) + (size_t)b * amp_bs * (amp_kind == PB_AMP_U8 ? 1 : rsize(dtype));
        f.out = reinterpret_cast<char*>(out) + (size_t)b * out_bs * out_elt();
        return f;
    }
};

int try_tuned_axis_pass(Handle* h, const AxisPass& p, cudaStream_t st);

int try_tuned_fft2_batch(Handle* h, const Fft2Args& a, cudaStream_t st);

}  // namespace pb
