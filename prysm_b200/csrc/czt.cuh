// Internal pieces of the chirp-z path shared between translation units (elementwise.cu, fft2.cu, polychromatic.cu).
#pragma once
#include "common.cuh"

namespace pb {

// pb_czt_plan with the K-element work vector `hk` supplied by the caller (the entry point takes it from scratch slot 2);
// Hadj may be null (forward-only use)
int czt_plan_impl(Handle* h, pb_handle_t hh, int dtype, int N, int M, int K, double shift, double alpha, int sign, double xc,
                  double f0, double df, void* b, void* post, void* H, void* Hadj, void* hk, void* stream);

// one fused Bluestein axis (pb_czt_axis / pb_czt_axis_intensity); dtype is checked by the caller
int czt_axis_impl(Handle* h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int K,
                  const void* pre_e, int pre_conj, const void* H, const void* post_e, int post_conj, int out_off,
                  int n_out, double scale, int out_kind, double weight, void* out, long long out_ld, cudaStream_t st);

}  // namespace pb
