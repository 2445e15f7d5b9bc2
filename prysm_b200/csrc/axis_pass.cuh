// One batched 1-D FFT pass along an arbitrary (strided) axis with fused pad / rotate /
// pre- and post-multiplies / crop / |.|^2.  Every 2-D operator of the library is a short
// sequence of these passes.
#pragma once
#include "common.cuh"

namespace pb {

// Logical model, for every batch b in [0, nb):
//   u[j], j in [0, L):   j >= Llog -> 0 ; else p = (j + rot_in) mod Llog,
//                        v = (in_off <= p < in_off + n_in) ? load(b, p - in_off) : 0
//                        u[j] = v * pre_mat(b, p - in_off) * pre_e[j - pre_off] * pre_b[b]   (multipliers optional)
//   U = DFT_L(u) with exp(dir * 2*pi*i*jk/L)
//   out(b, q), q in [0, n_out):  k = (q + crop_off - rot_out) mod Llog
//                        U[k] * post_e[k - post_off] * post_b[b] * post_mat(b, q) * scale
// Llog == L except inside Bluestein, where L is the padded power of two.
struct AxisPass {
    int dtype = PB_C64;
    // input
    const void* in = nullptr;
    int in_kind = PB_IN_COMPLEX;
    const void* amp = nullptr;
    int amp_kind = PB_AMP_NONE;
    double kturns = 0.0;  // phase[turns] = kturns * opd  (PB_IN_AMP_OPD)
    long long ibs = 0, ies = 1;
    int nb = 0;
    int L = 0, Llog = 0;   // Llog: modulus of the input rotation / pad window
    int Llog_out = 0;      // modulus of the output rotation (0 -> same as Llog)
    int n_in = 0, in_off = 0, rot_in = 0;
    const void* pre_e = nullptr; int pre_off = 0; int pre_e_conj = 0;
    const void* pre_e2 = nullptr; int pre_off2 = 0; int pre_e2_conj = 0;
    const void* pre_b = nullptr; int pre_b_conj = 0;
    // full-matrix pre-multiplier, indexed like the input (the between-plane phase screen of a free-space chain)
    const void* pre_mat = nullptr; long long pmi_bs = 0, pmi_es = 0; int pre_mat_conj = 0;
    // transform
    int dir = -1;
    // output
    void* out = nullptr;
    long long obs = 0, oes = 1;
    int n_out = 0, crop_off = 0, rot_out = 0;
    const void* post_e = nullptr; int post_off = 0; int post_e_conj = 0;
    const void* post_e2 = nullptr; int post_off2 = 0; int post_e2_conj = 0;
    const void* post_b = nullptr; int post_b_conj = 0;
    const void* post_mat = nullptr; long long pm_bs = 0, pm_es = 0; int pm_conj = 0;
    double scale = 1.0;
    int out_kind = PB_OUT_COMPLEX;
    double weight = 1.0;
    // mapping hint: 1 when consecutive batches are adjacent in memory (column pass)
    int batch_contiguous = 0;
    // tuned kernels only: forward transform, multiply by post_e/post_b, inverse transform, then crop/store
    // (the column half of a free-space step in one kernel); the generic kernel never sees this flag
    int roundtrip = 0;
};

// Points p at nlines lines of row-major planes with row pitches in_ld and out_ld (elements): axis 1 runs the pass along
// the rows (one line per row), axis 0 along the columns (one line per column, consecutive lines adjacent in memory).
inline void along(AxisPass& p, int axis, int nlines, long long in_ld, long long out_ld) {
    p.nb = nlines;
    if (axis == 1) { p.ibs = in_ld; p.ies = 1; p.obs = out_ld; p.oes = 1; p.batch_contiguous = 0; }
    else { p.ibs = 1; p.ies = in_ld; p.obs = 1; p.oes = out_ld; p.batch_contiguous = 1; }
}

// L must be a power of two here (Bluestein is composed one level up).
int launch_axis_pass(Handle* h, const AxisPass& p, cudaStream_t s);

// Largest power-of-two L the generic pass takes at dtype: one line of L elements must fit one CTA's opt-in shared
// memory (232,448 B on an H100: 16384 complex64 or 8192 complex128 points).
int generic_max_len(const Handle* h, int dtype);

}  // namespace pb
