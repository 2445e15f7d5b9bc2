/*
 * prysm_b200.h -- C ABI of the H100-native (sm_90a) propagation engine (libprysm_b200.so).
 *
 * This is the drop-in boundary for the prysm hot path (prysm.propagation + prysm.fttools +
 * the psf/otf reductions, reference v0.22).  The reference has no FFI of its own: its plug-in
 * surface is the Python module shim in prysm/mathops.py:11-116.  Each entry point below
 * states the reference call it replaces (paths relative to the reference tree).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes only.  All array pointers are DEVICE pointers owned
 *     by the caller (row-major, index order [y][x], interleaved complex) unless a parameter is
 *     documented as "host".  The library owns only the opaque handle (twiddle tables, scratch).
 *   - Every call is asynchronous on the `stream` argument (a cudaStream_t passed as void*;
 *     NULL = legacy default stream).  A handle is bound to one device and is not thread-safe.
 *   - Return value: PB_OK (0) or a negative pb_status; pb_last_error(h) gives the message.
 *     Nothing throws or exits across this boundary.  There is no CPU fallback.
 *   - dtype selects the working precision like prysm.conf.config.precision
 *     (prysm/conf.py:28-96): PB_C64 = complex64 fields / float32 reals, PB_C128 = complex128 /
 *     float64.
 */
#ifndef PRYSM_B200_H
#define PRYSM_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pb_handle_s* pb_handle_t;

typedef enum { PB_C64 = 0, PB_C128 = 1 } pb_dtype;

/* the element type of typed storage (frames, mosaics, Jones sources, slopes) in the entry points that take one */
typedef enum {
    PB_ELEM_F32 = 0, PB_ELEM_F64 = 1, PB_ELEM_C64 = 2, PB_ELEM_C128 = 3, PB_ELEM_U8 = 4, PB_ELEM_U16 = 5, PB_ELEM_U32 = 6,
    PB_ELEM_I32 = 7, PB_ELEM_I64 = 8
} pb_elem;

typedef enum {
    PB_OK = 0,
    PB_ERR_INVALID = -1,      /* bad argument */
    PB_ERR_UNSUPPORTED = -2,  /* shape / length outside what the kernels cover */
    PB_ERR_CUDA = -3,         /* CUDA runtime error (message has the cudaError string) */
    PB_ERR_ALLOC = -4
} pb_status;

/* how the input field of pb_fft2 is presented */
typedef enum {
    PB_IN_COMPLEX = 0,  /* in = complex (ny, nx) */
    PB_IN_REAL = 1,     /* in = real (ny, nx), imaginary part 0 (prysm/otf.py:31 takes a real PSF) */
    PB_IN_AMP_OPD = 2   /* field = amp * exp(i*kscale*opd): prysm/propagation/wavefront.py:59-79 fused in */
} pb_in_kind;

typedef enum { PB_AMP_NONE = 0, PB_AMP_REAL = 1, PB_AMP_U8 = 2 } pb_amp_kind;

typedef enum {
    PB_OUT_COMPLEX = 0,    /* complex field */
    PB_OUT_INTENSITY = 1,  /* re^2+im^2 (prysm/propagation/wavefront.py:147-151) into a real array */
    PB_OUT_ACCUMULATE = 2  /* out += weight*(re^2+im^2): the per-wavelength term of
                              prysm/polynomials/fitting.py:37 applied as it is produced */
} pb_out_kind;

/* ---- lifetime ------------------------------------------------------------------------ */
int pb_create(pb_handle_t* out, int device);
int pb_destroy(pb_handle_t h);
const char* pb_last_error(pb_handle_t h);
const char* pb_version(void);
/* number of kernels this handle has launched since creation (bench.py's gpu_launches) */
long long pb_launch_count(pb_handle_t h);
/* number of kernels this handle has launched on one route of the transform kernels, so that a caller (the test suite)
 * can tell which specialisation a call ran.  route = kind << 28 | L << 8 | flags:
 *   PB_ROUTE_AXIS_REG     axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE>; flags INV | COLS << 1 | RT << 2 | PM << 3 |
 *                         DENSE << 4
 *   PB_ROUTE_AXIS_GENERIC the generic shared-memory axis pass: every launch on L = 0, flags = 0, and each launch also
 *                         on its power-of-two length L, flags DTYPE | COLS << 1 (DTYPE: PB_C64 / PB_C128; COLS: a
 *                         column pass, consecutive lines adjacent in memory).  A Bluestein axis is two launches at its
 *                         padded length.
 *   PB_ROUTE_FOCUS_V2     focus_col4_kernel / focus_row4_kernel of N = L; flags INV (two kernels per field)
 *   PB_ROUTE_MDFT_TC      wgmma_gemm_kernel of the tensor-core matrix DFT; L = split-K pieces (1 when not split);
 *                         flags STREAMK | STAGE2 << 1 | PARTIALS << 2 (PARTIALS: writes split-K partial planes)
 *   PB_ROUTE_MDFT_REDUCE  reduce_splits_kernel, the sum of the split-K partial planes; L = pieces, flags = 0
 *   PB_ROUTE_CGEMM        cgemm_kernel<R, OPA, OPB> of the CUDA-core GEMM (pb_cgemm, pb_mdft_apply); L = 0,
 *                         flags DTYPE | OPA << 1 | OPB << 3 (DTYPE: PB_C64 / PB_C128; OP as in pb_cgemm)
 *   PB_ROUTE_CENTROID     centroid_kernel<T, O, V> of pb_subaperture_centroids; L = V (grid columns per thread: 4, or
 *                         1 for a row length or frame alignment that rules out vector loads, or more than 614 lenslet
 *                         columns), flags = the frame's pb_elem_type
 *   PB_ROUTE_PSI          psi_kernel of pb_psi; L = V (samples per thread: 16 / element size, or 1 for a misaligned
 *                         frame or output or an n that is not a multiple of it), flags = 1 for int64 sums, else 0
 * The key is a 32-bit int: kinds 8 and up set its sign bit.  Returns -1 for a NULL handle. */
typedef enum {
    PB_ROUTE_AXIS_REG = 1,
    PB_ROUTE_AXIS_GENERIC = 2,
    /* 3 is retired: it counted a second focus pair, since removed */
    PB_ROUTE_FOCUS_V2 = 4,
    PB_ROUTE_MDFT_TC = 5,
    PB_ROUTE_MDFT_REDUCE = 6,
    PB_ROUTE_CGEMM = 7,
    PB_ROUTE_CENTROID = 8,
    PB_ROUTE_PSI = 9
} pb_route_kind;
long long pb_route_launch_count(pb_handle_t h, int route);

/* ---- centred / plain 2-D FFT with fused pad, shifts, synthesis and |.|^2 ---------------
 * out = crop( S_out( FFT2_{dir}( S_in( pad( field ) ) ) ) ) * scale
 *   field : (ny, nx), see pb_in_kind; row pitch in_ld elements
 *   pad   : centred zero pad to (ky, kx) with the pad2d offset rule ceil((k-n)/2)
 *           (prysm/fttools.py:43-100)
 *   S_in  : ifftshift if shift_in, S_out: fftshift if shift_out (all axes)
 *   dir   : -1 forward (exp(-i..)), +1 inverse; scale is applied by the caller's norm rule
 *           (ortho: 1/sqrt(ky*kx); numpy default: 1 forward, 1/(ky*kx) inverse)
 *   crop  : centred (oy, ox) window with the crop_center rule (prysm/fttools.py:103-125)
 * Replaces: propagation.focus / unfocus and their adjoints (prysm/propagation/fft.py:7-85),
 *           fft.fft2 / ifft2 call sites (prysm/otf.py:31,59), Wavefront.from_amp_and_phase +
 *           .focus + .intensity chains (prysm/propagation/wavefront.py:59-79,147-151,478-504).
 * Any ky, kx >= 1 is accepted (non powers of two run Bluestein on the same kernels). */
int pb_fft2(pb_handle_t h, int dtype,
            const void* in, int in_kind, const void* amp, int amp_kind, double kscale,
            int ny, int nx, long long in_ld,
            int ky, int kx, int dir, double scale, int shift_in, int shift_out,
            void* out, int out_kind, double weight, int oy, int ox, long long out_ld,
            void* stream);
/* pb_fft2 over `batch` independent fields in one call: field b starts at in + b*in_bs, amp + b*amp_bs (0 = one
 * amplitude shared by all) and out + b*out_bs, strides in elements of the respective array's scalar type.  On the
 * fused focus shapes the fields share launches (eight per launch pair by default), which evens out the 3.46-wave
 * column pass and the 9.2-round row pass of a single 2048^2 field; other shapes run field by field.  The reference
 * has no batch form: fft.py:7-25 is called once per wavefront. */
int pb_fft2_batch(pb_handle_t h, int dtype, const void* in, int in_kind, const void* amp, int amp_kind,
                  double kscale, int batch, long long in_bs, long long amp_bs, int ny, int nx,
                  long long in_ld, int ky, int kx, int dir, double scale, int shift_in, int shift_out,
                  void* out, int out_kind, double weight, int oy, int ox, long long out_ld,
                  long long out_bs, void* stream);

/* ---- 1-D FFT along one axis of a 2-D array, numpy fft(a, n, axis) semantics ------------
 * Zero-extends or truncates to n along `axis` (0 = y/columns, 1 = x/rows).
 * Replaces fft.fft / fft.ifft call sites in prysm/fttools.py:301-321, 519-533. */
int pb_fft1(pb_handle_t h, int dtype, const void* in, int ny, int nx, long long in_ld,
            int axis, int n, int dir, double scale, void* out, long long out_ld, void* stream);

/* ---- the same, with fused multipliers and an output window -----------------------------
 * For every line b along `axis`:  u[j] = in_line[j] * pre_e[j] * pre_b[b]   (j < n_line, zero-extended to n)
 *                                 U = DFT_n(u);   out_line[q] = U[q + out_off] * post_e[q] * post_b[b] * scale
 * for q in [0, n_out).  Any multiplier may be NULL; *_conj conjugates it.  pre_e has n_line
 * entries, post_e has n_out entries, pre_b / post_b have one entry per line.
 * One call is one Bluestein half-step of CZT (prysm/fttools.py:298-324) or one FFTDFT axis
 * (prysm/fttools.py:443-459) with the chirp / ramp multiplies and the slice fused in. */
int pb_axis_dft(pb_handle_t h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis,
                int n, int dir, double scale,
                const void* pre_e, int pre_e_conj, const void* pre_b, int pre_b_conj,
                const void* post_e, int post_e_conj, const void* post_b, int post_b_conj,
                int out_off, int n_out, void* out, long long out_ld, void* stream);

/* ---- one Bluestein axis of the chirp-z transform, fused -----------------------------------
 * For every line along `axis`:  u = line * pre_e (zero-extended to K);  c = IFFT_K( FFT_K(u) * H );
 * out_line[q] = c[q + out_off] * post_e[q] * scale,  q in [0, n_out).   K must be a power of two.
 * On the tuned path the data stays in registers between the two transforms (one kernel, one read and one
 * write of the array).  Replaces the per-axis block of CZT.__call__ / adjoint, prysm/fttools.py:296-361. */
int pb_czt_axis(pb_handle_t h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int K,
                const void* pre_e, int pre_conj, const void* H, const void* post_e, int post_conj,
                int out_off, int n_out, double scale, void* out, long long out_ld, void* stream);

/* The same axis with the modulus fused into its store: out_kind = PB_OUT_INTENSITY writes |.|^2 (a REAL array),
 * PB_OUT_ACCUMULATE adds weight * |.|^2 to it -- the last pass of one wavelength of an incoherent sum never writes its
 * complex field.  Replaces the last axis of CZT.__call__ (prysm/fttools.py:296-325) followed by Wavefront.intensity
 * (prysm/propagation/wavefront.py:147-151) and the running term of sum_of_2d_modes (prysm/polynomials/fitting.py:37). */
int pb_czt_axis_intensity(pb_handle_t h, int dtype, const void* in, int ny, int nx, long long in_ld, int axis, int K,
                          const void* pre_e, int pre_conj, const void* H, const void* post_e, int post_conj,
                          int out_off, int n_out, double scale, int out_kind, double weight, void* out,
                          long long out_ld, void* stream);

/* ---- the wavelength loop of an incoherent (polychromatic) PSF as one call -------------------------------------
 * plane(m,m) += sum_i weight_i * | CZT_i( amp * exp(i * kscale_i * opd) ) |^2  over n_units wavelengths of a square n x n
 * pupil on a common square m x m focal grid.  Replaces, per wavelength, Wavefront.from_amp_and_phase
 * (prysm/propagation/wavefront.py:59-79) -> prepare_executor(kind='czt') (propagation/dft.py:69-117, fttools.py:257-291)
 * -> focus_dft (fttools.py:296-325) -> .intensity (wavefront.py:147-151) and the running weighted sum of
 * sum_of_2d_modes (polynomials/fitting.py:37) -- the loop of docs/source/how-tos/Polychromatic Propagation.ipynb:86-98.
 * units: n_units records of 8 doubles on the HOST: kscale (phase per unit of opd), then the pb_czt_plan scalars shift,
 * alpha, xc, f0, df of the (square, centred) geometry, the executor norm, the weight.  K: Bluestein length, a power of
 * two >= n + m - 1.  The plan of unit i+1 is built on the handle's helper stream while unit i transforms.
 * work: pb_polychromatic_czt_work_bytes(dtype, n, m, K) bytes, 256-byte aligned.  plane: real (float / double). */
long long pb_polychromatic_czt_work_bytes(int dtype, int n, int m, int K);
int pb_polychromatic_czt(pb_handle_t h, int dtype, const void* amp, int amp_kind, const void* opd, int n, int m, int K,
                         int n_units, const double* units, void* work, void* plane, void* stream);

/* The Bluestein pieces of one CZT axis built on the device from scalars (no host maths, no uploads):
 * b (N), post = a*phase (M), H = FFT_K(h) (K), Hadj (K) as consumed by pb_czt_axis.  alpha = dx*dfx,
 * shift = f[M/2]/df, xc = x[N/2], f0 = f[0], df the frequency step.  prysm/fttools.py:257-291, 372-389 */
int pb_czt_plan(pb_handle_t h, int dtype, int N, int M, int K, double shift, double alpha, int sign,
                double xc, double f0, double df, void* b, void* post, void* H, void* Hadj, void* stream);

/* ---- angular spectrum ------------------------------------------------------------------
 * out(ky,kx) = ifft2( fft2( pad(in -> ky,kx) ) * TF ), TF = outer(ty, tx) when tf == NULL,
 * else the full (ky,kx) array tf; conj_tf applies conj(TF) (adjoint); the result is cropped to
 * (oy, ox) with the crop_center rule (forward: oy=ky, ox=kx i.e. stays padded).
 * Replaces prysm/propagation/angular_spectrum.py:9-79. */
int pb_angular_spectrum(pb_handle_t h, int dtype, const void* in, int ny, int nx,
                        int ky, int kx, const void* ty, const void* tx, const void* tf,
                        int conj_tf, void* out, int oy, int ox, void* stream);

/* The same with the field multiplied by a complex (ny,nx) `screen` (conj_screen: by its conjugate) inside the first
 * transform pass: one step `wf = (wf * screen).free_space(dz)` of a plane-to-plane chain without the separate
 * elementwise pass.  Replaces prysm/propagation/wavefront.py:360-383 (Wavefront.__mul__) followed by
 * prysm/propagation/angular_spectrum.py:9-42. */
int pb_angular_spectrum_screen(pb_handle_t h, int dtype, const void* in, const void* screen, int conj_screen,
                               int ny, int nx, int ky, int kx, const void* ty, const void* tx, const void* tf,
                               int conj_tf, void* out, int oy, int ox, void* stream);

/* the two separable factors exp(-i*pi*wvl_mm*z*k^2), k = fftfreq(n, dx) rounded to the working
 * precision first (prysm/propagation/angular_spectrum.py:102-113).  ty: ky values, tx: kx. */
int pb_angular_spectrum_vectors(pb_handle_t h, int dtype, int ky, int kx, double wvl_um,
                                double dx_mm, double z_mm, void* ty, void* tx, void* stream);

/* ---- matrix DFT ------------------------------------------------------------------------
 * basis E[j,l] = exp(sign*2*pi*i*f[j]*x[l]), (m, n) complex.  f, x: HOST double arrays.
 * The phase is formed and range-reduced in fp64 before the sincos.  prysm/fttools.py:187-191 */
int pb_mdft_basis(pb_handle_t h, int dtype, const double* f_host, int m, const double* x_host,
                  int n, int sign, void* E, void* stream);

/* C(m,n) = alpha * opA(A) * opB(B); op (pb_op): PB_OP_N as is, PB_OP_T transpose, PB_OP_H conjugate transpose,
 * PB_OP_C conjugate.  A is (m,k) after op, B is (k,n) after op.  Complex, row-major.
 * Replaces the `@` chains of MDFT.__call__ / adjoint (prysm/fttools.py:201-228). */
typedef enum { PB_OP_N = 0, PB_OP_T = 1, PB_OP_H = 2, PB_OP_C = 3 } pb_op;
int pb_cgemm(pb_handle_t h, int dtype, int opA, int opB, int m, int n, int k, double alpha,
             const void* A, long long lda, const void* B, long long ldb, void* C, long long ldc,
             void* stream);

/* out(my,mx) = norm * Ey(my,ny) @ a(ny,nx) @ Ex(mx,nx)^T   (adjoint = 0), or
 * out(ny,nx) = norm * Ey^H @ g(my,mx) @ conj(Ex)            (adjoint = 1),
 * association order chosen by left_first (prysm/fttools.py:198-228).  `work` is caller scratch
 * of at least pb_mdft_work_elems(...) complex elements. */
int pb_mdft_apply(pb_handle_t h, int dtype, const void* Ey, const void* Ex, int my, int ny,
                  int mx, int nx, const void* a, void* out, double norm, int adjoint,
                  int left_first, void* work, void* stream);
long long pb_mdft_work_elems(int my, int ny, int mx, int nx, int adjoint, int left_first);

/* ---- matrix DFT on the wgmma tensor cores (complex64, forward) -------------------------
 * 3xTF32 split (fp32-accurate) real embedding of the complex product; see csrc/mdft_tc.cu.
 *   pb_mdft_tc_supported : 1 when (my, ny, mx, nx) is covered (multiples of 128 / 128 / 128 / 16)
 *   pb_mdft_tc_expand    : complex basis E (m,n) -> real expansions hi, lo, each (2m, 2n) fp32;
 *                          done once per executor for Ex and for Ey (prysm/fttools.py:187-191)
 *   pb_mdft_tc_apply     : out(my,mx) = norm * Ey @ a @ Ex^T   (prysm/fttools.py:201-207);
 *                          work: pb_mdft_tc_work_bytes() bytes of 16-byte aligned device scratch (the transposed
 *                          intermediate, split-K partial planes, and the partial tiles + flags of the stream-K form
 *                          that under-filled tile grids take) */
int pb_mdft_tc_supported(int my, int ny, int mx, int nx);
int pb_mdft_tc_expand(pb_handle_t h, const void* E, int m, int n, void* hi, void* lo, void* stream);
long long pb_mdft_tc_work_bytes(int my, int ny, int mx, int nx);
int pb_mdft_tc_apply(pb_handle_t h, const void* ExB_hi, const void* ExB_lo, const void* EyB_hi,
                     const void* EyB_lo, int my, int ny, int mx, int nx, const void* a, void* out,
                     double norm, void* work, void* stream);

/* ---- elementwise / reductions -----------------------------------------------------------
 * out = amp * exp(i*kscale*opd)   (amp optional).  prysm/propagation/wavefront.py:59-96 */
int pb_phase_screen(pb_handle_t h, int dtype, const void* amp, int amp_kind, const void* opd,
                    double kscale, long long count, void* out, void* stream);
/* out (+)= weight * |in|^2.  prysm/propagation/wavefront.py:147-151 */
int pb_intensity(pb_handle_t h, int dtype, const void* in, long long count, double weight,
                 int accumulate, void* out, void* stream);
/* out = a (op) b elementwise on complex arrays; b == NULL uses the scalar (s_re, s_im) instead;
 * reverse swaps the operands.  op: 0 mul, 1 div, 2 add, 3 sub.
 * Wavefront.__numerical_operation__ (prysm/propagation/wavefront.py:360-411). */
int pb_binary(pb_handle_t h, int dtype, int op, const void* a, const void* b, double s_re,
              double s_im, int reverse, long long count, void* out, void* stream);
/* out[y,x] = in[y,x] * vy[y] * vx[x] * scale (either vector may be NULL; conj flags per vector).
 * The chirp / phase-ramp multiplies of CZT and FFTDFT (prysm/fttools.py:298-324, 443-459). */
int pb_mul_outer(pb_handle_t h, int dtype, const void* in, long long in_ld, int ny, int nx,
                 const void* vy, int conj_y, const void* vx, int conj_x, double scale, void* out,
                 long long out_ld, void* stream);
/* out(n) = sum_k weights[k] * modes[k][n]; weights: HOST doubles.  prysm/polynomials/fitting.py:37 */
int pb_weighted_sum(pb_handle_t h, int dtype, const void* modes, int k, long long count,
                    const double* weights_host, void* out, void* stream);
/* centre-normalised transfer functions from the complex transform D (ny,nx):
 * n = D / D[ny/2, nx/2]; which bit0 -> mtf=|n| (real), bit1 -> ptf=angle(n) (real), bit2 -> otf=n.
 * prysm/otf.py:62-202 */
int pb_otf_normalize(pb_handle_t h, int dtype, const void* D, int ny, int nx, int which,
                     void* mtf, void* ptf, void* otf, void* stream);
/* Baliga-Cohn encircled energy of a real MTF array (ny,nx) with frequency spacing df [cy/mm] at nr radii
 * [mm] (HOST arrays in/out; synchronises the stream).  Deterministic.  prysm/otf.py:319-414 */
int pb_encircled_energy(pb_handle_t h, int dtype, const void* mtf, int ny, int nx, double df,
                        const double* radii_mm_host, int nr, double* out_host, void* stream);
/* moments of a real array: sums_host[0..2] = sum(d), sum(d*y), sum(d*x) (HOST doubles; this call
 * synchronises the stream).  Deterministic.  prysm/psf.py:174-203 */
int pb_moments(pb_handle_t h, int dtype, const void* data, int ny, int nx, double* sums_host,
               void* stream);


/* ---- adjoint twins and Lyot-coronagraph compositions (SURVEY.md 8(f)) -----------------------
 * masked multiply, the elementwise step of every composition in prysm/propagation/coronagraph.py and of
 * _adjoint_multiply (prysm/propagation/_kernels.py:30-38):
 *     out (+)= scale * (a - b) * f(m) * w
 * a: complex; b: complex or NULL; m: real / complex (m_kind) or NULL; w: real or NULL.  flags (OR of pb_mask_flags):
 * CONJ -> f = conj(m); ONE_MINUS -> f = 1 - m (Babinet complement, coronagraph.py:338); REAL_OUT -> out is a
 * REAL array receiving the real part (the real=True branch of _adjoint_multiply); ACCUMULATE -> out += ... */
typedef enum { PB_MASK_REAL = 0, PB_MASK_COMPLEX = 1 } pb_mask_kind;
typedef enum { PB_MASK_CONJ = 1, PB_MASK_ONE_MINUS = 2, PB_MASK_REAL_OUT = 4, PB_MASK_ACCUMULATE = 8 } pb_mask_flags;
int pb_mask_multiply(pb_handle_t h, int dtype, const void* a, const void* b, const void* m, int m_kind,
                     int flags, const void* w, double scale, long long count, void* out, void* stream);
/* adjoints of from_amp_and_phase (prysm/propagation/wavefront.py:172-242), kscale = 2*pi/(1e3*wavelength):
 * mode 0: out (complex) = i*kscale*imag(bar*conj(field))              -- w.r.t. phase (the reference's prefix is
 *         complex, so its result is purely imaginary; kept);
 * mode 1: out (real) = real(bar*conj(field))/|field|, 0 where field=0 -- w.r.t. amplitude, phasor from the field;
 * mode 2: out (real) = real(bar*conj(exp(i*kscale*opd)))              -- w.r.t. amplitude, phasor rebuilt from opd. */
int pb_field_adjoint(pb_handle_t h, int dtype, int mode, const void* field, const void* bar,
                     const void* opd, double kscale, long long count, void* out, void* stream);
/* real array out = re (which 0) / im (1) / angle (2) / abs (3) of a complex array: Wavefront.real / .imag / .phase
 * (prysm/propagation/wavefront.py:153-166). */
int pb_component(pb_handle_t h, int dtype, int which, const void* in, long long count, void* out,
                 void* stream);
/* out_host[0..1] = sum w * a * conj(b) (w real or NULL; fp64 accumulation, deterministic; synchronises the stream).
 * The reduction of thin_lens_adjoint (prysm/propagation/wavefront.py:244-280) and of <x, y> adjoint checks. */
int pb_dot(pb_handle_t h, int dtype, const void* a, const void* b, const void* w, long long count,
           double* out_host, void* stream);
/* out_host[2j..2j+1] = sum_n modes[j][n] * bar[n] for k real modes; bar real or complex (bar_complex).
 * sum_of_2d_modes_adjoint (prysm/polynomials/fitting.py:40-57).  Deterministic; synchronises the stream. */
int pb_mode_projection(pb_handle_t h, int dtype, const void* modes, int k, long long count,
                       const void* bar, int bar_complex, double* out_host, void* stream);
/* k-space gradient of mtf (which=1, bar real) / ptf (2, bar real) / otf (4, bar complex) _from_psf_adjoint given
 * the complex transform D (ny,nx), including the centre-normalisation term (prysm/otf.py:205-316); deterministic.  The
 * caller finishes with transform_psf_adjoint (pb_fft2, dir=+1) and takes the real part. */
int pb_otf_adjoint_seed(pb_handle_t h, int dtype, int which, const void* bar, const void* D, int ny,
                        int nx, void* data_bar, void* stream);
/* MTF-plane gradient of encircled_energy: mtf_bar = sum_r ee_bar[r]*r*J1(2 pi r nu)/nu*df^2, radii [mm] and
 * ee_bar HOST arrays (prysm/otf.py:417-471). */
int pb_encircled_energy_adjoint_seed(pb_handle_t h, int dtype, int ny, int nx, double df,
                                     const double* radii_mm_host, const double* ee_bar_host, int nr,
                                     void* mtf_bar, void* stream);
/* out = exp(i*charge*atan2(yf, xf)) on real coordinate arrays: vortex_phase_mask
 * (prysm/propagation/coronagraph.py:102-132). */
int pb_vortex_phase(pb_handle_t h, int dtype, int charge, const void* xf, const void* yf,
                    long long count, void* out, void* stream);
/* out = bilinear interpolation of the complex `map` (ny, nx) at col = (xf - cx)/dx + nx/2, row = (yf - cy)/dx + ny/2 with
 * edge replication, and `fill` (a complex array like out, or the scalar (fill_re, fill_im) when NULL) where a coordinate
 * leaves [0, n-1]: the fpm(xf, yf) callable of prepare_measured_fpm at order=1
 * (prysm/propagation/coronagraph.py:135-209; scipy.ndimage.map_coordinates(order=1, mode='nearest')). */
int pb_resample_bilinear(pb_handle_t h, int dtype, const void* map, int ny, int nx, const void* xf,
                         const void* yf, long long count, double cx, double cy, double dx, const void* fill,
                         double fill_re, double fill_im, void* out, void* stream);
/* one level of prepare_multiresolution (prysm/propagation/dft.py:155-167, 262-292): focal grids
 * xf = (ix - nx/2)*fdx + shift, yf likewise, and the hand-off window
 * taper(r; a0, b0) - taper(r; a1, b1), taper = 1 - smootherstep((r - a)/(b - a));
 * a0 < 0 -> first term 1 (coarsest level); a1 < 0 -> second term 0 (finest level).  Any output may be NULL. */
int pb_radial_window(pb_handle_t h, int dtype, int ny, int nx, double fdx, double shift, double a0,
                     double b0, double a1, double b1, void* win, void* xf, void* yf, void* stream);


/* ---- pupil synthesis: the step before the path (SURVEY.md 8(f) rank 3) ------------------------
 * x[iy,ix] = (ix - nx/2)*dx, y[iy,ix] = (iy - ny/2)*dx (make_xy_grid, prysm/coordinates.py:344-378) and their polar
 * form r = hypot(x, y), t = atan2(y, x) (cart_to_polar, coordinates.py:73-102), real arrays, any of them NULL. */
int pb_xy_grid(pb_handle_t h, int dtype, int ny, int nx, double dx, void* x, void* y, void* r, void* t,
               void* stream);
int pb_cart_to_polar(pb_handle_t h, int dtype, const void* x, const void* y, long long count, void* r,
                     void* t, void* stream);
/* aa_dx <= 0: out (uint8) = (r - radius <= 0): geometry.circle (prysm/geometry.py:337-372);
 * aa_dx  > 0: out (real)  = clip(0.5 - (r - radius)/aa_dx, 0, 1): antialias(circle_sdf(radius, r), aa_dx)
 *             (prysm/geometry.py:11-34), the grey-edge aperture coronagraph models need. */
int pb_circle(pb_handle_t h, int dtype, const void* r, long long count, double radius, double aa_dx,
              void* out, void* stream);
/* Jacobi polynomials P_j^(alpha,beta)(x), j = 0..nmax, by the three-term recurrence of
 * prysm/polynomials/jacobi.py:13-39, 147-175; order j is written to out[slots_host[j]] (a (n_out, count) real
 * array) when slots_host[j] >= 0.  nmax <= PB_POLY_NMAX (120). */
int pb_jacobi_seq(pb_handle_t h, int dtype, const void* x, long long count, int nmax, double alpha,
                  double beta, const int* slots_host, void* out, void* stream);
/* Zernike polynomials Z_n^m = norm * P_{(n-|m|)/2}^{(0,|m|)}(2r^2-1) * r^|m| * {cos(m t), sin(|m| t)} for k HOST
 * (n, m) pairs, the Jacobi recurrences shared per |m| (zernike_nm_seq, prysm/polynomials/zernike.py:74-166).
 * polar != 0: a = r, b = t; polar == 0: a = x, b = y (Cartesian; zernike_sum's input form).
 * pb_zernike_seq writes the basis out (k, count); pb_zernike_sum writes out (count) = sum_k coefs[k]*Z_k without
 * materialising the basis (zernike_sum, zernike.py:169-181; zero weights are skipped there too). */
int pb_zernike_seq(pb_handle_t h, int dtype, int polar, const void* a, const void* b, long long count,
                   int k, const int* n_host, const int* m_host, int norm, void* out, void* stream);
int pb_zernike_sum(pb_handle_t h, int dtype, int polar, const void* a, const void* b, long long count,
                   int k, const int* n_host, const int* m_host, const double* coefs_host, int norm,
                   void* out, void* stream);


/* ---- image-chain consumers of the same FFTs (SURVEY.md 8(f) rank 4) ------------------------------
 * conv(obj, psf) of two REAL arrays (prysm/convolution.py:9-32) as one forward and one inverse transform:
 * pb_balance_scale: *s_dev (a DEVICE double) = sqrt(sum a^2 / sum b^2) (1 if either sum is 0 / not finite): the two
 *   arrays share one transform whose rounding error is relative to the larger of them, so the PSF is scaled to the
 *   object's norm for the round trip -- on the device, no host synchronisation; deterministic;
 * pb_pack_complex: out = re + i*s*im (im NULL -> 0; im_scale_dev NULL -> s = 1); pb_fft2 of that gives Z = O + i*s*H;
 * pb_packed_spectrum_product: out[k] = scale/s * (Z[k]^2 - conj(Z[-k])^2)/(4i) = scale * O[k]*H[k], indices modulo
 *   (ny, nx), unshifted spectrum order; out must not alias Z. */
int pb_balance_scale(pb_handle_t h, int dtype, const void* a, const void* b, long long count, double* s_dev,
                     void* stream);
int pb_pack_complex(pb_handle_t h, int dtype, const void* re, const void* im, const double* im_scale_dev,
                    long long count, void* out, void* stream);
int pb_packed_spectrum_product(pb_handle_t h, int dtype, const void* Z, int ny, int nx, double scale,
                               const double* im_scale_dev, void* out, void* stream);

/* detector sampling of the image chain (prysm/detector.py:151-338), real arrays:
 * pb_bindown: out (ny/fy, nx/fx) = sum (mean != 0: mean) of each fy x fx block (bindown);
 * pb_tile:    out (ny*fy, nx*fx) = scale * in[y/fy, x/fx] (tile, the adjoint of bindown);
 * pb_separable_tf: out[y,x] = sinc(fx[x] wx) sinc(fy[y] wy) (kind 0, pixel_ft) or cos(2 wx fx[x]) cos(2 wy fy[y])
 *              (kind 1, olpf_ft) from the two frequency VECTORS. */
int pb_bindown(pb_handle_t h, int dtype, const void* in, int ny, int nx, int fy, int fx, int mean,
               void* out, void* stream);
int pb_tile(pb_handle_t h, int dtype, const void* in, int ny, int nx, int fy, int fx, double scale,
            void* out, void* stream);
int pb_separable_tf(pb_handle_t h, int dtype, int kind, const void* fx, const void* fy, int ny, int nx,
                    double wx, double wy, void* out, void* stream);


/* ---- deformable mirror and the cubic-spline warp (prysm/x/dm.py, prysm/coordinates.py:644-672) -------------------
 * pb_spline_prefilter: coef (ny, nx, always float64) = the order-3 B-spline coefficients of the real array `in` (or the
 *   real part of a complex one, in_complex != 0), both axes, mirror boundary: scipy.ndimage.spline_filter(in, 3,
 *   output=float64, mode='mirror'), which is also what map_coordinates(mode='constant') prefilters with.
 * pb_warp: out (oy, ox, real) = scale * map_coordinates(in, (y, x), order=3, mode='constant', cval=0) with
 *   x, y either the arrays xc, yc (oy*ox values, float when coord_dtype is PB_C64, double for PB_C128) or, when both
 *   are NULL, (x', y', w) = M (x, y, 1) / w at every output pixel (x = column, y = row) for the HOST row-major
 *   3 x 3 matrix matrix_host, evaluated in fp64 on the device.  The coefficients live in handle scratch.
 * pb_dm_scatter: poke (ny, nx, real) = act[(y - y0)/sy, (x - x0)/sx] at the lattice points y0 + k*sy, x0 + l*sx and 0
 *   elsewhere (every sample is written): poke_arr[iyy, ixx] = actuators (prysm/x/dm.py:251).
 * pb_dm_gather: act (nay, nax, real) = real(in)[y0 + k*sy, x0 + l*sx] (in real, or complex when in_complex != 0):
 *   in_actuator_space[iyy, ixx] (prysm/x/dm.py:331). */
int pb_spline_prefilter(pb_handle_t h, int dtype, const void* in, int in_complex, int ny, int nx, double* coef,
                        void* stream);
int pb_warp(pb_handle_t h, int dtype, const void* in, int in_complex, int ny, int nx, const void* xc, const void* yc,
            int coord_dtype, const double* matrix_host, int oy, int ox, double scale, void* out, void* stream);
int pb_dm_scatter(pb_handle_t h, int dtype, const void* act, int nay, int nax, int ny, int nx, int y0, int sy, int x0,
                  int sx, void* poke, void* stream);
int pb_dm_gather(pb_handle_t h, int dtype, const void* in, int in_complex, int ny, int nx, int nay, int nax, int y0,
                 int sy, int x0, int sx, void* act, void* stream);


/* ---- signed-distance geometry and segmented apertures (prysm/geometry.py, prysm/segmented.py:133-368) -------------
 * pb_sdf: out (ny, nx) = the signed distance (negative inside) of one shape at (x, y), computed in fp64 and rounded
 *   once to dtype's real type, or with mask != 0 the uint8 mask sdf <= 0.  separable != 0: x is a row of nx values and
 *   y a column of ny values (optimize_xy_separable's form); otherwise both are (ny, nx).  Parameters, HOST:
 *     PB_SDF_POLYGON          verts = nverts (x, y) vertices, any winding, even-odd parity   (geometry.py:419-463)
 *     PB_SDF_SPIDER           params = half width, cx, cy; verts = (cos, sin) of each vane's angle (geometry.py:550-594)
 *     PB_SDF_RECTANGLE        params = half width, half height, mode (0 none, 1 swap x/y, 2 rotate), cos, sin
 *                             (geometry.py:182-222)
 *     PB_SDF_FILLET_RECTANGLE params = half width, half height, fillet radius, cx, cy, rotate (0/1), cos, sin
 *                             (geometry.py:656-696)
 *     PB_SDF_ANNULUS          x = r (y unused); params = inner radius, outer radius        (geometry.py:375-395)
 *     PB_SDF_OFFSET_CIRCLE    params = radius, cx, cy                                       (geometry.py:627-653)
 *   At most 8 params and PB_SDF_MAX_VERTICES (128) vertices / vanes: the shape travels in kernel-parameter space.
 * pb_sdf_combine: out = min(a, b) (PB_SDF_UNION), max(a, b) (PB_SDF_INTERSECT) or max(a, -b) (PB_SDF_SUBTRACT)
 *   (geometry.py:37-93).
 * Segments: the DEVICE table `seg` has PB_SEGMENT_FIELDS int64 per segment: window row y0, column x0, height, width, the
 *   offset of its h*w samples in the packed per-segment buffers, and the offset of its (nmodes, h, w) basis in `bases`.
 *   tile_ptr (tiles_y*tiles_x + 1) / tile_seg (int32, DEVICE) list, per output tile of PB_SEGMENT_TILE_Y x
 *   PB_SEGMENT_TILE_X samples (row-major tiles), the segments whose windows meet it, in ascending segment order.
 * pb_hex_segments: for every listed segment, cover = clip(0.5 - polygon_sdf/dx, 0, 1) over its window, local_x = x - cx,
 *   local_y = y - cy (packed like cover); amp (ny, nx) = max of cover over the covering segments, 0 elsewhere.  geo
 *   (DEVICE fp64) holds per segment nverts (x, y) vertices, then (cx, cy); 3 <= nverts <= 8.
 * pb_segment_compose: out (ny, nx) += sum over segments s < ncoef of mask_s * sum_k coefs[s*coef_stride + k] *
 *   base_{s,k} over its window (compose_opd), accumulated per sample in fp64 in segment order and rounded once; coefs
 *   is a DEVICE fp64 array.  No atomics.
 * pb_segment_compose_adjoint: out (nseg, nmodes) = sum over segment s's window of opdbar * mask_s * base_{s,k}, with
 *   nchunk * PB_SEGMENT_CHUNK >= every window's h*w: a fixed-order two-level reduction. */
typedef enum {
    PB_SDF_POLYGON = 0, PB_SDF_SPIDER = 1, PB_SDF_RECTANGLE = 2, PB_SDF_FILLET_RECTANGLE = 3, PB_SDF_ANNULUS = 4,
    PB_SDF_OFFSET_CIRCLE = 5
} pb_sdf_kind;
typedef enum { PB_SDF_UNION = 0, PB_SDF_INTERSECT = 1, PB_SDF_SUBTRACT = 2 } pb_sdf_op;
enum { PB_SDF_MAX_VERTICES = 128 };
typedef enum {
    PB_SEGMENT_FIELDS = 6, PB_SEGMENT_TILE_Y = 32, PB_SEGMENT_TILE_X = 64, PB_SEGMENT_CHUNK = 2048
} pb_segment_layout;
int pb_sdf(pb_handle_t h, int dtype, int kind, const void* x, const void* y, int separable, int ny, int nx,
           const double* params_host, int nparams, const double* verts_host, int nverts, int mask, void* out,
           void* stream);
int pb_sdf_combine(pb_handle_t h, int dtype, int op, const void* a, const void* b, long long count, void* out,
                   void* stream);
int pb_hex_segments(pb_handle_t h, int dtype, const void* x, const void* y, int ny, int nx, int tiles_y, int tiles_x,
                    const int* tile_ptr, const int* tile_seg, const long long* seg, const double* geo, int nverts,
                    double dx, void* cover, void* local_x, void* local_y, void* amp, void* stream);
int pb_segment_compose(pb_handle_t h, int dtype, int ny, int nx, int tiles_y, int tiles_x, const int* tile_ptr,
                       const int* tile_seg, const long long* seg, const void* masks, const void* bases, int nmodes,
                       const double* coefs, long long coef_stride, int ncoef, void* out, void* stream);
int pb_segment_compose_adjoint(pb_handle_t h, int dtype, int ny, int nx, int nseg, const long long* seg,
                               const void* masks, const void* bases, int nmodes, const void* opdbar, int nchunk,
                               void* out, void* stream);

/* ---- Jones calculus (prysm/x/polarization.py) ----------------------------------------------------------------------
 * Element-planar layout: a Jones array of n pixels is 4 contiguous planes of n complex samples at dtype, plane 2*i + j
 * holding J[..., i, j]; Mueller and Kronecker arrays are 16 planes, plane 4*r + c (Mueller planes are real).
 * pb_jones_planar: src is a (rows, cols, 2, 2) array of src_type (PB_ELEM_F32 / F64 / C64 / C128) with strides s_row, s_col, s_i, s_j counted in
 *   elements of src_type (one complex value is one element); out = its 4 planes (n = rows*cols), converted to dtype.
 * pb_jones_product: out = op_a(A) * op_b(B) per pixel, the 2x2 matrix product (PB_JONES_MATMUL) or the elementwise
 *   product (PB_JONES_HADAMARD).  An operand is a constant 2x2 (PB_JONES_CONST: four complex values from consts_host,
 *   A's at [0, 8), B's at [8, 16)), 4 planes (PB_JONES_PLANES) or one complex / real plane broadcast to all four
 *   elements (PB_JONES_SCALAR / PB_JONES_SCALAR_REAL); op is PB_JONES_OP_N or PB_JONES_OP_H (conjugate transpose).
 *   out may be one of the operands.
 * pb_jones_elements: out = 4 planes of one constructor, phases evaluated in fp64.  params_host (host fp64):
 *   PB_JONES_FILL: 4 complex values (8 doubles);  PB_JONES_ROTATION: theta, scale (with a plane, theta = plane*scale);
 *   PB_JONES_RETARDER / PB_JONES_DIATTENUATOR: theta, retardance / alpha (a plane replaces the second);
 *   PB_JONES_VVR: charge, retardance, rotate, with the azimuth plane (required; it is not modified).
 *   plane: optional, n real values of plane_type PB_ELEM_F32 or PB_ELEM_F64.
 * pb_jones_reduce: PB_JONES_MUELLER: out = 16 real planes of real(U kron(conj a, a) U^-1);  PB_JONES_KRON: out = 16
 *   complex planes of kron(a, b);  PB_JONES_PAULI: out = 4 complex planes c0..c3. */
typedef enum { PB_JONES_CONST = 0, PB_JONES_PLANES = 1, PB_JONES_SCALAR = 2, PB_JONES_SCALAR_REAL = 3 } pb_jones_operand;
typedef enum { PB_JONES_MATMUL = 0, PB_JONES_HADAMARD = 1 } pb_jones_mode;
typedef enum { PB_JONES_OP_N = 0, PB_JONES_OP_H = 1 } pb_jones_op;
typedef enum {
    PB_JONES_FILL = 0, PB_JONES_ROTATION = 1, PB_JONES_RETARDER = 2, PB_JONES_DIATTENUATOR = 3, PB_JONES_VVR = 4
} pb_jones_element;
typedef enum { PB_JONES_MUELLER = 0, PB_JONES_KRON = 1, PB_JONES_PAULI = 2 } pb_jones_reduction;
int pb_jones_planar(pb_handle_t h, int dtype, const void* src, int src_type, long long rows, long long cols,
                    long long s_row, long long s_col, long long s_i, long long s_j, void* out, void* stream);
int pb_jones_product(pb_handle_t h, int dtype, int mode, long long n, int a_kind, const void* a, int a_op, int b_kind,
                     const void* b, int b_op, const double* consts_host, void* out, void* stream);
int pb_jones_elements(pb_handle_t h, int dtype, int kind, long long n, const void* plane, int plane_type,
                      const double* params_host, int nparams, void* out, void* stream);
int pb_jones_reduce(pb_handle_t h, int dtype, int kind, long long n, const void* a, const void* b, void* out,
                    void* stream);

/* ---- wavefront sensing (prysm/x/fibers.py, sri.py, pdi.py, psi.py) ---------------------------------------------------
 * pb_lp_modes: out = nmodes packed real fields (nmodes, n) of dtype's real type from the radius r and angle t grids
 *   (n values each; t may be NULL when no mode has an azimuth factor).  plan_host holds 6 doubles per mode:
 *   l, ld, U, W, rule, az.  rho = r / a and the core is r <= a (PB_LP_RULE_LP, compute_LP_modes) or rho = r * (1/a)
 *   and the core is rho < 1 (PB_LP_RULE_SMF, smf_mode_field).  Core: J_l(U rho) / J_ld(U); cladding:
 *   K_l(W rho) / K_ld(W), evaluated exponentially scaled; times cos(l t) (PB_LP_COS) or sin(l t) (PB_LP_SIN).
 * pb_overlap: for each of nmodes modes M_p (real or complex at dtype; packed (nmodes, n) in `modes`, or the host
 *   array mode_ptrs_host of nmodes device pointers when `modes` is NULL) and the complex field E (n values):
 *   eta[p] = |sum conj(M_p) E|^2 / (I_p I_E), I_p = sum |M_p|^2 (or ip_dev[p], fp64 on the device), I_E = sum |E|^2
 *   (or ie_dev[0]).  c_out (optional): sqrt(I_E eta[0]).  eta and c_out are dtype's real type.
 *   Deterministic: partials of PB_OVERLAP_CHUNK pixels summed in a fixed order.
 * pb_wfs_combine: out = alpha a + beta b (complex) or |alpha a + beta b|^2 (real_out: real).  coefs_host = re, im of
 *   alpha then of beta; each is multiplied by the device real scalar alpha_scale / beta_scale when given.  b may be
 *   NULL.
 * pb_grating: g = the grating of kind at x + shift (x real at dtype, the arithmetic in fp64); out = E g (complex), or
 *   g itself (real) when E is NULL.  PB_GRATING_SIN_AMP params: prefix (g = 1 - (sin(prefix x) + 1) / 2 * 0.1);
 *   PB_GRATING_RECTANGLE params: period, edge, hi, lo, mid, eps (numpy's mod by period, hi below edge else lo, mid
 *   where |x mod period| < eps).
 * pb_psi: num = sum s_k g_k, den = sum c_k g_k over nframes <= 64 frames of frame_type (PB_ELEM_F32 / F64 / U16 /
 *   I32; the host pointer array frames_host, or `stack` with frame_stride elements between frames) and phase =
 *   atan2(num, den).  Any of num, den and phase may be NULL.  Float frames: num_type = phase_type = frame_type.
 *   Integer frames: phase_type = PB_ELEM_F64 and num_type PB_ELEM_I64 (integer weights, exact) or PB_ELEM_F64. */
enum { PB_OVERLAP_CHUNK = 4096 };
typedef enum { PB_LP_RULE_LP = 0, PB_LP_RULE_SMF = 1 } pb_lp_rule;
typedef enum { PB_LP_NONE = 0, PB_LP_COS = 1, PB_LP_SIN = 2 } pb_lp_azimuth;
typedef enum { PB_GRATING_SIN_AMP = 0, PB_GRATING_RECTANGLE = 1 } pb_grating_kind;
int pb_lp_modes(pb_handle_t h, int dtype, const void* r, const void* t, long long n, double a, int nmodes,
                const double* plan_host, void* out, void* stream);
int pb_overlap(pb_handle_t h, int dtype, const void* E, long long n, int nmodes, const void* modes,
               const void* const* mode_ptrs_host, int modes_complex, const double* ip_dev, const double* ie_dev,
               void* eta, void* c_out, void* stream);
int pb_wfs_combine(pb_handle_t h, int dtype, long long n, const void* a, const void* b, const double* coefs_host,
                   const void* alpha_scale, const void* beta_scale, int real_out, void* out, void* stream);
int pb_grating(pb_handle_t h, int dtype, int kind, long long n, const void* x, double shift, const double* params_host,
               int nparams, const void* E, void* out, void* stream);
int pb_psi(pb_handle_t h, int frame_type, int nframes, const void* const* frames_host, const void* stack,
           long long frame_stride, long long n, const double* s_host, const double* c_host, int num_type, void* num,
           void* den, int phase_type, void* phase, void* stream);

/* ---- image sensors (prysm/detector.py, prysm/bayer.py) ---------------------------------------------------------------
 * pb_expose: frames exposures of the n-pixel aerial image (real at dtype; viewed as (n / nx, nx)) -> out, frame-major
 *   (frames, n).  lam = aerial t [* prnu] + dark [* dcnu], each step rounded at dtype; prnu / dcnu (optional, at dtype)
 *   are read at row * sr + col * sc, so a broadcast map is never materialised.  Per (pixel, frame): k ~ Poisson(lam)
 *   (exact: inversion below 10, PTRS from 10), x = k + read_sigma * N(0, 1) + bias, min(x, fwc) * scaling clipped to
 *   [0, cap] and truncated to an unsigned code of code_bytes (1, 2, 4); with a lut (lut_len entries of out_bytes), out =
 *   lut[code], else out_bytes = code_bytes.  params_host: t, dark, read_sigma, bias, fwc, scaling, cap.  Random
 *   numbers: Philox4x32-10 keyed by `key`, counter (pixel, frame, draw), independent of the launch shape.  flags: two
 *   zeroed uint32 on the device; bit 0 of flags[0]: some lam < 0 or NaN, bit 1: some lam > 9.2234e18 (numpy's
 *   POISSON_LAM_MAX), bit 2: some code >= lut_len, whose maximum is in flags[1].  Never synchronises.
 * pb_apply_lut: out[i] = lut[codes[i]] for unsigned codes of code_bytes; with check, a code >= lut_len sets bit 2 of
 *   flags[0] and raises flags[1] to it.
 * pb_pixel: out[i] = (x <= wx) & (x >= -wx) & (y <= wy) & (y >= -wy) as uint8, over an (n / nx, nx) view with x and y
 *   (real at dtype) read at row * sr + col * sc.
 * pb_bayer_interleave: out (M, N) with row pitch out_ld, elements of elem_bytes; the value at CFA site s (0 top-left,
 *   1 top-right, 2 bottom-left, 3 bottom-right of each 2x2 cell) comes from planes_host[s] (row pitch ld_host[s]) at
 *   (y, x), or at (y / 2, x / 2) with half (recomposite).
 * pb_demosaic_deinterlace: (m / 2, n / 2, 3) = (R, (G1 + G2) / 2, B) of an even-sided mosaic with row pitch ld; the
 *   green sum is formed in in_type (PB_ELEM_F32 / F64 / U8 / U16 / U32; wrapping for unsigned types), the halving in
 *   out_type (PB_ELEM_F32 / F64).
 * pb_white_balance: a *= gain in place (a contiguous, real at dtype): gains_host[site] for a mosaic (kind 0, rows of
 *   nx) or gains_host[i % 3] for interleaved RGB (kind 1).  With sat_host, every gain is first divided by max(1,
 *   max_p(max(plane p) gains_p / sat_p)), computed on the device.
 * pb_demosaic_malvar: (m, n, 3) RGB of out_type (PB_ELEM_F32 from f32 / u8 / u16, or PB_ELEM_F64) from an m x n
 *   mosaic of in_type with row pitch ld, rggb or bggr: Malvar-He-Cutler's 5x5 filters, scipy.ndimage's reflect
 *   boundary, accumulated in fp64.  One pass.
 * pb_bayer_assemble: (n, 3) = (Re rp, (Re g2p + g1) / 2, Re bp) for complex rp, g2p, bp and real g1 at dtype. */
int pb_expose(pb_handle_t h, int dtype, const void* aerial, long long n, long long nx, const void* prnu, long long prnu_sr,
              long long prnu_sc, const void* dcnu, long long dcnu_sr, long long dcnu_sc, const double* params_host,
              int frames, long long key, int code_bytes, const void* lut, long long lut_len, int out_bytes,
              void* out, void* flags, void* stream);
int pb_apply_lut(pb_handle_t h, int code_bytes, const void* codes, long long n, const void* lut, long long lut_len,
                 int out_bytes, int check, void* out, void* flags, void* stream);
int pb_pixel(pb_handle_t h, int dtype, const void* x, long long xsr, long long xsc, const void* y, long long ysr,
             long long ysc, long long n, long long nx, double wx, double wy, void* out, void* stream);
int pb_bayer_interleave(pb_handle_t h, int elem_bytes, const void* const* planes_host, const long long* ld_host, int half,
                        long long M, long long N, void* out, long long out_ld, void* stream);
int pb_demosaic_deinterlace(pb_handle_t h, int in_type, const void* img, long long m, long long n, long long ld, int bggr,
                            int out_type, void* out, void* stream);
int pb_white_balance(pb_handle_t h, int dtype, void* a, long long n, long long nx, int kind, const double* gains_host,
                     const double* sat_host, void* stream);
int pb_demosaic_malvar(pb_handle_t h, int in_type, const void* img, long long m, long long n, long long ld, int bggr,
                       int out_type, void* out, void* stream);
int pb_bayer_assemble(pb_handle_t h, int dtype, const void* rp, const void* g2p, const void* bp, const void* g1,
                      long long n, void* out, void* stream);

/* ---- Shack-Hartmann sensing (prysm/x/shack_hartmann.py) -------------------------------------------------------------
 * pb_lenslet_screen: the complex (H, W) screen exp(i kphase total) of dtype, one thread per sample.  total is the sum,
 *   in the storage precision and in lenslet order (row j outer, column i inner), of rsq / two_efl over the lenslets
 *   (j, i) whose window covers the sample and whose aperture admits it, with lx = x - xc[i], ly = y - yc[j],
 *   rsq = lx^2 + ly^2 in fp64 without fused multiply-add.  x, y: (H, W) real at dtype.  centres: fp64 device array,
 *   xc [ncols] then yc [nrows].  cand: int32 device array, per grid column (first, one past last) lenslet column whose
 *   window covers it [2 W], then the same per grid row [2 H].  params_host: half-width, half-height, angle (radians),
 *   lenslet r^2.  kind: PB_LENSLET_RECT (|lx| <= w and |ly| <= h), PB_LENSLET_RECT_SWAP (|ly| <= w and |lx| <= h),
 *   PB_LENSLET_RECT_ROTATED (the same after rotating (lx, ly) by the angle in polar form), PB_LENSLET_CIRCLE
 *   (rsq <= lenslet r^2).
 * pb_subaperture_centroids: for nframes frames of frame_type (PB_ELEM_F32 / F64 / U16 / I32; (H, W) each, frame_stride elements apart) and each
 *   subaperture (j, i): w = max(I - t, 0) with t = threshold max(I over the subaperture); disp (nframes, 2, nrows,
 *   ncols) = scale (sum w x / sum w - xc[i], sum w y / sum w - yc[j]), NaN where sum w = 0; flux (nframes, nrows, ncols) =
 *   sum I.  out_type: PB_ELEM_F64 for PB_ELEM_F64 frames, PB_ELEM_F32 otherwise; the sums are fp64 in a fixed order.
 *   dtab (fp64, device): x of each grid column [W], y of each grid row [H], xc [ncols], yc [nrows].  itab (int32,
 *   device): owning lenslet column of each grid column or -1 [W], each lenslet column's owned grid columns as
 *   [lo, hi): lo [ncols] then hi [ncols], each lenslet row's owned grid rows: lo [nrows] then hi [nrows].  One launch.
 * pb_sh_reconstruct: out[f, k] = sum_m R[k, m] (slopes[f][idx[m]] - ref[m]) for nframes slope vectors frame_stride
 *   elements apart, R (K, M) and ref (M, optional) fp64 on the device, idx int32; slopes and out of dtype
 *   (PB_ELEM_F32 / PB_ELEM_F64), accumulated in fp64.  A NaN in a selected slope propagates. */
typedef enum { PB_LENSLET_RECT = 0, PB_LENSLET_RECT_SWAP = 1, PB_LENSLET_RECT_ROTATED = 2, PB_LENSLET_CIRCLE = 3 } pb_lenslet_kind;
int pb_lenslet_screen(pb_handle_t h, int dtype, const void* x, const void* y, int H, int W, int ncols, int nrows,
                      const double* centres, const int* cand, int kind, const double* params_host, double two_efl,
                      double kphase, void* out, void* stream);
int pb_subaperture_centroids(pb_handle_t h, int frame_type, const void* frames, int nframes, int H, int W,
                             long long frame_stride, int ncols, int nrows, const double* dtab, const int* itab,
                             double threshold, double scale, int out_type, void* disp, void* flux, void* stream);
int pb_sh_reconstruct(pb_handle_t h, int dtype, const void* slopes, int nframes, long long frame_stride, const int* idx,
                      const double* ref, const double* R, int K, int M, void* out, void* stream);

/* ---- Forbes polynomials (prysm/polynomials/qpoly.py) ------------------------------------------------------------
 * family: PB_QPOLY_BFS (Q-bfs, oe-18-19-19700), PB_QPOLY_CON (Q-con, oe-18-13-13851), PB_QPOLY_2D (2D-Q, oe-20-3-2483;
 * m = 0 is Q-bfs, m < 0 a sine term).  Orders are limited to n and |m| <= PB_QPOLY_NMAX (64), a call to 256 recurrence steps
 * (the sum over its recurrences -- one for Q-bfs / Q-con, one per |m| for 2D-Q -- of the highest n + 1) and a basis
 * call to 1024 modes; outside these PB_ERR_UNSUPPORTED, n < 0 PB_ERR_INVALID, both before any launch.  Each call is
 * one kernel, one thread per sample, every recurrence run once in fp64 registers.
 * pb_qpoly_seq: k HOST (n, m) pairs (m_host may be NULL except for 2D-Q), in any order, repeats allowed; plane q of
 *   out0 (and out1), each (k, count), is mode q.
 *   kind PB_QPOLY_VALUE:  out0 = Q(a) (Q-bfs / Q-con: a = x) or Q(a = r, b = t) (2D-Q)       (Qbfs_seq, Qcon_seq, Q2d_seq)
 *   kind PB_QPOLY_DER:    out0 = d/dx (Q-bfs / Q-con), or d/dr -> out0 and d/dt -> out1 (2D-Q)
 *                         (Qbfs_der_seq, Qcon_der_seq, Q2d_der_seq)
 *   kind PB_QPOLY_DER_XY: 2D-Q only, a = x, b = y: d/dx -> out0, d/dy -> out1 through Re / Im (x + iy)^|m|, finite at
 *                         the origin (Q2d_der_xy_seq)
 * pb_qpoly_sum: the sag z = sum_q coefs[q] Q_q(u, t) and optionally dz/du, dz/dt (2D-Q) without the basis; zero
 *   coefficients are skipped, so trailing zeros trim.  z, dzdr, dzdt: (count) each, any may be NULL but not all.
 *   (compute_z_Qbfs, compute_z_zprime_Qbfs, compute_z_zprime_Qcon, compute_z_Q2d, compute_z_zprime_Q2d.)
 * pb_qpoly_tables (host, no handle): rows n = 0..nmax of 7 fp64 each of the recurrence tables the kernels use:
 *   PB_QPOLY_BFS: f(n), g(n), h(n) (f_qbfs, g_qbfs, h_qbfs);  PB_QPOLY_CON: A, B, C of order n (_qcon_abc);
 *   PB_QPOLY_2D (m >= 1): A, B, C (abc_q2d, NaN where its denominator is 0), G, F, g, f (G_q2d, F_q2d, g_q2d, f_q2d). */
typedef enum { PB_QPOLY_BFS = 0, PB_QPOLY_CON = 1, PB_QPOLY_2D = 2 } pb_qpoly_family;
typedef enum { PB_QPOLY_VALUE = 0, PB_QPOLY_DER = 1, PB_QPOLY_DER_XY = 2 } pb_qpoly_kind;
enum { PB_QPOLY_NMAX = 64 };
int pb_qpoly_seq(pb_handle_t h, int dtype, int family, int kind, const void* a, const void* b, long long count, int k,
                 const int* n_host, const int* m_host, void* out0, void* out1, void* stream);
int pb_qpoly_sum(pb_handle_t h, int dtype, int family, const void* u, const void* t, long long count, int k,
                 const int* n_host, const int* m_host, const double* coefs_host, void* z, void* dzdr, void* dzdt,
                 void* stream);
int pb_qpoly_tables(int family, int m, int nmax, double* out);

/* ---- Orthogonal polynomials, Zernike derivatives and polynomial sums (prysm/polynomials) ---------------------------
 * The 1-D families are one three-term recurrence P_k = (A_k x + B_k) P_{k-1} - C_k P_{k-2}, run once per sample in
 * fp64 registers by one kernel; outputs are rounded once to dtype.  Orders are limited to 0 <= n <= PB_POLY_NMAX (120):
 * n < 0 is PB_ERR_INVALID, n > PB_POLY_NMAX PB_ERR_UNSUPPORTED, both before any launch.  Each call is one launch.
 * pb_jacobi_seq (above) is served by the same kernel.
 * pb_poly_seq: k HOST orders n_host in any order, repeats allowed; alpha is Jacobi's and Laguerre's alpha and Dickson's
 *   alpha, beta Jacobi's beta (ignored otherwise).
 *   kind PB_POLY_VALUE:     plane q of out (k, count) = P_{n_q}(x)
 *   kind PB_POLY_DER:       plane q = dP_{n_q}/dx by the reference's route: Jacobi 0.5 (n + a + b + 1) P_{n-1}^(a+1,b+1),
 *                           Hermite kind n P_{n-1}, Laguerre -L_{n-1}^(a+1), the others the differentiated recurrence
 *   kind PB_POLY_VALUE_DER: planes 0..k-1 = P, k..2k-1 = dP/dx by the differentiated recurrence (jacobi_seq_with_der)
 *   k (2k for PB_POLY_VALUE_DER) <= 1024.
 * pb_jacobi_radial_sum: z = sum_q coefs[q] P_{n_q}^(alpha,beta)(u), u = 2 (x^2 + y^2) / radius^2 - 1, zero coefficients
 *   skipped; with dzdx and dzdy (both or neither) also dz/du 4x / radius^2 and dz/du 4y / radius^2, dz/du by the
 *   differentiated recurrence in the same pass.  (jacobi_radial_sum, jacobi_radial_sum_der_xy.)
 * pb_jacobi_clenshaw: Clenshaw's backward recurrence over the len (<= PB_POLY_NMAX + 1) HOST coefficients s_host for the
 *   sum and its first j (<= PB_CLENSHAW_JMAX, 8) derivatives, N = max(len, 2); table != 0: every alpha plane (jj, n) into out (j + 1, N, count), rows
 *   jj > len - 1 zero; table = 0: the sum alone into out (count).  (jacobi_sum_clenshaw, jacobi_sum_clenshaw_der.)
 * pb_zernike_der: the (n, m) pairs' derivatives into out (k, 2, count): cartesian = 0, (a, b) = (r, t): dZ/dr, dZ/dt;
 *   cartesian = 1, (a, b) = (x, y): dZ/dx, dZ/dy through Re / Im (x + iy)^|m|, finite at the origin.  norm as
 *   pb_zernike_seq.  One launch per Zernike plan.  (zernike_nm_der_seq, zernike_nm_der_xy_seq.)
 * pb_zernike_sum_der_xy: W, dW/dx, dW/dy of W = sum_q coefs[q] Z_q(x, y) into out (3, count) without the basis;
 *   duplicate (n, m) pairs add, zero coefficients are skipped.  One launch per Zernike plan.  (zernike_sum_der_xy.)
 * pb_xy_seq: plane q of out (k, count) is d^a/dx^a d^b/dy^b x^m y^n, (a, b) = bits 0 and 1 of kind_host[q];
 *   separable != 0: the grid is (count / nx, nx), x[column] and y[row]; otherwise x and y are elementwise.
 * pb_tensor_sum: z = sum_q coefs[q] P_{m_q}(x) P_{n_q}(y), P the monomials (PB_TSUM_MONOMIAL) or Chebyshev-1
 *   (PB_TSUM_CHEBY1), (max m + 1)(max n + 1) <= 1024; with dzdx and dzdy also dz/dx / x_norm and dz/dy / y_norm.  Grid
 *   as pb_xy_seq.  (xy_sum, xy_sum_der_xy, cheby1_2d_sum, cheby1_2d_sum_der_xy.) */
typedef enum {
    PB_POLY_JACOBI = 0, PB_POLY_CHEBY1 = 1, PB_POLY_CHEBY2 = 2, PB_POLY_CHEBY3 = 3, PB_POLY_CHEBY4 = 4, PB_POLY_LEGENDRE = 5,
    PB_POLY_HERMITE_HE = 6, PB_POLY_HERMITE_H = 7, PB_POLY_LAGUERRE = 8, PB_POLY_DICKSON1 = 9, PB_POLY_DICKSON2 = 10
} pb_poly_family;
typedef enum { PB_POLY_VALUE = 0, PB_POLY_DER = 1, PB_POLY_VALUE_DER = 2 } pb_poly_kind;
typedef enum { PB_TSUM_MONOMIAL = 0, PB_TSUM_CHEBY1 = 1 } pb_tsum_basis;
enum { PB_POLY_NMAX = 120, PB_CLENSHAW_JMAX = 8 };
int pb_poly_seq(pb_handle_t h, int dtype, int family, int kind, double alpha, double beta, const void* x, long long count,
                int k, const int* n_host, void* out, void* stream);
int pb_jacobi_radial_sum(pb_handle_t h, int dtype, double alpha, double beta, const void* x, const void* y, long long count,
                         int k, const int* n_host, const double* coefs_host, double radius, void* z, void* dzdx, void* dzdy,
                         void* stream);
int pb_jacobi_clenshaw(pb_handle_t h, int dtype, double alpha, double beta, const void* x, long long count, int len,
                       const double* s_host, int j, int table, void* out, void* stream);
int pb_zernike_der(pb_handle_t h, int dtype, int cartesian, const void* a, const void* b, long long count, int k,
                   const int* n_host, const int* m_host, int norm, void* out, void* stream);
int pb_zernike_sum_der_xy(pb_handle_t h, int dtype, const void* x, const void* y, long long count, int k, const int* n_host,
                          const int* m_host, const double* coefs_host, int norm, void* out, void* stream);
int pb_xy_seq(pb_handle_t h, int dtype, const void* x, const void* y, long long count, long long nx, int separable, int k,
              const int* m_host, const int* n_host, const int* kind_host, void* out, void* stream);
int pb_tensor_sum(pb_handle_t h, int dtype, int basis, const void* x, const void* y, long long count, long long nx,
                  int separable, int k, const int* m_host, const int* n_host, const double* coefs_host, double x_norm,
                  double y_norm, void* z, void* dzdx, void* dzdy, void* stream);

/* ---- Thin-film stacks (prysm/thinfilm.py multilayer_stack_rt, prysm/x/coatings stack.py and diff.py) ---------------
 * One thread per sample; the transfer-matrix chain runs in fp64 registers whatever dtype is, and outputs are rounded
 * once to dtype (PB_C64: complex64 / float32, PB_C128: complex128 / float64).  Layers are ambient side first.
 * Operands (HOST array in[PB_TF_NOPS] of device pointers, all fp64): wavelength and angle of incidence (radians) real,
 *   ambient index, substrate index and the per-layer index complex128, the per-layer thickness real.  Each is indexed
 *   over a collapsed calculation shape of ndim <= PB_TF_DIMS (4) dims (HOST shape[ndim], outermost first; count = its
 *   product): operand q reads element  sum_j idx_j strides[5 q + j]  (+ layer * strides[5 q + 4] for the per-layer
 *   operands),
 *   strides in elements, 0 where it broadcasts, slots j >= ndim ignored.
 * pb_stack_eval: the angle is theta_scale times the angle operand (pi / 180 for degrees).  Mode PB_TF_THINFILM
 *   assembles r, t as multilayer_stack_rt (nlayers >= 1; only the r and t outputs); PB_TF_COATINGS uses the
 *   admittance form of the coatings engine (nlayers >= 0).  flags is a bit mask of 1 << PB_TF_OUT_*; out[PB_TF_OUT_*] (HOST array of PB_TF_NOUT device pointers) is read for the bits set:
 *   r, t, eta0, eta_sub complex (count); E, H complex and Esq = |E|^2 real (nlayers + 1, count), E and H the tangential
 *   fields at every boundary; REFL = |r|^2, TRANS real (count); ABS real (nlayers, count) by flux telescoping.
 *   The field outputs are staged in fp64 before t scales them: in the outputs for PB_C128, in the handle's scratch for
 *   PB_C64.
 * pb_stack_grad: the thickness (PB_TF_GRAD_THICKNESS) and / or index (PB_TF_GRAD_INDEX) gradient of a scalar merit whose
 *   cotangents are the seeds (HOST array of 4 device pointers, fp64, NULL when absent): dR, dT (count), dA
 *   (nlayers, count), dEsq (nlayers + 1, count).  E and H are the complex128 boundary fields pb_stack_eval wrote in
 *   coatings mode.  grad: (nlayers) of dtype's real type, or (2, nlayers) thickness first when both kinds are asked.
 *   The sample sum is per-warp partials in the handle's scratch added in a fixed order by a second launch: no atomics,
 *   so repeated calls are bit-identical.
 * pb_field_at_depth: E, H (complex, nz) at depths z (fp64, nz) of a stack of nlayers >= 1 at one wavelength and angle:
 *   zb (fp64, nlayers + 1) the boundary depths, n (complex128, nlayers) the layer indices, E_b and H_b (complex128,
 *   nlayers + 1) the boundary fields pb_stack_eval wrote for that sample. */
typedef enum { PB_TF_THINFILM = 0, PB_TF_COATINGS = 1 } pb_tf_mode;
typedef enum { PB_TF_POL_S = 0, PB_TF_POL_P = 1 } pb_tf_pol;
typedef enum {
    PB_TF_IN_WVL = 0, PB_TF_IN_THETA = 1, PB_TF_IN_N0 = 2, PB_TF_IN_NSUB = 3, PB_TF_IN_N = 4, PB_TF_IN_D = 5,
    PB_TF_NOPS = 6
} pb_tf_operand;
typedef enum {
    PB_TF_OUT_R = 0, PB_TF_OUT_T = 1, PB_TF_OUT_E = 2, PB_TF_OUT_H = 3, PB_TF_OUT_REFL = 4, PB_TF_OUT_TRANS = 5,
    PB_TF_OUT_ABS = 6, PB_TF_OUT_ESQ = 7, PB_TF_OUT_ETA0 = 8, PB_TF_OUT_ETASUB = 9, PB_TF_NOUT = 10
} pb_tf_output;
typedef enum { PB_TF_GRAD_THICKNESS = 1, PB_TF_GRAD_INDEX = 2 } pb_tf_grad_kind;
enum { PB_TF_DIMS = 4 };
int pb_stack_eval(pb_handle_t h, int dtype, int mode, int pol, int flags, int nlayers, int ndim, const long long* shape,
                  const long long* strides, const void* const* in, double theta_scale, void* const* out, void* stream);
int pb_stack_grad(pb_handle_t h, int dtype, int pol, int kinds, int nlayers, int ndim, const long long* shape,
                  const long long* strides, const void* const* in, const void* E, const void* H, const void* const* seeds,
                  void* grad, void* stream);
int pb_field_at_depth(pb_handle_t h, int dtype, int pol, int nlayers, const void* z, long long nz, const void* zb,
                      const void* n, double n0_re, double n0_im, double wvl, double theta0, const void* E_b,
                      const void* H_b, void* E, void* H, void* stream);

/* ---- Coating design (prysm/x/coatings merit.py and needle.py) on the thin-film chain above ---------------------------
 * Operands: in[PB_CM_NOPS], strides[5 * PB_CM_NOPS] laid out as for pb_stack_eval; slots 0-5 are the six thin-film
 *   operands, then target and weight (fp64) and, for pb_needle only, the needle index (complex128; NULL otherwise).
 *   pol is PB_TF_POL_S, PB_TF_POL_P or PB_CM_POL_AVG: for avg one thread evaluates both polarisations, q is their mean
 *   and each is seeded with 2 w (q - target) / 2.  The quantity q (PB_CM_Q_*) of a sample is
 *   R; T; the absorptance of layer b0; |E|^2 at boundary b0; the largest |E|^2 over the nb boundaries of `blist`
 *   (device int array of 2 nb: the boundaries, then 1 where that listing is the boundary's last, else 0; the seed goes
 *   to the first maximum and only if its listing is the last); the mean of |E|^2 at boundaries b0 and b1.  Layer and
 *   boundary indices are non-negative and in range.
 * pb_coating_merit: flags (PB_CM_OUT_*) select the outputs: value (one fp64 device scalar) = sum of w (q - target)^2
 *   over the count samples; residuals (count, dtype's real type) = sqrt(w) (q - target); grad (nlayers, or (2, nlayers)
 *   thickness first when both kinds are asked) of the value.  With PB_CM_ACCUMULATE the value and the gradient are
 *   added to what value and grad hold (the gradient in dtype's real type).  One sample launch, then one fixed-order
 *   reduce launch when a value or gradient is asked; the forward vectors are staged in the handle's scratch, no
 *   atomics, so repeated calls are bit-identical.
 * pb_needle: P(z) of an R or T term at nz depths, summed over the samples.  zlist (device int array of nlayers + 1 +
 *   nz) holds the start offset of each layer's run and then the depth indices grouped by layer j, the layer a depth is
 *   evaluated in; zpart (fp64, (2, nz)) holds each depth's partial thicknesses z - Z_j, then Z_{j+1} - z.  P (nz, dtype's real type) is written, or added
 *   to with accumulate != 0.  Two launches, no atomics. */
typedef enum { PB_CM_IN_TARGET = 6, PB_CM_IN_WEIGHT = 7, PB_CM_IN_NEEDLE = 8, PB_CM_NOPS = 9 } pb_cm_operand;
typedef enum {
    PB_CM_Q_R = 0, PB_CM_Q_T = 1, PB_CM_Q_ABS = 2, PB_CM_Q_ESQ = 3, PB_CM_Q_PEAK = 4, PB_CM_Q_LAYER = 5
} pb_cm_quantity;
typedef enum { PB_CM_POL_AVG = 2 } pb_cm_pol;
typedef enum {
    PB_CM_OUT_VALUE = 1, PB_CM_OUT_RESIDUALS = 2, PB_CM_OUT_GRAD_THICKNESS = 4, PB_CM_OUT_GRAD_INDEX = 8,
    PB_CM_ACCUMULATE = 16
} pb_cm_flag;
int pb_coating_merit(pb_handle_t h, int dtype, int quantity, int pol, int flags, int nlayers, int ndim,
                     const long long* shape, const long long* strides, const void* const* in, int b0, int b1,
                     const void* blist, int nb, void* value, void* residuals, void* grad, void* stream);
int pb_needle(pb_handle_t h, int dtype, int quantity, int pol, int nlayers, int ndim, const long long* shape,
              const long long* strides, const void* const* in, const void* zpart, long long nz, const void* zlist, void* P,
              int accumulate, void* stream);

/* ---- Optical monitoring (prysm/x/coatings monitoring.py) on the thin-film chain above -------------------------------
 * The monitor signal of a (B, C) = v is R = |r|^2 (PB_MON_R) or T = Re eta_sub / Re eta0 |t|^2 (PB_MON_T), r and t as
 *   in coatings mode.  All arithmetic is fp64; outputs are rounded once to dtype's real type.
 * pb_monitor_runs: simulate_run for `runs` as-built runs in one launch, one CTA per run; run r monitors at candidate
 *   c = r / per_cand (runs <= ncand * per_cand).  in (HOST array of PB_TF_NOPS device pointers, dense): wavelength,
 *   angle (radians), ambient and substrate index (ncand each), the layer indices (complex128, (nlayers, ncand)) at each
 *   candidate's wavelength, and the nominal thicknesses (fp64, nlayers).  From v = [1, eta_sub], for k = nlayers - 1,
 *   ..., 0 the signal of M_k(d_j) v is taken on the grid d_j = numpy.linspace(start, max_factor d_k, n_points), and
 *   the layer stops at
 *     PB_MON_LEVEL: the crossing of the level levels[c, k] (+ err[r, k]) nearest d_k, the first on a tie, at
 *       d_i + frac (d_i+1 - d_i), frac = -s_i / (s_i+1 - s_i) (0 when equal), s = signal - level, a crossing wherever
 *       sign(s_i) != sign(s_i+1); with none, the d of the first minimum of |s|.  levels (fp64, (ncand, nlayers));
 *       n_points >= 1.
 *     PB_MON_TURNING: the turning_index-th (>= 1) turning point, i + 1 wherever sign(sig_i+1 - sig_i) changes, or d_k
 *       when there are fewer; then + err[r, k].
 *   asbuilt[r, k] = max(d_real, 0), and v <- M_k(asbuilt[r, k]) v in fp64.  err (fp64, (runs, nlayers)) may be NULL.
 *   Fixed-order block reductions, no atomics: repeated calls are bit-identical.
 * pb_monitor_cut: level_cut (PB_MON_LEVEL: out[0] = the cut at `level` nearest `target`, NaN for the first crossing;
 *   n >= 1) or turning_points (PB_MON_TURNING: out[0, *count) = the d of every turning point, count one device int64) of
 *   the trace d, sig (n each, dtype's real type), with the arithmetic in that type.  One launch.
 * pb_monitor_jacobian: J[c, w, k] = (Rr[c (nlayers + 1) + 1 + k, w] - Rr[c (nlayers + 1), w]) / eps for the realized
 *   reflectance Rr (fp64, (ncand (nlayers + 1), nw)) of each candidate's base run followed by its nlayers perturbed
 *   runs, and score[c] = sqrt(sum over w, k of J^2) by the fixed-order grid fold (DESIGN.md §4.4).  J ((ncand, nw,
 *   nlayers)) or score (ncand) may be NULL.  One launch, ncand <= 65535. */
typedef enum { PB_MON_LEVEL = 0, PB_MON_TURNING = 1 } pb_mon_strategy;
typedef enum { PB_MON_R = 0, PB_MON_T = 1 } pb_mon_mode;
int pb_monitor_runs(pb_handle_t h, int dtype, int strategy, int mode, int pol, int nlayers, long long ncand,
                    const void* const* in, long long runs, long long per_cand, const void* err, const void* levels,
                    long long n_points, double start, double max_factor, int turning_index, void* asbuilt, void* stream);
int pb_monitor_cut(pb_handle_t h, int dtype, int strategy, const void* d, const void* sig, long long n, double level,
                   double target, void* out, void* count, void* stream);
int pb_monitor_jacobian(pb_handle_t h, int dtype, int ncand, int nlayers, long long nw, const void* Rr, double eps,
                        void* J, void* score, void* stream);

/* ---- PSF / MTF analysis (prysm/_richdata.py, prysm/coordinates.py uniform_cart_to_polar, prysm/psf.py, prysm/otf.py) --
 * Data is (ny, nx) on the fp64 ascending axes xax (nx) and yax (ny), device arrays.  Every sampling entry point uses one
 * linear interpolator, scipy's RegularGridInterpolator(method='linear'): interval = the largest i with axis[i] <= p
 * clipped to [0, n - 2]; fp64 weights; the four corners summed in scipy's order without fused multiply-add, so a NaN
 * at any corner gives NaN even at weight 0; a point outside the axes gives `fill`.  An axis of one sample has weight 0.
 * The polar lattice is uniform_cart_to_polar's: rho_j = linspace(0, rmax, nx), phi_i = linspace(0, 2 pi, ny), the
 * point (rho_j cos phi_i, rho_j sin phi_i), fill 0, all in fp64; it is (ny, nx), phi along rows.
 * pb_interp2d_linear: type PB_ELEM_F32 / F64 / C64 / C128; rows of data are ld elements apart.  mode PB_INTERP_POINTS:
 *   out[k] = f(px[k], py[k]) (fp64 device arrays, count points); PB_INTERP_POLAR: out (ny, nx) = f on the lattice
 *   (px, py, count and fill unused).  out has data's type.  One launch.
 * pb_azimuthal_stats: type PB_ELEM_F32 / F64, data dense.  For every rho column j of the lattice, the statistics over
 *   phi that `stats` (a mask of pb_az_stat) asks for, ignoring NaN, into row log2(bit) of out (6, nx) of data's type:
 *   count, mean, variance (ddof 0, two passes), min, max, median (the mean of the two middle values for an even count).
 *   A column without a number gives NaN (count 0).  One launch; one block per column holds its ny samples in shared
 *   memory, so ny <= PB_AZ_MAX_NY (else PB_ERR_INVALID before any launch).  fp64 arithmetic, fixed-order reductions.
 * pb_polar_crossings: estimate_size's core.  The level is metric (relative = 0) or metric * the lattice maximum
 *   (relative != 0; NaN if any lattice sample is NaN).  Along each phi row, the first (last = 0) or last i with
 *   (v[i] > level) != (v[i + 1] > level) gives the radius rho_i + frac (rho_{i+1} - rho_i), frac = (level - v[i]) /
 *   (v[i + 1] - v[i]), 0 where v[i + 1] == v[i].  result (HOST, 2): the number of rows that cross, and the fixed-order
 *   fp64 mean of their radii.  A crossing next to a NaN sample counts and has a NaN radius, so the mean is NaN; only
 *   rows without a transition stay out.  Up to four launches in the handle's scratch; the call waits for them.
 * pb_analytic_radial: out[k] = f(x[k]) in fp64, rounded once to out_type (in_type, out_type PB_ELEM_F32 / F64);
 *   a = wavelength, b = F/#.  jinc(u) = j1(u) / u, 0.5 for |u| < 1e-8; core(s) = (2 / pi)(acos s - s sqrt(1 - s^2)).
 *   PB_AR_AIRYDISK (2 jinc(u))^2 and PB_AR_AIRYDISK_EFIELD 2 jinc(u), u = x pi / a / b;  PB_AR_AIRYDISK_FT core(min(|x| /
 *   (1 / (a b)), 1));  PB_AR_DIFFLIM_MTF core(min(|x / (1 / (a / 1000 b))|, 1));  PB_AR_DIFFLIM_NORMALIZED core(min(x,
 *   1));  PB_AR_EE_CIRCULAR 1 - J0(p)^2 - J1(p)^2, p = x pi / b / a.  One launch. */
typedef enum { PB_INTERP_POINTS = 0, PB_INTERP_POLAR = 1 } pb_interp_mode;
typedef enum {
    PB_AZ_COUNT = 1, PB_AZ_MEAN = 2, PB_AZ_VAR = 4, PB_AZ_MIN = 8, PB_AZ_MAX = 16, PB_AZ_MEDIAN = 32, PB_AZ_ALL = 63
} pb_az_stat;
typedef enum { PB_AZ_MAX_NY = 28672 } pb_az_limit;
typedef enum {
    PB_AR_AIRYDISK = 0, PB_AR_AIRYDISK_EFIELD = 1, PB_AR_AIRYDISK_FT = 2, PB_AR_DIFFLIM_MTF = 3, PB_AR_DIFFLIM_NORMALIZED = 4,
    PB_AR_EE_CIRCULAR = 5
} pb_analytic_kind;
int pb_interp2d_linear(pb_handle_t h, int type, const void* data, int ny, int nx, long long ld, const double* xax,
                       const double* yax, int mode, const double* px, const double* py, long long count, double rmax,
                       double fill, void* out, void* stream);
int pb_azimuthal_stats(pb_handle_t h, int type, const void* data, int ny, int nx, const double* xax, const double* yax,
                       double rmax, int stats, void* out, void* stream);
int pb_polar_crossings(pb_handle_t h, int type, const void* data, int ny, int nx, const double* xax, const double* yax,
                       double rmax, double metric, int relative, int last, double* result, void* stream);
int pb_analytic_radial(pb_handle_t h, int in_type, int out_type, int kind, const void* x, long long count, double a,
                       double b, void* out, void* stream);

/* ---- Interferometric metrology (prysm/interferogram.py, prysm/util.py, prysm/polynomials/fitting.py lstsq) ----------
 * Real data of dtype's real type (PB_C64: fp32, PB_C128: fp64), dense (ny, nx) or n elements.  Every reduction is the
 * library's fixed-order grid fold (DESIGN.md §4.4), so repeated calls give the same bits.
 * pb_nan_stats: res (DEVICE, 9 fp64) = finite count, sum, min, max and sum of squares of the finite values, NaN count,
 *   mean, then sum |x - mean| and sum (x - mean)^2 over the finite values (pass 2 reads the mean from res).  Two launches.
 * pb_masked_gram: modes (HOST array of k device pointers, NULL = the constant 1), each n elements; data n elements with
 *   NaN (or inf) for pixels to ignore.  out (DEVICE, fp64) = the packed row-major upper triangle of the (k+1) x (k+1)
 *   matrix [A d]^T [A d] over the finite pixels: A^T A, then A^T d in column k, and d^T d last.  1 <= k <= PB_GRAM_MAX_K.
 *   One launch.
 * pb_psd_prologue: the window w of make_window (PB_WIN_WELCH: 1 - |hypot(x, y) / rmax|^alpha on the fftrange * dx grid;
 *   PB_WIN_HANN: np.outer(np.hanning(ny), np.hanning(nx)); PB_WIN_USER: the array `user`; PB_WIN_AUTO: Welch when every
 *   sample of the four corner rectangles (HOST int[16], (y0, y1, x0, x1) each) is == 0, else Hann, decided on the
 *   device into flags (DEVICE int[4])).  Writes `window` = w and / or `shifted` = fftshift(height * w) (either may be
 *   NULL) and s2 (DEVICE fp64) = sum w^2.  One launch, two for PB_WIN_AUTO.
 * pb_psd_epilogue: psd = ifftshift(|F|^2) / (s2 fs^2) for the complex (ny, nx) F = pb_fft2 of `shifted`.  One launch.
 * pb_band_trapz: res (DEVICE fp64) = sum_ij wy_i wx_j psd_ij over the samples with flow <= r_ij <= fhigh, w = 1/2 on the
 *   edges of an axis (0 for an axis of one sample), the trapezoid of bandlimited_rms without its dx^2; r is the array r
 *   or, when r is NULL, hypot(fx[j], fy[i]) of the fp64 axes.  twod = 0: one trapezoid along the ny axis (nx = 1).
 * pb_filter_h: out0 (and out1, with fcn1) = the factors `parts` (PB_FILT_*) asks for: W = hann2d(ny, nx), H =
 *   ideal_lpf_iir2d(r, dx, fcn).  One launch.
 * pb_filter_apply: H from the complex transforms Hl (and Hh) by typ (PB_FILT_LOWPASS |Hl|, HIGHPASS 1 - |Hl|, BANDPASS
 *   1 - ((1 - |Hh|) + |Hl|), BANDREJECT (1 - |Hh|) + |Hl|); D *= H in place, or with D NULL H into the real Hout.
 * pb_gradient2d: gx, gy = np.gradient(f, dx) (central inside, one-sided first order on the edges) and gr = hypot(gx, gy);
 *   ny, nx >= 2.  One launch.
 * pb_finite_bounds: box (HOST int[4]) = max(ny - i), max(i + 1), max(nx - j), max(j + 1) over the finite samples (all 0
 *   when there is none).  One launch; the call waits for it.
 * pb_metro_pointwise: out (may be x) = PB_PW_FILL NaN -> a; KEEP NaN where the byte mask m is 0; CLIP NaN where |x| > a;
 *   RADIUS NaN where u / a > 1; SUB x - (a u + b v) (u NULL = 1, v NULL = 0); RHO2 rho^2 of np.linspace(-1, 1) axes whose steps
 *   2 / (n - 1) are a (x) and b (y), x unused; REAL the real part of the complex x; AXPBY a u + b v (v NULL = 0, x unused); DIV x / a; WELCH
 *   1 - |x / a|^b.  One launch. */
typedef enum { PB_GRAM_MAX_K = 64 } pb_gram_limit;
typedef enum { PB_WIN_AUTO = 0, PB_WIN_WELCH = 1, PB_WIN_HANN = 2, PB_WIN_USER = 3 } pb_window_kind;
typedef enum { PB_FILT_W = 1, PB_FILT_H = 2 } pb_filter_part;
typedef enum { PB_FILT_LOWPASS = 0, PB_FILT_HIGHPASS = 1, PB_FILT_BANDPASS = 2, PB_FILT_BANDREJECT = 3 } pb_filter_type;
typedef enum {
    PB_PW_FILL = 0, PB_PW_KEEP = 1, PB_PW_CLIP = 2, PB_PW_RADIUS = 3, PB_PW_SUB = 4, PB_PW_RHO2 = 5, PB_PW_REAL = 6,
    PB_PW_AXPBY = 7, PB_PW_DIV = 8, PB_PW_WELCH = 9
} pb_pointwise_op;
int pb_nan_stats(pb_handle_t h, int dtype, const void* x, long long n, double* res, void* stream);
int pb_masked_gram(pb_handle_t h, int dtype, const void* const* modes, int k, const void* data, long long n, double* out,
                   void* stream);
int pb_psd_prologue(pb_handle_t h, int dtype, const void* height, int ny, int nx, int kind, const void* user, double dx,
                    double alpha, double rmax, const int* corners, void* shifted, void* window, double* s2, int* flags,
                    void* stream);
int pb_psd_epilogue(pb_handle_t h, int dtype, const void* F, int ny, int nx, const double* s2, double fs, void* psd,
                    void* stream);
int pb_band_trapz(pb_handle_t h, int dtype, const void* psd, const void* r, const double* fx, const double* fy, int ny,
                  int nx, int twod, double flow, double fhigh, double* res, void* stream);
int pb_filter_h(pb_handle_t h, int dtype, const void* r, int ny, int nx, int parts, double dx, double fcn0, double fcn1,
                void* out0, void* out1, void* stream);
int pb_filter_apply(pb_handle_t h, int dtype, void* D, const void* Hl, const void* Hh, long long n, int typ, void* Hout,
                    void* stream);
int pb_gradient2d(pb_handle_t h, int dtype, const void* f, int ny, int nx, double dx, void* gx, void* gy, void* gr,
                  void* stream);
int pb_finite_bounds(pb_handle_t h, int dtype, const void* x, int ny, int nx, int* box, void* stream);
int pb_metro_pointwise(pb_handle_t h, int dtype, int op, const void* x, const void* u, const void* v, const void* m,
                       int ny, int nx, double a, double b, void* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PRYSM_B200_H */
