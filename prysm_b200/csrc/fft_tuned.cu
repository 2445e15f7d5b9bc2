// Tuned register-resident FFT kernels for the headline path: Wavefront.focus / unfocus with Q = 2
// on N x N complex64 pupils, N in {512, 1024, 2048}  (reference prysm/propagation/fft.py:7-65).
//
// Algebra.  K = 2N.  focus = fftshift(FFT2_K(ifftshift(pad(x)))).  Along one axis, with q = x
// zero-extended to K:   U[k] = (-dir*i)^k * Q[k]   (the centred pad + ifftshift is a circular
// shift by K/4), and the zero half makes the first radix-2 level trivial:
//      Q[2j]   = FFT_N(x)[j]                    ("even" half, lane A)
//      Q[2j+1] = FFT_N(x * w_K^n)[j]            ("odd" half,  lane B)
// so every length-K transform of the padded data is two length-N transforms of the un-padded
// data, the shifts are sign patterns / index rotations at the store, and no zero is ever read,
// written or multiplied.
//
// Two-lane arithmetic.  Each thread carries two transforms in structure-of-arrays form -- re = (re_A, re_B),
// im = (im_A, im_B) -- and every butterfly, twiddle multiply and store acts on the pair (add2 / mul2 / fma2 in
// fft_engine.cuh): one set of index arithmetic, shared-memory addressing and twiddle loads serves two transforms.
//
// Data flow (columns first so that the K x K output is written by the row kernel in full rows with 128-bit stores),
// one field per launch pair:
//   focus_col4_kernel : persistent, one 512-thread CTA per SM walking the 4-column tiles of the field.  Each tile comes
//                       in by tensor TMA (box = 4 columns x 256 rows, 32-byte runs gathered into a contiguous [row][4]
//                       image); a thread's two lanes are two adjacent columns, and group h of the CTA computes half h
//                       (h = 1 multiplies the input ramp w_K^n in: w_32^(n/NT) as immediates, w_2L^t per thread).
//                       Output: the intermediate [2][N][N] (plane p, row j  <->  output row 2j+p, rotated by K/2),
//                       TILE-MAJOR: [plane p][j / 4][column tile = col / 4][j % 4][col % 4] complex64, i.e. the 4 x 4
//                       block (4 output rows of one plane, 4 adjacent columns) is one 128-byte line and a warp stores
//                       two full lines per instruction.
//   focus_row4_kernel : persistent, four line groups per CTA (GeoR4); each intermediate row (512 runs of 32 bytes, 128
//                       bytes apart) is gathered by two tensor-TMA boxes, one row ahead; per row both half-transforms,
//                       lanes A and B, whose stage-1 twiddles differ by the per-thread w_2L^t; a thread owns outputs
//                       (2j, 2j+1) and stores them as one float4.
// Inputs tensor TMA cannot gather -- the fused phase-screen input PB_IN_AMP_OPD, a complex input with an odd pitch or a
// base off 16-byte alignment -- are first written, one field at a time, as a dense aligned N x N field in scratch slot 1
// (the phase-screen kernel of elementwise.cu, or one cudaMemcpy2DAsync) and then take the same pair.
//
// HBM traffic at N = 2048: pupil 8N^2 once, output 8K^2 once.  Plane 0 of the 16N^2-byte intermediate (the even output
// rows, 32 MiB) stays in L2: the column kernel writes it evict_last, the row kernel reads it first and then discards each
// line (discard.global.L2), so it never reaches HBM in either direction.  So do the first kPlane1KeepBytes of plane 1,
// which the row kernel reads next; the rest of plane 1 (30 MiB) is written evict_first and makes the trip.  A staged
// input adds the staging pass: its source read once and 8N^2 written.  The fields of a stack alternate between two
// intermediates, so that the column kernel of field f + 1 runs under the tail of field f's row kernel instead of
// waiting for it (focus_col4_kernel).
//
// FFT_N engine: N/16 threads per line, 16 points x 2 lanes per thread in registers, radix
// 16 x 16 x N/256, two shared-memory exchanges of float4 (1-in-16 padded, conflict free).
#include "fft_engine.cuh"

namespace pb {
namespace {

// share of plane 0's lines written evict_last (the rest evict_first): what the H100's 50 MB L2 keeps next to the
// streaming input and plane 1
constexpr float kPlane0Keep = 1.0f;
// bytes of plane 1 kept in L2 as well, from its first line group on: the row kernel reads them right after plane 0 and
// discards them in the same way.  Chosen by a sweep at N = 2048 (DESIGN §4.1)
constexpr long long kPlane1KeepBytes = 2LL << 20;
// ... in line groups of an L-point field (L/4 lines of 128 bytes each): at most all of plane 1, and a multiple of L/64
// (whole thread ranges of the column kernel's stores, so that its choice of policy is a compile-time one)
template <int L> constexpr int plane1_keep() {
    const long long g = kPlane1KeepBytes / (32LL * L);
    return (int)((g < L / 4 ? g : L / 4) / (L / 64) * (L / 64));
}


template <int L, bool INV, int HALF>
__device__ __forceinline__ void focus_col4_group(const CUtensorMap& in_map, const FocusParams& p, float4* smem4, uint64_t* bar) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    constexpr int NT = G::NT;
    const int lt = threadIdx.x & (2 * NT - 1);                       // thread within the group
    const int cp = lt & 1, t = lt >> 1;
    const float4* __restrict__ stage = smem4 + G4::STAGE;
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smem4 + G4::PLAN2);
    float4* S = smem4 + (HALF * 2 + cp) * G4::XBUF;
    const SyncGroup gsync{1 + HALF, 2 * NT};
    // plane 0 is read back first by the row kernel that follows: it stays in L2 (and is discarded there); plane 1 streams,
    // but for its first KEEP1 line groups (rows j < 4 KEEP1), which the row kernel reads next and which stay as well
    constexpr int KEEP1 = plane1_keep<L>();
    const uint64_t pol_tmp = (HALF == 0 && (p.hints & 4)) ? l2_policy_last_first(kPlane0Keep) : l2_policy((p.hints & 1) ? 1 : 0);
    const uint64_t pol_tmp1 = (HALF == 1 && KEEP1 > 0 && (p.hints & 4)) ? l2_policy_last_first(kPlane0Keep) : pol_tmp;
    const uint64_t pol_in = l2_policy((p.hints & 1) ? 1 : 0);
    auto request_tile = [&](int ww) {   // one thread: gather tile ww = (field, column tile) into the staging area
        const int fb = ww / G2::TILES, tile = ww - fb * G2::TILES;
        mbar_expect_tx(bar + 1, (uint32_t)(L * 4 * sizeof(float2)));
#pragma unroll
        for (int b = 0; b < G2::NBOX_IN; ++b)
            tma_load_3d(smem4 + G4::STAGE + b * G2::BOXR * 2, &in_map, tile * 4, b * G2::BOXR, fb, bar + 1, pol_in);
    };
    // Tiles are handed out at run time: the first wave statically (CTA b: tile b), every later one by an atomic counter,
    // so that the CTAs that start early -- on the SMs the previous row kernel's last wave leaves idle -- take more tiles.
    // The tile of iteration it goes to slot[it & 1] before the arrival on bar[1] that the gather completes, so a thread
    // reads it after its wait; p.ntiles there means "no more": the arrival is then a plain one.
    int* slot = reinterpret_cast<int*>(bar + 3);
    auto claim = [&](int it_next) {   // one thread, the staging area free: the CTA's tile of iteration it_next
        const int ww = it_next == 0 ? (int)blockIdx.x : (int)gridDim.x + (int)atomicAdd(p.tile_ctr, 1u);
        const int wc = ww < p.ntiles ? ww : p.ntiles;
        slot[it_next & 1] = wc;
        if (wc < p.ntiles) request_tile(wc);
        else mbar_arrive(bar + 1);
    };
    unsigned int* released = reinterpret_cast<unsigned int*>(bar + 2);   // warps that hold the inputs of the current tile, summed over tiles
    if (HALF == 0 && lt == 0) {
        mbar_expect_tx(bar, (uint32_t)(G4::PLANLEN * sizeof(float2)));
        bulk_g2s(smem4 + G4::PLAN2, p.plan, (uint32_t)(G4::PLANLEN * sizeof(float2)), bar);
        claim(0);
    }
    const float sgn = (t & 1) ? -1.0f : 1.0f;
    float2 u = make_float2(1.f, 0.f);
    if (HALF) { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u = make_float2(cs, sn); }   // w_2L^t = exp(-i pi t / L)
    mbar_wait(bar, 0);   // plan
    for (int it = 0;; ++it) {
        mbar_wait(bar + 1, it & 1);
        const int w = slot[it & 1];
        if (w >= p.ntiles) break;
        const int fb = w / G2::TILES, tile = w - fb * G2::TILES;
        auto sync = [&]() { gsync(); };
        P2 v[16];
        {
            float4 x[16];   // (col, col + 1) x (re, im)
            const float4* __restrict__ sg = stage + lt;   // ((n*NT + t)*2 + cp)
#pragma unroll
            for (int n = 0; n < 16; ++n) x[n] = sg[n * NT * 2];
            // lanes = the two columns; HALF 1 multiplies both by w_32^n (the n-dependent part of the input ramp)
#define PB_LANES2(n)                                                                                              \
            if (HALF == 0) v[n] = {make_float2(x[n].x, x[n].z), make_float2(x[n].y, x[n].w)};                          \
            else {                                                                                                     \
                const P2 a_ = make_lanes<INV, n>(make_float2(x[n].x, x[n].y)), b_ = make_lanes<INV, n>(make_float2(x[n].z, x[n].w)); \
                v[n] = {make_float2(a_.re.y, b_.re.y), make_float2(a_.im.y, b_.im.y)};                                 \
            }
            PB_LANES2(0) PB_LANES2(1) PB_LANES2(2) PB_LANES2(3) PB_LANES2(4) PB_LANES2(5) PB_LANES2(6) PB_LANES2(7)
            PB_LANES2(8) PB_LANES2(9) PB_LANES2(10) PB_LANES2(11) PB_LANES2(12) PB_LANES2(13) PB_LANES2(14) PB_LANES2(15)
#undef PB_LANES2
            __syncwarp();
            if ((threadIdx.x & 31) == 0) {   // this warp holds its inputs: one of 16 releases of the staging area per tile;
                __threadfence_block();       // the LAST warp to release it requests the next tile on the spot
                const unsigned int n = atomicAdd(released, 1u) + 1u;
                __threadfence_block();
                if (n == (unsigned int)(it + 1) * (4 * NT / 32)) {
                    fence_proxy_async();
                    claim(it + 1);
                }
            }
        }
        fft_two_stages_u<L, INV, HALF>(v, t, S, plan + G4::TW1, plan + G4::TW2, u, sync);
        fft_last_stage_load<L, INV>(v, t, S);
        sync();   // this group's exchange buffers are free for its next tile
#pragma unroll
        for (int g = 0; g < G::GI; ++g) dftR<G::R3, INV>(v + g * G::R3);
        // tile-major store: element (plane, j, tile, c) at ((plane*L/4 + j/4) * TILES + tile) * 16 + (j%4)*4 + c ; c = 2 cp
        float4* __restrict__ dst = reinterpret_cast<float4*>(
            p.tmp + fb * (2LL * L * L) + (long long)HALF * L * L + ((long long)(t >> 2) * G2::TILES + tile) * 16 + (t & 3) * 4 + 2 * cp);
#pragma unroll
        for (int g = 0; g < G::GI; ++g)
#pragma unroll
            for (int kk = 0; kk < G::R3; ++kk) {
                const P2 y = v[g * G::R3 + kk];
                const long long o = (long long)((g * NT + 256 * kk) >> 2) * (G2::TILES * 8);   // float4 units
                // (-dir*i)^k with k = 2j + HALF; j has the parity of t.  HALF 1: times (-dir*i): forward (-im, re), inverse (im, -re)
                float4 q;
                if (HALF == 0) q = make_float4(sgn * y.re.x, sgn * y.im.x, sgn * y.re.y, sgn * y.im.y);
                else q = INV ? make_float4(sgn * y.im.x, -sgn * y.re.x, sgn * y.im.y, -sgn * y.re.y)
                             : make_float4(-sgn * y.im.x, sgn * y.re.x, -sgn * y.im.y, sgn * y.re.y);
                // rows g NT + 256 kk + t, t < NT: all below 4 KEEP1 (a multiple of NT) or none
                st_hint(dst + o, q, (HALF == 1 && g * NT + 256 * kk < 4 * KEEP1) ? pol_tmp1 : pol_tmp);
            }
    }
}

template <int L, bool INV>
__global__ void __launch_bounds__(Geo4<L>::THREADS) focus_col4_kernel(const __grid_constant__ CUtensorMap in_map, const FocusParams p) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    extern __shared__ __align__(128) float4 smem4[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(smem4) + G4::BAR_OFF);   // [0] plan [1] tile full [2] tile free
    if (threadIdx.x == 0) {
        mbar_init(bar, 1);
        mbar_init(bar + 1, 1);
        *reinterpret_cast<unsigned int*>(bar + 2) = 0u;   // release counter of the staging area
        mbar_fence_init();
    }
    // every CTA of the grid is resident (one per SM, grid <= SMs): the row kernel that follows may take each SM this
    // kernel's last wave frees, and run its prologue there
    pdl_launch_dependents();
    if (!p.early_input) pdl_wait();
    __syncthreads();
    const int grp = threadIdx.x / (2 * G::NT);
    if (grp == 0) focus_col4_group<L, INV, 0>(in_map, p, smem4, bar);
    else focus_col4_group<L, INV, 1>(in_map, p, smem4, bar);
    // Field f of a call writes intermediate buffer f mod 2, so col(f + 1) writes the buffer row(f - 1) read and discarded,
    // never the one row(f), its predecessor in the stream, is reading: it does not wait before its stores.  That they
    // follow all of row(f - 1)'s reads and discards rests on griddepcontrol alone:
    //   * griddepcontrol.wait returns once the prerequisite grid has completed and its memory operations are performed
    //     and visible.  Every dependent column kernel executes it (here, or before its first gather when its input may
    //     overlap the output), so col(f) completes only after row(f - 1) has completed;
    //   * row(f) executes griddepcontrol.launch_dependents only after its own griddepcontrol.wait, i.e. after col(f) has
    //     completed, and col(f + 1) is launched only once every CTA of row(f) has done so (or exited).
    // So no CTA of col(f + 1) exists before row(f - 1) has completed.  The same chain orders row(f) after row(f - 1) --
    // their outputs may be the same plane (accumulated intensity) -- and the plain launch of a call's first column kernel
    // orders it after everything before it in the stream.
    if (p.early_input) pdl_wait();
}

template <int L, bool INV>
__global__ void __launch_bounds__(4 * L / 16) focus_row4_kernel(const __grid_constant__ CUtensorMap tmp_map, const FocusParams p) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using R4 = GeoR4<L, plane1_keep<L>()>;
    constexpr int NT = G::NT, R3 = G::R3, GI = G::GI;
    constexpr uint32_t ROW_BYTES = L * sizeof(float2);
    extern __shared__ __align__(128) unsigned char smraw[];
    const int grp = threadIdx.x / NT, t = threadIdx.x - grp * NT;
    float4* S = reinterpret_cast<float4*>(smraw + grp * R4::GROUP);      // this group's exchange buffer
    float2* inb = reinterpret_cast<float2*>(S + G::SBUF);                 // ... and L-element input row
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smraw + R4::PLAN_OFF);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smraw + R4::BAR_OFF);   // [0] plan, [1 + grp] row of group grp
    uint64_t* bar = bars + 1 + grp;
    const uint64_t pol_tmp = l2_policy((p.hints & 1) ? 1 : 0), pol_out = l2_policy((p.hints & 1) ? 1 : 0);
    // the kept rows, plane 0 and the first KEEP1 line groups of plane 1 (p.hints & 4): read evict_last so that no line
    // leaves L2 -- written back -- before all four of its rows are read; then discarded
    const uint64_t pol_keep = l2_policy((p.hints & 4) ? 2 : 0);
    auto request_row = [&](int R) {   // one thread: gather intermediate row R = (field, plane, j) into `inb`
        const int fb = R / (2 * L), rf = R - fb * (2 * L);
        const int ph = rf / L, j = rf - ph * L;
        const int grow = (fb * 2 + ph) * (L / 4) + (j >> 2);
        const uint64_t pol = rf < 4 * R4::NKEEP && (p.hints & 4) ? pol_keep : pol_tmp;
        mbar_expect_tx(bar, ROW_BYTES);
#pragma unroll
        for (int b = 0; b < G2::NBOX_ROW; ++b) tma_load_4d(inb + b * G2::BOXT * 4, &tmp_map, 0, j & 3, b * G2::BOXT, grow, bar, pol);
    };
    int r = blockIdx.x * 4 + grp;
    const int rstep = gridDim.x * 4;
    // Discard of the kept line groups (one field per launch: rows R < 4 NKEEP, R / 4 = line group; plane 1's follow plane
    // 0's).  The four groups of the CTA read the four rows j % 4 = 0..3 of the same line group at the same iteration, and
    // no other CTA reads those lines.  Each group counts itself in arrived[it] once its row is in shared memory; the last
    // of the four drops the group's lines from L2.
    unsigned int* arrived = reinterpret_cast<unsigned int*>(smraw + R4::CNT_OFF);
    unsigned int* last = arrived + R4::NKEEP;   // [grp]: this group arrived last at its current line group
    for (int i = threadIdx.x; i < R4::NCNT; i += blockDim.x) arrived[i] = 0u;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 5; ++i) mbar_init(bars + i, 1);
        mbar_fence_init();
        mbar_expect_tx(bars, (uint32_t)(G4::PLANLEN * sizeof(float2)));
        bulk_g2s(smraw + R4::PLAN_OFF, p.plan, (uint32_t)(G4::PLANLEN * sizeof(float2)), bars);
    }
    // The intermediate comes from the column kernel before this one: wait for it to complete (the prologue above -- the
    // static plan -- overlapped its tail).  Only then let the next field's column kernel be launched, to take the SMs
    // this grid's last wave frees: it writes the buffer the row kernel before this one read (see focus_col4_kernel)
    pdl_wait();
    pdl_launch_dependents();
    // the column kernel is complete: its tile counter is free for the column kernel two fields on, which starts only after
    // this kernel has completed (the chain in focus_col4_kernel)
    if (blockIdx.x == 0 && threadIdx.x == 0) *p.tile_ctr = 0u;
    __syncthreads();
    if (t == 0 && r < p.nrows) request_row(r);
    const SyncGroup gsync{1 + grp, NT};
    float2 u;
    { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u = make_float2(cs, sn); }   // w_2L^t
    const float sgn = ((t & 1) ? -1.0f : 1.0f) * p.scale;
    mbar_wait(bars, 0);
    for (int it = 0; r < p.nrows; ++it, r += rstep) {
        P2 v[16];
        mbar_wait(bar, it & 1);
        const bool drop = (p.hints & 4) && r < 4 * R4::NKEEP;
        if (drop && t == 0) {
            __threadfence_block();
            last[grp] = atomicAdd(arrived + it, 1u) == 3u;
        }
        {
            const float2* __restrict__ row = inb + t;
#define PB_X(n) row[(n) * NT]
            PB_MAKE_LANES_16(v, INV, PB_X)
#undef PB_X
        }
        const int rn = r + rstep;
        // ---- stage 1
        dft16<INV>(v);
        v[0] = mul_tw<INV>(v[0], make_float4(1.0f, u.x, 0.0f, u.y));
#pragma unroll
        for (int k = 1; k < 16; ++k) {
            const float2 w = plan[G4::TW1 + k * NT + t];
            const float2 wb = make_float2(fmaf(w.x, u.x, -w.y * u.y), fmaf(w.x, u.y, w.y * u.x));
            v[k] = mul_tw<INV>(v[k], make_float4(w.x, wb.x, w.y, wb.y));
        }
        {
            float4* __restrict__ d = S + t * 17;
#pragma unroll
            for (int k = 0; k < 16; ++k) d[k] = pack(v[k]);
        }
        gsync();   // every thread of the group holds its inputs in registers: the row buffer is free
        if (t == 0 && rn < p.nrows) {
            fence_proxy_async();
            request_row(rn);
        }
        if (drop && last[grp]) {   // all four rows of line group r / 4 are in shared memory: its lines are dead
            const char* lines = reinterpret_cast<const char*>(p.tmp) + (size_t)(r >> 2) * (G2::TILES * 128);
#pragma unroll
            for (int i = 0; i < G2::TILES / NT; ++i) l2_discard(lines + (size_t)(t + i * NT) * 128);
        }
        {
            const float4* __restrict__ s4 = S + pad16(t);
#pragma unroll
            for (int n = 0; n < 16; ++n) v[n] = unpack(s4[n * (NT + NT / 16)]);
        }
        gsync();
        // ---- stage 2
        dft16<INV>(v);
        {
            const int m = t >> 4, a = t & 15;
#pragma unroll
            for (int k = 1; k < 16; ++k) {
                const float2 w = plan[G4::TW2 + (k - 1) * (NT / 16) + m];
                v[k] = mul_tw<INV>(v[k], make_float4(w.x, w.x, w.y, w.y));
            }
            float4* __restrict__ d = S + m * 272 + a;
#pragma unroll
            for (int k = 0; k < 16; ++k) d[17 * k] = pack(v[k]);
        }
        gsync();
        fft_last_stage_load<L, INV>(v, t, S);
        gsync();  // exchange buffer is free for the next row
#pragma unroll
        for (int g = 0; g < GI; ++g) dftR<R3, INV>(v + g * R3);
        const int fb = r / (2 * L), rf = r - fb * (2 * L);   // field of the batch, row within its [2][L] planes
        const int phs = rf / L, rr = rf - phs * L;
        const int orow = (2 * rr + phs + L) & (2 * L - 1);  // fftshift along y
        if (p.out_kind == PB_OUT_COMPLEX) {
            float4* __restrict__ dst = reinterpret_cast<float4*>(reinterpret_cast<float2*>(p.out) + fb * p.out_bs + (long long)orow * p.out_ld);
#pragma unroll
            for (int g = 0; g < GI; ++g)
#pragma unroll
                for (int kk = 0; kk < R3; ++kk) {
                    const int j = t + g * NT + 256 * kk;
                    const P2 y = v[g * R3 + kk];
                    const float4 o = INV ? make_float4(sgn * y.re.x, sgn * y.im.x, sgn * y.im.y, -sgn * y.re.y)
                                         : make_float4(sgn * y.re.x, sgn * y.im.x, -sgn * y.im.y, sgn * y.re.y);
                    st_hint(dst + ((j + L / 2) & (L - 1)), o, pol_out);
                }
        } else {
            float2* __restrict__ dst = reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + fb * p.out_bs + (long long)orow * p.out_ld);
            const float2 s2 = make_float2(p.scale * p.scale, p.scale * p.scale);
            const float2 wgt = make_float2(p.weight, p.weight);
#pragma unroll
            for (int g = 0; g < GI; ++g)
#pragma unroll
                for (int kk = 0; kk < R3; ++kk) {
                    const int j = t + g * NT + 256 * kk;
                    const P2 y = v[g * R3 + kk];
                    float2 I = mul2(s2, fma2(y.re, y.re, mul2(y.im, y.im)));
                    float2* q = dst + ((j + L / 2) & (L - 1));
                    if (p.out_kind == PB_OUT_ACCUMULATE) I = fma2(wgt, I, ld_stream(q));
                    st_hint(q, I, pol_out);
                }
        }
    }
}


// ---- TMA descriptors, cached in the handle by (base pointer, geometry) -----------------------------
int get_map_c64(Handle* h, const MapKey& key, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                const cuuint32_t* box, const CUtensorMap** out) {
    auto it = h->maps.find(key);
    if (it != h->maps.end()) { *out = &it->second; return PB_OK; }
    CUtensorMap m;
    PB_TRY(encode_tensor_map(h, &m, CU_TENSOR_MAP_DATA_TYPE_UINT64, rank, key.base, dims, strides_bytes, box,
                             CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B));
    if (h->maps.size() > 256) h->maps.clear();
    *out = &(h->maps[key] = m);
    return PB_OK;
}

// one field: `p.tmp` holds its [2][L][L] intermediate.  col_dep: how the column kernel follows what precedes it in the
// stream -- 0: plain launch; 1: programmatic dependent of the previous field's row kernel; 2: the same, and its input does
// not overlap that kernel's output (the kernel waits for it at its end instead of its start)
template <int L, bool INV>
int launch_focus2(Handle* h, FocusParams p, int col_dep, cudaStream_t st) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using R4 = GeoR4<L, plane1_keep<L>()>;
    // one CTA per SM for both kernels: the column kernel's 512 threads fill the register file, and the row kernel keeps
    // its plan in shared memory, so it has no L1 working set to protect
    PB_TRY(set_smem_attrs(h, focus_col4_kernel<L, INV>, G4::SMEM, 1));
    PB_TRY(set_smem_attrs(h, focus_row4_kernel<L, INV>, R4::SMEM, 1));
    PB_TRY(get_col4_plan<L>(h, &p.plan));
    p.nrows = 2 * L;
    p.ntiles = G2::TILES;
    p.hints = 1 | 4;   // eviction hints, plane 0 and the head of plane 1 kept in L2 (FocusParams::hints)
    // (descriptors are copied out at once: the handle's cache may be flushed by the next lookup)
    const CUtensorMap* map = nullptr;
    CUtensorMap in_m, tmp_m;
    {   // intermediate: [group = (plane, j/4)][tile][j%4][c]
        const cuuint64_t dims[4] = {4, 4, (cuuint64_t)G2::TILES, (cuuint64_t)2 * (L / 4)};
        const cuuint64_t str[3] = {32, 128, (cuuint64_t)G2::TILES * 128};
        const cuuint32_t box[4] = {4, 1, (cuuint32_t)G2::BOXT, 1};
        PB_TRY(get_map_c64(h, MapKey{p.tmp, 1, L, 0, 0, 0}, 4, dims, str, box, &map));
        tmp_m = *map;
    }
    {   // input: (field, row, column) complex64, one field; box = one 4-column run of 256 rows
        const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)L, 1};
        const cuuint64_t str[2] = {(cuuint64_t)p.in_ld * 8, (cuuint64_t)L * p.in_ld * 8};
        const cuuint32_t box[3] = {4, (cuuint32_t)G2::BOXR, 1};
        PB_TRY(get_map_c64(h, MapKey{p.in, 2, L, p.in_ld, 0, 0}, 3, dims, str, box, &map));
        in_m = *map;
    }
    // Programmatic dependent launch: each kernel of the chain col(f), row(f), col(f + 1), ... is launched with
    // programmatic stream serialization, so that its CTAs take the SMs the previous kernel's last wave frees and run their
    // prologue (barriers, plan) while that wave finishes; griddepcontrol.wait orders everything that depends on the
    // previous kernel.  A column kernel with `early_input` writes the other intermediate buffer than the row kernel it
    // follows and runs its whole pass under that kernel's tail, waiting only at its end (focus_col4_kernel).  The column
    // kernel of the first field of a call is launched plainly: what precedes it is not known.  So is that of a staged field:
    // it follows its staging launch.
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr.val.programmaticStreamSerializationAllowed = 1;
    auto launch = [&](auto kern, int grid, int threads, size_t smem, bool dependent, const CUtensorMap& map) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid);
        cfg.blockDim = dim3(threads);
        cfg.dynamicSmemBytes = smem;
        cfg.stream = st;
        cfg.attrs = dependent ? &attr : nullptr;
        cfg.numAttrs = dependent ? 1 : 0;
        return cudaLaunchKernelEx(&cfg, kern, map, p);
    };
    // column pass: one CTA per SM walks the tiles of the field
    p.early_input = col_dep == 2;
    PB_CUDA(h, launch(focus_col4_kernel<L, INV>, std::min(h->sm_count, p.ntiles), G4::THREADS, G4::SMEM, col_dep > 0, in_m));
    h->launches++;
    // row pass: four line groups per CTA, plan in shared memory
    p.early_input = 0;
    PB_CUDA(h, launch(focus_row4_kernel<L, INV>, std::min(h->sm_count, (p.nrows + 3) / 4), 4 * G::NT, R4::SMEM, true, tmp_m));
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_FOCUS_V2, L, INV)] += 2;
    return PB_OK;
}

// =====================================================================================================
// Register-engine version of the generic axis pass (AxisPass semantics, complex64 in/out) for
// L in {1024, 2048, 4096}: two lines per thread group ride the two packed lanes.  ROWS: one CTA = 2 rows;
// COLS: one CTA = TP pairs of adjacent columns.  Used by pb_fft2 / pb_axis_dft / pb_angular_spectrum for
// every power-of-two pass the focus kernels above do not cover (CZT, FFTDFT, free space, psf -> otf).
// =====================================================================================================
__device__ __forceinline__ float2 cmul_s(float2 a, float2 b, int conj) {
    return conj ? make_float2(fmaf(a.x, b.x, a.y * b.y), fmaf(a.y, b.x, -a.x * b.y))
                : make_float2(fmaf(a.x, b.x, -a.y * b.y), fmaf(a.x, b.y, a.y * b.x));
}

// DENSE: the whole line is populated and kept -- no pad window, no rotation, no crop, an even number of lines, complex
// input (free-space steps at Q = 1, plain transforms): the per-element window tests and index arithmetic of the general
// form (about as many integer instructions as there are floating-point ones) compile away.
template <int L, bool INV, bool COLS, int TP, bool RT, bool PM, bool DENSE>
__global__ void __launch_bounds__((COLS ? TP : 1) * L / 16, (RT && (!COLS || TP == 1) && L >= 4096) ? 2 : 0) axis_reg_kernel(const AxisPass p, const float2* __restrict__ tw1,
                                                                            const float2* __restrict__ tw2) {
    using G = Geo<L>;
    constexpr int NT = G::NT;
    extern __shared__ __align__(16) float4 smem4[];
    const int c = COLS ? threadIdx.x % TP : 0, t = COLS ? threadIdx.x / TP : threadIdx.x;
    const int b0 = (blockIdx.x * (COLS ? TP : 1) + c) * 2;   // lines b0 (lane A) and b0 + 1 (lane B)
    const bool hasA = DENSE || b0 < p.nb, hasB = DENSE || b0 + 1 < p.nb;
    // column passes: a thread's two lines are adjacent columns, i.e. 16 contiguous bytes per sample -- one 128-bit access
    // instead of two 64-bit ones (half the LSU instructions and sector requests of the pass: `lg_throttle` was its second
    // stall).  vin / vout: unit line stride, even pitch, 16-byte aligned base, both lines present (host: dispatch_axis_reg).
    const bool vin = COLS && (DENSE || ((p.batch_contiguous & 2) && hasB));
    const bool vout = COLS && (DENSE || ((p.batch_contiguous & 4) && hasB));
    if (DENSE) {
        // L2 prefetch of the lines of the CTA that will run `pf` CTAs later: measured, no gain, and no launch sets pf
        // (bits 8 and up of batch_contiguous) any more.  The block stays because without it ptxas makes different code
        // for the DENSE kernels, and that code measured 3.7 % slower on the screened free-space chain (H100 SXM, 700 W)
        const int pf = p.batch_contiguous >> 8;
        if (pf) {
            const int nb0 = ((int)blockIdx.x + pf) * (COLS ? TP : 1) * 2;
            if (nb0 < p.nb) {
                if (!COLS) {
                    if (threadIdx.x < 2) {      // one bulk prefetch per line (contiguous: ies == 1), and of its screen row
                        const float2* src = reinterpret_cast<const float2*>(p.in) + (long long)(nb0 + threadIdx.x) * p.ibs;
                        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"((uint32_t)(L * sizeof(float2))) : "memory");
                        if (PM) {
                            const float2* sm = reinterpret_cast<const float2*>(p.pre_mat) + (long long)(nb0 + threadIdx.x) * p.pmi_bs;
                            asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(sm), "r"((uint32_t)(L * sizeof(float2))) : "memory");
                        }
                    }
                } else if (c == 0) {            // the 32-byte segments (TP = 2: four columns) of the next tile, one thread per segment
#pragma unroll
                    for (int n = 0; n < 16; ++n) {
                        const float2* src = reinterpret_cast<const float2*>(p.in) + (long long)nb0 * p.ibs + (long long)(n * NT + t) * p.ies;
                        asm volatile("prefetch.global.L2 [%0];" ::"l"(src) : "memory");
                    }
                }
            }
        }
    }
    const float2* __restrict__ in = reinterpret_cast<const float2*>(p.in);
    const float2* __restrict__ pre_e = reinterpret_cast<const float2*>(p.pre_e);
    const float2* __restrict__ pre_b = reinterpret_cast<const float2*>(p.pre_b);
    float2 pbA = make_float2(1.f, 0.f), pbB = pbA;
    if (pre_b) { if (hasA) pbA = pre_b[b0]; if (hasB) pbB = pre_b[b0 + 1]; }
    P2 v[16];
#pragma unroll
    for (int n = 0; n < 16; ++n) {
        const int j = n * NT + t;
        int li = j;
        if (!DENSE) {
            int pp = j + p.rot_in;
            if (pp >= L) pp -= L;
            li = pp - p.in_off;
        }
        float2 xa = make_float2(0.f, 0.f), xb = xa;
        if (DENSE || (li >= 0 && li < p.n_in)) {
            const long long o = (long long)b0 * p.ibs + (long long)li * p.ies;
            if (!DENSE && p.in_kind == PB_IN_REAL) {   // real field (the PSF going to transform_psf): imaginary part 0
                const float* __restrict__ inr = reinterpret_cast<const float*>(p.in);
                if (hasA) xa.x = __ldg(inr + o);
                if (hasB) xb.x = __ldg(inr + o + p.ibs);
            } else if (vin) {
                const float4 q = ld_stream4(reinterpret_cast<const float4*>(in + o));
                xa = make_float2(q.x, q.y); xb = make_float2(q.z, q.w);
            } else {
                if (hasA) xa = ld_stream(in + o);
                if (hasB) xb = ld_stream(in + o + p.ibs);
            }
            if (pre_e) { const float2 w = pre_e[j - p.pre_off]; xa = cmul_s(xa, w, p.pre_e_conj); xb = cmul_s(xb, w, p.pre_e_conj); }
            if (pre_b) { xa = cmul_s(xa, pbA, p.pre_b_conj); xb = cmul_s(xb, pbB, p.pre_b_conj); }
        }
        v[n] = {make_float2(xa.x, xb.x), make_float2(xa.y, xb.y)};
    }
    if (PM) {
        // full-matrix pre-multiplier (the phase screen of a free-space chain), same access pattern as the input.  A loop of
        // its own: the 32 loads are independent of the input loads above and of each other, so they overlap, and the
        // product is one packed complex multiply per point (lane A x mA, lane B x mB).
        const float2* __restrict__ pm = reinterpret_cast<const float2*>(p.pre_mat);
#pragma unroll
        for (int n = 0; n < 16; ++n) {
            const int j = n * NT + t;
            int li = j;
            if (!DENSE) {
                int pp = j + p.rot_in;
                if (pp >= L) pp -= L;
                li = pp - p.in_off;
            }
            if (DENSE || (li >= 0 && li < p.n_in)) {
                const long long om = (long long)b0 * p.pmi_bs + (long long)li * p.pmi_es;
                float2 ma = make_float2(1.f, 0.f), mb = ma;
                if (hasA) ma = ld_stream(pm + om);
                if (hasB) mb = ld_stream(pm + om + p.pmi_bs);
                const float4 w = make_float4(ma.x, mb.x, ma.y, mb.y);
                v[n] = p.pre_mat_conj ? mul_tw<true>(v[n], w) : mul_tw<false>(v[n], w);
            }
        }
    }
    // TP interleaved lines per CTA: consecutive exchange buffers are offset by 32 / TP banks (8 / TP float4 of padding), so
    // that the 8 threads of a 128-bit wavefront (8 / TP consecutive t  x  TP lines) cover all 32 banks
    float4* S = smem4 + c * (G::SBUF + 8 / (COLS ? TP : 1) % 8);
    fft_two_stages<L, INV>(v, t, S, tw1, tw2);
    fft_last_stage_load<L, INV>(v, t, S);
#pragma unroll
    for (int g = 0; g < G::GI; ++g) dftR<G::R3, INV>(v + g * G::R3);
    const float2* __restrict__ post_e = reinterpret_cast<const float2*>(p.post_e);
    const float2* __restrict__ post_b = reinterpret_cast<const float2*>(p.post_b);
    float2 qbA = make_float2(1.f, 0.f), qbB = qbA;
    if (post_b) { if (hasA) qbA = post_b[b0]; if (hasB) qbB = post_b[b0 + 1]; }
    const float scale = (float)p.scale;
    float2* __restrict__ out = reinterpret_cast<float2*>(p.out);
    if (RT) {
        // Round trip (free-space propagation along this axis): the spectrum is multiplied by the transfer
        // factors post_e[k] * post_b[line] and transformed straight back.  The forward pass leaves thread t
        // with X[t + NT*(g + GI*kk)], which IS the inverse pass's stage-1 register layout (n = g + GI*kk):
        // the data never leaves the registers between the two transforms.
        P2 w[16];
#pragma unroll
        for (int g = 0; g < G::GI; ++g)
#pragma unroll
            for (int kk = 0; kk < G::R3; ++kk) {
                const int k = t + g * NT + 256 * kk;
                const P2 y = v[g * G::R3 + kk];
                float2 ya = make_float2(y.re.x, y.im.x), yb = make_float2(y.re.y, y.im.y);
                if (post_e) { const float2 m = post_e[k - p.post_off]; ya = cmul_s(ya, m, p.post_e_conj); yb = cmul_s(yb, m, p.post_e_conj); }
                if (post_b) { ya = cmul_s(ya, qbA, p.post_b_conj); yb = cmul_s(yb, qbB, p.post_b_conj); }
                w[g + G::GI * kk] = {make_float2(ya.x, yb.x), make_float2(ya.y, yb.y)};
            }
        __syncthreads();   // all last-stage reads of S are done before the inverse pass overwrites it
        fft_two_stages<L, !INV>(w, t, S, tw1, tw2);
        fft_last_stage_load<L, !INV>(w, t, S);
#pragma unroll
        for (int g = 0; g < G::GI; ++g) dftR<G::R3, !INV>(w + g * G::R3);
        if (COLS && p.out_kind != PB_OUT_COMPLEX && (p.batch_contiguous & 8) && hasB) {
            // |.|^2 of a column pass onto a real plane, both columns of the thread as one aligned float2.  Three passes over
            // the thread's 16 samples -- form the intensities, read ALL the previous plane values, then store -- because a
            // read-modify-write per sample serialises: the compiler may not move sample i+1's load above sample i's store to
            // the same array, and sixteen DRAM latencies in a row were the C4 column pass's top stall (long_scoreboard 8.2).
            float* __restrict__ outr = reinterpret_cast<float*>(p.out);
            const float s2 = scale * scale, wgt = (float)p.weight;
            auto out_q = [&](int j) -> int {   // output sample of transform index j, or -1 when it is cropped away
                if (DENSE) return j;
                int q = j - p.crop_off + p.rot_out;
                if (q < 0) q += L;
                if (q >= L) q -= L;
                return q < p.n_out ? q : -1;
            };
            float2 I[16];
#pragma unroll
            for (int g = 0; g < G::GI; ++g)
#pragma unroll
                for (int kk = 0; kk < G::R3; ++kk) {
                    const int q = out_q(t + g * NT + 256 * kk);
                    const P2 y = w[g * G::R3 + kk];
                    float2 ya = make_float2(y.re.x, y.im.x), yb = make_float2(y.re.y, y.im.y);
                    if (p.post_e2 && q >= 0) {
                        const float2 m = reinterpret_cast<const float2*>(p.post_e2)[q];
                        ya = cmul_s(ya, m, p.post_e2_conj); yb = cmul_s(yb, m, p.post_e2_conj);
                    }
                    I[g * G::R3 + kk] = make_float2(s2 * fmaf(ya.x, ya.x, ya.y * ya.y), s2 * fmaf(yb.x, yb.x, yb.y * yb.y));
                }
            if (p.out_kind == PB_OUT_ACCUMULATE) {
#pragma unroll
                for (int g = 0; g < G::GI; ++g)
#pragma unroll
                    for (int kk = 0; kk < G::R3; ++kk) {
                        const int q = out_q(t + g * NT + 256 * kk);
                        if (q < 0) continue;
                        const float2 prev = *reinterpret_cast<const float2*>(outr + (long long)b0 * p.obs + (long long)q * p.oes);
                        float2& v2 = I[g * G::R3 + kk];
                        v2 = make_float2(fmaf(wgt, v2.x, prev.x), fmaf(wgt, v2.y, prev.y));
                    }
            }
#pragma unroll
            for (int g = 0; g < G::GI; ++g)
#pragma unroll
                for (int kk = 0; kk < G::R3; ++kk) {
                    const int q = out_q(t + g * NT + 256 * kk);
                    if (q < 0) continue;
                    *reinterpret_cast<float2*>(outr + (long long)b0 * p.obs + (long long)q * p.oes) = I[g * G::R3 + kk];
                }
            return;
        }
#pragma unroll
        for (int g = 0; g < G::GI; ++g)
#pragma unroll
            for (int kk = 0; kk < G::R3; ++kk) {
                const int j = t + g * NT + 256 * kk;
                int q = j;
                if (!DENSE) {
                    q = j - p.crop_off + p.rot_out;
                    if (q < 0) q += L;
                    if (q >= L) q -= L;
                    if (q >= p.n_out) continue;
                }
                const P2 y = w[g * G::R3 + kk];
                float2 ya = make_float2(y.re.x, y.im.x), yb = make_float2(y.re.y, y.im.y);
                if (p.post_e2) {  // final multiplier, indexed by the output sample (the CZT's a(m)*phase(m))
                    const float2 m = reinterpret_cast<const float2*>(p.post_e2)[q];
                    ya = cmul_s(ya, m, p.post_e2_conj); yb = cmul_s(yb, m, p.post_e2_conj);
                }
                const long long o = (long long)b0 * p.obs + (long long)q * p.oes;
                if (p.out_kind == PB_OUT_COMPLEX) {
                    if (vout) st_stream(reinterpret_cast<float4*>(out + o), make_float4(ya.x * scale, ya.y * scale, yb.x * scale, yb.y * scale));
                    else {
                        if (hasA) st_stream(out + o, make_float2(ya.x * scale, ya.y * scale));
                        if (hasB) st_stream(out + o + p.obs, make_float2(yb.x * scale, yb.y * scale));
                    }
                } else {   // |.|^2 (or weight * |.|^2 added to the plane): the complex field is never written
                    float* __restrict__ outr = reinterpret_cast<float*>(p.out);
                    const float s2 = scale * scale, wgt = (float)p.weight;
                    float ia = s2 * fmaf(ya.x, ya.x, ya.y * ya.y), ib = s2 * fmaf(yb.x, yb.x, yb.y * yb.y);
                    if (p.out_kind == PB_OUT_ACCUMULATE) {
                        if (hasA) ia = fmaf(wgt, ia, outr[o]);
                        if (hasB) ib = fmaf(wgt, ib, outr[o + p.obs]);
                    }
                    if (hasA) outr[o] = ia;
                    if (hasB) outr[o + p.obs] = ib;
                }
            }
        return;
    }
#pragma unroll
    for (int g = 0; g < G::GI; ++g)
#pragma unroll
        for (int kk = 0; kk < G::R3; ++kk) {
            const int k = t + g * NT + 256 * kk;
            int q = k;
            if (!DENSE) {
                q = k - p.crop_off + p.rot_out;
                if (q < 0) q += L;
                if (q >= L) q -= L;
                if (q >= p.n_out) continue;
            }
            const P2 y = v[g * G::R3 + kk];
            float2 ya = make_float2(y.re.x, y.im.x), yb = make_float2(y.re.y, y.im.y);
            if (post_e) { const float2 w = post_e[k - p.post_off]; ya = cmul_s(ya, w, p.post_e_conj); yb = cmul_s(yb, w, p.post_e_conj); }
            if (post_b) { ya = cmul_s(ya, qbA, p.post_b_conj); yb = cmul_s(yb, qbB, p.post_b_conj); }
            const long long o = (long long)b0 * p.obs + (long long)q * p.oes;
            if (vout) st_stream(reinterpret_cast<float4*>(out + o), make_float4(ya.x * scale, ya.y * scale, yb.x * scale, yb.y * scale));
            else {
                if (hasA) st_stream(out + o, make_float2(ya.x * scale, ya.y * scale));
                if (hasB) st_stream(out + o + p.obs, make_float2(yb.x * scale, yb.y * scale));
            }
        }
}

// plain twiddle tables: tw1[(k-1)*NT + t] = w_L^(t k), tw2[(k-1)*NT/16 + m] = w_L^(16 m k), contiguous
template <int L>
int get_plain_plan(Handle* h, const float2** tw1, const float2** tw2) {
    using G = Geo<L>;
    const void* d = nullptr;
    PB_TRY(cached_table(h, {L, PB_C64, TW_PLAIN_PLAN}, [](auto& tab) {
        tab.resize(15 * G::NT + 15 * (G::NT / 16));
        for (int k = 1; k < 16; ++k)
            for (int t = 0; t < G::NT; ++t) tab[(k - 1) * G::NT + t] = host_tw((long long)t * k, L);
        for (int k = 1; k < 16; ++k)
            for (int m = 0; m < G::NT / 16; ++m) tab[15 * G::NT + (k - 1) * (G::NT / 16) + m] = host_tw(16LL * m * k, L);
    }, &d));
    *tw1 = reinterpret_cast<const float2*>(d);
    *tw2 = *tw1 + 15 * G::NT;
    return PB_OK;
}

template <int L, bool INV, bool COLS, bool RT, bool PM = false, bool DENSE = false, int TPC = 2>
int launch_axis_reg(Handle* h, const AxisPass& p, cudaStream_t st) {
    using G = Geo<L>;
    constexpr int TP = COLS ? TPC : 1;
    const size_t smem = (size_t)TP * (G::SBUF + 8 / TP % 8) * sizeof(float4);
    if (attr_needed(h, reinterpret_cast<const void*>(axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE>))) {
        PB_CUDA(h, cudaFuncSetAttribute(axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        // Resident CTAs per SM: as many as leave >= 64 KB of the unified L1/shared array as L1 -- the twiddle tables are
        // re-read by every line and must hit there.  (Left to itself the driver picks the 228 KB carve-out and the tables
        // stream from L2 at ~300 cycles a load.)
        const size_t unified = 256 * 1024, l1_keep = 64 * 1024;
        const int ctas = std::max<int>(1, (int)((unified - l1_keep) / (smem + 1024)));
        const int pct = (int)std::min<size_t>(100, ((size_t)ctas * (smem + 1024) * 100 + h->max_smem_optin - 1) / h->max_smem_optin);
        PB_CUDA(h, cudaFuncSetAttribute(axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE>, cudaFuncAttributePreferredSharedMemoryCarveout, pct));
    }
    const float2 *tw1 = nullptr, *tw2 = nullptr;
    PB_TRY(get_plain_plan<L>(h, &tw1, &tw2));
    const int lines_per_cta = 2 * TP;
    const int grid = (p.nb + lines_per_cta - 1) / lines_per_cta;
    axis_reg_kernel<L, INV, COLS, TP, RT, PM, DENSE><<<grid, TP * G::NT, smem, st>>>(p, tw1, tw2);
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_AXIS_REG, L, INV | COLS << 1 | RT << 2 | PM << 3 | DENSE << 4)]++;
    return PB_OK;
}

template <int L>
int dispatch_axis_reg(Handle* h, const AxisPass& p0, cudaStream_t st) {
    AxisPass p = p0;
    const bool cols = p.batch_contiguous != 0;
    // 128-bit accesses of the column passes (two adjacent columns per thread): unit line stride, even pitch, aligned base
    const bool vec_in = cols && p.in_kind == PB_IN_COMPLEX && p.ibs == 1 && !(p.ies & 1) && !((uintptr_t)p.in & 15);
    const bool vec_out = cols && p.out_kind == PB_OUT_COMPLEX && p.obs == 1 && !(p.oes & 1) && !((uintptr_t)p.out & 15);
    const bool vec_int = cols && p.out_kind != PB_OUT_COMPLEX && p.obs == 1 && !(p.oes & 1) && !((uintptr_t)p.out & 7);
    if (cols) p.batch_contiguous = 1 | (vec_in ? 2 : 0) | (vec_out ? 4 : 0) | (vec_int ? 8 : 0);
    // the whole line populated and kept, lines in pairs, complex in: the index logic of the general kernel compiles away
    const bool dense = p.rot_in == 0 && p.in_off == 0 && p.n_in == L && p.crop_off == 0 && p.rot_out == 0 && p.n_out == L &&
                       !(p.nb & 1) && p.in_kind == PB_IN_COMPLEX && !p.post_e2 && p.pre_off == 0 && p.post_off == 0 &&
                       (!cols || (!(p.nb & 3) && vec_in && vec_out));
    if (p.pre_mat) {   // the screened first pass of a free-space step: rows, plain transform
        if (cols || p.roundtrip) return PB_ERR_UNSUPPORTED;
        if (dense) return p.dir < 0 ? launch_axis_reg<L, false, false, false, true, true>(h, p, st) : launch_axis_reg<L, true, false, false, true, true>(h, p, st);
        return p.dir < 0 ? launch_axis_reg<L, false, false, false, true>(h, p, st) : launch_axis_reg<L, true, false, false, true>(h, p, st);
    }
    if (dense && L >= 2048) {   // the free-space passes and plain transforms of the large configurations
        if (p.roundtrip) {
            if (cols) return p.dir < 0 ? launch_axis_reg<L, false, true, true, false, true>(h, p, st) : launch_axis_reg<L, true, true, true, false, true>(h, p, st);
        } else if (!cols) {
            return p.dir < 0 ? launch_axis_reg<L, false, false, false, false, true>(h, p, st) : launch_axis_reg<L, true, false, false, false, true>(h, p, st);
        } else {
            return p.dir < 0 ? launch_axis_reg<L, false, true, false, false, true>(h, p, st) : launch_axis_reg<L, true, true, false, false, true>(h, p, st);
        }
    }
    if (p.roundtrip) {
        if (p.dir < 0) return cols ? launch_axis_reg<L, false, true, true>(h, p, st) : launch_axis_reg<L, false, false, true>(h, p, st);
        return cols ? launch_axis_reg<L, true, true, true>(h, p, st) : launch_axis_reg<L, true, false, true>(h, p, st);
    }
    if (p.dir < 0) return cols ? launch_axis_reg<L, false, true, false>(h, p, st) : launch_axis_reg<L, false, false, false>(h, p, st);
    return cols ? launch_axis_reg<L, true, true, false>(h, p, st) : launch_axis_reg<L, true, false, false>(h, p, st);
}

}  // namespace

int try_tuned_axis_pass(Handle* h, const AxisPass& p, cudaStream_t st) {
    if (p.dtype != PB_C64 || p.in_kind == PB_IN_AMP_OPD) return PB_ERR_UNSUPPORTED;
    if (p.out_kind != PB_OUT_COMPLEX && !p.roundtrip) return PB_ERR_UNSUPPORTED;   // |.|^2 stores: round-trip epilogue only
    if (p.pre_e2 || (p.post_e2 && !p.roundtrip) || p.post_mat) return PB_ERR_UNSUPPORTED;
    if (p.Llog != p.L || (p.Llog_out != 0 && p.Llog_out != p.L)) return PB_ERR_UNSUPPORTED;
    // any batch: a single line (the kernel spectrum of a CZT plan, built per wavelength) would otherwise take the generic
    // kernel's six synchronised radix-4 stages
    switch (p.L) {
        case 1024: return dispatch_axis_reg<1024>(h, p, st);
        case 2048: return dispatch_axis_reg<2048>(h, p, st);
        case 4096: return dispatch_axis_reg<4096>(h, p, st);
        default: return PB_ERR_UNSUPPORTED;
    }
}

int try_tuned_fft2_batch(Handle* h, const Fft2Args& a, cudaStream_t st) {
    if (a.dtype != PB_C64 || a.ny != a.nx || a.ky != 2 * a.ny || a.kx != 2 * a.nx || !a.shift_in || !a.shift_out ||
        a.oy != a.ky || a.ox != a.kx)
        return PB_ERR_UNSUPPORTED;
    const int N = a.nx;
    if (N != 512 && N != 1024 && N != 2048) return PB_ERR_UNSUPPORTED;
    if (a.in_kind == PB_IN_REAL) return PB_ERR_UNSUPPORTED;
    if ((a.out_ld & 1) || (a.out_bs & 1) || ((uintptr_t)a.out & (a.out_kind == PB_OUT_COMPLEX ? 15 : 7)))
        return PB_ERR_UNSUPPORTED;  // vector stores need aligned rows
    // Inputs tensor TMA can gather (complex, 16-byte aligned base, even pitches) go to the pair as they are; every other
    // one is first written as a dense aligned field in scratch slot 1, one field at a time
    const bool staged = a.in_kind != PB_IN_COMPLEX || ((uintptr_t)a.in & 15) || (a.in_ld & 1) || (a.in_bs & 1);
    // the fields of a stack alternate between two intermediates (field f: buffer f mod 2), so that a column kernel never
    // writes what the row kernel before it reads (focus_col4_kernel)
    const int nbuf = a.batch > 1 ? 2 : 1;
    const size_t field_bytes = (size_t)N * N * sizeof(float2);
    void* tmp = nullptr;
    PB_TRY(ensure_scratch(h, 0, nbuf * 2 * field_bytes, &tmp));
    void* stage = nullptr;
    if (staged) PB_TRY(ensure_scratch(h, 1, field_bytes, &stage));
    // the column kernels' tile counters, one per buffer: zeroed once here, then by each field's row kernel
    const void* d = nullptr;
    PB_TRY(cached_table(h, {2, PB_C64, TW_TILE_COUNTERS}, [](auto& t) { t.resize(1); }, &d));   // one complex64 zero = two counters
    unsigned int* ctr = reinterpret_cast<unsigned int*>(const_cast<void*>(d));
    // fields after the first of an unstaged stack: the column kernel follows this call's previous row kernel
    // (programmatic dependent launch, see launch_focus2); it may gather its input early unless the input stack overlaps
    // the output stack.  A staged field's column kernel is launched plainly, after its staging launch, which is plain too
    // and so follows the previous field's row kernel.
    const uintptr_t in_lo = (uintptr_t)a.in,
                    in_hi = in_lo + (size_t)((long long)(a.batch - 1) * a.in_bs + (long long)(a.ny - 1) * a.in_ld + a.nx) * a.in_elt();
    const uintptr_t out_lo = (uintptr_t)a.out,
                    out_hi = out_lo + (size_t)((long long)(a.batch - 1) * a.out_bs + (long long)(a.ky - 1) * a.out_ld + a.kx) * a.out_elt();
    const int col_dep_next = staged ? 0 : (in_hi <= out_lo || out_hi <= in_lo) ? 2 : 1;
    for (int b = 0; b < a.batch; ++b) {
        const Fft2Args f = a.field(b);
        FocusParams p = {};
        p.in = f.in;   // (16-byte aligned if not staged: in_bs is even)
        p.in_ld = a.in_ld;
        if (staged) {
            if (a.in_kind == PB_IN_AMP_OPD) {
                PB_TRY(launch_phase_screen(h, PB_C64, f.amp, a.amp_kind, p.in, a.kturns(), (long long)N * N, N, a.in_ld, stage, st));
            } else {
                PB_CUDA(h, cudaMemcpy2DAsync(stage, N * sizeof(float2), p.in, a.in_ld * sizeof(float2), N * sizeof(float2), N,
                                             cudaMemcpyDeviceToDevice, st));
            }
            p.in = stage;
            p.in_ld = N;
        }
        p.tmp = reinterpret_cast<float2*>(reinterpret_cast<char*>(tmp) + (size_t)(b % nbuf) * 2 * field_bytes);
        p.out = f.out;
        p.out_ld = a.out_ld; p.out_kind = a.out_kind; p.scale = (float)a.scale; p.weight = (float)a.weight;
        p.out_bs = a.out_bs;
        p.tile_ctr = ctr + (b % nbuf);
        const int cd = b > 0 ? col_dep_next : 0;
        int rc;
        if (a.dir < 0) rc = N == 512 ? launch_focus2<512, false>(h, p, cd, st) : N == 1024 ? launch_focus2<1024, false>(h, p, cd, st) : launch_focus2<2048, false>(h, p, cd, st);
        else rc = N == 512 ? launch_focus2<512, true>(h, p, cd, st) : N == 1024 ? launch_focus2<1024, true>(h, p, cd, st) : launch_focus2<2048, true>(h, p, cd, st);
        if (rc != PB_OK) return rc;
    }
    return PB_OK;
}


}  // namespace pb
