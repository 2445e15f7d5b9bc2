// Fused focus pipeline for stacks of pupils: ONE persistent, role-specialised kernel instead of a column kernel and a
// row kernel per group of fields  (reference prysm/propagation/fft.py:7-65, Wavefront.focus / unfocus with Q = 2 on a
// (B, N, N) complex64 stack; algebra and FFT engine: fft_tuned.cu / fft_engine.cuh).
//
// Why.  With several fields per launch pair (needed to hide launch ramps and tails) the tile-major intermediates of a
// group (16 N^2 bytes each, 64 MiB at N = 2048) cannot stay in L2: each makes a round trip through HBM, 128 MB per
// propagation on top of 168 MB of algorithmic traffic.  Here the column pass of field f+1 and the row
// pass of field f run AT THE SAME TIME on disjoint sets of SMs, coupled by counters in global memory:
//   * `ncol` CTAs are column workers (focus_col4's two 256-thread groups), the rest row workers (focus_row4's four
//     128-thread line groups); one CTA per SM, all co-resident (cooperative launch), identical shared-memory layout
//     (4 exchange buffers, 64 KB tile staging = 4 row buffers, the float2 plan);
//   * column tiles and intermediate rows are handed out in order by two global counters, so every worker is busy as
//     long as there is work of its kind; a row of field f is gathered only after all tiles of f were signalled
//     (cols_done[f]), a tile of field f is stored only after all rows of field f - ring were read (rows_read[f - ring]):
//     the intermediates live in a ring of `ring` slots and only the one being consumed while the next is produced is
//     live at a time: 16 MiB at N = 1024 fits the H100's 50 MB L2, 64 MiB at N = 2048 does not and partly spills to HBM;
//   * the pipeline has no fill / drain bubble: every CTA starts in column mode (row workers help with field 0) and
//     every CTA ends in row mode (column workers join the row workers when the tiles run out).
// Cross-SM visibility: one thread per column group fences (gpu scope, cumulative over the group's barriers) and adds to
// cols_done a good part of a tile time AFTER the stores it signals (the fence then finds the stores drained); the row
// group's requesting thread load-acquires the counter and issues fence.proxy.async (all spaces, once per field) before
// the tensor-TMA gathers of that field's rows.
#include "fft_engine.cuh"

namespace pb {
namespace {

constexpr int FUSED_MAX_FIELDS = 64;   // fields per launch (size of the counter arrays)

struct FusedParams {
    const float2* plan;     // Geo4 float2 plan
    float2* tmp;            // ring of tile-major intermediates, [ring][2][L/4][TILES][4][4]
    int* sync;              // [0] next tile, [1] next row, [2 + f] cols_done[f], [2 + MAX + f] rows_read[f]
    void* out; long long out_ld, out_bs; int out_kind; float scale, weight;
    int batch, ring, ncol, help_tiles, hints;
    // plane-unit kernel only: tiles a column worker may run ahead of the row workers (< 0: no budget gate), and the
    // arrival counters of the line groups, [buffer][L/4]
    int slack_tiles;
    unsigned int* arrive;
};

template <int L> struct GeoF {
    using G4 = Geo4<L>;
    static constexpr size_t BAR_OFF = G4::BAR_OFF;               // 8 mbarriers: [0] plan, [1] tile, [2 + g] row of group g
    static constexpr size_t CTL_OFF = BAR_OFF + 8 * sizeof(uint64_t);
    // ints: [0] release counter of the staging area, [1], [2] tile of iteration it & 1, [3] prefetched tile, [4 + 2 g + (it & 1)] row of group g
    static constexpr size_t SMEM = CTL_OFF + 16 * sizeof(int);
    static constexpr int WARPS = G4::THREADS / 32;
};

__device__ __forceinline__ int ld_acquire(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ int ld_relaxed(const int* p) {
    int v;
    asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void spin_until(const int* p, int target) {
    while (ld_acquire(p) < target) __nanosleep(100);
}
__device__ __forceinline__ void fence_proxy_async_all() { asm volatile("fence.proxy.async;" ::: "memory"); }

// one thread: next column tile of the launch, or -1.  Row workers only help while tiles of the first field(s) remain.
__device__ __forceinline__ int next_tile(const FusedParams& p, const bool col_role, const int ntiles) {
    if (!col_role && ld_relaxed(p.sync) >= p.help_tiles) return -1;
    const int w = atomicAdd(p.sync, 1);
    return w < ntiles ? w : -1;
}

template <int L>
__device__ __forceinline__ void request_tile(const CUtensorMap& in_map, float4* smem4, uint64_t* bar_tile, const int ww, const uint64_t pol) {
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    const int fb = ww / G2::TILES, tile = ww - fb * G2::TILES;
    mbar_expect_tx(bar_tile, (uint32_t)(L * 4 * sizeof(float2)));
#pragma unroll
    for (int b = 0; b < G2::NBOX_IN; ++b)
        tma_load_3d(smem4 + G4::STAGE + b * G2::BOXR * 2, &in_map, tile * 4, b * G2::BOXR, fb, bar_tile, pol);
}

// ---- column mode: one of the CTA's two groups (HALF = half-transform / plane) -----------------------------------------
template <int L, bool INV, int HALF>
__device__ __forceinline__ void fused_col_group(const CUtensorMap& in_map, const FusedParams& p, float4* smem4, uint64_t* bar,
                                                volatile int* ctl, const bool col_role) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GF = GeoF<L>;
    constexpr int NT = G::NT;
    const int ntiles = p.batch * G2::TILES;
    const int lt = threadIdx.x & (2 * NT - 1);                       // thread within the group
    const int cp = lt & 1, t = lt >> 1;
    const int lane = threadIdx.x & 31;
    const float4* __restrict__ stage = smem4 + G4::STAGE;
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smem4 + G4::PLAN2);
    float4* S = smem4 + (HALF * 2 + cp) * G4::XBUF;
    const SyncGroup gsync{1 + HALF, 2 * NT};
    const uint64_t pol_tmp = l2_policy((p.hints & 1) ? 2 : 0), pol_in = l2_policy((p.hints & 1) ? 1 : 0);
    const float sgn = (t & 1) ? -1.0f : 1.0f;
    float2 u = make_float2(1.f, 0.f);
    if (HALF) { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u = make_float2(cs, sn); }   // w_2L^t = exp(-i pi t / L)
    int pending = -1;      // field of the tile whose stores this warp has not signalled yet
    int checked = -1;      // field whose ring slot is known to be free
    int pref = -1;         // (one lane) tile index fetched ahead, on its way to ctl[3]
    bool have_pref = false;
    for (int it = 0;; ++it) {
        mbar_wait(bar + 1, it & 1);
        const int w = ctl[1 + (it & 1)];
        if (w < 0) break;
        const int fb = w / G2::TILES, tile = w - fb * G2::TILES;
        auto sync = [&]() { gsync(); };
        P2 v[16];
        {
            float4 x[16];   // (col, col + 1) x (re, im)
            const float4* __restrict__ sg = stage + lt;   // ((n*NT + t)*2 + cp)
#pragma unroll
            for (int n = 0; n < 16; ++n) x[n] = sg[n * NT * 2];
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
            if (lane == 0) {   // this warp holds its inputs: one of WARPS releases of the staging area per tile;
                __threadfence_block();       // the LAST warp to release it requests the next tile on the spot
                const unsigned int n = atomicAdd(const_cast<unsigned int*>(reinterpret_cast<volatile unsigned int*>(ctl)), 1u) + 1u;
                __threadfence_block();
                if (n == (unsigned int)(it + 1) * GF::WARPS) {
                    const int wn = ctl[3];             // fetched a tile time ago
                    ctl[1 + ((it + 1) & 1)] = wn;
                    if (wn >= 0) {
                        fence_proxy_async();
                        request_tile<L>(in_map, smem4, bar + 1, wn, pol_in);
                        pref = next_tile(p, col_role, ntiles);   // the atomic's latency rides under the stages below
                    } else {
                        pref = -1;
                        mbar_arrive(bar + 1);
                    }
                    have_pref = true;
                }
            }
        }
        fft_two_stages_u<L, INV, HALF>(v, t, S, plan + G4::TW1, plan + G4::TW2, u, sync);
        if (have_pref) {
            ctl[3] = pref;
            have_pref = false;
            if ((p.hints & 2) && pref >= 0) {   // pull the tile after next from HBM into L2 now: its gather will be an L2 hit
                const int fb2 = pref / G2::TILES, tile2 = pref - fb2 * G2::TILES;
#pragma unroll
                for (int b = 0; b < G2::NBOX_IN; ++b) tma_prefetch_3d(&in_map, tile2 * 4, b * G2::BOXR, fb2);
            }
        }
        if (pending >= 0 && lt == 0) {   // the previous tile's stores of ALL warps of the group are three group barriers old:
            __threadfence();             // one cumulative gpu-scope fence by one thread publishes them
            atomicAdd(p.sync + 2 + pending, 1);
        }
        fft_last_stage_load<L, INV>(v, t, S);
        if (fb != checked) {   // ring slot of this field: every row of field fb - ring must have been gathered
            if (lt == 0 && fb >= p.ring) spin_until(p.sync + 2 + FUSED_MAX_FIELDS + fb - p.ring, 2 * L);
            checked = fb;
        }
        sync();   // this group's exchange buffers are free for its next tile (and the ring slot is free)
#pragma unroll
        for (int g = 0; g < G::GI; ++g) dftR<G::R3, INV>(v + g * G::R3);
        // tile-major store: element (plane, j, tile, c) at ((plane*L/4 + j/4) * TILES + tile) * 16 + (j%4)*4 + c ; c = 2 cp
        float4* __restrict__ dst = reinterpret_cast<float4*>(
            p.tmp + (long long)(fb % p.ring) * (2LL * L * L) + (long long)HALF * L * L + ((long long)(t >> 2) * G2::TILES + tile) * 16 + (t & 3) * 4 + 2 * cp);
#pragma unroll
        for (int g = 0; g < G::GI; ++g)
#pragma unroll
            for (int kk = 0; kk < G::R3; ++kk) {
                const P2 y = v[g * G::R3 + kk];
                const long long o = (long long)((g * NT + 256 * kk) >> 2) * (G2::TILES * 8);   // float4 units
                float4 q;
                if (HALF == 0) q = make_float4(sgn * y.re.x, sgn * y.im.x, sgn * y.re.y, sgn * y.im.y);
                else q = INV ? make_float4(sgn * y.im.x, -sgn * y.re.x, sgn * y.im.y, -sgn * y.re.y)
                             : make_float4(-sgn * y.im.x, sgn * y.re.x, -sgn * y.im.y, sgn * y.re.y);
                st_hint(dst + o, q, pol_tmp);
            }
        pending = fb;
    }
    gsync();   // every warp of the group has left the loop: its last tile's stores are ordered before the barrier
    if (pending >= 0 && lt == 0) {
        __threadfence();
        atomicAdd(p.sync + 2 + pending, 1);
    }
}

// ---- row epilogue: output row `orow` of field fb from the last stage's results (sgn = (-1)^t * scale) -------------------
template <int L, bool INV>
__device__ __forceinline__ void fused_row_store(const P2 (&v)[16], const int t, const FusedParams& p, const int fb, const int orow,
                                                const float sgn, const uint64_t pol_out) {
    using G = Geo<L>;
    constexpr int NT = G::NT, R3 = G::R3, GI = G::GI;
    if (p.out_kind == PB_OUT_COMPLEX) {
        float4* __restrict__ dst = reinterpret_cast<float4*>(reinterpret_cast<float2*>(p.out) + fb * p.out_bs + (long long)orow * p.out_ld);
#pragma unroll
        for (int g = 0; g < GI; ++g)
#pragma unroll
            for (int kk = 0; kk < R3; ++kk) {
                const int j = t + g * NT + 256 * kk;
                const P2 y = v[g * R3 + kk];
                // U[2j] = (-1)^j A,  U[2j+1] = (-1)^j (-dir*i) B ; fftshift along x: pair index (j + L/2) mod L
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

// ---- row mode: one of the CTA's four line groups ---------------------------------------------------------------------------
template <int L, bool INV>
__device__ __forceinline__ void fused_row_group(const CUtensorMap& tmp_map, const FusedParams& p, float4* smem4, uint64_t* bars,
                                                volatile int* ctl) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GF = GeoF<L>;
    constexpr int NT = G::NT, R3 = G::R3, GI = G::GI;
    constexpr uint32_t ROW_BYTES = L * sizeof(float2);
    const int grp = threadIdx.x / NT, t = threadIdx.x - grp * NT;
    float4* S = smem4 + grp * G4::XBUF;                                           // this group's exchange buffer
    float2* inb = reinterpret_cast<float2*>(smem4 + G4::STAGE) + grp * L;         // ... and L-element input row
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smem4 + G4::PLAN2);
    uint64_t* bar = bars + 2 + grp;
    volatile int* rslot = ctl + 4 + 2 * grp;
    const int nrows = p.batch * 2 * L;
    const uint64_t pol_tmp = l2_policy((p.hints & 1) ? 1 : 0), pol_out = l2_policy((p.hints & 1) ? 1 : 0);
    int ready_f = -1;   // (thread 0) fields whose column pass is known to be complete
    auto request_row = [&](int R) {   // one thread: gather intermediate row R = (field, plane, j) into `inb`
        const int fb = R / (2 * L), rf = R - fb * (2 * L);
        const int ph = rf / L, j = rf - ph * L;
        // generic -> async proxy: the row buffer's reads always; the column workers' (acquired) global stores once per field --
        // the all-space fence also waits for this thread's own output stores in flight, which is what made every group
        // barrier after it the kernel's top stall when it was issued per row
        if (fb > ready_f) { spin_until(p.sync + 2 + fb, G2::TILES * 2); ready_f = fb; fence_proxy_async_all(); }
        else fence_proxy_async();
        const int grow = ((fb % p.ring) * 2 + ph) * (L / 4) + (j >> 2);
        mbar_expect_tx(bar, ROW_BYTES);
#pragma unroll
        for (int b = 0; b < G2::NBOX_ROW; ++b) tma_load_4d(inb + b * G2::BOXT * 4, &tmp_map, 0, j & 3, b * G2::BOXT, grow, bar, pol_tmp);
    };
    if (t == 0) {
        const int r0 = atomicAdd(p.sync + 1, 1);
        rslot[0] = r0;
        if (r0 < nrows) request_row(r0);
        else mbar_arrive(bar);
    }
    const SyncGroup gsync{1 + grp, NT};
    float2 u;
    { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u = make_float2(cs, sn); }   // w_2L^t
    const float sgn = ((t & 1) ? -1.0f : 1.0f) * p.scale;
    for (int it = 0;; ++it) {
        P2 v[16];
        mbar_wait(bar, it & 1);
        const int r = rslot[it & 1];
        if (r >= nrows) break;
        int rn = 0;
        if (t == 0) rn = atomicAdd(p.sync + 1, 1);   // next row of this group; the latency rides under stage 1
        {
            const float2* __restrict__ row = inb + t;
#define PB_X(n) row[(n) * NT]
            PB_MAKE_LANES_16(v, INV, PB_X)
#undef PB_X
        }
        const int fb = r / (2 * L), rf = r - fb * (2 * L);   // field of the batch, row within its [2][L] planes
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
        if (t == 0) {
            atomicAdd(p.sync + 2 + FUSED_MAX_FIELDS + fb, 1);   // this row of the ring slot has been read
            rslot[(it + 1) & 1] = rn;
            if (rn < nrows) request_row(rn);
            else mbar_arrive(bar);
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
        const int phs = rf / L, rr = rf - phs * L;
        fused_row_store<L, INV>(v, t, p, fb, (2 * rr + phs + L) & (2 * L - 1), sgn, pol_out);   // fftshift along y
    }
}

template <int L, bool INV>
__global__ void __launch_bounds__(Geo4<L>::THREADS, 1)
focus_fused_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap tmp_map, const FusedParams p) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GF = GeoF<L>;
    extern __shared__ __align__(128) float4 smem4[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(smem4) + GF::BAR_OFF);
    volatile int* ctl = reinterpret_cast<volatile int*>(reinterpret_cast<unsigned char*>(smem4) + GF::CTL_OFF);
    const bool col_role = (int)blockIdx.x < p.ncol;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 6; ++i) mbar_init(bar + i, 1);
        ctl[0] = 0;
        mbar_fence_init();
        mbar_expect_tx(bar, (uint32_t)(G4::PLANLEN * sizeof(float2)));
        bulk_g2s(smem4 + G4::PLAN2, p.plan, (uint32_t)(G4::PLANLEN * sizeof(float2)), bar);
        const int ntiles = p.batch * G2::TILES;
        const int w0 = next_tile(p, col_role, ntiles);
        const int w1 = w0 >= 0 ? next_tile(p, col_role, ntiles) : -1;
        ctl[1] = w0;
        ctl[3] = w1;
        if (w0 >= 0) request_tile<L>(in_map, smem4, bar + 1, w0, l2_policy((p.hints & 1) ? 1 : 0));
        else mbar_arrive(bar + 1);
    }
    __syncthreads();
    mbar_wait(bar, 0);   // plan
    // ---- column mode: column workers until the tiles of the launch run out, row workers while tiles of the first field remain
    if (threadIdx.x < 2 * G::NT) fused_col_group<L, INV, 0>(in_map, p, smem4, bar, ctl, col_role);
    else fused_col_group<L, INV, 1>(in_map, p, smem4, bar, ctl, col_role);
    __syncthreads();     // the staging area becomes the four row buffers, the two groups become four
    // ---- row mode: until the rows of the launch run out
    fused_row_group<L, INV>(tmp_map, p, smem4, bar, ctl);
}

template <int L, bool INV>
int launch_fused(Handle* h, const void* in, long long in_ld, long long in_bs, int batch, void* out, int out_kind, long long out_ld,
                 long long out_bs, float scale, float weight, cudaStream_t st) {
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GF = GeoF<L>;
    auto kern = focus_fused_kernel<L, INV>;
    PB_TRY(set_smem_attrs(h, kern, GF::SMEM, 1));
    static const int ring_env = env_int("PB_FUSED_RING", 3);
    static const int ncol_env = env_int("PB_FUSED_NCOL", 0);
    static const int hints = env_int("PB_FOCUS_L2_HINTS", 1);
    const int grid = h->sm_count;
    const int ring = std::max(1, std::min(ring_env, batch));
    // column : row work of one field is ~ 0.37 : 0.63 of an SM-time (PB_FUSED_NCOL overrides the split)
    int ncol = ncol_env > 0 ? ncol_env : (grid * 37 + 50) / 100;
    ncol = std::max(1, std::min(ncol, grid - 1));
    void* scratch = nullptr;
    const size_t tmp_bytes = (size_t)ring * 2 * L * L * sizeof(float2);
    const size_t sync_bytes = (size_t)(2 + 2 * FUSED_MAX_FIELDS) * sizeof(int);
    PB_TRY(ensure_scratch(h, 0, tmp_bytes + sync_bytes, &scratch));
    FusedParams p;
    p.tmp = reinterpret_cast<float2*>(scratch);
    p.sync = reinterpret_cast<int*>(reinterpret_cast<char*>(scratch) + tmp_bytes);
    PB_TRY(get_col4_plan<L>(h, &p.plan));
    p.out = out; p.out_ld = out_ld; p.out_bs = out_bs; p.out_kind = out_kind; p.scale = scale; p.weight = weight;
    p.batch = batch; p.ring = ring; p.ncol = ncol; p.help_tiles = G2::TILES;
    static const int prefetch = env_int("PB_FUSED_PREFETCH", 0);
    p.hints = (hints & 1) | (prefetch ? 2 : 0);
    // (descriptors are copied out at once: the handle's cache may be flushed by the next lookup)
    const CUtensorMap* map = nullptr;
    CUtensorMap in_m, tmp_m;
    {   // intermediate ring: [group = (slot, plane, j/4)][tile][j%4][c]
        const cuuint64_t dims[4] = {4, 4, (cuuint64_t)G2::TILES, (cuuint64_t)ring * 2 * (L / 4)};
        const cuuint64_t str[3] = {32, 128, (cuuint64_t)G2::TILES * 128};
        const cuuint32_t box[4] = {4, 1, (cuuint32_t)G2::BOXT, 1};
        PB_TRY(get_map_c64(h, MapKey{p.tmp, 3, L, ring, 0, 0}, 4, dims, str, box, &map));
        tmp_m = *map;
    }
    {   // input: (field, row, column) complex64; box = one 4-column run of 256 rows
        const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)L, (cuuint64_t)batch};
        const cuuint64_t str[2] = {(cuuint64_t)in_ld * 8, (cuuint64_t)(batch > 1 ? in_bs : (long long)L * in_ld) * 8};
        const cuuint32_t box[3] = {4, (cuuint32_t)G2::BOXR, 1};
        PB_TRY(get_map_c64(h, MapKey{in, 2, L, batch, in_ld, batch > 1 ? in_bs : 0}, 3, dims, str, box, &map));
        in_m = *map;
    }
    PB_CUDA(h, cudaMemsetAsync(p.sync, 0, sync_bytes, st));
    void* args[3] = {&in_m, &tmp_m, &p};
    // cooperative: all CTAs are co-resident or the launch fails -- the workers spin on each other's counters
    PB_CUDA(h, cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(G4::THREADS), args, GF::SMEM, st));
    h->launches++;
    return PB_OK;
}

// =====================================================================================================================
// Plane-unit kernel (PB_FOCUS_V=4): the unit of work is ONE PLANE of one field, u = 2 f + p, so that what has to be live
// in L2 is 8 N^2 bytes (32 MiB at N = 2048) instead of a whole 64 MiB intermediate.  The input of a field is gathered
// twice, once per plane; every byte of the intermediate is written to L2 evict_last, read back from there and discarded.
//   * column work item = one 4-column tile of unit u: gather it, compute half-transform p only (fft_two_stages_u<HALF = p>,
//     the stores of the v2 column kernel).  Each of the CTA's two 256-thread groups takes tiles of its own; the groups
//     share the one 64 KB staging area in turn (tickets n = 0, 1, 2, ...; group n & 1 takes ticket n, on its own
//     "tile full" mbarrier): the last warp of ticket n's group to hold its inputs in registers requests ticket n + 1.
//   * intermediate = two plane buffers (unit u uses buffer u & 1), each in the tile-major [j/4][tile][j%4][c] layout.
//   * gates (one thread per group, before the stores of a tile; the group barrier after it orders the stores):
//       - buffer reuse: a tile of unit u >= 2 waits until every row of unit u - 2 was read (rows_read[u - 2] == L);
//       - L2 budget: tile k of unit u >= 1 waits until rows_read[u - 1] >= 4 (k - slack): the column workers stay at most
//         `slack` tiles ahead of what the row workers have freed (PB_FOCUS_L2_SLACK_MIB; < 0 disables the gate).
//     The rows of unit u are gathered once all TILES tiles of u were signalled (cols_done[u]).
//   * discard: a row counts itself at its line group (4 rows j % 4 = 0..3) once it is in shared memory; the 4th arrival
//     drops the group's TILES lines from L2 (discard.global.L2), fences, and only then counts the row in rows_read -- so
//     no discard can reach a line that the next unit of the same buffer has written.
//   * roles: row workers take tiles of unit 0 only (claimed by compare-and-swap: they never hold a gated tile); column
//     workers join the rows when the tiles run out.
// Progress.  No wait depends on a worker that is itself blocked:
//   (a) tiles are claimed in increasing order, per CTA in ticket order; a group signals a tile (cols_done) before it can
//       wait on a gate, and a group waiting for its next ticket holds (pending) only a tile claimed AFTER the tile its
//       sibling may be gated on -- the sibling frees the staging area before its gate.  So every tile below the lowest
//       gated tile gets signalled.
//   (b) a gated tile of unit u waits on rows of u - 1 and u - 2, whose tiles all lie below it: by (a) and induction over
//       units those rows become readable, and row workers (never gated; the help tiles of unit 0 have no gate) read them.
//   (c) a row group counts its row in rows_read before it can spin on cols_done of a later unit (its next row's gather
//       is deferred behind the count when that unit is not known complete), so the budget gate at the last tiles of a
//       unit, and the column -> row switch, always see the rows already taken.
// =====================================================================================================================
constexpr int PLANE_MAX_UNITS = 2 * FUSED_MAX_FIELDS;
// default L2 budget ahead of the row workers and share of column-role CTAs, from sweeps at N = 2048, 16 fields (H100
// SXM, 400 W): slack 0 / 4 / 8 / 16 MiB / no gate = 158.9 / 156.1 / 152.6 / 149.8 / 148.7 us per propagation; 46 / 53 /
// 60 column CTAs of 132 = 158.5 / 152.6 / 149.2 us (ENGINE_NOTES)
constexpr int kPlaneSlackMiB = 16;
constexpr int kPlaneNcolPct = 45;

template <int L> struct GeoP {
    using G4 = Geo4<L>;
    static constexpr size_t BAR_OFF = G4::BAR_OFF;    // 8 mbarriers: [0] plan, [1 + g] tile of column group g, [3 + g] row of line group g
    static constexpr size_t CTL_OFF = BAR_OFF + 8 * sizeof(uint64_t);
    // ints: [0] warp releases of the staging area, [3] tile of the next ticket (-2: not written yet), [4 + (n & 3)] tile of
    // ticket n, [8 + 2 g + (it & 1)] row of line group g, [16 + g] line group g arrived last at its row's line group
    static constexpr size_t SMEM = CTL_OFF + 32 * sizeof(int);
    static constexpr int GROUP_WARPS = G4::THREADS / 64;   // warps of one column group
};

// one thread: next tile (u * TILES + tile) or -1.  Row-role CTAs only take tiles of unit 0, and never past it.
__device__ __forceinline__ int plane_next_tile(const FusedParams& p, const bool col_role, const int ntiles) {
    if (col_role) {
        const int w = atomicAdd(p.sync, 1);
        return w < ntiles ? w : -1;
    }
    int w = ld_relaxed(p.sync);
    while (w < p.help_tiles) {
        const int seen = atomicCAS(p.sync, w, w + 1);
        if (seen == w) return w;
        w = seen;
    }
    return -1;
}

struct PlaneColState { int pending, checked, pref; bool have_pref; };

// one tile of ticket n (tile index w, unit w / TILES with plane HALF) by column group g
template <int L, bool INV, int HALF>
__device__ __forceinline__ void plane_col_tile(const CUtensorMap& in_map, const FusedParams& p, float4* smem4, uint64_t* bar,
                                               volatile int* ctl, const bool col_role, const int g, const int n, const int w,
                                               const float2 u, PlaneColState& s) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GP = GeoP<L>;
    constexpr int NT = G::NT;
    const int ntiles = 2 * p.batch * G2::TILES;
    const int lt = threadIdx.x & (2 * NT - 1);                       // thread within the group
    const int cp = lt & 1, t = lt >> 1;
    const int lane = threadIdx.x & 31;
    const int unit = w / G2::TILES, tile = w - unit * G2::TILES;
    const float4* __restrict__ stage = smem4 + G4::STAGE;
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smem4 + G4::PLAN2);
    float4* S = smem4 + (g * 2 + cp) * G4::XBUF;
    const SyncGroup gsync{1 + g, 2 * NT};
    const uint64_t pol_tmp = l2_policy((p.hints & 1) ? 2 : 0), pol_in = l2_policy((p.hints & 1) ? 1 : 0);
    const float sgn = (t & 1) ? -1.0f : 1.0f;
    auto sync = [&]() { gsync(); };
    P2 v[16];
    {
        float4 x[16];   // (col, col + 1) x (re, im)
        const float4* __restrict__ sg = stage + lt;   // ((n*NT + t)*2 + cp)
#pragma unroll
        for (int k = 0; k < 16; ++k) x[k] = sg[k * NT * 2];
#define PB_LANES2(n)                                                                                              \
        if (HALF == 0) v[n] = {make_float2(x[n].x, x[n].z), make_float2(x[n].y, x[n].w)};                              \
        else {                                                                                                         \
            const P2 a_ = make_lanes<INV, n>(make_float2(x[n].x, x[n].y)), b_ = make_lanes<INV, n>(make_float2(x[n].z, x[n].w)); \
            v[n] = {make_float2(a_.re.y, b_.re.y), make_float2(a_.im.y, b_.im.y)};                                     \
        }
        PB_LANES2(0) PB_LANES2(1) PB_LANES2(2) PB_LANES2(3) PB_LANES2(4) PB_LANES2(5) PB_LANES2(6) PB_LANES2(7)
        PB_LANES2(8) PB_LANES2(9) PB_LANES2(10) PB_LANES2(11) PB_LANES2(12) PB_LANES2(13) PB_LANES2(14) PB_LANES2(15)
#undef PB_LANES2
        __syncwarp();
        if (lane == 0) {   // this warp holds its inputs: the last of the group's warps hands the staging area to ticket n + 1
            __threadfence_block();
            const unsigned int c = atomicAdd(const_cast<unsigned int*>(reinterpret_cast<volatile unsigned int*>(ctl)), 1u) + 1u;
            __threadfence_block();
            if (c == (unsigned int)(n + 1) * GP::GROUP_WARPS) {
                int wn;
                while ((wn = ctl[3]) == -2) {}   // claimed by the previous ticket's requester, written after its first stages
                ctl[3] = -2;
                ctl[4 + ((n + 1) & 3)] = wn;
                if (wn >= 0) {
                    const int un = wn / G2::TILES;
                    fence_proxy_async();
                    request_tile<L>(in_map, smem4, bar + 2 - g, (un >> 1) * G2::TILES + (wn - un * G2::TILES), pol_in);
                    s.pref = plane_next_tile(p, col_role, ntiles);   // ticket n + 2; the atomic's latency rides under the stages below
                    s.have_pref = true;
                } else {   // no tiles left: tickets n + 1 (the other group) and n + 2 (this group) end the column mode
                    ctl[4 + ((n + 2) & 3)] = -1;
                    mbar_arrive(bar + 2 - g);
                    mbar_arrive(bar + 1 + g);
                }
            }
        }
    }
    fft_two_stages_u<L, INV, HALF>(v, t, S, plan + G4::TW1, plan + G4::TW2, u, sync);
    if (s.have_pref) {   // the other group's requester of ticket n + 2 waits for this
        ctl[3] = s.pref;
        s.have_pref = false;
    }
    if (s.pending >= 0 && lt == 0) {   // the previous tile's stores of ALL warps of the group are three group barriers old
        __threadfence();
        atomicAdd(p.sync + 2 + s.pending, 1);
    }
    fft_last_stage_load<L, INV>(v, t, S);
    if (lt == 0 && unit >= 1) {
        const int* rows_read = p.sync + 2 + PLANE_MAX_UNITS;
        if (unit >= 2 && unit != s.checked) { spin_until(rows_read + unit - 2, L); s.checked = unit; }   // buffer free
        if (p.slack_tiles >= 0 && tile > p.slack_tiles) spin_until(rows_read + unit - 1, 4 * (tile - p.slack_tiles));   // L2 budget
    }
    sync();   // this group's exchange buffers are free for its next tile (and the gates are passed)
#pragma unroll
    for (int gg = 0; gg < G::GI; ++gg) dftR<G::R3, INV>(v + gg * G::R3);
    // tile-major store: element (j, tile, c) of buffer unit & 1 at ((j/4) * TILES + tile) * 16 + (j%4)*4 + c ; c = 2 cp
    float4* __restrict__ dst = reinterpret_cast<float4*>(
        p.tmp + (long long)(unit & 1) * L * L + ((long long)(t >> 2) * G2::TILES + tile) * 16 + (t & 3) * 4 + 2 * cp);
#pragma unroll
    for (int gg = 0; gg < G::GI; ++gg)
#pragma unroll
        for (int kk = 0; kk < G::R3; ++kk) {
            const P2 y = v[gg * G::R3 + kk];
            const long long o = (long long)((gg * NT + 256 * kk) >> 2) * (G2::TILES * 8);   // float4 units
            float4 q;
            if (HALF == 0) q = make_float4(sgn * y.re.x, sgn * y.im.x, sgn * y.re.y, sgn * y.im.y);
            else q = INV ? make_float4(sgn * y.im.x, -sgn * y.re.x, sgn * y.im.y, -sgn * y.re.y)
                         : make_float4(-sgn * y.im.x, sgn * y.re.x, -sgn * y.im.y, sgn * y.re.y);
            st_hint(dst + o, q, pol_tmp);
        }
    s.pending = unit;
}

template <int L, bool INV>
__device__ __forceinline__ void plane_col_group(const CUtensorMap& in_map, const FusedParams& p, float4* smem4, uint64_t* bar,
                                                volatile int* ctl, const bool col_role, const int g) {
    using G2 = Geo2<L>;
    constexpr int NT = Geo<L>::NT;
    const int lt = threadIdx.x & (2 * NT - 1), t = lt >> 1;
    float2 u1;
    { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u1 = make_float2(cs, sn); }   // w_2L^t = exp(-i pi t / L)
    PlaneColState s{-1, -1, -1, false};
    for (int it = 0;; ++it) {
        const int n = 2 * it + g;   // ticket
        mbar_wait(bar + 1 + g, it & 1);
        const int w = ctl[4 + (n & 3)];
        if (w < 0) break;
        if ((w / G2::TILES) & 1) plane_col_tile<L, INV, 1>(in_map, p, smem4, bar, ctl, col_role, g, n, w, u1, s);
        else plane_col_tile<L, INV, 0>(in_map, p, smem4, bar, ctl, col_role, g, n, w, make_float2(1.f, 0.f), s);
    }
    const SyncGroup gsync{1 + g, 2 * NT};
    gsync();   // every warp of the group has left the loop: its last tile's stores are ordered before the barrier
    if (s.pending >= 0 && lt == 0) {
        __threadfence();
        atomicAdd(p.sync + 2 + s.pending, 1);
    }
}

template <int L, bool INV>
__device__ __forceinline__ void plane_row_group(const CUtensorMap& tmp_map, const FusedParams& p, float4* smem4, uint64_t* bars,
                                                volatile int* ctl) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    constexpr int NT = G::NT, R3 = G::R3, GI = G::GI;
    constexpr uint32_t ROW_BYTES = L * sizeof(float2);
    const int grp = threadIdx.x / NT, t = threadIdx.x - grp * NT;
    float4* S = smem4 + grp * G4::XBUF;                                           // this group's exchange buffer
    float2* inb = reinterpret_cast<float2*>(smem4 + G4::STAGE) + grp * L;         // ... and L-element input row
    const float2* __restrict__ plan = reinterpret_cast<const float2*>(smem4 + G4::PLAN2);
    uint64_t* bar = bars + 3 + grp;
    volatile int* rslot = ctl + 8 + 2 * grp;
    volatile int* last = ctl + 16 + grp;
    int* rows_read = p.sync + 2 + PLANE_MAX_UNITS;
    const int nrows = p.batch * 2 * L;   // rows of all units: R = u * L + j
    // the intermediate is read evict_last so that no line leaves L2 -- written back -- before all four of its rows are read
    const uint64_t pol_tmp = l2_policy((p.hints & 1) ? 2 : 0), pol_out = l2_policy((p.hints & 1) ? 1 : 0);
    int ready_u = -1;   // (thread 0) units whose column pass is known to be complete
    auto request_row = [&](int R) {   // one thread: gather intermediate row R = (unit, j) into `inb`
        const int u = R / L, j = R - u * L;
        if (u > ready_u) { spin_until(p.sync + 2 + u, G2::TILES); ready_u = u; fence_proxy_async_all(); }
        else fence_proxy_async();
        const int grow = (u & 1) * (L / 4) + (j >> 2);
        mbar_expect_tx(bar, ROW_BYTES);
#pragma unroll
        for (int b = 0; b < G2::NBOX_ROW; ++b) tma_load_4d(inb + b * G2::BOXT * 4, &tmp_map, 0, j & 3, b * G2::BOXT, grow, bar, pol_tmp);
    };
    if (t == 0) {
        const int r0 = atomicAdd(p.sync + 1, 1);
        rslot[0] = r0;
        if (r0 < nrows) request_row(r0);
        else mbar_arrive(bar);
    }
    const SyncGroup gsync{1 + grp, NT};
    float2 u;
    { float sn, cs; sincospif(-(float)t / (float)L, &sn, &cs); u = make_float2(cs, sn); }   // w_2L^t
    const float sgn = ((t & 1) ? -1.0f : 1.0f) * p.scale;
    for (int it = 0;; ++it) {
        P2 v[16];
        mbar_wait(bar, it & 1);
        const int r = rslot[it & 1];
        if (r >= nrows) break;
        const int unit = r / L, j = r - unit * L;
        const int lg = (unit & 1) * (L / 4) + (j >> 2);   // line group of the row in the plane buffers
        int rn = 0;
        bool arrived_last = false;
        if (t == 0) {   // next row of this group, and this row's arrival at its line group; both latencies ride under stage 1
            rn = atomicAdd(p.sync + 1, 1);
            arrived_last = atomicInc(p.arrive + lg, 3u) == 3u;   // (wraps to 0: the counter is ready for unit + 2)
        }
        {
            const float2* __restrict__ row = inb + t;
#define PB_X(n) row[(n) * NT]
            PB_MAKE_LANES_16(v, INV, PB_X)
#undef PB_X
        }
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
        if (t == 0) *last = arrived_last;
        gsync();   // every thread of the group holds its inputs in registers: the row buffer is free
        const bool drop = *last;
        bool requested = false;
        if (t == 0) {
            rslot[(it + 1) & 1] = rn;
            if (rn < nrows && rn / L <= ready_u) { request_row(rn); requested = true; }   // no wait: gather it now
        }
        if (drop) {   // all four rows of the line group are in shared memory: its lines are dead
            const char* lines = reinterpret_cast<const char*>(p.tmp) + (size_t)lg * (G2::TILES * 128);
#pragma unroll
            for (int i = 0; i < G2::TILES / NT; ++i) l2_discard(lines + (size_t)(t + i * NT) * 128);
        }
        {
            const float4* __restrict__ s4 = S + pad16(t);
#pragma unroll
            for (int n = 0; n < 16; ++n) v[n] = unpack(s4[n * (NT + NT / 16)]);
        }
        gsync();
        if (t == 0) {
            if (drop) __threadfence();   // the group's discards are ordered before the count that frees the buffer
            atomicAdd(rows_read + unit, 1);
            if (!requested) {
                if (rn < nrows) request_row(rn);   // may wait for the column pass of the next unit: after the count
                else mbar_arrive(bar);
            }
        }
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
        fused_row_store<L, INV>(v, t, p, unit >> 1, (2 * j + (unit & 1) + L) & (2 * L - 1), sgn, pol_out);   // fftshift along y
    }
}

template <int L, bool INV>
__global__ void __launch_bounds__(Geo4<L>::THREADS, 1)
focus_plane_kernel(const __grid_constant__ CUtensorMap in_map, const __grid_constant__ CUtensorMap tmp_map, const FusedParams p) {
    using G = Geo<L>;
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GP = GeoP<L>;
    extern __shared__ __align__(128) float4 smem4[];
    uint64_t* bar = reinterpret_cast<uint64_t*>(reinterpret_cast<unsigned char*>(smem4) + GP::BAR_OFF);
    volatile int* ctl = reinterpret_cast<volatile int*>(reinterpret_cast<unsigned char*>(smem4) + GP::CTL_OFF);
    const bool col_role = (int)blockIdx.x < p.ncol;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 7; ++i) mbar_init(bar + i, 1);
        ctl[0] = 0;
        mbar_fence_init();
        mbar_expect_tx(bar, (uint32_t)(G4::PLANLEN * sizeof(float2)));
        bulk_g2s(smem4 + G4::PLAN2, p.plan, (uint32_t)(G4::PLANLEN * sizeof(float2)), bar);
        const int ntiles = 2 * p.batch * G2::TILES;
        // tickets 0 and 1 (ticket n goes to group n & 1; n + 1 is requested when n has been read)
        const int w0 = plane_next_tile(p, col_role, ntiles);
        ctl[4] = w0;
        ctl[3] = w0 >= 0 ? plane_next_tile(p, col_role, ntiles) : -1;
        if (w0 >= 0) {
            const int u0 = w0 / G2::TILES;
            request_tile<L>(in_map, smem4, bar + 1, (u0 >> 1) * G2::TILES + (w0 - u0 * G2::TILES), l2_policy((p.hints & 1) ? 1 : 0));
        } else {   // no tiles for this CTA: tickets 0 and 1 end the column mode
            ctl[5] = -1;
            mbar_arrive(bar + 1);
            mbar_arrive(bar + 2);
        }
    }
    __syncthreads();
    mbar_wait(bar, 0);   // plan
    // ---- column mode: column workers until the tiles run out, row workers while tiles of unit 0 remain
    plane_col_group<L, INV>(in_map, p, smem4, bar, ctl, col_role, threadIdx.x < 2 * G::NT ? 0 : 1);
    __syncthreads();     // the staging area becomes the four row buffers, the two groups become four
    // ---- row mode: until the rows of the launch run out
    plane_row_group<L, INV>(tmp_map, p, smem4, bar, ctl);
}

template <int L, bool INV>
int launch_plane(Handle* h, const void* in, long long in_ld, long long in_bs, int batch, void* out, int out_kind, long long out_ld,
                 long long out_bs, float scale, float weight, cudaStream_t st) {
    using G2 = Geo2<L>;
    using G4 = Geo4<L>;
    using GP = GeoP<L>;
    auto kern = focus_plane_kernel<L, INV>;
    PB_TRY(set_smem_attrs(h, kern, GP::SMEM, 1));
    static const int ncol_env = env_int("PB_FUSED_NCOL", 0);
    static const int slack_mib = env_int("PB_FOCUS_L2_SLACK_MIB", kPlaneSlackMiB);
    static const int hints = env_int("PB_FOCUS_L2_HINTS", 1);
    const int grid = h->sm_count;
    // per unit the column side does 2 N length-N transforms and gathers 8 N^2 bytes, the row side 4 N transforms and
    // stores the output (PB_FUSED_NCOL overrides the split)
    int ncol = ncol_env > 0 ? ncol_env : (grid * kPlaneNcolPct + 50) / 100;
    ncol = std::max(1, std::min(ncol, grid - 1));
    void* scratch = nullptr;
    const size_t tmp_bytes = (size_t)2 * L * L * sizeof(float2);   // two plane buffers
    const size_t sync_bytes = (size_t)(2 + 2 * PLANE_MAX_UNITS + 2 * (L / 4)) * sizeof(int);
    PB_TRY(ensure_scratch(h, 0, tmp_bytes + sync_bytes, &scratch));
    FusedParams p;
    p.tmp = reinterpret_cast<float2*>(scratch);
    p.sync = reinterpret_cast<int*>(reinterpret_cast<char*>(scratch) + tmp_bytes);
    p.arrive = reinterpret_cast<unsigned int*>(p.sync + 2 + 2 * PLANE_MAX_UNITS);
    PB_TRY(get_col4_plan<L>(h, &p.plan));
    p.out = out; p.out_ld = out_ld; p.out_bs = out_bs; p.out_kind = out_kind; p.scale = scale; p.weight = weight;
    p.batch = batch; p.ring = 1; p.ncol = ncol; p.help_tiles = G2::TILES;
    p.hints = hints & 1;
    p.slack_tiles = slack_mib < 0 ? -1 : (int)(((size_t)slack_mib << 20) / ((size_t)L * 4 * sizeof(float2)));
    const CUtensorMap* map = nullptr;
    CUtensorMap in_m, tmp_m;
    {   // the two plane buffers: [group = (buffer, j/4)][tile][j%4][c]
        const cuuint64_t dims[4] = {4, 4, (cuuint64_t)G2::TILES, (cuuint64_t)2 * (L / 4)};
        const cuuint64_t str[3] = {32, 128, (cuuint64_t)G2::TILES * 128};
        const cuuint32_t box[4] = {4, 1, (cuuint32_t)G2::BOXT, 1};
        PB_TRY(get_map_c64(h, MapKey{p.tmp, 4, L, 1, 0, 0}, 4, dims, str, box, &map));
        tmp_m = *map;
    }
    {   // input: (field, row, column) complex64; box = one 4-column run of 256 rows
        const cuuint64_t dims[3] = {(cuuint64_t)L, (cuuint64_t)L, (cuuint64_t)batch};
        const cuuint64_t str[2] = {(cuuint64_t)in_ld * 8, (cuuint64_t)(batch > 1 ? in_bs : (long long)L * in_ld) * 8};
        const cuuint32_t box[3] = {4, (cuuint32_t)G2::BOXR, 1};
        PB_TRY(get_map_c64(h, MapKey{in, 2, L, batch, in_ld, batch > 1 ? in_bs : 0}, 3, dims, str, box, &map));
        in_m = *map;
    }
    PB_CUDA(h, cudaMemsetAsync(p.sync, 0, sync_bytes, st));
    void* args[3] = {&in_m, &tmp_m, &p};
    // cooperative: all CTAs are co-resident or the launch fails -- the workers spin on each other's counters
    PB_CUDA(h, cudaLaunchCooperativeKernel(reinterpret_cast<const void*>(kern), dim3(grid), dim3(G4::THREADS), args, GP::SMEM, st));
    h->launches++;
    return PB_OK;
}

}  // namespace

// Stacks of >= 2 pupils at N in {1024, 2048}: see the header of this file.  PB_ERR_UNSUPPORTED = not this path's shape.
int try_focus_fused(Handle* h, int N, int dir, const void* in, long long in_ld, long long in_bs, int batch, void* out, int out_kind,
                    long long out_ld, long long out_bs, double scale, double weight, cudaStream_t st) {
    static const int min_batch = env_int("PB_FUSED_MIN_BATCH", 2);
    if (batch < min_batch || (N != 2048 && N != 1024)) return PB_ERR_UNSUPPORTED;
    for (int b0 = 0; b0 < batch; b0 += FUSED_MAX_FIELDS) {
        const int nb = std::min(FUSED_MAX_FIELDS, batch - b0);
        const void* inb = reinterpret_cast<const char*>(in) + (size_t)b0 * in_bs * sizeof(float2);
        void* outb = reinterpret_cast<char*>(out) + (size_t)b0 * out_bs * (out_kind == PB_OUT_COMPLEX ? sizeof(float2) : sizeof(float));
        int rc;
        if (N == 2048) rc = dir < 0 ? launch_fused<2048, false>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st)
                                    : launch_fused<2048, true>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st);
        else rc = dir < 0 ? launch_fused<1024, false>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st)
                          : launch_fused<1024, true>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st);
        if (rc != PB_OK) return rc;
    }
    return PB_OK;
}

// The plane-unit kernel for stacks of >= 2 pupils at N in {1024, 2048}: see above.  PB_ERR_UNSUPPORTED = not this path's shape.
int try_focus_plane(Handle* h, int N, int dir, const void* in, long long in_ld, long long in_bs, int batch, void* out, int out_kind,
                    long long out_ld, long long out_bs, double scale, double weight, cudaStream_t st) {
    static const int min_batch = env_int("PB_FUSED_MIN_BATCH", 2);
    if (batch < min_batch || (N != 2048 && N != 1024)) return PB_ERR_UNSUPPORTED;
    for (int b0 = 0; b0 < batch; b0 += FUSED_MAX_FIELDS) {
        const int nb = std::min(FUSED_MAX_FIELDS, batch - b0);
        const void* inb = reinterpret_cast<const char*>(in) + (size_t)b0 * in_bs * sizeof(float2);
        void* outb = reinterpret_cast<char*>(out) + (size_t)b0 * out_bs * (out_kind == PB_OUT_COMPLEX ? sizeof(float2) : sizeof(float));
        int rc;
        if (N == 2048) rc = dir < 0 ? launch_plane<2048, false>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st)
                                    : launch_plane<2048, true>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st);
        else rc = dir < 0 ? launch_plane<1024, false>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st)
                          : launch_plane<1024, true>(h, inb, in_ld, in_bs, nb, outb, out_kind, out_ld, out_bs, (float)scale, (float)weight, st);
        if (rc != PB_OK) return rc;
    }
    return PB_OK;
}

}  // namespace pb
