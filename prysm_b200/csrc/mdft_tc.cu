// Matrix DFT (prysm/fttools.py:155-232, forward apply) as a wgmma complex GEMM for complex64 on sm_90a.
//
//   out(My,Mx) = norm * Ey(My,Ny) @ a(Ny,Nx) @ Ex(Mx,Nx)^T
//
// Mapping onto the Hopper tensor cores
//   * Complex -> real.  A complex matrix stored interleaved is a real matrix with twice the columns.
//     With the basis expanded once per executor to  B'[2j]   = ( E_re[j,:], -E_im[j,:] ) interleaved,
//                                                   B'[2j+1] = ( E_im[j,:],  E_re[j,:] ) interleaved,
//     the product  C'(m, 2j+c) = sum_k' A'(m,k') B'(2j+c,k')  is the complex product a @ E^T with its
//     (re, im) pairs already interleaved: the user's array is consumed exactly as it lies in memory,
//     both operands are K-major (the only layout wgmma takes for TF32), and 8 real flops are spent per
//     complex MAC (no wasted work).
//   * fp32 accuracy from TF32 MMAs.  x = hi + lo with hi = rn_tf32(x) and lo = rn_tf32(x - hi), both exactly
//     representable in TF32, so however the tensor core converts an fp32 operand it reads them unchanged.
//     a*b ~= hi*hi + hi*lo + lo*hi: three m64n128k8 TF32 wgmmas per K step, the two small products into a
//     second register accumulator so their low bits survive, summed in the epilogue.  Dropped term lo*lo ~ 2^-22.
//   * Association.  (a @ Ex^T) first, written TRANSPOSED by the epilogue; then out^T' = T1^T' @ Ey'^T with
//     split-K (or stream-K) over the long contraction, landing the result, scaled by `norm`, in (My,Mx)
//     orientation.  Same flop count as the reference's left-first order for square problems.
//   * Accumulation.  The tensor core's fp32 accumulate does not round to nearest: the error grows with the number
//     of accumulation steps.  The main accumulator is therefore restarted every CHUNK K-blocks and its value added
//     into an fp32 running sum on the CUDA cores (round-to-nearest), which keeps the result under 1e-6 of the fp64
//     reference; the correction accumulator is 2^-11 smaller and runs undrained.
//
// Kernel shape: one 128 x 128 output tile per CTA, 384 threads in three warpgroups.  Warpgroup 0 is the producer:
// warp 0 issues the TMA loads of a ring of three 64 KB stages (128-byte-swizzled K-major tiles of 32 fp32: A_hi,
// A_lo, B_hi, B_lo, 16 KB each), warps 2-3 form the TF32 split of the A tile in shared memory.  Warpgroups 1 and 2
// are the consumers: each owns 64 rows of the tile and keeps three 64 x 128 fp32 fragments in registers (main
// accumulator, correction accumulator, running sum: 192 registers, hence the setmaxnreg rebalancing).
#include <cuda.h>
#include <cstdlib>

#include "mdft_tc.cuh"

namespace pb {
namespace {

constexpr int BM = 128, BN = 128, BK = 32;   // BK = one 128-byte swizzle row of fp32
constexpr int STAGES = 3;
constexpr int NTHREADS = 384;                // warpgroup 0: TMA + TF32 split; warpgroups 1-2: wgmma + epilogue
constexpr int NCONV = 64;                    // converter threads (warps 2-3)
constexpr int NCONS = 256;                   // consumer threads
constexpr uint32_t A_TILE = BM * BK * 4;     // 16 KB
constexpr uint32_t B_TILE = BN * BK * 4;     // 16 KB
constexpr uint32_t STAGE_BYTES = 2 * A_TILE + 2 * B_TILE;  // 64 KB
constexpr uint32_t SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
static_assert(SMEM_BYTES <= 227 * 1024, "one CTA per SM within the 227 KB a block may opt in to");

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst)),
        "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
// wgmma shared-memory descriptor, K-major with 128-byte swizzle: rows of 32 fp32, 8-row groups 1024 bytes apart
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address
    d |= (uint64_t)1 << 16;                        // leading byte offset (unused for swizzled K-major)
    d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset between 8-row groups
    d |= (uint64_t)1 << 62;                        // SWIZZLE_128B
    return d;
}
// D(64 x 128, fp32 registers) (+)= A(64 x 8) B(128 x 8)^T, TF32 from shared memory; scale_d = 0 overwrites D
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t scale_d) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "setp.ne.b32 p, %66, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n"
        "}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accesses of accumulator registers across wgmma issue / wait
__device__ __forceinline__ void fence_regs(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

__device__ __forceinline__ int ld_acquire_gpu(const int* p) {
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ float tf32_rn(float v) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
    return __uint_as_float(u);
}

struct GemmParams {
    int kblocks;        // split-K: K blocks of 32 handled by one CTA; stream-K: K blocks per tile (a multiple of chunk)
    int chunk;          // K blocks accumulated by the tensor cores between drains into the fp32 running sum
    int mode;           // 0: write complex transposed, times `scale`; 1: write fp32 transposed split-K partials
    float* out;         // mode 0: complex (float2) [N/2][ldo]; mode 1: ws [split][N][ldo]
    long long ldo;      // leading dimension of the transposed output, in output elements
    long long split_stride;  // mode 1: elements between split-K partial planes
    float scale;
    // stream-K only (see wgmma_gemm_kernel<true>)
    int ntn;            // tiles along N
    int ntiles;         // tiles of the launch
    float* part;        // [gridDim.x][BM * BN] partial tiles
    int* flags;         // [gridDim.x] consumer warps of CTA g that have published its partial (zeroed before the launch)
};

// A CTA's work is a list of SEGMENTS (tile, K-block range).  Split-K: one segment, the tile of (blockIdx.x, blockIdx.y)
// and K-block piece blockIdx.z.  Stream-K, for grids that do not fill the GPU: the work of a launch -- tiles x K-blocks,
// in units of one drain chunk -- is cut into gridDim.x equal contiguous ranges, one per CTA (one CTA per SM).  A range
// covers the tail of one tile, possibly whole tiles, and the head of another; ring stage and phase counters simply run
// on across segments.  The segment that STARTS a tile's K range owns the tile's output; it is its CTA's last segment.
// Every segment that starts inside a tile is its CTA's FIRST: it writes its partial tile to the CTA's slot of the
// workspace and publishes it (gpu-scope fence + counter) before the CTA goes on, so a partial is never published after
// a wait.  The owner adds the partials of CTAs g+1, g+2, ... in that fixed order (deterministic) and stores.
struct Seg { int tile, kb0, kb1, m0, n0; };
// segment of the CTA's range [u, u1) that starts at unit u
__device__ __forceinline__ Seg sk_segment(int u, int u1, int upt, int chunk, int ntn) {
    Seg s;
    s.tile = u / upt;
    const int ub = u - s.tile * upt;
    const int ue = min(upt, ub + (u1 - u));
    s.kb0 = ub * chunk; s.kb1 = ue * chunk;
    s.m0 = (s.tile / ntn) * BM; s.n0 = (s.tile % ntn) * BN;
    return s;
}

template <bool SK>
__global__ void __launch_bounds__(NTHREADS, 1)
wgmma_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmBhi,
                  const __grid_constant__ CUtensorMap tmBlo, const GemmParams p) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
    uint64_t* full = bars;              // [STAGES]  TMA -> converters
    uint64_t* conv = bars + STAGES;     // [STAGES]  converters -> consumers: the split A tile is in shared memory
    uint64_t* empty = bars + 2 * STAGES;  // [STAGES]  consumers -> TMA: the wgmmas that read the stage completed

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int CHUNK = p.chunk;
    const int G = gridDim.x, g = blockIdx.x;
    int u0 = 0, u1 = 1, upt = 1;
    long long U = 1;
    if (SK) {
        upt = p.kblocks / CHUNK;
        U = (long long)p.ntiles * upt;
        u0 = (int)(U * g / G);
        u1 = (int)(U * (g + 1) / G);
    }
    auto segment = [&](int u) -> Seg {
        if (SK) return sk_segment(u, u1, upt, CHUNK, p.ntn);
        const int k0 = blockIdx.z * p.kblocks;
        return Seg{0, k0, k0 + p.kblocks, (int)blockIdx.x * BM, (int)blockIdx.y * BN};
    };
    auto units = [&](const Seg& sg) { return SK ? (sg.kb1 - sg.kb0) / CHUNK : 1; };

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBhi) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&tmBlo) : "memory");
        for (int s = 0; s < STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&conv[s], NCONV); mbar_init(&empty[s], NCONS / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;\n" ::: "memory");
        if (warp == 0 && lane == 0) {  // ===== TMA producer =====
            int i = 0;
            for (int u = u0; u < u1;) {
                const Seg sg = segment(u);
                for (int kb = sg.kb0; kb < sg.kb1; ++kb, ++i) {
                    const int s = i % STAGES;
                    const uint32_t ph = (i / STAGES) & 1;
                    mbar_wait(&empty[s], ph ^ 1);
                    unsigned char* st = smem + s * STAGE_BYTES;
                    mbar_expect_tx(&full[s], A_TILE + 2 * B_TILE);
                    const int kc = kb * BK;
                    tma_load_2d(st, &tmA, kc, sg.m0, &full[s]);
                    tma_load_2d(st + 2 * A_TILE, &tmBhi, kc, sg.n0, &full[s]);
                    tma_load_2d(st + 2 * A_TILE + B_TILE, &tmBlo, kc, sg.n0, &full[s]);
                }
                u += units(sg);
            }
        } else if (warp >= 2) {
            // ===== converters: hi = rn_tf32(x) in place, lo = rn_tf32(x - hi), element for element in the swizzled layout.
            // Forming the split on the tile in shared memory saves a streaming pre-pass over the input and a second
            // operand array.  All loads of a batch are issued before the first use: the conversion sits between the TMA
            // landing and the MMA issue, its latency is on the critical path.
            const int ct = threadIdx.x - 64;
            const int nkb = SK ? (u1 - u0) * CHUNK : p.kblocks;
            for (int i = 0; i < nkb; ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (i / STAGES) & 1;
                mbar_wait(&full[s], ph);
                float4* hi = reinterpret_cast<float4*>(smem + s * STAGE_BYTES);
                float4* lo = hi + A_TILE / 16;
                constexpr int BATCH = 4;     // A_TILE / 16 = 1024 float4 = 4 x (64 threads x 4)
                for (int i0 = ct; i0 < (int)(A_TILE / 16); i0 += NCONV * BATCH) {
                    float4 v[BATCH];
#pragma unroll
                    for (int j = 0; j < BATCH; ++j) v[j] = hi[i0 + NCONV * j];
#pragma unroll
                    for (int j = 0; j < BATCH; ++j) {
                        const float4 h = make_float4(tf32_rn(v[j].x), tf32_rn(v[j].y), tf32_rn(v[j].z), tf32_rn(v[j].w));
                        hi[i0 + NCONV * j] = h;
                        lo[i0 + NCONV * j] = make_float4(tf32_rn(v[j].x - h.x), tf32_rn(v[j].y - h.y), tf32_rn(v[j].z - h.z),
                                                         tf32_rn(v[j].w - h.w));
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> wgmma (async proxy) reads
                mbar_arrive(&conv[s]);
            }
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;\n" ::: "memory");
        // ===== consumers: wgmma mainloop, drains into the running sum, epilogue =====
        const int wg = (warp >> 2) - 1;      // rows [64 wg, 64 wg + 64) of the tile
        const int wl = warp & 3;             // warp inside the warpgroup: 16 rows each
        const int ct = threadIdx.x - 128;
        // fragment layout of a 64 x 128 accumulator: element 4j + e is row r0 + 8 (e >> 1), column 8j + c0 + (e & 1)
        const int r0 = 64 * wg + 16 * wl + (lane >> 2), c0 = 2 * (lane & 3);
        int i = 0;   // K-blocks of this CTA so far: ring position
        for (int u = u0; u < u1;) {
            const Seg sg = segment(u);
            float tot[64], acc[64], corr[64];
#pragma unroll
            for (int j = 0; j < 64; ++j) { tot[j] = 0.f; acc[j] = 0.f; corr[j] = 0.f; }
            for (int kb = sg.kb0; kb < sg.kb1; ++kb, ++i) {
                const int s = i % STAGES;
                const uint32_t ph = (i / STAGES) & 1;
                const int kin = (kb - sg.kb0) % CHUNK;
                mbar_wait(&conv[s], ph);
                const uint32_t sa = smem_u32(smem + s * STAGE_BYTES) + wg * (64 * BK * 4);
                const uint64_t a_hi = make_desc(sa), a_lo = make_desc(sa + A_TILE);
                const uint32_t sb = smem_u32(smem + s * STAGE_BYTES) + 2 * A_TILE;
                const uint64_t b_hi = make_desc(sb), b_lo = make_desc(sb + B_TILE);
                wgmma_fence();
                fence_regs(acc);
                fence_regs(corr);
#pragma unroll
                for (int ks = 0; ks < BK / 8; ++ks) {
                    const uint64_t adv = (uint64_t)(ks * 32 >> 4);  // 8 tf32 = 32 B along K inside the swizzle row
                    wgmma_tf32(acc, a_hi + adv, b_hi + adv, (kin | ks) != 0);
                    wgmma_tf32(corr, a_hi + adv, b_lo + adv, ((kb - sg.kb0) | ks) != 0);
                    wgmma_tf32(corr, a_lo + adv, b_hi + adv, 1u);
                }
                wgmma_commit();
                // the stage is released only once its wgmmas are done; with a drain every CHUNK = 2 K-blocks (which needs
                // the main accumulator complete anyway) keeping one group in flight could overlap at most every other
                // block -- not tried, the other warpgroup and the TMA ring cover this wait
                wgmma_wait_all();
                fence_regs(acc);
                fence_regs(corr);
                __syncwarp();
                if (lane == 0) mbar_arrive(&empty[s]);
                if (kin == CHUNK - 1 || kb == sg.kb1 - 1) {
#pragma unroll
                    for (int j = 0; j < 64; ++j) tot[j] += acc[j];
                }
            }
#pragma unroll
            for (int j = 0; j < 64; ++j) tot[j] += corr[j];
            u += units(sg);

            if (SK && sg.kb0 > 0) {
                // a tail or middle piece of its tile: always the FIRST segment of this CTA, so it is published early and
                // never after a wait -- the tile's owner (below) finds it ready when it gets there
                float* __restrict__ dst = p.part + (long long)g * (BM * BN) + ct;
#pragma unroll
                for (int j = 0; j < 64; ++j) __stcg(dst + j * NCONS, tot[j]);
                __threadfence();
                __syncwarp();
                if (lane == 0) atomicAdd(p.flags + g, 1);
                continue;
            }
            if (SK && sg.kb1 < p.kblocks) {
                // the head of a tile whose K range continues in CTAs g+1, g+2, ...: this CTA owns the tile (it is its LAST
                // segment) and adds their partials in that fixed order
                const long long tile_u1 = (long long)(sg.tile + 1) * upt;
                for (int gp = g + 1; gp < G; ++gp) {
                    while (ld_acquire_gpu(p.flags + gp) < NCONS / 32) __nanosleep(64);
                    const float* __restrict__ src = p.part + (long long)gp * (BM * BN) + ct;
#pragma unroll
                    for (int j = 0; j < 64; ++j) tot[j] += __ldcg(src + j * NCONS);
                    if (U * (gp + 1) / G >= tile_u1) break;   // that piece reached the tile's last K-block
                }
            }
            const int m = sg.m0 + r0;
            if (p.mode == 0) {
                float2* __restrict__ out = reinterpret_cast<float2*>(p.out);
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const long long o = (long long)((sg.n0 + 8 * j + c0) >> 1) * p.ldo + m;
                    out[o] = make_float2(p.scale * tot[4 * j], p.scale * tot[4 * j + 1]);
                    out[o + 8] = make_float2(p.scale * tot[4 * j + 2], p.scale * tot[4 * j + 3]);
                }
            } else {
                float* __restrict__ ws = p.out + (long long)blockIdx.z * p.split_stride;
#pragma unroll
                for (int j = 0; j < 16; ++j) {
                    const long long o = (long long)(sg.n0 + 8 * j + c0) * p.ldo + m;
                    ws[o] = tot[4 * j];
                    ws[o + p.ldo] = tot[4 * j + 1];
                    ws[o + 8] = tot[4 * j + 2];
                    ws[o + p.ldo + 8] = tot[4 * j + 3];
                }
            }
        }
    }
}

// complex basis E (m,n) -> real expansion (2m, 2n), hi and lo
__global__ void expand_basis_kernel(const float2* __restrict__ E, int m, int n, float* __restrict__ hi, float* __restrict__ lo) {
    const long long tot = (long long)m * n;
    PB_GRID_STRIDE(i, tot) {
        const int j = (int)(i / n), l = (int)(i - (long long)j * n);
        const float2 e = E[i];
        const long long r0 = (long long)(2 * j) * (2 * n) + 2 * l, r1 = r0 + 2 * n;
        const float v00 = e.x, v01 = -e.y, v10 = e.y, v11 = e.x;
        const float h00 = tf32_rn(v00), h01 = tf32_rn(v01), h10 = tf32_rn(v10), h11 = tf32_rn(v11);
        hi[r0] = h00; hi[r0 + 1] = h01; hi[r1] = h10; hi[r1 + 1] = h11;
        lo[r0] = tf32_rn(v00 - h00); lo[r0 + 1] = tf32_rn(v01 - h01); lo[r1] = tf32_rn(v10 - h10); lo[r1 + 1] = tf32_rn(v11 - h11);
    }
}

// out(i,j) = norm * sum_s ws[s][2i+c][j]
__global__ void reduce_splits_kernel(const float* __restrict__ ws, int splits, int my, int mx, float norm, float2* __restrict__ out) {
    const long long tot = (long long)my * mx;
    const long long plane = (long long)2 * my * mx;
    PB_GRID_STRIDE(e, tot) {
        const int i = (int)(e / mx), j = (int)(e - (long long)i * mx);
        float re = 0.f, im = 0.f;
        for (int s = 0; s < splits; ++s) {
            re += ws[s * plane + (long long)(2 * i) * mx + j];
            im += ws[s * plane + (long long)(2 * i + 1) * mx + j];
        }
        out[e] = make_float2(norm * re, norm * im);
    }
}

int make_map(Handle* h, CUtensorMap* map, const void* base, long long rows, long long cols, int box_rows) {
    const cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t gstr[1] = {(cuuint64_t)cols * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
    return encode_tensor_map(h, map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
}

// C'(M x N) = A'(M x K) @ B'(N x K)^T on the tensor cores; see GemmParams for the output modes.  Split-K: `splits`
// pieces of gp.kblocks K-blocks along grid z.  Stream-K (mode 0 only): one CTA per SM over all tiles, `work` =
// SK_WORK_BYTES of scratch.  `stage` (1 or 2) only keys the launch's route counter.
constexpr int SK_MAX_CTAS = 160;
constexpr long long SK_WORK_BYTES = (long long)SK_MAX_CTAS * BM * BN * 4 + 4096;   // partial tiles + flags

template <bool SK>
int launch_gemm(Handle* h, int stage, const float* A, const float* Bhi, const float* Blo, int M, int N, long long K,
                int splits, GemmParams gp, void* work, cudaStream_t st) {
    CUtensorMap mA, mBhi, mBlo;
    PB_TRY(make_map(h, &mA, A, M, K, BM));
    PB_TRY(make_map(h, &mBhi, Bhi, N, K, BN));
    PB_TRY(make_map(h, &mBlo, Blo, N, K, BN));
    const void* fn = reinterpret_cast<const void*>(wgmma_gemm_kernel<SK>);
    if (attr_needed(h, fn)) PB_CUDA(h, cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_BYTES));
    dim3 grid(M / BM, N / BN, splits);
    if (SK) {
        gp.ntn = N / BN;
        gp.ntiles = (M / BM) * (N / BN);
        gp.part = reinterpret_cast<float*>(work);
        gp.flags = reinterpret_cast<int*>(reinterpret_cast<char*>(work) + (long long)SK_MAX_CTAS * BM * BN * 4);
        grid = dim3(std::min(h->sm_count, SK_MAX_CTAS));
        PB_CUDA(h, cudaMemsetAsync(gp.flags, 0, SK_MAX_CTAS * sizeof(int), st));
    }
    wgmma_gemm_kernel<SK><<<grid, NTHREADS, SMEM_BYTES, st>>>(mA, mBhi, mBlo, gp);
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_MDFT_TC, splits, int(SK) | (stage == 2) << 1 | gp.mode << 2)]++;
    return PB_OK;
}

// stream-K when the tile grid leaves a good part of the SMs idle and each tile splits into few pieces (the owner's
// serial gather stays short); PB_MDFT_STREAMK=0 disables it, =2 forces it wherever it is legal
bool use_streamk(Handle* h, int tiles, int kblocks, int chunk) {
    static const int streamk = [] { const char* e = getenv("PB_MDFT_STREAMK"); return e ? atoi(e) : 1; }();
    return streamk && kblocks % chunk == 0 && tiles % h->sm_count != 0 &&
           (streamk >= 2 || (5 * tiles < 4 * h->sm_count && 4 * tiles >= h->sm_count)) &&
           (long long)tiles * (kblocks / chunk) >= 4LL * h->sm_count;
}

int pick_splits(int ny) {
    // stage 2 has only (Mx/128)*(2My/128) tiles; split its long contraction (2*Ny) to fill the GPU
    const long long kblocks = 2LL * ny / BK;
    int s = 8;
    while (s > 1 && (kblocks % s != 0 || kblocks / s < 4)) s >>= 1;   // at least 128 K elements per split
    return s;
}

}  // namespace

bool mdft_tc_shape_ok(int my, int ny, int mx, int nx) {
    return my % 128 == 0 && mx % 128 == 0 && ny % 128 == 0 && nx % 16 == 0 && ny >= 128 && nx >= 16;
}


}  // namespace pb

using namespace pb;

extern "C" int pb_mdft_tc_supported(int my, int ny, int mx, int nx) { return mdft_tc_shape_ok(my, ny, mx, nx) ? 1 : 0; }

extern "C" int pb_mdft_tc_expand(pb_handle_t hh, const void* E, int m, int n, void* hi, void* lo, void* stream) {
    PB_ENTER(hh);
    if (m < 1 || n < 1 || !E || !hi || !lo) return fail(h, PB_ERR_INVALID, "bad expand arguments");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const long long tot = (long long)m * n;
    const int g = (int)std::min<long long>((tot + 255) / 256, (long long)h->sm_count * 16);
    expand_basis_kernel<<<g, 256, 0, st>>>((const float2*)E, m, n, (float*)hi, (float*)lo);
    PB_LAUNCH_CHECK(h);
    return PB_OK;
}

extern "C" long long pb_mdft_tc_work_bytes(int my, int ny, int mx, int nx) {
    (void)nx;
    const long long t1 = 2LL * ny * mx * 4;                   // T1^T (complex mx x ny)
    const long long ws = (long long)pick_splits(ny) * 2 * my * mx * 4;
    return t1 + ws + 4096 + SK_WORK_BYTES;
}

extern "C" int pb_mdft_tc_apply(pb_handle_t hh, const void* ExB_hi, const void* ExB_lo, const void* EyB_hi,
                                const void* EyB_lo, int my, int ny, int mx, int nx, const void* a, void* out, double norm,
                                void* work, void* stream) {
    PB_ENTER(hh);
    if (!mdft_tc_shape_ok(my, ny, mx, nx)) return fail(h, PB_ERR_UNSUPPORTED, "shape not covered by the tensor-core MDFT");
    if (!ExB_hi || !ExB_lo || !EyB_hi || !EyB_lo || !a || !out || !work) return fail(h, PB_ERR_INVALID, "null pointer");
    // TMA needs 16-byte aligned global base addresses (the 1 KB alignment of the swizzle atoms is a shared-memory matter);
    // every sub-buffer of `work` below starts at a multiple of 16 bytes given the shape constraints
    if (((uintptr_t)a & 15) || ((uintptr_t)work & 15)) return fail(h, PB_ERR_INVALID, "data / work must be 16-byte aligned");
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    const int splits = pick_splits(ny);
    // 2 K-blocks (8 accumulation steps of the tensor core) per drain of the main accumulator
    static const int chunk = [] { const char* e = getenv("PB_MDFT_CHUNK"); return e ? std::max(1, atoi(e)) : 2; }();
    float* t1 = reinterpret_cast<float*>(work);
    float* ws = t1 + 2LL * ny * mx;
    char* skw = reinterpret_cast<char*>(ws + (long long)splits * 2 * my * mx);
    skw += (16 - ((uintptr_t)skw & 15)) & 15;
    {   // stage 1: T1^T(mx, ny) = (a @ Ex^T)^T : M = ny rows of a, N = 2*mx expanded basis rows, K = 2*nx
        GemmParams gp{};
        gp.kblocks = (int)(2LL * nx / BK); gp.chunk = chunk; gp.mode = 0; gp.out = t1; gp.ldo = ny; gp.scale = 1.0f;
        if (use_streamk(h, (ny / BM) * (2 * mx / BN), gp.kblocks, chunk))
            PB_TRY(launch_gemm<true>(h, 1, (const float*)a, (const float*)ExB_hi, (const float*)ExB_lo, ny, 2 * mx, 2LL * nx, 1, gp, skw, st));
        else PB_TRY(launch_gemm<false>(h, 1, (const float*)a, (const float*)ExB_hi, (const float*)ExB_lo, ny, 2 * mx, 2LL * nx, 1, gp, nullptr, st));
    }
    // stage 2: out^T' = T1^T' @ Ey'^T : M = mx, N = 2*my, K = 2*ny.  Few tiles and a long contraction: stream-K over all SMs
    // with the owner's store landing the result, scaled by `norm`, directly in (My, Mx) complex orientation (same index
    // arithmetic as stage 1's transposed complex store with ldo = mx) -- no partial planes, no reduce kernel.  Grids the
    // stream-K rule declines take split-K + reduce.
    {
        GemmParams gp{};
        gp.kblocks = (int)(2LL * ny / BK); gp.chunk = chunk; gp.mode = 0; gp.out = reinterpret_cast<float*>(out); gp.ldo = mx;
        gp.scale = (float)norm;
        if (use_streamk(h, (mx / BM) * (2 * my / BN), gp.kblocks, chunk))
            return launch_gemm<true>(h, 2, t1, (const float*)EyB_hi, (const float*)EyB_lo, mx, 2 * my, 2LL * ny, 1, gp, skw, st);
    }
    {   // split-K partials transposed into ws[s][2my][mx]
        GemmParams gp{};
        gp.kblocks = (int)(2LL * ny / BK / splits); gp.chunk = chunk; gp.mode = 1; gp.out = ws; gp.ldo = mx;
        gp.split_stride = 2LL * my * mx; gp.scale = 1.0f;
        PB_TRY(launch_gemm<false>(h, 2, t1, (const float*)EyB_hi, (const float*)EyB_lo, mx, 2 * my, 2LL * ny, splits, gp, nullptr, st));
    }
    {
        const long long tot = (long long)my * mx;
        const int g = (int)std::min<long long>((tot + 255) / 256, (long long)h->sm_count * 8);
        reduce_splits_kernel<<<g, 256, 0, st>>>(ws, splits, my, mx, (float)norm, (float2*)out);
        PB_LAUNCH_CHECK(h);
        h->route_launches[route_code(PB_ROUTE_MDFT_REDUCE, splits, 0)]++;
    }
    return PB_OK;
}
