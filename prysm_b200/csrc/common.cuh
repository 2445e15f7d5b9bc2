// Shared declarations for libprysm_b200: handle, error plumbing, complex helpers, fixed-order device reductions.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <algorithm>
#include <cstdint>
#include <complex>
#include <cstdio>
#include <map>
#include <set>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/prysm_b200.h"

namespace pb {

template <typename R> struct cplx_of;
template <> struct cplx_of<float> { using type = float2; };
template <> struct cplx_of<double> { using type = double2; };
template <typename R> using cplx = typename cplx_of<R>::type;

template <typename R> __host__ __device__ inline cplx<R> mk(R x, R y) { cplx<R> c; c.x = x; c.y = y; return c; }
template <typename C> __host__ __device__ inline C cmul(C a, C b) {
    C c; c.x = a.x * b.x - a.y * b.y; c.y = a.x * b.y + a.y * b.x; return c;
}
template <typename C> __host__ __device__ inline C cmulc(C a, C b) {  // a * conj(b)
    C c; c.x = a.x * b.x + a.y * b.y; c.y = a.y * b.x - a.x * b.y; return c;
}
template <typename C> __host__ __device__ inline C cadd(C a, C b) { C c; c.x = a.x + b.x; c.y = a.y + b.y; return c; }
template <typename C> __host__ __device__ inline C csub(C a, C b) { C c; c.x = a.x - b.x; c.y = a.y - b.y; return c; }
template <typename C> __host__ __device__ inline C cconj(C a) { a.y = -a.y; return a; }
template <typename C> __host__ __device__ inline C cscale(C a, decltype(a.x) s) { a.x *= s; a.y *= s; return a; }

// one rounding per operation and no contraction into an fma, like numpy
__device__ inline float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ inline double mul_rn(double a, double b) { return __dmul_rn(a, b); }
__device__ inline float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ inline double add_rn(double a, double b) { return __dadd_rn(a, b); }
__device__ inline float mul_add_rn(float a, float b, float c) { return __fadd_rn(__fmul_rn(a, b), c); }
__device__ inline double mul_add_rn(double a, double b, double c) { return __dadd_rn(__dmul_rn(a, b), c); }

// ---- fixed-order reductions: each combines the same values in the same order on every call ----------------------
struct OpAdd { __device__ double operator()(double a, double b) const { return a + b; } };
struct OpMin { __device__ double operator()(double a, double b) const { return fmin(a, b); } };   // NaN ignored
struct OpMax { __device__ double operator()(double a, double b) const { return fmax(a, b); } };   // NaN ignored
// NaN propagates (ndarray.max)
struct OpMaxNan { __device__ double operator()(double a, double b) const { return (isnan(a) || a > b) ? a : b; } };

// the fold of v over the warp, in lane 0
template <typename Op>
__device__ inline double warp_reduce(double v, Op op) {
    for (int o = 16; o; o >>= 1) v = op(v, __shfl_down_sync(0xffffffffu, v, o));
    return v;
}
template <int N, typename Op>
__device__ inline void warp_reduce(double (&v)[N], Op op) {
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = warp_reduce(v[k], op);
}

// the shared memory of block_reduce: one array per (THREADS, N) in a kernel whatever the op, so that the reductions
// of a kernel take no more shared memory than one of them
template <int THREADS, int N>
__device__ inline double (&block_reduce_smem())[N][THREADS / 32] {
    __shared__ double sh[N][THREADS / 32];
    return sh;
}

// the fold of each v[k] over the block (blockDim.x == THREADS), given to every thread: each warp folds, then warp 0
// folds the THREADS / 32 warp results
template <int THREADS, int N, typename Op>
__device__ inline void block_reduce(double (&v)[N], Op op) {
    double (&sh)[N][THREADS / 32] = block_reduce_smem<THREADS, N>();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    warp_reduce(v, op);
    __syncthreads();                 // sh may still be read by the previous reduction
    if (lane == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) sh[k][wid] = v[k];
    __syncthreads();
    if (wid == 0) {
#pragma unroll
        for (int k = 0; k < N; ++k) {
            double x = sh[k][lane < THREADS / 32 ? lane : 0];
            for (int o = THREADS / 64; o; o >>= 1) {
                const double w = __shfl_down_sync(0xffffffffu, x, o);
                if (lane < o) x = op(x, w);
            }
            if (lane == 0) sh[k][0] = x;
        }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < N; ++k) v[k] = sh[k][0];
}
template <int THREADS, typename Op>
__device__ inline double block_reduce(double v, Op op) {
    double a[1] = {v};
    block_reduce<THREADS>(a, op);
    return a[0];
}

// sh[w][k] = the fold of v[k] over warp w (blockDim.x == THREADS), then a block barrier; the caller combines the
// THREADS / 32 partials of each value in the order it needs
template <int THREADS, int N, typename Op>
__device__ inline void warp_partials(double (&v)[N], Op op, double (&sh)[THREADS / 32][N]) {
    warp_reduce(v, op);
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int k = 0; k < N; ++k) sh[threadIdx.x >> 5][k] = v[k];
    __syncthreads();
}

// ---- the grid fold of a reduction (DESIGN.md §4.4) ----------------------------------------------------------------
// Each block reduces its grid-stride share with block_reduce and thread 0 writes the block's N partials to
// part[(blockIdx.y * gridDim.x + blockIdx.x) * N + k]; the last block of its row to arrive then folds the row's partials
// in block order and runs the epilogue.  No float atomics: the same n on the same card gives the same bits.

// true in the last block of row blockIdx.y of the grid to arrive; the block's partials must be written before the call
__device__ inline bool arrive_last(unsigned* counter) {
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(counter + blockIdx.y, 1u) == gridDim.x - 1;
    __syncthreads();
    if (last) __threadfence();
    return last;
}

// the fold over the blocks of row blockIdx.y, in block order per thread then block_reduce, of column k of part
template <int THREADS, int N, typename Op>
__device__ inline double fold_partials(const double* part, int k, Op op, double init) {
    part += (size_t)blockIdx.y * gridDim.x * N;
    double v = init;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += THREADS) v = op(v, __ldcg(part + (size_t)b * N + k));
    return block_reduce<THREADS>(v, op);
}

// the sum of v over the block (blockDim.x == THREADS, a power of two) by a halving tree in sh, given to every thread
template <int THREADS>
__device__ inline double tree_sum(double v, double* sh) {
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int d = THREADS / 2; d > 0; d >>= 1) {
        if ((int)threadIdx.x < d) sh[threadIdx.x] += sh[threadIdx.x + d];
        __syncthreads();
    }
    return sh[0];
}

// exp(2*pi*i*turns) with the argument reduced in fp64 before the sincos.
__device__ inline float2 expi_turns(double turns, float) {
    double fr = turns - rint(turns);
    float s, c; sincospif(2.0f * (float)fr, &s, &c);
    return make_float2(c, s);
}
__device__ inline double2 expi_turns(double turns, double) {
    double fr = turns - rint(turns);
    double s, c; sincospi(2.0 * fr, &s, &c);
    return make_double2(c, s);
}

// what a table of Handle::tables holds (TwKey::kind)
enum TwKind {
    TW_ROOTS = 0,                    // w_n^k, k < n (get_twiddles)
    TW_CHIRP_FWD, TW_CHIRP_INV,      // Bluestein chirp of length n, dir -1 / +1
    TW_FILTER_FWD, TW_FILTER_INV,    // spectrum of the Bluestein filter, dir -1 / +1
    TW_PLAIN_PLAN,                   // stage twiddles of the register FFT engine, FFT_n (get_plain_plan)
    TW_FOCUS_PLAN,                   // plan of the focus pair, FFT_n (get_col4_plan)
    TW_TILE_COUNTERS,                // the focus column kernels' two tile counters (n = 2, one complex64 zero)
};

struct TwKey {
    int n; int dtype; int kind;  // kind: TwKind
    bool operator<(const TwKey& o) const {
        if (n != o.n) return n < o.n;
        if (dtype != o.dtype) return dtype < o.dtype;
        return kind < o.kind;
    }
};

// cache key of a TMA descriptor: everything cuTensorMapEncodeTiled was given
struct MapKey {
    const void* base; int kind; long long a, b, c, d;
    bool operator<(const MapKey& o) const {
        if (base != o.base) return base < o.base;
        if (kind != o.kind) return kind < o.kind;
        if (a != o.a) return a < o.a;
        if (b != o.b) return b < o.b;
        if (c != o.c) return c < o.c;
        return d < o.d;
    }
};

struct Handle {
    int device = 0;
    std::string err;
    long long launches = 0;
    // kernel launches per route of the transform kernels (pb_route_launch_count; the codes are in prysm_b200.h)
    std::map<int, long long> route_launches;
    std::map<TwKey, void*> tables;
    // scratch arenas, grown on demand (never on a warmed-up hot call); slot FOLD_SLOT holds the partials and arrival
    // counters of the grid folds
    void* scratch[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t scratch_bytes[4] = {0, 0, 0, 0};
    int sm_count = 132;
    int max_smem_optin = 0;
    // kernels whose opt-in attributes (dynamic shared memory, carve-out) were set on THIS handle's device.
    // cudaFuncSetAttribute acts on the current device's copy of the function, so the record is per handle
    // (= per device and stream), never a process-wide static.
    std::set<const void*> attr_done;
    std::map<MapKey, CUtensorMap> maps;   // TMA descriptors by (base pointer, geometry)
    // helper stream + events of the entry points that overlap small preparatory launches with the main sequence
    // (pb_polychromatic_czt: the Bluestein plan of unit i+1 beside the transforms of unit i); created on first use
    cudaStream_t side = nullptr;
    cudaEvent_t side_ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
};

// Makes the handle's device current for the duration of an entry point and restores the caller's device on
// the way out (one process may drive several GPUs; torch's current device must not change under the caller).
struct DeviceGuard {
    int prev = -1; bool switched = false;
    explicit DeviceGuard(int want) {
        if (cudaGetDevice(&prev) == cudaSuccess && prev != want) switched = cudaSetDevice(want) == cudaSuccess;
    }
    ~DeviceGuard() { if (switched) cudaSetDevice(prev); }
    DeviceGuard(const DeviceGuard&) = delete;
    DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// NVTX range per C-ABI call (SURVEY section 5): shows up in nsys / ncu --nvtx timelines, a no-op without a tool attached
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};

// First lines of every extern "C" entry point that takes a handle
#define PB_ENTER(hh)                                         \
    pb::Handle* h = reinterpret_cast<pb::Handle*>(hh);       \
    if (!h) return PB_ERR_INVALID;                           \
    pb::DeviceGuard pb_guard_(h->device);                    \
    pb::NvtxRange pb_range_(__func__)

// PB_ENTER for an entry point whose `dtype` selects fp32 (PB_C64) or fp64 (PB_C128) data and which takes `stream`
#define PB_ENTER_REAL(hh)                                                                                      \
    PB_ENTER(hh);                                                                                              \
    if (dtype != PB_C64 && dtype != PB_C128) return pb::fail(h, PB_ERR_INVALID, "dtype must be PB_C64 or PB_C128"); \
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream)

// blocks of a grid-stride launch over n items: enough to cover them, at most 16 per SM
inline int grid_for(long long n, int threads, int sm_count) {
    const long long g = (n + threads - 1) / threads;
    return (int)std::max<long long>(1, std::min<long long>(g, (long long)sm_count * 16));
}

// blocks of one row of a folded reduction over n items: enough to cover them in blocks of 256, at most 4 per SM
inline int fold_blocks(long long n, int sm_count) {
    return (int)std::max<long long>(1, std::min<long long>((n + 255) / 256, (long long)sm_count * 4));
}

#define PB_GRID_STRIDE(i, n) \
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < (n); i += (long long)gridDim.x * blockDim.x)

// calls f(float{}) for PB_C64 and f(double{}) for PB_C128; false for any other dtype.  A launch pair is written once
// as with_real(dtype, [&](auto r) { using R = decltype(r); kernel<R><<<...>>>(...); }), with PB_LAUNCH_CHECK after
// the call: it returns an error code, which the void lambda cannot.
template <typename F>
bool with_real(int dtype, F&& f) {
    if (dtype == PB_C64) { f(float{}); return true; }
    if (dtype == PB_C128) { f(double{}); return true; }
    return false;
}

// calls f with a value of the element type a pb_elem code names (float, double, float2, double2, uint8_t, uint16_t,
// uint32_t, int32_t, int64_t); false for an unknown code.  An entry point that takes only some types skips the others
// with `if constexpr` inside f, so that no kernel is instantiated for them, and reports them after the call.
template <typename F>
bool with_elem(int type, F&& f) {
    switch (type) {
        case PB_ELEM_F32: f(float{}); return true;
        case PB_ELEM_F64: f(double{}); return true;
        case PB_ELEM_C64: f(float2{}); return true;
        case PB_ELEM_C128: f(double2{}); return true;
        case PB_ELEM_U8: f(uint8_t{}); return true;
        case PB_ELEM_U16: f(uint16_t{}); return true;
        case PB_ELEM_U32: f(uint32_t{}); return true;
        case PB_ELEM_I32: f(int32_t{}); return true;
        case PB_ELEM_I64: f(int64_t{}); return true;
        default: return false;
    }
}

// bytes of one element of a pb_elem type; 0 for an unknown code
inline size_t elem_size(int type) {
    size_t s = 0;
    with_elem(type, [&](auto t) { s = sizeof(t); });
    return s;
}

template <typename T, typename... U> constexpr bool is_one_of = (std::is_same<T, U>::value || ...);

// true the first time a kernel is seen on this handle: the caller then sets its opt-in attributes
inline bool attr_needed(Handle* h, const void* fn) { return h->attr_done.insert(fn).second; }

inline int fail(Handle* h, int code, const std::string& msg) {
    if (h) h->err = msg;
    return code;
}

#define PB_CUDA(h, call)                                                                      \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return pb::fail(h, PB_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_)); \
    } while (0)

#define PB_LAUNCH_CHECK(h)                                                                    \
    do {                                                                                      \
        cudaError_t e_ = cudaGetLastError();                                                  \
        if (e_ != cudaSuccess)                                                                \
            return pb::fail(h, PB_ERR_CUDA, std::string("kernel launch: ") + cudaGetErrorString(e_)); \
        (h)->launches++;                                                                      \
    } while (0)

// key of Handle::route_launches (pb_route_launch_count); kinds 8 and up set the sign bit, so the key is formed unsigned
constexpr int route_code(int kind, int L, int flags) {
    return (int)((unsigned)kind << 28 | (unsigned)L << 8 | (unsigned)flags);
}

#define PB_TRY(expr)               \
    do {                           \
        int rc_ = (expr);          \
        if (rc_ != PB_OK) return rc_; \
    } while (0)

int ensure_scratch(Handle* h, int slot, size_t bytes, void** out);
constexpr int FOLD_SLOT = 3;
// the partials (rows * blocks * per doubles) and the rows arrival counters, zeroed on st, of a grid fold
int fold_scratch(Handle* h, int rows, int blocks, int per, cudaStream_t st, double** part, unsigned** counters);
// (A, B, C) of P_{n+1}^(alpha,beta) = (A x + B) P_n - C P_{n-1}, DLMF 18.9 as the reference writes them (synthesis.cu)
void jacobi_abc(int n, double alpha, double beta, double* abc);
// amp * exp(2 pi i kturns opd) into the dense complex array out (count elements in rows of nx); opd and amp (pb_amp_kind)
// have row pitch ld (elements)
int launch_phase_screen(Handle* h, int dtype, const void* amp, int amp_kind, const void* opd, double kturns, long long count,
                        long long nx, long long ld, void* out, cudaStream_t st);
// device table of w_n^k = exp(-2*pi*i*k/n), k in [0,n)
int get_twiddles(Handle* h, int n, int dtype, const void** out);
// upload a host fp64 complex table in the precision of key.dtype and cache it in the handle
int upload_table(Handle* h, const TwKey& key, const std::vector<std::complex<double>>& t, const void** out);
// the handle's device table `key`; on a miss, build(t) fills the empty host table t, which upload_table then uploads
template <typename F>
int cached_table(Handle* h, const TwKey& key, F&& build, const void** out) {
    auto it = h->tables.find(key);
    if (it != h->tables.end()) { *out = it->second; return PB_OK; }
    std::vector<std::complex<double>> t;
    build(t);
    return upload_table(h, key, t, out);
}
// cuTensorMapEncodeTiled (resolved once per process) with unit element strides, no interleave and no out-of-bounds fill
int encode_tensor_map(Handle* h, CUtensorMap* map, CUtensorMapDataType type, int rank, const void* base,
                      const cuuint64_t* dims, const cuuint64_t* strides_bytes, const cuuint32_t* box,
                      CUtensorMapSwizzle swizzle, CUtensorMapL2promotion l2);

inline bool is_pow2(int n) { return n > 0 && (n & (n - 1)) == 0; }
inline int ilog2(int n) { int l = 0; while ((1 << l) < n) ++l; return l; }
inline size_t csize(int dtype) { return dtype == PB_C64 ? 8 : 16; }
inline size_t rsize(int dtype) { return dtype == PB_C64 ? 4 : 8; }

}  // namespace pb
