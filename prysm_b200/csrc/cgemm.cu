// Complex GEMM on the CUDA cores (fp32 / fp64 FMA): the exact-precision matrix-DFT path.
// Used for complex128 (the TF32 tensor-core path is fp32-accurate only), for ragged shapes, and as the arbiter the
// tensor-core path in mdft_tc.cu is tested against.
#include "common.cuh"
#include "mdft_tc.cuh"

namespace pb {

template <typename R, int OP>
__device__ __forceinline__ cplx<R> ld_a(const cplx<R>* __restrict__ A, long long lda, int i, int kk) {
    cplx<R> v = (OP == PB_OP_N || OP == PB_OP_C) ? A[(long long)i * lda + kk] : A[(long long)kk * lda + i];
    if (OP == PB_OP_H || OP == PB_OP_C) v.y = -v.y;
    return v;
}
template <typename R, int OP>
__device__ __forceinline__ cplx<R> ld_b(const cplx<R>* __restrict__ B, long long ldb, int kk, int j) {
    cplx<R> v = (OP == PB_OP_N || OP == PB_OP_C) ? B[(long long)kk * ldb + j] : B[(long long)j * ldb + kk];
    if (OP == PB_OP_H || OP == PB_OP_C) v.y = -v.y;
    return v;
}

// 64x64 output tile, BK = 16, 256 threads, 4x4 micro-tile per thread.
template <typename R, int OPA, int OPB>
__global__ void __launch_bounds__(256) cgemm_kernel(int M, int N, int K, R alpha, const cplx<R>* __restrict__ A,
                                                    long long lda, const cplx<R>* __restrict__ B, long long ldb,
                                                    cplx<R>* __restrict__ C, long long ldc) {
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ R Ar[BK][BM + 4], Ai[BK][BM + 4], Br[BK][BN + 4], Bi[BK][BN + 4];
    const int tid = threadIdx.x;
    const int i0 = blockIdx.y * BM, j0 = blockIdx.x * BN;
    const int tx = tid & 15, ty = tid >> 4;
    // two-level accumulation: 64-term partial sums are folded into the running total, which keeps the
    // rounding error of a K = 4096 contraction near sqrt(64) + sqrt(K/64) ulp instead of sqrt(K)
    R tr[4][4] = {}, ti[4][4] = {};
    R cr[4][4] = {}, ci[4][4] = {};
    for (int k0 = 0; k0 < K; k0 += BK) {
        for (int e = tid; e < BM * BK; e += 256) {
            int ii, kk;
            if (OPA == PB_OP_N || OPA == PB_OP_C) { kk = e % BK; ii = e / BK; } else { ii = e % BM; kk = e / BM; }
            cplx<R> v = mk<R>(R(0), R(0));
            if (i0 + ii < M && k0 + kk < K) v = ld_a<R, OPA>(A, lda, i0 + ii, k0 + kk);
            Ar[kk][ii] = v.x; Ai[kk][ii] = v.y;
        }
        for (int e = tid; e < BN * BK; e += 256) {
            int jj, kk;
            if (OPB == PB_OP_N || OPB == PB_OP_C) { jj = e % BN; kk = e / BN; } else { kk = e % BK; jj = e / BK; }
            cplx<R> v = mk<R>(R(0), R(0));
            if (j0 + jj < N && k0 + kk < K) v = ld_b<R, OPB>(B, ldb, k0 + kk, j0 + jj);
            Br[kk][jj] = v.x; Bi[kk][jj] = v.y;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            R ar[4], ai[4], br[4], bi[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                ar[u] = Ar[kk][ty * 4 + u]; ai[u] = Ai[kk][ty * 4 + u];
                br[u] = Br[kk][tx * 4 + u]; bi[u] = Bi[kk][tx * 4 + u];
            }
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    cr[u][v] = fma(ar[u], br[v], cr[u][v]);
                    cr[u][v] = fma(-ai[u], bi[v], cr[u][v]);
                    ci[u][v] = fma(ar[u], bi[v], ci[u][v]);
                    ci[u][v] = fma(ai[u], br[v], ci[u][v]);
                }
        }
        __syncthreads();
        if (((k0 / BK) & 3) == 3) {
#pragma unroll
            for (int u = 0; u < 4; ++u)
#pragma unroll
                for (int v = 0; v < 4; ++v) {
                    tr[u][v] += cr[u][v]; ti[u][v] += ci[u][v];
                    cr[u][v] = R(0); ci[u][v] = R(0);
                }
        }
    }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int i = i0 + ty * 4 + u, j = j0 + tx * 4 + v;
            if (i < M && j < N) C[(long long)i * ldc + j] = mk<R>(alpha * (tr[u][v] + cr[u][v]), alpha * (ti[u][v] + ci[u][v]));
        }
}

template <typename R, int OPA>
static void launch_b(int opB, dim3 g, cudaStream_t st, int M, int N, int K, R alpha, const cplx<R>* A, long long lda,
                     const cplx<R>* B, long long ldb, cplx<R>* C, long long ldc) {
    switch (opB) {
        case PB_OP_N: cgemm_kernel<R, OPA, PB_OP_N><<<g, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        case PB_OP_T: cgemm_kernel<R, OPA, PB_OP_T><<<g, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        case PB_OP_H: cgemm_kernel<R, OPA, PB_OP_H><<<g, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        default: cgemm_kernel<R, OPA, PB_OP_C><<<g, 256, 0, st>>>(M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
    }
}

template <typename R>
static void launch_ab(int opA, int opB, dim3 g, cudaStream_t st, int M, int N, int K, R alpha, const cplx<R>* A,
                      long long lda, const cplx<R>* B, long long ldb, cplx<R>* C, long long ldc) {
    switch (opA) {
        case PB_OP_N: launch_b<R, PB_OP_N>(opB, g, st, M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        case PB_OP_T: launch_b<R, PB_OP_T>(opB, g, st, M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        case PB_OP_H: launch_b<R, PB_OP_H>(opB, g, st, M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
        default: launch_b<R, PB_OP_C>(opB, g, st, M, N, K, alpha, A, lda, B, ldb, C, ldc); break;
    }
}

int cgemm_simt(Handle* h, int dtype, int opA, int opB, int m, int n, int k, double alpha, const void* A,
               long long lda, const void* B, long long ldb, void* C, long long ldc, cudaStream_t st) {
    dim3 g((n + 63) / 64, (m + 63) / 64);
    if (dtype == PB_C64)
        launch_ab<float>(opA, opB, g, st, m, n, k, (float)alpha, (const float2*)A, lda, (const float2*)B, ldb, (float2*)C, ldc);
    else
        launch_ab<double>(opA, opB, g, st, m, n, k, alpha, (const double2*)A, lda, (const double2*)B, ldb, (double2*)C, ldc);
    PB_LAUNCH_CHECK(h);
    h->route_launches[route_code(PB_ROUTE_CGEMM, 0, dtype | opA << 1 | opB << 3)]++;
    return PB_OK;
}

}  // namespace pb

using namespace pb;

extern "C" int pb_cgemm(pb_handle_t hh, int dtype, int opA, int opB, int m, int n, int k, double alpha, const void* A,
                        long long lda, const void* B, long long ldb, void* C, long long ldc, void* stream) {
    PB_ENTER_REAL(hh);
    if (m < 1 || n < 1 || k < 1 || opA < PB_OP_N || opA > PB_OP_C || opB < PB_OP_N || opB > PB_OP_C)
        return fail(h, PB_ERR_INVALID, "bad gemm arguments");
    return cgemm_simt(h, dtype, opA, opB, m, n, k, alpha, A, lda, B, ldb, C, ldc, st);
}

extern "C" long long pb_mdft_work_elems(int my, int ny, int mx, int nx, int adjoint, int left_first) {
    if (!adjoint) return left_first ? (long long)my * nx : (long long)ny * mx;
    return left_first ? (long long)ny * mx : (long long)my * nx;
}

extern "C" int pb_mdft_apply(pb_handle_t hh, int dtype, const void* Ey, const void* Ex, int my, int ny, int mx, int nx,
                             const void* a, void* out, double norm, int adjoint, int left_first, void* work,
                             void* stream) {
    PB_ENTER_REAL(hh);
    if (my < 1 || ny < 1 || mx < 1 || nx < 1 || !Ey || !Ex || !a || !out || !work) return fail(h, PB_ERR_INVALID, "bad mdft arguments");
    if (!adjoint) {
        if (left_first) {  // (Ey @ a) @ Ex^T
            PB_TRY(cgemm_simt(h, dtype, PB_OP_N, PB_OP_N, my, nx, ny, 1.0, Ey, ny, a, nx, work, nx, st));
            return cgemm_simt(h, dtype, PB_OP_N, PB_OP_T, my, mx, nx, norm, work, nx, Ex, nx, out, mx, st);
        }
        PB_TRY(cgemm_simt(h, dtype, PB_OP_N, PB_OP_T, ny, mx, nx, 1.0, a, nx, Ex, nx, work, mx, st));
        return cgemm_simt(h, dtype, PB_OP_N, PB_OP_N, my, mx, ny, norm, Ey, ny, work, mx, out, mx, st);
    }
    if (left_first) {  // (Ey^H @ g) @ conj(Ex)
        PB_TRY(cgemm_simt(h, dtype, PB_OP_H, PB_OP_N, ny, mx, my, 1.0, Ey, ny, a, mx, work, mx, st));
        return cgemm_simt(h, dtype, PB_OP_N, PB_OP_C, ny, nx, mx, norm, work, mx, Ex, nx, out, nx, st);
    }
    PB_TRY(cgemm_simt(h, dtype, PB_OP_N, PB_OP_C, my, nx, mx, 1.0, a, mx, Ex, nx, work, nx, st));
    return cgemm_simt(h, dtype, PB_OP_H, PB_OP_N, ny, nx, my, norm, Ey, ny, work, nx, out, nx, st);
}
