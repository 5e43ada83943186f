// Principal coordinates of a subset K of the samples from the Gram of all of them (vpca_compute_pca_subset, DESIGN.md 8).
//
// The Gram of K is the principal submatrix S[K, K]: subset_gather copies it into a compact m x m buffer that the unchanged
// centring and eigensolver (eig.cu) read like the Gram of an m-sample context.  A removed sample r is then placed on the
// axes of K from its own Gram row: with u_c the eigenvectors of the subset solve, lambda_c its eigenvalues and rho_j the
// row sums of S[K, K], the projection of DESIGN.md 6 with the loadings of the kept samples is
//   p_c(r) = sum_v (x_rv - n_v / m) w_vc / lambda_c = (sum_{j in K} S[r][j] u_c[j] - (1/m) sum_{j in K} rho_j u_c[j]) / lambda_c
// since sum_v x_rv x_jv = S[r][j] and sum_v n_v x_jv = rho_j.  No genotype is read a second time.
//
// Summation order (fixed, so the output is bit-reproducible; no floating-point atomics): a block of kThreads threads
// owns one sum; thread t adds the terms q = t, t + kThreads, ... in increasing q (q indexes K in increasing sample
// order), the 32 partials of a warp are added by a butterfly (xor 16, 8, 4, 2, 1), then the warp sums in warp order.
// sum_j rho_j u_c[j] is computed once per c (subset_rho_kernel), and each p_c(r) ends with one division by lambda_c.
#include <cuda_runtime.h>

#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxK = 16;   // columns of the U buffer the loadings read, and components per block of the relatives kernel

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// grid (ceil(m / kThreads), m): block row q1 copies row idx[q1] of S at the columns of K (K is increasing, so the reads of a
// warp fall in few sectors of one row).
__global__ void __launch_bounds__(kThreads) subset_gather_kernel(const int32_t* __restrict__ S, int n,
                                                                  const int32_t* __restrict__ idx, int m,
                                                                  int32_t* __restrict__ out) {
    const int q1 = blockIdx.y;
    const int q2 = blockIdx.x * kThreads + threadIdx.x;
    if (q2 >= m) return;
    out[(int64_t)q1 * m + q2] = S[(int64_t)idx[q1] * n + idx[q2]];
}

// one thread per entry q of idx: the sample's row of U (u for kept samples, zeros for removed ones) and, for kept
// samples, its row of vecs
__global__ void subset_scatter_kernel(const int32_t* __restrict__ idx, int n, int m, const double* __restrict__ u, int k,
                                      double* __restrict__ U, double* __restrict__ vecs) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const int s = idx[q];
    for (int c = 0; c < max(k, kMaxK); ++c) {
        const double v = (q < m && c < k) ? u[(int64_t)c * m + q] : 0.0;
        if (c < kMaxK) U[(int64_t)c * n + s] = v;
        if (q < m && c < k) vecs[(int64_t)c * n + s] = v;
    }
}

// grid k: t[c] = sum_q rowsum[q] u_c[q]
__global__ void __launch_bounds__(kThreads) subset_rho_kernel(const double* __restrict__ rowsum, int m,
                                                              const double* __restrict__ u, double* __restrict__ t) {
    __shared__ double red[kWarps];
    const int c = blockIdx.x;
    double a = 0.0;
    for (int q = threadIdx.x; q < m; q += kThreads) a = fma(rowsum[q], u[(int64_t)c * m + q], a);
    a = warp_sum(a);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
    __syncthreads();
    if (threadIdx.x == 0) {
        double s = red[0];
        for (int w = 1; w < kWarps; ++w) s += red[w];
        t[c] = s;
    }
}

// grid (r removed samples, ceil(k / kMaxK)): block (b, y) places sample idx[m + b] on components [16 y, 16 y + 16) -- one
// pass over its Gram row at the columns of K for up to 16 components at once
__global__ void __launch_bounds__(kThreads) subset_relatives_kernel(const int32_t* __restrict__ S, int n,
                                                                    const int32_t* __restrict__ idx, int m,
                                                                    const double* __restrict__ u, int k,
                                                                    const double* __restrict__ t,
                                                                    const double* __restrict__ evals,
                                                                    double* __restrict__ vecs) {
    __shared__ double red[kWarps][kMaxK];
    const int row = idx[m + blockIdx.x];
    const int32_t* Sr = S + (int64_t)row * n;
    const int c0 = blockIdx.y * kMaxK;
    u += (int64_t)c0 * m;
    k = min(k - c0, kMaxK);   // components of this block
    double acc[kMaxK];
#pragma unroll
    for (int c = 0; c < kMaxK; ++c) acc[c] = 0.0;
    for (int q = threadIdx.x; q < m; q += kThreads) {
        const double s = (double)Sr[idx[q]];
#pragma unroll
        for (int c = 0; c < kMaxK; ++c)
            if (c < k) acc[c] = fma(s, u[(int64_t)c * m + q], acc[c]);
    }
#pragma unroll
    for (int c = 0; c < kMaxK; ++c) {
        if (c >= k) break;
        const double a = warp_sum(acc[c]);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5][c] = a;
    }
    __syncthreads();
    if (threadIdx.x < k) {
        const int c = threadIdx.x;
        double s = red[0][c];
        for (int w = 1; w < kWarps; ++w) s += red[w][c];
        vecs[(int64_t)(c0 + c) * n + row] = (s - t[c0 + c] / (double)m) / evals[c0 + c];
    }
}

}  // namespace

cudaError_t subset_gather(const int32_t* d_S, int n, const int32_t* d_idx, int m, int32_t* d_SKK, cudaStream_t stream) {
    subset_gather_kernel<<<dim3((m + kThreads - 1) / kThreads, m), kThreads, 0, stream>>>(d_S, n, d_idx, m, d_SKK);
    return cudaGetLastError();
}

cudaError_t subset_place(const int32_t* d_S, int n, const int32_t* d_idx, int m, const double* d_u, const double* d_evals,
                         const double* d_rowsum, int k, double* d_U, double* d_vecs, double* d_t, cudaStream_t stream) {
    subset_scatter_kernel<<<(n + kThreads - 1) / kThreads, kThreads, 0, stream>>>(d_idx, n, m, d_u, k, d_U, d_vecs);
    if (m < n) {
        subset_rho_kernel<<<k, kThreads, 0, stream>>>(d_rowsum, m, d_u, d_t);
        const dim3 grid((unsigned)(n - m), (unsigned)((k + kMaxK - 1) / kMaxK));
        subset_relatives_kernel<<<grid, kThreads, 0, stream>>>(d_S, n, d_idx, m, d_u, k, d_t, d_evals, d_vecs);
    }
    return cudaGetLastError();
}

}  // namespace vpca
