// GRM loadings and projection (DESIGN.md 14): per-variant weights w = Z^T U of the variance-standardized relationship
// matrix's eigenvectors, and new samples placed on those axes, both straight from 2-bit .bed rows on the device.
//
// With z = tab[v][code] (grm.cu's table, indexed by the .bed code; 0 for a missing call and for an unused variant),
//   loadings    w[v][c] = sum_s tab[v][code(s, v)] u_c[s]
//   projection  p_c(y)  = sum_v tab[v][y_v] w[v][c]        (the caller divides by M lambda_c)
// Neither expands Z: a cell is decoded from its two bits through the variant's four doubles in registers or shared
// memory, and multiplied by U or w with one DFMA per component.
//   grm_loadings_kernel: a thread owns VT variants and walks ALL samples in order 0 .. n-1; the CTA's rows go through
//     shared memory in 32-byte tiles (128 samples, a warp reading 32 consecutive bytes of one row), U in the same sample
//     tiles.  w[v] depends on row v's codes, its table, U and n only: not on the rows beside it, the chunk split or the
//     stride.  Each component is its own chain of FMAs, so the first k' columns have the same bits at any k >= k'.
//   grm_project_kernel: a thread owns one byte of the sample axis (4 samples) and walks the variants of a fixed panel
//     in order (a warp reads 32 consecutive bytes of a row); each panel leaves a partial per (sample, component), and
//     grm_project_reduce_kernel adds the partials into the accumulator in panel order.
// No floating-point atomics anywhere, so every result is bitwise reproducible.
#include <cuda_runtime.h>

#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

// z of a .bed code from the variant's table (00 HOM_A1, 01 missing = 0, 10 HET, 11 HOM_A2)
__device__ __forceinline__ double zsel(const double4& t, uint32_t code) {
    const double lo = (code & 1) ? 0.0 : t.x;
    const double hi = (code & 1) ? t.w : t.z;
    return (code & 2) ? hi : lo;
}

template <int KMAX>
__device__ __forceinline__ void load_u(const double* p, double (&u)[KMAX]) {
#pragma unroll
    for (int c = 0; c < KMAX; c += 2) {
        const double2 uu = *reinterpret_cast<const double2*>(p + c);
        u[c] = uu.x;
        u[c + 1] = uu.y;
    }
}

// ---- loadings ------------------------------------------------------------------------------------------------------
constexpr int kLThreads = 128;
constexpr int kLTileBytes = 32;                 // row bytes per tile (128 samples)
constexpr int kLPitch = kLTileBytes / 4 + 1;    // words per staged row: odd, so 32 consecutive rows hit 32 banks
constexpr int kLTileS = 4 * kLTileBytes;        // samples per tile

// grid ceil(nv / (kLThreads VT)).  Row r of the CTA (variant v0 + r, r = i kLThreads + thread) is staged at srow[r
// kLPitch ..].  Samples >= n (padding bits, bytes past ceil(n / 4)) meet U = 0 in the tile: fma(z, 0, a) = a for the
// finite z of a table and an accumulator that never holds -0, so they leave every bit unchanged.
template <int KMAX, int VT>
__global__ void __launch_bounds__(kLThreads) grm_loadings_kernel(const uint8_t* __restrict__ rows, int64_t stride, int nv,
                                                                 int n, const double* __restrict__ tab,
                                                                 const double* __restrict__ U, int k,
                                                                 double* __restrict__ w) {
    constexpr int RB = kLThreads * VT;
    __shared__ uint32_t srow[RB * kLPitch];
    __shared__ __align__(16) double su[kLTileS * KMAX];
    uint8_t* sb = reinterpret_cast<uint8_t*>(srow);
    const int v0 = blockIdx.x * RB;
    const int nb = (n + 3) / 4;
    double4 t[VT];
    double acc[VT][KMAX];
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int v = v0 + i * kLThreads + threadIdx.x;
        t[i] = v < nv ? reinterpret_cast<const double4*>(tab)[v] : make_double4(0.0, 0.0, 0.0, 0.0);
#pragma unroll
        for (int c = 0; c < KMAX; ++c) acc[i][c] = 0.0;
    }
#pragma unroll 1
    for (int b0 = 0; b0 < nb; b0 += kLTileBytes) {
        __syncthreads();
        for (int q = threadIdx.x; q < RB * kLTileBytes; q += kLThreads) {
            const int r = q / kLTileBytes, j = q % kLTileBytes;
            const int v = v0 + r, b = b0 + j;
            sb[r * 4 * kLPitch + j] = (v < nv && b < nb) ? rows[(int64_t)v * stride + b] : 0;
        }
        const int s0 = 4 * b0;
        for (int q = threadIdx.x; q < kLTileS * KMAX; q += kLThreads) {
            const int s = q / KMAX, c = q % KMAX;
            su[q] = (c < k && s0 + s < n) ? U[(int64_t)c * n + s0 + s] : 0.0;
        }
        __syncthreads();
#pragma unroll 1
        for (int wd = 0; wd < kLTileBytes / 4; ++wd) {
            uint32_t word[VT];
#pragma unroll
            for (int i = 0; i < VT; ++i) word[i] = srow[(i * kLThreads + threadIdx.x) * kLPitch + wd];
#pragma unroll 4
            for (int j = 0; j < 16; ++j) {   // sample s0 + 16 wd + j is bits 2j, 2j + 1 of the word
                double u[KMAX];
                load_u<KMAX>(su + (wd * 16 + j) * KMAX, u);
#pragma unroll
                for (int i = 0; i < VT; ++i) {
                    const double z = zsel(t[i], (word[i] >> (2 * j)) & 3u);
#pragma unroll
                    for (int c = 0; c < KMAX; ++c) acc[i][c] = fma(z, u[c], acc[i][c]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int v = v0 + i * kLThreads + threadIdx.x;
        if (v >= nv) continue;
#pragma unroll
        for (int c = 0; c < KMAX; ++c)
            if (c < k) w[(int64_t)v * k + c] = acc[i][c];
    }
}

// ---- projection ----------------------------------------------------------------------------------------------------
constexpr int kPThreads = 128;
constexpr int kPPanel = 1024;   // variants per partial sum: a constant, so the order depends on the call's rows alone

__host__ __device__ constexpr int project_tile(int kmax) { return kmax >= 16 ? 16 : 32; }   // variants per smem tile

// grid (panels, ceil(ceil(n / 4) / kPThreads)).  part[(p * n + s) * KMAX + c] = sum over the variants of panel p, in
// order, of tab[v][code(s, v)] w[v][c].
template <int KMAX>
__global__ void __launch_bounds__(kPThreads) grm_project_kernel(const uint8_t* __restrict__ rows, int64_t stride, int nv,
                                                                int n, const double* __restrict__ tab,
                                                                const double* __restrict__ w, int k,
                                                                double* __restrict__ part) {
    constexpr int TV = project_tile(KMAX);
    __shared__ __align__(16) double sw[TV * KMAX];
    __shared__ double st[TV * 4];
    const int p = blockIdx.x;
    const int b = blockIdx.y * kPThreads + threadIdx.x;   // byte of the sample axis: samples 4 b .. 4 b + 3
    const bool active = b < (n + 3) / 4;
    const int v0 = p * kPPanel, v1 = min(nv, v0 + kPPanel);
    double acc[4][KMAX];
#pragma unroll
    for (int e = 0; e < 4; ++e)
#pragma unroll
        for (int c = 0; c < KMAX; ++c) acc[e][c] = 0.0;
#pragma unroll 1
    for (int t0 = v0; t0 < v1; t0 += TV) {
        __syncthreads();
        for (int q = threadIdx.x; q < TV * KMAX; q += kPThreads) {
            const int vl = q / KMAX, c = q % KMAX;
            const int v = t0 + vl;
            sw[q] = (c < k && v < v1) ? w[(int64_t)v * k + c] : 0.0;
        }
        for (int q = threadIdx.x; q < TV * 4; q += kPThreads) {
            const int v = t0 + q / 4;
            st[q] = v < v1 ? tab[4 * (int64_t)v + (q & 3)] : 0.0;   // past v1: z = 0 and w = 0, no change
        }
        __syncthreads();
        if (!active) continue;
        uint32_t by[TV];
#pragma unroll
        for (int j = 0; j < TV; ++j) by[j] = t0 + j < v1 ? rows[(int64_t)(t0 + j) * stride + b] : 0u;
#pragma unroll
        for (int j = 0; j < TV; ++j) {
            double z[4], u[KMAX];
#pragma unroll
            for (int e = 0; e < 4; ++e) z[e] = st[j * 4 + ((by[j] >> (2 * e)) & 3u)];
            load_u<KMAX>(sw + j * KMAX, u);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
                for (int c = 0; c < KMAX; ++c) acc[e][c] = fma(z[e], u[c], acc[e][c]);
        }
    }
    if (!active) return;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const int s = 4 * b + e;
        if (s >= n) break;
        double* out = part + ((int64_t)p * n + s) * KMAX;
#pragma unroll
        for (int c = 0; c < KMAX; ++c) out[c] = acc[e][c];
    }
}

// acc[s * acc_ld + c] += part[0][s][c] + part[1][s][c] + ...  (panel order)
template <int KMAX>
__global__ void grm_project_reduce_kernel(const double* __restrict__ part, int npanels, int n, int k,
                                          double* __restrict__ acc, int acc_ld) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (int64_t)n * k) return;
    const int s = (int)(q / k), c = (int)(q - (int64_t)s * k);
    double a = acc[(int64_t)s * acc_ld + c];
    for (int p = 0; p < npanels; ++p) a += part[((int64_t)p * n + s) * KMAX + c];
    acc[(int64_t)s * acc_ld + c] = a;
}

int kmax_of(int k) { return k <= 2 ? 2 : k <= 4 ? 4 : k <= 8 ? 8 : 16; }

template <int KMAX>
void launch_loadings(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_U, int k,
                     double* d_w, cudaStream_t stream) {
    constexpr int VT = 2;
    const unsigned grid = (unsigned)((nv + kLThreads * VT - 1) / (kLThreads * VT));
    grm_loadings_kernel<KMAX, VT><<<grid, kLThreads, 0, stream>>>(d_rows, stride, nv, n, d_tab, d_U, k, d_w);
}

template <int KMAX>
void launch_project(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_w, int k,
                    double* d_part, double* d_acc, int acc_ld, cudaStream_t stream) {
    const int npanels = (nv + kPPanel - 1) / kPPanel;
    const int nb = (n + 3) / 4;
    const dim3 grid((unsigned)npanels, (unsigned)((nb + kPThreads - 1) / kPThreads));
    grm_project_kernel<KMAX><<<grid, kPThreads, 0, stream>>>(d_rows, stride, nv, n, d_tab, d_w, k, d_part);
    const int64_t cells = (int64_t)n * k;
    grm_project_reduce_kernel<KMAX><<<(unsigned)((cells + 255) / 256), 256, 0, stream>>>(d_part, npanels, n, k, d_acc,
                                                                                       acc_ld);
}

}  // namespace

cudaError_t grm_loadings(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_U,
                         int k, double* d_w, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    switch (kmax_of(k)) {
        case 2: launch_loadings<2>(d_rows, stride, nv, n, d_tab, d_U, k, d_w, stream); break;
        case 4: launch_loadings<4>(d_rows, stride, nv, n, d_tab, d_U, k, d_w, stream); break;
        case 8: launch_loadings<8>(d_rows, stride, nv, n, d_tab, d_U, k, d_w, stream); break;
        default: launch_loadings<16>(d_rows, stride, nv, n, d_tab, d_U, k, d_w, stream); break;
    }
    return cudaGetLastError();
}

int64_t grm_project_scratch_doubles(int n, int64_t nv, int k) {
    return (nv + kPPanel - 1) / kPPanel * (int64_t)n * kmax_of(k);
}

cudaError_t grm_project(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_w,
                        int k, double* d_part, double* d_acc, int acc_ld, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    switch (kmax_of(k)) {
        case 2: launch_project<2>(d_rows, stride, nv, n, d_tab, d_w, k, d_part, d_acc, acc_ld, stream); break;
        case 4: launch_project<4>(d_rows, stride, nv, n, d_tab, d_w, k, d_part, d_acc, acc_ld, stream); break;
        case 8: launch_project<8>(d_rows, stride, nv, n, d_tab, d_w, k, d_part, d_acc, acc_ld, stream); break;
        default: launch_project<16>(d_rows, stride, nv, n, d_tab, d_w, k, d_part, d_acc, acc_ld, stream); break;
    }
    return cudaGetLastError();
}

}  // namespace vpca
