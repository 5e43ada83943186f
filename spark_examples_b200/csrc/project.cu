// Variant loadings and projection of new samples onto computed principal coordinates (DESIGN.md §6).
//
// With C = J S J (the centering of VariantsPca.scala:199-223) and C u_c = lambda_c u_c (what vpca_compute_pca returns),
//   loadings    w[v][c] = sum_s x[s][v] u_c[s]          n_v = sum_s x[s][v]
//   projection  p_c(y)  = sum_v (y_v - n_v / N) w[v][c] / lambda_c
// and projecting a reference sample j with its own loadings gives u_c[j] back.
//
// Both kernels stream dense sample-major cells in the panel layout of the Gram kernel (vpca_internal.h), int8, bf16
// (integers 0/1/2.. held exactly) or packed e2m1 (cell m is the code 2 m, encode.cu).  No floating-point atomics: every
// sum runs in a fixed order, so results are bitwise reproducible.
//   loadings_kernel: a thread owns VT adjacent variants of a panel and walks ALL samples in order 0 .. N-1; U goes
//     through shared memory in sample tiles.  w[v] depends on column v alone, so it is the same bits whichever path
//     (CSR, .bed, panels) staged the cells and whatever the panel width.
//   above kSplitMinN samples the sum is cut into kRanges fixed ranges whose bounds depend on N alone, the range sums
//     added in range order: loadings_split_kernel (k <= 8) gives each range its own warps, loadings_ranged_kernel
//     (k > 8) walks the ranges one after another in each thread.  w[v] is still a function of column v, U and N only.
//   masked loadings (after vpca_compute_pca_subset): loadings_kernel<..., MASK = true> reads U with zero rows for the
//     samples outside the PCA set and a keep byte per sample next to the U tile; the count adds only kept cells.  A zero U
//     row leaves every accumulator's bits unchanged (fma(d, 0, a) = a, as a never holds -0), so w[v] has the bits of the
//     same kernel run over the kept samples alone.
//   project_kernel: a thread owns one sample and walks the variants of one panel in order; the panel's slice of w and of
//     the means goes through shared memory in variant tiles.  Each panel leaves a partial sum per (sample, component);
//     project_reduce_kernel adds the partials into the accumulator in panel order.
// Cells become doubles without a conversion instruction (the 64-bit I2F runs at a quarter of the DFMA rate on sm_90):
// the integer m goes into the low word of 2^52 and 2^52 is subtracted, one DADD.
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdlib>
#include <cstring>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kThreads = 128;

// cell i (0-based) of a little-endian word of packed cells -> its integer value
template <int BITS>
__device__ __forceinline__ int cell_value(uint64_t word, int i) {
    if constexpr (BITS == 8) {
        return (int)((word >> (8 * i)) & 0xFFu);
    } else if constexpr (BITS == 4) {
        return (int)((word >> (4 * i)) & 0xFu) >> 1;   // code 2 m
    } else {
        // bf16 holding a non-negative integer <= 256: 1.mmmmmmm x 2^e with e = exp - 127 in [0, 8]
        const uint32_t b = (uint32_t)((word >> (16 * i)) & 0xFFFFu);
        const int e = (int)((b >> 7) & 0xFFu) - 127;
        return b == 0 ? 0 : (int)(((0x80u | (b & 0x7Fu)) << (e & 15)) >> 7);
    }
}

__device__ __forceinline__ double int_to_f64(int m) {   // exact for 0 <= m < 2^31
    return __hiloint2double(0x43300000, m) - 4503599627370496.0;
}

template <int BYTES>
__device__ __forceinline__ uint64_t load_word(const uint8_t* p) {
    if constexpr (BYTES == 1) return *p;
    else if constexpr (BYTES == 2) return *reinterpret_cast<const uint16_t*>(p);
    else if constexpr (BYTES == 4) return *reinterpret_cast<const uint32_t*>(p);
    else return *reinterpret_cast<const unsigned long long*>(p);
}

// ---- loadings ------------------------------------------------------------------------------------------------------
// acc[i][c] += x[s][v0 + i] U[s][c] and cnt[i] += x[s][v0 + i] for the ts sample rows of a tile, in order, from the
// thread's cells `r` (row_bytes apart) and the tile's U in shared memory (su[s * KMAX + c]).  MASK: cnt[i] only counts the
// rows whose keep byte sk[s] is nonzero.
template <int BITS, int KMAX, int VT, bool MASK = false>
__device__ __forceinline__ void sum_tile(const uint8_t* r, int64_t row_bytes, const double* su, int ts,
                                         double (&acc)[VT][KMAX], int (&cnt)[VT], const uint8_t* sk = nullptr) {
    constexpr int WB = VT * BITS / 8; // bytes of my VT cells in one sample row
#pragma unroll 8
    for (int s = 0; s < ts; ++s) {
        const uint64_t word = load_word<WB>(r + (int64_t)s * row_bytes);
        double u[KMAX];
#pragma unroll
        for (int c = 0; c < KMAX; c += 2) {
            const double2 uu = *reinterpret_cast<const double2*>(&su[s * KMAX + c]);
            u[c] = uu.x;
            u[c + 1] = uu.y;
        }
#pragma unroll
        for (int i = 0; i < VT; ++i) {
            const int m = cell_value<BITS>(word, i);
            if constexpr (MASK) cnt[i] += sk[s] ? m : 0;
            else cnt[i] += m;
            const double d = int_to_f64(m);
#pragma unroll
            for (int c = 0; c < KMAX; ++c) acc[i][c] = fma(d, u[c], acc[i][c]);
        }
    }
}

// grid (panels, ceil(P / (kThreads * VT))).  U: n x k column-major (ld n).  w: nv x k variant-major, count: nv.
// MASK: keep (n bytes) selects the samples the count adds up; their tile of keep bytes follows the U tile in shared memory.
template <int BITS, int KMAX, int VT, bool MASK = false>
__global__ void __launch_bounds__(kThreads) loadings_kernel(const uint8_t* __restrict__ x, int n, int64_t nv,
                                                            int64_t panel, const double* __restrict__ U, int k,
                                                            double* __restrict__ w, int32_t* __restrict__ count,
                                                            const uint8_t* __restrict__ keep = nullptr) {
    constexpr int TS = 4096 / KMAX;   // samples of U per shared-memory tile (32 KB)
    __shared__ __align__(16) double su[TS * KMAX + (MASK ? TS / 8 : 0)];
    uint8_t* sk = reinterpret_cast<uint8_t*>(su + TS * KMAX);
    const int64_t p = blockIdx.x;
    const int64_t vloc = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * VT;
    const int64_t vg = p * panel + vloc;
    const bool active = vloc < panel && vg < nv;
    const int64_t row_bytes = panel * BITS / 8;
    const uint8_t* col = x + (p * (int64_t)n * panel + vloc) * BITS / 8;
    double acc[VT][KMAX];
    int cnt[VT];
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        cnt[i] = 0;
#pragma unroll
        for (int c = 0; c < KMAX; ++c) acc[i][c] = 0.0;
    }
    for (int s0 = 0; s0 < n; s0 += TS) {
        const int ts = min(TS, n - s0);
        __syncthreads();
        for (int q = threadIdx.x; q < ts * KMAX; q += kThreads) {
            const int s = q / KMAX, c = q - s * KMAX;
            su[q] = c < k ? U[(int64_t)c * n + s0 + s] : 0.0;
        }
        if constexpr (MASK)
            for (int s = threadIdx.x; s < ts; s += kThreads) sk[s] = keep[s0 + s];
        __syncthreads();
        if (!active) continue;
        sum_tile<BITS, KMAX, VT, MASK>(col + (int64_t)s0 * row_bytes, row_bytes, su, ts, acc, cnt, sk);
    }
    if (!active) return;
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int64_t v = vg + i;
        if (v >= nv) break;
        count[v] = cnt[i];
#pragma unroll
        for (int c = 0; c < KMAX; ++c)
            if (c < k) w[v * k + c] = acc[i][c];
    }
}

// Above kSplitMinN samples the sum over the samples is cut into kRanges ranges of `span` samples (the last one shorter),
// span = round_up(ceil(n / kRanges), 32), each summed in order from zero, and the range partials are added in range
// order: w = ((p_0 + p_1) + p_2) + p_3.  The bounds and the order depend on n alone -- not on nv, the panel width, the
// input form or k -- so every path gives w[v] the same bits.  Two kernels sum in this order:
//   loadings_ranged_kernel: loadings_kernel's grid, each thread summing the ranges one after another (a second set of
//     accumulators); used at KMAX 16, where 2 variants per thread already give enough CTAs;
//   loadings_split_kernel (below): the ranges side by side in the warps of a CTA, for KMAX <= 8.
constexpr int kRanges = 4;

__host__ __device__ inline int split_span(int n) { return ((n + kRanges - 1) / kRanges + 31) / 32 * 32; }

template <int BITS, int KMAX, int VT>
__global__ void __launch_bounds__(kThreads) loadings_ranged_kernel(const uint8_t* __restrict__ x, int n, int64_t nv,
                                                                   int64_t panel, const double* __restrict__ U, int k,
                                                                   double* __restrict__ w, int32_t* __restrict__ count) {
    constexpr int TS = 4096 / KMAX;
    __shared__ __align__(16) double su[TS * KMAX];
    const int64_t p = blockIdx.x;
    const int64_t vloc = ((int64_t)blockIdx.y * kThreads + threadIdx.x) * VT;
    const int64_t vg = p * panel + vloc;
    const bool active = vloc < panel && vg < nv;
    const int64_t row_bytes = panel * BITS / 8;
    const uint8_t* col = x + (p * (int64_t)n * panel + vloc) * BITS / 8;
    const int span = split_span(n);
    double acc[VT][KMAX];   // the sum of the running range
    double tot[VT][KMAX];   // the sum of the ranges so far
    int cnt[VT];
#pragma unroll
    for (int i = 0; i < VT; ++i) cnt[i] = 0;
#pragma unroll 1
    for (int jr = 0; jr < kRanges; ++jr) {
        const int lo = min(n, jr * span), hi = min(n, (jr + 1) * span);
#pragma unroll
        for (int i = 0; i < VT; ++i)
#pragma unroll
            for (int c = 0; c < KMAX; ++c) acc[i][c] = 0.0;
        for (int s0 = lo; s0 < hi; s0 += TS) {
            const int ts = min(TS, hi - s0);
            __syncthreads();
            for (int q = threadIdx.x; q < ts * KMAX; q += kThreads) {
                const int s = q / KMAX, c = q - s * KMAX;
                su[q] = c < k ? U[(int64_t)c * n + s0 + s] : 0.0;
            }
            __syncthreads();
            if (active) sum_tile<BITS, KMAX, VT>(col + (int64_t)s0 * row_bytes, row_bytes, su, ts, acc, cnt);
        }
#pragma unroll
        for (int i = 0; i < VT; ++i)
#pragma unroll
            for (int c = 0; c < KMAX; ++c) tot[i][c] = jr == 0 ? acc[i][c] : tot[i][c] + acc[i][c];
    }
    if (!active) return;
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int64_t v = vg + i;
        if (v >= nv) break;
        count[v] = cnt[i];
#pragma unroll
        for (int c = 0; c < KMAX; ++c)
            if (c < k) w[v * k + c] = tot[i][c];
    }
}

// ---- loadings, sample axis split across warps ----------------------------------------------------------------------
// The range order of loadings_ranged_kernel, with the ranges side by side: a CTA is G x kRanges warps, warp (group g,
// range j) owns the VT adjacent variants of lane l of group g and sums range j in order; the range partials are then
// added in shared memory, range by range.  The grid has kRanges times the warps of loadings_kernel's for the same
// variants, which is what keeps enough loads in flight when few variants meet many samples.
// G (variant groups per CTA) only decides which variants a CTA covers, never an order: 2 at KMAX 2 (half the re-reads of
// U per variant); 1 at KMAX 4 and 8, where the accumulators take up to ~200 registers and two CTAs per SM hide each
// other's tile barriers.
__host__ __device__ constexpr int split_groups(int kmax) { return kmax <= 2 ? 2 : 1; }

// grid (panels, ceil(P / (32 * G * VT))), 32 * kRanges * G threads.  Arguments as for loadings_kernel.
template <int BITS, int KMAX, int VT>
__global__ void __launch_bounds__(32 * kRanges * split_groups(KMAX), 2)
    loadings_split_kernel(const uint8_t* __restrict__ x, int n, int64_t nv, int64_t panel, const double* __restrict__ U,
                          int k, double* __restrict__ w, int32_t* __restrict__ count) {
    constexpr int G = split_groups(KMAX);
    constexpr int NT = 32 * kRanges * G;
    constexpr int TS = 1024 / KMAX;    // samples of U per range and tile (kRanges tiles: 32 KB)
    constexpr int R = VT * KMAX;       // partial sums per thread
    __shared__ __align__(16) double su[kRanges * TS * KMAX];   // later: the range partials, G x R x 32
    __shared__ int scnt[G * VT * 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int g = warp % G, j = warp / G;
    const int span = split_span(n);
    const int lo = min(n, j * span), hi = min(n, (j + 1) * span);
    const int64_t p = blockIdx.x;
    const int64_t vloc = (((int64_t)blockIdx.y * G + g) * 32 + lane) * VT;
    const int64_t vg = p * panel + vloc;
    const bool active = vloc < panel && vg < nv;
    const int64_t row_bytes = panel * BITS / 8;
    const uint8_t* col = x + (p * (int64_t)n * panel + vloc) * BITS / 8;
    double acc[VT][KMAX];
    int cnt[VT];
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        cnt[i] = 0;
#pragma unroll
        for (int c = 0; c < KMAX; ++c) acc[i][c] = 0.0;
    }
    for (int t0 = 0; t0 < span; t0 += TS) {   // every warp takes the same number of tiles: the barriers line up
        __syncthreads();
        for (int q = threadIdx.x; q < kRanges * TS * KMAX; q += NT) {
            const int jr = q / (TS * KMAX), rem = q - jr * (TS * KMAX);
            const int s = rem / KMAX, c = rem - s * KMAX;
            const int sg = jr * span + t0 + s;
            su[q] = (c < k && t0 + s < span && sg < n) ? U[(int64_t)c * n + sg] : 0.0;
        }
        __syncthreads();
        const int s0 = lo + t0;
        const int ts = min(TS, hi - s0);
        if (!active || ts <= 0) continue;
        sum_tile<BITS, KMAX, VT>(col + (int64_t)s0 * row_bytes, row_bytes, su + j * TS * KMAX, ts, acc, cnt);
    }
    // range partials, added in range order; lanes are the fastest index, so the shared accesses do not conflict
    double* red = su + g * R * 32 + lane;
    int* rc = scnt + g * VT * 32 + lane;
#pragma unroll 1
    for (int jr = 0; jr < kRanges; ++jr) {
        __syncthreads();
        if (j != jr) continue;
#pragma unroll
        for (int i = 0; i < VT; ++i) {
            if (jr > 0) cnt[i] += rc[i * 32];
#pragma unroll
            for (int c = 0; c < KMAX; ++c)
                if (jr > 0) acc[i][c] = red[(i * KMAX + c) * 32] + acc[i][c];
        }
        if (jr < kRanges - 1) {
#pragma unroll
            for (int i = 0; i < VT; ++i) {
                rc[i * 32] = cnt[i];
#pragma unroll
                for (int c = 0; c < KMAX; ++c) red[(i * KMAX + c) * 32] = acc[i][c];
            }
        }
    }
    if (j != kRanges - 1 || !active) return;
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int64_t v = vg + i;
        if (v >= nv) break;
        count[v] = cnt[i];
#pragma unroll
        for (int c = 0; c < KMAX; ++c)
            if (c < k) w[v * k + c] = acc[i][c];
    }
}

// ---- projection ----------------------------------------------------------------------------------------------------
// grid (panels, ceil(m / kThreads)).  part[(p * m + s) * KMAX + c] = sum over the variants of panel p of
// (y[s][v] - mean[v]) w[v][c], in variant order.
template <int BITS, int KMAX>
__global__ void __launch_bounds__(kThreads) project_kernel(const uint8_t* __restrict__ y, int m, int64_t nv,
                                                           int64_t panel, const double* __restrict__ w,
                                                           const double* __restrict__ mean, int k,
                                                           double* __restrict__ part) {
    constexpr int VTILE = KMAX <= 4 ? 1024 : 256;   // variants of w per shared-memory tile
    constexpr int CPS = 256 / BITS;                 // cells per 32-byte step of a sample row
    __shared__ __align__(16) double sw[VTILE * KMAX];
    __shared__ double smean[VTILE];
    const int64_t p = blockIdx.x;
    const int s = blockIdx.y * kThreads + threadIdx.x;
    const int64_t v0 = p * panel;
    const uint8_t* row = y + (p * (int64_t)m * panel + (int64_t)s * panel) * BITS / 8;
    double acc[KMAX];
#pragma unroll
    for (int c = 0; c < KMAX; ++c) acc[c] = 0.0;
    for (int64_t t0 = 0; t0 < panel && v0 + t0 < nv; t0 += VTILE) {
        const int tv = (int)min((int64_t)VTILE, panel - t0);   // a multiple of 128 (panels are)
        __syncthreads();
        for (int q = threadIdx.x; q < tv * KMAX; q += kThreads) {
            const int vl = q / KMAX, c = q - vl * KMAX;
            const int64_t v = v0 + t0 + vl;
            sw[q] = (c < k && v < nv) ? w[v * k + c] : 0.0;
        }
        for (int q = threadIdx.x; q < tv; q += kThreads) {
            const int64_t v = v0 + t0 + q;
            smean[q] = v < nv ? mean[v] : 0.0;   // cells after nv are zero: (0 - 0) * 0
        }
        __syncthreads();
        if (s >= m) continue;
        const uint4* r = reinterpret_cast<const uint4*>(row + t0 * BITS / 8);
        for (int j = 0; j < tv; j += CPS, r += 2) {
            const uint4 a = r[0], b = r[1];
            const uint64_t q[4] = {(uint64_t)a.x | ((uint64_t)a.y << 32), (uint64_t)a.z | ((uint64_t)a.w << 32),
                                   (uint64_t)b.x | ((uint64_t)b.y << 32), (uint64_t)b.z | ((uint64_t)b.w << 32)};
#pragma unroll
            for (int h = 0; h < 4; ++h) {
#pragma unroll
                for (int i = 0; i < 64 / BITS; ++i) {
                    const int vl = j + h * (64 / BITS) + i;
                    const double d = int_to_f64(cell_value<BITS>(q[h], i)) - smean[vl];
#pragma unroll
                    for (int c = 0; c < KMAX; c += 2) {
                        const double2 ww = *reinterpret_cast<const double2*>(&sw[vl * KMAX + c]);
                        acc[c] = fma(d, ww.x, acc[c]);
                        acc[c + 1] = fma(d, ww.y, acc[c + 1]);
                    }
                }
            }
        }
    }
    if (s >= m) return;
    double* out = part + (p * m + s) * KMAX;
#pragma unroll
    for (int c = 0; c < KMAX; ++c) out[c] = acc[c];
}

// acc[s * acc_ld + c] += part[0][s][c] + part[1][s][c] + ...  (panel order)
template <int KMAX>
__global__ void project_reduce_kernel(const double* __restrict__ part, int64_t npanels, int m, int k,
                                      double* __restrict__ acc, int acc_ld) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= (int64_t)m * k) return;
    const int s = (int)(q / k), c = (int)(q - (int64_t)s * k);
    double a = acc[(int64_t)s * acc_ld + c];
    for (int64_t p = 0; p < npanels; ++p) a += part[(p * m + s) * KMAX + c];
    acc[(int64_t)s * acc_ld + c] = a;
}

int kmax_for(int k) { return k <= 2 ? 2 : k <= 4 ? 4 : k <= 8 ? 8 : 16; }

template <int BITS, int KMAX>
void launch_loadings(const void* d_x, int n, int64_t nv, int64_t panel, const double* d_U, int k, double* d_w,
                     int32_t* d_count, bool split, const uint8_t* d_keep, cudaStream_t stream) {
    constexpr int VT = KMAX >= 16 ? 2 : 4;
    const int64_t npanels = (nv + panel - 1) / panel;
    const uint8_t* x = static_cast<const uint8_t*>(d_x);
    const dim3 grid((unsigned)npanels, (unsigned)((panel + kThreads * VT - 1) / (kThreads * VT)));
    if (d_keep != nullptr) {   // a subset solve: n <= 65 535, the whole order
        loadings_kernel<BITS, KMAX, VT, true><<<grid, kThreads, 0, stream>>>(x, n, nv, panel, d_U, k, d_w, d_count, d_keep);
        return;
    }
    if constexpr (KMAX >= 16) {
        // 2 variants per thread leave enough CTAs already; the warp split would re-read U 4 x as often
        if (split) {
            loadings_ranged_kernel<BITS, KMAX, VT><<<grid, kThreads, 0, stream>>>(x, n, nv, panel, d_U, k, d_w, d_count);
            return;
        }
    } else if (split) {
        constexpr int G = split_groups(KMAX);
        constexpr int CV = 32 * G * VT;   // variants of one CTA
        const dim3 sgrid((unsigned)npanels, (unsigned)((panel + CV - 1) / CV));
        loadings_split_kernel<BITS, KMAX, VT><<<sgrid, 32 * kRanges * G, 0, stream>>>(x, n, nv, panel, d_U, k, d_w, d_count);
        return;
    }
    loadings_kernel<BITS, KMAX, VT><<<grid, kThreads, 0, stream>>>(x, n, nv, panel, d_U, k, d_w, d_count);
}

template <int BITS, int KMAX>
void launch_project(const void* d_y, int m, int64_t nv, int64_t panel, const double* d_w, const double* d_mean, int k,
                    double* d_part, double* d_acc, int acc_ld, cudaStream_t stream) {
    const int64_t npanels = (nv + panel - 1) / panel;
    const dim3 grid((unsigned)npanels, (unsigned)((m + kThreads - 1) / kThreads));
    project_kernel<BITS, KMAX><<<grid, kThreads, 0, stream>>>(static_cast<const uint8_t*>(d_y), m, nv, panel, d_w, d_mean,
                                                              k, d_part);
    const int64_t cells = (int64_t)m * k;
    project_reduce_kernel<KMAX><<<(unsigned)((cells + 255) / 256), 256, 0, stream>>>(d_part, npanels, m, k, d_acc, acc_ld);
}

template <int BITS>
void loadings_bits(const void* d_x, int n, int64_t nv, int64_t panel, const double* d_U, int k, double* d_w,
                   int32_t* d_count, bool split, const uint8_t* d_keep, cudaStream_t stream) {
    switch (kmax_for(k)) {
        case 2: launch_loadings<BITS, 2>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream); break;
        case 4: launch_loadings<BITS, 4>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream); break;
        case 8: launch_loadings<BITS, 8>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream); break;
        default: launch_loadings<BITS, 16>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream); break;
    }
}

template <int BITS>
void project_bits(const void* d_y, int m, int64_t nv, int64_t panel, const double* d_w, const double* d_mean, int k,
                  double* d_part, double* d_acc, int acc_ld, cudaStream_t stream) {
    switch (kmax_for(k)) {
        case 2: launch_project<BITS, 2>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream); break;
        case 4: launch_project<BITS, 4>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream); break;
        case 8: launch_project<BITS, 8>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream); break;
        default: launch_project<BITS, 16>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream); break;
    }
}

}  // namespace

cudaError_t loadings_launch(const void* d_x, int elem_bits, int n, int64_t nv, int64_t panel, const double* d_U, int k,
                            double* d_w, int32_t* d_count, const uint8_t* d_keep, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    // VPCA_LOADINGS_KERNEL=whole|split forces one kernel (to time both at one N, or to test the split below the
    // threshold); the default is the split above kSplitMinN samples
    bool split = n > kSplitMinN;
    if (const char* e = getenv("VPCA_LOADINGS_KERNEL")) {
        if (strcmp(e, "whole") == 0) split = false;
        else if (strcmp(e, "split") == 0) split = true;
    }
    if (elem_bits == 8) loadings_bits<8>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream);
    else if (elem_bits == 16) loadings_bits<16>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream);
    else loadings_bits<4>(d_x, n, nv, panel, d_U, k, d_w, d_count, split, d_keep, stream);
    return cudaGetLastError();
}

int64_t project_scratch_doubles(int m, int64_t nv, int64_t panel, int k) {
    return ((nv + panel - 1) / panel) * (int64_t)m * kmax_for(k);
}

cudaError_t project_launch(const void* d_y, int elem_bits, int m, int64_t nv, int64_t panel, const double* d_w,
                           const double* d_mean, int k, double* d_part, double* d_acc, int acc_ld, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    if (elem_bits == 8) project_bits<8>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream);
    else if (elem_bits == 16) project_bits<16>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream);
    else project_bits<4>(d_y, m, nv, panel, d_w, d_mean, k, d_part, d_acc, acc_ld, stream);
    return cudaGetLastError();
}

}  // namespace vpca
