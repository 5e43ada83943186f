// Variant quality control (DESIGN.md 10): the four genotype counts of PLINK .bed rows, and the exact Hardy-Weinberg
// p-value of each variant from its counts.
//
// Counts.  A 64-bit word of a row holds 32 samples, two bits each, low bits first.  Its even bits (lo) and odd bits (hi),
// with the padding samples past n cleared, give MISSING = popc(lo & ~hi) (code 01), HET = popc(hi & ~lo) (10) and
// HOM_A2 = popc(lo & hi) (11); HOM_A1 = n - the three (code 00, which is also what zero padding would read as).  One warp
// per variant, or one block for rows of more than kQcWarpBytes bytes; integer sums only, so the counts are exact.
//
// HWE.  One thread per variant walks the relative probabilities of the het counts (vpca.h, vpca_hwe_exact) twice: first
// the total and the observed term, then the tail.  Every double operation is an explicitly rounded intrinsic, so nothing
// is contracted into an FMA and a host restatement with the same operations in the same order gives the same bits.
#include <cuda_runtime.h>

#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kQcThreads = 256;
constexpr int64_t kQcWarpBytes = 4096;   // rows up to this many bytes (16 384 samples) take one warp per variant

// Bytes [8k, 8k + 8) of a row of `nb` bytes as a little-endian word; bytes past nb read as zero.
template <bool ALIGNED>
__device__ __forceinline__ uint64_t row_word(const uint8_t* __restrict__ row, int64_t k, int64_t nb) {
    if (ALIGNED) return reinterpret_cast<const uint64_t*>(row)[k];   // the pitch is a multiple of 8: in bounds
    uint64_t w = 0;
    const int64_t b0 = 8 * k;
#pragma unroll
    for (int i = 0; i < 8; ++i)
        if (b0 + i < nb) w |= (uint64_t)row[b0 + i] << (8 * i);
    return w;
}

// MISSING, HET, HOM_A2 of row words [k0, nw) stepping by `step`
template <bool ALIGNED>
__device__ __forceinline__ void count_words(const uint8_t* __restrict__ row, int n, int64_t k0, int64_t step, int& miss,
                                            int& het, int& hom2) {
    const int64_t nb = ((int64_t)n + 3) / 4, nw = ((int64_t)n + 31) / 32;
    for (int64_t k = k0; k < nw; k += step) {
        const uint64_t w = row_word<ALIGNED>(row, k, nb);
        const int64_t valid = (int64_t)n - 32 * k;   // samples of this word, >= 1
        const uint64_t m = 0x5555555555555555ull & (valid >= 32 ? ~0ull : (1ull << (2 * valid)) - 1ull);
        const uint64_t lo = w & m, hi = (w >> 1) & m;
        miss += __popcll(lo & ~hi);
        het += __popcll(hi & ~lo);
        hom2 += __popcll(lo & hi);
    }
}

__device__ __forceinline__ void store_counts(int32_t* __restrict__ out, int64_t v, int n, int miss, int het, int hom2) {
    int4 c;
    c.x = n - miss - het - hom2;
    c.y = het;
    c.z = hom2;
    c.w = miss;
    reinterpret_cast<int4*>(out)[v] = c;
}

template <bool ALIGNED>
__global__ void __launch_bounds__(kQcThreads) qc_count_warp_kernel(const uint8_t* __restrict__ rows, int64_t pitch, int nv,
                                                                   int n, int32_t* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int64_t v = ((int64_t)blockIdx.x * kQcThreads + threadIdx.x) >> 5;
    if (v >= nv) return;
    int miss = 0, het = 0, hom2 = 0;
    count_words<ALIGNED>(rows + v * pitch, n, lane, 32, miss, het, hom2);
    miss = __reduce_add_sync(0xffffffffu, miss);
    het = __reduce_add_sync(0xffffffffu, het);
    hom2 = __reduce_add_sync(0xffffffffu, hom2);
    if (lane == 0) store_counts(out, v, n, miss, het, hom2);
}

template <bool ALIGNED>
__global__ void __launch_bounds__(kQcThreads) qc_count_block_kernel(const uint8_t* __restrict__ rows, int64_t pitch,
                                                                    int n, int32_t* __restrict__ out) {
    __shared__ int part[3][kQcThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t v = blockIdx.x;
    int miss = 0, het = 0, hom2 = 0;
    count_words<ALIGNED>(rows + v * pitch, n, threadIdx.x, kQcThreads, miss, het, hom2);
    miss = __reduce_add_sync(0xffffffffu, miss);
    het = __reduce_add_sync(0xffffffffu, het);
    hom2 = __reduce_add_sync(0xffffffffu, hom2);
    if (lane == 0) {
        part[0][warp] = miss;
        part[1][warp] = het;
        part[2][warp] = hom2;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        miss = het = hom2 = 0;
        for (int w = 0; w < kQcThreads / 32; ++w) {   // a fixed order; integer sums are exact in any order anyway
            miss += part[0][w];
            het += part[1][w];
            hom2 += part[2][w];
        }
        store_counts(out, v, n, miss, het, hom2);
    }
}

// Sum of the relative probabilities t(h) <= thr over the het counts of (n, r), the mode first, then downward, then upward
// (vpca.h); *t_obs = t(het), or 0 when het lies beyond the first exact zero of its direction.  The counts h, homr, homc
// are held as doubles: integers below 2^53, so every step of them is exact and no conversion sits in the loop.
__device__ double hwe_walk(double n, double r, double m, double het, double thr, double* t_obs) {
    double sum = 1.0 <= thr ? 1.0 : 0.0;
    *t_obs = m == het ? 1.0 : 0.0;
    const double homr0 = (r - m) * 0.5, homc0 = n - m - homr0;
    {
        double t = 1.0, h = m, homr = homr0, homc = homc0;
        while (h >= 2.0) {
            const double num = __dmul_rn(__dmul_rn(t, h), h - 1.0);
            const double den = __dmul_rn(__dmul_rn(4.0, homr + 1.0), homc + 1.0);
            t = __ddiv_rn(num, den);
            h -= 2.0;
            homr += 1.0;
            homc += 1.0;
            if (t == 0.0) break;
            if (h == het) *t_obs = t;
            if (t <= thr) sum = __dadd_rn(sum, t);
        }
    }
    {
        double t = 1.0, h = m, homr = homr0, homc = homc0;
        while (h + 2.0 <= r) {
            const double num = __dmul_rn(__dmul_rn(__dmul_rn(t, 4.0), homr), homc);
            const double den = __dmul_rn(h + 2.0, h + 1.0);
            t = __ddiv_rn(num, den);
            h += 2.0;
            homr -= 1.0;
            homc -= 1.0;
            if (t == 0.0) break;
            if (h == het) *t_obs = t;
            if (t <= thr) sum = __dadd_rn(sum, t);
        }
    }
    return sum;
}

__global__ void __launch_bounds__(kQcThreads) qc_hwe_kernel(const int32_t* __restrict__ counts, int nv,
                                                            double* __restrict__ p) {
    const int64_t v = (int64_t)blockIdx.x * kQcThreads + threadIdx.x;
    if (v >= nv) return;
    const int4 c = reinterpret_cast<const int4*>(counts)[v];
    const int64_t n = (int64_t)c.x + c.y + c.z, het = c.y;
    const int64_t r = 2 * (int64_t)min(c.x, c.z) + het;
    if (r == 0) {   // monomorphic or nothing called
        p[v] = 1.0;
        return;
    }
    int64_t m = r * (2 * n - r) / (2 * n);
    if ((m ^ r) & 1) ++m;
    double t_obs, unused;
    const double dn = (double)n, dr = (double)r, dm = (double)m, dh = (double)het;
    const double total = hwe_walk(dn, dr, dm, dh, __longlong_as_double(0x7ff0000000000000ll), &t_obs);
    const double tail = hwe_walk(dn, dr, dm, dh, __dmul_rn(t_obs, 1.0 + 0x1p-40), &unused);
    p[v] = fmin(__ddiv_rn(tail, total), 1.0);
}

}  // namespace

cudaError_t qc_count(const uint8_t* d_rows, int64_t pitch, int nv, int n, int32_t* d_counts, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    const bool aligned = pitch % 8 == 0 && reinterpret_cast<uintptr_t>(d_rows) % 8 == 0;
    if ((int64_t)(n + 3) / 4 <= kQcWarpBytes) {
        const unsigned grid = (unsigned)(((int64_t)nv * 32 + kQcThreads - 1) / kQcThreads);
        if (aligned)
            qc_count_warp_kernel<true><<<grid, kQcThreads, 0, stream>>>(d_rows, pitch, nv, n, d_counts);
        else
            qc_count_warp_kernel<false><<<grid, kQcThreads, 0, stream>>>(d_rows, pitch, nv, n, d_counts);
    } else if (aligned) {
        qc_count_block_kernel<true><<<(unsigned)nv, kQcThreads, 0, stream>>>(d_rows, pitch, n, d_counts);
    } else {
        qc_count_block_kernel<false><<<(unsigned)nv, kQcThreads, 0, stream>>>(d_rows, pitch, n, d_counts);
    }
    return cudaGetLastError();
}

cudaError_t qc_hwe(const int32_t* d_counts, int nv, double* d_p, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    qc_hwe_kernel<<<(unsigned)(((int64_t)nv + kQcThreads - 1) / kQcThreads), kQcThreads, 0, stream>>>(d_counts, nv, d_p);
    return cudaGetLastError();
}

}  // namespace vpca
