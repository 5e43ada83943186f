// Sample QC (DESIGN.md 11): the missing calls of every sample over a block of PLINK .bed rows, and the rows repacked to a
// subset of their samples.
//
// Missing counts.  A 32-bit column word of a row holds 16 samples, two bits each, low bits first; sample s of the word is
// missing (code 01) where bit 2s of w & ~(w >> 1) is set.  One thread per column word walks a slab of rows with four SWAR
// registers: register r holds an 8-bit counter for each of the samples r, r + 4, r + 8, r + 12 (bits 2r + 8k of the
// missing mask, shifted down by 2r).  A byte counts at most 255 rows before it is flushed into 16 int32 totals; the thread
// ends with one integer atomicAdd per sample, so the counts are exact whatever the order of the slabs and the split of
// the rows into calls.  Grids have at most kSmMaxSlabs rows of blocks; a block row takes every gridDim.y-th slab.  Padding samples past n are masked off, and bytes past ceil(n / 4) are never read.
//
// Subsetting.  One thread per output 32-bit word (16 kept samples) holds the 16 source sample indices in registers and
// walks a slab of rows: each output code is read from byte src >> 2, shift 2 (src & 3), of the staged source row.  The
// codes past m in the last word are 0, and only the ceil(m / 4) bytes of an output row are stored.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kSmThreads = 128;
constexpr int kSmMissSlab = 1020;   // rows per missing-count thread: four flushes of the byte counters
constexpr int kSmSubSlab = 64;      // rows per subsetting thread
constexpr int64_t kSmMaxSlabs = 8192;   // rows of blocks per grid

// Bytes [4c, 4c + 4) of a row as a little-endian word; bytes at or past `left` (bytes of the row from 4c on) read as zero.
template <bool ALIGNED>
__device__ __forceinline__ uint32_t column_word(const uint8_t* __restrict__ p, int64_t left) {
    if (ALIGNED) return __ldg(reinterpret_cast<const uint32_t*>(p));   // pitch and base are multiples of 4: in bounds
    uint32_t w = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if (i < left) w |= (uint32_t)__ldg(p + i) << (8 * i);
    return w;
}

template <bool ALIGNED>
__global__ void __launch_bounds__(kSmThreads) sample_missing_kernel(const uint8_t* __restrict__ rows, int64_t pitch,
                                                                    int nv, int n, int32_t* __restrict__ out) {
    const int64_t c = (int64_t)blockIdx.x * kSmThreads + threadIdx.x;   // column word
    if (c >= ((int64_t)n + 15) / 16) return;
    const int valid = (int)min((int64_t)16, (int64_t)n - 16 * c);
    const uint32_t mask = 0x55555555u & (valid >= 16 ? ~0u : (1u << (2 * valid)) - 1u);
    const int64_t left = ((int64_t)n + 3) / 4 - 4 * c;
    int32_t total[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) total[s] = 0;
    for (int64_t v0 = (int64_t)blockIdx.y * kSmMissSlab; v0 < nv; v0 += (int64_t)gridDim.y * kSmMissSlab) {
        const int64_t v1 = min(v0 + kSmMissSlab, (int64_t)nv);
        const uint8_t* p = rows + v0 * pitch + 4 * c;
        for (int64_t v = v0; v < v1;) {
            const int64_t end = min(v + 255, v1);
            uint32_t acc0 = 0, acc1 = 0, acc2 = 0, acc3 = 0;
            for (; v < end; ++v, p += pitch) {
                const uint32_t w = column_word<ALIGNED>(p, left);
                const uint32_t miss = w & ~(w >> 1) & mask;
                acc0 += miss & 0x01010101u;
                acc1 += (miss >> 2) & 0x01010101u;
                acc2 += (miss >> 4) & 0x01010101u;
                acc3 += (miss >> 6) & 0x01010101u;
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                total[4 * k + 0] += (acc0 >> (8 * k)) & 0xFF;
                total[4 * k + 1] += (acc1 >> (8 * k)) & 0xFF;
                total[4 * k + 2] += (acc2 >> (8 * k)) & 0xFF;
                total[4 * k + 3] += (acc3 >> (8 * k)) & 0xFF;
            }
        }
    }
#pragma unroll
    for (int s = 0; s < 16; ++s)
        if (s < valid && total[s] != 0) atomicAdd(out + 16 * c + s, total[s]);
}

template <bool ALIGNED_OUT>
__global__ void __launch_bounds__(kSmThreads) subset_samples_kernel(const uint8_t* __restrict__ rows, int64_t pitch,
                                                                    int nv, const int32_t* __restrict__ keep_idx, int m,
                                                                    uint8_t* __restrict__ out, int64_t out_pitch) {
    const int64_t c = (int64_t)blockIdx.x * kSmThreads + threadIdx.x;   // output word
    if (c >= ((int64_t)m + 15) / 16) return;
    const int valid = (int)min((int64_t)16, (int64_t)m - 16 * c);
    int32_t src[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) src[j] = j < valid ? __ldg(keep_idx + 16 * c + j) : -1;
    const int64_t bytes = min((int64_t)4, ((int64_t)m + 3) / 4 - 4 * c);   // bytes of this word inside the output row
    for (int64_t v0 = (int64_t)blockIdx.y * kSmSubSlab; v0 < nv; v0 += (int64_t)gridDim.y * kSmSubSlab) {
        const int64_t v1 = min(v0 + kSmSubSlab, (int64_t)nv);
        for (int64_t v = v0; v < v1; ++v) {
            const uint8_t* row = rows + v * pitch;
            uint32_t w = 0;
#pragma unroll
            for (int j = 0; j < 16; ++j)
                if (src[j] >= 0) w |= (uint32_t)((__ldg(row + (src[j] >> 2)) >> (2 * (src[j] & 3))) & 3) << (2 * j);
            uint8_t* dst = out + v * out_pitch + 4 * c;
            if (ALIGNED_OUT) {
                *reinterpret_cast<uint32_t*>(dst) = w;
            } else {
#pragma unroll
                for (int i = 0; i < 4; ++i)
                    if (i < bytes) dst[i] = (uint8_t)(w >> (8 * i));
            }
        }
    }
}

}  // namespace

cudaError_t sample_missing(const uint8_t* d_rows, int64_t pitch, int nv, int n, int32_t* d_missing, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    const bool aligned = pitch % 4 == 0 && reinterpret_cast<uintptr_t>(d_rows) % 4 == 0;
    const dim3 grid((unsigned)((((int64_t)n + 15) / 16 + kSmThreads - 1) / kSmThreads),
                    (unsigned)std::min<int64_t>(kSmMaxSlabs, ((int64_t)nv + kSmMissSlab - 1) / kSmMissSlab));
    if (aligned)
        sample_missing_kernel<true><<<grid, kSmThreads, 0, stream>>>(d_rows, pitch, nv, n, d_missing);
    else
        sample_missing_kernel<false><<<grid, kSmThreads, 0, stream>>>(d_rows, pitch, nv, n, d_missing);
    return cudaGetLastError();
}

cudaError_t subset_samples(const uint8_t* d_rows, int64_t pitch, int nv, const int32_t* d_keep_idx, int m, uint8_t* d_out,
                           int64_t out_pitch, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    const bool aligned = out_pitch % 4 == 0 && reinterpret_cast<uintptr_t>(d_out) % 4 == 0;
    const dim3 grid((unsigned)((((int64_t)m + 15) / 16 + kSmThreads - 1) / kSmThreads),
                    (unsigned)std::min<int64_t>(kSmMaxSlabs, ((int64_t)nv + kSmSubSlab - 1) / kSmSubSlab));
    if (aligned)
        subset_samples_kernel<true><<<grid, kSmThreads, 0, stream>>>(d_rows, pitch, nv, d_keep_idx, m, d_out, out_pitch);
    else
        subset_samples_kernel<false><<<grid, kSmThreads, 0, stream>>>(d_rows, pitch, nv, d_keep_idx, m, d_out, out_pitch);
    return cudaGetLastError();
}

}  // namespace vpca
