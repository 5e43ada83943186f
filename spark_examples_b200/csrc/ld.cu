// LD pruning (DESIGN.md 9): Pearson r^2 of allele counts between nearby variants, with pairwise deletion of missing calls,
// read from the int32 Gram G = Y Y^T of the three planes Y of a chunk of c variants (encode_ld_planes: rows [0, c) the A1
// count D, [c, 2c) Q = D^2, [2c, 3c) M = called).  For chunk rows a < b (a the earlier variant i, b the later j) every sum
// over the samples called at both is a lower-triangle entry of G:
//   Sxy = G[b][a]   Sx = G[2c+b][a]   Sy = G[2c+a][b]   Sxx = G[2c+b][c+a]   Syy = G[2c+a][c+b]   n = G[2c+b][2c+a]
//   cov = n Sxy - Sx Sy, vx = n Sxx - Sx^2, vy = n Syy - Sy^2 (exact int64), r2 = (cov * cov) / (vx * vy) in double, each
//   operation rounded once; the pair is in LD iff vx > 0 && vy > 0 && r2 > r2_max.
// A block takes a 32 x 32 tile of pairs (rows b, columns a) of the band the windows cover; the two column reads
// (G[2c+a][b], G[2c+a][c+b]) are staged through shared memory so that every global load runs along a row.  Pass 1 writes
// one bit per pair and scans the bit counts along each row; pass 2 (only when pairs are listed) recomputes the same pairs
// and writes each to its position, in order of b, then a.  The keep-first sweep is one warp walking the owned rows in order.
// Integer sums, three rounded double operations per pair, integer atomics only: the output is bit-reproducible.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kTile = 32;
constexpr int kWarps = 8;

struct PairOut {
    int64_t* pairs;
    double* r2;
    const int64_t* row_start;
    int64_t base, end;
};

// grid (T, row tiles): block (w, y) is row tile bt = bt_lo + y against column tile bt - (T - 1) + w
template <bool EMIT, bool MASKED>
__global__ void __launch_bounds__(kTile * kWarps)
ld_pairs_kernel(LdChunk ch, int bt_lo, uint32_t* __restrict__ bits, const int32_t* __restrict__ seg, PairOut out) {
    __shared__ int32_t t_sy[kTile][kTile + 1];    // [al][bl] = G[2c+a][b]
    __shared__ int32_t t_syy[kTile][kTile + 1];   // [al][bl] = G[2c+a][c+b]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int T = ch.T, w = blockIdx.x, bt = bt_lo + blockIdx.y, at = bt - (T - 1) + w;
    const int b0 = bt * kTile;
    if (at < 0) {   // before the first variant of the chunk: no pairs
        if (!EMIT && threadIdx.x < kTile) bits[(int64_t)(b0 + threadIdx.x) * T + w] = 0u;
        return;
    }
    const int c = ch.c, a0 = at * kTile;
    const int64_t R = 3 * (int64_t)c;
    const int32_t* __restrict__ G = ch.G;
    {   // column reads, coalesced along b
        const int b = b0 + lane;
        for (int al = warp; al < kTile; al += kWarps) {
            const int32_t* ra = G + (2 * (int64_t)c + a0 + al) * R;
            t_sy[al][lane] = ra[b];
            t_syy[al][lane] = ra[c + b];
        }
    }
    __syncthreads();
    const int a = a0 + lane;
    const bool ea = !MASKED || (a < ch.nc && ch.elig[ch.s0 + a] != 0);
    for (int bl = warp; bl < kTile; bl += kWarps) {
        const int b = b0 + bl;
        bool sel = false;
        double r2 = 0.0;
        if (ea && b >= ch.own_lo && b < ch.nc && a < b && ch.s0 + a >= ch.wlo[b] && (!MASKED || ch.elig[ch.s0 + b] != 0)) {
            const int32_t* rb = G + (int64_t)b * R;
            const int32_t* rm = G + (2 * (int64_t)c + b) * R;
            const int64_t n = rm[2 * c + a], sx = rm[a], sxx = rm[c + a], sxy = rb[a];
            const int64_t sy = t_sy[lane][bl], syy = t_syy[lane][bl];
            const int64_t cov = n * sxy - sx * sy, vx = n * sxx - sx * sx, vy = n * syy - sy * sy;
            if (vx > 0 && vy > 0) {
                const double dc = (double)cov;
                r2 = __ddiv_rn(__dmul_rn(dc, dc), __dmul_rn((double)vx, (double)vy));
                sel = r2 > ch.r2_max;
            }
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, sel);
        const int64_t word = (int64_t)b * T + w;
        if (!EMIT) {
            if (lane == 0) bits[word] = mask;
        } else if (sel) {
            const int64_t pos = out.row_start[b] + seg[word] + __popc(mask & ((1u << lane) - 1u));
            if (pos >= out.base && pos < out.end) {
                const int64_t q = pos - out.base;
                out.pairs[2 * q] = ch.s0 + a;
                out.pairs[2 * q + 1] = ch.s0 + b;
                out.r2[q] = r2;
            }
        }
    }
}

// One warp per row b: exclusive scan of the bit counts of its T words into seg, the row total into row_total[b] and onto
// *total.
__global__ void ld_row_scan_kernel(const uint32_t* __restrict__ bits, int32_t* __restrict__ seg,
                                   int32_t* __restrict__ row_total, unsigned long long* __restrict__ total, int row0,
                                   int rows, int T) {
    const int lane = threadIdx.x & 31;
    const int r = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (r >= rows) return;
    const int64_t b = row0 + r;
    int32_t carry = 0;
    for (int t0 = 0; t0 < T; t0 += 32) {
        const int t = t0 + lane;
        const int32_t v = t < T ? __popc(bits[b * T + t]) : 0;
        int32_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int32_t u = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += u;
        }
        if (t < T) seg[b * T + t] = carry + inc - v;
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) {
        row_total[b] = carry;
        if (carry > 0) atomicAdd(total, (unsigned long long)carry);
    }
}

// One warp.  kb holds the kept bits of the chunk rows (rows before own_lo from keep, as the previous chunk decided them);
// the owned rows are decided in order.  A row without an in-LD partner is kept outright; a row with partners is kept iff
// none of its in-LD bits meets a kept bit.  Bits of later rows never matter to a row's test (its bits only name a < b).
// The bit words of 32 rows are contiguous: they are staged in shared memory with one coalesced pass, so the serial
// per-row tests wait on shared memory only.  MASKED: an ineligible row has no pairs and is never kept.
template <bool MASKED>
__global__ void __launch_bounds__(32) ld_sweep_kernel(LdChunk ch, const uint32_t* __restrict__ bits,
                                                      const int32_t* __restrict__ row_total, uint8_t* __restrict__ keep) {
    __shared__ uint32_t kb[kLdMaxChunk / kTile];
    __shared__ uint32_t rb[kTile * (kLdMaxWindow / kTile + 1)];   // bit words of the current 32 rows
    const int lane = threadIdx.x;
    const int T = ch.T;
    for (int wi = 0; wi < ch.c / kTile; ++wi) {
        const int r = wi * kTile + lane;
        const uint32_t k = __ballot_sync(0xffffffffu, r < ch.own_lo && keep[ch.s0 + r] != 0);
        if (lane == 0) kb[wi] = k;
    }
    __syncwarp();
    for (int wi = ch.own_lo / kTile; wi * kTile < ch.nc; ++wi) {
        const int r = wi * kTile + lane;
        const bool owned = r >= ch.own_lo && r < ch.nc;
        const uint32_t om = __ballot_sync(0xffffffffu, owned);
        uint32_t todo = __ballot_sync(0xffffffffu, owned && row_total[r] != 0);
        const uint32_t em = MASKED ? __ballot_sync(0xffffffffu, owned && ch.elig[ch.s0 + r] != 0) : om;
        uint32_t word = kb[wi] | (em & ~todo);
        if (todo != 0u) {
            const uint32_t* src = bits + (int64_t)wi * kTile * T;
            for (int t = lane; t < kTile * T; t += 32) rb[t] = src[t];
            __syncwarp();
        }
        while (todo != 0u) {
            const int bit = __ffs(todo) - 1;
            todo &= todo - 1u;
            bool hit = false;
            for (int k = lane; k < T; k += 32) {
                const int at = wi - (T - 1) + k;
                if (at >= 0) hit |= (rb[bit * T + k] & (at == wi ? word : kb[at])) != 0u;
            }
            if (!__any_sync(0xffffffffu, hit)) word |= 1u << bit;
        }
        if (lane == 0) kb[wi] = word;
        __syncwarp();   // kb[wi] for the next rows, rb free for the next 32 rows
        if (owned) keep[ch.s0 + r] = (uint8_t)((word >> lane) & 1u);
    }
}

}  // namespace

cudaError_t ld_count(LdWork& w, const LdChunk& ch, cudaStream_t stream) {
    const int bt_lo = ch.own_lo / kTile, bt_hi = (ch.nc + kTile - 1) / kTile;
    if (bt_hi <= bt_lo) return cudaSuccess;
    PairOut none{};
    const dim3 grid((unsigned)ch.T, (unsigned)(bt_hi - bt_lo));
    if (ch.elig != nullptr)
        ld_pairs_kernel<false, true><<<grid, kTile * kWarps, 0, stream>>>(ch, bt_lo, w.d_bits.get(), nullptr, none);
    else
        ld_pairs_kernel<false, false><<<grid, kTile * kWarps, 0, stream>>>(ch, bt_lo, w.d_bits.get(), nullptr, none);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int rows = (bt_hi - bt_lo) * kTile, threads = 256;
    ld_row_scan_kernel<<<(unsigned)(((int64_t)rows * 32 + threads - 1) / threads), threads, 0, stream>>>(
        w.d_bits.get(), w.d_seg.get(), w.d_row_total.get(), reinterpret_cast<unsigned long long*>(w.d_total.get()), bt_lo * kTile, rows, ch.T);
    return cudaGetLastError();
}

cudaError_t ld_sweep(LdWork& w, const LdChunk& ch, uint8_t* d_keep, cudaStream_t stream) {
    if (ch.elig != nullptr)
        ld_sweep_kernel<true><<<1, 32, 0, stream>>>(ch, w.d_bits.get(), w.d_row_total.get(), d_keep);
    else
        ld_sweep_kernel<false><<<1, 32, 0, stream>>>(ch, w.d_bits.get(), w.d_row_total.get(), d_keep);
    return cudaGetLastError();
}

cudaError_t ld_emit(LdWork& w, const LdChunk& ch, int bt_lo, int bt_hi, int64_t base, int64_t end, cudaStream_t stream) {
    if (bt_hi <= bt_lo) return cudaSuccess;
    PairOut out{w.d_pairs.get(), w.d_r2.get(), w.d_row_start.get(), base, end};
    const dim3 grid((unsigned)ch.T, (unsigned)(bt_hi - bt_lo));
    if (ch.elig != nullptr)
        ld_pairs_kernel<true, true><<<grid, kTile * kWarps, 0, stream>>>(ch, bt_lo, w.d_bits.get(), w.d_seg.get(), out);
    else
        ld_pairs_kernel<true, false><<<grid, kTile * kWarps, 0, stream>>>(ch, bt_lo, w.d_bits.get(), w.d_seg.get(), out);
    return cudaGetLastError();
}

}  // namespace vpca
