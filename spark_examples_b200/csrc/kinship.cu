// KING-robust kinship (Manichaikul et al., Bioinformatics 26:2867, 2010; the between-family estimator) of every sample
// pair, read from the int32 Gram G = Y Y^T of the three indicator planes Y (encode_bed_planes: rows [0, n) het,
// [n, 2n) hom A1, [2n, 3n) hom A2).  For a pair a < b every count is a lower-triangle entry of G (DESIGN.md 7):
//   HETHET    = G[b][a]
//   IBS0      = G[2n+b][n+a] + G[2n+a][n+b]          (opposite homozygotes)
//   HET1_HOM2 = G[n+b][a]    + G[2n+b][a]            (a het, b hom)
//   HET2_HOM1 = G[n+a][b]    + G[2n+a][b]            (b het, a hom)
//   NSNP      = HETHET + IBS0 + HET1_HOM2 + HET2_HOM1 + G[n+b][n+a] + G[2n+b][2n+a]
//   KINSHIP   = (HETHET - 2 IBS0) / (2 HETHET + HET1_HOM2 + HET2_HOM1), NaN when the denominator is 0.
// A block takes a 32 x 32 tile of pairs (rows b, columns a); the three column reads (G[2n+a][n+b], G[n+a][b], G[2n+a][b])
// are staged through shared memory so that every global load runs along a row.  Selection is two passes without a sort:
// kin_count writes the selected pairs of every (row, tile) segment and scans them along the row; the host turns the row
// totals into row offsets; kin_emit recomputes the same pairs and writes each to its position (row-major lower-triangle
// order: by b, then a).  Integer counts, one double division per pair, no atomics: the output is bit-reproducible.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kTile = 32;
constexpr int kWarps = 8;

struct PairOut {
    int32_t* ids;
    int32_t* counts;
    double* kin;
    const int64_t* row_start;
    int64_t base, end;
};

// linear index of a lower-triangle tile (at <= bt) -> (bt, at)
__device__ __forceinline__ void tile_of(int64_t i, int* bt, int* at) {
    int t = (int)((sqrt(8.0 * (double)i + 1.0) - 1.0) * 0.5);
    while ((int64_t)t * (t + 1) / 2 > i) --t;
    while ((int64_t)(t + 1) * (t + 2) / 2 <= i) ++t;
    *bt = t;
    *at = (int)(i - (int64_t)t * (t + 1) / 2);
}

template <bool EMIT>
__global__ void __launch_bounds__(kTile * kWarps)
kin_pairs_kernel(const int32_t* __restrict__ G, int n, int tiles, int64_t tile0, double thr, int select_all,
                 int32_t* __restrict__ seg, PairOut out) {
    __shared__ int32_t t_ibs0[kTile][kTile + 1];   // [al][bl] = G[2n+a][n+b]
    __shared__ int32_t t_het2[kTile][kTile + 1];   // [al][bl] = G[n+a][b] + G[2n+a][b]
    int bt, at;
    tile_of(tile0 + blockIdx.x, &bt, &at);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t R = 3 * (int64_t)n;
    const int a0 = at * kTile, b0 = bt * kTile;
    {   // column reads, coalesced along b
        const int b = b0 + lane;
        for (int al = warp; al < kTile; al += kWarps) {
            const int a = a0 + al;
            int32_t v1 = 0, v2 = 0;
            if (a < n && b < n) {
                v1 = G[(2 * (int64_t)n + a) * R + n + b];
                v2 = G[((int64_t)n + a) * R + b] + G[(2 * (int64_t)n + a) * R + b];
            }
            t_ibs0[al][lane] = v1;
            t_het2[al][lane] = v2;
        }
    }
    __syncthreads();
    const int a = a0 + lane;
    for (int bl = warp; bl < kTile; bl += kWarps) {
        const int b = b0 + bl;
        if (b >= n) break;   // warp-uniform
        const bool valid = a < b;
        int64_t hethet = 0, ibs0 = 0, het1 = 0, het2 = 0, nsnp = 0;
        double kin = 0.0;
        bool sel = false;
        if (valid) {
            const int32_t* rb = G + (int64_t)b * R;
            const int32_t* r1 = G + ((int64_t)n + b) * R;
            const int32_t* r2 = G + (2 * (int64_t)n + b) * R;
            hethet = rb[a];
            ibs0 = (int64_t)r2[n + a] + t_ibs0[lane][bl];
            het1 = (int64_t)r1[a] + r2[a];
            het2 = t_het2[lane][bl];
            nsnp = hethet + ibs0 + het1 + het2 + r1[n + a] + r2[2 * (int64_t)n + a];
            const int64_t num = hethet - 2 * ibs0, den = 2 * hethet + het1 + het2;
            kin = den == 0 ? __longlong_as_double(0x7ff8000000000000ll) : (double)num / (double)den;
            sel = select_all != 0 || kin >= thr;
        }
        const uint32_t mask = __ballot_sync(0xffffffffu, sel);
        int32_t* sp = seg + (int64_t)b * tiles + at;
        if (!EMIT) {
            if (lane == 0) *sp = __popc(mask);
        } else if (sel) {
            const int64_t pos = out.row_start[b] + *sp + __popc(mask & ((1u << lane) - 1u));
            if (pos >= out.base && pos < out.end) {
                const int64_t q = pos - out.base;
                out.ids[2 * q] = a;
                out.ids[2 * q + 1] = b;
                int32_t* c = out.counts + 5 * q;
                c[0] = (int32_t)nsnp;
                c[1] = (int32_t)hethet;
                c[2] = (int32_t)ibs0;
                c[3] = (int32_t)het1;
                c[4] = (int32_t)het2;
                out.kin[q] = kin;
            }
        }
    }
}

// One warp per row b: exclusive scan of its segment counts (tiles 0 .. b / 32) in place, the row total into row_total[b].
__global__ void kin_row_scan_kernel(int32_t* __restrict__ seg, int32_t* __restrict__ row_total, int n, int tiles) {
    const int lane = threadIdx.x & 31;
    const int b = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (b >= n) return;
    int32_t* s = seg + (int64_t)b * tiles;
    const int nseg = b / kTile + 1;
    int32_t carry = 0;
    for (int t0 = 0; t0 < nseg; t0 += 32) {
        const int t = t0 + lane;
        const int32_t v = t < nseg ? s[t] : 0;
        int32_t inc = v;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int32_t u = __shfl_up_sync(0xffffffffu, inc, d);
            if (lane >= d) inc += u;
        }
        if (t < nseg) s[t] = carry + inc - v;
        carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (lane == 0) row_total[b] = carry;
}

}  // namespace

cudaError_t kin_pair_alloc(KinPairWork& w, int n) {
    if (w.n == n) return cudaSuccess;
    w = KinPairWork{};   // a new sample count: every buffer is allocated afresh
    const int tiles = (n + kTile - 1) / kTile;
    // a tile row (32 rows b) holds fewer than 32 n pairs: one always fits the scratch
    const int64_t cap = std::max<int64_t>(int64_t(1) << 21, (int64_t)kTile * n);
    cudaError_t e = w.d_seg.ensure((int64_t)n * tiles);
    if (e == cudaSuccess) e = w.d_row_total.ensure(n);
    if (e == cudaSuccess) e = w.d_row_start.ensure(n);
    if (e == cudaSuccess) e = w.d_ids.ensure(cap * 2);
    if (e == cudaSuccess) e = w.d_counts.ensure(cap * 5);
    if (e == cudaSuccess) e = w.d_kin.ensure(cap);
    if (e == cudaSuccess) w.n = n;
    return e;
}

cudaError_t kin_count(KinPairWork& w, const int32_t* d_G, int n, double min_kinship, bool select_all, cudaStream_t stream) {
    const int tiles = (n + kTile - 1) / kTile;
    const int64_t num_tiles = (int64_t)tiles * (tiles + 1) / 2;
    PairOut none{};
    kin_pairs_kernel<false><<<(unsigned)num_tiles, kTile * kWarps, 0, stream>>>(d_G, n, tiles, 0, min_kinship,
                                                                               select_all ? 1 : 0, w.d_seg.get(), none);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    const int threads = 256;
    kin_row_scan_kernel<<<(unsigned)(((int64_t)n * 32 + threads - 1) / threads), threads, 0, stream>>>(w.d_seg.get(), w.d_row_total.get(),
                                                                                                      n, tiles);
    return cudaGetLastError();
}

cudaError_t kin_emit(KinPairWork& w, const int32_t* d_G, int n, double min_kinship, bool select_all, int bt_lo, int bt_hi,
                     int64_t base, int64_t end, cudaStream_t stream) {
    const int tiles = (n + kTile - 1) / kTile;
    const int64_t t0 = (int64_t)bt_lo * (bt_lo + 1) / 2, t1 = (int64_t)bt_hi * (bt_hi + 1) / 2;
    if (t1 <= t0) return cudaSuccess;
    PairOut out{w.d_ids.get(), w.d_counts.get(), w.d_kin.get(), w.d_row_start.get(), base, end};
    kin_pairs_kernel<true><<<(unsigned)(t1 - t0), kTile * kWarps, 0, stream>>>(d_G, n, tiles, t0, min_kinship,
                                                                              select_all ? 1 : 0, w.d_seg.get(), out);
    return cudaGetLastError();
}

}  // namespace vpca
