// Multi-dataset keying on the device: variant keys, the 2-way join and the N-way merge that feed the encoder.
//
// Replaces (reference: src/main/scala/com/google/cloud/genomics/spark/examples/VariantsPca.scala)
//   :62-78    getVariantKey: Guava Hashing.murmur3_128() over contig, start, end, reference bases, alternate bases;
//   :115-128  joinDatasets: keyBy(getVariantKey) on both sides, RDD.join, calls of the two sides concatenated;
//   :136-148  mergeDatasets: union, groupByKey, keep the keys seen exactly variantSetCount times, calls flattened.
// The reference shuffles (key, Seq[CallData]) records between executors; here the rows of all datasets sit in one CSR
// (offsets + sample indices, rows of dataset 0 first) next to their key bytes, and
//   1. one thread per row hashes the key bytes (MurmurHash3_x64_128, seed 0: the published algorithm Guava implements;
//      Guava is an un-vendored dependency, shaded at build.sbt:44 -- pinned by the KATs in tests/test_host.py);
//   2. every row is inserted into an open-addressing table (linear probing, load <= 1/2) keyed by h1;
//   3. every row walks its probe cluster once and finds the rows with the same 128-bit key: its group size, the group's
//      first row (leader) and the calls that precede it inside the group (merge), or its partners on the right (join);
//   4. two exclusive scans turn per-row output sizes into CSR offsets, and one warp per output row copies the calls.
// The output CSR stays on the device: vpca_accumulate_joined hands it to encode_calls -> Gram without a host round trip.
// Everything is integer work with a fixed output order (merge: groups by first row, members in row order; join: by
// left row, then right row), so the joined rows are reproducible and equal to the host implementation's.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

__device__ __forceinline__ uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }

__device__ __forceinline__ uint64_t fmix64(uint64_t k) {
    k ^= k >> 33;
    k *= 0xFF51AFD7ED558CCDull;
    k ^= k >> 33;
    k *= 0xC4CEB9FE1A85EC53ull;
    k ^= k >> 33;
    return k;
}

__device__ __forceinline__ uint64_t load_le(const uint8_t* p, int nbytes) {   // nbytes <= 8, unaligned
    uint64_t v = 0;
    for (int b = 0; b < nbytes; ++b) v |= (uint64_t)p[b] << (8 * b);
    return v;
}

// MurmurHash3_x64_128 (Austin Appleby, public domain), seed 0; out = (h1, h2): the little-endian halves of Guava's
// HashCode.asBytes().
__global__ void hash_keys_kernel(const uint8_t* __restrict__ payload, const int64_t* __restrict__ off, int64_t nkeys,
                                 uint64_t* __restrict__ out) {
    const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nkeys) return;
    const uint8_t* data = payload + off[q];
    const int64_t len = off[q + 1] - off[q];
    const uint64_t c1 = 0x87C37B91114253D5ull, c2 = 0x4CF5AD432745937Full;
    uint64_t h1 = 0, h2 = 0;
    const int64_t nblocks = len / 16;
    for (int64_t i = 0; i < nblocks; ++i) {
        uint64_t k1 = load_le(data + i * 16, 8), k2 = load_le(data + i * 16 + 8, 8);
        k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
        h1 = rotl64(h1, 27); h1 += h2; h1 = h1 * 5 + 0x52DCE729ull;
        k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
        h2 = rotl64(h2, 31); h2 += h1; h2 = h2 * 5 + 0x38495AB5ull;
    }
    const uint8_t* tail = data + nblocks * 16;
    const int t = (int)(len & 15);
    if (t > 8) {
        uint64_t k2 = load_le(tail + 8, t - 8);
        k2 *= c2; k2 = rotl64(k2, 33); k2 *= c1; h2 ^= k2;
    }
    if (t > 0) {
        uint64_t k1 = load_le(tail, t > 8 ? 8 : t);
        k1 *= c1; k1 = rotl64(k1, 31); k1 *= c2; h1 ^= k1;
    }
    h1 ^= (uint64_t)len; h2 ^= (uint64_t)len;
    h1 += h2; h2 += h1;
    h1 = fmix64(h1); h2 = fmix64(h2);
    h1 += h2; h2 += h1;
    out[2 * q] = h1;
    out[2 * q + 1] = h2;
}

__global__ void fill_i32_kernel(int32_t* __restrict__ p, int64_t count, int32_t v) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) p[i] = v;
}

__global__ void insert_kernel(const uint64_t* __restrict__ h, int64_t nrows, int32_t* __restrict__ table, uint32_t mask) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows) return;
    uint32_t slot = (uint32_t)h[2 * i] & mask;
    while (atomicCAS(&table[slot], -1, (int32_t)i) != -1) slot = (slot + 1) & mask;
}

// One thread per row: walk the probe cluster from the row's home slot to the first empty slot; every row with the same
// 128-bit key is in there (linear probing never skips an empty slot on insertion, and nothing is ever deleted).
//   merge: rows_out[i] = 1 for the first row of a group of exactly `vsc` rows, len_out[i] = calls of the whole group;
//          leader[i] = first row of i's group or -1 if the group is dropped; prefix[i] = calls of the members before i.
//   join : for a left row, rows_out[i] = number of right rows with its key, len_out[i] = calls of all its output rows.
__global__ void analyze_kernel(const uint64_t* __restrict__ h, const int64_t* __restrict__ off, int64_t nrows, int64_t n_left,
                               int mode, int vsc, const int32_t* __restrict__ table, uint32_t mask,
                               int64_t* __restrict__ rows_out, int64_t* __restrict__ len_out, int32_t* __restrict__ leader,
                               int64_t* __restrict__ prefix) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nrows) return;
    const uint64_t k1 = h[2 * i], k2 = h[2 * i + 1];
    const int64_t my_len = off[i + 1] - off[i];
    uint32_t slot = (uint32_t)k1 & mask;
    int64_t cnt = 0, total = 0, before = 0;
    int32_t first = (int32_t)i;
    if (mode == VPCA_JOIN && i >= n_left) {   // right rows produce nothing themselves
        rows_out[i] = 0;
        len_out[i] = 0;
        leader[i] = -1;
        prefix[i] = 0;
        return;
    }
    while (true) {
        const int32_t e = table[slot];
        if (e < 0) break;
        if (h[2 * (int64_t)e] == k1 && h[2 * (int64_t)e + 1] == k2) {
            const int64_t elen = off[e + 1] - off[e];
            if (mode == VPCA_MERGE) {
                ++cnt;
                total += elen;
                if (e < i) before += elen;
                if (e < first) first = e;
            } else if (e >= n_left) {
                ++cnt;
                total += my_len + elen;
            }
        }
        slot = (slot + 1) & mask;
    }
    if (mode == VPCA_MERGE) {
        const bool kept = cnt == vsc;
        rows_out[i] = (kept && first == (int32_t)i) ? 1 : 0;
        len_out[i] = (kept && first == (int32_t)i) ? total : 0;
        leader[i] = kept ? first : -1;
        prefix[i] = before;
    } else {
        rows_out[i] = cnt;
        len_out[i] = total;
        leader[i] = (int32_t)i;
        prefix[i] = 0;
    }
}

// ---- exclusive scan of int64 (three kernels: block totals, scan of the totals by one block, block scans + base) ----
constexpr int kScanBlock = 1024;

__device__ __forceinline__ int64_t block_exclusive_scan(int64_t v, int64_t* sh, int64_t* total) {
    // sh: >= 33 int64
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int64_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) sh[wid] = x;
    __syncthreads();
    if (wid == 0) {
        int64_t s = sh[lane];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int64_t y = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += y;
        }
        sh[lane] = s;   // inclusive scan of the warp totals
    }
    __syncthreads();
    const int64_t base = wid > 0 ? sh[wid - 1] : 0;
    if (total != nullptr) *total = sh[31];
    __syncthreads();
    return base + x - v;
}

__global__ void __launch_bounds__(kScanBlock) scan_totals_kernel(const int64_t* __restrict__ in, int64_t count,
                                                                 int64_t* __restrict__ block_tot) {
    __shared__ int64_t sh[33];
    const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
    int64_t tot;
    block_exclusive_scan(i < count ? in[i] : 0, sh, &tot);
    if (threadIdx.x == 0) block_tot[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(kScanBlock) scan_blocks_kernel(int64_t* __restrict__ block_tot, int64_t nblocks,
                                                                 int64_t* __restrict__ grand) {
    __shared__ int64_t sh[33];
    __shared__ int64_t carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t b0 = 0; b0 < nblocks; b0 += kScanBlock) {
        const int64_t i = b0 + threadIdx.x;
        const int64_t v = i < nblocks ? block_tot[i] : 0;
        int64_t tot;
        const int64_t ex = block_exclusive_scan(v, sh, &tot);
        if (i < nblocks) block_tot[i] = carry + ex;
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) *grand = carry;
}

__global__ void __launch_bounds__(kScanBlock) scan_apply_kernel(const int64_t* __restrict__ in, int64_t count,
                                                                const int64_t* __restrict__ block_base,
                                                                int64_t* __restrict__ out) {
    __shared__ int64_t sh[33];
    const int64_t i = (int64_t)blockIdx.x * kScanBlock + threadIdx.x;
    const int64_t ex = block_exclusive_scan(i < count ? in[i] : 0, sh, nullptr);
    if (i < count) out[i] = block_base[blockIdx.x] + ex;
}

cudaError_t exclusive_scan(const int64_t* in, int64_t count, int64_t* out, int64_t* block_tmp, int64_t* grand,
                           cudaStream_t stream) {
    const int64_t nblocks = (count + kScanBlock - 1) / kScanBlock;
    scan_totals_kernel<<<(unsigned)nblocks, kScanBlock, 0, stream>>>(in, count, block_tmp);
    scan_blocks_kernel<<<1, kScanBlock, 0, stream>>>(block_tmp, nblocks, grand);
    scan_apply_kernel<<<(unsigned)nblocks, kScanBlock, 0, stream>>>(in, count, block_tmp, out);
    return cudaGetLastError();
}

// One warp per input row.
//   merge: a member of a kept group copies its calls to (CSR offset of the group's row) + (calls of the members before
//          it); the leader also writes the row's offset.
//   join : left row i writes one output row per right partner, partners in ascending row order.
__global__ void __launch_bounds__(256) emit_kernel(const uint64_t* __restrict__ h, const int64_t* __restrict__ off,
                                                   const int32_t* __restrict__ idx, int64_t nrows, int64_t n_left, int mode,
                                                   const int32_t* __restrict__ table, uint32_t mask,
                                                   const int64_t* __restrict__ row_base, const int64_t* __restrict__ nnz_base,
                                                   const int32_t* __restrict__ leader, const int64_t* __restrict__ prefix,
                                                   int64_t* __restrict__ out_off, int32_t* __restrict__ out_idx) {
    const int64_t i = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (i >= nrows) return;
    const int32_t L = leader[i];
    if (L < 0) return;
    const int64_t src = off[i], len = off[i + 1] - off[i];
    if (mode == VPCA_MERGE) {
        const int64_t dst = nnz_base[L] + prefix[i];
        for (int64_t c = lane; c < len; c += 32) out_idx[dst + c] = idx[src + c];
        if (L == (int32_t)i && lane == 0) out_off[row_base[i]] = nnz_base[i];
        return;
    }
    // join: partners in ascending row order -- repeatedly take the smallest partner above the last one written
    const uint64_t k1 = h[2 * i], k2 = h[2 * i + 1];
    int64_t row = row_base[i], dst = nnz_base[i];
    int32_t last = -1;
    while (true) {
        int32_t next = 0x7fffffff;
        uint32_t slot = (uint32_t)k1 & mask;
        while (true) {
            const int32_t e = table[slot];
            if (e < 0) break;
            if (e >= n_left && e > last && e < next && h[2 * (int64_t)e] == k1 && h[2 * (int64_t)e + 1] == k2) next = e;
            slot = (slot + 1) & mask;
        }
        if (next == 0x7fffffff) break;
        const int64_t rsrc = off[next], rlen = off[next + 1] - off[next];
        if (lane == 0) out_off[row] = dst;
        for (int64_t c = lane; c < len; c += 32) out_idx[dst + c] = idx[src + c];          // related._1 ++ related._2 (:127)
        for (int64_t c = lane; c < rlen; c += 32) out_idx[dst + len + c] = idx[rsrc + c];
        dst += len + rlen;
        ++row;
        last = next;
    }
}

__global__ void set_i64_kernel(int64_t* __restrict__ p, const int64_t* __restrict__ rows, const int64_t* __restrict__ v) {
    p[*rows] = *v;   // out_off[nrows_out] = nnz_out
}

}  // namespace

cudaError_t hash_keys(const uint8_t* d_payload, const int64_t* d_off, int64_t nkeys, uint64_t* d_hash, cudaStream_t stream) {
    if (nkeys <= 0) return cudaSuccess;
    hash_keys_kernel<<<(unsigned)((nkeys + 255) / 256), 256, 0, stream>>>(d_payload, d_off, nkeys, d_hash);
    return cudaGetLastError();
}

void join_free(JoinWork& w) {
    if (w.h_totals) cudaFreeHost(w.h_totals);
    w = JoinWork{};
}

// Sizes the per-row workspace for `nrows` rows (grow-only).  d_rows is emptied first and grows last, so its capacity is
// the rows every buffer holds: after a failed call it is 0 and the next call reserves again.
static cudaError_t join_reserve(JoinWork& w, int64_t nrows) {
    if (nrows <= w.d_rows.capacity()) return cudaSuccess;
    const int64_t cap = with_slack(nrows);
    uint64_t slots = 1024;
    while (slots < 2 * (uint64_t)cap) slots <<= 1;
    w.d_rows.reset();
    w.d_table.reset();   // the table and the scan scratch are sized for `cap` rows: reallocated whenever the rows grow
    w.d_block.reset();
    cudaError_t e;
#define VPCA_TRY(x) if ((e = (x)) != cudaSuccess) return e
    VPCA_TRY(w.d_hash.ensure(2 * nrows, 2 * cap));
    VPCA_TRY(w.d_table.ensure((int64_t)slots));
    w.table_slots = slots;
    VPCA_TRY(w.d_len.ensure(nrows, cap));
    VPCA_TRY(w.d_row_base.ensure(nrows, cap));
    VPCA_TRY(w.d_nnz_base.ensure(nrows, cap));
    VPCA_TRY(w.d_leader.ensure(nrows, cap));
    VPCA_TRY(w.d_prefix.ensure(nrows, cap));
    VPCA_TRY(w.d_block.ensure((cap + kScanBlock - 1) / kScanBlock + 1));
    VPCA_TRY(w.d_totals.ensure(2));
    if (w.h_totals == nullptr) VPCA_TRY(cudaHostAlloc(&w.h_totals, 2 * sizeof(int64_t), cudaHostAllocPortable));
    VPCA_TRY(w.d_rows.ensure(nrows, cap));
#undef VPCA_TRY
    return cudaSuccess;
}

// Keys + CSR on the device -> joined / merged CSR on the device (w.d_out_off: out_rows + 1 offsets, w.d_out_idx).
// Synchronises the stream once (the output sizes decide the output allocation).
cudaError_t join_rows(JoinWork& w, int mode, int variant_set_count, int64_t n_left, const uint8_t* d_payload,
                      const int64_t* d_key_off, const int64_t* d_off, const int32_t* d_idx, int64_t nrows, cudaStream_t stream,
                      int64_t* out_rows, int64_t* out_nnz, int64_t* launches) {
    *out_rows = 0;
    *out_nnz = 0;
    cudaError_t e = join_reserve(w, nrows > 0 ? nrows : 1);
    if (e != cudaSuccess) return e;
    if (nrows > 0) {
        const unsigned gb = (unsigned)((nrows + 255) / 256);
        const uint32_t mask = (uint32_t)(w.table_slots - 1);
        hash_keys_kernel<<<gb, 256, 0, stream>>>(d_payload, d_key_off, nrows, w.d_hash.get());
        fill_i32_kernel<<<1184, 256, 0, stream>>>(w.d_table.get(), (int64_t)w.table_slots, -1);
        insert_kernel<<<gb, 256, 0, stream>>>(w.d_hash.get(), nrows, w.d_table.get(), mask);
        analyze_kernel<<<gb, 256, 0, stream>>>(w.d_hash.get(), d_off, nrows, n_left, mode, variant_set_count, w.d_table.get(), mask, w.d_rows.get(),
                                               w.d_len.get(), w.d_leader.get(), w.d_prefix.get());
        if ((e = exclusive_scan(w.d_rows.get(), nrows, w.d_row_base.get(), w.d_block.get(), w.d_totals.get(), stream)) != cudaSuccess) return e;
        if ((e = exclusive_scan(w.d_len.get(), nrows, w.d_nnz_base.get(), w.d_block.get(), w.d_totals.get() + 1, stream)) != cudaSuccess) return e;
        if (launches) *launches += 4 + 6;
        if ((e = cudaMemcpyAsync(w.h_totals, w.d_totals.get(), 2 * sizeof(int64_t), cudaMemcpyDeviceToHost, stream)) != cudaSuccess) return e;
        if ((e = cudaStreamSynchronize(stream)) != cudaSuccess) return e;
        *out_rows = w.h_totals[0];
        *out_nnz = w.h_totals[1];
    }
    if ((e = w.d_out_off.ensure(*out_rows + 1, with_slack(*out_rows))) != cudaSuccess) return e;
    // never left null, even after a join without calls
    if ((e = w.d_out_idx.ensure(std::max<int64_t>(*out_nnz, 1), with_slack(*out_nnz))) != cudaSuccess) return e;
    if (nrows > 0) {
        const uint32_t mask = (uint32_t)(w.table_slots - 1);
        emit_kernel<<<(unsigned)((nrows + 7) / 8), 256, 0, stream>>>(w.d_hash.get(), d_off, d_idx, nrows, n_left, mode, w.d_table.get(), mask,
                                                                      w.d_row_base.get(), w.d_nnz_base.get(), w.d_leader.get(), w.d_prefix.get(),
                                                                      w.d_out_off.get(), w.d_out_idx.get());
        set_i64_kernel<<<1, 1, 0, stream>>>(w.d_out_off.get(), w.d_totals.get(), w.d_totals.get() + 1);
        if (launches) *launches += 2;
    } else {
        if ((e = cudaMemsetAsync(w.d_out_off.get(), 0, 8, stream)) != cudaSuccess) return e;
    }
    return cudaGetLastError();
}

}  // namespace vpca
