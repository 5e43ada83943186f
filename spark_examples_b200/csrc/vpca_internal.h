// Internal declarations shared by the libvpca translation units (not part of the ABI).
#pragma once
#include <algorithm>
#include <atomic>
#include <cstdint>
#include <cuda_runtime.h>
#include <string>
#include <vector>

#include "../../include/vpca.h"

namespace vpca {

// ---- device memory -----------------------------------------------------------------------------------------------------
// Device bytes held by every DeviceBuffer of the process (vpca_debug_device_bytes).
inline std::atomic<int64_t> g_device_bytes{0};

// Owner of one cudaMalloc allocation of `capacity()` elements, freed on destruction, reset() or when it grows.  There is no
// conversion to T*: a pointer leaves the buffer through get() only, so no caller can free or replace the allocation.
// Frees run on whatever device is current; an owner whose buffers live on another device selects it first.
template <class T>
class DeviceBuffer {
public:
    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    DeviceBuffer(DeviceBuffer&& o) noexcept : p_(o.p_), cap_(o.cap_) {
        o.p_ = nullptr;
        o.cap_ = 0;
    }
    DeviceBuffer& operator=(DeviceBuffer&& o) noexcept {
        if (this != &o) {
            reset();
            p_ = o.p_;
            cap_ = o.cap_;
            o.p_ = nullptr;
            o.cap_ = 0;
        }
        return *this;
    }
    ~DeviceBuffer() { reset(); }

    // Grow-only: nothing happens while count <= capacity(); otherwise the old allocation is freed (its contents are not
    // kept) and max(count, alloc) elements are allocated.  On failure the buffer is empty.
    cudaError_t ensure(int64_t count, int64_t alloc) {
        if (count <= cap_) return cudaSuccess;
        reset();
        alloc = std::max(alloc, count);
        void* p = nullptr;
        const cudaError_t e = cudaMalloc(&p, (size_t)alloc * sizeof(T));
        if (e != cudaSuccess) return e;
        p_ = static_cast<T*>(p);
        cap_ = alloc;
        g_device_bytes += alloc * (int64_t)sizeof(T);
        return cudaSuccess;
    }
    cudaError_t ensure(int64_t count) { return ensure(count, count); }
    void reset() {
        if (p_ == nullptr) return;
        cudaFree(p_);
        g_device_bytes -= cap_ * (int64_t)sizeof(T);
        p_ = nullptr;
        cap_ = 0;
    }
    T* get() const { return p_; }
    int64_t capacity() const { return cap_; }

private:
    T* p_ = nullptr;
    int64_t cap_ = 0;
};

// Allocation size of the buffers that grow with headroom, so that slowly growing inputs do not reallocate on every call.
inline int64_t with_slack(int64_t n) { return n + n / 4 + 1024; }

// ---- Gram (gram_sm90.cu) --------------------------------------------------------------------
struct GramPlan {
    int cta_group = 2;        // CTAs per tile (1: 128 x 256 tiles per CTA; 2: 256 x 256 per CTA pair, one A block each,
                              // the pair launched as a 2-CTA cluster that fetches the B rows once and multicasts them)
    int kb_window = 0;        // k-blocks per L2 window (0 -> automatic)
    int num_sms = 0;
    int max_pairs[3] = {};    // 2-CTA clusters of the int8 / bf16 / e2m1 kernel the device holds at once (0: not queried)
    DeviceBuffer<uint8_t> d_tiles;   // device tile list (TileDesc, gram_sm90.cu)
    std::vector<int32_t> h_tiles;   // the same list on the host (8 ints per tile): resident / accumulator-fit decisions
    int num_tiles = 0;
    int num_full = 0;         // leading full-weight tiles (whole-tile waves of the large-N schedule)
    int total_weight = 0;     // sum over tiles of n_eff / 16
    int tiles_col_limit = 256;   // accumulator columns (B rows) one worker may hold
    bool exact_cover = false; // VPCA_EXACT_COVER=1: the exact 128-block cover of the lower triangle (4.5 % fewer MMAs at
                              // 2504 samples) instead of square 256 x 256 tiles.  Off by default: a one-row tile (128 B rows)
                              // still takes a worker's whole 256-row accumulator, and with one accumulator per worker its
                              // unequal tiles split less evenly (2504 samples, 66 workers: the busiest worker gets 1.30 x the
                              // mean share against 1.24 x for the rectangles)
    int tiles_for_n = -1;     // n_samples the tile list was built for
    int tiles_for_cg = 0;
    int tiles_for_bn = 0;
    int tiles_row_lo = 0, tiles_row_hi = 0;   // rows of S the tile list covers
    int own_lo = 0, own_hi = 0;   // band-only context: the rows of S it stores (own_hi == 0: the whole matrix); without
                                  // peers the Gram kernel then computes exactly those rows (owner-computes)
    int last_resident = 0;
    int* d_err = nullptr;     // device debug words written before a watchdog trap
    static constexpr int kMaxWindows = 1 << 16;
    int sync_lead = 0;        // VPCA_SYNC_LEAD: windows a worker may lead the slowest one by (0 = no pacing)
    DeviceBuffer<int> d_win_done;
    bool self_b = true;       // VPCA_SELF_B=0: diagonal tiles load their B rows although they are the pair's own A blocks
    bool red64 = true;        // VPCA_RED64=0: one 32-bit red per cell in the flush instead of two cells per 64-bit red
    double gain = 0.5;        // VPCA_REBALANCE_GAIN: how far a launch moves the shares towards the measured speeds
    bool adaptive = true;     // VPCA_ADAPTIVE=0 keeps the stream-K split equal instead of speed-weighted
    DeviceBuffer<uint8_t> d_cum;   // cumulative worker shares (workers + 1 doubles), front/tail split point (a double), update
                                   // counter (an int)
    int cum_workers = 0, cum_tiles = 0, cum_kbw = 0, cum_for_n = 0, cum_dev = 0, cum_elem = 0;   // what the split in d_cum was made for
    // fused multi-GPU reduction: Gram buffers / barrier flags of all ranks, peer-mapped through CUDA IPC
    int num_peers = 0, peer_rank = 0, peer_epoch = 0;
    int32_t* peer_S[16] = {};     // Gram of rank d as seen from this device: the address of row 0 (for a rank that stores
                                  // only a row band this is a VIRTUAL origin, valid for the rows of the band only)
    int32_t* peer_base[16] = {};  // start of rank d's allocation (what an IPC mapping must be closed with)
    int32_t* peer_flags[16] = {};
    int band_row0[16] = {}, band_rows[16] = {};   // rows rank d stores (band_rows 0 or n: all of them)
    bool peers_ipc = false;       // peer mappings came from cudaIpcOpenMemHandle (other processes), not from peer access
    int peer_mode = 0;        // 0: every flush goes to all ranks' Grams; 1: to the owner of the row only (+ gather)
    int own_end[16] = {};     // peer_mode 1: rank q owns Gram rows [own_end[q-1], own_end[q])
    bool profile = false;     // VPCA_GRAM_PROF=1: per-CTA timestamps in d_prof
    DeviceBuffer<long long> d_prof;
};
// Copies the per-CTA timestamps of the last profiled launch (4 per CTA) to host; returns the CTA count.
int gram_read_profile(GramPlan& plan, long long* out, int max_ctas);

// S(lower triangle, row >= col) += X X^T for the nv variants of a dense sample-major tile.
//   d_x : device, element (s, v) at index s * ld + v; elem_bits 8 (int8), 16 (bf16) or 4 (packed e2m1: two cells per
//         byte, ld % 128 == 0 and zero cells up to the next multiple of 128 variants)
//   d_S : device int32 n x n row-major
// Returns cudaSuccess or the first CUDA error; never synchronises.
// panel > 0: the tile is stored as ceil(nv / panel) consecutive panels of `panel` variants, each panel n rows of
// `panel` cells (cell (s, v) at (v / panel) * n * panel + s * panel + v % panel, zero cells after nv in the last
// panel); `ld` is ignored.  Keeps the pages touched per L2 window few (a row-major tile with a multi-MB pitch puts
// every sample row on its own 2 MB page and thrashes the TLBs).
cudaError_t gram_accumulate(GramPlan& plan, const void* d_x, int elem_bits, int n, int64_t nv, int64_t ld, int64_t panel,
                            int32_t* d_S, cudaStream_t stream, std::string* err);
cudaError_t gram_symmetrize(int32_t* d_S, int n, cudaStream_t stream);
cudaError_t gram_add(int32_t* d_dst, const int32_t* d_src, int64_t count, cudaStream_t stream);
cudaError_t gram_add_peers(GramPlan& plan, const int32_t* d_src, int64_t count, cudaStream_t stream);
cudaError_t gram_add_owners(GramPlan& plan, const int32_t* d_src, int n, cudaStream_t stream);
cudaError_t gram_gather_rows(GramPlan& plan, int32_t* d_S, int n, cudaStream_t stream);
cudaError_t gram_peer_barrier(GramPlan& plan, cudaStream_t stream);
cudaError_t gram_preload_kernels(cudaStream_t stream);   // see gram_sm90.cu: lazy module loading vs spinning barriers
cudaError_t encode_preload_kernels();
void gram_plan_free(GramPlan& plan);
int gram_debug_max_clusters(int cluster_size);
int gram_debug_band_tiles(int n, int cta_group, int row_lo, int row_hi, int32_t* out, int max_tiles);
int gram_debug_tiles(int n, int cta_group, int exact, int32_t* out, int max_tiles);
int gram_debug_plan(const int32_t* tiles8, int num_tiles, int workers, int kbw, int32_t* out, int max_pieces);
int gram_debug_schedule(int n, int cta_group, int exact, int workers, int kbw, int kb_total, double frac, int32_t* out,
                        int max_pieces, int32_t* info);
int gram_debug_repair(const int32_t* tiles8, int num_tiles, int workers, int kbw, int col_limit, double* cum, int32_t* out,
                      int max_pieces);

// ---- encode (encode.cu) ------------------------------------------------------------------------
// CSR rows [0, nv) (d_off has nv+1 entries; entry e of row v is d_idx[d_off[v] - base + ...]) -> dense
// sample-major tile, zero-filled first.  d_flags[0] is OR-ed with 1 on an out-of-range index and 2 on a
// multiplicity overflow.
cudaError_t encode_calls(const int64_t* d_off, int64_t base, const void* d_idx, int idx_bytes, int64_t nv, int n,
                         int elem_bits, int max_mult, void* d_x, int64_t ld, int64_t panel, int* d_flags,
                         cudaStream_t stream);   // idx_bytes: 4 (int32) or 2 (uint16)

// Packed rows (`stride` bytes apart) -> dense cells (binary carriers).  code 0: one N-bit bitmap per variant, LSB
// first; code 1 / 2: PLINK .bed rows (2 bits per sample), carriers of A1 / of A2.
cudaError_t encode_bits(const uint8_t* d_bits, int64_t stride, int64_t nv, int n, int elem_bits, void* d_x, int64_t ld,
                        int64_t panel, int code, cudaStream_t stream);

// PLINK .bed rows (`stride` bytes apart) -> the three int8 kinship planes in panel layout over 3n rows: row s het, row
// n + s hom A1, row 2n + s hom A2 (missing calls and padding samples set nothing).  Zeroes a partial last panel first.
cudaError_t encode_bed_planes(const uint8_t* d_rows, int64_t stride, int64_t nv, int n, void* d_x, int64_t panel,
                              cudaStream_t stream);

// PLINK .bed rows -> the three int8 LD planes of a chunk of c variants (DESIGN.md 9) over samples [s0, s0 + len), panel
// layout over 3c rows: row v the A1 count D, row c + v D^2, row 2c + v 1 if called (missing calls 0 in all three).  Row v of
// the input is `pitch` bytes at d_rows + v * pitch holding samples s0 .. (its first `width` bytes are meaningful); rows
// v >= nv and samples >= n are written as zero, and so is every cell up to the end of the last panel.
cudaError_t encode_ld_planes(const uint8_t* d_rows, int64_t pitch, int64_t width, int nv, int c, int64_t s0, int64_t len,
                             int n, void* d_x, int64_t panel, cudaStream_t stream);

// ---- LD pruning from the 3c x 3c plane Gram of a chunk (ld.cu) -------------------------------------------------------
constexpr int kLdMaxWindow = VPCA_LD_MAX_WINDOW;   // H: variants a window may reach back (vpca_ld_prune_bed)
constexpr int kLdMaxChunk = 2 * kLdMaxWindow;   // C: variants per chunk (a multiple of 32)
// One chunk: chunk rows [0, nc) are variants s0 + [0, nc), rows [own_lo, nc) are the ones it decides; wlo[v] is the global
// window start of chunk row v.  Words: T = ceil(H / 32) + 1 per row; word w of row b holds the pairs (a, b) with a in
// tile b / 32 - (T - 1) + w, bit a % 32.
struct LdChunk {
    const int32_t* G;      // 3c x 3c int32 plane Gram (lower triangle)
    const int64_t* wlo;
    int64_t s0;
    int c, nc, own_lo, T;
    double r2_max;
    const uint8_t* elig;   // vpca_ld_prune_bed_masked: eligible[v] of every variant v of the call; nullptr = all eligible
};
struct LdWork {
    DeviceBuffer<uint32_t> d_bits;      // c x T in-LD bits
    DeviceBuffer<int32_t> d_seg;        // c x T: pairs before word w in row b
    DeviceBuffer<int32_t> d_row_total;  // c: in-LD pairs of row b
    DeviceBuffer<int64_t> d_row_start;  // c: output position of the first pair of row b
    DeviceBuffer<int64_t> d_total;      // in-LD pairs of the call so far
    DeviceBuffer<int64_t> d_pairs;      // pair scratch: (i, j) of each pair, then its r2
    DeviceBuffer<double> d_r2;          // (its capacity is the pairs the scratch holds)
};
// Pass 1: bits, per-word prefix, row totals (and their sum into *d_total) of the owned rows.  Never synchronises.
cudaError_t ld_count(LdWork& w, const LdChunk& ch, cudaStream_t stream);
// Keep-first sweep over the owned rows, in order: keep[s0 + b] = no kept a in b's window is in LD with b.  Reads keep of
// the rows before own_lo (decided by the previous chunk).  Never synchronises.
cudaError_t ld_sweep(LdWork& w, const LdChunk& ch, uint8_t* d_keep, cudaStream_t stream);
// Pass 2: the in-LD pairs of row tiles [bt_lo, bt_hi) whose output position p lies in [base, end) go to scratch slot
// p - base (needs w.d_row_start).  Never synchronises.
cudaError_t ld_emit(LdWork& w, const LdChunk& ch, int bt_lo, int bt_hi, int64_t base, int64_t end, cudaStream_t stream);

// ---- variant QC (qc.cu, DESIGN.md 10) ------------------------------------------------------------------------------
// HOM_A1, HET, HOM_A2, MISSING of nv .bed rows of n samples, row v at d_rows + v * pitch, into d_counts[4v ..] (16-byte
// aligned).  Bytes past ceil(n / 4) and the padding bits of the last byte are ignored.  Never synchronises.
cudaError_t qc_count(const uint8_t* d_rows, int64_t pitch, int nv, int n, int32_t* d_counts, cudaStream_t stream);
// The exact HWE p-value (vpca.h) of each of nv count rows (layout above, 16-byte aligned).  Never synchronises.
cudaError_t qc_hwe(const int32_t* d_counts, int nv, double* d_p, cudaStream_t stream);

// ---- variance-standardized relationship matrix (grm.cu, DESIGN.md 13) -----------------------------------------------
// Used variants per FP64 panel: a constant, so that the panel boundaries, and with them the bits of the sum, depend only
// on the ordered sequence of used variants.
constexpr int kGrmPanelK = 1024;
// Rows of a panel: n rounded up to the SYRK's tile edge (rows >= n stay zero).
int64_t grm_panel_rows(int n);
// From nv count rows (qc_count's layout): d_tab[4v ..] = z of each .bed code (0 for missing calls and unused variants),
// d_used[v] in {0, 1}, d_inv[0 .. *d_total) = the used variants in row order.  Never synchronises.
cudaError_t grm_tables(const int32_t* d_counts, int nv, double* d_tab, int32_t* d_used, int32_t* d_inv, int* d_total,
                       cudaStream_t stream);
// Panel columns [col0, col0 + cnt) = the z columns of rows d_inv[0 .. cnt) (row v at d_rows + v * stride), samples < n.
cudaError_t grm_expand(const uint8_t* d_rows, int64_t stride, const int32_t* d_inv, const double* d_tab, int cnt, int n,
                       double* d_Z, int col0, cudaStream_t stream);
// Lower-triangle tiles of d_C (n x n row-major) += Z Z^T over the kGrmPanelK columns of the panel.  Never synchronises.
cudaError_t grm_syrk(const double* d_Z, int n, double* d_C, cudaStream_t stream);
// d_C = its lower triangle / m, mirrored to the upper one.
cudaError_t grm_finish(double* d_C, int n, int64_t m, cudaStream_t stream);
// The z tables and used flags of grm_tables alone (no used list).  Never synchronises.
cudaError_t grm_table(const int32_t* d_counts, int nv, double* d_tab, int32_t* d_used, cudaStream_t stream);

// ---- GRM loadings and projection (grm_project.cu, DESIGN.md 14) -----------------------------------------------------
// d_w[v * k + c] = sum over samples s < n, in order, of tab[v][code(s, v)] U[c * n + s] for nv rows (row v at d_rows +
// v * stride), U n x k column-major, k in [1, 16].  Never synchronises.
cudaError_t grm_loadings(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_U,
                         int k, double* d_w, cudaStream_t stream);
// Scratch (doubles) grm_project needs for nv rows of n samples at k components.
int64_t grm_project_scratch_doubles(int n, int64_t nv, int k);
// d_acc[s * acc_ld + c] += sum over the nv rows of tab[v][code(s, v)] w[v * k + c]: fixed panels of variants summed in
// variant order, the panel partials (d_part) added in panel order.  Never synchronises.
cudaError_t grm_project(const uint8_t* d_rows, int64_t stride, int nv, int n, const double* d_tab, const double* d_w,
                        int k, double* d_part, double* d_acc, int acc_ld, cudaStream_t stream);

// ---- linear association tests (glm.cu, DESIGN.md 15) ----------------------------------------------------------------
// Doubles per variant of the sums: b_0 .. b_KMAX (b_c = sum g' q_c for c < q, b_q = sum g' y~, zero past q, g' the
// centred dosage of glm.cu), then OBS_CT, sum g and sum g^2 of the raw dosage (exact integers).
constexpr int kGlmRec = VPCA_GLM_MAX_Q + 4;
// Columns of Q the kernels are instantiated for (2, 4, 8, 16 or 32); Qx has glm_kmax(q) + 2 doubles per sample.
int glm_kmax(int q);
// nv .bed rows (row v at d_rows + v * stride) of n samples: the sums into d_sums (nv x kGlmRec), then
// d_out[v * 6 ..] = OBS_CT, A1_FREQ, BETA, SE, T_STAT, P and d_err[v] (VPCA_GLM_*).  d_Qx: n rows [q_0 .. q_{q-1}, y~, 0 ..,
// mask]; d_mask: bit e of byte j = sample 4 j + e is a regression sample; d_z0 = Q^T y~ (q); yty = y~^T y~; n_reg the
// regression samples; counted 1 (A1) or 2 (A2).  Never synchronises.
cudaError_t glm_linear(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, int n_reg, const double* d_Qx,
                       const uint8_t* d_mask, const double* d_z0, double yty, int counted, double* d_sums, double* d_out,
                       int32_t* d_err, cudaStream_t stream);
// Logistic tests (DESIGN.md 16) of nv .bed rows: the counts into d_cnt (nv x 6: OBS_CT, sum g, sum g^2 under d_mask, then
// under d_case), then d_out[v * 6 ..] = OBS_CT, A1_FREQ, BETA, SE, Z, P, d_err[v] (VPCA_GLM_*) and d_passes[v] (Newton
// passes, 0 for a variant flagged before any).  d_Qx: n rows [q_0 .. q_{q-1}, y, 0 .., mask] with y in {0, 1}; d_case:
// the regression samples with y = 1 as bits; d_theta0: the null fit in the basis Q (q).  firth_mode 0: the
// maximum-likelihood fit alone.  With Firth's penalized likelihood (DESIGN.md 17): VPCA_GLM_FIRTH_FALLBACK, then the
// Firth fit of the variants the maximum-likelihood fit ends with LOGISTIC_CONVERGE_FAIL after a pass, listed on the
// device in d_idx (nv) and d_nf (1); VPCA_GLM_FIRTH_ALWAYS, the Firth fit alone; d_firth[v] (nv) = 1 where the Firth fit
// ran.  d_firth, d_idx and d_nf are unused in mode 0.  Never synchronises.
cudaError_t glm_logistic(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, const double* d_Qx,
                         const uint8_t* d_mask, const uint8_t* d_case, const double* d_theta0, int counted, double* d_cnt,
                         double* d_out, int32_t* d_err, int32_t* d_passes, int firth_mode, uint8_t* d_firth,
                         int32_t* d_idx, int32_t* d_nf, cudaStream_t stream);

// ---- sample QC (samples.cu, DESIGN.md 11) ---------------------------------------------------------------------------
// Adds the MISSING calls (code 01) of each of the n samples over nv .bed rows (row v at d_rows + v * pitch) to
// d_missing[0 .. n) with integer atomics.  Bytes past ceil(n / 4) and the padding bits of the last byte are ignored.
// Never synchronises.
cudaError_t sample_missing(const uint8_t* d_rows, int64_t pitch, int nv, int n, int32_t* d_missing, cudaStream_t stream);
// Out row v (at d_out + v * out_pitch, ceil(m / 4) bytes written, padding bits 0) = the codes of samples d_keep_idx[0 .. m)
// of source row v (at d_rows + v * pitch).  Never synchronises.
cudaError_t subset_samples(const uint8_t* d_rows, int64_t pitch, int nv, const int32_t* d_keep_idx, int m, uint8_t* d_out,
                           int64_t out_pitch, cudaStream_t stream);

// ---- KING-robust kinship pairs from the 3n x 3n plane Gram (kinship.cu) ----------------------------------------------
constexpr int kKinMaxN = 21845;   // 3n <= 65 535: the plane Gram stays below 2^32 cells
// Device scratch of vpca_kinship_pairs, owned by the context and kept between calls.
struct KinPairWork {
    int n = 0;
    DeviceBuffer<int32_t> d_seg;        // n x ceil(n / 32): selected pairs per (row b, 32-column tile), then their row-wise scan
    DeviceBuffer<int32_t> d_row_total;  // n: selected pairs per row b
    DeviceBuffer<int64_t> d_row_start;  // n: output position of the first selected pair of row b
    DeviceBuffer<int32_t> d_ids;        // pair scratch: 2 ids, 5 counts, 1 kinship each (d_kin's capacity: the pairs it holds)
    DeviceBuffer<int32_t> d_counts;
    DeviceBuffer<double> d_kin;
};
cudaError_t kin_pair_alloc(KinPairWork& w, int n);
// Pass 1: w.d_seg / w.d_row_total for the threshold (select_all: every pair, NaN included).  Never synchronises.
cudaError_t kin_count(KinPairWork& w, const int32_t* d_G, int n, double min_kinship, bool select_all, cudaStream_t stream);
// Pass 2: the selected pairs of tile rows [bt_lo, bt_hi) whose output position p lies in [base, end) go to scratch slot
// p - base (needs w.d_row_start).  Never synchronises.
cudaError_t kin_emit(KinPairWork& w, const int32_t* d_G, int n, double min_kinship, bool select_all, int bt_lo, int bt_hi,
                     int64_t base, int64_t end, cudaStream_t stream);

// ---- multi-dataset keying: variant keys, join, merge (join.cu)---------------------------------------------
struct JoinWork {
    DeviceBuffer<uint64_t> d_hash;       // 2 per row: MurmurHash3_x64_128 of the variant key
    DeviceBuffer<int32_t> d_table;       // open-addressing table of row indices (-1 = empty)
    uint64_t table_slots = 0;
    DeviceBuffer<int64_t> d_rows;        // output rows / calls each input row is responsible for, and their exclusive scans
    DeviceBuffer<int64_t> d_len;
    DeviceBuffer<int64_t> d_row_base;
    DeviceBuffer<int64_t> d_nnz_base;
    DeviceBuffer<int32_t> d_leader;
    DeviceBuffer<int64_t> d_prefix;
    DeviceBuffer<int64_t> d_block;       // scan scratch
    DeviceBuffer<int64_t> d_totals;      // {output rows, output calls}
    int64_t* h_totals = nullptr;         // pinned copy
    DeviceBuffer<int64_t> d_out_off;     // the joined CSR: out_rows + 1 offsets, out_nnz sample indices
    DeviceBuffer<int32_t> d_out_idx;
    int64_t out_rows = -1, out_nnz = 0;   // result of the last join (-1: none)
    // device copies of the caller's input (grow-only)
    DeviceBuffer<uint8_t> d_payload;
    DeviceBuffer<int64_t> d_key_off;
    DeviceBuffer<int64_t> d_off;
    DeviceBuffer<int32_t> d_idx;
};
cudaError_t hash_keys(const uint8_t* d_payload, const int64_t* d_off, int64_t nkeys, uint64_t* d_hash, cudaStream_t stream);
cudaError_t join_rows(JoinWork& w, int mode, int variant_set_count, int64_t n_left, const uint8_t* d_payload,
                      const int64_t* d_key_off, const int64_t* d_off, const int32_t* d_idx, int64_t nrows, cudaStream_t stream,
                      int64_t* out_rows, int64_t* out_nnz, int64_t* launches);
void join_free(JoinWork& w);

// ---- top-k of a Gram held as row bands across contexts (eig.cu, vpca_compute_pca_bands) ------------------------------
// One rank's share: its band of S (rows [row0, row0 + rows), lower-triangle cells meaningful) and the buffers of its part
// of the sharded mat-vec, all on the rank's device.  Owned by the rank's context (or by an EigWork for its one-band
// solves), kept between solves.
struct BandPart {
    int device = 0;
    cudaStream_t stream = nullptr;
    const int32_t* d_S = nullptr;   // row row0 of the band
    const double* d_Sd = nullptr;   // or, when set, the band of an FP64 matrix that is solved as it is (no centring)
    int n = 0, row0 = 0, rows = 0;
    DeviceBuffer<double> d_v;       // n: the Lanczos vector of the step
    DeviceBuffer<double> d_y;       // row0 + rows: the partial product (or partial row sums as int64)
    DeviceBuffer<double> d_scratch; // tile row partials, then tile column partials
    int alloc_n = 0, alloc_row0 = -1, alloc_rows = 0;
    cudaEvent_t ev_done = nullptr;  // the partial has landed on rank 0
};
void band_part_free(BandPart& p);

// Solver state on rank 0: the Lanczos basis (n x kLzCap), w ping-pong, the small Lanczos scalars, `world` slots of n
// doubles for the partials, row sums; no n x n matrix.
struct BandEigWork {
    int n = 0, kmax = 0;
    DeviceBuffer<double> d_V;
    DeviceBuffer<double> d_w;       // 2 n
    DeviceBuffer<double> d_small;   // alpha | beta | h1 | h2 | e2 | Y | theta2 | res | scal2 | sc | part
    DeviceBuffer<double> d_slots;   // 16 n
    DeviceBuffer<double> d_rowsum;  // n
    DeviceBuffer<double> d_rbar;    // n
    DeviceBuffer<double> d_scal;    // 16: [0] matrixMean, [2] ||T||
    DeviceBuffer<double> d_evals;   // kmax
    DeviceBuffer<double> d_evecs;   // n x kmax, column-major
    DeviceBuffer<double> d_lu;      // 8 kLzCap: inverse-iteration scratch
    DeviceBuffer<int> d_nz;
    DeviceBuffer<int> d_st;         // {step, flag, ticket, step cap}
    cudaEvent_t ev_v = nullptr;  // v_j is ready on rank 0
    int last_iters = 0;
};
void band_eig_free(BandEigWork& w);

// ---- centering + eigensolve (eig.cu) ---------------------------------------------------------------
struct EigWork {
    int n = 0;
    DeviceBuffer<double> d_C;     // n x n centered matrix, overwritten by the tridiagonalisation
    DeviceBuffer<double> d_rowsum;
    DeviceBuffer<double> d_v;     // Householder vector of the current step (n)
    DeviceBuffer<double> d_w;     // w vector of the current step (n)
    DeviceBuffer<double> d_p;     // p = tau A v (n)
    DeviceBuffer<double> d_diag;  // n
    DeviceBuffer<double> d_off;   // n
    DeviceBuffer<double> d_tau;   // n
    DeviceBuffer<double> d_scal;  // small scalar scratch
    DeviceBuffer<double> d_evals; // k
    DeviceBuffer<double> d_evecs; // n x k (column-major)
    DeviceBuffer<double> d_lu;    // 8 n scratch for inverse iteration
    DeviceBuffer<int> d_nz;
    DeviceBuffer<int> d_step;               // {next step, step of the pending trailing update}
    cudaGraphExec_t graph_exec = nullptr; // kGraphSteps tridiagonalisation steps, replayed n / kGraphSteps times
    int graph_n = 0;
    bool graph_fused = false;
    int kmax = 0;
    // persistent Lanczos workspace (allocated on the first solve in that form)
    DeviceBuffer<double> d_V;      // n x kLzCap orthonormal basis, column-major
    DeviceBuffer<double> d_lzw;    // 2 n: w ping-pong
    DeviceBuffer<double> d_lzs;    // alpha | beta | e2 | Y | theta2 | res | scal2 | part | hpart
    DeviceBuffer<int> d_lzst;      // {step, flag, ticket, step cap}
    DeviceBuffer<unsigned> d_lzbar;   // grid barrier counter of the persistent Lanczos kernel
    DeviceBuffer<double> d_lzG;       // kLzCap x kLzCap: V^T V of the Lanczos basis (one-reduction Gram-Schmidt)
    DeviceBuffer<long long> d_lzprof; // VPCA_LZ_PROF=1: phase timestamps of block 0 (first 64 steps)
    bool c_valid = false;       // d_C holds the centred matrix of the last center_gram()
    int lz_blocks = -1;         // blocks of the persistent kernel (= SMs; 0: cooperative launch unavailable or
                                // VPCA_LZ_PERSIST=0; -1: not queried yet, at the first Lanczos solve)
    size_t lz_smem_max = 0;     // dynamic shared memory a block of the persistent kernel may take (opt-in limit - static)
    const int32_t* d_S = nullptr;   // the (symmetrised) int32 Gram the last center_gram() read
    BandEigWork band_eig;       // Lanczos where the persistent form does not run: the band solver, the whole Gram as one
    BandPart band_part;         // band
    int last_method = 0;        // 1 direct, 2 Lanczos, 3 Lanczos abandoned -> direct
    int last_iters = 0;         // Lanczos steps of the last solve
    int mode = 0;               // 0 auto, 1 direct, 2 Lanczos whenever n allows
    bool grm = false;           // eig_topk solves d_C as it is (the GRM, symmetric): the band solver's Lanczos on FP64
                                // cells, or the direct reduction, which consumes d_C
};
cudaError_t eig_alloc(EigWork& w, int n, int kmax);
void eig_free(EigWork& w);
// row sums + matrix mean always; the FP64 matrix C only when `materialise` (or later, on demand, through center_matrix)
cudaError_t center_gram(EigWork& w, const int32_t* d_S, cudaStream_t stream, bool materialise);
cudaError_t center_matrix(EigWork& w, cudaStream_t stream);
cudaError_t eig_topk(EigWork& w, int k, cudaStream_t stream, int64_t* launches);

// Lanczos on the bands of `world` ranks (vpca_compute_pca_bands; eig_topk past the persistent form's fit, on one band).
// outcome: 0 converged (d_evals / d_evecs / d_nz hold the answer), 2 breakdown, 3 a missed eigenvalue found by the
// deflated verification run, 4 no convergence within the step budget.  Synchronises rank 0's stream at every convergence
// test; the bands are only read.
cudaError_t band_eig_topk(BandEigWork& w, BandPart* const* parts, int world, int kmax, int k, int64_t* launches,
                          int* outcome);

// ---- variant loadings and projection (project.cu) -----------------------------------------------------------------
// Both read cells in the panel layout (see gram_accumulate; zero cells after nv in the last panel), k in [1, 16].
// w[v * k + c] = sum_s x[s][v] U[s][c] (FP64, samples summed in order), count[v] = sum_s x[s][v] (exact) for v < nv;
// U: n x k column-major (ld n).  Never synchronises.  Above kSplitMinN samples the samples are summed in 4 ranges whose
// bounds depend on n alone, the range sums added in range order (project.cu): w[v] still depends on n, column v and U only.
constexpr int kSplitMinN = 65535;
// d_keep != nullptr (n bytes, after a subset solve; needs n <= kSplitMinN): count[v] adds only the samples whose keep byte is
// nonzero, U is zero on the others, and the samples are summed in the whole order whatever VPCA_LOADINGS_KERNEL says.
cudaError_t loadings_launch(const void* d_x, int elem_bits, int n, int64_t nv, int64_t panel, const double* d_U, int k,
                            double* d_w, int32_t* d_count, const uint8_t* d_keep, cudaStream_t stream);
// acc[s * acc_ld + c] += sum_v (y[s][v] - mean[v]) w[v * k + c] for the m samples: a partial sum per panel (variants in
// order) into d_part (project_scratch_doubles entries), then the partials added in panel order.
cudaError_t project_launch(const void* d_y, int elem_bits, int m, int64_t nv, int64_t panel, const double* d_w,
                           const double* d_mean, int k, double* d_part, double* d_acc, int acc_ld, cudaStream_t stream);
int64_t project_scratch_doubles(int m, int64_t nv, int64_t panel, int k);

// ---- principal coordinates of a subset of the samples (subset.cu, vpca_compute_pca_subset) ------------------------------
// d_idx: the m kept samples in increasing order, then the r removed ones in increasing order (m + r = n).
// S_KK[q1 * m + q2] = S[idx[q1]][idx[q2]] for q1, q2 < m (S: the finalized n x n Gram).  Never synchronises.
cudaError_t subset_gather(const int32_t* d_S, int n, const int32_t* d_idx, int m, int32_t* d_SKK, cudaStream_t stream);
// From the subset solve (u: m x k column-major, ld m; evals: k; rowsum: the m row sums of S_KK):
//   U[c * n + s]    = u_c of sample s for kept s, 0 for removed s (c < 16; the buffer the masked loadings read)
//   vecs[c * n + s] = u_c of sample s for kept s, p_c(s) for removed s (c < k, any k), where
//   p_c(r) = (sum_q S[r][idx[q]] u_c[q] - (sum_q rowsum[q] u_c[q]) / m) / evals[c]
// both sums over q in a fixed order (subset.cu), no floating-point atomics; d_t: k doubles of scratch.  Never synchronises.
cudaError_t subset_place(const int32_t* d_S, int n, const int32_t* d_idx, int m, const double* d_u, const double* d_evals,
                         const double* d_rowsum, int k, double* d_U, double* d_vecs, double* d_t, cudaStream_t stream);

// ---- synthetic generator (synth.cu) ----------------------------------------------------------------
cudaError_t synth_dense(uint64_t seed, int n, int64_t v0, int64_t nv, int mode, int elem_bits, void* d_x,
                        int64_t ld, int64_t panel, cudaStream_t stream);

}  // namespace vpca
