// Gram / similarity accumulation  S += X X^T  on sm_90a tensor cores.
//
// Replaces the hot loop of VariantsPcaDriver.getSimilarityMatrix
// (reference: src/main/scala/com/google/cloud/genomics/spark/examples/VariantsPca.scala:182-191,
//  `for (c1 <- callset; c2 <- callset) matrix(c1, c2) += 1` over every variant) by a dense symmetric
// rank-V update on the genotype matrix X (samples x variants, sample-major in HBM):
//
//   TMA (cp.async.bulk.tensor, SWIZZLE_128B)  ->  shared memory ring  ->  wgmma (s8 -> s32 / bf16 -> f32)
//   ->  accumulators in the registers of two consumer warpgroups  ->  red.global.add into the lower triangle of S.
//
// CTA pairs (VPCA_CTA_GROUP=2, the default) are 2-CTA clusters: both CTAs multiply the same B rows, so B box r is fetched
// once, by CTA r, and multicast into both CTAs' shared memory, while each CTA loads its own A block.  Per k-block a CTA
// pulls 32 KB from L2 instead of 48 KB (16 KB instead of 32 KB on a self-B tile).  Both CTAs walk the same k-blocks.
//
// Work decomposition ("window-synchronous stream-K"):
//   * an output tile is the product of A row blocks (128 samples each: one per CTA, so two for a CTA pair with
//     VPCA_CTA_GROUP=2) and up to 256 B rows; the B rows are the wgmma M side (128 per consumer warpgroup), the A block
//     the N side, and the accumulator D[m][n] = sum_v X[rowB + m][v] X[rowA + n][v] is cell S[rowB + m][rowA + n];
//   * default tiling: rectangles of 256 A rows (two adjacent 128-blocks, one per CTA of a pair) x up to 256 B rows that
//     touch row >= col, the B strips of nearly equal width (2504 samples: 7 x 256 + 3 x 240);
//   * EXACT BLOCK COVER (VPCA_EXACT_COVER=1, off by default): in units of 128 x 128 blocks the lower triangle of S has
//     nb (nb + 1) / 2 blocks; the A blocks of a pair need not be adjacent, the B rows may be a single block (N = 128), and
//     a block above the diagonal may be computed in place of its mirror image and written transposed; with that freedom
//     the tile list of build_tiles covers every needed block exactly once (2504 samples: 210 blocks instead of 220);
//   * owner-computes bands: a context that stores only rows [own_lo, own_hi) of S and has no peers enumerates only the
//     tiles of those rows (every variant is fed to every band's context; nothing is flushed anywhere else);
//   * the variant axis is cut into k-blocks of 128 bytes (one swizzle atom; packed e2m1 cells are expanded to that
//     layout in shared memory) and into windows of `kb_window` k-blocks; in every window the (tile, k-block) units are
//     split over the workers (CTAs, or CTA pairs), and all workers walk the windows in the same order, so the slice of X
//     a window needs (n x kb_window * 128 B, sized to sit in L2) is fetched from HBM once and re-read from L2 by the
//     other tiles;
//   * a worker holds ONE accumulator (128 x 256 int32 / fp32 in registers); when the split of a window gives every
//     worker a piece of a single tile (N = 2504: 55 tiles, 66 pairs) that piece is the same in every window and the
//     accumulator is flushed once at the end of the launch; otherwise (large N) it is whole-tile waves + a stream-K tail
//     whose pieces are flushed one after the other;
//   * with more tiles than half the workers but fewer than all of them (N = 2504: 55 tiles, 66 pairs) that split would
//     leave some workers a whole tile in every window: there each tile has a front worker that multiplies it over the
//     k-blocks [0, s), and the remaining workers share the tiles over [s, K) (front/tail schedule, see Sched);
//   * the split of a window over the workers is speed-weighted from launch to launch (rebalance_kernel, repair_split);
//   * the flush packs two cells into one 64-bit red (no carry between the halves: counts are non-negative, sums < 2^31).
// Integer atomics make the result independent of the order of the flushes: S is bit-exact.
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstring>

#include <algorithm>
#include <map>
#include <mutex>
#include <tuple>
#include <type_traits>
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "ptx_sm90.cuh"
#include "vpca_internal.h"

namespace vpca {

namespace {

constexpr int kThreads = 384;                   // warpgroup 0: TMA producer; warpgroups 1 and 2: wgmma consumers
constexpr int kKBytes = 128;                    // bytes of K per k-block in the operand layout: one SWIZZLE_128B atom
constexpr int kBoxRows = 128;                   // rows per TMA box
constexpr int kUmmaN = 256;                     // B rows of a tile (wgmma M of the two consumer warpgroups)
constexpr int kAccCols = 256;                   // accumulator budget of one worker: one tile of up to 256 B rows
constexpr long long kWatchdogCycles = 20000000000LL;   // ~10 s: a stuck barrier traps instead of hanging the box

template <int KIND>
struct Cfg {
    // KIND 0 (int8) / 1 (bf16): 128-byte rows, swizzled by TMA; KIND 2 (packed e2m1): 64-byte rows of 128 cells that
    // the consumers expand into two 128-byte-row buffers (ping-pong) of 384 rows: 256 B rows, then the A block
    static constexpr int BOX_BYTES = kBoxRows * (KIND == 2 ? kKBytes / 2 : kKBytes);
    static constexpr int B_BYTES = 2 * BOX_BYTES;
    static constexpr int STAGE_BYTES = 3 * BOX_BYTES;
    static constexpr int STAGES = 4;
    static constexpr int XBUF_BYTES = KIND == 2 ? 3 * kBoxRows * kKBytes : 0;
    static constexpr int BAR_BYTES = 256;
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 2 * XBUF_BYTES + BAR_BYTES + 1024;   // + 1024 B alignment slack
};

constexpr int kMaxPeers = 16;

// One output tile: (A block of CTA 0, A block of CTA 1) x (n_eff B rows from rowB).
struct TileDesc {
    int rowA0, rowA1;   // first sample of the A block of CTA 0 / CTA 1 (one CTA per tile: rowA0 only)
    int rowB;           // first sample of the B rows
    int n_eff;          // MMA N: B rows that exist, rounded up to 16
    int wstart;         // sum of the weights (n_eff / 16) of the tiles before this one
    int flags;          // kTileXpose: a 128-block above the diagonal is written transposed (it stands in for its mirror
                        // image) instead of being skipped; kTileFiller: CTA 1's A block only pads the pair, drop its output
    int acc_cols;       // accumulator columns it takes in the plan of a worker: always kAccCols (the register
                        // accumulator of a CTA spans 256 B rows whatever n_eff is)
    int pad1;
};
constexpr int kTileXpose = 1, kTileFiller = 2, kTileSelfB = 4;   // kTileSelfB: the B rows ARE the pair's two A blocks (a
                                                                  // diagonal 256 x 256 tile): B is read from the A tile, no B load
constexpr int kMaxSegs = 4;   // (tile, k-range) pieces a plan may hold (the accumulator budget admits one per window)

struct GramArgs {
    int32_t* S;
    int32_t* peer[kMaxPeers];   // num_peers > 0: the flush goes to peer-mapped Grams (own included) over NVLink:
    int num_peers;              //   peer_mode 0: into ALL of them (replicated reduce);
    int peer_mode;              //   peer_mode 1: only into the Gram of the rank that owns the row (reduce-scatter)
    int own_end[kMaxPeers];     // rank q owns Gram rows [own_end[q-1], own_end[q]); multiples of 32, >= 32 apart
    const TileDesc* tiles;
    int* err;          // mapped host memory: watchdog diagnostics
    int n;
    int num_tiles;
    int num_full;      // leading tiles of full weight: what the large-N schedule deals out in whole-tile waves
    int total_weight;  // sum of n_eff / 16 over all tiles
    int kb_total;
    int kb_window;
    int num_workers;
    int resident;
    int kc_per_kb;     // TMA coordinate units (cells; bytes for packed e2m1) per k-block
    int kb_per_panel;  // k-blocks per panel of the genotype matrix (row-major input = one panel)
    int sync_lead;     // > 0: a worker may run at most this many windows ahead of the slowest one (soft barrier)
    int active_workers;
    int* win_done;     // win_done[w] = number of workers whose producer has issued every load of window w
    long long* prof;   // optional per-CTA timestamps (globaltimer ns): start, first MMA, MMA done, end
    const double* cum; // cum[w] = fraction of every window's units owned by workers < w (cum[0] = 0, cum[W] = 1)
    int front_tiles;   // > 0: the front/tail schedule (see Sched), with this many tiles (= front workers)
    const double* front_frac;   // front/tail schedule: the front ends at k-block front_split(*front_frac, kb_total)
    int col_limit;     // accumulator columns of one worker (kAccCols)
    int acc_stride;    // unused by the register accumulator (Seg.col of the large-N schedule)
    int row_limit;     // rows of S at or beyond this one are never written (n, or the end of an owner-computes band)
    int red64;         // epilogue packs two cells per 64-bit red (VPCA_RED64=0: one 32-bit red per cell)
};

struct Seg {
    int tile, kb0, kb1, col, slot, first, flush, use, win, last_in_win;   // slot: which accumulator barrier pair
    int rowA0, rowA1, rowB, n_eff, flags;
};

// The pieces of a weighted unit range [u_begin, u_end) -- tile t occupies [wstart_t * len, (wstart_t + w_t) * len) and its
// k-block q sits at wstart_t * len + q * w_t -- as (tile, k-range, accumulator column) triples.  Two workers that share a
// boundary u agree on the k-block it falls in (both take floor((u - base) / w_t)), so the pieces partition every tile.
// Shared by the kernel, by the host (which decides whether the accumulators of a worker fit its budget) and by the rebalancer.
struct SegPlan {
    int n;
    int tile[kMaxSegs], lo[kMaxSegs], hi[kMaxSegs], col[kMaxSegs];
    int cols;      // accumulator columns needed
    int overflow;  // more than kMaxSegs pieces
};

__host__ __device__ inline void plan_segments(const TileDesc* tiles, int num_tiles, int first_tile, long long u_begin,
                                              long long u_end, int len, SegPlan& p) {
    p.n = 0;
    p.cols = 0;
    p.overflow = 0;
    const long long origin = (long long)tiles[first_tile].wstart * len;
    long long u = u_begin;
    int t = first_tile;
    while (u < u_end && t < num_tiles) {
        const int w = tiles[t].n_eff >> 4;
        const long long base = (long long)tiles[t].wstart * len - origin;
        const long long tend = base + (long long)w * len;
        if (tend <= u) {
            ++t;
            continue;
        }
        const long long e = u_end < tend ? u_end : tend;
        const int lo = (int)((u - base) / w);
        const int hi = e == tend ? len : (int)((e - base) / w);
        u = e;
        if (lo >= hi) continue;   // a sliver thinner than one k-block: the neighbour owns that k-block
        if (p.n == kMaxSegs) {
            p.overflow = 1;
            return;
        }
        p.tile[p.n] = t;
        p.lo[p.n] = lo;
        p.hi[p.n] = hi;
        p.col[p.n] = p.cols;
        p.cols += tiles[t].acc_cols;
        ++p.n;
    }
}

// Largest e <= u_end such that the pieces of [u_begin, e) fit one worker's accumulator budget (at most kMaxSegs pieces,
// at most col_limit columns): u_end itself, or the start of the first tile whose accumulator no longer fits.
// `hint`: a tile index at or before the tile that holds u_begin (advanced to it; callers walk u_begin upwards).
__host__ __device__ inline long long feasible_end(const TileDesc* tiles, int num_tiles, long long u_begin, long long u_end,
                                                  int len, int col_limit, int& hint) {
    int n = 0, cols = 0;
    long long u = u_begin;
    int t = hint;
    bool first = true;
    while (u < u_end && t < num_tiles) {
        const int w = tiles[t].n_eff >> 4;
        const long long base = (long long)tiles[t].wstart * len;
        const long long tend = base + (long long)w * len;
        if (tend <= u) {
            ++t;
            continue;
        }
        if (first) {
            hint = t;
            first = false;
        }
        const long long e = u_end < tend ? u_end : tend;
        const int lo = (int)((u - base) / w);
        const int hi = e == tend ? len : (int)((e - base) / w);
        if (lo < hi) {
            if (n == kMaxSegs || cols + tiles[t].acc_cols > col_limit) return u;
            ++n;
            cols += tiles[t].acc_cols;
        }
        u = e;
    }
    return u_end;
}

// Makes a candidate split (cand[0] = 0 <= cand[1] <= ... <= cand[workers] = 1, fractions of the uw units of a window)
// feasible: worker i ends where feasible_end says it must, and worker i + 1 starts there.  A worker is never cut
// below need[i + 1], the earliest point from which workers i + 1 .. workers - 1 can still cover the rest of the window
// within their budgets (a worker's budget may hold only one tile, so trimming every cut worker to its tile edge would
// leave the last ones short).  need: scratch of workers + 1 entries.  False if no split fits (the caller keeps the old one).
__host__ __device__ inline bool repair_split(const TileDesc* tiles, int num_tiles, int workers, long long uw, int len,
                                             int col_limit, double* cand, long long* need) {
    need[workers] = uw;
    for (int j = workers - 1; j >= 1; --j) {
        // smallest start from which one worker reaches need[j + 1] (a later start only drops pieces: monotone)
        long long lo = 0, hi = need[j + 1];
        while (lo < hi) {
            const long long mid = lo + (hi - lo) / 2;
            int h = 0;
            if (feasible_end(tiles, num_tiles, mid, need[j + 1], len, col_limit, h) >= need[j + 1]) hi = mid;
            else lo = mid + 1;
        }
        need[j] = hi;
    }
    long long ub = 0;
    int hint = 0;
    for (int i = 0; i < workers; ++i) {
        long long ue = (i + 1 == workers) ? uw : (long long)((double)uw * cand[i + 1]);
        if (ue < ub) ue = ub;
        if (i + 1 < workers && ue < need[i + 1]) ue = need[i + 1];
        const long long fe = feasible_end(tiles, num_tiles, ub, ue, len, col_limit, hint);
        if (fe < ue) {
            if (i + 1 == workers || fe < need[i + 1]) return false;
            ue = fe;
        }
        if (i + 1 < workers) cand[i + 1] = ((double)ue + 0.5) / (double)uw;   // floor(uw * cand) == ue in the kernel
        ub = ue;
    }
    return true;
}

// The front/tail schedule applies when W / 2 < T < W (T tiles, W workers): an equal split of every window would give some
// workers a whole tile and the others a sliver, so the critical path would be a whole tile in every window.
__host__ __device__ inline bool front_tail_applies(int num_tiles, int workers) {
    return 2 * num_tiles > workers && num_tiles < workers;
}

// Its split point s: the front covers k-blocks [0, s), the tail [s, kb_total).
__host__ __device__ inline int front_split(double frac, int kb_total) {
    const double f = frac < 0.0 ? 0.0 : (frac > 1.0 ? 1.0 : frac);
    const int s = (int)(f * (double)kb_total);
    return s < kb_total ? s : kb_total;
}

// Every role of a worker (TMA producer, MMA issuer, epilogue) replays the same deterministic schedule.
//   resident (every worker's accumulators fit its budget):  window-synchronous stream-K -- the worker owns the same pieces
//               (tile, k-range) in every window, so its accumulator stays in registers for the whole launch;
//   front/tail (resident, W / 2 < T < W): front worker t < T owns tile t for k-blocks [0, s) and walks the windows like
//               the resident schedule (one flush); the W - T tail workers split the region T tiles x [s, kb_total),
//               tile-major, into contiguous equal shares, and flush every piece when it completes.  The tail stays out
//               of the window pacing (Seg.win = -1).  s moves from launch to launch (rebalance_front_kernel);
//   otherwise:  full tiles in waves (wave i = tiles [i W, (i+1) W), one per worker, whole K) -- the tile list is ordered
//               so that a wave is a compact 2-D block of S and shares few row panels of X -- then the leftover
//               tiles are split stream-K style over all workers; accumulators double-buffered against the epilogue.
// Host-callable so that vpca_debug_schedule replays exactly what the kernel runs.
struct Sched {
    SegPlan plan;
    long long u_begin, u_end, u;
    int kbw, nwin, kb_total, kb_end, resident, win, seg_i, nflush, acc_stride;
    int worker, workers, num_tiles, wave, full_waves, tail_first;
    int tail, kb_split;   // front/tail schedule: this worker is in the tail; the split point s
    const TileDesc* tiles;

    // false if the worker's resident pieces do not fit its accumulator (the kernel then traps)
    __host__ __device__ bool init(const GramArgs& a, int w) {
        kbw = a.kb_window;
        kb_total = a.kb_total;
        kb_end = kb_total;
        resident = a.resident;
        acc_stride = a.acc_stride;
        worker = w;
        workers = a.num_workers;
        num_tiles = a.num_tiles;
        tiles = a.tiles;
        win = 0;
        seg_i = 0;
        nflush = 0;
        wave = 0;
        tail = 0;
        kb_split = kb_total;
        u_begin = u_end = 0;
        if (a.front_tiles > 0) {
            kb_split = front_split(*a.front_frac, kb_total);
            if (worker < a.front_tiles) {   // one piece of a whole tile's width in every window of [0, s)
                kb_end = kb_split;
                plan.n = 1;
                plan.tile[0] = worker;
                plan.lo[0] = 0;
                plan.hi[0] = kbw;
                plan.col[0] = 0;
                plan.cols = tiles[worker].acc_cols;
                plan.overflow = 0;
            } else {                        // units of the tail: tile-major, kb_total - s per tile
                tail = 1;
                const long long units = (long long)a.front_tiles * (kb_total - kb_split);
                const int tw = workers - a.front_tiles, j = worker - a.front_tiles;
                u_begin = units * j / tw;
                u_end = units * (j + 1) / tw;
                plan.n = 0;
            }
        } else if (resident) {
            const long long uw = (long long)a.total_weight * kbw;
            // speed-weighted split (equal shares until the first launches have been timed, see rebalance_kernel)
            u_begin = (long long)((double)uw * a.cum[worker]);
            u_end = (worker + 1 == a.num_workers) ? uw : (long long)((double)uw * a.cum[worker + 1]);
            plan_segments(tiles, num_tiles, 0, u_begin, u_end, kbw, plan);
            if (plan.overflow || plan.cols > a.col_limit) {   // overlapping accumulators would corrupt S silently
#ifdef __CUDA_ARCH__
                if (a.err != nullptr && threadIdx.x == 0) {
                    a.err[0] = 9;
                    a.err[1] = (int)blockIdx.x;
                    a.err[2] = plan.cols;
                    a.err[3] = plan.n;
                    __threadfence_system();
                }
                __trap();
#else
                return false;
#endif
            }
        } else {
            full_waves = a.num_full / workers;
            tail_first = full_waves * workers;
            const long long tail_units =
                tail_first < num_tiles ? (long long)(a.total_weight - tiles[tail_first].wstart) * kb_total : 0;
            u_begin = tail_units * worker / workers;       // weighted units of the leftover tiles
            u_end = tail_units * (worker + 1) / workers;
            plan.n = 0;
        }
        nwin = (kb_end + kbw - 1) / kbw;
        u = u_begin;
        return true;
    }
    __host__ __device__ void fill(Seg& s, int t) const {
#ifdef __CUDA_ARCH__
        const int4 lo = __ldg(reinterpret_cast<const int4*>(tiles + t));
        const int4 hi = __ldg(reinterpret_cast<const int4*>(tiles + t) + 1);
#else
        const int4 lo = reinterpret_cast<const int4*>(tiles + t)[0];
        const int4 hi = reinterpret_cast<const int4*>(tiles + t)[1];
#endif
        s.tile = t;
        s.rowA0 = lo.x;
        s.rowA1 = lo.y;
        s.rowB = lo.z;
        s.n_eff = lo.w;
        s.flags = hi.y;
    }
    __host__ __device__ bool next(Seg& s) {
        if (tail) {   // one piece at a time: [u, end of its tile or of the share), flushed when it completes
            if (u >= u_end) return false;
            const int span = kb_total - kb_split;
            const int t = (int)(u / span);
            const long long e = u_end < (long long)(t + 1) * span ? u_end : (long long)(t + 1) * span;
            fill(s, t);
            s.kb0 = kb_split + (int)(u - (long long)t * span);
            s.kb1 = kb_split + (int)(e - (long long)t * span);
            s.win = -1;
            s.last_in_win = 0;
            s.first = 1;
            s.flush = 1;
            s.col = 0;
            s.slot = 0;
            s.use = 0;
            u = e;
            return true;
        }
        if (!resident) {
            s.win = 0;
            s.last_in_win = 0;
            s.first = 1;
            s.flush = 1;
            s.slot = nflush & 1;
            s.col = s.slot * acc_stride;
            s.use = nflush >> 1;
            if (wave < full_waves) {                        // one whole tile of the current wave
                fill(s, wave * workers + worker);
                s.kb0 = 0;
                s.kb1 = kb_total;
                ++wave;
                ++nflush;
                return true;
            }
            // stream-K tail: at most kMaxSegs pieces are planned at a time
            while (true) {
                if (seg_i < plan.n) {
                    fill(s, plan.tile[seg_i]);
                    s.kb0 = plan.lo[seg_i];
                    s.kb1 = plan.hi[seg_i];
                    ++seg_i;
                    ++nflush;
                    return true;
                }
                if (u >= u_end) return false;
                // plan the next pieces: advance u to the end of what was planned
                plan_segments(tiles, num_tiles, tail_first, u, u_end, kb_total, plan);
                seg_i = 0;
                if (plan.n == 0) return false;
                const int lt = plan.tile[plan.n - 1];
                const long long base = (long long)(tiles[lt].wstart - tiles[tail_first].wstart) * kb_total;
                const long long endu = base + (long long)plan.hi[plan.n - 1] * (tiles[lt].n_eff >> 4);
                u = plan.overflow ? endu : u_end;
            }
        }
        if (plan.n == 0) return false;
        if (seg_i == plan.n) {
            ++win;
            seg_i = 0;
        }
        if (win >= nwin) return false;
        const int i = seg_i++;
        fill(s, plan.tile[i]);
        const int base = win * kbw;
        const int cnt = kbw < kb_end - base ? kbw : kb_end - base;
        s.kb0 = base + (plan.lo[i] < cnt ? plan.lo[i] : cnt);
        s.kb1 = base + (plan.hi[i] < cnt ? plan.hi[i] : cnt);
        s.win = win;
        s.last_in_win = (seg_i == plan.n);
        s.col = plan.col[i];
        s.slot = i;
        s.first = (win == 0);
        s.flush = (win == nwin - 1);
        s.use = 0;
        return true;
    }
};

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity, int* err, int code) {
    if (ptx::mbar_try_wait(bar, parity)) return;
    const long long t0 = clock64();
    while (!ptx::mbar_try_wait(bar, parity)) {
        if (clock64() - t0 > kWatchdogCycles) {
            if (err != nullptr) {
                err[0] = code;
                err[1] = (int)blockIdx.x;
                err[2] = (int)bar;
                err[3] = (int)parity;
                __threadfence_system();
            }
            __trap();
        }
    }
}

__device__ __forceinline__ long long globaltimer_ns() {
    long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Soft inter-worker barrier: wait (bounded) until `need` workers have finished issuing window `w`.  Purely a pacing
// hint that keeps all workers inside the same few L2-resident windows of X; correctness never depends on it.
__device__ __forceinline__ void wait_window(const int* win_done, int w, int need) {
    const long long t0 = globaltimer_ns();
    while (true) {
        int v;
        asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(win_done + w) : "memory");
        if (v >= need) return;
        if (globaltimer_ns() - t0 > 200000) return;   // 200 us: give up (e.g. not all workers co-resident)
        __nanosleep(256);
    }
}

// wgmma shared-memory descriptor of a K-major SWIZZLE_128B operand: rows of 128 B, 8-row groups 1024 B apart (SBO), one
// atom along K (LBO unused), layout type 1 = 128-byte swizzle.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024 >> 4) << 32) | (1ull << 62);
}

// Packed e2m1 cells -> int8 holding TWICE the cell value (0, 0.5, 1, 1.5, 2, 3, 4, 6 -> 0, 1, 2, 3, 4, 6, 8, 12; the sign
// bit negates), four cells (one 16-bit word, low nibble first) per call.  The Gram of the doubled cells is 4 S exactly.
__device__ __forceinline__ uint32_t e2m1x4_to_s8x2(uint32_t w) {
    const uint32_t mag = __byte_perm(0x03020100u, 0x0C080604u, w & 0x7777u);
    const uint32_t sgn = ((w >> 3) & 1u) | (((w >> 7) & 1u) << 8) | (((w >> 11) & 1u) << 16) | (((w >> 15) & 1u) << 24);
    const uint32_t m = sgn * 0xFFu;
    return (mag & ~m) | (__vneg4(mag) & m);
}

// Round-to-nearest-even of acc / 4 (the e2m1 path accumulates doubled cells), the rounding __float2int_rn gives.
__device__ __forceinline__ int quarter_rn(int acc) {
    const int q = acc >> 2, r = acc & 3;
    return q + ((r > 2 || (r == 2 && (q & 1))) ? 1 : 0);
}

// accumulator element: fp32 for bf16 operands, int32 (as its bit pattern) otherwise
template <int KIND>
using AccT = typename std::conditional<KIND == 1, float, uint32_t>::type;

template <int KIND>
__device__ __forceinline__ int acc_to_int(AccT<KIND> v) {
    if constexpr (KIND == 0) return (int)v;
    else if constexpr (KIND == 1) return __float2int_rn(v);
    else return quarter_rn((int)v);
}

// One CTA: warpgroup 0 produces (TMA), warpgroups 1 and 2 consume.  An output tile of one CTA is its A block (128 samples,
// the wgmma N side) times up to 256 B rows (the M side, 128 per consumer warpgroup = two m64 wgmmas); the accumulator
// stays in the consumers' registers, D[m][n] = sum_v X[rowB + m][v] X[rowA + n][v] = S[rowB + m][rowA + n], so that a
// thread's two adjacent accumulator columns are two adjacent int32 of one row of S (one 64-bit red).
template <int CG, int KIND>
__global__ void __launch_bounds__(kThreads, 1) gram_kernel(const __grid_constant__ CUtensorMap tmap, const GramArgs a) {
    using C = Cfg<KIND>;
    extern __shared__ uint8_t smem_raw[];
    // aligned in the shared window itself: a generic pointer of a cluster kernel carries the CTA's rank, and converting
    // one back to a shared address re-reads it (ptxas re-derived and spilled the base in every k-block)
    const uint32_t smem_base = (ptx::smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t bar_base = smem_base + C::STAGES * C::STAGE_BYTES + C::XBUF_BYTES * 2;
    // stage st: the B rows (M operand, 256 rows) then the A block (N operand, 128 rows), as TMA delivers them
    auto sB = [&](uint32_t st) { return smem_base + st * C::STAGE_BYTES; };
    auto sA = [&](uint32_t st) { return smem_base + st * C::STAGE_BYTES + C::B_BYTES; };
    auto full_bar = [&](uint32_t i) { return bar_base + 8u * i; };
    auto empty_bar = [&](uint32_t i) { return bar_base + 8u * (C::STAGES + i); };

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const uint32_t lane = ptx::lane_id();
    // CG == 2: the pair is a 2-CTA cluster of a 1-D grid, so its rank in the cluster is blockIdx.x & 1 (taken from
    // %ctaid: a rank read through inline asm from %cluster_ctarank was spilled and reloaded in every k-block)
    const uint32_t cta_rank = (CG == 2) ? (blockIdx.x & 1u) : 0u;
    const int worker = (CG == 2) ? (int)(blockIdx.x >> 1) : (int)blockIdx.x;
    // a consumer warpgroup frees a stage in its own CTA and, with CTA pairs, in the peer (whose producer multicasts into it)
    auto release = [&](uint32_t st) {
        if constexpr (CG == 2) {
            ptx::mbar_arrive_cluster(ptx::mapa(empty_bar(st), 0));
            ptx::mbar_arrive_cluster(ptx::mapa(empty_bar(st), 1));
        } else {
            ptx::mbar_arrive(empty_bar(st));
        }
    };

    if (warp == 0 && ptx::elect_one()) {
        ptx::prefetch_tensormap(&tmap);
        for (uint32_t i = 0; i < (uint32_t)C::STAGES; ++i) {
            ptx::mbar_init(full_bar(i), 1);         // producer's arrive.expect_tx
            ptx::mbar_init(empty_bar(i), 2 * CG);   // one arrive per consumer warpgroup of the cluster
        }
        ptx::fence_mbar_init();
    }
    // the peer's barriers must be initialised before the first multicast or remote arrive reaches them
    if constexpr (CG == 2) ptx::cluster_sync();
    else __syncthreads();
    if (a.prof != nullptr && threadIdx.x == 0) a.prof[(size_t)blockIdx.x * 4 + 0] = globaltimer_ns();

    if (warp < 4) {
        // ===================================== TMA producer =====================================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // registers go to the consumers' accumulators
        if (warp == 0 && ptx::elect_one()) {
            const bool leader = cta_rank == 0;
            Sched sc;
            sc.init(a, worker);
            Seg s;
            uint32_t it = 0;
            int synced_win = -1;
            while (sc.next(s)) {
                // CTA r of a pair multiplies its own A block.  Both CTAs walk every tile, filler tiles included, so that
                // their k-block sequences (and the stages the multicasts fill) stay in lockstep.
                const int rowA = (CG == 2 && cta_rank != 0) ? s.rowA1 : s.rowA0;
                const bool two_boxes = s.n_eff > kBoxRows;
                const bool self_b = (CG == 2) && (s.flags & kTileSelfB) != 0;   // the A block is half of the B rows
                const uint32_t tx = (uint32_t)((two_boxes ? 2 : 1) + (self_b ? 0 : 1)) * C::BOX_BYTES;
                if (a.sync_lead > 0 && leader && s.win != synced_win) {
                    synced_win = s.win;
                    if (s.win >= a.sync_lead) wait_window(a.win_done, s.win - a.sync_lead, a.active_workers);
                }
                for (int kb = s.kb0; kb < s.kb1; ++kb, ++it) {
                    const uint32_t st = it % C::STAGES, ph = (it / C::STAGES) & 1u;
                    mbar_wait(empty_bar(st), ph ^ 1u, a.err, 1);
                    const int pnl = kb / a.kb_per_panel;
                    const int kc = (kb - pnl * a.kb_per_panel) * a.kc_per_kb;
                    ptx::mbar_arrive_expect_tx(full_bar(st), tx);
                    if constexpr (CG == 2) {
                        // B box r is fetched once, by CTA r, into both CTAs (on a self-B tile it is CTA r's A block);
                        // the empty barrier waited on above counts the consumers of both CTAs
                        if (two_boxes || cta_rank == 0)
                            ptx::tma_load_3d_multicast(sB(st) + cta_rank * C::BOX_BYTES, &tmap, full_bar(st), kc,
                                                       s.rowB + (int)cta_rank * kBoxRows, pnl, 0x3);
                    } else {
                        ptx::tma_load_3d(sB(st), &tmap, full_bar(st), kc, s.rowB, pnl);
                        if (two_boxes) ptx::tma_load_3d(sB(st) + C::BOX_BYTES, &tmap, full_bar(st), kc, s.rowB + kBoxRows, pnl);
                    }
                    if (!self_b) ptx::tma_load_3d(sA(st), &tmap, full_bar(st), kc, rowA, pnl);
                }
                if (a.sync_lead > 0 && leader && s.last_in_win)
                    asm volatile("red.release.gpu.global.add.s32 [%0], 1;" ::"l"(a.win_done + s.win) : "memory");
            }
        }
    } else {
        // ===================================== consumers: wgmma + flush =====================================
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int cw = (warp >> 2) - 1;          // consumer warpgroup: B rows [128 cw, 128 cw + 128) of the tile
        const int wq = warp & 3;                 // warp within the warpgroup: accumulator rows 16 wq .. 16 wq + 15
        const uint32_t ctid = threadIdx.x - 128; // 0 .. 255 over both consumer warpgroups
        AccT<KIND> acc[2][64];
        Sched sc;
        sc.init(a, worker);
        Seg s;
        uint32_t it = 0;
        while (sc.next(s)) {
            // CTA 1's A block of a filler tile only pads the pair: multiplied in lockstep with CTA 0, never flushed
            const bool filler = (CG == 2) && cta_rank != 0 && (s.flags & kTileFiller) != 0;
            const bool self_b = (CG == 2) && (s.flags & kTileSelfB) != 0;
            // m64 blocks of this warpgroup that hold B rows of the tile (n_eff is a multiple of 16)
            const int mrow0 = cw * 128;
            const bool act0 = mrow0 < s.n_eff, act1 = mrow0 + 64 < s.n_eff;
            if (s.first) {
#pragma unroll
                for (int i = 0; i < 64; ++i) {
                    acc[0][i] = 0;
                    acc[1][i] = 0;
                }
            }
            // the A block follows the 256 B rows; on a self-B tile it is CTA r's half of them
            const uint32_t a_off = (self_b ? cta_rank : 2u) * (uint32_t)(kBoxRows * 128);
            int pending = -1;   // stage whose wgmmas may still be in flight
            for (int kb = s.kb0; kb < s.kb1; ++kb, ++it) {
                const uint32_t st = it % C::STAGES, ph = (it / C::STAGES) & 1u;
                mbar_wait(full_bar(st), ph, a.err, 3);
                uint32_t opB, opA;   // operand tiles in the 128-byte-swizzled int8 / bf16 layout wgmma reads
                if constexpr (KIND == 2) {
                    // packed e2m1 stage (64 bytes per row, unswizzled) -> doubled int8 cells in the swizzled layout of
                    // expansion buffer it % 2.  Its previous contents fed the wgmmas of k-block it - 2, which both
                    // warpgroups have waited for (wait_group 1 after issuing it - 1) before the first named barrier.
                    const uint32_t xb = smem_base + C::STAGES * C::STAGE_BYTES + (it & 1u) * C::XBUF_BYTES;
                    ptx::named_sync(1, 256);
                    const int nb = s.n_eff > kBoxRows ? 2 * kBoxRows : kBoxRows;   // B rows TMA delivered
                    const int rows = nb + (self_b ? 0 : kBoxRows);
                    for (int c = (int)ctid; c < rows * 8; c += 256) {   // 8 chunks of 8 packed bytes (16 cells) per row
                        const int r = c >> 3, j = c & 7;
                        // B row r -> expanded row r; A row r - nb -> expanded row 256 + r - nb (after the 256 B rows)
                        const uint32_t src = (r < nb ? sB(st) + (uint32_t)r * 64u : sA(st) + (uint32_t)(r - nb) * 64u) + (uint32_t)j * 8u;
                        const int xr = r < nb ? r : 2 * kBoxRows + (r - nb);
                        uint32_t lo, hi;
                        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(lo), "=r"(hi) : "r"(src));
                        const uint32_t o0 = e2m1x4_to_s8x2(lo & 0xFFFFu), o1 = e2m1x4_to_s8x2(lo >> 16);
                        const uint32_t o2 = e2m1x4_to_s8x2(hi & 0xFFFFu), o3 = e2m1x4_to_s8x2(hi >> 16);
                        const uint32_t dst = xb + (uint32_t)xr * 128u + (((uint32_t)j ^ ((uint32_t)xr & 7u)) << 4);
                        asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "r"(o0), "r"(o1), "r"(o2), "r"(o3)
                                     : "memory");
                    }
                    ptx::fence_proxy_async();   // generic-proxy stores -> visible to wgmma (async proxy)
                    ptx::named_sync(1, 256);
                    if (threadIdx.x % 128 == 0) release(st);   // the packed stage is free again
                    opB = xb;
                } else {
                    opB = sB(st);
                }
                opA = opB + a_off;
                const uint64_t bdesc = make_smem_desc(opA);
                const uint64_t adesc0 = make_smem_desc(opB + (uint32_t)mrow0 * 128u);
                const uint64_t adesc1 = make_smem_desc(opB + (uint32_t)(mrow0 + 64) * 128u);
                ptx::wgmma_fence_acc(acc[0]);
                ptx::wgmma_fence_acc(acc[1]);
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < kKBytes / 32; ++k) {   // 32 bytes of K per wgmma: +2 in the descriptor's 16-byte units
                    // both m64 blocks always (a branch would serialise the wgmmas); rows past n_eff are not flushed
                    if constexpr (KIND == 1) {
                        ptx::wgmma_bf16(acc[0], adesc0 + 2 * k, bdesc + 2 * k);
                        ptx::wgmma_bf16(acc[1], adesc1 + 2 * k, bdesc + 2 * k);
                    } else {
                        ptx::wgmma_s8(acc[0], adesc0 + 2 * k, bdesc + 2 * k);
                        ptx::wgmma_s8(acc[1], adesc1 + 2 * k, bdesc + 2 * k);
                    }
                }
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();   // the wgmmas of the previous k-block are done: release its stage
                ptx::wgmma_fence_acc(acc[0]);
                ptx::wgmma_fence_acc(acc[1]);
                if constexpr (KIND != 2) {
                    if (pending >= 0 && threadIdx.x % 128 == 0) release((uint32_t)pending);
                }
                pending = (int)st;
            }
            ptx::wgmma_wait<0>();
            ptx::wgmma_fence_acc(acc[0]);
            ptx::wgmma_fence_acc(acc[1]);
            if constexpr (KIND != 2) {
                if (pending >= 0 && threadIdx.x % 128 == 0) release((uint32_t)pending);
            }
            if (!s.flush || filler) continue;

            // ---- flush: S[row][col] += D, lower triangle only (or the transposed cell, exact block cover) ----
            const int colA = (CG == 2 && cta_rank != 0) ? s.rowA1 : s.rowA0;
            const int row_end = min(a.row_limit, s.rowB + s.n_eff);   // B rows this tile owns
            const bool pair64 = a.red64 != 0 && (a.n & 1) == 0;       // 8-byte aligned pairs of an even column
#pragma unroll
            for (int j = 0; j < 2; ++j) {
                if (!(j == 0 ? act0 : act1)) continue;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = s.rowB + mrow0 + 64 * j + 16 * wq + (int)(lane >> 2) + 8 * h;
                    if (row >= row_end) continue;
                    int32_t* own = a.S;   // owner-rows mode: the Gram of the rank that owns this row
                    if (a.num_peers != 0 && a.peer_mode == 1) {
                        int o = 0;
                        while (o + 1 < a.num_peers && row >= a.own_end[o]) ++o;
                        own = a.peer[o];
                    }
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const int col = colA + 8 * i + 2 * (int)(lane & 3);
                        if (col >= a.n) continue;
                        int v0 = acc_to_int<KIND>(acc[j][4 * i + 2 * h]);
                        int v1 = acc_to_int<KIND>(acc[j][4 * i + 2 * h + 1]);
                        if ((s.flags & kTileXpose) != 0 && (row >> 7) < (col >> 7)) {
                            // a 128-block above the diagonal computed in place of its mirror image: S[col][row] (a pair of
                            // even columns never straddles a block edge)
                            for (int e = 0; e < 2; ++e) {
                                const int v = e ? v1 : v0, c = col + e;
                                if (v == 0 || c >= a.n) continue;
                                const size_t o = (size_t)c * (size_t)a.n + (size_t)row;
                                if (a.num_peers == 0) {
                                    asm volatile("red.global.add.s32 [%0], %1;" ::"l"(a.S + o), "r"(v) : "memory");
                                } else if (a.peer_mode == 1) {
                                    int q = 0;
                                    while (q + 1 < a.num_peers && c >= a.own_end[q]) ++q;
                                    asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(a.peer[q] + o), "r"(v) : "memory");
                                } else {
                                    for (int d = 0; d < a.num_peers; ++d)
                                        asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(a.peer[d] + o), "r"(v)
                                                     : "memory");
                                }
                            }
                            continue;
                        }
                        if (row < col) v0 = 0;
                        if (row < col + 1 || col + 1 >= a.n) v1 = 0;
                        if ((v0 | v1) == 0) continue;
                        const size_t o = (size_t)row * (size_t)a.n + (size_t)col;
                        if (pair64) {
                            // two cells per atomic: counts are non-negative and every sum stays below 2^31, so a 64-bit
                            // add of (cell c | cell c + 1 << 32) never carries between the halves
                            const unsigned long long packed = (unsigned long long)(unsigned)v0 | ((unsigned long long)(unsigned)v1 << 32);
                            if (a.num_peers == 0) {
                                asm volatile("red.global.add.u64 [%0], %1;" ::"l"(a.S + o), "l"(packed) : "memory");
                            } else if (a.peer_mode == 1) {
                                asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(own + o), "l"(packed) : "memory");
                            } else {
                                for (int d = 0; d < a.num_peers; ++d)
                                    asm volatile("red.relaxed.sys.global.add.u64 [%0], %1;" ::"l"(a.peer[d] + o), "l"(packed)
                                                 : "memory");
                            }
                        } else {
                            for (int e = 0; e < 2; ++e) {
                                const int v = e ? v1 : v0;
                                if (v == 0) continue;
                                if (a.num_peers == 0) {
                                    asm volatile("red.global.add.s32 [%0], %1;" ::"l"(a.S + o + e), "r"(v) : "memory");
                                } else if (a.peer_mode == 1) {
                                    asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(own + o + e), "r"(v) : "memory");
                                } else {
                                    for (int d = 0; d < a.num_peers; ++d)
                                        asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(a.peer[d] + o + e), "r"(v)
                                                     : "memory");
                                }
                            }
                        }
                    }
                }
            }
        }
        if (a.prof != nullptr && threadIdx.x == 128) a.prof[(size_t)blockIdx.x * 4 + 2] = globaltimer_ns();
    }

    // no CTA of a pair exits while its peer may still arrive on its barriers
    if constexpr (CG == 2) ptx::cluster_sync();
    else __syncthreads();
    if (a.prof != nullptr && threadIdx.x == 0) a.prof[(size_t)blockIdx.x * 4 + 3] = globaltimer_ns();
}

// ---------------------------------------------------------------------------------------------------
// Adaptive stream-K split.  Workers need not all run at the same speed (the SMs of different GPCs may get different
// shares of the L2 -> SM bandwidth the operand loads run against), and an equal split waits for the slowest worker.  After every sufficiently long launch this kernel turns the
// per-worker timestamps into speeds (units / time) and moves the shares of the next launch towards them.  The Gram
// stays exact whatever the split is (integer atomics); shares are clamped so that a worker never spans more than
// the tile its accumulator holds.
__global__ void rebalance_kernel(const long long* __restrict__ prof, double* __restrict__ cum, int workers, int cta_group,
                                 double gain, double max_share, long long min_ns, int* __restrict__ gen, const TileDesc* __restrict__ tiles,
                                 int num_tiles, int total_weight, int kbw, int col_limit) {
    __shared__ double sh[1024];
    __shared__ double cand[1025];
    __shared__ long long need[1025];
    __shared__ double red_sum, red_min;
    __shared__ int reject, need_repair;
    const int w = threadIdx.x;
    const bool active = w < workers;
    double t = 0.0, share_old = 0.0;
    if (active) {
        const long long t0 = prof[(size_t)w * cta_group * 4 + 0], t1 = prof[(size_t)w * cta_group * 4 + 2];
        t = (double)(t1 - t0);
        share_old = cum[w + 1] - cum[w];
    }
    sh[w] = active ? t : 1e30;
    if (w == 0) {
        reject = 0;
        need_repair = 0;
    }
    __syncthreads();
    if (w == 0) {
        double mn = 1e30, mx = 0.0;
        for (int i = 0; i < workers; ++i) {
            mn = fmin(mn, sh[i]);
            mx = fmax(mx, sh[i]);
        }
        // too short to time, or already balanced to within 3 %: keep the shares (hysteresis against noise)
        red_min = (mn < (double)min_ns || (mx - mn) < 0.03 * mx) ? -1.0 : mn;
    }
    __syncthreads();
    if (red_min < 0.0) return;
    const double speed = active ? share_old / t : 0.0;
    sh[w] = speed;
    __syncthreads();
    if (w == 0) {
        double sum = 0.0;
        for (int i = 0; i < workers; ++i) sum += sh[i];
        red_sum = sum;
    }
    __syncthreads();
    double share = 0.0;
    if (active) {
        const double est = speed / red_sum;
        share = (1.0 - gain) * share_old + gain * est;
        const double avg = 1.0 / workers;
        share = fmin(fmax(share, 0.5 * avg), max_share * avg);
    }
    __syncthreads();
    sh[w] = share;
    __syncthreads();
    if (w == 0) {
        double sum = 0.0;
        for (int i = 0; i < workers; ++i) sum += sh[i];
        double acc = 0.0;
        cand[0] = 0.0;
        for (int i = 0; i < workers; ++i) {
            acc += sh[i] / sum;
            cand[i + 1] = (i + 1 == workers) ? 1.0 : acc;
        }
    }
    __syncthreads();
    // Repair, then publish: a worker whose pieces under the candidate split would not fit its accumulator budget (more than kMaxSegs
    // accumulators or more than col_limit columns: e.g. the tail of one tile, a whole 13-unit tile and the head of a
    // third) stops at the edge of the tile that does not fit, and its neighbour starts there.  One thread walks the
    // workers in order; the tile cursor only moves forward, so the walk is O(workers + tiles).
    // common case: every worker's pieces fit under the candidate as it is -- checked by all workers in parallel; only
    // when one does not, one thread walks the workers in order and repairs (tens of microseconds: kept off the usual path)
    if (active) {
        const long long uw = (long long)total_weight * kbw;
        const long long ub = (long long)((double)uw * cand[w]);
        const long long ue = (w + 1 == workers) ? uw : (long long)((double)uw * cand[w + 1]);
        int hint = 0;
        if (feasible_end(tiles, num_tiles, ub, ue, kbw, col_limit, hint) < ue) atomicExch(&need_repair, 1);
    }
    __syncthreads();
    if (need_repair && w == 0 && !repair_split(tiles, num_tiles, workers, (long long)total_weight * kbw, kbw, col_limit, cand, need)) reject = 1;
    __syncthreads();
    if (reject) return;
    if (w <= workers) cum[w] = cand[w];
    if (w == 0) *gen += 1;
}

// The front/tail schedule's counterpart: moves the split point s so that the slowest front worker (s k-blocks, one
// flush) and the slowest tail worker (T (K - s) / (W - T) k-blocks, a flush per piece, its own L2 traffic) finish
// together.  Each side's time is taken as proportional to its k-blocks, so the fixed point is where both finish
// together, whatever the tail's flushes cost.  *frac stays within [lo, hi].
__global__ void rebalance_front_kernel(const long long* __restrict__ prof, double* __restrict__ frac, int front, int workers,
                                       int cta_group, int kb_total, double gain, double lo, double hi, long long min_ns,
                                       int* __restrict__ gen) {
    __shared__ long long tmax[2][32];
    const int w = threadIdx.x;
    long long t = 0;
    if (w < workers) t = prof[(size_t)w * cta_group * 4 + 2] - prof[(size_t)w * cta_group * 4 + 0];
    const int side = w < front ? 0 : 1;
    // per-side max: a warp's lanes may straddle the two sides, so reduce each side with the other side's lanes at 0
    long long m0 = side == 0 ? t : 0, m1 = side == 1 ? t : 0;
    for (int o = 16; o > 0; o >>= 1) {
        m0 = max(m0, __shfl_xor_sync(0xffffffffu, m0, o));
        m1 = max(m1, __shfl_xor_sync(0xffffffffu, m1, o));
    }
    if ((w & 31) == 0) {
        tmax[0][w >> 5] = m0;
        tmax[1][w >> 5] = m1;
    }
    __syncthreads();
    if (w != 0) return;
    long long tf = 0, tt = 0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) {
        tf = max(tf, tmax[0][i]);
        tt = max(tt, tmax[1][i]);
    }
    const double f = *frac;
    const int s = front_split(f, kb_total);
    if (s <= 0 || s >= kb_total) return;                  // one side did no work: nothing to compare
    if (tf < min_ns || tt < min_ns) return;                // too short to time
    if (llabs(tf - tt) < (max(tf, tt) >> 8)) return;       // balanced to within 0.4 %: keep s (hysteresis against noise)
    const double a = (double)tf / (double)s, b = (double)tt / (double)(kb_total - s);   // ns per k-block of each side
    const double target = b / (a + b);                     // a s = b (K - s)
    const double nf = fmin(fmax((1.0 - gain) * f + gain * target, lo), hi);
    *frac = nf;
    *gen += 1;
}

__global__ void symmetrize_kernel(int32_t* __restrict__ S, int n) {
    // block (bx >= by): read lower tile (bx, by), write it transposed into the upper tile (by, bx)
    __shared__ int32_t tile[32][33];
    const int bx = blockIdx.x, by = blockIdx.y;
    if (bx < by) return;
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    for (int r = ty; r < 32; r += 8) {
        const int row = bx * 32 + r, col = by * 32 + tx;
        tile[r][tx] = (row < n && col < n) ? S[(size_t)row * n + col] : 0;
    }
    __syncthreads();
    for (int r = ty; r < 32; r += 8) {
        const int row = by * 32 + r, col = bx * 32 + tx;   // target (upper)
        if (row < n && col < n && row < col) S[(size_t)row * n + col] = tile[tx][r];
    }
}

__global__ void add_i32_kernel(int32_t* __restrict__ dst, const int32_t* __restrict__ src, int64_t count) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) dst[i] += src[i];
}

struct PeerPtrs {
    int32_t* p[kMaxPeers];
};

__global__ void add_i32_peers_kernel(PeerPtrs dst, int npeers, const int32_t* __restrict__ src, int64_t count) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (; i < count; i += stride) {
        const int v = src[i];
        if (v != 0)
            for (int d = 0; d < npeers; ++d)
                asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(dst.p[d] + i), "r"(v) : "memory");
    }
}

struct OwnEnds {
    int e[kMaxPeers];
};

__device__ __forceinline__ int owner_of_row(const OwnEnds& own, int npeers, int row) {
    int q = 0;
    while (q + 1 < npeers && row >= own.e[q]) ++q;
    return q;
}

// Staged partition -> owners: element (row, col) of the lower triangle is added into the Gram of the row's owner.
__global__ void add_i32_owner_kernel(PeerPtrs dst, OwnEnds own, int npeers, const int32_t* __restrict__ src, int n) {
    for (int row = blockIdx.x; row < n; row += gridDim.x) {
        int32_t* d = dst.p[owner_of_row(own, npeers, row)] + (size_t)row * n;
        const int32_t* s = src + (size_t)row * n;
        for (int c = threadIdx.x; c <= row; c += blockDim.x) {
            const int v = s[c];
            if (v != 0) asm volatile("red.relaxed.sys.global.add.s32 [%0], %1;" ::"l"(d + c), "r"(v) : "memory");
        }
    }
}

// All-gather after the reduce-scatter: every rank pulls the lower-triangle part of the rows it does not own from the
// owner's Gram (peer loads over NVLink, 16-byte when the row pitch allows).
__global__ void __launch_bounds__(256) gather_rows_kernel(PeerPtrs src, int32_t* __restrict__ dst, OwnEnds own, int npeers,
                                                          int rank, int n) {
    const bool vec = (n & 3) == 0;
    for (int row = blockIdx.x; row < n; row += gridDim.x) {
        const int q = owner_of_row(own, npeers, row);
        if (q == rank) continue;
        const int32_t* s = src.p[q] + (size_t)row * n;
        int32_t* d = dst + (size_t)row * n;
        if (vec) {
            const int4* s4 = reinterpret_cast<const int4*>(s);
            int4* d4 = reinterpret_cast<int4*>(d);
            for (int c = threadIdx.x; c < (row + 4) / 4; c += blockDim.x) d4[c] = s4[c];   // up to 3 cells past the diagonal: zeros
        } else {
            for (int c = threadIdx.x; c <= row; c += blockDim.x) d[c] = s[c];
        }
    }
}

// The same all-gather as posted writes: every rank pushes the lower-triangle part of the rows it owns into the Gram of
// every other rank (remote stores are fire-and-forget; remote loads pay a NVLink round trip each).
__global__ void __launch_bounds__(256) push_rows_kernel(PeerPtrs dst, const int32_t* __restrict__ src, OwnEnds own,
                                                        int npeers, int rank, int n) {
    const bool vec = (n & 3) == 0;
    const int row_lo = rank == 0 ? 0 : own.e[rank - 1], row_hi = own.e[rank];
    for (int row = row_lo + blockIdx.x; row < row_hi; row += gridDim.x) {
        const int32_t* s = src + (size_t)row * n;
        if (vec) {
            const int4* s4 = reinterpret_cast<const int4*>(s);
            for (int c = threadIdx.x; c < (row + 4) / 4; c += blockDim.x) {
                const int4 v = s4[c];
                for (int d = 0; d < npeers; ++d)
                    if (d != rank) reinterpret_cast<int4*>(dst.p[d] + (size_t)row * n)[c] = v;
            }
        } else {
            for (int c = threadIdx.x; c <= row; c += blockDim.x) {
                const int v = s[c];
                for (int d = 0; d < npeers; ++d)
                    if (d != rank) dst.p[d][(size_t)row * n + c] = v;
            }
        }
    }
}

// All-rank barrier over peer-mapped flag words: rank r publishes `epoch` in slot r of every rank's flag array, then
// waits until every slot of its own array shows it.  One thread per peer.
__global__ void peer_barrier_kernel(PeerPtrs flags, int npeers, int rank, int epoch) {
    const int d = threadIdx.x;
    if (d < npeers) {
        __threadfence_system();
        asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(flags.p[d] + rank), "r"(epoch) : "memory");
        int v;
        const long long t0 = globaltimer_ns();
        do {
            asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(flags.p[rank] + d) : "memory");
            // a peer that died or never reached the barrier must surface as an error, not hang the box
            if (v < epoch && globaltimer_ns() - t0 > 30000000000LL) __trap();
        } while (v < epoch);
    }
    __syncthreads();
    __threadfence_system();
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
    }
    return fn;
}

template <int CG, int KIND>
cudaError_t launch(const CUtensorMap& tmap, const GramArgs& args, int grid, cudaStream_t stream) {
    using C = Cfg<KIND>;
    // per launch, not cached: the attribute is per device and one process may drive several GPUs
    cudaError_t ea = cudaFuncSetAttribute(gram_kernel<CG, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES);
    if (ea != cudaSuccess) return ea;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = C::SMEM_BYTES;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    if (CG == 2) {   // the two CTAs of a worker form a cluster (TMA multicast of the B rows they share)
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = 2;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
    }
    return cudaLaunchKernelEx(&cfg, gram_kernel<CG, KIND>, tmap, args);
}

// How many clusters of `cluster_size` CTAs of gram_kernel<2, KIND> (1 CTA per SM: ~200 KB of shared memory each) the
// current device can hold at once; -1 if the query fails.
template <int KIND>
int max_clusters(int cluster_size) {
    using C = Cfg<KIND>;
    if (cudaFuncSetAttribute(gram_kernel<2, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::SMEM_BYTES) != cudaSuccess)
        return -1;
    if (cluster_size > 8 &&
        cudaFuncSetAttribute(gram_kernel<2, KIND>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) return -1;
    int sms = 0, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)(sms / cluster_size * cluster_size));
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = C::SMEM_BYTES;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cluster_size;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    if (cudaOccupancyMaxActiveClusters(&clusters, gram_kernel<2, KIND>, &cfg) != cudaSuccess) {
        cudaGetLastError();
        return -1;
    }
    return clusters;
}

}  // namespace

// Process-wide memory of the speed-weighted splits the rebalancer converged to: the per-worker speeds it measures are a
// property of the device (which SMs get how much L2 bandwidth), so a new context for the same (device, cohort size, tile
// list, window) starts from the split the last one ended with instead of relearning it over its first launches.
namespace {
struct SplitKey {
    int dev, n, tiles, kbw, workers, elem;
    bool operator<(const SplitKey& o) const {
        return std::tie(dev, n, tiles, kbw, workers, elem) < std::tie(o.dev, o.n, o.tiles, o.kbw, o.workers, o.elem);
    }
};
std::mutex g_split_mu;
std::map<SplitKey, std::vector<double>> g_splits;
}  // namespace

static void remember_split(GramPlan& plan) {
    if (plan.d_cum.get() == nullptr || plan.cum_workers <= 0 || !plan.adaptive) return;
    if (plan.own_hi > plan.own_lo && plan.num_peers <= 1) return;   // a band's tile list is not the cohort's
    std::vector<double> cum((size_t)plan.cum_workers + 2);   // the split and the front/tail split point
    if (cudaMemcpy(cum.data(), plan.d_cum.get(), cum.size() * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) {
        cudaGetLastError();
        return;
    }
    std::lock_guard<std::mutex> lk(g_split_mu);
    g_splits[SplitKey{plan.cum_dev, plan.cum_for_n, plan.cum_tiles, plan.cum_kbw, plan.cum_workers, plan.cum_elem}] = std::move(cum);
}

void gram_plan_free(GramPlan& plan) {
    remember_split(plan);
    plan.h_tiles.clear();
    if (plan.d_err) cudaFreeHost(plan.d_err);
    plan.d_err = nullptr;
    plan.tiles_for_n = -1;
}

int gram_read_profile(GramPlan& plan, long long* out, int max_ctas) {
    if (plan.d_prof.get() == nullptr) return 0;
    const int ctas = std::min(max_ctas, std::min(1024, plan.num_sms));
    if (cudaMemcpy(out, plan.d_prof.get(), (size_t)ctas * 4 * sizeof(long long), cudaMemcpyDeviceToHost) != cudaSuccess) return 0;
    return ctas;
}

// Tile list of the lower triangle of S.
//   exact == false: BM x BN rectangles that touch row >= col, in strips of 8 row blocks walked column by
//     column, so that a run of ~num_sms / 2 consecutive tiles (one wave of the large-N schedule) is a compact patch of S.
//   exact == true: the exact block cover.  Units: 128 x 128 blocks (col block c, row block r), needed iff c <= r.  A tile
//     multiplies `cg` A (column) blocks -- any blocks, one per CTA -- with one or two adjacent B (row) blocks.  With
//     CTA pairs a tile holds an even number of blocks of every row it touches, but row r needs r + 1 of them, so for
//     r = 4t the block (col 4t, row 4t + 2) is taken out of row 4t + 2 and computed in row 4t as its mirror image
//     (col 4t + 2, row 4t), written transposed: both rows become even and every needed block is covered exactly once.
//     Two-row tiles come first, one-row tiles last.
static void make_tiles(int n, int cg, bool exact, int bn, int row_lo, int row_hi, bool self_b, std::vector<TileDesc>& out,
                       int* num_full) {
    // [row_lo, row_hi): the rows of S to produce (the whole triangle, or the band an owner-computes context stores)
    out.clear();
    auto n_eff = [&](int row0, int want) { return std::min(want, ((n - row0) + 15) & ~15); };
    if (!exact) {
        // B strips of nearly equal width: ceil(n / 16) units of 16 rows dealt over ceil(n / bn) strips (2504 samples,
        // bn = 256: 7 strips of 256 rows and 3 of 240 instead of 9 of 256 and one of 200).  Tiles of nearly equal
        // weight keep the pieces of an even split close to one worker's one-tile accumulator budget.
        const int BM = 128 * cg;
        const int span = row_hi - row_lo;
        const int nbn = (span + bn - 1) / bn, nbm = (n + BM - 1) / BM;
        const int units = (span + 15) / 16;
        std::vector<int> row0(nbn + 1, row_lo);
        for (int b = 0; b < nbn; ++b) row0[b + 1] = row0[b] + 16 * (units / nbn + (b < units % nbn ? 1 : 0));
        constexpr int kStrip = 8;
        for (int bb = 0; bb < nbn; bb += kStrip)
            for (int am = 0; am < nbm; ++am)
                for (int b = bb; b < std::min(nbn, bb + kStrip); ++b) {
                    const int max_row = std::min(row_hi, row0[b + 1]) - 1;
                    if (am * BM > max_row) continue;   // wholly above the diagonal
                    TileDesc t{};
                    t.rowA0 = am * BM;
                    t.rowA1 = am * BM + 128;
                    t.rowB = row0[b];
                    t.n_eff = std::min(row0[b + 1], ((row_hi + 15) & ~15)) - row0[b];
                    t.acc_cols = bn;
                    // diagonal tile whose 256 B rows are exactly the two A blocks of the pair: CTA r's half of B is its own
                    // A block, so the MMA reads B through the A tile and the producer loads nothing for B (half the
                    // L2 -> SM bytes of the tile)
                    if (self_b && cg == 2 && t.rowB == t.rowA0 && t.n_eff == 2 * 128) t.flags |= kTileSelfB;
                    out.push_back(t);
                }
    } else {
        const int nb = (n + 127) / 128;
        std::vector<TileDesc> two, one;
        auto emit = [&](std::vector<TileDesc>& dst, int c0, int c1, int r0, int rows, bool filler) {
            TileDesc t{};
            t.rowA0 = c0 * 128;
            t.rowA1 = c1 * 128;
            t.rowB = r0 * 128;
            t.n_eff = n_eff(r0 * 128, rows * 128);
            t.acc_cols = kAccCols;
            t.flags = kTileXpose | (filler ? kTileFiller : 0);
            dst.push_back(t);
        };
        // column blocks each row block needs (a value > the row index = the mirror image of a block of a later row)
        std::vector<std::vector<int>> need(nb);
        for (int r = 0; r < nb; ++r)
            for (int c = 0; c <= r; ++c) need[r].push_back(c);
        if (cg == 2)
            for (int r = 0; r + 2 < nb; r += 4) {
                need[r].push_back(r + 2);                                        // (col r + 2, row r): transposed
                need[r + 2].erase(std::find(need[r + 2].begin(), need[r + 2].end(), r));
            }
        for (int r0 = 0; r0 < nb; r0 += 2) {
            const bool pair = r0 + 1 < nb;
            std::vector<int> common, left0, left1;
            if (pair) {
                for (int c : need[r0])
                    if (std::find(need[r0 + 1].begin(), need[r0 + 1].end(), c) != need[r0 + 1].end()) common.push_back(c);
                if (cg == 2 && (common.size() & 1)) common.pop_back();          // an odd one out joins the one-row tiles
            }
            for (int c : need[r0])
                if (std::find(common.begin(), common.end(), c) == common.end()) left0.push_back(c);
            if (pair)
                for (int c : need[r0 + 1])
                    if (std::find(common.begin(), common.end(), c) == common.end()) left1.push_back(c);
            for (size_t i = 0; i < common.size(); i += cg) emit(two, common[i], common[cg == 2 ? i + 1 : i], r0, 2, false);
            for (int side = 0; side < (pair ? 2 : 1); ++side) {
                const std::vector<int>& left = side == 0 ? left0 : left1;
                for (size_t i = 0; i < left.size(); i += cg) {
                    const bool filler = cg == 2 && i + 1 >= left.size();
                    emit(one, left[i], filler ? left[i] : left[cg == 2 ? i + 1 : i], r0 + side, 1, filler);
                }
            }
        }
        // large-N schedule: whole-tile waves want equal tiles that share row panels of X -- the full-weight two-row
        // tiles go in front, in strips of 8 row blocks walked column pair by column pair (a wave of one tile per
        // worker -- 66 consecutive tiles on 132 SMs -- is then a compact patch of S that needs ~34 row blocks of X instead
        // of ~150)
        auto mid = std::stable_partition(two.begin(), two.end(), [&](const TileDesc& t) { return t.n_eff == 256; });
        std::stable_sort(two.begin(), mid, [](const TileDesc& x, const TileDesc& y) {
            const int sx = x.rowB / 1024, sy = y.rowB / 1024;
            if (sx != sy) return sx < sy;
            const int cx = std::min(x.rowA0, x.rowA1) / 256, cy = std::min(y.rowA0, y.rowA1) / 256;
            if (cx != cy) return cx < cy;
            return x.rowB < y.rowB;
        });
        *num_full = (int)(mid - two.begin());
        out = two;
        out.insert(out.end(), one.begin(), one.end());
    }
    if (!exact) *num_full = (int)out.size();   // the rectangles go out in whole-tile waves whatever their edge trim
    int w = 0;
    for (auto& t : out) {
        t.wstart = w;
        w += t.n_eff >> 4;
    }
}

static cudaError_t build_tiles(GramPlan& plan, int n, bool exact, int BN, int row_lo, int row_hi, cudaStream_t stream) {
    std::vector<TileDesc> tiles;
    int num_full = 0;
    make_tiles(n, plan.cta_group, exact, BN, row_lo, row_hi, plan.self_b, tiles, &num_full);
    plan.d_tiles.reset();
    cudaError_t e = plan.d_tiles.ensure((int64_t)(tiles.size() * sizeof(TileDesc)));
    if (e != cudaSuccess) return e;
    e = cudaMemcpyAsync(plan.d_tiles.get(), tiles.data(), tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice, stream);
    if (e != cudaSuccess) return e;
    e = cudaStreamSynchronize(stream);   // `tiles` is a stack vector
    plan.h_tiles.assign(reinterpret_cast<const int32_t*>(tiles.data()),
                        reinterpret_cast<const int32_t*>(tiles.data() + tiles.size()));
    plan.num_tiles = (int)tiles.size();
    plan.num_full = num_full;
    plan.total_weight = tiles.empty() ? 0 : tiles.back().wstart + (tiles.back().n_eff >> 4);
    plan.tiles_for_n = n;
    plan.tiles_for_cg = plan.cta_group;
    plan.tiles_for_bn = exact ? -1 : BN;
    plan.tiles_row_lo = row_lo;
    plan.tiles_row_hi = row_hi;
    plan.tiles_col_limit = kAccCols;
    return e;
}

// Whether a launch takes the front/tail schedule, and its split point as a fraction of K: initially T / W, the balance
// when a k-block costs the same on both sides; the adaptation keeps it within half the distance to either end.
// Owner-computes bands keep the within-window split.
struct FrontRange {
    bool on = false;
    double init = 0.0, lo = 0.0, hi = 0.0;
};

static FrontRange front_range(int num_tiles, int workers, bool banded) {
    FrontRange r;
    r.on = !banded && front_tail_applies(num_tiles, workers);
    if (r.on) {
        r.init = (double)num_tiles / (double)workers;
        r.lo = 0.5 * r.init;
        r.hi = r.init + 0.5 * (1.0 - r.init);
    }
    return r;
}

// Resident schedule (accumulators stay in registers for the whole launch) iff the equal split of a window of `kbw`
// k-blocks, after the same repair the rebalancer applies (a worker stops at the edge of a tile whose accumulator would not
// fit any more), lets every worker keep its pieces in its accumulator budget.  `cum` receives that initial split
// (workers + 1 fractions).
static bool initial_split(const GramPlan& plan, int workers, int kbw, std::vector<double>& cum) {
    if (plan.total_weight <= 0) return false;
    const TileDesc* tiles = reinterpret_cast<const TileDesc*>(plan.h_tiles.data());
    const long long uw = (long long)plan.total_weight * kbw;
    cum.resize((size_t)workers + 1);
    for (int w = 0; w <= workers; ++w) cum[w] = (double)w / (double)workers;
    std::vector<long long> need((size_t)workers + 1);
    if (!repair_split(tiles, plan.num_tiles, workers, uw, kbw, plan.tiles_col_limit, cum.data(), need.data())) return false;
    for (int w = 0; w < workers; ++w) {   // belt and braces: what the kernel will plan from these fractions must fit
        const long long ub = (long long)((double)uw * cum[w]);
        const long long ue = (w + 1 == workers) ? uw : (long long)((double)uw * cum[w + 1]);
        SegPlan p;
        plan_segments(tiles, plan.num_tiles, 0, ub, ue, kbw, p);
        if (p.overflow || p.cols > plan.tiles_col_limit) return false;
    }
    return true;
}

// Host-only introspection of the schedule (no device needed): the tile list for n samples, and the pieces
// (tile, k-block range, accumulator column) each worker owns in a window of `kbw` k-blocks under an equal split.
int gram_debug_tiles(int n, int cta_group, int exact, int32_t* out, int max_tiles) {
    std::vector<TileDesc> tiles;
    int num_full = 0;
    make_tiles(n, cta_group == 1 ? 1 : 2, exact != 0, kUmmaN, 0, n, true, tiles, &num_full);
    const int cnt = std::min<int>((int)tiles.size(), max_tiles);
    if (out != nullptr && cnt > 0) memcpy(out, tiles.data(), (size_t)cnt * sizeof(TileDesc));
    return (int)tiles.size();
}

int gram_debug_band_tiles(int n, int cta_group, int row_lo, int row_hi, int32_t* out, int max_tiles) {
    std::vector<TileDesc> tiles;
    int num_full = 0;
    make_tiles(n, cta_group == 1 ? 1 : 2, false, kUmmaN, row_lo, row_hi, true, tiles, &num_full);
    const int cnt = std::min<int>((int)tiles.size(), max_tiles);
    if (out != nullptr && cnt > 0) memcpy(out, tiles.data(), (size_t)cnt * sizeof(TileDesc));
    return (int)tiles.size();
}

int gram_debug_plan(const int32_t* tiles8, int num_tiles, int workers, int kbw, int32_t* out, int max_pieces) {
    // the split a first launch uses: equal shares, repaired like initial_split does
    if (num_tiles <= 0) return 0;
    const int col_limit = kAccCols;
    std::vector<double> cum((size_t)workers + 1);
    for (int w = 0; w <= workers; ++w) cum[w] = (double)w / (double)workers;
    return gram_debug_repair(tiles8, num_tiles, workers, kbw, col_limit, cum.data(), out, max_pieces);
}

// Host-only: the rebalancer's repair step on a caller-supplied split (cum: workers + 1 fractions, in / out) followed by
// the plan it yields, in the same format as gram_debug_plan.  -1000: no feasible repair.
int gram_debug_repair(const int32_t* tiles8, int num_tiles, int workers, int kbw, int col_limit, double* cum, int32_t* out,
                      int max_pieces) {
    const TileDesc* tiles = reinterpret_cast<const TileDesc*>(tiles8);
    if (num_tiles <= 0) return 0;
    const long long total = tiles[num_tiles - 1].wstart + (tiles[num_tiles - 1].n_eff >> 4);
    const long long uw = total * kbw;
    std::vector<long long> need((size_t)workers + 1);
    if (!repair_split(tiles, num_tiles, workers, uw, kbw, col_limit, cum, need.data())) return -1000;
    int cnt = 0;
    for (int w = 0; w < workers; ++w) {
        const long long ub = (long long)((double)uw * cum[w]);
        const long long ue = (w + 1 == workers) ? uw : (long long)((double)uw * cum[w + 1]);
        SegPlan p;
        plan_segments(tiles, num_tiles, 0, ub, ue, kbw, p);
        if (p.overflow || p.cols > col_limit) return -1 - w;
        for (int i = 0; i < p.n; ++i, ++cnt)
            if (cnt < max_pieces) {
                int32_t* o = out + (size_t)cnt * 6;
                o[0] = w; o[1] = p.tile[i]; o[2] = p.lo[i]; o[3] = p.hi[i]; o[4] = p.col[i]; o[5] = p.cols;
            }
    }
    return cnt;
}

// Host-only: every piece each worker of a launch replays, in launch order, under the schedule gram_accumulate picks for a
// whole-cohort context (no band) with the initial split.  frac >= 0 sets the front/tail split point instead of T / W.
// info: {schedule (0 waves, 1 resident, 2 front/tail), split point s (kb_total unless front/tail)}.
int gram_debug_schedule(int n, int cta_group, int exact, int workers, int kbw, int kb_total, double frac, int32_t* out,
                        int max_pieces, int32_t* info) {
    GramPlan plan;
    plan.cta_group = cta_group == 1 ? 1 : 2;
    std::vector<TileDesc> tiles;
    int num_full = 0;
    make_tiles(n, plan.cta_group, exact != 0, kUmmaN, 0, n, true, tiles, &num_full);
    plan.h_tiles.assign(reinterpret_cast<const int32_t*>(tiles.data()), reinterpret_cast<const int32_t*>(tiles.data() + tiles.size()));
    plan.num_tiles = (int)tiles.size();
    plan.num_full = num_full;
    plan.total_weight = tiles.back().wstart + (tiles.back().n_eff >> 4);
    kbw = std::min(kbw, kb_total);
    std::vector<double> cum;
    const FrontRange front = front_range(plan.num_tiles, workers, false);
    GramArgs a{};
    a.tiles = tiles.data();
    a.n = n;
    a.num_tiles = plan.num_tiles;
    a.num_full = num_full;
    a.total_weight = plan.total_weight;
    a.kb_total = kb_total;
    a.num_workers = workers;
    a.col_limit = plan.tiles_col_limit;
    a.resident = front.on || (plan.num_tiles <= 4 * workers && initial_split(plan, workers, kbw, cum)) ? 1 : 0;
    a.kb_window = a.resident ? kbw : kb_total;
    a.cum = cum.data();
    const double f = frac >= 0.0 ? frac : front.init;
    if (front.on) {
        a.front_tiles = plan.num_tiles;
        a.front_frac = &f;
    }
    info[0] = front.on ? 2 : a.resident;
    info[1] = front.on ? front_split(f, kb_total) : kb_total;
    int cnt = 0;
    for (int w = 0; w < workers; ++w) {
        Sched sc;
        if (!sc.init(a, w)) return -1 - w;
        Seg s;
        for (; sc.next(s); ++cnt)
            if (cnt < max_pieces) {
                int32_t* o = out + (size_t)cnt * 6;
                o[0] = w; o[1] = s.tile; o[2] = s.kb0; o[3] = s.kb1; o[4] = s.first; o[5] = s.flush;
            }
    }
    return cnt;
}

cudaError_t gram_accumulate(GramPlan& plan, const void* d_x, int elem_bits, int n, int64_t nv, int64_t ld, int64_t panel,
                            int32_t* d_S, cudaStream_t stream, std::string* err) {
    if (nv <= 0) return cudaSuccess;
    EncodeTiledFn encode = get_encode_fn();
    if (encode == nullptr) {
        if (err) *err = "cuTensorMapEncodeTiled entry point not available";
        return cudaErrorNotSupported;
    }
    if (plan.num_sms == 0) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&plan.num_sms, cudaDevAttrMultiProcessorCount, dev);
        const char* cg = getenv("VPCA_CTA_GROUP");
        if (cg != nullptr) plan.cta_group = (atoi(cg) == 1) ? 1 : 2;
        const char* kw = getenv("VPCA_KB_WINDOW");
        if (kw != nullptr) plan.kb_window = atoi(kw);
        const char* sl = getenv("VPCA_SYNC_LEAD");
        if (sl != nullptr) plan.sync_lead = atoi(sl);
        const char* pf = getenv("VPCA_GRAM_PROF");
        plan.profile = (pf != nullptr && atoi(pf) != 0);
        const char* ad = getenv("VPCA_ADAPTIVE");
        if (ad != nullptr) plan.adaptive = atoi(ad) != 0;
        const char* sb = getenv("VPCA_SELF_B");
        if (sb != nullptr) plan.self_b = atoi(sb) != 0;
        const char* r64 = getenv("VPCA_RED64");
        if (r64 != nullptr) plan.red64 = atoi(r64) != 0;
        const char* gain = getenv("VPCA_REBALANCE_GAIN");
        if (gain != nullptr) plan.gain = std::min(1.0, std::max(0.1, atof(gain)));
        const char* ex = getenv("VPCA_EXACT_COVER");
        if (ex != nullptr) plan.exact_cover = atoi(ex) != 0;
    }
    if (cudaError_t e = plan.d_win_done.ensure(GramPlan::kMaxWindows); e != cudaSuccess) return e;
    if ((plan.profile || plan.adaptive) && plan.d_prof.get() == nullptr) {
        cudaError_t e = plan.d_prof.ensure(1024 * 4);
        if (e != cudaSuccess) return e;
        e = cudaMemsetAsync(plan.d_prof.get(), 0, 1024 * 4 * sizeof(long long), stream);
        if (e != cudaSuccess) return e;
    }
    if (plan.d_err == nullptr) {
        cudaError_t e = cudaHostAlloc(&plan.d_err, 4 * sizeof(int), cudaHostAllocMapped);
        if (e != cudaSuccess) return e;
        for (int i = 0; i < 4; ++i) plan.d_err[i] = 0;
    }
    const int tile_bn = kUmmaN;
    // Owner-computes band (a context that stores only rows [own_lo, own_hi) of S and has no peers to flush to): only the
    // tiles of those rows are enumerated -- the caller feeds every variant of the cohort to every band's context and no
    // cell is produced twice anywhere (SURVEY 8e "shard output tiles across GPUs ... no reduction").
    const bool banded = plan.own_hi > plan.own_lo && plan.num_peers <= 1;
    const int row_lo = banded ? plan.own_lo : 0, row_hi = banded ? plan.own_hi : n;
    const bool exact = plan.exact_cover && !banded;
    if (plan.tiles_for_n != n || plan.tiles_for_cg != plan.cta_group || plan.tiles_for_bn != (exact ? -1 : tile_bn) ||
        plan.tiles_row_lo != row_lo || plan.tiles_row_hi != row_hi) {
        cudaError_t e = build_tiles(plan, n, exact, tile_bn, row_lo, row_hi, stream);
        if (e != cudaSuccess) return e;
    }
    if (panel > 0) {
        if ((panel % 128) != 0) {
            if (err) *err = "panel_variants must be a multiple of 128";
            return cudaErrorInvalidValue;
        }
        ld = panel;   // rows of a panel are `panel` cells apart, panels n * panel cells apart
    }
    const uintptr_t align = (elem_bits == 4) ? 31 : 15;
    if ((reinterpret_cast<uintptr_t>(d_x) & align) != 0 || (((ld * elem_bits) / 8) & align) != 0 ||
        (elem_bits == 4 && (ld % 128) != 0)) {
        if (err) *err = "dense tile must be 16-byte aligned with a 16-byte multiple row pitch (32 / ld % 128 == 0 for e2m1)";
        return cudaErrorInvalidValue;
    }

    const int cgp = plan.cta_group;
    // one k-block = one 128-byte swizzle atom of the operand layout: 128 int8, 64 bf16 or 128 e2m1 cells (64 packed bytes,
    // expanded to one byte each in shared memory)
    const int elems_per_kb = (elem_bits == 16) ? 64 : 128;
    const int kind = (elem_bits == 8) ? 0 : (elem_bits == 16 ? 1 : 2);
    int workers = plan.num_sms;
    if (cgp == 2) {
        // a pair is a 2-CTA cluster: as many pairs as the device holds at once, so that all of them are co-resident
        int& pairs = plan.max_pairs[kind];
        if (pairs == 0) pairs = kind == 0 ? max_clusters<0>(2) : (kind == 1 ? max_clusters<1>(2) : max_clusters<2>(2));
        if (pairs <= 0) {
            if (err) *err = "cudaOccupancyMaxActiveClusters found no room for a 2-CTA cluster of the Gram kernel";
            return cudaErrorNotSupported;
        }
        workers = std::min(plan.num_sms / 2, pairs);
    }

    CUtensorMap tmap;
    // Panel layout: dim0 = cells of one panel row (bytes for e2m1), dim1 = samples, dim2 = panels.  Row-major input is one
    // panel as wide as the tile.  e2m1: the caller guarantees zero cells up to a multiple of 128.
    const int64_t npanels = panel > 0 ? (nv + panel - 1) / panel : 1;
    const int64_t cells0 = panel > 0 ? panel : (elem_bits == 4 ? ((nv + 127) / 128) * 128 : nv);
    const int64_t dim0 = elem_bits == 4 ? cells0 / 2 : cells0;
    const cuuint64_t gdim[3] = {(cuuint64_t)dim0, (cuuint64_t)n, (cuuint64_t)npanels};
    const cuuint64_t gstride[2] = {(cuuint64_t)ld * (cuuint64_t)elem_bits / 8,
                                   (cuuint64_t)n * (cuuint64_t)ld * (cuuint64_t)elem_bits / 8};
    const int kc_per_kb = elem_bits == 4 ? elems_per_kb / 2 : elems_per_kb;
    const cuuint32_t box[3] = {(cuuint32_t)kc_per_kb, (cuuint32_t)kBoxRows, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    const CUtensorMapDataType tmtype = elem_bits == 16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_UINT8;
    CUresult r = encode(&tmap, tmtype, 3,
                        const_cast<void*>(d_x), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        elem_bits == 4 ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
                        CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        if (err) *err = "cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r);
        return cudaErrorInvalidValue;
    }

    GramArgs args{};
    // a band is addressed through the virtual origin of the full matrix: row r lives at d_S + (r - own_lo) * n
    args.S = banded ? d_S - (ptrdiff_t)plan.own_lo * n : d_S;
    args.num_peers = (plan.num_peers > 1 && d_S == plan.peer_base[plan.peer_rank]) ? plan.num_peers : 0;
    for (int d = 0; d < kMaxPeers; ++d) args.peer[d] = d < plan.num_peers ? plan.peer_S[d] : nullptr;
    args.peer_mode = plan.peer_mode;
    for (int d = 0; d < kMaxPeers; ++d) args.own_end[d] = plan.own_end[d];
    args.tiles = reinterpret_cast<const TileDesc*>(plan.d_tiles.get());
    cudaHostGetDevicePointer(reinterpret_cast<void**>(&args.err), plan.d_err, 0);
    args.n = n;
    args.num_tiles = plan.num_tiles;
    args.num_full = plan.num_full;
    args.total_weight = plan.total_weight;
    args.kb_total = (int)((nv + elems_per_kb - 1) / elems_per_kb);
    args.kb_per_panel = panel > 0 ? (int)(panel / elems_per_kb) : args.kb_total;
    args.num_workers = workers;
    args.kc_per_kb = kc_per_kb;
    args.acc_stride = 0;
    args.col_limit = plan.tiles_col_limit;
    args.row_limit = row_hi;
    args.red64 = plan.red64 ? 1 : 0;
    FrontRange front;
    {
        int kbw = plan.kb_window;
        if (kbw <= 0 && panel > 0) kbw = args.kb_per_panel;   // one L2 window per panel
        if (kbw <= 0) {
            // window of X sized to ~16 MiB so that every tile re-reads it from L2 (50 MB) rather than HBM
            const long long target = 16ll << 20;
            kbw = (int)std::max<long long>(8, std::min<long long>(4096, target / ((long long)n * kKBytes)));
        }
        kbw = std::min(kbw, args.kb_total);
        std::vector<double> cum0;
        front = front_range(plan.num_tiles, workers, banded);
        if (front.on) {
            args.resident = 1;
            cum0.assign((size_t)workers + 1, 0.0);   // the within-window split is not used
        } else {
            // cheap upper bound first (a worker with less than a tile's worth of work can touch few tiles), then the exact test
            args.resident = (plan.num_tiles <= 4 * workers && initial_split(plan, workers, kbw, cum0)) ? 1 : 0;
        }
        double frac0 = front.init;
        int dev = 0;
        cudaGetDevice(&dev);
        args.kb_window = args.resident ? kbw : args.kb_total;
        // the device-side split (speed-weighted by rebalance_kernel, or the front/tail split point moved by
        // rebalance_front_kernel, from launch to launch) starts from the repaired equal split / the initial split point;
        // it is only meaningful for one (workers, tile list, window length)
        if (args.resident && (plan.d_cum.get() == nullptr || plan.cum_workers != workers || plan.cum_tiles != plan.num_tiles ||
                              plan.cum_kbw != kbw || plan.cum_for_n != n || plan.cum_elem != elem_bits)) {
            remember_split(plan);
            if (plan.adaptive && !banded) {   // a split learned earlier on this device for the same schedule, if it still fits the accumulator budget
                std::lock_guard<std::mutex> lk(g_split_mu);
                auto it = g_splits.find(SplitKey{dev, n, plan.num_tiles, kbw, workers, elem_bits});
                if (it != g_splits.end()) {
                    std::vector<double> learned = it->second;
                    if (front.on) {
                        const double f = learned.size() > (size_t)workers + 1 ? learned[(size_t)workers + 1] : -1.0;
                        if (f >= front.lo && f <= front.hi) frac0 = f;
                    } else {
                        const TileDesc* tiles = reinterpret_cast<const TileDesc*>(plan.h_tiles.data());
                        std::vector<long long> need((size_t)workers + 1);
                        learned.resize((size_t)workers + 1);
                        if (repair_split(tiles, plan.num_tiles, workers, (long long)plan.total_weight * kbw, kbw,
                                         plan.tiles_col_limit, learned.data(), need.data()))
                            cum0 = learned;
                    }
                }
            }
            plan.d_cum.reset();
            cudaError_t e = plan.d_cum.ensure((int64_t)(workers + 2) * sizeof(double) + sizeof(int));
            if (e != cudaSuccess) return e;
            cum0.push_back(frac0);                                 // [workers + 1]: the front/tail split point (fraction of K)
            cum0.push_back(0.0);                                   // [workers + 2]: the update counter (int)
            e = cudaMemcpyAsync(plan.d_cum.get(), cum0.data(), (size_t)(workers + 2) * sizeof(double) + sizeof(int),
                                cudaMemcpyHostToDevice, stream);   // pageable source: staged before the call returns
            if (e != cudaSuccess) return e;
            plan.cum_workers = workers;
            plan.cum_tiles = plan.num_tiles;
            plan.cum_kbw = kbw;
            plan.cum_for_n = n;
            plan.cum_dev = dev;
            plan.cum_elem = elem_bits;
        }
    }
    plan.last_resident = args.resident;
    double* cum = reinterpret_cast<double*>(plan.d_cum.get());   // the split (see GramPlan::d_cum)
    const int nwin = (args.kb_total + args.kb_window - 1) / args.kb_window;
    const long long uw = (long long)args.total_weight * args.kb_window;
    args.active_workers = (int)std::min<long long>(workers, uw);
    if (front.on) {   // only the front workers take part in the window pacing
        args.front_tiles = plan.num_tiles;
        args.front_frac = cum + workers + 1;
        args.active_workers = plan.num_tiles;
    }
    args.sync_lead = (args.resident && nwin <= GramPlan::kMaxWindows) ? plan.sync_lead : 0;
    args.win_done = plan.d_win_done.get();
    const bool adapt = plan.adaptive && args.resident && workers <= 1024 && (front.on || args.active_workers == workers);
    args.prof = (plan.profile || adapt) ? plan.d_prof.get() : nullptr;
    args.cum = cum;
    if (args.sync_lead > 0) {
        cudaError_t e = cudaMemsetAsync(plan.d_win_done.get(), 0, (size_t)nwin * sizeof(int), stream);
        if (e != cudaSuccess) return e;
    }

    const int grid = workers * cgp;
    cudaError_t le;
    if (cgp == 2)
        le = kind == 0 ? launch<2, 0>(tmap, args, grid, stream)
                       : (kind == 1 ? launch<2, 1>(tmap, args, grid, stream) : launch<2, 2>(tmap, args, grid, stream));
    else
        le = kind == 0 ? launch<1, 0>(tmap, args, grid, stream)
                       : (kind == 1 ? launch<1, 1>(tmap, args, grid, stream) : launch<1, 2>(tmap, args, grid, stream));
    if (le != cudaSuccess) return le;
    if (adapt && front.on) {
        rebalance_front_kernel<<<1, (workers + 31) / 32 * 32, 0, stream>>>(
            plan.d_prof.get(), cum + workers + 1, plan.num_tiles, workers, cgp, args.kb_total, plan.gain, front.lo, front.hi,
            300000, reinterpret_cast<int*>(cum + workers + 2));
        le = cudaGetLastError();
    } else if (adapt) {
        // shares move towards the measured speeds, at most 35 % above the mean; a split under which some worker's
        // accumulators would not fit its budget is rejected by the kernel itself
        rebalance_kernel<<<1, 1024, 0, stream>>>(plan.d_prof.get(), cum, workers, cgp, plan.gain, 1.35, 300000,
                                                 reinterpret_cast<int*>(cum + workers + 2), reinterpret_cast<const TileDesc*>(plan.d_tiles.get()), plan.num_tiles,
                                                 plan.total_weight, args.kb_window, plan.tiles_col_limit);
        le = cudaGetLastError();
    }
    return le;
}

// Loads every kernel of this translation unit on the current device.  With CUDA's lazy module loading the FIRST launch of
// a kernel loads it, and that load can wait for the device to go idle; a host thread that has just enqueued a spinning
// peer_barrier_kernel for one context and then launches a not-yet-loaded kernel (for this or another context of the same
// process) would wait for a barrier that can only complete once the thread has enqueued the other contexts' barriers --
// a deadlock (two contexts in one process: the 30 s barrier watchdog fires).  One process driving
// several contexts (vpca_gram_set_peers_local, vpca_pool) therefore loads everything up front: cudaFuncGetAttributes
// for all kernels, plus an empty launch of those that are enqueued behind a barrier.
cudaError_t gram_preload_kernels(cudaStream_t stream) {
    cudaFuncAttributes fa;
    cudaError_t e = cudaSuccess;
#define VPCA_LOAD(k) if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, k)
    VPCA_LOAD((gram_kernel<1, 0>)); VPCA_LOAD((gram_kernel<1, 1>)); VPCA_LOAD((gram_kernel<1, 2>));
    VPCA_LOAD((gram_kernel<2, 0>)); VPCA_LOAD((gram_kernel<2, 1>)); VPCA_LOAD((gram_kernel<2, 2>));
    VPCA_LOAD(rebalance_kernel); VPCA_LOAD(rebalance_front_kernel); VPCA_LOAD(symmetrize_kernel); VPCA_LOAD(add_i32_kernel); VPCA_LOAD(add_i32_peers_kernel);
    VPCA_LOAD(add_i32_owner_kernel); VPCA_LOAD(gather_rows_kernel); VPCA_LOAD(push_rows_kernel); VPCA_LOAD(peer_barrier_kernel);
#undef VPCA_LOAD
    if (e != cudaSuccess) return e;
    PeerPtrs pp{};
    OwnEnds own{};
    peer_barrier_kernel<<<1, 32, 0, stream>>>(pp, 0, 0, 0);                 // npeers = 0: no thread touches a flag
    push_rows_kernel<<<1, 32, 0, stream>>>(pp, nullptr, own, 0, 0, 0);        // own.e[0] = 0: no rows
    gather_rows_kernel<<<1, 32, 0, stream>>>(pp, nullptr, own, 0, 0, 0);      // n = 0
    add_i32_owner_kernel<<<1, 32, 0, stream>>>(pp, own, 0, nullptr, 0);       // n = 0
    add_i32_peers_kernel<<<1, 32, 0, stream>>>(pp, 0, nullptr, 0);            // count = 0
    add_i32_kernel<<<1, 32, 0, stream>>>(nullptr, nullptr, 0);
    symmetrize_kernel<<<dim3(1, 1), dim3(32, 8), 0, stream>>>(nullptr, 0);    // n = 0: every access is masked
    return cudaGetLastError();
}

// How many clusters of `cluster_size` CTAs of the int8 Gram kernel the current device can hold at once -- the GPC
// layout decides whether a 4- or 8-CTA cluster could still use every SM.  Diagnostic only.
int gram_debug_max_clusters(int cluster_size) { return max_clusters<0>(cluster_size); }

cudaError_t gram_symmetrize(int32_t* d_S, int n, cudaStream_t stream) {
    const int nb = (n + 31) / 32;
    symmetrize_kernel<<<dim3(nb, nb), dim3(32, 8), 0, stream>>>(d_S, n);
    return cudaGetLastError();
}

cudaError_t gram_add(int32_t* d_dst, const int32_t* d_src, int64_t count, cudaStream_t stream) {
    add_i32_kernel<<<592, 256, 0, stream>>>(d_dst, d_src, count);
    return cudaGetLastError();
}

cudaError_t gram_add_peers(GramPlan& plan, const int32_t* d_src, int64_t count, cudaStream_t stream) {
    PeerPtrs pp{};
    for (int d = 0; d < plan.num_peers; ++d) pp.p[d] = plan.peer_S[d];
    add_i32_peers_kernel<<<592, 256, 0, stream>>>(pp, plan.num_peers, d_src, count);
    return cudaGetLastError();
}

cudaError_t gram_add_owners(GramPlan& plan, const int32_t* d_src, int n, cudaStream_t stream) {
    PeerPtrs pp{};
    OwnEnds own{};
    for (int d = 0; d < plan.num_peers; ++d) pp.p[d] = plan.peer_S[d];
    for (int d = 0; d < kMaxPeers; ++d) own.e[d] = plan.own_end[d];
    add_i32_owner_kernel<<<592, 256, 0, stream>>>(pp, own, plan.num_peers, d_src, n);
    return cudaGetLastError();
}

cudaError_t gram_gather_rows(GramPlan& plan, int32_t* d_S, int n, cudaStream_t stream) {
    PeerPtrs pp{};
    OwnEnds own{};
    for (int d = 0; d < plan.num_peers; ++d) pp.p[d] = plan.peer_S[d];
    for (int d = 0; d < kMaxPeers; ++d) own.e[d] = plan.own_end[d];
    // VPCA_GATHER=push (default) | pull | copy: posted peer stores, peer loads, or copy-engine 2-D copies per band
    const char* how = getenv("VPCA_GATHER");
    if (how != nullptr && strcmp(how, "pull") == 0) {
        gather_rows_kernel<<<1184, 256, 0, stream>>>(pp, d_S, own, plan.num_peers, plan.peer_rank, n);
    } else if (how != nullptr && strcmp(how, "copy") == 0) {
        for (int q = 0; q < plan.num_peers; ++q) {
            if (q == plan.peer_rank) continue;
            const int r0 = q == 0 ? 0 : plan.own_end[q - 1], r1 = plan.own_end[q];
            cudaError_t e = cudaMemcpy2DAsync(d_S + (size_t)r0 * n, (size_t)n * 4, plan.peer_S[q] + (size_t)r0 * n,
                                              (size_t)n * 4, (size_t)std::min(n, r1) * 4, (size_t)(r1 - r0),
                                              cudaMemcpyDeviceToDevice, stream);
            if (e != cudaSuccess) return e;
        }
    } else {
        push_rows_kernel<<<1184, 256, 0, stream>>>(pp, d_S, own, plan.num_peers, plan.peer_rank, n);
    }
    return cudaGetLastError();
}

cudaError_t gram_peer_barrier(GramPlan& plan, cudaStream_t stream) {
    PeerPtrs pp{};
    for (int d = 0; d < plan.num_peers; ++d) pp.p[d] = plan.peer_flags[d];
    plan.peer_epoch += 1;
    peer_barrier_kernel<<<1, 32, 0, stream>>>(pp, plan.num_peers, plan.peer_rank, plan.peer_epoch);
    return cudaGetLastError();
}

}  // namespace vpca
