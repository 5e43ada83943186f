// libvpca C ABI (include/vpca.h): context management, host<->device staging and the call sequence
// encode -> Gram -> (cross-GPU reduce) -> symmetrize -> centering -> eigensolve.
// Mirrors the method set of the reference's VariantsPcaDriver
// (src/main/scala/com/google/cloud/genomics/spark/examples/VariantsPca.scala:81-286); see vpca.h for the mapping.
//
// Threading model (the reference runs the bodies of `mapPartitions` concurrently, one task thread per core,
// VariantsPca.scala:184-189): host-input calls (accumulate_calls / _u16 / _bits / _bed / dense-from-host) take one
// of `staging_lanes` LANES -- a private stream pair, double-buffered staging and a private Gram schedule -- and hold
// the context mutex only for bookkeeping, never across a copy, a kernel or a stream synchronisation.  So the H2D copy
// and encode of one task overlap the Gram kernel of another; a partition's staging Gram (slot) is private to the
// task that owns the partition id, and `commit` folds it into the Gram with integer adds on the context's stream.
#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <cmath>
#include <condition_variable>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "vpca_internal.h"

using namespace vpca;

namespace {
thread_local std::string tls_error;
thread_local const vpca_ctx* tls_error_ctx = nullptr;
thread_local std::string tls_error_copy;
}   // namespace

struct vpca_ctx {
    vpca_config cfg{};
    int n = 0;
    int elem_bits = 8;   // 8 = int8, 16 = bf16, 4 = packed e2m1
    int max_mult = 2;
    int num_pc = 2;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    int32_t* d_S = nullptr;          // the Gram: cfg.d_gram, or owned_S
    DeviceBuffer<int32_t> owned_S;   // a library-owned Gram, with the barrier flags of the peer-reduce mode after it
    int band_row0 = 0, band_rows = 0;   // rows of the Gram this context stores (band_rows == n: all of them)
    bool finalized = false;
    bool pca_done = false;
    GramPlan plan;        // schedule state of the launches on `stream` (device-resident input)
    EigWork eig;
    bool eig_ready = false;
    BandEigWork band_eig;   // vpca_compute_pca_bands with this context as rank 0: the solver's state
    BandPart band_part;     // vpca_compute_pca_bands: this context's share of the sharded mat-vec
    JoinWork join;        // multi-dataset keying (join.cu); one join at a time (join_mu)
    std::mutex join_mu;
    int pca_k = 0;        // k of the last solve whose U / eigenvalues are still valid on the device (0: none)
    const double* d_U = nullptr;     // that U (n x min(pca_k, 16), column-major): eig.d_evecs after vpca_compute_pca;
                                     // band_eig.d_evecs or d_band_U after vpca_compute_pca_bands
    DeviceBuffer<double> d_band_U;   // n x 16: this rank's copy of U from a band solve driven by another context
    // vpca_compute_pca_subset: a solver of its own for the m kept samples (ctx->eig is never touched), their m x m Gram,
    // U scattered to n x 16 with zero rows for the removed samples (d_U points here after a subset solve, which is what
    // makes the loadings apply d_sub_keep), the n x k output, the sample lists and the keep bytes
    EigWork sub_eig;
    DeviceBuffer<int32_t> d_sub_S;
    DeviceBuffer<double> d_sub_U;
    DeviceBuffer<double> d_sub_vecs;    // n x max(num_pc, 16) (the first k columns used)
    DeviceBuffer<double> d_sub_t;       // max(num_pc, 16): sum_j rho_j u_c[j]
    DeviceBuffer<int32_t> d_sub_idx;    // n: kept samples, then removed ones, each in increasing order
    DeviceBuffer<uint8_t> d_sub_keep;   // n: 1 for kept samples
    int proj_k = 0;       // k of the projection begun by vpca_project_begin (0: none in progress)
    DeviceBuffer<double> d_proj_acc;    // n x kProjLd partial projection sums (project.cu)
    DeviceBuffer<double> d_proj_part;   // per-panel partial sums of one launch
    DeviceBuffer<double> d_lp_w;        // host-input loadings / projection: one chunk of w (loadings out, projection in)
    DeviceBuffer<double> d_lp_mean;     // and of the means (projection)
    DeviceBuffer<int32_t> d_lp_count;   // and of the carrier counts (loadings)
    // kinship (vpca_kinship_bed / _pairs): the 3n x 3n int32 Gram of the indicator planes, allocated on the first call, with
    // a Gram schedule and plane staging of its own (the PCA Gram's tiles and stream-K split are never touched)
    DeviceBuffer<int32_t> d_kin;
    GramPlan kin_plan;
    DeviceBuffer<uint8_t> d_kin_x[2];
    int64_t kin_chunk = 0, kin_panel = 0;   // rows per staged chunk, variants per panel of the 3n-row plane tile
    int64_t kin_variants = 0;               // rows added since creation / the last vpca_reset
    KinPairWork kin_pairs;
    // LD pruning (vpca_ld_prune_bed): the 3c x 3c plane Gram of one chunk, its plane tile, double-buffered raw rows, the
    // chunk's window starts, the pair scratch and the keep bytes; all grow-only, with a Gram schedule of their own
    DeviceBuffer<int32_t> d_ld_G;
    DeviceBuffer<uint8_t> d_ld_x;
    DeviceBuffer<uint8_t> d_ld_rows[2];
    DeviceBuffer<int64_t> d_ld_wlo;
    DeviceBuffer<uint8_t> d_ld_keep;
    DeviceBuffer<uint8_t> d_ld_elig;    // vpca_ld_prune_bed_masked: the eligible bytes of the call
    // .bed rows of the driver-side calls (GRM, its loadings and projection, GLM, variant and sample QC), double-buffered:
    // those calls never run at the same time, so they share this pair (stage_rows); grow-only
    DeviceBuffer<uint8_t> d_bed_rows[2];
    // variant QC (vpca_variant_qc_bed / vpca_hwe_exact): the counts and p-values of one batch; grow-only
    DeviceBuffer<int32_t> d_qc_counts;
    DeviceBuffer<double> d_qc_p;
    // sample QC (vpca_sample_missing_bed / vpca_subset_bed_samples): double-buffered repacked rows of one chunk, the
    // per-sample counts, the kept indices, and a stream and events of their own for the D2H copies; grow-only
    DeviceBuffer<uint8_t> d_sm_out[2];
    DeviceBuffer<int32_t> d_sm_miss;
    DeviceBuffer<int32_t> d_sm_idx;
    cudaStream_t sm_d2h_stream = nullptr;
    cudaEvent_t sm_ev_copy[2] = {nullptr, nullptr}, sm_ev_kern[2] = {nullptr, nullptr};
    GramPlan ld_plan;
    LdWork ld;
    // GRM (vpca_grm_bed / _finalize, grm.cu): the chunk's counts, z tables, used flags and used list, and one FP64 panel;
    // the sum itself accumulates in eig.d_C.  All grow-only.
    DeviceBuffer<int32_t> d_grm_counts, d_grm_used, d_grm_inv;
    DeviceBuffer<double> d_grm_tab, d_grm_Z;
    DeviceBuffer<int> d_grm_total;
    int grm_state = 0;      // 0 none, 1 accumulating, 2 finalized (eig.d_C holds the GRM), 3 unusable until vpca_reset
                            // (finalized with no used variant, or d_C overwritten by another solve)
    int64_t grm_used = 0;   // used variants so far (M)
    int grm_fill = 0;       // of which in the current, not yet multiplied panel
    // GRM loadings and projection (grm_project.cu): U of the last successful vpca_compute_pca_grm (n x 16 column-major,
    // the first grm_k columns valid; its own buffer, so it outlives the direct solve that consumes d_C), and one chunk of
    // loadings (out) or of the caller's w and tables (projection, in)
    DeviceBuffer<double> d_grm_U, d_grm_w, d_grm_ptab;
    int grm_k = 0;          // 0: no GRM U
    // linear association tests (vpca_glm_*, glm.cu): Q, y~ and the mask of the last vpca_glm_begin (n rows of
    // glm_kmax(q) + 2 doubles), the regression mask as bits, Q^T y~, and one chunk of sums and outputs.  All grow-only.
    // The logistic tests (vpca_glm_logistic_*) keep y in place of y~, the null fit in d_glm_z0, the cases as bits in
    // d_glm_case, the counts in d_glm_sums and the passes in d_glm_passes.
    DeviceBuffer<double> d_glm_Qx, d_glm_z0, d_glm_sums, d_glm_out;
    // The Firth tests (vpca_glm_firth_bed) add the chunk's Firth flags, and for a fallback the list of the variants to
    // refit and its length, built on the device.
    DeviceBuffer<uint8_t> d_glm_mask, d_glm_case, d_glm_firth;
    DeviceBuffer<int32_t> d_glm_err, d_glm_passes, d_glm_idx, d_glm_nf;
    int glm_q = 0;          // 0: no GLM state
    int glm_logistic = 0;   // the model of the GLM state: 0 linear (vpca_glm_begin), 1 logistic
    int glm_nreg = 0;       // regression samples
    double glm_yty = 0.0;   // y~^T y~

    struct Slot {
        int64_t pid = -1;
        DeviceBuffer<int32_t> d_S;
        bool used = false;
        bool busy = false;             // a call of the owning task is in flight
        bool fresh = false;            // still to be zeroed by its first batch
        int64_t nv = 0;
        cudaEvent_t ev_free = nullptr; // recorded after the commit that last read the slot
    };
    std::vector<Slot> slots;

    // One lane = everything a host-input call needs to run without the other lanes: streams, double-buffered CSR /
    // dense staging, error flags and its own Gram schedule (the speed-weighted stream-K shares must not change under
    // a running kernel, so they are per stream).
    struct Lane {
        cudaStream_t stream = nullptr, copy_stream = nullptr;
        DeviceBuffer<int64_t> d_off[2];
        DeviceBuffer<int32_t> d_idx[2];
        DeviceBuffer<uint8_t> d_x[2];
        cudaEvent_t ev_copy[2] = {nullptr, nullptr};
        cudaEvent_t ev_done[2] = {nullptr, nullptr};
        cudaEvent_t ev_order = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
        DeviceBuffer<int> d_flags;
        int* h_flags = nullptr;
        GramPlan plan;
        bool ready = false, busy = false;
    };
    std::vector<Lane> lanes;
    int64_t chunk_variants = 0, chunk_nnz = 0;
    int64_t panel = 8192;   // cells per panel row of the internal dense staging tiles (VPCA_PANEL)

    cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr, ev_e0 = nullptr, ev_e1 = nullptr;
    bool gram_timed = false, eig_timed = false;

    int64_t total_variants = 0;      // committed + direct
    int64_t inflight_variants = 0;   // staged in slots, not yet committed
    vpca_stats st{};
    std::atomic<int64_t> c_launches{0}, c_gram{0}, c_h2d{0}, c_d2h{0};
    std::atomic<float> lane_gram_ms{0.f};
    std::mutex mu;
    std::condition_variable cv;
    std::mutex err_mu;
    std::string err;
};

namespace {

int fail(vpca_ctx* ctx, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    tls_error = buf;
    tls_error_ctx = ctx;
    if (ctx) {
        std::lock_guard<std::mutex> lk(ctx->err_mu);
        ctx->err = buf;
    }
    return code;
}

#define CUDA_OK(ctx, call)                                                                                      \
    do {                                                                                                        \
        cudaError_t _e = (call);                                                                                \
        if (_e != cudaSuccess)                                                                                  \
            return fail(ctx, VPCA_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__,   \
                        __LINE__);                                                                              \
    } while (0)

// every similarity count is at most (#variants) * max_mult^2 and must stay a Java Int (VariantsPca.scala:185).
// `extra` = variants about to be added on top of everything committed AND everything staged in uncommitted partitions.
int check_overflow(vpca_ctx* ctx, int64_t extra) {
    const long double worst =
        (long double)(ctx->total_variants + ctx->inflight_variants + extra) * ctx->max_mult * ctx->max_mult;
    if (worst > 2147483647.0L)
        return fail(ctx, VPCA_ERR_OVERFLOW, "%lld variants x multiplicity %d^2 could overflow an int32 similarity count",
                    (long long)(ctx->total_variants + ctx->inflight_variants + extra), ctx->max_mult);
    return VPCA_OK;
}

void free_lane(vpca_ctx::Lane& L) {
    if (L.stream) cudaStreamSynchronize(L.stream);
    if (L.copy_stream) cudaStreamSynchronize(L.copy_stream);
    for (int b = 0; b < 2; ++b) {
        if (L.ev_copy[b]) cudaEventDestroy(L.ev_copy[b]);
        if (L.ev_done[b]) cudaEventDestroy(L.ev_done[b]);
        L.ev_copy[b] = L.ev_done[b] = nullptr;
    }
    for (cudaEvent_t* ev : {&L.ev_order, &L.ev_t0, &L.ev_t1})
        if (*ev) {
            cudaEventDestroy(*ev);
            *ev = nullptr;
        }
    if (L.h_flags) cudaFreeHost(L.h_flags);
    L.h_flags = nullptr;
    gram_plan_free(L.plan);
    if (L.copy_stream) cudaStreamDestroy(L.copy_stream);
    if (L.stream) cudaStreamDestroy(L.stream);
    L.copy_stream = L.stream = nullptr;
    L.ready = false;
}

void copy_peers(const GramPlan& from, GramPlan& to) {
    to.own_lo = from.own_lo;
    to.own_hi = from.own_hi;
    to.num_peers = from.num_peers;
    to.peer_rank = from.peer_rank;
    to.peer_mode = from.peer_mode;
    for (int d = 0; d < 16; ++d) {
        to.peer_S[d] = from.peer_S[d];
        to.peer_flags[d] = from.peer_flags[d];
        to.own_end[d] = from.own_end[d];
    }
}

void sync_peers_to_lanes(vpca_ctx* ctx) {
    for (auto& L : ctx->lanes) copy_peers(ctx->plan, L.plan);
}

void staging_geometry(vpca_ctx* ctx) {
    if (ctx->chunk_variants != 0) return;
    const int n = ctx->n, bits = ctx->elem_bits;
    int64_t cv = ctx->cfg.chunk_variants;
    if (cv <= 0) {
        cv = (256ll << 20) * 8 / ((int64_t)n * bits);
        cv = std::max<int64_t>(1024, std::min<int64_t>(cv, 1 << 20));
    }
    if (const char* pe = getenv("VPCA_PANEL")) {
        const int64_t pv = atoll(pe);
        if (pv >= 128 && pv % 128 == 0) ctx->panel = pv;
    }
    cv = std::max<int64_t>(ctx->panel, (cv / ctx->panel) * ctx->panel);   // whole panels
    int64_t cz = ctx->cfg.chunk_nnz;
    if (cz <= 0) cz = 64ll << 20;
    cz = std::max<int64_t>(cz, 1024);
    ctx->chunk_variants = cv;
    ctx->chunk_nnz = cz;
}

// Allocates the lane's streams and staging buffers on first use; on any failure the streams and events are released
// again, so a later call retries instead of running on half a lane.
int ensure_lane(vpca_ctx* ctx, vpca_ctx::Lane& L) {
    if (L.ready) return VPCA_OK;
    const int n = ctx->n, bits = ctx->elem_bits;
    const int64_t cv = ctx->chunk_variants, cz = ctx->chunk_nnz;
    cudaError_t e = cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&L.copy_stream, cudaStreamNonBlocking);
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
        e = L.d_off[b].ensure(cv + 1);
        if (e == cudaSuccess) e = L.d_idx[b].ensure(cz);
        if (e == cudaSuccess) e = L.d_x[b].ensure((int64_t)n * cv * bits / 8);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&L.ev_copy[b], cudaEventDisableTiming);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&L.ev_done[b], cudaEventDisableTiming);
    }
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&L.ev_order, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreate(&L.ev_t0);
    if (e == cudaSuccess) e = cudaEventCreate(&L.ev_t1);
    if (e == cudaSuccess) e = L.d_flags.ensure(1);
    if (e == cudaSuccess) e = cudaHostAlloc(&L.h_flags, sizeof(int), cudaHostAllocPortable);
    if (e != cudaSuccess) {
        free_lane(L);
        return fail(ctx, e == cudaErrorMemoryAllocation ? VPCA_ERR_NOMEM : VPCA_ERR_CUDA, "staging lane: %s",
                    cudaGetErrorString(e));
    }
    copy_peers(ctx->plan, L.plan);
    L.ready = true;
    return VPCA_OK;
}

// A free lane, blocking while all are taken.  Also orders the lane's stream after everything enqueued on the context's
// stream so far (a preceding vpca_reset / vpca_load_partial_gram).
struct LaneGuard {
    vpca_ctx* ctx;
    vpca_ctx::Lane* lane = nullptr;
    int rc = VPCA_OK;
    explicit LaneGuard(vpca_ctx* c) : ctx(c) {
        std::unique_lock<std::mutex> lk(ctx->mu);
        staging_geometry(ctx);
        ctx->cv.wait(lk, [&] {
            for (auto& L : ctx->lanes)
                if (!L.busy) return true;
            return false;
        });
        for (auto& L : ctx->lanes)
            if (!L.busy) {
                lane = &L;
                break;
            }
        lane->busy = true;
        rc = ensure_lane(ctx, *lane);
        if (rc == VPCA_OK) {
            cudaError_t e = cudaEventRecord(lane->ev_order, ctx->stream);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(lane->stream, lane->ev_order, 0);
            if (e != cudaSuccess) rc = fail(ctx, VPCA_ERR_CUDA, "lane ordering: %s", cudaGetErrorString(e));
        }
    }
    ~LaneGuard() {
        {
            std::lock_guard<std::mutex> lk(ctx->mu);
            lane->busy = false;
        }
        ctx->cv.notify_one();
    }
};

int launch_gram(vpca_ctx* ctx, GramPlan& plan, cudaStream_t stream, cudaEvent_t t0, cudaEvent_t t1, const void* d_x,
                int64_t nv, int64_t ld, int64_t panel, int32_t* d_target) {
    // fp32 accumulation (bf16) is exact only below 2^24: bound the variants one launch may fold (e2m1, whose doubled
    // cells accumulate 4 S in int32, keeps the same bound).
    // vpca_create guarantees that the bound is at least one panel.
    int64_t limit = nv;
    if (ctx->elem_bits != 8) {
        limit = (int64_t)(16777216ll / ((int64_t)ctx->max_mult * ctx->max_mult));
        const int64_t q = panel > 0 ? panel : 128;
        limit = (limit / q) * q;
        if (limit <= 0)
            return fail(ctx, VPCA_ERR_UNSUPPORTED, "max_multiplicity %d leaves no exact fp32 accumulation window for panels of "
                        "%lld variants", ctx->max_mult, (long long)q);
    }
    for (int64_t v0 = 0; v0 < nv; v0 += limit) {
        const int64_t cnt = std::min<int64_t>(limit, nv - v0);
        std::string msg;
        cudaEventRecord(t0, stream);
        // sub-launches start on a panel boundary (panel layout) or at column v0 (row-major)
        const size_t byte_off = panel > 0 ? (size_t)(v0 / panel) * (size_t)ctx->n * (size_t)panel * ctx->elem_bits / 8
                                          : (size_t)v0 * ctx->elem_bits / 8;
        cudaError_t e = gram_accumulate(plan, static_cast<const char*>(d_x) + byte_off, ctx->elem_bits, ctx->n, cnt, ld,
                                        panel, d_target, stream, &msg);
        cudaEventRecord(t1, stream);
        if (e != cudaSuccess)
            return fail(ctx, VPCA_ERR_CUDA, "Gram launch failed: %s %s", cudaGetErrorString(e), msg.c_str());
        ctx->c_gram += 1;
        ctx->c_launches += 1;
    }
    return VPCA_OK;
}

// Caller holds ctx->mu.
vpca_ctx::Slot* find_slot(vpca_ctx* ctx, int64_t pid, bool create, int* rc) {
    *rc = VPCA_OK;
    for (auto& s : ctx->slots)
        if (s.used && s.pid == pid) return &s;
    if (!create) return nullptr;
    for (auto& s : ctx->slots)
        if (!s.used) {
            cudaError_t e = s.d_S.ensure((int64_t)ctx->n * ctx->n);
            if (e == cudaSuccess && s.ev_free == nullptr) e = cudaEventCreateWithFlags(&s.ev_free, cudaEventDisableTiming);
            if (e != cudaSuccess) {
                *rc = fail(ctx, VPCA_ERR_NOMEM, "cudaMalloc of a partition Gram failed: %s", cudaGetErrorString(e));
                return nullptr;
            }
            s.used = true;
            s.fresh = true;
            s.busy = false;
            s.pid = pid;
            s.nv = 0;
            return &s;
        }
    *rc = fail(ctx, VPCA_ERR_STATE, "more than %d partitions in flight; commit or abort one first",
               (int)ctx->slots.size());
    return nullptr;
}

// Bookkeeping that brackets every host-input accumulate call.  begin(): state + overflow checks, slot lookup.
// end(): counters, slot release; a failed batch poisons its partition (the staging Gram may be partially updated).
struct CallScope {
    vpca_ctx* ctx;
    int64_t pid, nv;
    vpca_ctx::Slot* slot = nullptr;
    int32_t* target = nullptr;
    bool fresh = false;
    int begin() {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
        int rc = check_overflow(ctx, nv);
        if (rc != VPCA_OK) return rc;
        target = ctx->d_S;
        if (pid >= 0) {
            slot = find_slot(ctx, pid, true, &rc);
            if (slot == nullptr) return rc;
            if (slot->busy) {
                slot = nullptr;
                return fail(ctx, VPCA_ERR_STATE, "partition %lld is being written by another thread (spark.speculation "
                            "must stay off)", (long long)pid);
            }
            slot->busy = true;
            fresh = slot->fresh;
            slot->fresh = false;
            target = slot->d_S.get();
            ctx->inflight_variants += nv;   // reserved now, so that concurrent tasks cannot jointly pass the bound
        } else if (ctx->band_rows != ctx->n) {
            return fail(ctx, VPCA_ERR_STATE, "a band-only Gram takes device-resident input (vpca_accumulate_panels / "
                        "vpca_accumulate_dense with on_device = 1)");
        }
        return VPCA_OK;
    }
    int end(int rc) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (slot != nullptr) {
            slot->busy = false;
            if (rc == VPCA_OK) {
                slot->nv += nv;
            } else {
                ctx->inflight_variants -= nv + slot->nv;
                ctx->st.variants_accumulated -= slot->nv;
                slot->used = false;
            }
        } else if (rc == VPCA_OK) {
            ctx->total_variants += nv;
        } else if (rc == VPCA_ERR_INDEX_OUT_OF_RANGE || rc == VPCA_ERR_OVERFLOW) {
            std::lock_guard<std::mutex> lk2(ctx->err_mu);
            ctx->err += " [direct accumulation: the Gram may hold a partial batch, call vpca_reset]";
            tls_error = ctx->err;
        }
        if (rc == VPCA_OK) ctx->st.variants_accumulated += nv;
        return rc;
    }
};

// First batch of a partition: zero its staging Gram on the lane's stream, after the commit that last read it.
int prepare_slot(vpca_ctx* ctx, vpca_ctx::Lane& L, CallScope& sc) {
    if (sc.slot == nullptr || !sc.fresh) return VPCA_OK;
    CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, sc.slot->ev_free, 0));
    CUDA_OK(ctx, cudaMemsetAsync(sc.slot->d_S.get(), 0, (size_t)ctx->n * ctx->n * sizeof(int32_t), L.stream));
    return VPCA_OK;
}

void lane_gram_time(vpca_ctx* ctx, vpca_ctx::Lane& L) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, L.ev_t0, L.ev_t1) == cudaSuccess) {
        ctx->lane_gram_ms.store(ms);
        std::lock_guard<std::mutex> lk(ctx->mu);
        ctx->gram_timed = false;
        ctx->st.gram_cta_group = L.plan.cta_group;
        ctx->st.gram_resident = L.plan.last_resident;
    }
}

// What a staging loop does with one encoded chunk: rows [v, v + nvc) of the call sit in L.d_x[b] in panel layout
// (ctx->panel); work is enqueued on L.stream.
using ChunkFn = std::function<int(vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc)>;

// CSR rows -> encode -> consume(chunk), on lane L.  gram: the consumer launches the Gram (its time is recorded).
int process_calls(vpca_ctx* ctx, vpca_ctx::Lane& L, const int64_t* offsets, const void* sample_idx, int idx_bytes,
                  int64_t nv, const ChunkFn& consume, bool gram) {
    const int bits = ctx->elem_bits;
    // validate the whole offsets array before anything is sized from it
    if (offsets[0] < 0) return fail(ctx, VPCA_ERR_BAD_ARG, "offsets[0] must be >= 0");
    for (int64_t q = 0; q < nv; ++q)
        if (offsets[q + 1] < offsets[q]) return fail(ctx, VPCA_ERR_BAD_ARG, "offsets must be non-decreasing (row %lld)", (long long)q);
    *L.h_flags = 0;
    CUDA_OK(ctx, cudaMemsetAsync(L.d_flags.get(), 0, sizeof(int), L.stream));
    int64_t v = 0;
    int chunk = 0;
    while (v < nv) {
        // largest run of rows that fits both the variant and the index budget
        int64_t vend = std::min(nv, v + ctx->chunk_variants);
        if (offsets[vend] - offsets[v] > ctx->chunk_nnz) {
            const int64_t* hi = std::upper_bound(offsets + v, offsets + vend + 1, offsets[v] + ctx->chunk_nnz);
            vend = (hi - offsets) - 1;
            if (bits == 4 && vend - v >= 128) vend = v + ((vend - v) / 128) * 128;   // keep packed rows byte aligned
            if (vend <= v)
                return fail(ctx, VPCA_ERR_BAD_ARG, "row %lld has %lld entries, more than chunk_nnz=%lld", (long long)v,
                            (long long)(offsets[v + 1] - offsets[v]), (long long)ctx->chunk_nnz);
        }
        const int64_t nvc = vend - v, nnz = offsets[vend] - offsets[v];
        if (nnz > ctx->chunk_nnz || nvc > ctx->chunk_variants)
            return fail(ctx, VPCA_ERR_BAD_ARG, "internal: chunk of %lld rows / %lld entries exceeds the staging buffers",
                        (long long)nvc, (long long)nnz);
        const int b = chunk & 1;
        // the copy stream may overwrite buffer b only after the kernels that read it have run
        CUDA_OK(ctx, cudaStreamWaitEvent(L.copy_stream, L.ev_done[b], 0));
        CUDA_OK(ctx, cudaMemcpyAsync(L.d_off[b].get(), offsets + v, (size_t)(nvc + 1) * sizeof(int64_t), cudaMemcpyHostToDevice,
                                     L.copy_stream));
        if (nnz > 0)
            CUDA_OK(ctx, cudaMemcpyAsync(L.d_idx[b].get(), static_cast<const char*>(sample_idx) + (size_t)offsets[v] * idx_bytes,
                                         (size_t)nnz * idx_bytes, cudaMemcpyHostToDevice, L.copy_stream));
        CUDA_OK(ctx, cudaEventRecord(L.ev_copy[b], L.copy_stream));
        ctx->c_h2d += (nvc + 1) * 8 + nnz * idx_bytes;
        CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, L.ev_copy[b], 0));
        const int64_t P = ctx->panel;
        CUDA_OK(ctx, encode_calls(L.d_off[b].get(), offsets[v], L.d_idx[b].get(), idx_bytes, nvc, ctx->n, bits, ctx->max_mult, L.d_x[b].get(), P, P,
                                  L.d_flags.get(), L.stream));
        ctx->c_launches += 2;
        int rc = consume(L, b, v, nvc);
        if (rc != VPCA_OK) return rc;
        CUDA_OK(ctx, cudaEventRecord(L.ev_done[b], L.stream));
        v = vend;
        ++chunk;
    }
    CUDA_OK(ctx, cudaMemcpyAsync(L.h_flags, L.d_flags.get(), sizeof(int), cudaMemcpyDeviceToHost, L.stream));
    // the caller's buffers are read asynchronously: do not return before every copy has completed
    CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
    if (gram && nv > 0) lane_gram_time(ctx, L);
    if (*L.h_flags & 1)
        return fail(ctx, VPCA_ERR_INDEX_OUT_OF_RANGE, "sample index outside [0, %d) (the reference throws at "
                    "VariantsPca.scala:59/:188)", ctx->n);
    if (*L.h_flags & 2)
        return fail(ctx, VPCA_ERR_OVERFLOW, "a sample is listed more than max_multiplicity=%d times in one row",
                    ctx->max_mult);
    return VPCA_OK;
}


// What the row stager does with one staged chunk: rows [v, v + nvc) of the call sit in d_rows, which is dst[b]; work is
// enqueued on L.stream.
using RowsFn = std::function<int(int b, const uint8_t* d_rows, int64_t v, int64_t nvc)>;

// Rows [0, nv) of `rows` (host, `stride` bytes apart) go to the device `step` rows at a time, chunk c into dst[c & 1] on
// L.copy_stream once the work that last read that buffer (chunk c - 2, L.ev_done) is done; work(b, d_rows, v, nvc)
// enqueues chunk c's kernels on L.stream and may synchronise it.  The copy of chunk c is enqueued after work(c - 1), not
// before: from pageable memory cudaMemcpyAsync blocks the host until its stream reaches the copy, so this order is the
// one that keeps chunk c - 1's kernels running while chunk c is copied.  Counts c_h2d; returns work's first error, else
// after L.stream has drained (the caller's rows are free on return).
int stage_rows(vpca_ctx* ctx, vpca_ctx::Lane& L, const uint8_t* rows, int64_t nv, int64_t stride, int64_t step,
               const std::array<uint8_t*, 2>& dst, const RowsFn& work) {
    for (int64_t v = 0, c = 0; v < nv; v += step, ++c) {
        const int b = (int)(c & 1);
        const int64_t nvc = std::min(step, nv - v);
        CUDA_OK(ctx, cudaStreamWaitEvent(L.copy_stream, L.ev_done[b], 0));
        CUDA_OK(ctx, cudaMemcpyAsync(dst[b], rows + (size_t)v * stride, (size_t)(nvc * stride), cudaMemcpyHostToDevice,
                                     L.copy_stream));
        CUDA_OK(ctx, cudaEventRecord(L.ev_copy[b], L.copy_stream));
        ctx->c_h2d += nvc * stride;
        CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, L.ev_copy[b], 0));
        if (int rc = work(b, dst[b], v, nvc)) return rc;
        CUDA_OK(ctx, cudaEventRecord(L.ev_done[b], L.stream));
    }
    CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
    return VPCA_OK;
}

// The argument checks of every packed-row call: nv >= 0, the rows and the outputs (outs_set) given when nv > 0, and rows
// at least min_stride bytes apart.  The message names fn.
int rows_args(vpca_ctx* ctx, const char* fn, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int64_t min_stride,
              bool outs_set = true) {
    if (nv < 0 || (nv > 0 && (rows == nullptr || !outs_set)) || stride_bytes < min_stride)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: bad argument (nv = %lld must be >= 0, rows and outputs set when nv > 0, "
                    "stride_bytes = %lld >= %lld)", fn, (long long)nv, (long long)stride_bytes, (long long)min_stride);
    return VPCA_OK;
}

// The context's staging pair for driver-side calls (d_bed_rows); calls on task threads use their lane's L.d_idx instead.
std::array<uint8_t*, 2> bed_rows(vpca_ctx* ctx) { return {ctx->d_bed_rows[0].get(), ctx->d_bed_rows[1].get()}; }

// Raw rows in the lane's index buffers (the packed accumulate, loadings and projection calls, and kinship).
std::array<uint8_t*, 2> lane_rows(vpca_ctx::Lane& L) {
    return {reinterpret_cast<uint8_t*>(L.d_idx[0].get()), reinterpret_cast<uint8_t*>(L.d_idx[1].get())};
}

// Packed rows (code 0: bitmaps; 1 / 2: PLINK .bed rows counting A1 / A2, see encode.cu) -> encode -> consume(chunk), on
// lane L; returns after the lane's stream has drained (the caller's buffer is free to reuse).
int process_packed(vpca_ctx* ctx, vpca_ctx::Lane& L, const uint8_t* bits, int64_t nv, int64_t stride_bytes, int code,
                   const ChunkFn& consume) {
    // bits beyond sample n-1 in the last byte of a row would be read as carriers of non-existent samples: the kernel
    // masks them (smp >= n), nothing to validate on the host.
    const int64_t P = ctx->panel;
    const int64_t cap_rows = std::min<int64_t>(ctx->chunk_variants, (ctx->chunk_nnz * (int64_t)sizeof(int32_t)) / stride_bytes);
    if (cap_rows < 32) return fail(ctx, VPCA_ERR_BAD_ARG, "stride_bytes too large for the staging buffer");
    const int64_t whole = std::max<int64_t>(P, (cap_rows / P) * P);
    const int64_t step = whole <= cap_rows ? whole : (cap_rows / 32) * 32;
    return stage_rows(ctx, L, bits, nv, stride_bytes, step, lane_rows(L), [&](int b, const uint8_t* d_rows, int64_t v, int64_t nvc) -> int {
        CUDA_OK(ctx, encode_bits(d_rows, stride_bytes, nvc, ctx->n, ctx->elem_bits, L.d_x[b].get(), P, P, code, L.stream));
        ctx->c_launches += 1;
        return consume(L, b, v, nvc);
    });
}

}  // namespace

extern "C" {

int vpca_version(void) { return VPCA_VERSION_MAJOR * 1000 + VPCA_VERSION_MINOR; }

const char* vpca_last_error(const vpca_ctx* ctx) {
    // a thread that just failed on `ctx` reads its own message, whatever other threads have done to the context since
    if (ctx == nullptr || tls_error_ctx == ctx) return tls_error.c_str();
    vpca_ctx* c = const_cast<vpca_ctx*>(ctx);
    std::lock_guard<std::mutex> lk(c->err_mu);
    tls_error_copy = c->err;
    return tls_error_copy.c_str();
}

int vpca_create(const vpca_config* cfg, vpca_ctx** out) {
    if (out == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "out is NULL");
    *out = nullptr;
    if (cfg == nullptr || cfg->struct_size != sizeof(vpca_config))
        return fail(nullptr, VPCA_ERR_BAD_ARG, "cfg is NULL or struct_size != sizeof(vpca_config) (%zu)",
                    sizeof(vpca_config));
    if (cfg->n_samples < 2) return fail(nullptr, VPCA_ERR_BAD_ARG, "n_samples must be >= 2");
    if (cfg->dtype != VPCA_DTYPE_I8 && cfg->dtype != VPCA_DTYPE_BF16 && cfg->dtype != VPCA_DTYPE_E2M1)
        return fail(nullptr, VPCA_ERR_BAD_ARG, "unknown dtype %d", cfg->dtype);
    if (cfg->staging_lanes < 0 || cfg->staging_lanes > 16)
        return fail(nullptr, VPCA_ERR_BAD_ARG, "staging_lanes must be in [0, 16]");
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return fail(nullptr, VPCA_ERR_CUDA, "no CUDA device: %s (libvpca has no CPU fallback)", cudaGetErrorString(e));
    if (cfg->device < 0 || cfg->device >= ndev) return fail(nullptr, VPCA_ERR_BAD_ARG, "device %d of %d", cfg->device, ndev);
    CUDA_OK(nullptr, cudaSetDevice(cfg->device));
    cudaDeviceProp prop;
    CUDA_OK(nullptr, cudaGetDeviceProperties(&prop, cfg->device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(nullptr, VPCA_ERR_UNSUPPORTED, "device %d is sm_%d%d; libvpca is built for sm_90a (H100) only",
                    cfg->device, prop.major, prop.minor);
    vpca_ctx* ctx = new (std::nothrow) vpca_ctx();
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_NOMEM, "out of host memory");
    ctx->cfg = *cfg;
    ctx->n = cfg->n_samples;
    ctx->elem_bits = cfg->dtype == VPCA_DTYPE_I8 ? 8 : (cfg->dtype == VPCA_DTYPE_BF16 ? 16 : 4);
    ctx->max_mult = cfg->max_multiplicity > 0 ? cfg->max_multiplicity : 2;
    ctx->num_pc = cfg->num_pc > 0 ? cfg->num_pc : 2;
    if (ctx->elem_bits == 4 && ctx->max_mult > 2) {
        delete ctx;
        return fail(nullptr, VPCA_ERR_BAD_ARG, "VPCA_DTYPE_E2M1 represents multiplicities 0, 1, 2 only (max_multiplicity <= 2)");
    }
    if (ctx->elem_bits != 8 && 16777216ll / ((int64_t)ctx->max_mult * ctx->max_mult) < 8192) {
        // fp32 tensor accumulation is exact below 2^24 only: a launch folds at least one panel (8192 variants), so the
        // largest count of one panel, 8192 * max_mult^2, must stay below that (bf16: max_multiplicity <= 45)
        const int mm = ctx->max_mult;
        delete ctx;
        return fail(nullptr, VPCA_ERR_BAD_ARG, "max_multiplicity %d is too large for exact fp32 accumulation of bf16 cells "
                    "(<= 45); use VPCA_DTYPE_I8", mm);
    }
    const bool band = cfg->gram_band_rows > 0;
    if (band && (cfg->d_gram != nullptr || cfg->gram_band_row0 < 0 || cfg->gram_band_row0 + cfg->gram_band_rows > ctx->n)) {
        delete ctx;
        return fail(nullptr, VPCA_ERR_BAD_ARG, "gram_band_row0/rows must lie in [0, n_samples] and need a library-owned Gram");
    }
    ctx->band_row0 = band ? cfg->gram_band_row0 : 0;
    ctx->band_rows = band ? cfg->gram_band_rows : ctx->n;
    if (band) {   // without peers the Gram kernel computes exactly these rows (owner-computes), with peers it flushes to owners
        ctx->plan.own_lo = ctx->band_row0;
        ctx->plan.own_hi = ctx->band_row0 + ctx->band_rows;
    }
    if (cfg->stream != nullptr) {
        ctx->stream = static_cast<cudaStream_t>(cfg->stream);
    } else {
        e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking);
        ctx->own_stream = true;
    }
    const size_t gram_cells = (size_t)ctx->band_rows * ctx->n;
    if (e == cudaSuccess) {
        if (cfg->d_gram != nullptr) {
            ctx->d_S = static_cast<int32_t*>(cfg->d_gram);
        } else {
            e = ctx->owned_S.ensure((int64_t)gram_cells + 64);   // + barrier flags of the peer-reduce mode
            ctx->d_S = ctx->owned_S.get();
            if (e == cudaSuccess) e = cudaMemsetAsync(ctx->d_S + gram_cells, 0, 64 * sizeof(int32_t), ctx->stream);
        }
    }
    if (e == cudaSuccess) e = cudaMemsetAsync(ctx->d_S, 0, gram_cells * sizeof(int32_t), ctx->stream);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev_t0);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev_t1);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev_e0);
    if (e == cudaSuccess) e = cudaEventCreate(&ctx->ev_e1);
    if (e != cudaSuccess) {
        const int rc = fail(nullptr, e == cudaErrorMemoryAllocation ? VPCA_ERR_NOMEM : VPCA_ERR_CUDA, "vpca_create: %s",
                            cudaGetErrorString(e));
        vpca_destroy(ctx);
        return rc;
    }
    const int nslots = cfg->partitions_in_flight > 0 ? cfg->partitions_in_flight : 4;
    ctx->slots.resize(nslots);
    ctx->lanes.resize(cfg->staging_lanes > 0 ? cfg->staging_lanes : 2);
    *out = ctx;
    return VPCA_OK;
}

int vpca_destroy(vpca_ctx* ctx) {
    if (ctx == nullptr) return VPCA_OK;
    cudaSetDevice(ctx->cfg.device);
    if (ctx->stream) cudaStreamSynchronize(ctx->stream);
    for (auto& L : ctx->lanes) free_lane(L);
    for (auto& s : ctx->slots)
        if (s.ev_free) cudaEventDestroy(s.ev_free);
    if (ctx->plan.peers_ipc)
        for (int d = 0; d < ctx->plan.num_peers; ++d)
            if (d != ctx->plan.peer_rank && ctx->plan.peer_S[d] != nullptr) cudaIpcCloseMemHandle(ctx->plan.peer_base[d]);
    if (ctx->eig_ready) eig_free(ctx->eig);
    band_eig_free(ctx->band_eig);
    band_part_free(ctx->band_part);
    if (ctx->sub_eig.n != 0) eig_free(ctx->sub_eig);
    join_free(ctx->join);
    gram_plan_free(ctx->kin_plan);
    for (cudaEvent_t ev : {ctx->sm_ev_copy[0], ctx->sm_ev_copy[1], ctx->sm_ev_kern[0], ctx->sm_ev_kern[1]})
        if (ev) cudaEventDestroy(ev);
    if (ctx->sm_d2h_stream) cudaStreamDestroy(ctx->sm_d2h_stream);
    gram_plan_free(ctx->ld_plan);
    gram_plan_free(ctx->plan);
    for (cudaEvent_t ev : {ctx->ev_t0, ctx->ev_t1, ctx->ev_e0, ctx->ev_e1})
        if (ev) cudaEventDestroy(ev);
    if (ctx->own_stream && ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;   // frees every device buffer, on the device selected above
    return VPCA_OK;
}

int vpca_synchronize(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return VPCA_OK;
}

int vpca_reset(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> jl(ctx->join_mu);   // lock order everywhere: join_mu, then mu
    std::lock_guard<std::mutex> lk(ctx->mu);
    for (auto& L : ctx->lanes)
        if (L.busy) return fail(ctx, VPCA_ERR_STATE, "vpca_reset while an accumulate call is in flight");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaMemsetAsync(ctx->d_S, 0, (size_t)ctx->band_rows * ctx->n * sizeof(int32_t), ctx->stream));
    if (ctx->d_kin.get() != nullptr)
        CUDA_OK(ctx, cudaMemsetAsync(ctx->d_kin.get(), 0, (size_t)9 * ctx->n * ctx->n * sizeof(int32_t), ctx->stream));
    ctx->kin_variants = 0;
    ctx->grm_state = 0;
    ctx->grm_used = 0;
    ctx->grm_fill = 0;
    for (auto& s : ctx->slots) s.used = false;
    ctx->finalized = false;
    ctx->pca_done = false;
    ctx->pca_k = 0;
    ctx->grm_k = 0;
    ctx->proj_k = 0;
    ctx->glm_q = 0;
    ctx->total_variants = 0;
    ctx->inflight_variants = 0;
    ctx->st.variants_accumulated = 0;
    ctx->join.out_rows = -1;   // joined rows of an earlier analysis do not outlive a reset (join_mu is held, see above)
    return VPCA_OK;
}

int vpca_encode_calls(vpca_ctx* ctx, const int64_t* offsets, const int32_t* sample_idx, int64_t nv, void* out,
                      int64_t ld) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (offsets == nullptr || out == nullptr || nv < 0 || ld < nv || (nv > 0 && sample_idx == nullptr && offsets[nv] > offsets[0]))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_encode_calls: bad argument");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    const int bits = ctx->elem_bits;
    const int64_t P = ctx->panel;
    // panel layout -> the caller's row-major tile, one 2-D copy per panel (chunk boundaries are multiples of 128
    // variants, so 4-bit rows split on byte boundaries)
    auto copy_out = [&](vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc) -> int {
        for (int64_t pv = 0; pv < nvc; pv += P) {
            const int64_t wv = std::min(P, nvc - pv);
            CUDA_OK(ctx, cudaMemcpy2DAsync(static_cast<char*>(out) + (size_t)(v + pv) * bits / 8, (size_t)ld * bits / 8,
                                           L.d_x[b].get() + (size_t)(pv / P) * ctx->n * P * bits / 8,
                                           (size_t)P * bits / 8, (size_t)(wv * bits + 7) / 8, (size_t)ctx->n,
                                           cudaMemcpyDeviceToHost, L.stream));
        }
        ctx->c_d2h += (nvc * bits + 7) / 8 * (int64_t)ctx->n;
        return VPCA_OK;
    };
    return process_calls(ctx, *lg.lane, offsets, sample_idx, 4, nv, copy_out, false);
}

static int accumulate_calls_impl(vpca_ctx* ctx, int64_t partition_id, const int64_t* offsets, const void* sample_idx,
                                 int idx_bytes, int64_t nv) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (offsets == nullptr || nv < 0 || (nv > 0 && sample_idx == nullptr && offsets[nv] > offsets[0]))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_accumulate_calls: bad argument");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
        return VPCA_OK;
    }
    CallScope sc{ctx, partition_id, nv};
    int rc = sc.begin();
    if (rc != VPCA_OK) return rc;
    {
        LaneGuard lg(ctx);
        rc = lg.rc;
        if (rc == VPCA_OK) rc = prepare_slot(ctx, *lg.lane, sc);
        auto gram = [&](vpca_ctx::Lane& L, int b, int64_t, int64_t nvc) -> int {
            return launch_gram(ctx, L.plan, L.stream, L.ev_t0, L.ev_t1, L.d_x[b].get(), nvc, ctx->panel, ctx->panel, sc.target);
        };
        if (rc == VPCA_OK) rc = process_calls(ctx, *lg.lane, offsets, sample_idx, idx_bytes, nv, gram, true);
    }
    return sc.end(rc);
}

int vpca_accumulate_calls(vpca_ctx* ctx, int64_t partition_id, const int64_t* offsets, const int32_t* sample_idx,
                          int64_t nv) {
    return accumulate_calls_impl(ctx, partition_id, offsets, sample_idx, 4, nv);
}

int vpca_accumulate_calls_u16(vpca_ctx* ctx, int64_t partition_id, const int64_t* offsets, const uint16_t* sample_idx,
                              int64_t nv) {
    if (ctx != nullptr && ctx->n > 65536) return fail(ctx, VPCA_ERR_BAD_ARG, "16-bit sample indices need n_samples <= 65536");
    return accumulate_calls_impl(ctx, partition_id, offsets, sample_idx, 2, nv);
}

// code 0: bitmap rows; 1 / 2: PLINK .bed rows counting A1 / A2 (see encode.cu)
static int accumulate_packed(vpca_ctx* ctx, int64_t partition_id, const uint8_t* bits, int64_t nv, int64_t stride_bytes,
                             int code) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (int rc = rows_args(ctx, code == 0 ? "vpca_accumulate_bits" : "vpca_accumulate_bed", bits, nv, stride_bytes,
                           code == 0 ? (ctx->n + 7) / 8 : (ctx->n + 3) / 4))
        return rc;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
        return VPCA_OK;
    }
    CallScope sc{ctx, partition_id, nv};
    int rc = sc.begin();
    if (rc != VPCA_OK) return rc;
    auto body = [&](vpca_ctx::Lane& L) -> int {
        int r = prepare_slot(ctx, L, sc);
        if (r != VPCA_OK) return r;
        auto gram = [&](vpca_ctx::Lane& L2, int b, int64_t, int64_t nvc) -> int {
            return launch_gram(ctx, L2.plan, L2.stream, L2.ev_t0, L2.ev_t1, L2.d_x[b].get(), nvc, ctx->panel, ctx->panel, sc.target);
        };
        r = process_packed(ctx, L, bits, nv, stride_bytes, code, gram);
        if (r != VPCA_OK) return r;
        lane_gram_time(ctx, L);
        return VPCA_OK;
    };
    {
        LaneGuard lg(ctx);
        rc = lg.rc;
        if (rc == VPCA_OK) rc = body(*lg.lane);
    }
    return sc.end(rc);
}

int vpca_accumulate_bits(vpca_ctx* ctx, int64_t partition_id, const uint8_t* bits, int64_t nv, int64_t stride_bytes) {
    return accumulate_packed(ctx, partition_id, bits, nv, stride_bytes, 0);
}

int vpca_accumulate_bed(vpca_ctx* ctx, int64_t partition_id, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                        int32_t counted_allele) {
    if (counted_allele != 1 && counted_allele != 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_accumulate_bed: counted_allele must be 1 (A1) or 2 (A2)");
    return accumulate_packed(ctx, partition_id, rows, nv, stride_bytes, counted_allele);
}

// ---- multi-dataset keying (join.cu) -----------------------------------------------------------------------------
int vpca_hash_keys(vpca_ctx* ctx, const uint8_t* payload, const int64_t* key_offsets, int64_t nkeys, uint64_t* out) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (nkeys < 0 || key_offsets == nullptr || (nkeys > 0 && out == nullptr))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_hash_keys: bad argument");
    if (nkeys == 0) return VPCA_OK;
    for (int64_t q = 0; q < nkeys; ++q)
        if (key_offsets[q + 1] < key_offsets[q] || key_offsets[0] < 0)
            return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_hash_keys: key_offsets must be non-negative and non-decreasing (key %lld)", (long long)q);
    const int64_t bytes = key_offsets[nkeys] - key_offsets[0];
    if (bytes > 0 && payload == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_hash_keys: payload is NULL");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    DeviceBuffer<uint8_t> d_pay;
    DeviceBuffer<int64_t> d_koff;
    DeviceBuffer<uint64_t> d_out;
    cudaError_t e = d_pay.ensure(bytes + 16);
    if (e == cudaSuccess) e = d_koff.ensure(nkeys + 1);
    if (e == cudaSuccess) e = d_out.ensure(2 * nkeys);
    if (e == cudaSuccess && bytes > 0)
        e = cudaMemcpyAsync(d_pay.get(), payload + key_offsets[0], (size_t)bytes, cudaMemcpyHostToDevice, ctx->stream);
    if (e == cudaSuccess)
        e = cudaMemcpyAsync(d_koff.get(), key_offsets, (size_t)(nkeys + 1) * 8, cudaMemcpyHostToDevice, ctx->stream);
    // the device copy starts at the first key: shift the base pointer instead of rebasing the offsets
    if (e == cudaSuccess) e = hash_keys(d_pay.get() - key_offsets[0], d_koff.get(), nkeys, d_out.get(), ctx->stream);
    if (e == cudaSuccess) e = cudaMemcpyAsync(out, d_out.get(), (size_t)nkeys * 16, cudaMemcpyDeviceToHost, ctx->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) return fail(ctx, VPCA_ERR_CUDA, "vpca_hash_keys: %s", cudaGetErrorString(e));
    ctx->c_launches += 1;
    ctx->c_h2d += bytes + (nkeys + 1) * 8;
    ctx->c_d2h += nkeys * 16;
    return VPCA_OK;
}

int vpca_join_rows(vpca_ctx* ctx, int32_t mode, int32_t variant_set_count, int64_t n_left, const uint8_t* key_payload,
                   const int64_t* key_offsets, const int64_t* offsets, const int32_t* sample_idx, int64_t nrows,
                   int64_t* out_rows, int64_t* out_nnz) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if ((mode != VPCA_JOIN && mode != VPCA_MERGE) || nrows < 0 || nrows > 0x7ffffff0ll || key_offsets == nullptr ||
        offsets == nullptr || out_rows == nullptr || out_nnz == nullptr)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: bad argument");
    if (mode == VPCA_JOIN && (n_left < 0 || n_left > nrows))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: n_left must be in [0, nrows]");
    if (mode == VPCA_MERGE && variant_set_count < 1)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: variant_set_count must be >= 1");
    if (key_offsets[0] < 0 || offsets[0] < 0) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: negative offset");
    for (int64_t q = 0; q < nrows; ++q)
        if (key_offsets[q + 1] < key_offsets[q] || offsets[q + 1] < offsets[q])
            return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: offsets must be non-decreasing (row %lld)", (long long)q);
    const int64_t kbytes = key_offsets[nrows] - key_offsets[0], nnz = offsets[nrows] - offsets[0];
    if ((kbytes > 0 && key_payload == nullptr) || (nnz > 0 && sample_idx == nullptr))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_join_rows: NULL payload");
    std::lock_guard<std::mutex> jl(ctx->join_mu);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    JoinWork& w = ctx->join;
    w.out_rows = -1;
    CUDA_OK(ctx, w.d_payload.ensure(kbytes + 16, with_slack(kbytes + 16)));
    CUDA_OK(ctx, w.d_key_off.ensure(nrows + 1, with_slack(nrows)));
    CUDA_OK(ctx, w.d_off.ensure(nrows + 1, with_slack(nrows)));
    CUDA_OK(ctx, w.d_idx.ensure(nnz + 1, with_slack(nnz + 1)));
    if (kbytes > 0)
        CUDA_OK(ctx, cudaMemcpyAsync(w.d_payload.get(), key_payload + key_offsets[0], (size_t)kbytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(w.d_key_off.get(), key_offsets, (size_t)(nrows + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(w.d_off.get(), offsets, (size_t)(nrows + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (nnz > 0)
        CUDA_OK(ctx, cudaMemcpyAsync(w.d_idx.get(), sample_idx + offsets[0], (size_t)nnz * 4, cudaMemcpyHostToDevice, ctx->stream));
    ctx->c_h2d += kbytes + 2 * (nrows + 1) * 8 + nnz * 4;
    int64_t launches = 0, rows = 0, calls = 0;
    // the device copies start at the first key / first call: shift the base pointers instead of rebasing the offsets
    cudaError_t e = join_rows(w, mode, variant_set_count, n_left, w.d_payload.get() - key_offsets[0], w.d_key_off.get(), w.d_off.get(),
                              w.d_idx.get() - offsets[0], nrows, ctx->stream, &rows, &calls, &launches);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);   // the caller's buffers were read asynchronously
    ctx->c_launches += launches;
    if (e != cudaSuccess)
        return fail(ctx, e == cudaErrorMemoryAllocation ? VPCA_ERR_NOMEM : VPCA_ERR_CUDA, "vpca_join_rows: %s", cudaGetErrorString(e));
    w.out_rows = rows;
    w.out_nnz = calls;
    *out_rows = rows;
    *out_nnz = calls;
    return VPCA_OK;
}

int vpca_join_fetch(vpca_ctx* ctx, int64_t* out_offsets, int32_t* out_idx) {
    if (ctx == nullptr || out_offsets == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> jl(ctx->join_mu);
    JoinWork& w = ctx->join;
    if (w.out_rows < 0) return fail(ctx, VPCA_ERR_STATE, "no joined rows: call vpca_join_rows first");
    if (w.out_nnz > 0 && out_idx == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "out_idx is NULL");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaMemcpyAsync(out_offsets, w.d_out_off.get(), (size_t)(w.out_rows + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (w.out_nnz > 0)
        CUDA_OK(ctx, cudaMemcpyAsync(out_idx, w.d_out_idx.get(), (size_t)w.out_nnz * 4, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (w.out_rows + 1) * 8 + w.out_nnz * 4;
    return VPCA_OK;
}

int vpca_join_size(vpca_ctx* ctx, int64_t* out_rows, int64_t* out_nnz) {
    if (ctx == nullptr || out_rows == nullptr || out_nnz == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> jl(ctx->join_mu);
    if (ctx->join.out_rows < 0) return fail(ctx, VPCA_ERR_STATE, "no joined rows: call vpca_join_rows first");
    *out_rows = ctx->join.out_rows;
    *out_nnz = ctx->join.out_nnz;
    return VPCA_OK;
}

int vpca_accumulate_joined(vpca_ctx* ctx, int64_t partition_id) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> jl(ctx->join_mu);
    JoinWork& w = ctx->join;
    if (w.out_rows < 0) return fail(ctx, VPCA_ERR_STATE, "no joined rows: call vpca_join_rows first");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const int64_t nv = w.out_rows;
    if (nv == 0) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
        return VPCA_OK;
    }
    CallScope sc{ctx, partition_id, nv};
    int rc = sc.begin();
    if (rc != VPCA_OK) return rc;
    auto body = [&](vpca_ctx::Lane& L) -> int {
        int r = prepare_slot(ctx, L, sc);
        if (r != VPCA_OK) return r;
        *L.h_flags = 0;
        CUDA_OK(ctx, cudaMemsetAsync(L.d_flags.get(), 0, sizeof(int), L.stream));
        const int64_t P = ctx->panel;
        int chunk = 0;
        for (int64_t v = 0; v < nv; v += ctx->chunk_variants, ++chunk) {
            const int64_t nvc = std::min(ctx->chunk_variants, nv - v);
            const int b = chunk & 1;
            // the joined CSR is device-resident: rows [v, v + nvc) are encoded straight from it (absolute offsets, base 0)
            CUDA_OK(ctx, encode_calls(w.d_out_off.get() + v, 0, w.d_out_idx.get(), 4, nvc, ctx->n, ctx->elem_bits, ctx->max_mult, L.d_x[b].get(),
                                      P, P, L.d_flags.get(), L.stream));
            ctx->c_launches += 2;
            r = launch_gram(ctx, L.plan, L.stream, L.ev_t0, L.ev_t1, L.d_x[b].get(), nvc, P, P, sc.target);
            if (r != VPCA_OK) return r;
        }
        CUDA_OK(ctx, cudaMemcpyAsync(L.h_flags, L.d_flags.get(), sizeof(int), cudaMemcpyDeviceToHost, L.stream));
        CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
        lane_gram_time(ctx, L);
        if (*L.h_flags & 1)
            return fail(ctx, VPCA_ERR_INDEX_OUT_OF_RANGE, "sample index outside [0, %d) (the reference throws at "
                        "VariantsPca.scala:59/:188)", ctx->n);
        if (*L.h_flags & 2)
            return fail(ctx, VPCA_ERR_OVERFLOW, "a sample is listed more than max_multiplicity=%d times in one joined row "
                        "(a sample present in both datasets counts twice, VariantsPca.scala:127/:187)", ctx->max_mult);
        return VPCA_OK;
    };
    {
        LaneGuard lg(ctx);   // orders the lane after the join kernels on the context's stream
        rc = lg.rc;
        if (rc == VPCA_OK) rc = body(*lg.lane);
    }
    return sc.end(rc);
}

int vpca_commit(vpca_ctx* ctx, int64_t partition_id) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized");
    int rc;
    vpca_ctx::Slot* s = find_slot(ctx, partition_id, false, &rc);
    if (s == nullptr) return VPCA_OK;   // an empty partition never staged anything
    if (s->busy) return fail(ctx, VPCA_ERR_STATE, "partition %lld still has an accumulate call in flight", (long long)partition_id);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    // the partition's variants were reserved against the int32 bound when they were staged (CallScope::begin)
    if (s->nv > 0) {
        // every accumulate call of the partition synchronised its lane before returning: the staging Gram is complete
        if (ctx->plan.num_peers > 1 && ctx->plan.peer_mode == 1)
            CUDA_OK(ctx, gram_add_owners(ctx->plan, s->d_S.get(), ctx->n, ctx->stream));
        else if (ctx->plan.num_peers > 1)
            CUDA_OK(ctx, gram_add_peers(ctx->plan, s->d_S.get(), (int64_t)ctx->n * ctx->n, ctx->stream));
        else   // an owner-computes band staged only its own rows, at the band Gram's own offsets
            CUDA_OK(ctx, gram_add(ctx->d_S, s->d_S.get(), (int64_t)ctx->band_rows * ctx->n, ctx->stream));
        CUDA_OK(ctx, cudaEventRecord(s->ev_free, ctx->stream));
        ctx->c_launches += 1;
    }
    ctx->total_variants += s->nv;
    ctx->inflight_variants -= s->nv;
    s->used = false;
    return VPCA_OK;
}

int vpca_abort(vpca_ctx* ctx, int64_t partition_id) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    int rc;
    vpca_ctx::Slot* s = find_slot(ctx, partition_id, false, &rc);
    if (s != nullptr) {
        if (s->busy) return fail(ctx, VPCA_ERR_STATE, "partition %lld still has an accumulate call in flight", (long long)partition_id);
        ctx->st.variants_accumulated -= s->nv;
        ctx->inflight_variants -= s->nv;
        s->used = false;
    }
    return VPCA_OK;
}

int vpca_accumulate_dense(vpca_ctx* ctx, const void* x, int64_t nv, int64_t ld, int on_device) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (x == nullptr || nv < 0 || ld < nv) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_accumulate_dense: bad argument");
    const int bits = ctx->elem_bits;
    if (bits == 4 && (ld % 128) != 0)
        return fail(ctx, VPCA_ERR_BAD_ARG, "packed e2m1 tiles need ld %% 128 == 0 (and zero padding up to a multiple of 128 variants)");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (on_device) {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
        if (nv == 0) return VPCA_OK;
        int rc = check_overflow(ctx, nv);
        if (rc != VPCA_OK) return rc;
        const int align = bits == 4 ? 31 : 15;
        if ((reinterpret_cast<uintptr_t>(x) & align) != 0 || ((ld * bits / 8) & align) != 0)
            return fail(ctx, VPCA_ERR_BAD_ARG, "device tile must be %d-byte aligned with a %d-byte multiple row pitch",
                        align + 1, align + 1);
        rc = launch_gram(ctx, ctx->plan, ctx->stream, ctx->ev_t0, ctx->ev_t1, x, nv, ld, 0, ctx->d_S);
        if (rc != VPCA_OK) return rc;
        ctx->gram_timed = true;
        ctx->st.gram_cta_group = ctx->plan.cta_group;
        ctx->st.gram_resident = ctx->plan.last_resident;
        ctx->total_variants += nv;
        ctx->st.variants_accumulated += nv;
        return VPCA_OK;
    }
    if (nv == 0) return VPCA_OK;
    CallScope sc{ctx, -1, nv};
    int rc = sc.begin();
    if (rc != VPCA_OK) return rc;
    auto body = [&](vpca_ctx::Lane& L) -> int {
        int chunk = 0;
        for (int64_t v = 0; v < nv; v += ctx->chunk_variants, ++chunk) {
            const int64_t nvc = std::min(ctx->chunk_variants, nv - v);
            const int b = chunk & 1;
            CUDA_OK(ctx, cudaStreamWaitEvent(L.copy_stream, L.ev_done[b], 0));
            // the caller's row-major tile -> panel layout, one 2-D copy per panel; a partial last panel is zeroed first
            const int64_t P = ctx->panel;
            if ((nvc % P) != 0)
                CUDA_OK(ctx, cudaMemsetAsync(L.d_x[b].get() + (size_t)(nvc / P) * ctx->n * P * bits / 8, 0,
                                             (size_t)ctx->n * P * bits / 8, L.copy_stream));
            for (int64_t pv = 0; pv < nvc; pv += P) {
                const int64_t wv = std::min(P, nvc - pv);
                CUDA_OK(ctx, cudaMemcpy2DAsync(L.d_x[b].get() + (size_t)(pv / P) * ctx->n * P * bits / 8,
                                               (size_t)P * bits / 8, static_cast<const char*>(x) + (size_t)(v + pv) * bits / 8,
                                               (size_t)ld * bits / 8, (size_t)(wv * bits + 7) / 8, (size_t)ctx->n,
                                               cudaMemcpyHostToDevice, L.copy_stream));
            }
            CUDA_OK(ctx, cudaEventRecord(L.ev_copy[b], L.copy_stream));
            ctx->c_h2d += (nvc * bits + 7) / 8 * (int64_t)ctx->n;
            CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, L.ev_copy[b], 0));
            int r = launch_gram(ctx, L.plan, L.stream, L.ev_t0, L.ev_t1, L.d_x[b].get(), nvc, P, P, ctx->d_S);
            if (r != VPCA_OK) return r;
            CUDA_OK(ctx, cudaEventRecord(L.ev_done[b], L.stream));
        }
        CUDA_OK(ctx, cudaStreamSynchronize(L.stream));   // caller's buffer is free to reuse on return
        lane_gram_time(ctx, L);
        return VPCA_OK;
    };
    {
        LaneGuard lg(ctx);
        rc = lg.rc;
        if (rc == VPCA_OK) rc = body(*lg.lane);
    }
    return sc.end(rc);
}

int vpca_accumulate_panels(vpca_ctx* ctx, const void* d_x, int64_t nv, int64_t panel_variants) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (d_x == nullptr || nv < 0 || panel_variants < 128 || (panel_variants % 128) != 0)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_accumulate_panels: panel_variants must be a positive multiple of 128");
    if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
    if ((reinterpret_cast<uintptr_t>(d_x) & 31) != 0) return fail(ctx, VPCA_ERR_BAD_ARG, "panels must be 32-byte aligned");
    // a band-only Gram either has peers in owner-rows mode (every context gets a variant shard and flushes each row to
    // its owner) or no peers at all (owner-computes: every context gets ALL variants and produces only its own rows)
    if (ctx->band_rows != ctx->n && ctx->plan.num_peers > 1 && ctx->plan.peer_mode != 1)
        return fail(ctx, VPCA_ERR_STATE, "a band-only Gram with peers needs VPCA_PEER_OWNER_ROWS");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    int rc = check_overflow(ctx, nv);
    if (rc != VPCA_OK) return rc;
    rc = launch_gram(ctx, ctx->plan, ctx->stream, ctx->ev_t0, ctx->ev_t1, d_x, nv, panel_variants, panel_variants, ctx->d_S);
    if (rc != VPCA_OK) return rc;
    ctx->gram_timed = true;
    ctx->st.gram_cta_group = ctx->plan.cta_group;
    ctx->st.gram_resident = ctx->plan.last_resident;
    ctx->total_variants += nv;
    ctx->st.variants_accumulated += nv;
    return VPCA_OK;
}

int vpca_synth_panels_device(vpca_ctx* ctx, uint64_t seed, int64_t v0, int64_t nv, int mode, void* d_x,
                             int64_t panel_variants) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (d_x == nullptr || nv < 0 || v0 < 0 || (mode != 0 && mode != 1) || panel_variants < 128 || (panel_variants % 128) != 0)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_synth_panels_device: bad argument");
    if (mode == 1 && ctx->max_mult < 2) return fail(ctx, VPCA_ERR_BAD_ARG, "dosage mode needs max_multiplicity >= 2");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    cudaError_t e = synth_dense(seed, ctx->n, v0, nv, mode, ctx->elem_bits, d_x, panel_variants, panel_variants, ctx->stream);
    if (e != cudaSuccess) return fail(ctx, VPCA_ERR_CUDA, "synthetic generator: %s", cudaGetErrorString(e));
    ctx->c_launches += 2 * ((nv + (1 << 22) - 1) >> 22);
    return VPCA_OK;
}

int vpca_gram_device_ptr(vpca_ctx* ctx, void** d_gram) {
    if (ctx == nullptr || d_gram == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    *d_gram = ctx->d_S;
    return VPCA_OK;
}

int vpca_finalize_gram(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->finalized) return VPCA_OK;
    for (auto& s : ctx->slots)
        if (s.used)
            return fail(ctx, VPCA_ERR_STATE, "partition %lld is neither committed nor aborted", (long long)s.pid);
    for (auto& L : ctx->lanes)
        if (L.busy) return fail(ctx, VPCA_ERR_STATE, "vpca_finalize_gram while an accumulate call is in flight");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (ctx->band_rows == ctx->n) {   // a row band stays a band of the lower triangle: nothing to mirror into
        CUDA_OK(ctx, gram_symmetrize(ctx->d_S, ctx->n, ctx->stream));
        ctx->c_launches += 1;
    }
    ctx->finalized = true;
    ctx->pca_done = false;
    ctx->pca_k = 0;
    ctx->grm_k = 0;
    return VPCA_OK;
}

static int copy_gram_out(vpca_ctx* ctx, int32_t* out, size_t cells) {
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaMemcpyAsync(out, ctx->d_S, cells * sizeof(int32_t), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)(cells * sizeof(int32_t));
    return VPCA_OK;
}

int vpca_get_gram(vpca_ctx* ctx, int32_t* out) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "call vpca_finalize_gram first");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band: use vpca_get_gram_band");
    return copy_gram_out(ctx, out, (size_t)ctx->n * ctx->n);
}

int vpca_get_gram_band(vpca_ctx* ctx, int32_t row0, int32_t rows, int32_t* out) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (rows <= 0 || row0 < ctx->band_row0 || row0 + rows > ctx->band_row0 + ctx->band_rows)
        return fail(ctx, VPCA_ERR_BAD_ARG, "rows [%d, %d) are outside the band [%d, %d) this context stores", row0, row0 + rows,
                    ctx->band_row0, ctx->band_row0 + ctx->band_rows);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t cells = (size_t)rows * ctx->n;
    CUDA_OK(ctx, cudaMemcpyAsync(out, ctx->d_S + (size_t)(row0 - ctx->band_row0) * ctx->n, cells * sizeof(int32_t),
                                 cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)(cells * sizeof(int32_t));
    return VPCA_OK;
}

int vpca_get_partial_gram(vpca_ctx* ctx, int32_t* out, int64_t* variants_in_gram) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized: use vpca_get_gram");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band: use vpca_get_gram_band");
    if (variants_in_gram) *variants_in_gram = ctx->total_variants;
    return copy_gram_out(ctx, out, (size_t)ctx->n * ctx->n);
}

int vpca_load_partial_gram(vpca_ctx* ctx, const int32_t* gram, int64_t variants_in_gram) {
    if (ctx == nullptr || gram == nullptr || variants_in_gram < 0) return fail(ctx, VPCA_ERR_BAD_ARG, "bad argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized; call vpca_reset first");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band");
    for (auto& s : ctx->slots)
        if (s.used) return fail(ctx, VPCA_ERR_STATE, "partition %lld is in flight", (long long)s.pid);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t bytes = (size_t)ctx->n * ctx->n * sizeof(int32_t);
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_S, gram, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_h2d += (int64_t)bytes;
    // the restored counts keep counting against the int32 bound (VariantsPca.scala:185)
    ctx->total_variants = variants_in_gram;
    ctx->inflight_variants = 0;
    ctx->pca_k = 0;
    ctx->grm_k = 0;
    return check_overflow(ctx, 0);
}

int vpca_set_gram(vpca_ctx* ctx, const int32_t* gram) {
    if (ctx == nullptr || gram == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t bytes = (size_t)ctx->n * ctx->n * sizeof(int32_t);
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_S, gram, bytes, cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_h2d += (int64_t)bytes;
    for (auto& s : ctx->slots) s.used = false;
    ctx->inflight_variants = 0;
    ctx->finalized = true;
    ctx->pca_done = false;
    ctx->pca_k = 0;
    ctx->grm_k = 0;
    return VPCA_OK;
}

int64_t vpca_variant_count(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    return ctx->total_variants;
}

static int run_center(vpca_ctx* ctx, bool materialise) {
    if (!ctx->eig_ready) {
        cudaError_t e = eig_alloc(ctx->eig, ctx->n, std::max(ctx->num_pc, 16));
        if (e != cudaSuccess) return fail(ctx, VPCA_ERR_NOMEM, "eigensolver workspace: %s", cudaGetErrorString(e));
        ctx->eig_ready = true;
    }
    CUDA_OK(ctx, center_gram(ctx->eig, ctx->d_S, ctx->stream, materialise));
    ctx->c_launches += materialise ? 3 : 2;
    return VPCA_OK;
}

int vpca_compute_pca(vpca_ctx* ctx, int32_t k, double* vecs, double* evals, int32_t* non_zero_rows) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (vecs == nullptr || k < 1 || k > ctx->n || k > std::max(ctx->num_pc, 16))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_compute_pca: k=%d out of range", k);
    if (!ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "call vpca_finalize_gram first");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band of the Gram");
    if (ctx->n > 65535)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "computePca is limited to 65535 samples, like the reference (MLlib RowMatrix "
                    "behind VariantsPca.scala:226 refuses more columns); the Gram itself has no such limit");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->pca_k = 0;   // U is overwritten from here on
    ctx->grm_k = 0;
    if (ctx->grm_state != 0) ctx->grm_state = 3;   // the solve may use d_C
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e0, ctx->stream));
    int rc = run_center(ctx, false);   // row sums + mean; the solver materialises C only if it needs it
    if (rc != VPCA_OK) return rc;
    {   // VPCA_EIG=direct|lanczos|auto (default auto: Lanczos from 512 samples up, direct reduction as its fallback)
        const char* em = getenv("VPCA_EIG");
        ctx->eig.mode = (em != nullptr && strcmp(em, "direct") == 0) ? 1 : (em != nullptr && strcmp(em, "lanczos") == 0) ? 2 : 0;
    }
    int64_t launches = 0;
    CUDA_OK(ctx, eig_topk(ctx->eig, k, ctx->stream, &launches));
    ctx->c_launches += launches;
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e1, ctx->stream));
    ctx->st.eig_method = ctx->eig.last_method;
    ctx->st.eig_iterations = ctx->eig.last_iters;
    ctx->eig_timed = true;
    const size_t nb = (size_t)ctx->n * k * sizeof(double);
    CUDA_OK(ctx, cudaMemcpyAsync(vecs, ctx->eig.d_evecs.get(), nb, cudaMemcpyDeviceToHost, ctx->stream));
    if (evals) CUDA_OK(ctx, cudaMemcpyAsync(evals, ctx->eig.d_evals.get(), k * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    int nz = 0;
    CUDA_OK(ctx, cudaMemcpyAsync(&nz, ctx->eig.d_nz.get(), sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    if (non_zero_rows) *non_zero_rows = nz;
    ctx->c_d2h += (int64_t)nb + (evals ? k * 8 : 0) + 4;
    ctx->pca_done = true;
    ctx->pca_k = k;
    ctx->d_U = ctx->eig.d_evecs.get();
    return VPCA_OK;
}

int vpca_get_centered(vpca_ctx* ctx, double* out) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "call vpca_finalize_gram first");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "this context stores a row band of the Gram");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (ctx->grm_state != 0) ctx->grm_state = 3;   // d_C is about to hold the centred Gram
    int rc = run_center(ctx, true);   // the eigensolve overwrites C, so recompute it
    if (rc != VPCA_OK) return rc;
    const size_t bytes = (size_t)ctx->n * ctx->n * sizeof(double);
    CUDA_OK(ctx, cudaMemcpyAsync(out, ctx->eig.d_C.get(), bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)bytes;
    ctx->pca_done = false;
    return VPCA_OK;
}

int vpca_get_tridiagonal(vpca_ctx* ctx, double* diag, double* offdiag) {
    if (ctx == nullptr || diag == nullptr || offdiag == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->pca_done) return fail(ctx, VPCA_ERR_STATE, "call vpca_compute_pca first");
    if (ctx->eig.last_method == 2)
        return fail(ctx, VPCA_ERR_STATE, "the last solve used Lanczos and did not tridiagonalise C (set VPCA_EIG=direct)");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaMemcpyAsync(diag, ctx->eig.d_diag.get(), (size_t)ctx->n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(offdiag, ctx->eig.d_off.get(), (size_t)(ctx->n - 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return VPCA_OK;
}

// Principal coordinates of the kept samples K from S[K, K], the removed samples placed from their Gram rows (subset.cu,
// DESIGN.md 8).  The solve is vpca_compute_pca's centring and eigensolver on an m-sample workspace of its own, so the
// kept rows have the bits of vpca_compute_pca in an m-sample context holding S[K, K].
int vpca_compute_pca_subset(vpca_ctx* ctx, const uint8_t* keep, int32_t k, double* vecs, double* evals,
                            int32_t* non_zero_rows) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    // checked in vpca_compute_pca's order: arguments, then the Gram's state, then what the context can hold
    if (keep == nullptr || vecs == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_compute_pca_subset: NULL argument");
    const int n = ctx->n;
    std::vector<int32_t> idx;
    idx.reserve(n);
    for (int s = 0; s < n; ++s)
        if (keep[s]) idx.push_back(s);
    const int m = (int)idx.size();
    for (int s = 0; s < n; ++s)
        if (!keep[s]) idx.push_back(s);
    const int kmax = std::max(ctx->num_pc, 16);
    if (m < 2) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_compute_pca_subset: %d kept samples, at least 2 needed", m);
    if (k < 1 || k > m || k > kmax)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_compute_pca_subset: k=%d out of range [1, %d]", k, std::min(m, kmax));
    if (!ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "call vpca_finalize_gram first");
    if (ctx->band_rows != ctx->n)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "vpca_compute_pca_subset needs a context that stores the whole Gram");
    if (n > 65535)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "vpca_compute_pca_subset is limited to 65535 samples, like vpca_compute_pca");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->pca_k = 0;   // U is overwritten from here on
    ctx->grm_k = 0;
    ctx->pca_done = false;   // the tridiagonal form of ctx->eig does not belong to this solve
    if (ctx->sub_eig.n != m) {
        eig_free(ctx->sub_eig);   // a new subset size: the whole workspace is allocated afresh
        const cudaError_t e = eig_alloc(ctx->sub_eig, m, kmax);
        if (e != cudaSuccess) return fail(ctx, VPCA_ERR_NOMEM, "subset eigensolver workspace: %s", cudaGetErrorString(e));
    }
    {
        // U keeps the 16 columns the loadings read; the output and t take every component a solve may ask for
        cudaError_t e = ctx->d_sub_U.ensure((int64_t)n * 16);
        if (e == cudaSuccess) e = ctx->d_sub_vecs.ensure((int64_t)n * kmax);
        if (e == cudaSuccess) e = ctx->d_sub_t.ensure(kmax);
        if (e == cudaSuccess) e = ctx->d_sub_idx.ensure(n);
        if (e == cudaSuccess) e = ctx->d_sub_keep.ensure(n);
        if (e != cudaSuccess) return fail(ctx, VPCA_ERR_NOMEM, "subset buffers: %s", cudaGetErrorString(e));
    }
    CUDA_OK(ctx, ctx->d_sub_S.ensure((int64_t)m * m, with_slack((int64_t)m * m)));
    std::vector<uint8_t> keep01(n);
    for (int s = 0; s < n; ++s) keep01[s] = keep[s] != 0;
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e0, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_sub_idx.get(), idx.data(), (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_sub_keep.get(), keep01.data(), (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    ctx->c_h2d += (int64_t)n * 5;
    CUDA_OK(ctx, subset_gather(ctx->d_S, n, ctx->d_sub_idx.get(), m, ctx->d_sub_S.get(), ctx->stream));
    EigWork& w = ctx->sub_eig;
    CUDA_OK(ctx, center_gram(w, ctx->d_sub_S.get(), ctx->stream, false));
    {   // VPCA_EIG as for vpca_compute_pca
        const char* em = getenv("VPCA_EIG");
        w.mode = (em != nullptr && strcmp(em, "direct") == 0) ? 1 : (em != nullptr && strcmp(em, "lanczos") == 0) ? 2 : 0;
    }
    int64_t launches = 3;
    CUDA_OK(ctx, eig_topk(w, k, ctx->stream, &launches));
    CUDA_OK(ctx, subset_place(ctx->d_S, n, ctx->d_sub_idx.get(), m, w.d_evecs.get(), w.d_evals.get(), w.d_rowsum.get(), k, ctx->d_sub_U.get(),
                              ctx->d_sub_vecs.get(), ctx->d_sub_t.get(), ctx->stream));
    launches += m < n ? 3 : 1;
    ctx->c_launches += launches;
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e1, ctx->stream));
    ctx->st.eig_method = w.last_method;
    ctx->st.eig_iterations = w.last_iters;
    ctx->eig_timed = true;
    const size_t nb = (size_t)n * k * sizeof(double);
    CUDA_OK(ctx, cudaMemcpyAsync(vecs, ctx->d_sub_vecs.get(), nb, cudaMemcpyDeviceToHost, ctx->stream));
    if (evals) CUDA_OK(ctx, cudaMemcpyAsync(evals, w.d_evals.get(), k * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    int nz = 0;
    CUDA_OK(ctx, cudaMemcpyAsync(&nz, w.d_nz.get(), sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    if (non_zero_rows) *non_zero_rows = nz;
    ctx->c_d2h += (int64_t)nb + (evals ? k * 8 : 0) + 4;
    ctx->pca_k = k;
    ctx->d_U = ctx->d_sub_U.get();
    return VPCA_OK;
}

// Top-k of a Gram stored as row bands in `world` contexts (eig.cu, band_eig_topk): Lanczos driven from rank 0 with the
// mat-vec sharded over the bands.  Neither S nor the FP64 centred matrix is ever assembled, so neither the 65 535-sample
// limit of vpca_compute_pca nor its N x N workspace applies.  The direct reduction that backs the one-GPU Lanczos needs
// C, so there is no fallback here: every Lanczos failure is reported as VPCA_ERR_UNSUPPORTED.
int vpca_compute_pca_bands(vpca_ctx* const* ctxs, int32_t world, int32_t k, double* vecs, double* evals,
                           int32_t* non_zero_rows) {
    if (ctxs == nullptr || world < 1 || world > 16)
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_compute_pca_bands: world must be in [1, 16]");
    for (int r = 0; r < world; ++r)
        if (ctxs[r] == nullptr) return fail(ctxs[0], VPCA_ERR_BAD_ARG, "vpca_compute_pca_bands: ctxs[%d] is NULL", r);
    vpca_ctx* c0 = ctxs[0];
    const int n = c0->n;
    const int kmax = std::max(c0->num_pc, 16);
    if (vecs == nullptr || k < 1 || k > n || k > kmax)
        return fail(c0, VPCA_ERR_BAD_ARG, "vpca_compute_pca_bands: k=%d out of range [1, %d]", k, std::min(n, kmax));
    // n, band_row0 and band_rows are fixed at vpca_create: the bands can be checked before any lock is taken
    int next = 0;
    for (int r = 0; r < world; ++r) {
        const vpca_ctx* c = ctxs[r];
        if (c->n != n) return fail(c0, VPCA_ERR_BAD_ARG, "ctxs[%d] has %d samples, ctxs[0] %d", r, c->n, n);
        for (int q = 0; q < r; ++q)
            if (ctxs[q] == c) return fail(c0, VPCA_ERR_BAD_ARG, "ctxs[%d] and ctxs[%d] are the same context", q, r);
        if (c->band_row0 != next)
            return fail(c0, VPCA_ERR_BAD_ARG, "the bands must cover [0, %d) in rank order: ctxs[%d] stores rows [%d, %d), "
                        "expected a band starting at row %d", n, r, c->band_row0, c->band_row0 + c->band_rows, next);
        next = c->band_row0 + c->band_rows;
    }
    if (next != n) return fail(c0, VPCA_ERR_BAD_ARG, "the bands end at row %d, not at %d", next, n);
    std::vector<std::unique_lock<std::mutex>> locks;   // rank order
    locks.reserve(world);
    for (int r = 0; r < world; ++r) locks.emplace_back(ctxs[r]->mu);
    for (int r = 0; r < world; ++r) ctxs[r]->pca_k = ctxs[r]->grm_k = 0;   // a failed solve leaves no U behind, never a stale one
    BandPart* parts[16];
    for (int r = 0; r < world; ++r) {
        vpca_ctx* c = ctxs[r];
        if (!c->finalized) return fail(c0, VPCA_ERR_STATE, "ctxs[%d]: call vpca_finalize_gram first", r);
        for (auto& L : c->lanes)
            if (L.busy) return fail(c0, VPCA_ERR_STATE, "ctxs[%d]: an accumulate call is in flight", r);
        BandPart& p = c->band_part;
        p.device = c->cfg.device;
        p.stream = c->stream;
        p.d_S = c->d_S;
        p.n = n;
        p.row0 = c->band_row0;
        p.rows = c->band_rows;
        parts[r] = &p;
    }
    CUDA_OK(c0, cudaSetDevice(c0->cfg.device));
    CUDA_OK(c0, cudaEventRecord(c0->ev_e0, c0->stream));
    int64_t launches = 0;
    int outcome = 0;
    const cudaError_t e = band_eig_topk(c0->band_eig, parts, world, kmax, k, &launches, &outcome);
    cudaSetDevice(c0->cfg.device);
    c0->c_launches += launches;
    if (e != cudaSuccess)
        return fail(c0, e == cudaErrorMemoryAllocation ? VPCA_ERR_NOMEM : VPCA_ERR_CUDA, "band eigensolver: %s",
                    cudaGetErrorString(e));
    CUDA_OK(c0, cudaEventRecord(c0->ev_e1, c0->stream));
    c0->st.eig_method = 4;
    c0->st.eig_iterations = c0->band_eig.last_iters;
    c0->eig_timed = true;
    if (outcome != 0) {
        CUDA_OK(c0, cudaStreamSynchronize(c0->stream));
        const char* why = outcome == 2 ? "Lanczos broke down (a zero Gram, or a Krylov space exhausted before convergence)"
                        : outcome == 3 ? "the deflated verification run found an eigenvalue above the computed ones (a "
                                         "multiple top eigenvalue)"
                                       : "Lanczos did not converge within the step budget (kLzMaxIter, VPCA_EIG_MAXIT)";
        return fail(c0, VPCA_ERR_UNSUPPORTED, "vpca_compute_pca_bands after %d steps: %s; the bands have no direct-solver "
                    "fallback", c0->band_eig.last_iters, why);
    }
    const size_t nb = (size_t)n * k * sizeof(double);
    CUDA_OK(c0, cudaMemcpyAsync(vecs, c0->band_eig.d_evecs.get(), nb, cudaMemcpyDeviceToHost, c0->stream));
    if (evals) CUDA_OK(c0, cudaMemcpyAsync(evals, c0->band_eig.d_evals.get(), k * sizeof(double), cudaMemcpyDeviceToHost, c0->stream));
    int nz = 0;
    CUDA_OK(c0, cudaMemcpyAsync(&nz, c0->band_eig.d_nz.get(), sizeof(int), cudaMemcpyDeviceToHost, c0->stream));
    // U for the loadings on every rank: rank 0 reads its solver's vectors, every other rank gets a copy of the first
    // min(k, 16) columns on its own device, in stream order after the solve (ev_e1), as v_j travels during it
    const int kc = std::min(k, 16);
    for (int r = 1; r < world; ++r) {
        vpca_ctx* c = ctxs[r];
        CUDA_OK(c0, cudaSetDevice(c->cfg.device));
        if (const cudaError_t ae = c->d_band_U.ensure((int64_t)n * 16); ae != cudaSuccess)
            return fail(c0, VPCA_ERR_NOMEM, "ctxs[%d]: U for the loadings: %s", r, cudaGetErrorString(ae));
        CUDA_OK(c0, cudaStreamWaitEvent(c->stream, c0->ev_e1, 0));
        CUDA_OK(c0, cudaMemcpyPeerAsync(c->d_band_U.get(), c->cfg.device, c0->band_eig.d_evecs.get(), c0->cfg.device,
                                        (size_t)n * kc * sizeof(double), c->stream));
    }
    for (int r = 1; r < world; ++r) {   // the source is rank 0's solver state, which the next solve overwrites
        CUDA_OK(c0, cudaSetDevice(ctxs[r]->cfg.device));
        CUDA_OK(c0, cudaStreamSynchronize(ctxs[r]->stream));
    }
    CUDA_OK(c0, cudaSetDevice(c0->cfg.device));
    CUDA_OK(c0, cudaStreamSynchronize(c0->stream));
    if (non_zero_rows) *non_zero_rows = nz;
    c0->c_d2h += (int64_t)nb + (evals ? k * 8 : 0) + 4;
    for (int r = 0; r < world; ++r) {
        ctxs[r]->pca_k = k;
        ctxs[r]->d_U = r == 0 ? c0->band_eig.d_evecs.get() : ctxs[r]->d_band_U.get();
    }
    return VPCA_OK;
}

// ---- variant loadings and projection (project.cu) --------------------------------------------------------------
// Driver-side calls, one at a time per context and never concurrent with accumulation, so the chunk buffers below are
// the context's own; host-input calls run on a staging lane (encode as for the Gram), panel calls on the ctx stream.
static constexpr int kProjLd = 16;   // row pitch (doubles) of the projection accumulator

// On success *U is the U the loadings read (valid until the next solve, reset or Gram change of this context), and *keep
// the keep bytes of the subset solve that made it (nullptr after any other solve).
static int loadings_check(vpca_ctx* ctx, int32_t k, const double** U, const uint8_t** keep) {   // caller holds ctx->mu
    if (ctx->band_rows != ctx->n && ctx->pca_k == 0)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "loadings on a context that stores a row band need the eigenvectors of a "
                    "successful vpca_compute_pca_bands that named it, since its last reset / finalize_gram");
    if (k < 1 || k > 16) return fail(ctx, VPCA_ERR_BAD_ARG, "loadings: k=%d out of range [1, 16]", k);
    if (ctx->pca_k == 0)
        return fail(ctx, VPCA_ERR_STATE, "loadings need a vpca_compute_pca or vpca_compute_pca_bands since the last reset / "
                    "set_gram / load_partial_gram / finalize_gram");
    if (k > ctx->pca_k) return fail(ctx, VPCA_ERR_BAD_ARG, "loadings of %d components, the last solve computed %d", k, ctx->pca_k);
    *U = ctx->d_U;
    *keep = ctx->d_U == ctx->d_sub_U.get() ? ctx->d_sub_keep.get() : nullptr;
    return VPCA_OK;
}

static int project_check(vpca_ctx* ctx) {   // caller holds ctx->mu
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_UNSUPPORTED, "projection needs a context that stores the whole Gram");
    if (ctx->proj_k == 0) return fail(ctx, VPCA_ERR_STATE, "call vpca_project_begin first");
    return VPCA_OK;
}

// The projection of one encoded chunk [v, v + nvc) on lane L: the chunk's slice of w / mean goes to the device on the
// lane's stream (the single buffer is reused in stream order), then the projection kernels add into the accumulator.
static int project_chunk(vpca_ctx* ctx, vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc, const double* w, const double* mean) {
    const int k = ctx->proj_k;
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_lp_w.get(), w + v * k, (size_t)nvc * k * sizeof(double), cudaMemcpyHostToDevice, L.stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_lp_mean.get(), mean + v, (size_t)nvc * sizeof(double), cudaMemcpyHostToDevice, L.stream));
    ctx->c_h2d += nvc * (k + 1) * (int64_t)sizeof(double);
    CUDA_OK(ctx, project_launch(L.d_x[b].get(), ctx->elem_bits, ctx->n, nvc, ctx->panel, ctx->d_lp_w.get(), ctx->d_lp_mean.get(), k,
                                ctx->d_proj_part.get(), ctx->d_proj_acc.get(), kProjLd, L.stream));
    ctx->c_launches += 2;
    return VPCA_OK;
}

static int loadings_chunk(vpca_ctx* ctx, vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc, const double* U,
                          const uint8_t* keep, int k, double* out_w, int32_t* out_count) {
    CUDA_OK(ctx, loadings_launch(L.d_x[b].get(), ctx->elem_bits, ctx->n, nvc, ctx->panel, U, k, ctx->d_lp_w.get(),
                                 ctx->d_lp_count.get(), keep, L.stream));
    CUDA_OK(ctx, cudaMemcpyAsync(out_w + v * k, ctx->d_lp_w.get(), (size_t)nvc * k * sizeof(double), cudaMemcpyDeviceToHost, L.stream));
    CUDA_OK(ctx, cudaMemcpyAsync(out_count + v, ctx->d_lp_count.get(), (size_t)nvc * sizeof(int32_t), cudaMemcpyDeviceToHost, L.stream));
    ctx->c_launches += 1;
    ctx->c_d2h += nvc * (k * (int64_t)sizeof(double) + 4);
    return VPCA_OK;
}

// chunk buffers for host-input loadings (project == false) or projection; after LaneGuard (it fixes chunk_variants)
static int lp_buffers(vpca_ctx* ctx, int k, bool project) {
    const int64_t cv = ctx->chunk_variants;
    CUDA_OK(ctx, ctx->d_lp_w.ensure(cv * k, with_slack(cv * k)));
    if (project) {
        const int64_t part = project_scratch_doubles(ctx->n, cv, ctx->panel, k);
        CUDA_OK(ctx, ctx->d_lp_mean.ensure(cv, with_slack(cv)));
        CUDA_OK(ctx, ctx->d_proj_part.ensure(part, with_slack(part)));
    } else {
        CUDA_OK(ctx, ctx->d_lp_count.ensure(cv, with_slack(cv)));
    }
    return VPCA_OK;
}

int vpca_loadings_calls(vpca_ctx* ctx, int32_t k, const int64_t* offsets, const int32_t* sample_idx, int64_t nv,
                        double* out_w, int32_t* out_count) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (offsets == nullptr || nv < 0 || (nv > 0 && (out_w == nullptr || out_count == nullptr)) ||
        (nv > 0 && sample_idx == nullptr && offsets[nv] > offsets[0]))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_loadings_calls: bad argument");
    const double* U = nullptr;
    const uint8_t* keep = nullptr;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        int rc = loadings_check(ctx, k, &U, &keep);
        if (rc != VPCA_OK) return rc;
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    int rc = lp_buffers(ctx, k, false);
    if (rc != VPCA_OK) return rc;
    auto consume = [&](vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc) {
        return loadings_chunk(ctx, L, b, v, nvc, U, keep, k, out_w, out_count);
    };
    return process_calls(ctx, *lg.lane, offsets, sample_idx, 4, nv, consume, false);
}

int vpca_loadings_bed(vpca_ctx* ctx, int32_t k, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                      double* out_w, int32_t* out_count) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (counted_allele != 1 && counted_allele != 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_loadings_bed: counted_allele must be 1 (A1) or 2 (A2)");
    if (int rc = rows_args(ctx, "vpca_loadings_bed", rows, nv, stride_bytes, (ctx->n + 3) / 4,
                           out_w != nullptr && out_count != nullptr))
        return rc;
    const double* U = nullptr;
    const uint8_t* keep = nullptr;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        int rc = loadings_check(ctx, k, &U, &keep);
        if (rc != VPCA_OK) return rc;
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    int rc = lp_buffers(ctx, k, false);
    if (rc != VPCA_OK) return rc;
    auto consume = [&](vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc) {
        return loadings_chunk(ctx, L, b, v, nvc, U, keep, k, out_w, out_count);
    };
    return process_packed(ctx, *lg.lane, rows, nv, stride_bytes, counted_allele, consume);
}

int vpca_loadings_panels(vpca_ctx* ctx, int32_t k, const void* d_x, int64_t nv, int64_t panel_variants, double* d_w,
                         int32_t* d_count) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    const double* U = nullptr;
    const uint8_t* keep = nullptr;
    int rc = loadings_check(ctx, k, &U, &keep);
    if (rc != VPCA_OK) return rc;
    if (d_x == nullptr || nv < 0 || panel_variants < 128 || (panel_variants % 128) != 0 || (nv > 0 && (d_w == nullptr || d_count == nullptr)))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_loadings_panels: panel_variants must be a positive multiple of 128");
    if ((reinterpret_cast<uintptr_t>(d_x) & 31) != 0) return fail(ctx, VPCA_ERR_BAD_ARG, "panels must be 32-byte aligned");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, loadings_launch(d_x, ctx->elem_bits, ctx->n, nv, panel_variants, U, k, d_w, d_count, keep, ctx->stream));
    ctx->c_launches += nv > 0 ? 1 : 0;
    return VPCA_OK;
}

int vpca_project_begin(vpca_ctx* ctx, int32_t k) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_UNSUPPORTED, "projection needs a context that stores the whole Gram");
    if (k < 1 || k > 16) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_project_begin: k=%d out of range [1, 16]", k);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, ctx->d_proj_acc.ensure((int64_t)ctx->n * kProjLd));
    CUDA_OK(ctx, cudaMemsetAsync(ctx->d_proj_acc.get(), 0, (size_t)ctx->n * kProjLd * sizeof(double), ctx->stream));
    ctx->proj_k = k;
    return VPCA_OK;
}

int vpca_project_calls(vpca_ctx* ctx, const int64_t* offsets, const int32_t* sample_idx, int64_t nv, const double* w,
                       const double* mean) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        int rc = project_check(ctx);
        if (rc != VPCA_OK) return rc;
    }
    if (offsets == nullptr || nv < 0 || (nv > 0 && (w == nullptr || mean == nullptr)) ||
        (nv > 0 && sample_idx == nullptr && offsets[nv] > offsets[0]))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_project_calls: bad argument");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    int rc = lp_buffers(ctx, ctx->proj_k, true);
    if (rc != VPCA_OK) return rc;
    auto consume = [&](vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc) { return project_chunk(ctx, L, b, v, nvc, w, mean); };
    return process_calls(ctx, *lg.lane, offsets, sample_idx, 4, nv, consume, false);
}

int vpca_project_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                     const double* w, const double* mean) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        int rc = project_check(ctx);
        if (rc != VPCA_OK) return rc;
    }
    if (counted_allele != 1 && counted_allele != 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_project_bed: counted_allele must be 1 (A1) or 2 (A2)");
    if (int rc = rows_args(ctx, "vpca_project_bed", rows, nv, stride_bytes, (ctx->n + 3) / 4, w != nullptr && mean != nullptr))
        return rc;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    int rc = lp_buffers(ctx, ctx->proj_k, true);
    if (rc != VPCA_OK) return rc;
    auto consume = [&](vpca_ctx::Lane& L, int b, int64_t v, int64_t nvc) { return project_chunk(ctx, L, b, v, nvc, w, mean); };
    return process_packed(ctx, *lg.lane, rows, nv, stride_bytes, counted_allele, consume);
}

int vpca_project_panels(vpca_ctx* ctx, const void* d_x, int64_t nv, int64_t panel_variants, const double* d_w,
                        const double* d_mean) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    int rc = project_check(ctx);
    if (rc != VPCA_OK) return rc;
    if (d_x == nullptr || nv < 0 || panel_variants < 128 || (panel_variants % 128) != 0 || (nv > 0 && (d_w == nullptr || d_mean == nullptr)))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_project_panels: panel_variants must be a positive multiple of 128");
    if ((reinterpret_cast<uintptr_t>(d_x) & 31) != 0) return fail(ctx, VPCA_ERR_BAD_ARG, "panels must be 32-byte aligned");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int64_t need = project_scratch_doubles(ctx->n, nv, panel_variants, ctx->proj_k);
    if (need > ctx->d_proj_part.capacity()) {
        // the scratch may still be read by an earlier launch on this stream
        CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
        CUDA_OK(ctx, ctx->d_proj_part.ensure(need, with_slack(need)));
    }
    CUDA_OK(ctx, project_launch(d_x, ctx->elem_bits, ctx->n, nv, panel_variants, d_w, d_mean, ctx->proj_k, ctx->d_proj_part.get(),
                                ctx->d_proj_acc.get(), kProjLd, ctx->stream));
    ctx->c_launches += 2;
    return VPCA_OK;
}

int vpca_project_get(vpca_ctx* ctx, const double* evals, double* out) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    int rc = project_check(ctx);
    if (rc != VPCA_OK) return rc;
    if (evals == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_project_get: NULL argument");
    const int k = ctx->proj_k, n = ctx->n;
    std::vector<double> acc((size_t)n * kProjLd);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaMemcpyAsync(acc.data(), ctx->d_proj_acc.get(), acc.size() * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)(acc.size() * sizeof(double));
    for (int c = 0; c < k; ++c)
        for (int s = 0; s < n; ++s) out[s + (size_t)c * n] = acc[(size_t)s * kProjLd + c] / evals[c];
    return VPCA_OK;
}

// ---- KING-robust kinship (kinship.cu, DESIGN.md 7) --------------------------------------------------------------
// Driver-side calls like the loadings: one at a time per context, never concurrent with accumulation.  Rows are staged on
// a lane (their H2D copy overlaps the encode and Gram of the previous chunk); the planes and the Gram are the kinship's own.
static int kinship_check(vpca_ctx* ctx) {
    if (ctx->n > kKinMaxN)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "kinship is limited to %d samples (the 3N x 3N plane Gram must stay below 2^32 "
                    "cells); this context has %d", kKinMaxN, ctx->n);
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_UNSUPPORTED, "kinship needs a context that stores the whole Gram");
    return VPCA_OK;
}

// Plane staging geometry and buffers, and the kinship Gram (zeroed on the lane's stream), on the first call.
static int kinship_buffers(vpca_ctx* ctx, vpca_ctx::Lane& L) {
    const int64_t R = 3 * (int64_t)ctx->n, budget = 256ll << 20;   // bytes per plane staging buffer
    if (ctx->kin_panel == 0) {
        const int64_t p = std::max<int64_t>(128, (budget / R / 128) * 128);
        ctx->kin_panel = std::min<int64_t>(ctx->panel, p);
        ctx->kin_chunk = std::max<int64_t>(ctx->kin_panel, (budget / R / ctx->kin_panel) * ctx->kin_panel);
        for (int b = 0; b < 2; ++b) {
            cudaError_t e = ctx->d_kin_x[b].ensure(R * ctx->kin_chunk);
            if (e != cudaSuccess) {
                ctx->kin_panel = ctx->kin_chunk = 0;
                return fail(ctx, VPCA_ERR_NOMEM, "kinship plane staging: %s", cudaGetErrorString(e));
            }
        }
    }
    if (ctx->d_kin.get() == nullptr) {
        cudaError_t e = ctx->d_kin.ensure(R * R);
        if (e != cudaSuccess)
            return fail(ctx, VPCA_ERR_NOMEM, "kinship Gram of %lld x %lld int32: %s", (long long)R, (long long)R,
                        cudaGetErrorString(e));
        CUDA_OK(ctx, cudaMemsetAsync(ctx->d_kin.get(), 0, (size_t)R * R * sizeof(int32_t), L.stream));
    }
    return VPCA_OK;
}

int vpca_kinship_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    int rc = kinship_check(ctx);
    if (rc != VPCA_OK) return rc;
    rc = rows_args(ctx, "vpca_kinship_bed", rows, nv, stride_bytes, (ctx->n + 3) / 4);
    if (rc != VPCA_OK) return rc;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->kin_variants + nv > 2147483647ll)
            return fail(ctx, VPCA_ERR_OVERFLOW, "%lld kinship variants could overflow an int32 count",
                        (long long)(ctx->kin_variants + nv));
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    rc = kinship_buffers(ctx, L);
    if (rc != VPCA_OK) return rc;
    const int n = ctx->n;
    const int64_t R = 3 * (int64_t)n, P = ctx->kin_panel;
    const int64_t cap_rows = (ctx->chunk_nnz * (int64_t)sizeof(int32_t)) / stride_bytes;   // raw rows in L.d_idx[b]
    if (cap_rows < 32) return fail(ctx, VPCA_ERR_BAD_ARG, "stride_bytes too large for the staging buffer");
    const int64_t step = std::min(ctx->kin_chunk, (cap_rows / 32) * 32);
    rc = stage_rows(ctx, L, rows, nv, stride_bytes, step, lane_rows(L), [&](int b, const uint8_t* d_rows, int64_t, int64_t nvc) -> int {
        CUDA_OK(ctx, encode_bed_planes(d_rows, stride_bytes, nvc, n, ctx->d_kin_x[b].get(), P, L.stream));
        std::string msg;
        cudaError_t e = gram_accumulate(ctx->kin_plan, ctx->d_kin_x[b].get(), 8, (int)R, nvc, P, P, ctx->d_kin.get(), L.stream, &msg);
        if (e != cudaSuccess)
            return fail(ctx, VPCA_ERR_CUDA, "kinship Gram launch failed: %s %s [the kinship counts may hold a partial "
                        "batch, call vpca_reset]", cudaGetErrorString(e), msg.c_str());
        ctx->c_launches += 2;
        ctx->c_gram += 1;
        return VPCA_OK;
    });
    if (rc != VPCA_OK) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->kin_variants += nv;
    return VPCA_OK;
}

int vpca_kinship_pairs(vpca_ctx* ctx, double min_kinship, int64_t max_pairs, int32_t* out_ids, int32_t* out_counts,
                       double* out_kinship, int64_t* n_pairs) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    int rc = kinship_check(ctx);
    if (rc != VPCA_OK) return rc;
    if (n_pairs == nullptr || max_pairs < 0 ||
        (max_pairs > 0 && (out_ids == nullptr || out_counts == nullptr || out_kinship == nullptr)))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_kinship_pairs: bad argument");
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->kin_variants == 0)
            return fail(ctx, VPCA_ERR_STATE, "no kinship rows since the context was created or reset: call vpca_kinship_bed");
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const int n = ctx->n, tile_rows = (n + 31) / 32;
    const bool all = std::isinf(min_kinship) && min_kinship < 0;
    KinPairWork& w = ctx->kin_pairs;
    cudaError_t e = kin_pair_alloc(w, n);
    if (e != cudaSuccess) return fail(ctx, VPCA_ERR_NOMEM, "kinship pair scratch: %s", cudaGetErrorString(e));
    CUDA_OK(ctx, kin_count(w, ctx->d_kin.get(), n, min_kinship, all, ctx->stream));
    std::vector<int32_t> row_total(n);
    CUDA_OK(ctx, cudaMemcpyAsync(row_total.data(), w.d_row_total.get(), (size_t)n * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                 ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_launches += 2;
    std::vector<int64_t> start(n + 1, 0);   // output position of the first pair of row b (row-major lower triangle)
    for (int b = 0; b < n; ++b) start[b + 1] = start[b] + row_total[b];
    *n_pairs = start[n];
    const int64_t limit = std::min(start[n], max_pairs);
    if (limit == 0) return VPCA_OK;
    CUDA_OK(ctx, cudaMemcpyAsync(w.d_row_start.get(), start.data(), (size_t)n * sizeof(int64_t), cudaMemcpyHostToDevice, ctx->stream));
    ctx->c_h2d += (int64_t)n * 8;
    auto row_end = [&](int bt) { return start[std::min(n, 32 * bt)]; };   // position after tile rows [0, bt)
    for (int lo = 0; lo < tile_rows && row_end(lo) < limit;) {
        int hi = lo + 1;   // as many tile rows as the scratch holds (one always fits, kin_pair_alloc)
        while (hi < tile_rows && row_end(hi + 1) - row_end(lo) <= w.d_kin.capacity() && row_end(hi) < limit) ++hi;
        const int64_t base = row_end(lo), end = std::min(row_end(hi), limit), cnt = end - base;
        if (cnt > 0) {
            CUDA_OK(ctx, kin_emit(w, ctx->d_kin.get(), n, min_kinship, all, lo, hi, base, end, ctx->stream));
            CUDA_OK(ctx, cudaMemcpyAsync(out_ids + 2 * base, w.d_ids.get(), (size_t)cnt * 2 * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                         ctx->stream));
            CUDA_OK(ctx, cudaMemcpyAsync(out_counts + 5 * base, w.d_counts.get(), (size_t)cnt * 5 * sizeof(int32_t),
                                         cudaMemcpyDeviceToHost, ctx->stream));
            CUDA_OK(ctx, cudaMemcpyAsync(out_kinship + base, w.d_kin.get(), (size_t)cnt * sizeof(double), cudaMemcpyDeviceToHost,
                                         ctx->stream));
            ctx->c_launches += 1;
            ctx->c_d2h += cnt * 36;
        }
        lo = hi;
    }
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return VPCA_OK;
}

// ---- LD pruning (ld.cu, DESIGN.md 9) ----------------------------------------------------------------------------------
// Driver-side and synchronous.  The variants are walked in chunks of c rows that overlap by H = max_j (j - window_lo[j]);
// a chunk decides the rows it does not share with the previous one, whose windows then lie inside it.  The samples of a
// chunk are split into pieces of at most kLdMaxPiece, each staged on a lane (its H2D copy overlaps the previous piece's
// encode and Gram) and added into the same plane Gram, so staging is bounded whatever the cohort size.
namespace {
constexpr int64_t kLdMaxPiece = 32768;            // samples per staged piece
constexpr int64_t kLdPlaneBudget = 256ll << 20;   // bytes of the plane tile of one piece
constexpr int64_t kLdWindowBytes = 16ll << 20;    // bytes of one panel of the plane tile (the Gram kernel's L2 window)

// Grows every buffer of one call: the 3c x 3c Gram, the plane tile (x_bytes), two row buffers (row_bytes each), the window
// starts and the row arrays (c), the bit words (c T), a pair scratch that holds a whole row tile (32 rows of at most 32 T
// pairs) and the keep bytes (nv).
cudaError_t ld_buffers(vpca_ctx* ctx, int64_t c, int T, int64_t x_bytes, int64_t row_bytes, int64_t nv) {
    LdWork& w = ctx->ld;
    const int64_t pairs = std::max<int64_t>(int64_t(1) << 20, 1024 * (int64_t)T);
    cudaError_t e = ctx->d_ld_G.ensure(9 * c * c);
    if (e == cudaSuccess) e = ctx->d_ld_x.ensure(x_bytes);
    if (e == cudaSuccess) e = ctx->d_ld_rows[0].ensure(row_bytes);
    if (e == cudaSuccess) e = ctx->d_ld_rows[1].ensure(row_bytes);
    if (e == cudaSuccess) e = ctx->d_ld_wlo.ensure(c);
    if (e == cudaSuccess) e = ctx->d_ld_keep.ensure(nv);
    if (e == cudaSuccess) e = w.d_bits.ensure(c * T);
    if (e == cudaSuccess) e = w.d_seg.ensure(c * T);
    if (e == cudaSuccess) e = w.d_row_total.ensure(c);
    if (e == cudaSuccess) e = w.d_row_start.ensure(c);
    if (pairs > w.d_r2.capacity() || 2 * pairs > w.d_pairs.capacity()) {
        // the pair scratch holds d_r2.capacity() pairs in both buffers: they are reallocated together
        w.d_pairs.reset();
        w.d_r2.reset();
    }
    if (e == cudaSuccess) e = w.d_pairs.ensure(2 * pairs);
    if (e == cudaSuccess) e = w.d_r2.ensure(pairs);
    if (e == cudaSuccess) e = w.d_total.ensure(1);
    return e;
}
}   // namespace

int vpca_ld_prune_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, const int64_t* window_lo,
                      double r2_max, uint8_t* keep, int64_t max_pairs, int64_t* out_pairs, double* out_r2,
                      int64_t* n_pairs) {
    return vpca_ld_prune_bed_masked(ctx, rows, nv, stride_bytes, window_lo, nullptr, r2_max, keep, max_pairs, out_pairs,
                                    out_r2, n_pairs);
}

int vpca_ld_prune_bed_masked(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                             const int64_t* window_lo, const uint8_t* eligible, double r2_max, uint8_t* keep,
                             int64_t max_pairs, int64_t* out_pairs, double* out_r2, int64_t* n_pairs) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    const int n = ctx->n;
    if (rows == nullptr || window_lo == nullptr || keep == nullptr || n_pairs == nullptr || nv < 0 ||
        stride_bytes < (n + 3) / 4 || max_pairs < 0 || (max_pairs > 0 && (out_pairs == nullptr || out_r2 == nullptr)))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_ld_prune_bed: bad argument (rows, window_lo, keep and n_pairs must be set, "
                    "stride_bytes >= ceil(n_samples / 4))");
    if (!std::isfinite(r2_max) || r2_max < 0.0 || r2_max >= 1.0)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_ld_prune_bed: r2_max must be in [0, 1), not %g", r2_max);
    int64_t H = 0;
    for (int64_t j = 0; j < nv; ++j) {
        const int64_t lo = window_lo[j];
        if (lo < 0 || lo > j || (j > 0 && lo < window_lo[j - 1]))
            return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_ld_prune_bed: window_lo[%lld] = %lld must lie in [window_lo[j - 1], j]",
                        (long long)j, (long long)lo);
        H = std::max(H, j - lo);
    }
    if (H > kLdMaxWindow) {
        int64_t j = 0;
        while (j - window_lo[j] <= kLdMaxWindow) ++j;
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "vpca_ld_prune_bed: the window of variant %lld reaches back %lld variants; "
                    "the limit is %d", (long long)j, (long long)(j - window_lo[j]), kLdMaxWindow);
    }
    if (eligible != nullptr)
        for (int64_t j = 0; j < nv; ++j)
            if (eligible[j] > 1)
                return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_ld_prune_bed_masked: eligible[%lld] = %d must be 0 or 1",
                            (long long)j, (int)eligible[j]);
    *n_pairs = 0;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;

    // geometry: c = 2H minimises the Gram per decided variant, 4.5 c^2 / (c - H) products per sample (DESIGN.md 9)
    int64_t c = ((std::max<int64_t>(2 * H, 1024) + 31) / 32) * 32;
    if (nv <= c) c = ((nv + 31) / 32) * 32;
    const int T = (int)((H + 31) / 32) + 1;
    const int64_t R = 3 * c;
    const int64_t n128 = ((int64_t)n + 127) / 128 * 128;
    const int64_t P = std::min(n128, std::max<int64_t>(128, std::min<int64_t>(8192, kLdWindowBytes / R / 128 * 128)));
    int64_t piece = std::max(P, std::min(kLdMaxPiece, kLdPlaneBudget / R) / P * P);
    piece = std::min(piece, ((int64_t)n + P - 1) / P * P);
    const int64_t rp = piece / 4;                       // staged bytes per row and piece
    const int64_t row_bytes = ((int64_t)n + 3) / 4;     // meaningful bytes of a .bed row

    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    LdWork& w = ctx->ld;
    {
        cudaError_t e = ld_buffers(ctx, c, T, R * piece, c * rp, nv);
        if (e == cudaSuccess && eligible != nullptr) e = ctx->d_ld_elig.ensure(nv);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "LD pruning buffers for chunks of %lld variants: %s", (long long)c,
                        cudaGetErrorString(e));
        }
    }
    CUDA_OK(ctx, cudaMemsetAsync(w.d_total.get(), 0, sizeof(int64_t), L.stream));
    if (eligible != nullptr) {
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_ld_elig.get(), eligible, (size_t)nv, cudaMemcpyHostToDevice, L.stream));
        ctx->c_h2d += nv;
    }
    int64_t listed = 0;                   // pairs counted (and listed) before the current chunk while listing
    bool listing = max_pairs > 0;
    std::vector<int32_t> row_total((size_t)c);
    std::vector<int64_t> start((size_t)c + 1);
    int unit = 0;                         // staged pieces so far: selects the row buffer
    for (int64_t s = 0;;) {
        const int64_t e_end = std::min(s + c, nv);
        LdChunk ch{ctx->d_ld_G.get(), ctx->d_ld_wlo.get(), s, (int)c, (int)(e_end - s), s == 0 ? 0 : (int)H, T, r2_max,
                   eligible != nullptr ? ctx->d_ld_elig.get() : nullptr};
        CUDA_OK(ctx, cudaMemsetAsync(ctx->d_ld_G.get(), 0, (size_t)(R * R) * sizeof(int32_t), L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_ld_wlo.get(), window_lo + s, (size_t)ch.nc * sizeof(int64_t), cudaMemcpyHostToDevice,
                                     L.stream));
        ctx->c_h2d += ch.nc * 8;
        for (int64_t s0 = 0; s0 < n; s0 += piece, ++unit) {
            const int64_t len = std::min<int64_t>(piece, n - s0);
            const int64_t width = std::min(rp, row_bytes - s0 / 4);
            const int b = unit & 1;
            CUDA_OK(ctx, cudaStreamWaitEvent(L.copy_stream, L.ev_done[b], 0));
            CUDA_OK(ctx, cudaMemcpy2DAsync(ctx->d_ld_rows[b].get(), (size_t)rp, rows + (size_t)s * stride_bytes + s0 / 4,
                                           (size_t)stride_bytes, (size_t)width, (size_t)ch.nc, cudaMemcpyHostToDevice,
                                           L.copy_stream));
            CUDA_OK(ctx, cudaEventRecord(L.ev_copy[b], L.copy_stream));
            ctx->c_h2d += width * ch.nc;
            CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, L.ev_copy[b], 0));
            CUDA_OK(ctx, encode_ld_planes(ctx->d_ld_rows[b].get(), rp, width, ch.nc, (int)c, s0, len, n, ctx->d_ld_x.get(), P, L.stream));
            CUDA_OK(ctx, cudaEventRecord(L.ev_done[b], L.stream));   // the row buffer is free again
            std::string msg;
            cudaError_t e = gram_accumulate(ctx->ld_plan, ctx->d_ld_x.get(), 8, (int)R, len, P, P, ctx->d_ld_G.get(), L.stream, &msg);
            if (e != cudaSuccess)
                return fail(ctx, VPCA_ERR_CUDA, "LD plane Gram launch failed: %s %s", cudaGetErrorString(e), msg.c_str());
            ctx->c_launches += 2;
            ctx->c_gram += 1;
        }
        CUDA_OK(ctx, ld_count(w, ch, L.stream));
        CUDA_OK(ctx, ld_sweep(w, ch, ctx->d_ld_keep.get(), L.stream));
        ctx->c_launches += 3;
        if (listing) {
            const int lo = ch.own_lo, nc = ch.nc;
            CUDA_OK(ctx, cudaMemcpyAsync(row_total.data(), w.d_row_total.get() + lo, (size_t)(nc - lo) * sizeof(int32_t),
                                         cudaMemcpyDeviceToHost, L.stream));
            CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
            start[lo] = listed;
            for (int b = lo; b < nc; ++b) start[b + 1] = start[b] + row_total[b - lo];
            CUDA_OK(ctx, cudaMemcpyAsync(w.d_row_start.get() + lo, start.data() + lo, (size_t)(nc - lo) * sizeof(int64_t),
                                         cudaMemcpyHostToDevice, L.stream));
            const int64_t limit = std::min(start[nc], max_pairs);
            auto row_end = [&](int bt) { return start[std::min(nc, std::max(lo, 32 * bt))]; };   // position after tile rows < bt
            const int tiles_hi = (nc + 31) / 32;
            for (int tlo = lo / 32; tlo < tiles_hi && row_end(tlo) < limit;) {
                int thi = tlo + 1;   // as many row tiles as the scratch holds (one always fits, ld_buffers)
                while (thi < tiles_hi && row_end(thi + 1) - row_end(tlo) <= w.d_r2.capacity() && row_end(thi) < limit) ++thi;
                const int64_t base = row_end(tlo), end = std::min(row_end(thi), limit), cnt = end - base;
                if (cnt > 0) {
                    CUDA_OK(ctx, ld_emit(w, ch, tlo, thi, base, end, L.stream));
                    CUDA_OK(ctx, cudaMemcpyAsync(out_pairs + 2 * base, w.d_pairs.get(), (size_t)cnt * 2 * sizeof(int64_t),
                                                 cudaMemcpyDeviceToHost, L.stream));
                    CUDA_OK(ctx, cudaMemcpyAsync(out_r2 + base, w.d_r2.get(), (size_t)cnt * sizeof(double), cudaMemcpyDeviceToHost,
                                                 L.stream));
                    ctx->c_launches += 1;
                    ctx->c_d2h += cnt * 24;
                }
                tlo = thi;
            }
            listed = start[nc];
            listing = listed < max_pairs;
        }
        if (e_end == nv) break;
        s = e_end - H;
    }
    CUDA_OK(ctx, cudaMemcpyAsync(keep, ctx->d_ld_keep.get(), (size_t)nv, cudaMemcpyDeviceToHost, L.stream));
    CUDA_OK(ctx, cudaMemcpyAsync(n_pairs, w.d_total.get(), sizeof(int64_t), cudaMemcpyDeviceToHost, L.stream));
    ctx->c_d2h += nv + 8;
    CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
    return VPCA_OK;
}

// ---- variant QC (qc.cu, DESIGN.md 10) -----------------------------------------------------------------------------------
// Driver-side and synchronous.  Rows are staged in chunks of at most kQcStageBytes through stage_rows and counted; the
// counts of whole chunks gather into batches of about kQcHweChunk rows, each tested with one HWE launch and copied back,
// so that the HWE kernel fills the GPU even when a chunk holds a few thousand wide rows, and device memory stays bounded
// whatever the number of variants.
namespace {
constexpr int64_t kQcStageBytes = 64ll << 20;   // raw .bed bytes per staged chunk
constexpr int64_t kQcHweChunk = 1ll << 18;      // count rows per HWE launch (and per vpca_hwe_exact chunk)

// grows the QC buffers to `rows` count / p-value rows
cudaError_t qc_buffers(vpca_ctx* ctx, int64_t rows) {
    cudaError_t e = ctx->d_qc_counts.ensure(4 * rows);
    if (e == cudaSuccess) e = ctx->d_qc_p.ensure(rows);
    return e;
}
}   // namespace

int vpca_variant_qc_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t* out_counts,
                        double* out_hwe_p) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    const int n = ctx->n;
    if (int rc = rows_args(ctx, "vpca_variant_qc_bed", rows, nv, stride_bytes, (n + 3) / 4, out_counts != nullptr)) return rc;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int64_t step = std::max<int64_t>(1, std::min(nv, kQcStageBytes / stride_bytes));
    const int64_t batch = std::min(nv, step * std::max<int64_t>(1, kQcHweChunk / step));   // whole chunks
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = qc_buffers(ctx, batch);
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "variant QC buffers for %lld rows of %lld bytes: %s", (long long)step,
                        (long long)stride_bytes, cudaGetErrorString(e));
        }
    }
    // chunk boundaries fall on batch boundaries: the last chunk of a batch tests and copies back the whole batch
    return stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t v, int64_t nvc) -> int {
        const int64_t b0 = v / batch * batch, nb = std::min(batch, nv - b0);
        CUDA_OK(ctx, qc_count(d_rows, stride_bytes, (int)nvc, n, ctx->d_qc_counts.get() + 4 * (v - b0), L.stream));
        ctx->c_launches += 1;
        if (v + nvc < b0 + nb) return VPCA_OK;
        CUDA_OK(ctx, cudaMemcpyAsync(out_counts + 4 * b0, ctx->d_qc_counts.get(), (size_t)(4 * nb) * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, L.stream));
        ctx->c_d2h += 16 * nb;
        if (out_hwe_p != nullptr) {
            CUDA_OK(ctx, qc_hwe(ctx->d_qc_counts.get(), (int)nb, ctx->d_qc_p.get(), L.stream));
            CUDA_OK(ctx, cudaMemcpyAsync(out_hwe_p + b0, ctx->d_qc_p.get(), (size_t)nb * sizeof(double), cudaMemcpyDeviceToHost,
                                         L.stream));
            ctx->c_launches += 1;
            ctx->c_d2h += 8 * nb;
        }
        return VPCA_OK;
    });
}

int vpca_hwe_exact(vpca_ctx* ctx, const int32_t* counts, int64_t nv, double* out_p) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (nv < 0 || (nv > 0 && (counts == nullptr || out_p == nullptr)))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_hwe_exact: bad argument (counts and out_p must be set)");
    for (int64_t v = 0; v < nv; ++v) {
        const int64_t a = counts[4 * v], h = counts[4 * v + 1], b = counts[4 * v + 2];
        if (a < 0 || h < 0 || b < 0 || a + h + b > 2147483647ll)
            return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_hwe_exact: counts of row %lld (%lld, %lld, %lld) must be non-negative "
                        "with a sum below 2^31", (long long)v, (long long)a, (long long)h, (long long)b);
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int64_t step = std::min(nv, kQcHweChunk);
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = qc_buffers(ctx, step);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "HWE buffers for %lld rows: %s", (long long)step, cudaGetErrorString(e));
        }
    }
    for (int64_t v = 0; v < nv; v += step) {
        const int64_t nvc = std::min(step, nv - v);
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_qc_counts.get(), counts + 4 * v, (size_t)(4 * nvc) * sizeof(int32_t),
                                     cudaMemcpyHostToDevice, L.stream));
        ctx->c_h2d += 16 * nvc;
        CUDA_OK(ctx, qc_hwe(ctx->d_qc_counts.get(), (int)nvc, ctx->d_qc_p.get(), L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(out_p + v, ctx->d_qc_p.get(), (size_t)nvc * sizeof(double), cudaMemcpyDeviceToHost, L.stream));
        ctx->c_launches += 1;
        ctx->c_d2h += 8 * nvc;
    }
    CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
    return VPCA_OK;
}

// ---- variance-standardized relationship matrix (grm.cu, DESIGN.md 13) ---------------------------------------------------
// Driver-side and synchronous.  Rows are staged in chunks of at most kGrmStageBytes and kGrmMaxChunk rows through
// stage_rows, the upload of chunk i + 1 overlapping the work on chunk i.  Per chunk: counts, tables and the used list,
// then (after one small read-back of the used count) the used columns expanded into the panel, which is multiplied into
// eig.d_C whenever it is full.
namespace {
constexpr int64_t kGrmStageBytes = 64ll << 20;   // raw .bed bytes per staged chunk
constexpr int64_t kGrmMaxChunk = 1ll << 20;      // rows per staged chunk

int64_t grm_step(int64_t nv, int64_t stride) { return std::max<int64_t>(1, std::min({nv, kGrmStageBytes / stride, kGrmMaxChunk})); }

int grm_check(vpca_ctx* ctx) {
    if (ctx->n > 65535)
        return fail(ctx, VPCA_ERR_UNSUPPORTED, "the GRM is limited to 65535 samples, like vpca_compute_pca; this context has %d",
                    ctx->n);
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_UNSUPPORTED, "the GRM needs a context that stores the whole Gram");
    return VPCA_OK;
}

// The eigensolver workspace (whose d_C holds the sum) and the staging buffers; d_C and the panel zeroed on the first call.
int grm_buffers(vpca_ctx* ctx, vpca_ctx::Lane& L, int64_t step, int64_t stride) {
    if (!ctx->eig_ready) {
        cudaError_t e = eig_alloc(ctx->eig, ctx->n, std::max(ctx->num_pc, 16));
        if (e != cudaSuccess) return fail(ctx, VPCA_ERR_NOMEM, "eigensolver workspace: %s", cudaGetErrorString(e));
        ctx->eig_ready = true;
    }
    const int64_t zc = grm_panel_rows(ctx->n) * kGrmPanelK;
    cudaError_t e = cudaSuccess;
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride);
    if (e == cudaSuccess) e = ctx->d_grm_counts.ensure(4 * step);
    if (e == cudaSuccess) e = ctx->d_grm_tab.ensure(4 * step);
    if (e == cudaSuccess) e = ctx->d_grm_used.ensure(step);
    if (e == cudaSuccess) e = ctx->d_grm_inv.ensure(step);
    if (e == cudaSuccess) e = ctx->d_grm_total.ensure(1);
    if (e == cudaSuccess) e = ctx->d_grm_Z.ensure(zc);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(ctx, VPCA_ERR_NOMEM, "GRM buffers: %s", cudaGetErrorString(e));
    }
    if (ctx->grm_state == 0) {
        CUDA_OK(ctx, cudaMemsetAsync(ctx->eig.d_C.get(), 0, (size_t)ctx->n * ctx->n * sizeof(double), L.stream));
        CUDA_OK(ctx, cudaMemsetAsync(ctx->d_grm_Z.get(), 0, (size_t)zc * sizeof(double), L.stream));
        ctx->eig.c_valid = false;
        ctx->grm_used = 0;
        ctx->grm_fill = 0;
        ctx->grm_state = 1;
    }
    return VPCA_OK;
}
}   // namespace

int vpca_grm_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    const int n = ctx->n;
    int rc = rows_args(ctx, "vpca_grm_bed", rows, nv, stride_bytes, (n + 3) / 4);
    if (rc != VPCA_OK) return rc;
    rc = grm_check(ctx);
    if (rc != VPCA_OK) return rc;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->grm_state >= 2)
            return fail(ctx, VPCA_ERR_STATE, "the GRM was finalized (or its matrix overwritten) since the last vpca_reset");
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int64_t step = grm_step(nv, stride_bytes);
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    rc = grm_buffers(ctx, L, step, stride_bytes);
    if (rc != VPCA_OK) return rc;
    double* Z = ctx->d_grm_Z.get();
    double* C = ctx->eig.d_C.get();
    return stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t, int64_t nvc) -> int {
        CUDA_OK(ctx, qc_count(d_rows, stride_bytes, (int)nvc, n, ctx->d_grm_counts.get(), L.stream));
        CUDA_OK(ctx, grm_tables(ctx->d_grm_counts.get(), (int)nvc, ctx->d_grm_tab.get(), ctx->d_grm_used.get(),
                                ctx->d_grm_inv.get(), ctx->d_grm_total.get(), L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(L.h_flags, ctx->d_grm_total.get(), sizeof(int), cudaMemcpyDeviceToHost, L.stream));
        CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
        ctx->c_launches += 3;
        const int used = *L.h_flags;
        for (int j = 0; j < used;) {
            const int cnt = std::min(kGrmPanelK - ctx->grm_fill, used - j);
            CUDA_OK(ctx, grm_expand(d_rows, stride_bytes, ctx->d_grm_inv.get() + j, ctx->d_grm_tab.get(), cnt, n, Z,
                                    ctx->grm_fill, L.stream));
            ctx->c_launches += 1;
            ctx->grm_fill += cnt;
            j += cnt;
            if (ctx->grm_fill == kGrmPanelK) {
                CUDA_OK(ctx, grm_syrk(Z, n, C, L.stream));
                ctx->c_launches += 1;
                ctx->grm_fill = 0;
            }
        }
        ctx->grm_used += used;
        return VPCA_OK;
    });
}

int vpca_grm_finalize(vpca_ctx* ctx, int64_t* n_used) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    int rc = grm_check(ctx);
    if (rc != VPCA_OK) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->grm_state == 3)
        return fail(ctx, VPCA_ERR_STATE, "the GRM has no used variant or its matrix was overwritten: call vpca_reset");
    if (ctx->grm_state == 2) {
        if (n_used) *n_used = ctx->grm_used;
        return VPCA_OK;
    }
    if (ctx->grm_used == 0) {
        ctx->grm_state = 3;
        return fail(ctx, VPCA_ERR_STATE, "no variant of the GRM varies among its called samples (M = 0)");
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const int n = ctx->n;
    if (ctx->grm_fill > 0) {   // the partial panel, its unfilled columns zeroed
        double* Z = ctx->d_grm_Z.get();
        CUDA_OK(ctx, cudaMemset2DAsync(Z + ctx->grm_fill, kGrmPanelK * sizeof(double), 0,
                                       (size_t)(kGrmPanelK - ctx->grm_fill) * sizeof(double), (size_t)n, ctx->stream));
        CUDA_OK(ctx, grm_syrk(Z, n, ctx->eig.d_C.get(), ctx->stream));
        ctx->c_launches += 1;
        ctx->grm_fill = 0;
    }
    CUDA_OK(ctx, grm_finish(ctx->eig.d_C.get(), n, ctx->grm_used, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_launches += 1;
    ctx->grm_state = 2;
    if (n_used) *n_used = ctx->grm_used;
    return VPCA_OK;
}

int vpca_get_grm(vpca_ctx* ctx, double* out) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->grm_state != 2) return fail(ctx, VPCA_ERR_STATE, "no finalized GRM (call vpca_grm_finalize; a solve that "
                                         "overwrote it needs vpca_reset and the rows again)");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t bytes = (size_t)ctx->n * ctx->n * sizeof(double);
    CUDA_OK(ctx, cudaMemcpyAsync(out, ctx->eig.d_C.get(), bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)bytes;
    return VPCA_OK;
}

int vpca_compute_pca_grm(vpca_ctx* ctx, int32_t k, double* vecs, double* evals) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (vecs == nullptr || k < 1 || k > ctx->n || k > std::max(ctx->num_pc, 16))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_compute_pca_grm: k=%d out of range", k);
    if (ctx->grm_state != 2) return fail(ctx, VPCA_ERR_STATE, "no finalized GRM (call vpca_grm_finalize; a solve that "
                                         "overwrote it needs vpca_reset and the rows again)");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    ctx->pca_k = 0;   // a GRM solve leaves no U for the carrier loadings
    ctx->grm_k = 0;   // and a failed one none for the GRM loadings
    ctx->pca_done = false;
    {
        const char* em = getenv("VPCA_EIG");
        ctx->eig.mode = (em != nullptr && strcmp(em, "direct") == 0) ? 1 : (em != nullptr && strcmp(em, "lanczos") == 0) ? 2 : 0;
    }
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e0, ctx->stream));
    int64_t launches = 0;
    ctx->eig.grm = true;
    const cudaError_t e = eig_topk(ctx->eig, k, ctx->stream, &launches);
    ctx->eig.grm = false;
    if (e != cudaSuccess || ctx->eig.last_method != 2) ctx->grm_state = 3;   // the direct reduction consumed d_C
    CUDA_OK(ctx, e);
    ctx->c_launches += launches;
    CUDA_OK(ctx, cudaEventRecord(ctx->ev_e1, ctx->stream));
    ctx->st.eig_method = ctx->eig.last_method;
    ctx->st.eig_iterations = ctx->eig.last_iters;
    ctx->eig_timed = true;
    const size_t nb = (size_t)ctx->n * k * sizeof(double);
    CUDA_OK(ctx, cudaMemcpyAsync(vecs, ctx->eig.d_evecs.get(), nb, cudaMemcpyDeviceToHost, ctx->stream));
    if (evals) CUDA_OK(ctx, cudaMemcpyAsync(evals, ctx->eig.d_evals.get(), k * sizeof(double), cudaMemcpyDeviceToHost, ctx->stream));
    const int ku = std::min(k, 16);   // U for vpca_grm_loadings_bed
    CUDA_OK(ctx, ctx->d_grm_U.ensure((int64_t)ctx->n * 16));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_grm_U.get(), ctx->eig.d_evecs.get(), (size_t)ctx->n * ku * sizeof(double),
                                 cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_d2h += (int64_t)nb + (evals ? k * 8 : 0);
    ctx->grm_k = ku;
    return VPCA_OK;
}

// ---- GRM loadings and projection (grm_project.cu, DESIGN.md 14) ----------------------------------------------------------
// Driver-side and synchronous.  Rows are staged as in vpca_grm_bed: chunks of grm_step rows through stage_rows.
int vpca_grm_loadings_bed(vpca_ctx* ctx, int32_t k, const uint8_t* rows, int64_t nv, int64_t stride_bytes, double* out_w,
                          double* out_tab) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    int rc = rows_args(ctx, "vpca_grm_loadings_bed", rows, nv, stride_bytes, (ctx->n + 3) / 4,
                       out_w != nullptr && out_tab != nullptr);
    if (rc != VPCA_OK) return rc;
    rc = grm_check(ctx);
    if (rc != VPCA_OK) return rc;
    const double* U = nullptr;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->grm_k == 0)
            return fail(ctx, VPCA_ERR_STATE, "GRM loadings need a vpca_compute_pca_grm since the last reset / solve / Gram "
                        "change");
        if (k < 1 || k > ctx->grm_k)
            return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_grm_loadings_bed: k=%d out of range [1, %d]", k, ctx->grm_k);
        U = ctx->d_grm_U.get();
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int n = ctx->n;
    const int64_t step = grm_step(nv, stride_bytes);
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = cudaSuccess;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
        if (e == cudaSuccess) e = ctx->d_grm_counts.ensure(4 * step);
        if (e == cudaSuccess) e = ctx->d_grm_tab.ensure(4 * step);
        if (e == cudaSuccess) e = ctx->d_grm_used.ensure(step);
        if (e == cudaSuccess) e = ctx->d_grm_w.ensure(step * k);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "GRM loadings buffers: %s", cudaGetErrorString(e));
        }
    }
    return stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t v, int64_t nvc) -> int {
        CUDA_OK(ctx, qc_count(d_rows, stride_bytes, (int)nvc, n, ctx->d_grm_counts.get(), L.stream));
        CUDA_OK(ctx, grm_table(ctx->d_grm_counts.get(), (int)nvc, ctx->d_grm_tab.get(), ctx->d_grm_used.get(), L.stream));
        CUDA_OK(ctx, grm_loadings(d_rows, stride_bytes, (int)nvc, n, ctx->d_grm_tab.get(), U, k, ctx->d_grm_w.get(), L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(out_w + v * k, ctx->d_grm_w.get(), (size_t)nvc * k * sizeof(double),
                                     cudaMemcpyDeviceToHost, L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(out_tab + 4 * v, ctx->d_grm_tab.get(), (size_t)nvc * 4 * sizeof(double),
                                     cudaMemcpyDeviceToHost, L.stream));
        ctx->c_launches += 3;
        ctx->c_d2h += nvc * (k + 4) * (int64_t)sizeof(double);
        return VPCA_OK;
    });
}

int vpca_grm_project_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, const double* tab,
                         const double* w) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    int k = 0;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        int rc = project_check(ctx);
        if (rc != VPCA_OK) return rc;
        k = ctx->proj_k;
    }
    int rc = rows_args(ctx, "vpca_grm_project_bed", rows, nv, stride_bytes, (ctx->n + 3) / 4, tab != nullptr && w != nullptr);
    if (rc != VPCA_OK) return rc;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int n = ctx->n;
    const int64_t step = grm_step(nv, stride_bytes);
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        const int64_t part = grm_project_scratch_doubles(n, step, k);
        cudaError_t e = cudaSuccess;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
        if (e == cudaSuccess) e = ctx->d_grm_ptab.ensure(4 * step);
        if (e == cudaSuccess) e = ctx->d_grm_w.ensure(step * k);
        if (e == cudaSuccess) e = ctx->d_proj_part.ensure(part, with_slack(part));
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "GRM projection buffers: %s", cudaGetErrorString(e));
        }
    }
    return stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t v, int64_t nvc) -> int {
        // the single w / table buffers are reused in stream order: the previous chunk's kernels read them first
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_grm_w.get(), w + v * k, (size_t)nvc * k * sizeof(double),
                                     cudaMemcpyHostToDevice, L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_grm_ptab.get(), tab + 4 * v, (size_t)nvc * 4 * sizeof(double),
                                     cudaMemcpyHostToDevice, L.stream));
        ctx->c_h2d += nvc * (k + 4) * (int64_t)sizeof(double);
        CUDA_OK(ctx, grm_project(d_rows, stride_bytes, (int)nvc, n, ctx->d_grm_ptab.get(), ctx->d_grm_w.get(), k,
                                 ctx->d_proj_part.get(), ctx->d_proj_acc.get(), kProjLd, L.stream));
        ctx->c_launches += 2;
        return VPCA_OK;
    });
}

// ---- linear association tests (glm.cu, DESIGN.md 15) ---------------------------------------------------------------------
// vpca_glm_begin is host FP64 work and one upload; vpca_glm_linear_bed is driver-side and synchronous, its rows staged as
// vpca_grm_loadings_bed stages them.
namespace {
// The checks and the regression samples both begins share; VPCA_OK or the refusal (the message names fn).
int glm_samples(vpca_ctx* ctx, const char* fn, const double* pheno, const double* covar, int32_t n_covar,
                std::vector<int>& idx) {
    if (pheno == nullptr || n_covar < 0 || (n_covar > 0 && covar == nullptr))
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: bad argument (pheno must be set, n_covar >= 0, covar set when "
                    "n_covar > 0)", fn);
    const int q = n_covar + 1;
    if (q > VPCA_GLM_MAX_Q)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: %d covariates and the intercept exceed %d columns", fn, n_covar,
                    VPCA_GLM_MAX_Q);
    const int n = ctx->n;
    for (int s = 0; s < n; ++s) {
        bool ok = std::isfinite(pheno[s]);
        if (std::isinf(pheno[s])) return fail(ctx, VPCA_ERR_BAD_ARG, "%s: the phenotype of sample %d is infinite", fn, s);
        for (int j = 0; j < n_covar; ++j) {
            const double x = covar[(size_t)s * n_covar + j];
            if (std::isinf(x))
                return fail(ctx, VPCA_ERR_BAD_ARG, "%s: covariate %d of sample %d is infinite", fn, j + 1, s);
            ok = ok && std::isfinite(x);
        }
        if (ok) idx.push_back(s);
    }
    const int R = (int)idx.size();
    if (R < q + 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: %d regression samples; %d covariates and the intercept need at "
                    "least %d", fn, R, n_covar, q + 2);
    return VPCA_OK;
}

// Q (q x R, column-major by covariate): the columns of C over the regression samples orthonormalised in order, modified
// Gram-Schmidt applied twice; VPCA_OK or the refusal of a collinear covariate.
int glm_basis(vpca_ctx* ctx, const char* fn, const double* covar, int32_t n_covar, const std::vector<int>& idx,
              std::vector<double>& Q) {
    const int q = n_covar + 1, R = (int)idx.size();
    Q.assign((size_t)q * R, 0.0);
    for (int c = 0; c < q; ++c) {
        double* col = Q.data() + (size_t)c * R;
        for (int i = 0; i < R; ++i) col[i] = c == 0 ? 1.0 : covar[(size_t)idx[i] * n_covar + c - 1];
        double nrm0 = 0.0;
        for (int i = 0; i < R; ++i) nrm0 += col[i] * col[i];
        for (int pass = 0; pass < 2; ++pass)
            for (int k = 0; k < c; ++k) {
                const double* qk = Q.data() + (size_t)k * R;
                double r = 0.0;
                for (int i = 0; i < R; ++i) r += qk[i] * col[i];
                for (int i = 0; i < R; ++i) col[i] -= r * qk[i];
            }
        double nrm = 0.0;
        for (int i = 0; i < R; ++i) nrm += col[i] * col[i];
        if (!(nrm > 1e-18 * nrm0))
            return fail(ctx, VPCA_ERR_BAD_ARG, "%s: covariate %d is collinear with the intercept and the "
                        "covariates before it over the %d regression samples", fn, c, R);
        const double inv = 1.0 / std::sqrt(nrm);
        for (int i = 0; i < R; ++i) col[i] *= inv;
    }
    return VPCA_OK;
}

// Uploads Qx (n rows [q_0 .. q_{q-1}, y, 0 .., mask], y[i] the value of regression sample idx[i]), the regression mask,
// z0 (q doubles) and, when cases is set, the regression samples with y = 1 as bits.
int glm_upload(vpca_ctx* ctx, int q, const std::vector<int>& idx, const std::vector<double>& Q, const std::vector<double>& y,
               const std::vector<double>& z0, bool cases) {
    const int n = ctx->n, R = (int)idx.size();
    const int ld = glm_kmax(q) + 2;
    std::vector<double> Qx((size_t)n * ld, 0.0);
    std::vector<uint8_t> mask((n + 3) / 4, 0), cmask(cases ? (n + 3) / 4 : 0, 0);
    for (int i = 0; i < R; ++i) {
        double* xr = Qx.data() + (size_t)idx[i] * ld;
        for (int c = 0; c < q; ++c) xr[c] = Q[(size_t)c * R + i];
        xr[q] = y[i];
        xr[ld - 1] = 1.0;
        mask[idx[i] / 4] |= (uint8_t)(1u << (idx[i] % 4));
        if (cases && y[i] != 0.0) cmask[idx[i] / 4] |= (uint8_t)(1u << (idx[i] % 4));
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    {
        cudaError_t e = ctx->d_glm_Qx.ensure((int64_t)n * ld);
        if (e == cudaSuccess) e = ctx->d_glm_mask.ensure((n + 3) / 4);
        if (e == cudaSuccess && cases) e = ctx->d_glm_case.ensure((n + 3) / 4);
        if (e == cudaSuccess) e = ctx->d_glm_z0.ensure(VPCA_GLM_MAX_Q);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "GLM buffers: %s", cudaGetErrorString(e));
        }
    }
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_glm_Qx.get(), Qx.data(), Qx.size() * sizeof(double), cudaMemcpyHostToDevice,
                                 ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_glm_mask.get(), mask.data(), mask.size(), cudaMemcpyHostToDevice, ctx->stream));
    if (cases)
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_glm_case.get(), cmask.data(), cmask.size(), cudaMemcpyHostToDevice,
                                     ctx->stream));
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_glm_z0.get(), z0.data(), q * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->c_h2d += (int64_t)(Qx.size() * sizeof(double) + mask.size() + cmask.size() + q * sizeof(double));
    return VPCA_OK;
}

// Sets the GLM state under ctx->mu: q columns (0: none), the model, R regression samples and y~^T y~ (linear).
void glm_commit(vpca_ctx* ctx, int q, bool logistic, int R, double yty, int64_t* n_used) {
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->glm_q = q;
    ctx->glm_logistic = logistic;
    ctx->glm_nreg = R;
    ctx->glm_yty = yty;
    if (n_used) *n_used = R;
}

// The logistic null fit: theta (q) maximising l over all R regression samples with Q alone, by the Newton passes of
// glm_logistic_kernel (DESIGN.md 16) from theta = 0, in FP64 on the host.  Returns the passes, or 0 without convergence.
int glm_null_fit(const std::vector<double>& Q, const std::vector<double>& y, int q, std::vector<double>& theta) {
    const int R = (int)y.size();
    std::vector<double> Qr((size_t)R * q);   // row-major copy: one sample's q values together
    for (int c = 0; c < q; ++c)
        for (int i = 0; i < R; ++i) Qr[(size_t)i * q + c] = Q[(size_t)c * R + i];
    std::vector<double> th(q, 0.0), thp(q, 0.0), del(q, 0.0), H((size_t)q * q), gr(q), sr(q);
    double lp = 0.0;
    int halv = 0;
    for (int k = 1; k <= 25; ++k) {
        std::fill(H.begin(), H.end(), 0.0);
        std::fill(gr.begin(), gr.end(), 0.0);
        double l = 0.0;
        for (int i = 0; i < R; ++i) {
            const double* x = Qr.data() + (size_t)i * q;
            double eta = 0.0;
            for (int c = 0; c < q; ++c) eta += x[c] * th[c];
            const double e = std::exp(-std::fabs(eta)), rd = 1.0 / (1.0 + e);
            const double mu = eta >= 0.0 ? rd : e * rd, w = e * rd * rd, r = y[i] - mu;
            const double m = y[i] != 0.0 ? -eta : eta;
            l -= std::fmax(m, 0.0) + std::log1p(e);
            for (int a = 0; a < q; ++a) {
                gr[a] += r * x[a];
                const double wa = w * x[a];
                for (int b = 0; b <= a; ++b) H[(size_t)a * q + b] += wa * x[b];
            }
        }
        if (!std::isfinite(l)) return 0;
        if (k > 1 && l < lp - 1e-10 * std::fabs(lp)) {
            if (halv == 8) return 0;
            ++halv;
            for (int c = 0; c < q; ++c) {
                del[c] *= 0.5;
                th[c] = thp[c] + del[c];
            }
            continue;
        }
        halv = 0;
        for (int j = 0; j < q; ++j) {   // Cholesky, L below the diagonal of H, sr = 1 / L_jj
            double d = H[(size_t)j * q + j];
            for (int c = 0; c < j; ++c) d -= H[(size_t)j * q + c] * H[(size_t)j * q + c];
            if (!(d > 0.0)) return 0;
            sr[j] = 1.0 / std::sqrt(d);
            for (int i = j + 1; i < q; ++i) {
                double x = H[(size_t)i * q + j];
                for (int c = 0; c < j; ++c) x -= H[(size_t)i * q + c] * H[(size_t)j * q + c];
                H[(size_t)i * q + j] = x * sr[j];
            }
        }
        double dd = 0.0;
        for (int i = 0; i < q; ++i) {
            double z = gr[i];
            for (int c = 0; c < i; ++c) z -= H[(size_t)i * q + c] * gr[c];
            gr[i] = z * sr[i];
            dd += gr[i] * gr[i];
        }
        for (int i = q - 1; i >= 0; --i) {
            double x = gr[i];
            for (int c = i + 1; c < q; ++c) x -= H[(size_t)c * q + i] * del[c];
            del[i] = x * sr[i];
        }
        if (!std::isfinite(dd)) return 0;
        if (dd <= 1e-18) {
            for (int c = 0; c < q; ++c) theta[c] = th[c] + del[c];
            return k;
        }
        lp = l;
        for (int c = 0; c < q; ++c) {
            thp[c] = th[c];
            th[c] += del[c];
        }
    }
    return 0;
}
}  // namespace

int vpca_glm_begin(vpca_ctx* ctx, const double* pheno, const double* covar, int32_t n_covar, int64_t* n_used) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    glm_commit(ctx, 0, false, 0, 0.0, nullptr);   // a refused call leaves no GLM state
    std::vector<int> idx;   // the regression samples
    int rc = glm_samples(ctx, "vpca_glm_begin", pheno, covar, n_covar, idx);
    if (rc != VPCA_OK) return rc;
    const int q = n_covar + 1, R = (int)idx.size();
    bool constant = true;
    for (int i = 1; i < R && constant; ++i) constant = pheno[idx[i]] == pheno[idx[0]];
    if (constant) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_glm_begin: the phenotype is constant over the regression samples");
    std::vector<double> Q, y(R);
    rc = glm_basis(ctx, "vpca_glm_begin", covar, n_covar, idx, Q);
    if (rc != VPCA_OK) return rc;
    for (int i = 0; i < R; ++i) y[i] = pheno[idx[i]];
    for (int pass = 0; pass < 2; ++pass)
        for (int k = 0; k < q; ++k) {
            const double* qk = Q.data() + (size_t)k * R;
            double r = 0.0;
            for (int i = 0; i < R; ++i) r += qk[i] * y[i];
            for (int i = 0; i < R; ++i) y[i] -= r * qk[i];
        }
    std::vector<double> z0(q, 0.0);
    double yty = 0.0;
    for (int i = 0; i < R; ++i) yty += y[i] * y[i];
    for (int k = 0; k < q; ++k)
        for (int i = 0; i < R; ++i) z0[k] += Q[(size_t)k * R + i] * y[i];
    rc = glm_upload(ctx, q, idx, Q, y, z0, false);
    if (rc != VPCA_OK) return rc;
    glm_commit(ctx, q, false, R, yty, n_used);
    return VPCA_OK;
}

int vpca_glm_logistic_begin(vpca_ctx* ctx, const double* pheno, const double* covar, int32_t n_covar, int64_t* n_used) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    glm_commit(ctx, 0, false, 0, 0.0, nullptr);   // a refused call leaves no GLM state
    const char* fn = "vpca_glm_logistic_begin";
    std::vector<int> idx;
    int rc = glm_samples(ctx, fn, pheno, covar, n_covar, idx);
    if (rc != VPCA_OK) return rc;
    for (int s = 0; s < ctx->n; ++s)
        if (std::isfinite(pheno[s]) && pheno[s] != 0.0 && pheno[s] != 1.0)
            return fail(ctx, VPCA_ERR_BAD_ARG, "%s: the phenotype of sample %d is %.17g, not 0 (control), 1 (case) or "
                        "NaN (missing)", fn, s, pheno[s]);
    const int q = n_covar + 1, R = (int)idx.size();
    std::vector<double> y(R);
    int cases = 0;
    for (int i = 0; i < R; ++i) {
        y[i] = pheno[idx[i]];
        cases += y[i] != 0.0;
    }
    if (cases == 0 || cases == R)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: %d cases and %d controls among the %d regression samples; a logistic test "
                    "needs both", fn, cases, R - cases, R);
    std::vector<double> Q;
    rc = glm_basis(ctx, fn, covar, n_covar, idx, Q);
    if (rc != VPCA_OK) return rc;
    std::vector<double> theta(q, 0.0);
    if (glm_null_fit(Q, y, q, theta) == 0)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: the null model (the intercept and the %d covariates, without a variant) "
                    "does not converge in 25 Newton passes: a covariate separates the cases from the controls", fn,
                    n_covar);
    rc = glm_upload(ctx, q, idx, Q, y, theta, true);
    if (rc != VPCA_OK) return rc;
    glm_commit(ctx, q, true, R, 0.0, n_used);
    return VPCA_OK;
}

namespace {
// The three GLM *_bed calls: the argument and state rules (the state's model must be logistic, or linear), then the
// rows through stage_rows with the model's kernels per chunk: glm_linear, or glm_logistic in firth_mode.  out_passes and
// out_firth (logistic only) may be null.
int glm_bed_rows(vpca_ctx* ctx, const char* fn, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                 int32_t counted_allele, bool logistic, int firth_mode, double* out, int32_t* out_err, int32_t* out_passes,
                 uint8_t* out_firth) {
    int rc = rows_args(ctx, fn, rows, nv, stride_bytes, (ctx->n + 3) / 4, out != nullptr && out_err != nullptr);
    if (rc != VPCA_OK) return rc;
    if (counted_allele != 1 && counted_allele != 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "%s: counted_allele must be 1 (A1) or 2 (A2), not %d", fn, counted_allele);
    const char* begin = logistic ? "vpca_glm_logistic_begin" : "vpca_glm_begin";
    int q = 0, n_reg = 0;
    double yty = 0.0;
    {
        std::lock_guard<std::mutex> lk(ctx->mu);
        if (ctx->glm_q == 0) return fail(ctx, VPCA_ERR_STATE, "%s needs a %s since the last reset", fn, begin);
        if (ctx->glm_logistic != (int)logistic)
            return fail(ctx, VPCA_ERR_STATE, "%s: the GLM state is %s (%s); a %s test needs %s", fn,
                        logistic ? "linear" : "logistic", logistic ? "vpca_glm_begin" : "vpca_glm_logistic_begin",
                        logistic ? "logistic" : "linear", begin);
        q = ctx->glm_q;
        n_reg = ctx->glm_nreg;
        yty = ctx->glm_yty;
    }
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int n = ctx->n;
    const int64_t step = grm_step(nv, stride_bytes);
    const bool fallback = firth_mode == VPCA_GLM_FIRTH_FALLBACK;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = cudaSuccess;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
        if (e == cudaSuccess) e = ctx->d_glm_sums.ensure(step * (logistic ? 6 : kGlmRec));
        if (e == cudaSuccess) e = ctx->d_glm_out.ensure(step * 6);
        if (e == cudaSuccess) e = ctx->d_glm_err.ensure(step);
        if (e == cudaSuccess && logistic) e = ctx->d_glm_passes.ensure(step);
        if (e == cudaSuccess && firth_mode) e = ctx->d_glm_firth.ensure(step);
        if (e == cudaSuccess && fallback) e = ctx->d_glm_idx.ensure(step);
        if (e == cudaSuccess && fallback) e = ctx->d_glm_nf.ensure(1);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "GLM buffers: %s", cudaGetErrorString(e));
        }
    }
    return stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t v, int64_t nvc) -> int {
        if (logistic)
            CUDA_OK(ctx, glm_logistic(d_rows, stride_bytes, (int)nvc, n, q, ctx->d_glm_Qx.get(), ctx->d_glm_mask.get(),
                                      ctx->d_glm_case.get(), ctx->d_glm_z0.get(), counted_allele, ctx->d_glm_sums.get(),
                                      ctx->d_glm_out.get(), ctx->d_glm_err.get(), ctx->d_glm_passes.get(), firth_mode,
                                      firth_mode ? ctx->d_glm_firth.get() : nullptr,
                                      fallback ? ctx->d_glm_idx.get() : nullptr, fallback ? ctx->d_glm_nf.get() : nullptr,
                                      L.stream));
        else
            CUDA_OK(ctx, glm_linear(d_rows, stride_bytes, (int)nvc, n, q, n_reg, ctx->d_glm_Qx.get(), ctx->d_glm_mask.get(),
                                    ctx->d_glm_z0.get(), yty, counted_allele, ctx->d_glm_sums.get(), ctx->d_glm_out.get(),
                                    ctx->d_glm_err.get(), L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(out + v * 6, ctx->d_glm_out.get(), (size_t)nvc * 6 * sizeof(double),
                                     cudaMemcpyDeviceToHost, L.stream));
        CUDA_OK(ctx, cudaMemcpyAsync(out_err + v, ctx->d_glm_err.get(), (size_t)nvc * sizeof(int32_t),
                                     cudaMemcpyDeviceToHost, L.stream));
        if (out_passes)
            CUDA_OK(ctx, cudaMemcpyAsync(out_passes + v, ctx->d_glm_passes.get(), (size_t)nvc * sizeof(int32_t),
                                         cudaMemcpyDeviceToHost, L.stream));
        if (out_firth)
            CUDA_OK(ctx, cudaMemcpyAsync(out_firth + v, ctx->d_glm_firth.get(), (size_t)nvc, cudaMemcpyDeviceToHost,
                                         L.stream));
        // linear: 3 as counted since the linear tests began; logistic: the count kernels, then the maximum-likelihood
        // and finish kernels (5 as counted before the Firth tests), the selection and the Firth kernel (fallback), or
        // the Firth and finish kernels (always)
        ctx->c_launches += !logistic ? 3 : firth_mode == 0 ? 5 : fallback ? 6 : 4;
        ctx->c_d2h += nvc * (6 * (int64_t)sizeof(double) + (out_passes ? 2 : 1) * (int64_t)sizeof(int32_t) +
                             (out_firth ? 1 : 0));
        return VPCA_OK;
    });
}
}  // namespace

int vpca_glm_linear_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                        double* out, int32_t* out_err) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    return glm_bed_rows(ctx, "vpca_glm_linear_bed", rows, nv, stride_bytes, counted_allele, false, 0, out, out_err,
                        nullptr, nullptr);
}

int vpca_glm_logistic_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                          double* out, int32_t* out_err, int32_t* out_passes) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    return glm_bed_rows(ctx, "vpca_glm_logistic_bed", rows, nv, stride_bytes, counted_allele, true, 0, out, out_err,
                        out_passes, nullptr);
}

int vpca_glm_firth_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                       int32_t mode, double* out, int32_t* out_err, int32_t* out_passes, uint8_t* out_firth) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (mode != VPCA_GLM_FIRTH_FALLBACK && mode != VPCA_GLM_FIRTH_ALWAYS)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_glm_firth_bed: mode must be 1 (fallback) or 2 (always), not %d", mode);
    return glm_bed_rows(ctx, "vpca_glm_firth_bed", rows, nv, stride_bytes, counted_allele, true, mode, out, out_err,
                        out_passes, out_firth);
}

// ---- sample QC (samples.cu, DESIGN.md 11) -------------------------------------------------------------------------------
// Driver-side and synchronous, on rows of their own sample count: the context lends its device, a lane and scratch.  Rows
// are staged in chunks of at most kSmStageBytes in the context's driver-side pair (d_bed_rows).  The subset pass copies
// both ways: chunk i + 1 goes up on the lane's copy stream while a helper thread brings chunk i down on a stream of its
// own, so that the two copies (pageable, hence each blocking the thread that issues it) run at once on the two copy
// engines.
namespace {
constexpr int64_t kSmStageBytes = 64ll << 20;   // raw .bed bytes per staged chunk

// The D2H side of vpca_subset_bed_samples: copies chunk i down once the main thread has launched its kernel, and
// reports each finished copy, which frees the chunk's two buffers for chunk i + 2.
struct SubsetDownloader {
    std::mutex mu;
    std::condition_variable cv;
    int64_t launched = 0, copied = 0;   // chunks whose kernel is enqueued / whose rows are on the host
    bool stop = false;
    cudaError_t err = cudaSuccess;
    std::thread th;

    void launched_chunk(int64_t i) {
        {
            std::lock_guard<std::mutex> lk(mu);
            launched = i + 1;
        }
        cv.notify_all();
    }
    // blocks until `count` chunks are on the host; false on a copy error
    bool wait_copied(int64_t count) {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return copied >= count || err != cudaSuccess; });
        return err == cudaSuccess;
    }
    ~SubsetDownloader() {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv.notify_all();
        if (th.joinable()) th.join();
    }
};
}   // namespace

int vpca_sample_missing_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t n_samples,
                            int32_t* out_missing) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (n_samples < 1) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_sample_missing_bed: n_samples = %d must be >= 1", (int)n_samples);
    if (int rc = rows_args(ctx, "vpca_sample_missing_bed", rows, nv, stride_bytes, ((int64_t)n_samples + 3) / 4,
                           out_missing != nullptr))
        return rc;
    if (nv > 2147483647ll)
        return fail(ctx, VPCA_ERR_OVERFLOW, "vpca_sample_missing_bed: %lld rows could overflow an int32 count",
                    (long long)nv);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) {
        if (out_missing != nullptr) memset(out_missing, 0, (size_t)n_samples * sizeof(int32_t));
        return VPCA_OK;
    }
    const int64_t step = std::max<int64_t>(1, std::min(nv, kSmStageBytes / stride_bytes));
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = ctx->d_sm_miss.ensure(n_samples);
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "sample QC buffers for %lld rows of %lld bytes: %s", (long long)step,
                        (long long)stride_bytes, cudaGetErrorString(e));
        }
    }
    CUDA_OK(ctx, cudaMemsetAsync(ctx->d_sm_miss.get(), 0, (size_t)n_samples * sizeof(int32_t), L.stream));
    int rc = stage_rows(ctx, L, rows, nv, stride_bytes, step, bed_rows(ctx), [&](int, const uint8_t* d_rows, int64_t, int64_t nvc) -> int {
        CUDA_OK(ctx, sample_missing(d_rows, stride_bytes, (int)nvc, n_samples, ctx->d_sm_miss.get(), L.stream));
        ctx->c_launches += 1;
        return VPCA_OK;
    });
    if (rc != VPCA_OK) return rc;
    CUDA_OK(ctx, cudaMemcpyAsync(out_missing, ctx->d_sm_miss.get(), (size_t)n_samples * sizeof(int32_t), cudaMemcpyDeviceToHost,
                                 L.stream));
    ctx->c_d2h += 4 * (int64_t)n_samples;
    CUDA_OK(ctx, cudaStreamSynchronize(L.stream));
    return VPCA_OK;
}

int vpca_subset_bed_samples(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t n_samples,
                            const int32_t* keep_idx, int32_t m, uint8_t* out_rows, int64_t out_stride) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    if (n_samples < 1) return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_subset_bed_samples: n_samples = %d must be >= 1", (int)n_samples);
    if (int rc = rows_args(ctx, "vpca_subset_bed_samples", rows, nv, stride_bytes, ((int64_t)n_samples + 3) / 4,
                           keep_idx != nullptr && out_rows != nullptr))
        return rc;
    if (m < 1 || out_stride < ((int64_t)m + 3) / 4)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_subset_bed_samples: bad argument (m = %d must be >= 1, out_stride = %lld "
                    ">= ceil(m / 4))", (int)m, (long long)out_stride);
    if (keep_idx != nullptr)
        for (int32_t j = 0; j < m; ++j)
            if (keep_idx[j] < 0 || keep_idx[j] >= n_samples || (j > 0 && keep_idx[j] <= keep_idx[j - 1]))
                return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_subset_bed_samples: keep_idx[%d] = %d must be in [0, %d) and "
                            "above the entry before it", (int)j, (int)keep_idx[j], (int)n_samples);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (nv == 0) return VPCA_OK;
    const int64_t mb = ((int64_t)m + 3) / 4;
    const int64_t step = std::max<int64_t>(1, std::min(nv, kSmStageBytes / stride_bytes));
    const int64_t chunks = (nv + step - 1) / step;
    LaneGuard lg(ctx);
    if (lg.rc != VPCA_OK) return lg.rc;
    vpca_ctx::Lane& L = *lg.lane;
    {
        cudaError_t e = cudaSuccess;
        for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
            e = ctx->d_bed_rows[b].ensure(step * stride_bytes);
            if (e == cudaSuccess) e = ctx->d_sm_out[b].ensure(step * mb);
            if (e == cudaSuccess && ctx->sm_ev_copy[b] == nullptr)
                e = cudaEventCreateWithFlags(&ctx->sm_ev_copy[b], cudaEventDisableTiming);
            if (e == cudaSuccess && ctx->sm_ev_kern[b] == nullptr)
                e = cudaEventCreateWithFlags(&ctx->sm_ev_kern[b], cudaEventDisableTiming);
        }
        if (e == cudaSuccess) e = ctx->d_sm_idx.ensure(m);
        if (e == cudaSuccess && ctx->sm_d2h_stream == nullptr)
            e = cudaStreamCreateWithFlags(&ctx->sm_d2h_stream, cudaStreamNonBlocking);
        if (e != cudaSuccess) {
            cudaGetLastError();
            return fail(ctx, VPCA_ERR_NOMEM, "sample subset buffers for %lld rows of %lld bytes: %s", (long long)step,
                        (long long)stride_bytes, cudaGetErrorString(e));
        }
    }
    CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_sm_idx.get(), keep_idx, (size_t)m * sizeof(int32_t), cudaMemcpyHostToDevice, L.stream));
    ctx->c_h2d += 4 * (int64_t)m;
    SubsetDownloader down;
    const int device = ctx->cfg.device;
    down.th = std::thread([&down, ctx, device, chunks, step, nv, mb, out_rows, out_stride] {
        cudaError_t e = cudaSetDevice(device);
        for (int64_t i = 0; i < chunks && e == cudaSuccess; ++i) {
            {
                std::unique_lock<std::mutex> lk(down.mu);
                down.cv.wait(lk, [&] { return down.launched > i || down.stop; });
                if (down.launched <= i) return;
            }
            const int b = (int)(i & 1);
            const int64_t v = i * step, nvc = std::min(step, nv - v);
            e = cudaStreamWaitEvent(ctx->sm_d2h_stream, ctx->sm_ev_kern[b], 0);
            if (e == cudaSuccess)
                e = out_stride == mb
                        ? cudaMemcpyAsync(out_rows + (size_t)(v * mb), ctx->d_sm_out[b].get(), (size_t)(nvc * mb),
                                          cudaMemcpyDeviceToHost, ctx->sm_d2h_stream)
                        : cudaMemcpy2DAsync(out_rows + (size_t)(v * out_stride), (size_t)out_stride, ctx->d_sm_out[b].get(),
                                            (size_t)mb, (size_t)mb, (size_t)nvc, cudaMemcpyDeviceToHost, ctx->sm_d2h_stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->sm_d2h_stream);
            {
                std::lock_guard<std::mutex> lk(down.mu);
                if (e == cudaSuccess)
                    down.copied = i + 1;
                else
                    down.err = e;
            }
            down.cv.notify_all();
        }
        if (e != cudaSuccess) {   // cudaSetDevice failed before the first chunk
            std::lock_guard<std::mutex> lk(down.mu);
            down.err = e;
            down.cv.notify_all();
        }
    });
    for (int64_t i = 0; i < chunks; ++i) {
        const int b = (int)(i & 1);
        const int64_t v = i * step, nvc = std::min(step, nv - v);
        if (!down.wait_copied(i - 1)) break;   // chunk i - 2, the last user of buffers b, is on the host
        CUDA_OK(ctx, cudaMemcpyAsync(ctx->d_bed_rows[b].get(), rows + (size_t)v * stride_bytes, (size_t)(nvc * stride_bytes),
                                     cudaMemcpyHostToDevice, L.copy_stream));
        CUDA_OK(ctx, cudaEventRecord(ctx->sm_ev_copy[b], L.copy_stream));
        ctx->c_h2d += nvc * stride_bytes;
        CUDA_OK(ctx, cudaStreamWaitEvent(L.stream, ctx->sm_ev_copy[b], 0));
        CUDA_OK(ctx, subset_samples(ctx->d_bed_rows[b].get(), stride_bytes, (int)nvc, ctx->d_sm_idx.get(), m, ctx->d_sm_out[b].get(), mb,
                                    L.stream));
        CUDA_OK(ctx, cudaEventRecord(ctx->sm_ev_kern[b], L.stream));
        ctx->c_launches += 1;
        down.launched_chunk(i);
    }
    if (!down.wait_copied(chunks))
        return fail(ctx, VPCA_ERR_CUDA, "vpca_subset_bed_samples: device-to-host copy failed: %s",
                    cudaGetErrorString(down.err));
    ctx->c_d2h += nv * mb;
    return VPCA_OK;
}

int vpca_synth_dense_device(vpca_ctx* ctx, uint64_t seed, int64_t v0, int64_t nv, int mode, void* d_x, int64_t ld) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (d_x == nullptr || nv < 0 || ld < nv || v0 < 0 || (mode != 0 && mode != 1))
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_synth_dense_device: bad argument");
    if (mode == 1 && ctx->max_mult < 2)
        return fail(ctx, VPCA_ERR_BAD_ARG, "dosage mode needs max_multiplicity >= 2");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    cudaError_t e = synth_dense(seed, ctx->n, v0, nv, mode, ctx->elem_bits, d_x, ld, 0, ctx->stream);
    if (e != cudaSuccess) return fail(ctx, VPCA_ERR_CUDA, "synthetic generator: %s", cudaGetErrorString(e));
    ctx->c_launches += 2 * ((nv + (1 << 22) - 1) >> 22);
    return VPCA_OK;
}

int vpca_get_stats(vpca_ctx* ctx, vpca_stats* out) {
    if (ctx == nullptr || out == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    if (ctx->gram_timed && cudaEventSynchronize(ctx->ev_t1) == cudaSuccess) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ctx->ev_t0, ctx->ev_t1) == cudaSuccess) ctx->st.last_gram_ms = ms;
    } else if (!ctx->gram_timed) {
        ctx->st.last_gram_ms = ctx->lane_gram_ms.load();
    }
    if (ctx->eig_timed && cudaEventSynchronize(ctx->ev_e1) == cudaSuccess) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, ctx->ev_e0, ctx->ev_e1) == cudaSuccess) ctx->st.last_eig_ms = ms;
    }
    ctx->st.gram_launches = ctx->c_gram.load();
    ctx->st.kernel_launches = ctx->c_launches.load();
    ctx->st.h2d_bytes = ctx->c_h2d.load();
    ctx->st.d2h_bytes = ctx->c_d2h.load();
    *out = ctx->st;
    return VPCA_OK;
}

int vpca_gram_export_ipc(vpca_ctx* ctx, void* handle64) {
    if (ctx == nullptr || handle64 == nullptr) return fail(ctx, VPCA_ERR_BAD_ARG, "NULL argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->owned_S.get() == nullptr) return fail(ctx, VPCA_ERR_STATE, "the peer-reduce mode needs a library-owned Gram (vpca_config.d_gram == NULL)");
    if (ctx->band_rows != ctx->n) return fail(ctx, VPCA_ERR_STATE, "band-only Grams are shared with vpca_gram_set_peers_local");
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    cudaIpcMemHandle_t h;
    CUDA_OK(ctx, cudaIpcGetMemHandle(&h, ctx->d_S));
    memcpy(handle64, &h, sizeof(h));
    return VPCA_OK;
}

int vpca_gram_set_peers(vpca_ctx* ctx, const void* handles, int32_t world, int32_t rank) {
    if (ctx == nullptr || handles == nullptr || world < 1 || world > 16 || rank < 0 || rank >= world)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_gram_set_peers: bad argument (world <= 16)");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->owned_S.get() == nullptr) return fail(ctx, VPCA_ERR_STATE, "the peer-reduce mode needs a library-owned Gram");
    if (ctx->plan.num_peers != 0) return fail(ctx, VPCA_ERR_STATE, "peers already set");
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    const size_t nn = (size_t)ctx->n * ctx->n;
    for (int d = 0; d < world; ++d) {
        int32_t* base = ctx->d_S;
        if (d != rank) {
            cudaIpcMemHandle_t h;
            memcpy(&h, static_cast<const char*>(handles) + (size_t)d * sizeof(h), sizeof(h));
            void* ptr = nullptr;
            cudaError_t e = cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess);
            if (e != cudaSuccess) {
                for (int q = 0; q < d; ++q)
                    if (q != rank) cudaIpcCloseMemHandle(ctx->plan.peer_base[q]);
                return fail(ctx, VPCA_ERR_NCCL, "cudaIpcOpenMemHandle(rank %d) failed: %s", d, cudaGetErrorString(e));
            }
            base = static_cast<int32_t*>(ptr);
        }
        ctx->plan.peer_base[d] = base;
        ctx->plan.peer_S[d] = base;
        ctx->plan.peer_flags[d] = base + nn;
    }
    CUDA_OK(ctx, gram_preload_kernels(ctx->stream));   // nothing is loaded lazily behind a spinning barrier
    CUDA_OK(ctx, encode_preload_kernels());
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->plan.peers_ipc = true;
    ctx->plan.peer_rank = rank;
    ctx->plan.num_peers = world;
    sync_peers_to_lanes(ctx);
    return VPCA_OK;
}

// Same-process form of vpca_gram_set_peers: the caller owns all `world` contexts (one JVM driving the GPUs of the box,
// SURVEY 8b "process model"), so the Gram buffers are shared by enabling peer access between the devices instead of
// through IPC handles.  Contexts may also sit on the same device (tests on a 1-GPU box).
int vpca_gram_set_peers_local(vpca_ctx* const* ctxs, int32_t world) {
    if (ctxs == nullptr || world < 1 || world > 16) return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_gram_set_peers_local: world must be in [1, 16]");
    for (int r = 0; r < world; ++r) {
        if (ctxs[r] == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctxs[%d] is NULL", r);
        if (ctxs[r]->owned_S.get() == nullptr) return fail(ctxs[r], VPCA_ERR_STATE, "the peer-reduce mode needs a library-owned Gram");
        if (ctxs[r]->n != ctxs[0]->n) return fail(ctxs[r], VPCA_ERR_BAD_ARG, "all contexts must have the same n_samples");
        if (ctxs[r]->plan.num_peers != 0) return fail(ctxs[r], VPCA_ERR_STATE, "peers already set");
        for (int q = 0; q < r; ++q)
            if (ctxs[q] == ctxs[r]) return fail(ctxs[r], VPCA_ERR_BAD_ARG, "ctxs[%d] and ctxs[%d] are the same context", q, r);
    }
    for (int r = 0; r < world; ++r) {
        vpca_ctx* c = ctxs[r];
        CUDA_OK(c, cudaSetDevice(c->cfg.device));
        for (int d = 0; d < world; ++d) {
            const int od = ctxs[d]->cfg.device;
            if (od == c->cfg.device) continue;
            int can = 0;
            CUDA_OK(c, cudaDeviceCanAccessPeer(&can, c->cfg.device, od));
            if (!can) return fail(c, VPCA_ERR_NCCL, "device %d cannot access device %d (no NVLink / PCIe peer path)", c->cfg.device, od);
            cudaError_t e = cudaDeviceEnablePeerAccess(od, 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) {
                cudaGetLastError();
            } else if (e != cudaSuccess) {
                return fail(c, VPCA_ERR_NCCL, "cudaDeviceEnablePeerAccess(%d -> %d): %s", c->cfg.device, od, cudaGetErrorString(e));
            }
        }
    }
    // one host thread will enqueue barriers for several contexts: no kernel may be loaded lazily behind a spinning one
    for (int r = 0; r < world; ++r) {
        vpca_ctx* c = ctxs[r];
        CUDA_OK(c, cudaSetDevice(c->cfg.device));
        CUDA_OK(c, gram_preload_kernels(c->stream));
        CUDA_OK(c, encode_preload_kernels());
        CUDA_OK(c, cudaStreamSynchronize(c->stream));
    }
    for (int r = 0; r < world; ++r) {
        vpca_ctx* c = ctxs[r];
        std::lock_guard<std::mutex> lk(c->mu);
        for (int d = 0; d < world; ++d) {
            vpca_ctx* o = ctxs[d];
            // a band-only Gram is addressed through the virtual origin of the full matrix: row r of rank d lives at
            // base + (r - band_row0) * n, so (base - band_row0 * n) + r * n is valid for every row the rank owns
            c->plan.peer_base[d] = o->d_S;
            c->plan.peer_S[d] = o->d_S - (ptrdiff_t)o->band_row0 * o->n;
            c->plan.peer_flags[d] = o->d_S + (size_t)o->band_rows * o->n;
            c->plan.band_row0[d] = o->band_row0;
            c->plan.band_rows[d] = o->band_rows;
        }
        c->plan.peers_ipc = false;
        c->plan.peer_rank = r;
        c->plan.num_peers = world;
        sync_peers_to_lanes(c);
    }
    return VPCA_OK;
}

int vpca_gram_set_peer_mode(vpca_ctx* ctx, int32_t mode) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (mode != VPCA_PEER_REPLICATE && mode != VPCA_PEER_OWNER_ROWS)
        return fail(ctx, VPCA_ERR_BAD_ARG, "vpca_gram_set_peer_mode: unknown mode %d", mode);
    if (ctx->plan.num_peers < 1) return fail(ctx, VPCA_ERR_STATE, "call vpca_gram_set_peers first");
    const int world = ctx->plan.num_peers, n = ctx->n;
    if (mode == VPCA_PEER_OWNER_ROWS) {
        if (n < 64 * world)
            return fail(ctx, VPCA_ERR_UNSUPPORTED, "owner-rows mode needs n_samples >= 64 x world (%d < %d)", n, 64 * world);
        int ends[16];
        vpca_owner_row_bands(n, world, ends);
        for (int q = 0; q < 16; ++q) ctx->plan.own_end[q] = q < world ? ends[q] : n;
        // band-only Grams must hold exactly the rows their rank owns
        for (int q = 0; q < world; ++q) {
            const int lo = q == 0 ? 0 : ends[q - 1];
            if (ctx->plan.band_rows[q] != 0 && ctx->plan.band_rows[q] != n &&
                (ctx->plan.band_row0[q] != lo || ctx->plan.band_rows[q] != ends[q] - lo))
                return fail(ctx, VPCA_ERR_BAD_ARG, "rank %d stores rows [%d, %d) but owns [%d, %d) (see vpca_owner_row_bands)", q,
                            ctx->plan.band_row0[q], ctx->plan.band_row0[q] + ctx->plan.band_rows[q], lo, ends[q]);
        }
    } else if (ctx->band_rows != n) {
        return fail(ctx, VPCA_ERR_BAD_ARG, "a band-only Gram supports VPCA_PEER_OWNER_ROWS only");
    }
    ctx->plan.peer_mode = mode;
    sync_peers_to_lanes(ctx);
    return VPCA_OK;
}

int vpca_owner_row_bands(int32_t n_samples, int32_t world, int32_t* row_end) {
    if (row_end == nullptr || world < 1 || world > 16 || n_samples < 64 * world)
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_owner_row_bands: need 1 <= world <= 16 and n_samples >= 64 x world");
    // equal shares of the lower triangle: rows [0, R) hold R^2 / 2 cells -> R_q = n sqrt(q / world), on multiples of 32
    const int n = n_samples;
    int prev = 0;
    for (int q = 0; q < world; ++q) {
        int end = (q + 1 == world) ? n : (int)(std::sqrt((double)(q + 1) / world) * n / 32.0 + 0.5) * 32;
        end = std::max(end, prev + 32);
        // leave 32 rows for each later band without leaving the multiples of 32 (n itself need not be one)
        if (q + 1 < world) end = std::min(end, (n / 32) * 32 - 32 * (world - 1 - q));
        row_end[q] = end;
        prev = end;
    }
    return VPCA_OK;
}

int vpca_gram_gather(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->finalized) return fail(ctx, VPCA_ERR_STATE, "Gram already finalized");
    if (ctx->plan.num_peers < 2) return VPCA_OK;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, gram_peer_barrier(ctx->plan, ctx->stream));          // every rank's contributions have landed
    ctx->c_launches += 1;
    if (ctx->plan.peer_mode == 1 && ctx->band_rows == ctx->n) {
        CUDA_OK(ctx, gram_gather_rows(ctx->plan, ctx->d_S, ctx->n, ctx->stream));
        CUDA_OK(ctx, gram_peer_barrier(ctx->plan, ctx->stream));      // nobody resets a Gram a peer is still reading
        ctx->c_launches += 2;
    }
    return VPCA_OK;
}

int vpca_peer_barrier(vpca_ctx* ctx) {
    if (ctx == nullptr) return fail(nullptr, VPCA_ERR_BAD_ARG, "ctx is NULL");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (ctx->plan.num_peers < 2) return VPCA_OK;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, gram_peer_barrier(ctx->plan, ctx->stream));
    ctx->c_launches += 1;
    return VPCA_OK;
}

int vpca_debug_gram_profile(vpca_ctx* ctx, int64_t* out, int32_t max_ctas) {
    if (ctx == nullptr || out == nullptr || max_ctas <= 0) return fail(ctx, VPCA_ERR_BAD_ARG, "bad argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    return gram_read_profile(ctx->plan, reinterpret_cast<long long*>(out), max_ctas);
}

int vpca_debug_lanczos_profile(vpca_ctx* ctx, int64_t* out, int32_t max_steps) {
    if (ctx == nullptr || out == nullptr || max_steps <= 0) return fail(ctx, VPCA_ERR_BAD_ARG, "bad argument");
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!ctx->eig_ready || ctx->eig.d_lzprof.get() == nullptr) return 0;
    CUDA_OK(ctx, cudaSetDevice(ctx->cfg.device));
    CUDA_OK(ctx, cudaStreamSynchronize(ctx->stream));
    const int steps = std::min(max_steps, 32);
    CUDA_OK(ctx, cudaMemcpy(out, ctx->eig.d_lzprof.get(), (size_t)steps * 8 * sizeof(long long), cudaMemcpyDeviceToHost));
    return steps;
}

int64_t vpca_debug_device_bytes(void) { return g_device_bytes.load(); }

int vpca_debug_band_tiles(int32_t n_samples, int32_t cta_group, int32_t row0, int32_t rows, int32_t* out, int32_t max_tiles) {
    if (n_samples < 2 || max_tiles < 0 || row0 < 0 || rows < 1 || row0 + rows > n_samples)
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_debug_band_tiles: bad argument");
    return gram_debug_band_tiles(n_samples, cta_group, row0, row0 + rows, out, max_tiles);
}

int vpca_debug_max_clusters(int32_t device, int32_t cluster_size) {
    if (cluster_size < 1 || cluster_size > 16) return fail(nullptr, VPCA_ERR_BAD_ARG, "cluster_size must be in [1, 16]");
    if (cudaSetDevice(device) != cudaSuccess) return fail(nullptr, VPCA_ERR_CUDA, "cudaSetDevice(%d) failed", device);
    const int c = gram_debug_max_clusters(cluster_size);
    if (c < 0) return fail(nullptr, VPCA_ERR_CUDA, "cudaOccupancyMaxActiveClusters failed for cluster size %d", cluster_size);
    return c;
}

int vpca_debug_tiles(int32_t n_samples, int32_t cta_group, int32_t exact, int32_t* out, int32_t max_tiles) {
    if (n_samples < 2 || max_tiles < 0) return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_debug_tiles: bad argument");
    return gram_debug_tiles(n_samples, cta_group, exact, out, max_tiles);
}

int vpca_debug_plan(const int32_t* tiles, int32_t num_tiles, int32_t workers, int32_t kb_window, int32_t* out, int32_t max_pieces) {
    if (tiles == nullptr || num_tiles < 1 || workers < 1 || kb_window < 1 || (out == nullptr && max_pieces > 0))
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_debug_plan: bad argument");
    const int rc = gram_debug_plan(tiles, num_tiles, workers, kb_window, out, max_pieces);
    if (rc < 0) return fail(nullptr, VPCA_ERR_STATE, "vpca_debug_plan: the accumulators of a worker do not fit its budget (large-N schedule)");
    return rc;
}

int vpca_debug_schedule(int32_t n_samples, int32_t cta_group, int32_t exact, int32_t workers, int32_t kb_window,
                        int32_t kb_total, double front_frac, int32_t* out, int32_t max_pieces, int32_t* info) {
    if (n_samples < 2 || workers < 1 || workers > 1024 || kb_window < 1 || kb_total < 1 || !(front_frac <= 1.0) ||
        info == nullptr || max_pieces < 0 || (out == nullptr && max_pieces > 0))
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_debug_schedule: bad argument");
    const int rc = gram_debug_schedule(n_samples, cta_group, exact, workers, kb_window, kb_total, front_frac, out, max_pieces, info);
    if (rc < 0) return fail(nullptr, VPCA_ERR_STATE, "vpca_debug_schedule: the accumulators of a worker do not fit its budget");
    return rc;
}

int vpca_debug_rebalance(const int32_t* tiles, int32_t num_tiles, int32_t workers, int32_t kb_window, int32_t col_limit,
                         double* cum, int32_t* out, int32_t max_pieces) {
    if (tiles == nullptr || num_tiles < 1 || workers < 1 || kb_window < 1 || cum == nullptr || col_limit < 32 ||
        (out == nullptr && max_pieces > 0))
        return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_debug_rebalance: bad argument");
    const int rc = gram_debug_repair(tiles, num_tiles, workers, kb_window, col_limit, cum, out, max_pieces);
    if (rc < 0) return fail(nullptr, VPCA_ERR_STATE, "vpca_debug_rebalance: no feasible repair of this split");
    return rc;
}

/* Pinned host memory for callers that stage rows themselves (JNI direct ByteBuffers): the H2D copies of accumulate_*
 * then run at full PCIe rate and truly asynchronously.  Portable across devices. */
int vpca_host_alloc(size_t bytes, void** out) {
    if (out == nullptr || bytes == 0) return fail(nullptr, VPCA_ERR_BAD_ARG, "vpca_host_alloc: bad argument");
    cudaError_t e = cudaHostAlloc(out, bytes, cudaHostAllocPortable);
    if (e != cudaSuccess) {
        *out = nullptr;
        return fail(nullptr, VPCA_ERR_NOMEM, "cudaHostAlloc(%zu): %s", bytes, cudaGetErrorString(e));
    }
    return VPCA_OK;
}

int vpca_host_free(void* p) {
    if (p == nullptr) return VPCA_OK;
    cudaError_t e = cudaFreeHost(p);
    if (e != cudaSuccess) return fail(nullptr, VPCA_ERR_CUDA, "cudaFreeHost: %s", cudaGetErrorString(e));
    return VPCA_OK;
}

}  // extern "C"
