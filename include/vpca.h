/*
 * vpca.h -- C ABI of libvpca.so: the H100-native VariantsPca hot path
 *           (genotype encode -> N x N similarity/Gram accumulation -> centering + top-k eigenvectors).
 *
 * Drop-in boundary.  The reference (googlegenomics/spark-examples) has no FFI; the boundary is the
 * public method set of `class VariantsPcaDriver` as used by `main`
 * (src/main/scala/com/google/cloud/genomics/spark/examples/VariantsPca.scala:38-50).  Each entry
 * point below names the reference lines whose work it replaces; INTEGRATION.md shows the JNI class
 * (`NativePca`) and the Scala changes a maintainer would add to bind them.
 *
 * Conventions
 *   - plain C, no C++/torch types; every pointer is either HOST memory owned by the caller or a raw
 *     CUDA device pointer where the parameter name starts with `d_`.
 *   - every function returns VPCA_OK (0) or a negative vpca_status; vpca_last_error() gives the text.
 *     No C++ exception crosses the ABI.
 *   - a vpca_ctx owns one GPU's worth of state (device buffers, streams, staging); a vpca_pool owns one ctx per GPU
 *     of the box and is what one driver JVM holds (the reference's process model, VariantsPca.scala:38-50).
 *   - threading: accumulate_* / commit / abort may be called concurrently from many threads (the task threads of
 *     `mapPartitions`, VariantsPca.scala:184-189).  Host-input calls run on one of `staging_lanes` private lanes
 *     (streams + staging buffers): the context mutex is held for bookkeeping only, never across a copy, a kernel or
 *     a synchronisation, so the H2D copy and encode of one task overlap the Gram kernel of another.  One partition
 *     id belongs to one thread at a time (spark.speculation off).  reset / finalize / get_* / compute_pca are
 *     driver-side calls made when no accumulate call is in flight.
 *   - device-resident input (on_device tiles, panels) and everything driver-side is ordered on the stream given in
 *     vpca_config.stream (or a private stream); functions that return host data synchronise before returning.
 *   - there is no CPU fallback: vpca_create fails with VPCA_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef VPCA_H_
#define VPCA_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VPCA_VERSION_MAJOR 0
#define VPCA_VERSION_MINOR 2

typedef enum vpca_status {
    VPCA_OK = 0,
    VPCA_ERR_BAD_ARG = -1,
    VPCA_ERR_INDEX_OUT_OF_RANGE = -2, /* sample index outside [0, n_samples): the reference would throw
                                         (VariantsPca.scala:59 NoSuchElementException / :188 Breeze bounds) */
    VPCA_ERR_CUDA = -3,
    VPCA_ERR_NCCL = -4,     /* the cross-GPU reduction (`reduceByKey`, VariantsPca.scala:190) cannot run: no peer path
                               between two devices, or a peer mapping failed */
    VPCA_ERR_OVERFLOW = -5, /* an int32 similarity count (VariantsPca.scala:185) could exceed 2^31-1,
                               or a multiplicity does not fit the encoding */
    VPCA_ERR_STATE = -6,
    VPCA_ERR_NOMEM = -7,
    VPCA_ERR_UNSUPPORTED = -8
} vpca_status;

typedef enum vpca_dtype {
    VPCA_DTYPE_I8 = 0,  /* int8 genotype encoding, wgmma s8, exact int32 accumulation            */
    VPCA_DTYPE_BF16 = 1, /* bf16 genotype encoding, wgmma bf16, fp32 register accumulation flushed
                            into the int32 Gram before 2^24 could be reached (exact)              */
    VPCA_DTYPE_E2M1 = 2  /* 4-bit e2m1 cells (0, 1, 2 exact), two per byte in HBM; expanded in shared
                            memory to int8 holding twice the cell value, wgmma s8 with int32
                            accumulation, the flush divides by 4 (exact).  Half the HBM/L2 bytes per
                            cell, but the expansion makes its Gram several times slower than int8
                            (README): choose it only for the memory footprint.  Dense tiles need ld % 128 == 0 (panels: % 128), 32-byte alignment
                            and zero cells up to the next multiple of 128 variants;
                            max_multiplicity <= 2.                                                 */
} vpca_dtype;

typedef struct vpca_ctx vpca_ctx;

typedef struct vpca_config {
    uint32_t struct_size;      /* sizeof(vpca_config), for forward compatibility                     */
    int32_t n_samples;         /* N = common.indexes.size (VariantsPca.scala:183,199)                 */
    int32_t device;            /* CUDA device ordinal                                                  */
    int32_t dtype;             /* vpca_dtype                                                           */
    int32_t num_pc;            /* PcaConf.numPc (GenomicsConf.scala:85); default 2 when 0             */
    int32_t max_multiplicity;  /* largest value a genotype cell may take (1 = binary carriers, the
                                  reference rule VariantsPca.scala:58; 2 = dosage / a sample listed
                                  twice).  0 -> 2.  Used for the overflow guards.                     */
    int32_t partitions_in_flight; /* staging Grams for uncommitted partitions; 0 -> 4                 */
    int32_t staging_lanes;     /* host-input calls that may run concurrently on this GPU (each lane: two
                                  streams + double-buffered staging, ~1 GB); 0 -> 2, at most 16            */
    int64_t chunk_variants;    /* variants per device staging chunk for CSR input; 0 -> automatic     */
    int64_t chunk_nnz;         /* sample-index entries per device staging chunk; 0 -> automatic       */
    void* stream;              /* cudaStream_t to order all work on; NULL -> private stream           */
    void* d_gram;              /* optional caller-owned device buffer of n_samples^2 int32 (e.g. the
                                  tensor the host all-reduces with NCCL); NULL -> library-owned       */
    int32_t gram_band_row0;    /* gram_band_rows > 0: this context stores ONLY rows [row0, row0 + rows) of the   */
    int32_t gram_band_rows;    /* Gram -- the band it owns in VPCA_PEER_OWNER_ROWS mode (vpca_owner_row_bands);
                                  for cohorts whose full Gram should not be replicated per GPU (100 k
                                  samples: 40 GB; the reference's sizing note at VariantsPca.scala:176-177).
                                  0 -> the whole matrix                                                 */
} vpca_config;

/* ---- lifecycle ---------------------------------------------------------------------------- */
int vpca_version(void);                                  /* major * 1000 + minor */
int vpca_create(const vpca_config* cfg, vpca_ctx** out); /* replaces `new VariantsPcaDriver(conf)` state
                                                            that lives on the executor side
                                                            (VariantsPca.scala:81-85, :185)             */
int vpca_destroy(vpca_ctx* ctx);
/* Last error text of `ctx` (or of the calling thread when ctx == NULL).  Never NULL. */
const char* vpca_last_error(const vpca_ctx* ctx);
/* Zero the Gram and forget all partitions: start a new analysis on the same ctx. */
int vpca_reset(vpca_ctx* ctx);
/* Wait for everything enqueued on the context's stream (kernels of device-resident input, commits, gathers). */
int vpca_synchronize(vpca_ctx* ctx);
/* Pinned (page-locked, portable) host memory for callers that stage rows themselves -- the JNI binding wraps it in
 * direct ByteBuffers so that Spark tasks pack RDD[Seq[Int]] rows (VariantsPca.scala:153-168) straight into memory the
 * copy engines read at full PCIe rate, with no JVM array pinning. */
int vpca_host_alloc(size_t bytes, void** out);
int vpca_host_free(void* p);

/* ---- encode (VariantsPca.scala:56-60 extractCallInfo, :153-168 getCallsRdd) ---------------------
 * Host-side records arrive already projected to `RDD[Seq[Int]]` rows (CSR: row v = the sample indices
 * with hasVariation at variant v, duplicates allowed, any order; offsets has nv+1 entries).
 * vpca_encode_calls runs ONLY the device encode (CSR -> dense sample-major tile) and copies the tile
 * back: out[s * ld + v] = multiplicity of sample s in row v.  It exists so the encode kernel can be
 * parity-checked on its own; accumulate_calls below fuses it with the Gram.
 * Element type of `out` follows cfg.dtype (int8_t or bf16 bits as uint16_t); ld in elements, >= nv. */
int vpca_encode_calls(vpca_ctx* ctx, const int64_t* offsets, const int32_t* sample_idx, int64_t nv, void* out,
                      int64_t ld);

/* ---- similarity / Gram accumulation (VariantsPca.scala:182-191 getSimilarityMatrix) --------------
 * vpca_accumulate_calls = the body of `mapPartitions` (:184-189) for one batch of rows of Spark
 * partition `partition_id`: encode on device + S_partition += X X^T on wgmma tensor cores.  May be
 * called many times per partition.  Nothing is visible in the Gram until vpca_commit(partition_id)
 * (task success); vpca_abort discards it (task failure / retry), so a retried task is counted exactly
 * once -- the property the reference gets from returning a fresh matrix per task (:185).
 * partition_id < 0 means "no staging": accumulate straight into the Gram (single-shot callers). */
int vpca_accumulate_calls(vpca_ctx* ctx, int64_t partition_id, const int64_t* offsets, const int32_t* sample_idx,
                          int64_t nv);
/* Same, with 16-bit sample indices -- halves the host->device bytes of the dominant e2e cost.  Valid whenever
 * n_samples <= 65536, which covers every cohort the reference itself can process (MLlib's RowMatrix refuses more
 * than 65535 columns at VariantsPca.scala:226). */
int vpca_accumulate_calls_u16(vpca_ctx* ctx, int64_t partition_id, const int64_t* offsets, const uint16_t* sample_idx,
                              int64_t nv);
/* Packed wire format (SURVEY 8f-1): one bitmap per variant instead of an index list -- bit s (least significant bit
 * first) of row v is `hasVariation` of sample s (VariantsPca.scala:58), rows stride_bytes apart
 * (>= ceil(n_samples / 8)).  N/8 bytes per variant on the wire whatever the carrier count (313 B at N = 2504 against
 * ~4.3 KB of int32 indices for the synthetic cohort); expanded to cells on the device by a bit-matrix transpose.
 * Binary carriers only (a sample cannot be listed twice).  Same staging / commit semantics as vpca_accumulate_calls. */
int vpca_accumulate_bits(vpca_ctx* ctx, int64_t partition_id, const uint8_t* bits, int64_t nv, int64_t stride_bytes);
/* PLINK 1 .bed rows as they are on disk (variant-major; 2 bits per sample, low bits first: 00 homozygous A1,
 * 01 missing, 10 heterozygous, 11 homozygous A2), rows stride_bytes apart (>= ceil(n_samples / 4)).  `hasVariation`
 * (:58) = "carries the counted allele": counted_allele 1 -> codes {00, 10} (A1, PLINK's minor / alternate allele),
 * 2 -> codes {10, 11}; a missing call carries nothing, like a no-call.  Stands in for the retired ingestion
 * (rdd/VariantsRDD.scala:187-236) at N/4 bytes per variant.  Same staging / commit semantics as vpca_accumulate_calls. */
int vpca_accumulate_bed(vpca_ctx* ctx, int64_t partition_id, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                        int32_t counted_allele);
int vpca_commit(vpca_ctx* ctx, int64_t partition_id);
int vpca_abort(vpca_ctx* ctx, int64_t partition_id);

/* Pre-encoded dense input, sample-major: x[s * ld + v], s in [0, n_samples), v in [0, nv); element
 * type per cfg.dtype; ld (elements) must make rows 16-byte aligned.  on_device != 0: `x` is a device
 * pointer and is consumed in place (no copy) -- the resident-in-HBM path of bench.py; otherwise it is
 * host memory and is staged through the device in chunks.  Accumulates straight into the Gram. */
int vpca_accumulate_dense(vpca_ctx* ctx, const void* x, int64_t nv, int64_t ld, int on_device);

/* Device-resident input in PANEL layout -- the layout to keep a whole cohort in HBM: the nv variants are cut into
 * panels of `panel_variants` (a multiple of 128); panel p is a contiguous n_samples x panel_variants row-major block,
 * panels follow each other:  cell (s, v) at  (v / P) * n_samples * P + s * P + v % P  (cells; e2m1: two per byte),
 * cells after nv in the last panel are zero, d_x 32-byte aligned.  One Gram launch consumes everything.  Why: with a
 * row-major tile whose rows are megabytes apart every sample row sits on its own 2 MB page and each 128-row TMA box
 * touches 128 pages; panels keep the pages live per L2 window to a few dozen (measured 2x on 2504 x 5M int8). */
int vpca_accumulate_panels(vpca_ctx* ctx, const void* d_x, int64_t nv, int64_t panel_variants);

/* `reduceByKey(_ + _)` (:190) across GPUs is ONE all-reduce of the raw Gram buffer, driven by the host
 * (torch.distributed / NCCL in this repo, see INTEGRATION.md): all-reduce the n_samples^2 int32 at
 * vpca_gram_device_ptr() between the last commit and vpca_finalize_gram().  Until finalize only the
 * lower triangle (row >= col) of the buffer is meaningful. */
int vpca_gram_device_ptr(vpca_ctx* ctx, void** d_gram);
/* Fused alternative to the host-driven all-reduce (one process per GPU, all GPUs of one NVLink box): once every
 * rank has exchanged the 64-byte handle of vpca_gram_export_ipc() and called vpca_gram_set_peers() with the handles
 * of all ranks (rank order; needs a library-owned Gram, vpca_config.d_gram == NULL), the epilogue of the Gram
 * kernel adds every flushed accumulator straight into the Gram of EVERY rank (red.global.add.s32 on peer-mapped
 * memory), so compute and reduceByKey (:190) are one kernel.  Protocol per pass, on every rank:
 *   vpca_reset -> vpca_peer_barrier -> accumulate ... (commit) -> vpca_peer_barrier -> vpca_finalize_gram.
 * vpca_peer_barrier enqueues an all-rank barrier over peer-mapped flags on the context's stream. */
int vpca_gram_export_ipc(vpca_ctx* ctx, void* handle64);
int vpca_gram_set_peers(vpca_ctx* ctx, const void* handles, int32_t world, int32_t rank);
/* The same wiring when ONE process owns all `world` contexts (the reference's process model: one driver JVM whose task
 * threads share the executors' state, VariantsPca.scala:38-50, :184-190): peer access is enabled between the devices and
 * ctxs[r] becomes rank r.  Contexts may share a device (a 1-GPU box exercises the same kernels).  VPCA_ERR_NCCL when two
 * of the devices have no peer path.  vpca_pool_create does this for the contexts it creates. */
int vpca_gram_set_peers_local(vpca_ctx* const* ctxs, int32_t world);
int vpca_peer_barrier(vpca_ctx* ctx);
/* How the fused epilogue reduces across the peers set above:
 *   VPCA_PEER_REPLICATE (default): every flush goes into the Gram of every rank -- world x the remote traffic, no
 *     second phase.  Best at 2 GPUs.
 *   VPCA_PEER_OWNER_ROWS: reduce-scatter + all-gather.  Rank q owns a band of Gram rows (equal shares of the lower
 *     triangle, boundaries on multiples of 32); a flush goes only to the owner of its row, and vpca_gram_gather()
 *     (barrier, pull the rows owned by the other ranks over NVLink, barrier) completes every rank's copy.
 *     Protocol per pass:  vpca_reset -> vpca_peer_barrier -> accumulate ... (commit) -> vpca_gram_gather ->
 *     vpca_finalize_gram.  vpca_gram_gather() is valid in both modes (REPLICATE: just the closing barrier). */
enum { VPCA_PEER_REPLICATE = 0, VPCA_PEER_OWNER_ROWS = 1 };
int vpca_gram_set_peer_mode(vpca_ctx* ctx, int32_t mode);
int vpca_gram_gather(vpca_ctx* ctx);
/* Row bands of VPCA_PEER_OWNER_ROWS: rank q owns Gram rows [row_end[q-1], row_end[q]) (row_end[-1] = 0).  A context
 * created with vpca_config.gram_band_row0 / gram_band_rows set to its band stores nothing else: its kernels still
 * compute the whole lower triangle of their variant shard, but every flush leaves for the owner of its row, the bands
 * ARE the result (no gather), and vpca_get_gram_band reads them.  This is the biobank-scale form (100 k samples: a
 * 40 GB matrix, 2.6 - 14 GB per GPU at 8 GPUs) of `reduceByKey` (VariantsPca.scala:190). */
int vpca_owner_row_bands(int32_t n_samples, int32_t world, int32_t* row_end /* world entries */);
/* Rows [row0, row0 + rows) of the Gram as this context holds them (lower triangle meaningful before finalize;
 * n_samples int32 per row). */
int vpca_get_gram_band(vpca_ctx* ctx, int32_t row0, int32_t rows, int32_t* out);

/* Mirror the lower triangle into the upper one: after this the buffer equals the reference's
 * similarity matrix with all N^2 entries present (:189-190). */
int vpca_finalize_gram(vpca_ctx* ctx);
/* Copy the finalized Gram to host, row-major n_samples x n_samples int32 (the collected
 * RDD[((Int, Int), Int)] in key order). */
int vpca_get_gram(vpca_ctx* ctx, int32_t* out);
/* Checkpoint / resume of a long accumulation (SURVEY 8f-2): copy out / restore the Gram as accumulated so far
 * (committed partitions only, NOT finalized: lower triangle meaningful).  After vpca_load_partial_gram accumulation
 * continues on top of the restored counts; the caller keeps the watermark (which partitions are in it). */
int vpca_get_partial_gram(vpca_ctx* ctx, int32_t* out, int64_t* variants_in_gram /* may be NULL */);
/* variants_in_gram: how many variants the restored counts stand for (what vpca_get_partial_gram reported); they keep
 * counting against the int32 bound of a similarity count (VariantsPca.scala:185). */
int vpca_load_partial_gram(vpca_ctx* ctx, const int32_t* gram, int64_t variants_in_gram);
/* Variants folded into the Gram so far (committed partitions + direct input); negative vpca_status on error. */
int64_t vpca_variant_count(vpca_ctx* ctx);
/* Load a Gram (checkpoint restore / tests); marks it finalized. */
int vpca_set_gram(vpca_ctx* ctx, const int32_t* gram);

/* ---- computePca (VariantsPca.scala:198-231) --------------------------------------------------------
 * Centering (:199-223) in FP64 with the reference's operation order, then the top-k eigenvectors of the
 * centered matrix (= the first k columns of U that MLlib's RowMatrix.computePrincipalComponents returns
 * at :226) by Householder tridiagonalisation + Sturm bisection + inverse iteration on the GPU.
 *   vecs : n_samples x k, column-major -- the layout of `pca.toArray` (:227); vecs[i + c*n] is PC c of
 *          sample i.  Each column is unit-norm and sign-normalised (largest-|.| entry positive).
 *   evals: k eigenvalues of the centered matrix, descending (may be NULL).
 *   non_zero_rows: `rowSums.filter(_ > 0).size` (:207), may be NULL.
 * Like MLlib's RowMatrix, limited to 65 535 samples, and needs the whole Gram in this context plus an N x N FP64
 * workspace; for a Gram held as row bands, or for more samples, use vpca_compute_pca_bands below. */
int vpca_compute_pca(vpca_ctx* ctx, int32_t k, double* vecs, double* evals, int32_t* non_zero_rows);
/* Top-k principal coordinates of a Gram stored as row bands in `world` contexts of this process (beyond
 * VariantsPca.scala:224-227: no replica of S and no N x N FP64 matrix, no 65 535-sample limit).
 *   ctxs[q] holds rows [row0_q, row0_q + rows_q) (vpca_config.gram_band_row0 / _rows); the bands cover [0, N) in rank order
 *   with no gap or overlap, all with the same n_samples; a context that stores the whole Gram is the band [0, N), so
 *   world = 1 with an ordinary context is legal.  Every context must be finalized (VPCA_ERR_STATE otherwise); owner-flush
 *   (VPCA_PEER_OWNER_ROWS + vpca_gram_gather) and owner-computes (no peers) bands are both accepted.  The bands are only
 *   read.  1 <= world <= 16, 1 <= k <= min(N, max(num_pc of ctxs[0], 16)), else VPCA_ERR_BAD_ARG.
 *   vecs / evals / non_zero_rows as for vpca_compute_pca.
 * Lanczos with full reorthogonalisation driven from ctxs[0]; each step's product S v is sharded over the bands (every
 * stored lower-triangle cell read once, for its row and for its transpose) and the partials are added in rank order, so
 * repeated calls on the same bands give the same bits.  There is no direct-solver fallback (it would need the N x N
 * matrix): breakdown (e.g. a zero Gram), no convergence within the step budget (VPCA_EIG_MAXIT) or an eigenvalue missed
 * by a single Krylov sequence returns VPCA_ERR_UNSUPPORTED, with the reason in vpca_last_error(ctxs[0]).  ctxs[0]'s
 * vpca_stats report the solve (eig_method 4).  Driver-side: no accumulation may be in flight in any of the contexts.
 * On success every context in ctxs holds U (N x k, FP64, column-major) and the k eigenvalues on its own device for the
 * loadings below, as after vpca_compute_pca: ctxs[0] reads its solver's vectors, every other context gets a copy of the
 * first min(k, 16) columns in a buffer of N x 16 doubles it allocates on the first such solve (cudaMemcpyPeerAsync after
 * the solve, also between contexts on one device).  The call clears U on every context it names before it starts, so a
 * failed solve leaves no vectors behind; the most recent successful vpca_compute_pca / _bands of a context wins. */
int vpca_compute_pca_bands(vpca_ctx* const* ctxs, int32_t world, int32_t k, double* vecs, double* evals,
                           int32_t* non_zero_rows);
/* The centered matrix itself (row-major N x N doubles) for parity tests of :199-223. */
int vpca_get_centered(vpca_ctx* ctx, double* out);
/* Tridiagonal form of the centered matrix after the last vpca_compute_pca (diag: n, offdiag: n-1). */
int vpca_get_tridiagonal(vpca_ctx* ctx, double* diag, double* offdiag);

/* ---- variant loadings and projection (beyond VariantsPca.scala:224-230) ---------------------------------------------
 * The reference returns U (:226-227) and prints pc1 / pc2 per sample (:229-246); U alone means nothing without the
 * cohort's genotypes.  With C = J S J (the centering of :199-223) and C u_c = lambda_c u_c (vpca_compute_pca), u_c is
 * orthogonal to the ones vector, so
 *   loadings of variant v:   w[v][c] = sum_s x[s][v] u_c[s]      carriers n_v = sum_s x[s][v]   (x as encoded at :56-60)
 *   projection of cells y:   p_c = sum_v (y_v - n_v / N) w[v][c] / lambda_c
 * and a reference sample projected with its own loadings gets u_c back, in the units of the pc1 / pc2 columns of :229-246.
 * Cells are staged and encoded exactly as for the Gram (:56-60, :164; no-calls are 0); every sum runs in a fixed order,
 * no floating-point atomics, so results are bitwise reproducible.  w[v] depends on column v only: the three input forms
 * give the same bits.  Driver-side calls: one at a time per context, never concurrent with accumulation.
 *
 * After vpca_compute_pca(ctx, k, ...), or a vpca_compute_pca_bands(..., k, ...) that named ctx, U and the eigenvalues stay
 * on the device until the next vpca_reset / vpca_set_gram / vpca_load_partial_gram / vpca_finalize_gram of this context or
 * the next band solve that names it; the most recent successful solve wins.  Without them: VPCA_ERR_STATE on a context
 * that stores the whole Gram, VPCA_ERR_UNSUPPORTED on a band-only one (never solved, reset, or named by a failed band
 * solve).  A band-only context with U from a band solve computes loadings of any variants, whatever rows it stores; its
 * host forms run on the staging lanes it has for staged partitions.  Loadings of k' <= k components, k' in [1, 16]:
 *   out_w[v * k' + c] = sum_s x[s][v] * U[s][c] (FP64), out_count[v] = sum_s x[s][v] (exact).  Rows without carriers are
 *   legal (w = 0).  VPCA_ERR_INDEX_OUT_OF_RANGE for a sample index >= n_samples.  _panels: device input in the layout of
 *   vpca_accumulate_panels, device outputs, ordered on the ctx stream.
 * Up to 65 535 samples a thread sums each variant over all samples in order; above, the samples are cut into 4 ranges
 * whose bounds depend on n_samples alone and the 4 partials are added in range order.  Either way w[v] depends on column
 * v, U and n_samples only: every rank, input form and panel width gives it the same bits.  (Diagnostic:
 * VPCA_LOADINGS_KERNEL=whole|split forces one of the two orders at any n_samples.) */
int vpca_loadings_calls(vpca_ctx* ctx, int32_t k, const int64_t* offsets, const int32_t* sample_idx, int64_t nv,
                        double* out_w, int32_t* out_count);
int vpca_loadings_bed(vpca_ctx* ctx, int32_t k, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                      double* out_w, int32_t* out_count);
int vpca_loadings_panels(vpca_ctx* ctx, int32_t k, const void* d_x, int64_t nv, int64_t panel_variants,
                         double* d_w, int32_t* d_count);
/* Projection, in a context whose n_samples is the NEW cohort's size M (its Gram is unused; a band-only context is refused
 * with VPCA_ERR_UNSUPPORTED, so a cohort placed on the axes of a band solve is projected in an ordinary context).  vpca_project_begin zeroes
 * the M x k FP64 accumulator (k in [1, 16]); vpca_reset drops it.  Every row passed is a variant of the new cohort,
 * aligned with w (nv x k, variant-major, as vpca_loadings_* wrote it) and mean (nv, n_v / N of the reference): rows with
 * no carriers still contribute -mean * w.  Successive calls add up (per call in variant order; across calls in call
 * order).  VPCA_ERR_STATE before vpca_project_begin.
 * vpca_project_get: out[s + c*M] = acc[s][c] / evals[c] (column-major like vpca_compute_pca); evals = 1 reads the raw
 * sums (e.g. to add the sums of several GPUs before dividing). */
int vpca_project_begin(vpca_ctx* ctx, int32_t k);
int vpca_project_calls(vpca_ctx* ctx, const int64_t* offsets, const int32_t* sample_idx, int64_t nv, const double* w,
                       const double* mean);
int vpca_project_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                     const double* w, const double* mean);
int vpca_project_panels(vpca_ctx* ctx, const void* d_x, int64_t nv, int64_t panel_variants, const double* d_w,
                        const double* d_mean);
int vpca_project_get(vpca_ctx* ctx, const double* evals, double* out);

/* ---- KING-robust kinship between the samples (beyond VariantsPca.scala: which samples to leave out of the PCA) ------------
 * Related samples add excess sharing to S (VariantsPca.scala:182-191) that the top components can pick up as an axis of
 * their own; the usual remedy is kinship first, PCs of an unrelated subset, projection of the relatives (above).  The
 * estimator is KING-robust's between-family kinship (Manichaikul et al., Bioinformatics 26:2867, 2010; PLINK 2's
 * --make-king-table).  PLINK 1 .bed rows (as vpca_accumulate_bed) are encoded into three int8 indicator planes stacked as
 * 3N rows -- het (code 10), hom A1 (00), hom A2 (11); a missing call (01) sets none -- and G = Y Y^T runs on the int8 Gram
 * kernel, exact int32, with a Gram schedule of its own.  For a pair a < b (lower-triangle entries of G, DESIGN.md 7):
 *   HETHET = G[b][a]   IBS0 = G[2N+b][N+a] + G[2N+a][N+b]   HET1_HOM2 = G[N+b][a] + G[2N+b][a]
 *   HET2_HOM1 = G[N+a][b] + G[2N+a][b]   NSNP = the four + G[N+b][N+a] + G[2N+b][2N+a]   (variants both samples called)
 *   KINSHIP = (HETHET - 2 IBS0) / (2 HETHET + HET1_HOM2 + HET2_HOM1), numerator and denominator exact int64 converted to
 *   double, one correctly rounded division: bit-reproducible; NaN when the denominator is 0.
 * Driver-side calls: one at a time per context, never concurrent with accumulation.  The planes are int8 whatever
 * cfg.dtype is.  The 3N x 3N int32 counts (9 N^2 x 4 bytes: 17 GB at the limit) are allocated on the first
 * vpca_kinship_bed; vpca_reset zeroes them; vpca_set_gram / finalize_gram / compute_pca* and accumulation leave them alone,
 * and kinship calls leave the PCA Gram alone.  VPCA_ERR_UNSUPPORTED when n_samples > 21 845 (3N <= 65 535) or on a
 * band-only context.
 * vpca_kinship_bed: adds the rows (stride_bytes >= ceil(n_samples / 4)) to the counts; successive calls add up, and any split
 *   of the rows into calls gives the same counts.  Rows are staged on a lane (H2D overlapped with the previous chunk's
 *   work); returns after the last chunk is counted.  VPCA_ERR_OVERFLOW, before any row is staged, when the kinship
 *   variants would pass 2^31 - 1.
 * vpca_kinship_pairs: selects pairs -- every pair, NaN included, when min_kinship = -INFINITY, else KINSHIP >= min_kinship
 *   (NaN never passes) -- and writes the first min(total, max_pairs) in order of b, then a (row-major lower triangle):
 *   out_ids[2p] = a, out_ids[2p + 1] = b (a < b); out_counts[5p ..] = NSNP, HETHET, IBS0, HET1_HOM2, HET2_HOM1;
 *   out_kinship[p].  *n_pairs = the total selected (may exceed max_pairs); max_pairs = 0 with NULL outputs counts only.
 *   May be called any number of times on the same counts.  Two passes (count + scan, then emit in row batches through a
 *   bounded device scratch), no sort, no floating-point atomics.  VPCA_ERR_STATE when no kinship row was added since
 *   vpca_create / vpca_reset. */
int vpca_kinship_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes);
int vpca_kinship_pairs(vpca_ctx* ctx, double min_kinship, int64_t max_pairs, int32_t* out_ids, int32_t* out_counts,
                       double* out_kinship, int64_t* n_pairs);

/* ---- principal coordinates of an unrelated subset (kinship, then PCs of the unrelated, then the relatives placed) -------
 * vpca_compute_pca_subset: the PCs of the samples K with keep[s] != 0 (keep: n_samples bytes), M = |K| >= 2, from the
 * finalized Gram of all the samples -- no genotype is read again (DESIGN.md 8).  S[K, K] is copied into an M x M buffer and
 * centred and solved exactly as vpca_compute_pca does in an M-sample context (VPCA_EIG, the same eigensolver selection,
 * sign rule and fallback), on a workspace of its own that is allocated on the first call and again whenever M changes.
 *   vecs (n_samples x k, column-major): rows of kept samples hold u_c -- the bits of vpca_set_gram(S[K, K]) +
 *     vpca_compute_pca in an M-sample context; rows of removed samples r hold their projection onto the axes of K,
 *       p_c(r) = (sum_{j in K} S[r][j] u_c[j] - (1/M) sum_{j in K} rho_j u_c[j]) / lambda_c     rho_j = sum_{i in K} S[j][i]
 *     which is vpca_project_* of r's genotypes with the kept samples' loadings (FP64, sums in a fixed order, no
 *     floating-point atomics).  All samples kept: the bits of vpca_compute_pca.
 *   evals: the k eigenvalues of the subset (may be NULL); non_zero_rows: the nonzero row sums of S[K, K] (may be NULL).
 * Afterwards vpca_loadings_* return the kept samples' loadings: w[v][c] = sum_{s in K} x[s][v] u_c[s] and
 * count[v] = sum_{s in K} x[s][v], with the bits of vpca_loadings_* in an M-sample context fed only the kept columns (they
 * always sum the samples in the whole order, so this holds unless VPCA_LOADINGS_KERNEL=split forces that context's split);
 * projection is unaffected; vpca_get_tridiagonal returns VPCA_ERR_STATE; vpca_stats report this solve's eig_method /
 * eig_iterations.  The next vpca_compute_pca / _bands, vpca_reset, vpca_set_gram, vpca_load_partial_gram or
 * vpca_finalize_gram ends the subset state as it ends U.  The Gram and the kinship counts are only read.
 * Checked in vpca_compute_pca's order: VPCA_ERR_BAD_ARG for keep / vecs NULL, M < 2 or k outside
 * [1, min(M, max(num_pc, 16))]; then VPCA_ERR_STATE before vpca_finalize_gram; then VPCA_ERR_UNSUPPORTED on a band-only
 * context or above 65 535 samples.  k > 16 (num_pc > 16) is served in full; the loadings afterwards take k' <= 16. */
int vpca_compute_pca_subset(vpca_ctx* ctx, const uint8_t* keep, int32_t k, double* vecs, double* evals,
                            int32_t* non_zero_rows);

/* ---- LD pruning of the variants (beyond VariantsPca.scala: which variants go into S, VariantsPca.scala:182-191) ---------
 * Blocks of correlated nearby variants make the top components follow local haplotype structure instead of ancestry; the
 * usual remedy is to keep roughly independent variants only.  For variants i < j, over the samples called at both, with x
 * and y their A1 counts (0 / 1 / 2) and n, Sx, Sy, Sxx, Syy, Sxy the exact integer sums:
 *   cov = n Sxy - Sx Sy   vx = n Sxx - Sx^2   vy = n Syy - Sy^2     (int64, exact)
 *   r2 = (double(cov) * double(cov)) / (double(vx) * double(vy))     (each operation rounded once)
 * i and j are in LD iff vx > 0 && vy > 0 && r2 > r2_max.  The rows (PLINK 1 .bed, as vpca_accumulate_bed) are unpacked into
 * three int8 planes per chunk of variants -- A1 count, its square, called -- with the samples as the K axis, and every sum
 * is one lower-triangle entry of their Gram on the int8 Gram kernel (DESIGN.md 9).  The result does not depend on which
 * allele is counted (x -> 2 - x leaves r2 unchanged).
 * vpca_ld_prune_bed: window_lo[j] (nv entries, 0 <= window_lo[j] <= j, non-decreasing) is the first variant of j's window;
 *   keep[j] (nv bytes) = 1 iff no kept variant i with window_lo[j] <= i < j is in LD with j (keep-first, in order; the
 *   unique set in which no two kept variants of a window are in LD and every pruned variant is in LD with an earlier kept
 *   one of its window).  *n_pairs = the number of in-LD pairs (i, j) with window_lo[j] <= i < j; the first
 *   min(total, max_pairs) of them, in order of j, then i, go to out_pairs[2p] = i, out_pairs[2p + 1] = j and out_r2[p];
 *   max_pairs = 0 with NULL outputs counts only.  Driver-side and synchronous; int8 planes whatever cfg.dtype is.  The
 *   variants are walked in chunks that overlap by H = max_j (j - window_lo[j]), the samples in pieces of at most 32 768,
 *   so device memory grows with H but not with the number of samples or variants, apart from nv keep bytes: up to about
 *   2.8 GB at H = VPCA_LD_MAX_WINDOW (a 24 576 x 24 576 int32 Gram).  Buffers are allocated on the first call and freed
 *   by vpca_destroy; the PCA Gram, U, the kinship counts and the subset state are left alone.
 *   VPCA_ERR_BAD_ARG, before any row is staged: rows, window_lo, keep or n_pairs NULL, stride_bytes < ceil(n_samples / 4),
 *   a window_lo outside [0, j] or decreasing, r2_max not finite or outside [0, 1), max_pairs > 0 with NULL outputs.
 *   VPCA_ERR_UNSUPPORTED, before any row is staged, when H > VPCA_LD_MAX_WINDOW. */
#define VPCA_LD_MAX_WINDOW 4096
int vpca_ld_prune_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, const int64_t* window_lo,
                      double r2_max, uint8_t* keep, int64_t max_pairs, int64_t* out_pairs, double* out_r2,
                      int64_t* n_pairs);
/* vpca_ld_prune_bed_masked: vpca_ld_prune_bed with eligible[j] in {0, 1} (nv bytes; NULL = all eligible, which is
 *   vpca_ld_prune_bed bit for bit): keep[j] = 0 where eligible[j] = 0, and pairs are counted and listed only between
 *   eligible variants.  keep and the pairs equal vpca_ld_prune_bed on the eligible rows alone, with their window_lo
 *   recomputed (the first eligible variant at or after window_lo[j]), the pairs' indices staying those of all nv rows.
 *   The window limit is still checked on the window_lo given.  VPCA_ERR_BAD_ARG also for an eligible byte above 1. */
int vpca_ld_prune_bed_masked(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                             const int64_t* window_lo, const uint8_t* eligible, double r2_max, uint8_t* keep,
                             int64_t max_pairs, int64_t* out_pairs, double* out_r2, int64_t* n_pairs);

/* ---- variant quality control (beyond VariantsPca.scala: which variants go into S; DESIGN.md 10) ------------------------
 * The three usual variant filters before an ancestry PCA -- minor-allele frequency, missing-call rate, Hardy-Weinberg
 * equilibrium -- depend on four exact counts per variant, over all n_samples samples: HOM_A1 (code 00), HET (10), HOM_A2
 * (11), MISSING (01).  With n = HOM_A1 + HET + HOM_A2 the called samples and r = 2 min(HOM_A1, HOM_A2) + HET the copies of
 * the rarer allele, the HWE p-value is the exact test of Wigginton, Cutler & Abecasis (AJHG 76:887, 2005), in FP64:
 *   the relative probability t(h) of h hets given r and n is 1 at m = floor(r (2n - r) / (2n)) (+1 when its parity differs
 *   from r's), the mode or next to it; downward t(h - 2) = ((t(h) * h) * (h - 1)) / ((4 * (homr + 1)) * (homc + 1)), upward
 *   t(h + 2) = (((t(h) * 4) * homr) * homc) / ((h + 2) * (h + 1)), with homr = (r - h) / 2, homc = n - h - homr at h;
 *   each operation rounded once (no contraction).  A direction ends at its range end or at the first t that is exactly 0.
 *   T = sum of t, S = sum of the t <= t(obs) * (1 + 2^-40), both summed m first, then downward, then upward;
 *   p = min(S / T, 1), and p = 1 when r = 0 or n = 0.  A t(obs) that underflows to 0 gives p = 0 (true p below ~1e-300).
 * vpca_variant_qc_bed: rows are PLINK 1 .bed rows (as vpca_accumulate_bed; bytes past ceil(n_samples / 4) and the padding
 *   bits of the last byte are ignored); out_counts[4v ..] = HOM_A1, HET, HOM_A2, MISSING (exact, whatever the split of
 *   the rows into calls); out_hwe_p (may be NULL) = the p-value of each row.
 * vpca_hwe_exact: the same p-values from host counts in the layout above (MISSING ignored), for any n.
 * Driver-side and synchronous.  Rows are staged in chunks of at most 64 MB, the upload of chunk i + 1 overlapping the
 * count of chunk i, and tested in batches of about 2^18 rows (at least one chunk), so device memory does not grow with
 * nv: two chunk buffers (shared with the other driver-side .bed calls) and 24 bytes per batch row are allocated on the
 * first call and freed by vpca_destroy.  The PCA Gram, U, the kinship counts, the subset state and the LD state are left
 * alone.
 * VPCA_ERR_BAD_ARG, before any row is staged: rows / out_counts / counts / out_p NULL (nv > 0), nv < 0,
 *   stride_bytes < ceil(n_samples / 4), negative counts or counts whose sum exceeds 2^31 - 1. */
int vpca_variant_qc_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t* out_counts,
                        double* out_hwe_p);
int vpca_hwe_exact(vpca_ctx* ctx, const int32_t* counts, int64_t nv, double* out_p);

/* ---- variance-standardized genomic relationship matrix (beyond VariantsPca.scala: PLINK 2 / GCTA / EIGENSOFT's PCA;
 * DESIGN.md 13) ------------------------------------------------------------------------------------------------------
 * For each variant of PLINK 1 .bed rows (as vpca_accumulate_bed; bytes past ceil(n_samples / 4) and the padding bits of
 * the last byte are ignored), with HOM_A1, HET, HOM_A2 the exact counts of vpca_variant_qc_bed over all n_samples
 * samples, n = HOM_A1 + HET + HOM_A2 and a = 2 HOM_A1 + HET: the variant is USED iff 0 < a < 2n.  For a used variant,
 * r = min(a, 2n - a) counts the less common allele (A1 at a tie), and, each operation rounded once (no contraction),
 *   mu = r / n   q = r / (2n)   s = 1 / sqrt(mu (1 - q))   z_d = (d - mu) s
 * for that allele's count d of a called sample, z = 0 for a missing call.  GRM = (1/M) sum over the M used variants of
 * z z^T, FP64, each finished cell divided by M once.  Counting A1 or A2 gives the same GRM bit for bit.
 * The used variants are packed in row order into panels of a fixed number of variants and each panel is multiplied on the
 * FP64 tensor cores, so the GRM's bits depend only on the ordered sequence of used variants: not on how the rows are
 * split into calls, on stride_bytes or on skipped variants anywhere.
 * The sum accumulates in the eigensolver's FP64 N x N matrix (the one vpca_get_centered returns; 34 GB at 65 535
 * samples), allocated on the first call if no solve has allocated it.  The GRM calls leave the PCA Gram, U, the kinship
 * counts, the LD state, the QC counts and the subset state alone.  vpca_compute_pca and vpca_get_centered overwrite
 * the matrix, and so does a GRM solve by the direct reduction: afterwards vpca_get_grm, vpca_compute_pca_grm and
 * vpca_grm_bed return VPCA_ERR_STATE until vpca_reset.  Driver-side and synchronous.
 * vpca_grm_bed: adds the rows; successive calls add up.  Rows are staged in chunks of at most 64 MB on a lane (H2D of
 *   chunk i + 1 overlapped with the work on chunk i).  VPCA_ERR_STATE after vpca_grm_finalize (until vpca_reset).
 * vpca_grm_finalize: multiplies the last partial panel, divides by M and mirrors the lower triangle; *n_used = M (may be
 *   NULL).  Calling it again returns M again.  VPCA_ERR_STATE when M = 0, and from then on every GRM call until vpca_reset.
 * vpca_get_grm: the finalized GRM, symmetric N x N row-major.
 * vpca_compute_pca_grm: the k largest eigenpairs of the GRM as it is (no second centring), with the shapes, sign rule and
 *   k range of vpca_compute_pca: vecs N x k column-major, evals k (may be NULL), 1 <= k <= min(N, max(num_pc, 16)).
 *   The band solver's Lanczos on the FP64 cells from 512 samples up (the GRM stays valid); below that, with
 *   VPCA_EIG=direct and as the Lanczos fallback the direct reduction, which consumes the GRM.  It leaves no U for the
 *   carrier loadings: vpca_loadings_* return VPCA_ERR_STATE afterwards.  It keeps the first min(k, 16) columns of U in
 *   a buffer of its own (N x 16 doubles) for vpca_grm_loadings_bed, valid even after the direct reduction consumed the
 *   GRM, until the next vpca_reset / vpca_compute_pca* / vpca_set_gram / vpca_load_partial_gram / vpca_finalize_gram.
 * VPCA_ERR_BAD_ARG, before any row is staged: NULL ctx / rows (nv > 0) / out / vecs, nv < 0, stride_bytes <
 *   ceil(n_samples / 4), k out of range.  VPCA_ERR_UNSUPPORTED above 65 535 samples or on a band-only context. */
int vpca_grm_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes);
int vpca_grm_finalize(vpca_ctx* ctx, int64_t* n_used);
int vpca_get_grm(vpca_ctx* ctx, double* out);
int vpca_compute_pca_grm(vpca_ctx* ctx, int32_t k, double* vecs, double* evals);

/* ---- GRM loadings and projection (DESIGN.md 14) ----------------------------------------------------------------------
 * With Z the N x M matrix of used z values above (0 for a missing call and for an unused variant), GRM = Z Z^T / M and
 * GRM u_c = lambda_c u_c:
 *   loadings of variant v:          w[v][c] = sum_s tab[v][code(s, v)] u_c[s]          (the columns of Z^T U)
 *   projection of a sample's codes: p_c = sum_v tab_ref[v][y_v] w[v][c] / (M lambda_c)
 * so a sample of the reference projected with the reference's own tables and loadings gets u_c back.  A missing call
 * contributes 0 (mean imputation); the new cohort's own frequencies play no part.  Rows are PLINK 1 .bed rows of the
 * context's n_samples (as vpca_grm_bed; bytes past ceil(n_samples / 4) and padding bits are ignored), staged in chunks
 * of at most 64 MB and 2^20 rows on a lane.  FP64, no floating-point atomics, every sum in a fixed order.
 * vpca_grm_loadings_bed: out_w[v * k + c] (nv x k, variant-major) and out_tab[4 v + code] (nv x 4, indexed by the .bed
 *   code, all zero for an unused variant) for the U of the last vpca_compute_pca_grm.  The tables are recomputed from
 *   the rows given, with the bits of vpca_grm_bed's, so pass the rows the GRM was built from.  w[v] is the sum over the
 *   samples in order 0 .. n_samples - 1, one FMA chain per component: it depends on row v's codes, its table, U and
 *   n_samples only (not on nv, the chunk split or stride_bytes), and the first k' columns have the same bits at any
 *   k >= k'.  VPCA_ERR_STATE without GRM U; VPCA_ERR_BAD_ARG for k outside [1, min(k solved, 16)] or the argument rules
 *   of vpca_grm_bed (out_w / out_tab set when nv > 0); VPCA_ERR_UNSUPPORTED where vpca_grm_bed is.
 * vpca_grm_project_bed: adds sum_v tab[v][code(s, v)] w[v][c] (tab nv x 4 and w nv x k of the reference, aligned with
 *   the rows; k of vpca_project_begin) into the accumulator of vpca_project_begin; read it with vpca_project_get and
 *   evals[c] = M lambda_c.  Order: per staged chunk, fixed panels of 1024 variants each summed in variant order, the
 *   panel sums added into the accumulator in panel order; chunks in row order, calls in call order.  So the bits
 *   depend on the rows, tables, w and stride_bytes of each call, never on the run.  VPCA_ERR_STATE before
 *   vpca_project_begin; VPCA_ERR_UNSUPPORTED on a band-only context; VPCA_ERR_BAD_ARG as above. */
int vpca_grm_loadings_bed(vpca_ctx* ctx, int32_t k, const uint8_t* rows, int64_t nv, int64_t stride_bytes, double* out_w,
                          double* out_tab);
int vpca_grm_project_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, const double* tab,
                         const double* w);

/* ---- linear association tests (beyond VariantsPca.scala: PLINK 2's linear --glm; DESIGN.md 15) ---------------------
 * A quantitative trait y, an additive model, per variant on the complete cases.  The REGRESSION SAMPLES are the samples
 * with a finite phenotype and finite values for every covariate; C (N x q) is an intercept followed by the n_covar
 * covariate columns over them, q = n_covar + 1 <= 32.  For variant v, g is the count of the counted allele (0 for a
 * missing call), A_v the regression samples called at v and OBS_CT = |A_v|; least squares over A_v of
 * y = C gamma + beta g + e gives BETA = beta, SE = sqrt(sigma^2 [(X^T X)^-1]_gg) with sigma^2 = RSS / df and
 * df = OBS_CT - q - 1, T_STAT = BETA / SE, P = the two-sided Student t p-value I_{df / (df + T^2)}(df / 2, 1 / 2) (0 below
 * the double range), A1_FREQ = sum over A_v of g / (2 OBS_CT).  ERRCODE, checked in this order:
 *   VPCA_GLM_TOO_FEW_OBS   df < 1
 *   VPCA_GLM_CONST_ALLELE  g constant over A_v
 *   VPCA_GLM_VIF_INFINITE  the Schur term s = sum g^2 - (b^T P^-1 b) is <= 1e-10 x (sum g^2 - (sum g)^2 / OBS_CT), or the
 *                          covariates are collinear over A_v (a Cholesky pivot of P <= 1e-10; P = Q_A^T Q_A, see below)
 *   VPCA_GLM_NO_RESIDUAL   RSS <= 1e-12 x the residual phenotype's sum of squares over A_v
 * A flagged variant has BETA, SE, T_STAT and P NaN; so has A1_FREQ at OBS_CT = 0.
 * vpca_glm_begin: in FP64 on the host, orthonormalises C over the regression samples into Q (modified Gram-Schmidt applied
 *   twice), sets y~ = y - Q Q^T y and uploads Q, y~ and the regression mask.  pheno: N doubles, covar: N x n_covar
 *   row-major (may be NULL when n_covar = 0); NaN is missing.  *n_used (may be NULL) = the regression samples.
 *   VPCA_ERR_BAD_ARG, leaving no GLM state: pheno NULL, +-Inf in any input, n_covar < 0 or n_covar + 1 > 32, fewer than
 *   q + 2 regression samples, a constant phenotype, or a covariate collinear with the intercept and the columns before it
 *   (its residual norm <= 1e-9 x its norm; the message names it).  The state lasts until the next vpca_glm_begin or
 *   vpca_reset.
 * vpca_glm_linear_bed: out[6 v ..] = OBS_CT, A1_FREQ, BETA, SE, T_STAT, P and out_err[v] = ERRCODE of each of nv .bed rows
 *   of n_samples samples (as vpca_grm_bed; bytes past ceil(n_samples / 4) and the padding bits are ignored), counting
 *   A1 (counted_allele 1) or A2 (2).  Rows are staged as vpca_grm_loadings_bed stages them: chunks of at most 64 MB and
 *   2^20 rows on a lane.  Per variant one pass over its row sums b = Q^T g, sum g y~, sum g, sum g^2 and OBS_CT in sample
 *   order (FP64 FMA chains, exact integers), then over the fewer of its missing and its called regression samples the
 *   terms that turn Q^T Q = I into P = Q_A^T Q_A; a Cholesky solve of the bordered system follows.  Every output of a
 *   variant depends on its row's codes, Q, y~ and n_samples only: not on the chunk split, stride_bytes or the call.
 *   VPCA_ERR_STATE without GLM state; VPCA_ERR_BAD_ARG for counted_allele outside {1, 2} or the argument rules of
 *   vpca_grm_bed (out / out_err set when nv > 0).
 * Driver-side and synchronous.  The GLM calls leave the PCA Gram, U, the GRM, the kinship counts and the projection
 * accumulator alone; Q, y~ and the mask take N (q rounded up to 2, 4, 8, 16 or 32, plus 2) doubles and N / 4 bytes. */
enum {
    VPCA_GLM_OK = 0,
    VPCA_GLM_TOO_FEW_OBS = 1,
    VPCA_GLM_CONST_ALLELE = 2,
    VPCA_GLM_VIF_INFINITE = 3,
    VPCA_GLM_NO_RESIDUAL = 4,
    VPCA_GLM_LOGISTIC_CONVERGE_FAIL = 5,
    VPCA_GLM_FIRTH_CONVERGE_FAIL = 6
};
#define VPCA_GLM_MAX_Q 32
int vpca_glm_begin(vpca_ctx* ctx, const double* pheno, const double* covar, int32_t n_covar, int64_t* n_used);
int vpca_glm_linear_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                        double* out, int32_t* out_err);

/* ---- logistic association tests (beyond VariantsPca.scala: PLINK 2's --glm no-firth for case/control traits;
 * DESIGN.md 16) ---------------------------------------------------------------------------------------------------------
 * A case/control trait y in {0 (control), 1 (case)}, an additive model, per variant on the complete cases: with the
 * regression samples, C, q, g, A_v and OBS_CT as above, maximum likelihood over A_v of logit P(y = 1) = C gamma + beta g
 * gives BETA = beta, SE = sqrt([H^-1]_gg) with H = X^T W X at the fit, Z = BETA / SE, P = erfc(|Z| / sqrt(2)) (0 below the
 * double range) and A1_FREQ as in the linear test.  The fit runs in the orthonormal basis Q of C and the centred dosage
 * of the linear test, by Newton passes from (the null fit, beta = 0): each pass evaluates l, grad l and H over A_v;
 * a fall of l by more than 1e-10 |l| against the last accepted pass halves the step (at most 8 times in a row);
 * otherwise H = L L^T and the pass stops at a Newton decrement ||L^-1 grad l|| <= 1e-9, reporting beta + the step's
 * last entry and SE = 1 / L_gg; at most 25 passes.  ERRCODE, checked in this order:
 *   VPCA_GLM_TOO_FEW_OBS             OBS_CT - q - 1 < 1
 *   VPCA_GLM_CONST_ALLELE            g constant over A_v
 *   VPCA_GLM_LOGISTIC_CONVERGE_FAIL  A_v holds no case or no control (exact counts)
 *   VPCA_GLM_VIF_INFINITE            on the first pass a Cholesky pivot of H <= 1e-10 x that diagonal entry of H
 *   VPCA_GLM_LOGISTIC_CONVERGE_FAIL  no convergence in 25 passes or 8 halvings, a pivot <= 0 after the first pass, or a
 *                                    non-finite l or step (separation lands here)
 * A flagged variant has BETA, SE, Z and P NaN.
 * vpca_glm_logistic_begin: pheno is 0, 1 or NaN (missing) per sample, covar as vpca_glm_begin.  Refuses with
 *   VPCA_ERR_BAD_ARG, leaving no GLM state, everything vpca_glm_begin refuses, a phenotype outside {0, 1, NaN}, no case or
 *   no control among the regression samples, and a null fit (Q alone, all regression samples, on the host in FP64 by the
 *   rules above) that does not converge, as when a covariate separates cases from controls; the message names the
 *   problem.  The GLM state records its model: vpca_glm_linear_bed after this call, and vpca_glm_logistic_bed after
 *   vpca_glm_begin, return VPCA_ERR_STATE.
 * vpca_glm_logistic_bed: out[6 v ..] = OBS_CT, A1_FREQ, BETA, SE, Z, P, out_err[v] = ERRCODE and out_passes[v] (may be
 *   NULL) = the Newton passes run (0 for a variant flagged before the first), with the row, chunk and argument rules of
 *   vpca_glm_linear_bed.  Every output of a variant depends on its row's codes, Q, y, the null fit and n_samples only. */
int vpca_glm_logistic_begin(vpca_ctx* ctx, const double* pheno, const double* covar, int32_t n_covar, int64_t* n_used);
int vpca_glm_logistic_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                          double* out, int32_t* out_err, int32_t* out_passes);

/* ---- Firth-penalized logistic tests (beyond VariantsPca.scala: PLINK 2's --glm firth-fallback / firth; DESIGN.md 17) --
 * The model, samples, basis and start of the logistic tests above, maximising the penalized log-likelihood
 * l*(theta) = l(theta) + log det(H(theta)) / 2 (H = X^T W X) instead of l.  It has a finite maximum where l has none, as
 * when every carrier of a rare allele is a case.  Each pass evaluates l and H at a trial point, H = L L^T, and
 * l* = l + sum log L_jj, then the Firth score U* = sum_i x_i (y_i - mu_i + h_i (1/2 - mu_i)), h_i = w_i ||L^-1 x_i||^2.
 * A trial point theta_prev + t Delta is backtracked (t halved) when l is not finite, a pivot of H is <= 0 or l* fell by
 * more than 1e-10 |l*_prev|, and by the secant t <- t s0 / (s0 - s1) when s1 = U*^T Delta < -0.45 s0, s0 = delta^2 at
 * theta_prev; at most 30 backtracks in a row.  An accepted point takes z = L^-1 U*, delta^2 = z^T z, Delta = L^-T z, and
 * stops at delta <= 1e-9, reporting BETA = beta + Delta_g and SE = 1 / L_gg (sqrt([H^-1]_gg) of the unpenalized
 * information), Z = BETA / SE and P = erfc(|Z| / sqrt(2)); else the next trial point is at t = min(1, 5 / delta).  At most
 * 100 passes, backtracked ones included.
 * vpca_glm_firth_bed: as vpca_glm_logistic_bed (the same state, rows, chunks, outputs and argument rules), in one of two
 *   modes:
 *   VPCA_GLM_FIRTH_FALLBACK  the maximum-likelihood fit of vpca_glm_logistic_bed (the same bits), and the Firth fit, from
 *                            the same start, of the variants it ends with VPCA_GLM_LOGISTIC_CONVERGE_FAIL after at least
 *                            one pass.  A variant without a case or a control among its called samples keeps that code.
 *   VPCA_GLM_FIRTH_ALWAYS    the Firth fit of every variant past the checks that come before the first pass.
 *   The Firth fit's ERRCODE is VPCA_GLM_VIF_INFINITE by the first-pass rule of the logistic test, or
 *   VPCA_GLM_FIRTH_CONVERGE_FAIL (100 passes, 30 backtracks in a row, or a non-finite l or step on the first pass or at
 *   an accepted point).  out_passes[v] (may be NULL) = the passes of the fit reported; out_firth[v] (may be NULL) = 1
 *   where the Firth fit ran.  A variant's Firth outputs depend on its row's codes, Q, y, the null fit and n_samples only,
 *   and are the same bits in both modes.  VPCA_ERR_STATE without vpca_glm_logistic_begin state (after vpca_glm_begin
 *   too); VPCA_ERR_BAD_ARG for a mode outside {1, 2}, besides the rules of vpca_glm_logistic_bed. */
enum { VPCA_GLM_FIRTH_FALLBACK = 1, VPCA_GLM_FIRTH_ALWAYS = 2 };
int vpca_glm_firth_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t counted_allele,
                       int32_t mode, double* out, int32_t* out_err, int32_t* out_passes, uint8_t* out_firth);

/* ---- sample quality control (beyond VariantsPca.scala: which samples go into S; DESIGN.md 11) -------------------------
 * --keep / --remove / --mind decide the samples of a run before its context exists: the per-sample missing-call counts
 * over every row of a fileset, then the rows repacked to the kept samples, which a plain run reads as its fileset.
 * n_samples is the rows' own sample count; the context supplies only its device, a lane and scratch buffers (its own
 * n_samples plays no part), so the driver can run these before it knows the size of the run's context.  Rows are PLINK 1
 * .bed rows (as vpca_accumulate_bed; bytes past ceil(n_samples / 4) and the padding bits of the last byte are ignored).
 * vpca_sample_missing_bed: out_missing[s] = the rows where sample s has code 01 (exact int32 sums, whatever the split of
 *   the rows into calls); all n_samples entries are overwritten, with zeros when nv = 0.
 * vpca_subset_bed_samples: out row v (at out_rows + v * out_stride) = the codes of samples keep_idx[0 .. m) of row v, in
 *   that order, packed as a .bed row of m samples: the padding bits of its last byte are 0, as PLINK writes them, so the
 *   bytes equal those of a fileset of the kept samples.  Bytes of an out row past ceil(m / 4) are not written.
 * Driver-side and synchronous.  Rows are staged in chunks of at most 64 MB in two buffers (shared with the other
 *   driver-side .bed calls), so device memory does not grow with nv or n_samples; the upload of chunk i + 1 overlaps the
 *   work on chunk i, and the subset pass also overlaps it with the download of chunk i.  The buffers are allocated on the
 *   first call and freed by vpca_destroy.  The PCA Gram, U, the kinship counts, the subset state, the LD state and the
 *   variant QC counts are left alone.
 * VPCA_ERR_BAD_ARG, before any row is staged and with the outputs untouched: a NULL rows / out_missing / keep_idx /
 *   out_rows when nv > 0, nv < 0, n_samples < 1, stride_bytes < ceil(n_samples / 4), m < 1, keep_idx not strictly
 *   increasing or outside [0, n_samples), out_stride < ceil(m / 4).  VPCA_ERR_OVERFLOW: nv > 2^31 - 1 for the counts. */
int vpca_sample_missing_bed(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t n_samples,
                            int32_t* out_missing /* n_samples entries, overwritten */);
int vpca_subset_bed_samples(vpca_ctx* ctx, const uint8_t* rows, int64_t nv, int64_t stride_bytes, int32_t n_samples,
                            const int32_t* keep_idx, int32_t m, uint8_t* out_rows, int64_t out_stride);

/* ---- one process, all GPUs of the box (SURVEY 8b "process model") --------------------------------------------------
 * A vpca_pool is what `class VariantsPcaDriver` holds on a multi-GPU host: one vpca_ctx per GPU, wired with
 * vpca_gram_set_peers_local in VPCA_PEER_OWNER_ROWS mode (VPCA_PEER_REPLICATE when n_samples < 64 x n_gpus).  Spark
 * partition p is served by GPU p % n_gpus (`mapPartitionsWithIndex`, VariantsPca.scala:184); all entry points below
 * except create / destroy / reset / reduce / get / compute may be called concurrently from the task threads.
 *   vpca_pool_create(cfg, n_gpus, devices, &pool)      cfg.device / stream / d_gram / gram_band_* are ignored
 *   task p:  vpca_pool_accumulate_* (pool, p, ...) ...  vpca_pool_commit(pool, p)   |  vpca_pool_abort(pool, p)
 *   driver:  vpca_pool_reduce_and_finalize(pool)        `reduceByKey(_ + _)` (:190): every commit has already been
 *                                                       added into the owners of its Gram rows over NVLink; this is the
 *                                                       closing barrier + all-gather of the bands + symmetrize
 *            vpca_pool_get_gram / vpca_pool_compute_pca  (:189-190, :198-227), served by GPU 0 of the pool */
typedef struct vpca_pool vpca_pool;
int vpca_pool_create(const vpca_config* cfg, int32_t n_gpus, const int32_t* devices /* NULL: 0 .. n_gpus-1 */,
                     vpca_pool** out);
int vpca_pool_destroy(vpca_pool* pool);
int32_t vpca_pool_size(const vpca_pool* pool);
/* The context that serves partition_id (partition_id < 0: GPU 0). */
vpca_ctx* vpca_pool_ctx(vpca_pool* pool, int64_t partition_id);
const char* vpca_pool_last_error(const vpca_pool* pool);
int vpca_pool_reset(vpca_pool* pool);
int vpca_pool_accumulate_calls(vpca_pool* pool, int64_t partition_id, const int64_t* offsets, const int32_t* sample_idx,
                               int64_t nv);
int vpca_pool_accumulate_calls_u16(vpca_pool* pool, int64_t partition_id, const int64_t* offsets,
                                   const uint16_t* sample_idx, int64_t nv);
int vpca_pool_accumulate_bits(vpca_pool* pool, int64_t partition_id, const uint8_t* bits, int64_t nv, int64_t stride_bytes);
int vpca_pool_accumulate_bed(vpca_pool* pool, int64_t partition_id, const uint8_t* rows, int64_t nv, int64_t stride_bytes,
                             int32_t counted_allele);
int vpca_pool_commit(vpca_pool* pool, int64_t partition_id);
int vpca_pool_abort(vpca_pool* pool, int64_t partition_id);
int vpca_pool_reduce_and_finalize(vpca_pool* pool);
int vpca_pool_get_gram(vpca_pool* pool, int32_t* out);
int vpca_pool_compute_pca(vpca_pool* pool, int32_t k, double* vecs, double* evals, int32_t* non_zero_rows);
/* Sum of the per-GPU statistics (times: the maximum). */
struct vpca_stats;
int vpca_pool_get_stats(vpca_pool* pool, struct vpca_stats* out);

/* ---- synthetic cohort (stands in for the retired Genomics API ingestion, rdd/VariantsRDD.scala:187-236;
 *      specification in DESIGN.md "Synthetic generator") --------------------------------------------------
 * Fill a dense sample-major device tile d_x[s * ld + (v - v0)] for variants [v0, v0+nv).
 * mode 0: binary carrier x = (dosage > 0) (reference encode rule); mode 1: dosage 0/1/2. */
int vpca_synth_dense_device(vpca_ctx* ctx, uint64_t seed, int64_t v0, int64_t nv, int mode, void* d_x, int64_t ld);

/* Same generator, writing the panel layout of vpca_accumulate_panels (buffer: ceil(nv / P) * n_samples * P cells). */
int vpca_synth_panels_device(vpca_ctx* ctx, uint64_t seed, int64_t v0, int64_t nv, int mode, void* d_x,
                             int64_t panel_variants);

/* ---- introspection ---------------------------------------------------------------------------------- */
typedef struct vpca_stats {
    int64_t variants_accumulated; /* rows folded into the Gram or into staged partitions                  */
    int64_t gram_launches;        /* Gram kernel launches                                                 */
    int64_t kernel_launches;      /* all kernels launched by this ctx                                     */
    int64_t h2d_bytes;            /* bytes copied host -> device by accumulate_* / encode / set_gram      */
    int64_t d2h_bytes;            /* bytes copied device -> host by get_* / compute_pca                   */
    float last_gram_ms;           /* device time of the most recent Gram launch (CUDA events)             */
    float last_eig_ms;            /* device time of the most recent centering + eigensolve                */
    int32_t gram_cta_group;       /* 1 or 2: CTAs per Gram tile                                           */
    int32_t gram_resident;        /* 1 when the last launch kept accumulators in registers for the whole K loop */
    int32_t eig_method;           /* last vpca_compute_pca: 1 direct reduction, 2 Lanczos, 3 Lanczos abandoned -> direct;
                                     4 Lanczos on row bands (vpca_compute_pca_bands, reported by ctxs[0])    */
    int32_t eig_iterations;       /* Lanczos steps taken by the last solve (0 for a direct solve)             */
} vpca_stats;
int vpca_get_stats(vpca_ctx* ctx, vpca_stats* out);
/* Diagnostic (set VPCA_GRAM_PROF=1 before the first Gram launch): per-CTA timestamps of the last Gram launch,
 * 4 x int64 nanoseconds per CTA {start, -, last MMA issued, end}; returns the number of CTAs written (<= max_ctas)
 * or a negative vpca_status.  Synchronises the stream. */
int vpca_debug_gram_profile(vpca_ctx* ctx, int64_t* out, int32_t max_ctas);
/* Diagnostic (set VPCA_LZ_PROF=1 before the first vpca_compute_pca): block 0's timestamps of the persistent Lanczos kernel,
 * 8 x int64 nanoseconds per step {step start, start vector staged + norms, mat-vec done, y and the new basis column written,
 * shares of V^T y and V^T v_j written, first grid barrier passed, fused Gram-Schmidt pass done, next start vector written
 * (second grid barrier next)}
 * for steps 0..31 (each slot holds the last launch that ran that step index); returns the number of steps written or a
 * negative vpca_status. */
int vpca_debug_lanczos_profile(vpca_ctx* ctx, int64_t* out, int32_t max_steps);
/* Host-only diagnostic: the bytes of device memory every context of the process holds right now (their Grams, staging
 * and solver workspaces; not caller-owned Grams or pinned host memory).  vpca_destroy brings it back to what it was
 * before the context was created. */
int64_t vpca_debug_device_bytes(void);

/* ---- Multi-dataset keying on the device (SURVEY 8 f-3) ------------------------------------------------------------
 * The 2-dataset and N-dataset branches of VariantsPcaDriver.getCallsRdd (VariantsPca.scala:153-168) key every variant by
 * getVariantKey (:62-78: Guava Hashing.murmur3_128() over contig, start, end, reference bases, alternate bases) and then
 * join (:115-128) or merge (:136-148) the datasets on that key.  Here the rows of ALL datasets are handed over as one CSR
 * (rows of dataset 0 first) next to the key bytes of every row; hashing, the hash join / group-by and the concatenation
 * of the calls run on the GPU, and the joined rows can be accumulated without leaving it.
 *
 * vpca_hash_keys: MurmurHash3_x64_128 (seed 0) of nkeys byte strings, key q = payload[key_offsets[q], key_offsets[q+1]);
 *   out[2q], out[2q+1] = the two little-endian 64-bit halves of Guava's HashCode.asBytes() (HashCode.toString is their
 *   bytes in hex).  Host buffers in and out.
 * vpca_join_rows: mode VPCA_JOIN -- rows [0, n_left) are the left dataset, rows [n_left, nrows) the right one; one
 *   output row per (left, right) pair with equal keys, left calls then right calls (`related._1 ++ related._2`, :127),
 *   ordered by left row, then right row.  mode VPCA_MERGE -- n_left is ignored; keys that occur exactly
 *   variant_set_count times (:144) yield one row: the calls of the group's rows in input order (:145), rows ordered by
 *   the group's first input row.  sample_idx holds the calls that survive `_.hasVariation` (:164), already mapped to
 *   [0, n_samples).  The result stays on the device inside the context until the next vpca_join_rows / vpca_reset;
 *   *out_rows / *out_nnz report its size.  Driver-side step (the reference's join is a shuffle stage that precedes the
 *   mapPartitions tasks): one join at a time per context.  Every argument check runs on the host before anything is
 *   copied: a call refused with VPCA_ERR_BAD_ARG keeps the previous result, a call that fails later drops it.
 * vpca_join_fetch: copies the retained result to the host (out_offsets: out_rows + 1, out_idx: out_nnz entries).
 * vpca_accumulate_joined: encodes the retained rows and accumulates them into the staging Gram of partition_id, exactly
 *   like vpca_accumulate_calls would for the same rows (commit / abort as usual); no host round trip of the joined rows. */
#define VPCA_JOIN 0
#define VPCA_MERGE 1
int vpca_hash_keys(vpca_ctx* ctx, const uint8_t* payload, const int64_t* key_offsets, int64_t nkeys, uint64_t* out);
int vpca_join_rows(vpca_ctx* ctx, int32_t mode, int32_t variant_set_count, int64_t n_left, const uint8_t* key_payload,
                   const int64_t* key_offsets, const int64_t* offsets, const int32_t* sample_idx, int64_t nrows,
                   int64_t* out_rows, int64_t* out_nnz);
int vpca_join_fetch(vpca_ctx* ctx, int64_t* out_offsets, int32_t* out_idx);
/* rows / calls of the retained result (what vpca_join_fetch will write); VPCA_ERR_STATE when there is none */
int vpca_join_size(vpca_ctx* ctx, int64_t* out_rows, int64_t* out_nnz);
int vpca_accumulate_joined(vpca_ctx* ctx, int64_t partition_id);

/* Host-only introspection of the Gram schedule (works without a GPU; what tests/test_schedule.py checks).
 * vpca_debug_tiles: the output tiles the kernel enumerates for n_samples -- 8 int32 per tile {rowA of CTA 0, rowA of CTA 1,
 *   rowB, n_eff (MMA N), weight prefix, flags (1: a 128-block above the diagonal is written transposed, 2: CTA 1 is a
 *   filler), 0, 0}; exact != 0: the exact 128-block cover of the lower triangle (every block of
 *   `for (c1 <- callset; c2 <- callset)`, VariantsPca.scala:186-188, with c2 <= c1 computed exactly once), 0: the 256 x (<= 256)
 *   rectangles of the default tiling.  Returns the tile count (may exceed max_tiles).
 * vpca_debug_plan: the (worker, tile, first k-block, end k-block, accumulator column, accumulator columns of the worker) pieces of one
 *   window of kb_window k-blocks under an equal split -- 6 int32 per piece; returns the piece count, or -(1 + worker) when
 *   a worker would own more pieces than the kernel supports.
 * vpca_debug_rebalance: what the on-device rebalancer does with a candidate speed-weighted split before it publishes it --
 *   `cum` (workers + 1 fractions of a window, cum[0] = 0, cum[workers] = 1; in / out) is repaired so that the accumulators
 *   of every worker fit `col_limit` accumulator columns (256: one tile), then the pieces are written like
 *   vpca_debug_plan.  Returns the piece count, or VPCA_ERR_STATE when no repair exists (the device keeps the old split). */
int vpca_debug_rebalance(const int32_t* tiles, int32_t num_tiles, int32_t workers, int32_t kb_window, int32_t col_limit,
                         double* cum, int32_t* out, int32_t max_pieces);
int vpca_debug_tiles(int32_t n_samples, int32_t cta_group, int32_t exact, int32_t* out, int32_t max_tiles);
/* Host-only: the tiles (int8 / bf16 rectangles, same 8-int records as vpca_debug_tiles) an owner-computes context that
 * stores rows [row0, row0 + rows) of the Gram enumerates -- only products whose rows of S lie in the band. */
int vpca_debug_band_tiles(int32_t n_samples, int32_t cta_group, int32_t row0, int32_t rows, int32_t* out, int32_t max_tiles);
/* Diagnostic: how many clusters of cluster_size CTAs of the Gram kernel (one CTA per SM) `device` can hold at once
 * (cudaOccupancyMaxActiveClusters); negative vpca_status on error. */
int vpca_debug_max_clusters(int32_t device, int32_t cluster_size);
int vpca_debug_plan(const int32_t* tiles, int32_t num_tiles, int32_t workers, int32_t kb_window, int32_t* out, int32_t max_pieces);
/* Host-only: every (tile, k-range) piece each of `workers` workers replays in one launch of kb_total k-blocks, in launch
 * order, under the schedule the Gram kernel takes for a whole-cohort context of n_samples (tiles as vpca_debug_tiles)
 * with windows of kb_window k-blocks and the initial split -- 6 int32 per piece {worker, tile, first k-block, end k-block,
 * first (the accumulator starts from zero), flush (the accumulator is added into S after it)}.  front_frac >= 0 sets the
 * split point s = floor(front_frac * kb_total) of the front/tail schedule (taken when workers / 2 < tiles < workers:
 * worker t < tiles owns tile t for k-blocks [0, s), the others split the tiles x [s, kb_total)); < 0: its initial
 * tiles / workers.  info (2 int32): {schedule: 0 whole-tile waves, 1 resident, 2 front/tail; s, or kb_total for the
 * others}.  Returns the piece count (may exceed max_pieces), or VPCA_ERR_STATE when a worker's accumulators would not fit. */
int vpca_debug_schedule(int32_t n_samples, int32_t cta_group, int32_t exact, int32_t workers, int32_t kb_window,
                        int32_t kb_total, double front_frac, int32_t* out, int32_t max_pieces, int32_t* info);

#ifdef __cplusplus
}
#endif
#endif /* VPCA_H_ */
