/*
 * vpca_oracle.c -- CPU restatement of the VariantsPca hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * This file is the parity oracle for the CUDA path.  It is NOT product code: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 *
 * PINNING: the reference (googlegenomics/spark-examples) ships no tests, fixtures or golden vectors
 * for this path and its Scala driver cannot be executed here (no JVM/Spark in the image).  What
 * pins this restatement: (a) for encode, similarity and centering, vectors produced by the
 * reference's OWN Python twin of these steps (src/main/python/variants_pca.py:19-121, executed
 * by tests/golden/make_reference_twin_golden.py; tests/test_reference_twin.py holds this file to
 * them bit for bit); (b) a line-by-line reading of the Scala below; (c) a second, independent
 * numpy restatement (oracle/oracle.py); (d) hand-computed cases in tests/.  The eigen step has no
 * reference-produced vector (it needs the JVM): PARITY UNPINNED for that step.
 *
 * Every function cites the reference lines it follows; paths are relative to
 * /root/reference/src/main/scala/com/google/cloud/genomics/spark/examples/ .
 *
 * Build: see oracle/Makefile  (gcc -O2 -fopenmp -ffp-contract=off -shared -fPIC).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* ------------------------------------------------------------------------------------------
 * a-1 / a-2  encode:  VariantsPca.scala:56-60 (extractCallInfo) and :153-168 (getCallsRdd).
 *
 * Columnar form of RDD[Variant]: variant v owns calls [call_off[v], call_off[v+1]); call c has
 * callset index callset[c] (the value of mapping(call.callsetId), VariantsPca.scala:59) and
 * alleles genotype[gt_off[c] .. gt_off[c+1])  (Call.genotype, rdd/VariantsRDD.scala:46-48).
 *
 *   hasVariation = genotype.foldLeft(false)(_ || _ > 0)          (:58)   -- no-call (-1) is NOT variation
 *   calls.filter(_.hasVariation)                                  (:164)
 *   .filter(_.size > 0)                                           (:166)  -- drop variants with no carrier
 *   .map(_.map(_.callsetId))                                      (:167)  -- order of calls preserved,
 *                                                                            duplicates preserved
 * Output: CSR (out_off[nv_out+1], out_idx[]).  Returns nv_out, or -1 if a callset index is
 * outside [0, n_samples) (the reference would throw: NoSuchElementException at :59 for an
 * unknown id, IndexOutOfBounds from Breeze at :188 for a bad index).
 * ------------------------------------------------------------------------------------------ */
int64_t vo_encode_calls(int32_t n_samples, int64_t nv,
                        const int64_t *call_off, const int32_t *callset,
                        const int64_t *gt_off, const int32_t *genotype,
                        int64_t *out_off, int32_t *out_idx)
{
    int64_t nv_out = 0, nnz = 0;
    out_off[0] = 0;
    for (int64_t v = 0; v < nv; ++v) {
        int64_t start = nnz;
        for (int64_t c = call_off[v]; c < call_off[v + 1]; ++c) {
            int has_variation = 0;                         /* foldLeft(false) */
            for (int64_t g = gt_off[c]; g < gt_off[c + 1]; ++g)
                has_variation = has_variation || (genotype[g] > 0);
            if (callset[c] < 0 || callset[c] >= n_samples) return -1;
            if (has_variation) out_idx[nnz++] = callset[c];
        }
        if (nnz > start) out_off[++nv_out] = nnz;          /* .filter(_.size > 0) */
    }
    return nv_out;
}

/* ------------------------------------------------------------------------------------------
 * a-3  getSimilarityMatrix:  VariantsPca.scala:182-191.
 *
 *   callsets.mapPartitions(callsInPartition => {
 *     val matrix = DenseMatrix.zeros[Int](size, size)                      (:185)
 *     callsInPartition.foreach(callset =>
 *       for (c1 <- callset; c2 <- callset) matrix(c1, c2) += 1)            (:186-188)
 *     matrix.iterator }).reduceByKey(_ + _)                                (:189-190)
 *
 * One "partition" per thread (contiguous variant ranges), a private dense int32 N x N each,
 * scalar += 1 over the full cartesian square, then the partition matrices are summed.
 * S is row-major N x N int32, all N^2 entries present.  Returns 0, -1 on bad index.
 * ------------------------------------------------------------------------------------------ */
int vo_similarity(int32_t n, int64_t nv, const int64_t *off, const int32_t *idx,
                  int32_t n_partitions, int32_t *S)
{
    if (n_partitions < 1) n_partitions = 1;
    const size_t nn = (size_t)n * (size_t)n;
    for (int64_t e = 0; e < off[nv]; ++e)
        if (idx[e] < 0 || idx[e] >= n) return -1;
    memset(S, 0, nn * sizeof(int32_t));
    int32_t **part = (int32_t **)calloc((size_t)n_partitions, sizeof(int32_t *));
#pragma omp parallel for schedule(static, 1) num_threads(n_partitions)
    for (int p = 0; p < n_partitions; ++p) {
        int32_t *M = (int32_t *)calloc(nn, sizeof(int32_t));          /* DenseMatrix.zeros :185 */
        part[p] = M;
        int64_t v0 = nv * p / n_partitions, v1 = nv * (p + 1) / n_partitions;
        for (int64_t v = v0; v < v1; ++v) {
            const int32_t *cs = idx + off[v];
            const int64_t c = off[v + 1] - off[v];
            for (int64_t a = 0; a < c; ++a) {                          /* c1 <- callset */
                int32_t *row = M + (size_t)cs[a] * n;
                for (int64_t b = 0; b < c; ++b) row[cs[b]] += 1;       /* c2 <- callset */
            }
        }
    }
    /* reduceByKey(_ + _) :190 */
#pragma omp parallel for schedule(static) num_threads(n_partitions)
    for (int64_t i = 0; i < (int64_t)nn; ++i) {
        int32_t acc = 0;
        for (int p = 0; p < n_partitions; ++p) acc += part[p][i];
        S[i] = acc;
    }
    for (int p = 0; p < n_partitions; ++p) free(part[p]);
    free(part);
    return 0;
}

/* a-3'  getSimilarityMatrixStream: VariantsPca.scala:262-279 -- pairs with c1 <= c2, summed,
 * mirrored.  Same S wherever it is non-zero; implemented densely (zero rows present) because
 * SURVEY.md 2 row 3 says not to replicate the sparse-row bug. */
int vo_similarity_stream(int32_t n, int64_t nv, const int64_t *off, const int32_t *idx, int32_t *S)
{
    const size_t nn = (size_t)n * (size_t)n;
    memset(S, 0, nn * sizeof(int32_t));
    for (int64_t v = 0; v < nv; ++v) {
        const int32_t *cs = idx + off[v];
        const int64_t c = off[v + 1] - off[v];
        for (int64_t a = 0; a < c; ++a)
            for (int64_t b = 0; b < c; ++b) {
                if (cs[a] < 0 || cs[a] >= n || cs[b] < 0 || cs[b] >= n) return -1;
                if (cs[a] <= cs[b]) S[(size_t)cs[a] * n + cs[b]] += 1;         /* :267 */
            }
    }
    for (int32_t i = 0; i < n; ++i)                                             /* :272-278 */
        for (int32_t j = i + 1; j < n; ++j) S[(size_t)j * n + i] = S[(size_t)i * n + j];
    return 0;
}

/* ------------------------------------------------------------------------------------------
 * a-4  computePca part 1 (centering):  VariantsPca.scala:199-223.
 *
 *   rowSums(i)  = entries(i).foldLeft(0D)(_ + _._2)     (:206)  exact: integer-valued doubles
 *   matrixSum   = rowSums.reduce(_ + _)                  (:210)
 *   matrixMean  = matrixSum / rowCount / rowCount        (:211)  two successive divisions
 *   rowMean     = rowSums(i) / rowCount                  (:216)
 *   colMean     = rowSums(j) / rowCount                  (:220)
 *   C(i,j)      = data - rowMean - colMean + matrixMean  (:221)  evaluated left to right
 *
 * C is row-major N x N double.  *non_zero_rows receives rowSums.filter(_ > 0).size (:207).
 * ------------------------------------------------------------------------------------------ */
void vo_center(int32_t n, const int32_t *S, double *C, double *row_sums_out, int32_t *non_zero_rows)
{
    double *rs = (double *)malloc((size_t)n * sizeof(double));
    int32_t nz = 0;
    for (int32_t i = 0; i < n; ++i) {
        double acc = 0.0;
        for (int32_t j = 0; j < n; ++j) acc = acc + (double)S[(size_t)i * n + j];
        rs[i] = acc;
        if (acc > 0) ++nz;
    }
    double matrix_sum = rs[0];
    for (int32_t i = 1; i < n; ++i) matrix_sum = matrix_sum + rs[i];   /* reduce(_ + _) */
    const double row_count = (double)n;
    const double matrix_mean = matrix_sum / row_count / row_count;
    for (int32_t i = 0; i < n; ++i) {
        const double row_mean = rs[i] / row_count;
        for (int32_t j = 0; j < n; ++j) {
            const double col_mean = rs[j] / row_count;
            const double data = (double)S[(size_t)i * n + j];
            C[(size_t)i * n + j] = data - row_mean - col_mean + matrix_mean;
        }
    }
    if (row_sums_out) memcpy(row_sums_out, rs, (size_t)n * sizeof(double));
    if (non_zero_rows) *non_zero_rows = nz;
    free(rs);
}

/* ------------------------------------------------------------------------------------------
 * a-5 (first half)  spark-mllib 1.6.1 RowMatrix.computeCovariance, reached from
 * VariantsPca.scala:225-226 (un-vendored dependency, build.sbt:11,25; restated from the
 * published source, tag v1.6.1, mllib/.../linalg/distributed/RowMatrix.scala):
 *     m    = numRows,  mean = column means of the rows
 *     G    = sum_rows r r^T            (computeGramianMatrix, BLAS.spr on the packed upper half)
 *     Cov(i,j) = G(i,j)/(m-1) - (m/(m-1)) * mean(i)*mean(j)
 * The SVD of Cov (Breeze svd -> LAPACK dgesdd) is done in oracle.py with numpy, which calls the
 * same LAPACK driver.
 * ------------------------------------------------------------------------------------------ */
void vo_mllib_covariance(int32_t n, const double *C, double *Cov)
{
    const double m = (double)n;
    double *mean = (double *)calloc((size_t)n, sizeof(double));
    for (int32_t i = 0; i < n; ++i)
        for (int32_t j = 0; j < n; ++j) mean[j] += C[(size_t)i * n + j];
    for (int32_t j = 0; j < n; ++j) mean[j] /= m;
#pragma omp parallel for schedule(dynamic, 16)
    for (int32_t i = 0; i < n; ++i)
        for (int32_t j = i; j < n; ++j) {
            double g = 0.0;
            for (int32_t r = 0; r < n; ++r) g += C[(size_t)r * n + i] * C[(size_t)r * n + j];
            double c = g / (m - 1.0) - (m / (m - 1.0)) * mean[i] * mean[j];
            Cov[(size_t)i * n + j] = c;
            Cov[(size_t)j * n + i] = c;
        }
    free(mean);
}

/* ==========================================================================================
 * Synthetic genotype generator (SURVEY.md 8d).  Not part of the reference; it stands in for the
 * retired Genomics API ingestion (rdd/VariantsRDD.scala:187-236) and produces the record shape
 * the hot path consumes (RDD[Seq[Int]], VariantsPca.scala:153-168).  Counter-based so that any
 * (variant, sample) cell can be regenerated independently on CPU and GPU, bit for bit:
 *
 *   Philox4x32-10, key = (seed_lo, seed_hi)
 *   per variant v:  r[0..3] = philox(ctr = (v_lo, v_hi, 0, TAG_VARIANT)),
 *                   r[4..7] = philox(ctr = (v_lo, v_hi, 1, TAG_VARIANT))
 *       u       = (r[0] + 0.5) * 2^-32
 *       p_anc   = 0.02 + 0.48 * u                                  ancestral AF ~ U(0.02, 0.5)
 *       z_k     = (b0+b1+b2+b3 - 510) / 147.80054127               bytes of r[1+k]: Irwin-Hall(4),
 *                                                                   mean 0, variance 1
 *       p_k     = clip(p_anc + sqrt(F_k * p_anc * (1 - p_anc)) * z_k, 0.001, 0.999)
 *                 -- a moment-matched stand-in for the Balding-Nichols Beta draw (same mean p and
 *                    variance F p (1-p)) that needs no libm, so CPU and GPU agree exactly
 *       T_k     = floor(p_k * 2^32)
 *   K = 5 populations, F = (.15,.10,.07,.05,.03); sample s belongs to population k where
 *       bounds_k = (cum_pct_k * N) / 100 (integer division), cum_pct = (26,40,60,80,100)
 *   per cell (v, s): w[0..3] = philox(ctr = (v_lo, v_hi, s >> 1, TAG_CELL));
 *       alleles a1 = w[2*(s&1)] < T_pop(s), a2 = w[2*(s&1)+1] < T_pop(s); dosage g = a1 + a2
 *       binary carrier x = (g > 0)   (the reference's encode rule, VariantsPca.scala:58)
 * All floating point is IEEE double with no FMA contraction (-ffp-contract=off here).
 * ========================================================================================== */
#define VO_TAG_VARIANT 0xA11E1E00u
#define VO_TAG_CELL    0xC0FFEE00u
#define VO_NPOP 5

static inline void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                 uint32_t k0, uint32_t k1, uint32_t out[4])
{
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

void vo_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
    philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1], out);
}

void vo_pop_bounds(int32_t n, int32_t bounds[VO_NPOP])
{
    static const int cum[VO_NPOP] = {26, 40, 60, 80, 100};
    for (int k = 0; k < VO_NPOP; ++k) bounds[k] = (int32_t)(((int64_t)cum[k] * n) / 100);
}

void vo_variant_thresholds(uint64_t seed, int64_t v, uint32_t thr[VO_NPOP])
{
    static const double F[VO_NPOP] = {0.15, 0.10, 0.07, 0.05, 0.03};
    uint32_t r[8];
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    const uint32_t v0 = (uint32_t)(uint64_t)v, v1 = (uint32_t)((uint64_t)v >> 32);
    philox4x32_10(v0, v1, 0u, VO_TAG_VARIANT, k0, k1, r);
    philox4x32_10(v0, v1, 1u, VO_TAG_VARIANT, k0, k1, r + 4);
    const double u = ((double)r[0] + 0.5) * (1.0 / 4294967296.0);
    const double p = 0.02 + 0.48 * u;
    const double pq = p * (1.0 - p);
    for (int k = 0; k < VO_NPOP; ++k) {
        uint32_t w = r[1 + k];
        int sum4 = (int)(w & 255u) + (int)((w >> 8) & 255u) + (int)((w >> 16) & 255u) + (int)(w >> 24);
        double z = (double)(sum4 - 510) / 147.80054127;
        double pk = p + sqrt(F[k] * pq) * z;
        if (pk < 0.001) pk = 0.001;
        if (pk > 0.999) pk = 0.999;
        thr[k] = (uint32_t)(pk * 4294967296.0);
    }
}

/* dosage (0,1,2) of cell (v, s) */
static inline int cell_dosage(uint32_t k0, uint32_t k1, int64_t v, int32_t s, uint32_t T)
{
    uint32_t w[4];
    philox4x32_10((uint32_t)(uint64_t)v, (uint32_t)((uint64_t)v >> 32), (uint32_t)(s >> 1),
                  VO_TAG_CELL, k0, k1, w);
    const int h = (s & 1) * 2;
    return (int)(w[h] < T) + (int)(w[h + 1] < T);
}

/* Dense tile, sample-major: X[s * ld + (v - v0)] for s in [0,n), v in [v0, v0+nv).
 * mode 0: binary carrier (g > 0); mode 1: dosage g. */
void vo_synth_dense(uint64_t seed, int32_t n, int64_t v0, int64_t nv, int mode, int64_t ld, int8_t *X)
{
    int32_t bounds[VO_NPOP];
    vo_pop_bounds(n, bounds);
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < nv; ++j) {
        uint32_t thr[VO_NPOP];
        vo_variant_thresholds(seed, v0 + j, thr);
        int pop = 0;
        for (int32_t s = 0; s < n; ++s) {
            while (s >= bounds[pop]) ++pop;
            int g = cell_dosage(k0, k1, v0 + j, s, thr[pop]);
            X[(size_t)s * ld + j] = (int8_t)(mode ? g : (g > 0));
        }
    }
}

/* RDD[Seq[Int]] form (binary carriers, ascending sample order, variants with no carrier dropped,
 * VariantsPca.scala:164-167).  Two-pass: call with idx == NULL to size (returns nnz and fills
 * off[0..nv_out]); *nv_out receives the number of kept variants. */
int64_t vo_synth_calls(uint64_t seed, int32_t n, int64_t v0, int64_t nv, int64_t *off, int32_t *idx,
                       int64_t *nv_out)
{
    int32_t bounds[VO_NPOP];
    vo_pop_bounds(n, bounds);
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
    int64_t *cnt = (int64_t *)malloc((size_t)(nv > 0 ? nv : 1) * sizeof(int64_t));
#pragma omp parallel for schedule(static)
    for (int64_t j = 0; j < nv; ++j) {
        uint32_t thr[VO_NPOP];
        vo_variant_thresholds(seed, v0 + j, thr);
        int pop = 0;
        int64_t c = 0;
        for (int32_t s = 0; s < n; ++s) {
            while (s >= bounds[pop]) ++pop;
            c += cell_dosage(k0, k1, v0 + j, s, thr[pop]) > 0;
        }
        cnt[j] = c;
    }
    int64_t kept = 0, nnz = 0;
    off[0] = 0;
    for (int64_t j = 0; j < nv; ++j)
        if (cnt[j] > 0) { nnz += cnt[j]; off[++kept] = nnz; }
    *nv_out = kept;
    if (idx) {
        /* map kept slot -> source variant */
        int64_t *src = (int64_t *)malloc((size_t)(kept > 0 ? kept : 1) * sizeof(int64_t));
        int64_t q = 0;
        for (int64_t j = 0; j < nv; ++j) if (cnt[j] > 0) src[q++] = j;
#pragma omp parallel for schedule(static)
        for (int64_t q2 = 0; q2 < kept; ++q2) {
            uint32_t thr[VO_NPOP];
            const int64_t j = src[q2];
            vo_variant_thresholds(seed, v0 + j, thr);
            int pop = 0;
            int64_t w = off[q2];
            for (int32_t s = 0; s < n; ++s) {
                while (s >= bounds[pop]) ++pop;
                if (cell_dosage(k0, k1, v0 + j, s, thr[pop]) > 0) idx[w++] = s;
            }
        }
        free(src);
    }
    free(cnt);
    return nnz;
}

/* torchrun exports OMP_NUM_THREADS=1; the CPU arm of bench.py raises the thread count explicitly. */
void vo_set_threads(int n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int vo_num_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
