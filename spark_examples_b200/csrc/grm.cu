// Variance-standardized genomic relationship matrix (DESIGN.md 13): per-variant z tables from the exact genotype counts,
// the used variants compacted into FP64 panels of kGrmPanelK columns, and the panels multiplied into the running sum
// C += Z Z^T by an FP64 tensor-core SYRK (DMMA m16n8k16) over the lower-triangle tiles.
//
// Table.  For a used variant (0 < a < 2n, a = 2 HOM_A1 + HET the A1 copies over the n called samples), r = min(a, 2n - a)
// counts the less common allele (A1 at a tie), and
//   mu = r / n   q = r / (2n)   s = 1 / sqrt(mu (1 - q))   z_d = (d - mu) s  (d: that allele's count; missing calls 0)
// every operation an explicitly rounded intrinsic, so a host restatement with the same operations gives the same bits.
//
// SYRK.  One CTA per 64 x 64 tile of the lower triangle (diagonal tiles whole), four warps of 32 x 32, the tile's
// accumulators in registers over the panel's whole K, z tiles double-buffered in shared memory with cp.async.  The tile
// is added into C with one read-add-write per cell: no atomics and no split-K, so every cell is the same sequence of
// roundings whatever the launch geometry.
#include <cuda_runtime.h>

#include <cstdint>

#include "vpca_internal.h"

namespace vpca {
namespace {

constexpr int kTile = 64;               // samples per tile edge
constexpr int kStageK = 32;             // variants per shared-memory stage
constexpr int kPitch = kStageK + 4;     // doubles per staged row: rows 4 apart hit disjoint banks (fragment loads)
constexpr int kSyrkThreads = 128;
constexpr int kStageDoubles = kTile * kPitch;

__global__ void grm_table_kernel(const int32_t* __restrict__ counts, int nv, double* __restrict__ tab,
                                 int32_t* __restrict__ used) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const int4 c = reinterpret_cast<const int4*>(counts)[v];
    const int64_t n = (int64_t)c.x + c.y + c.z, a = 2 * (int64_t)c.x + c.y;
    double4 t = make_double4(0.0, 0.0, 0.0, 0.0);   // indexed by the .bed code: 00 HOM_A1, 01 missing, 10 HET, 11 HOM_A2
    const bool u = a > 0 && a < 2 * n;
    if (u) {
        const bool a1 = a <= 2 * n - a;   // count A1 when it is the less common allele or at a tie
        const int64_t r = a1 ? a : 2 * n - a;
        const double dn = (double)n, dr = (double)r;
        const double mu = __ddiv_rn(dr, dn);
        const double q = __ddiv_rn(dr, 2.0 * dn);
        const double s = __ddiv_rn(1.0, __dsqrt_rn(__dmul_rn(mu, __dsub_rn(1.0, q))));
        t.x = __dmul_rn(__dsub_rn(a1 ? 2.0 : 0.0, mu), s);
        t.z = __dmul_rn(__dsub_rn(1.0, mu), s);
        t.w = __dmul_rn(__dsub_rn(a1 ? 0.0 : 2.0, mu), s);
    }
    reinterpret_cast<double4*>(tab)[v] = t;
    used[v] = u ? 1 : 0;
}

// One block: inv[0 .. total) = the used variants of the chunk in row order, *total their number.
constexpr int kCompactThreads = 1024;
__global__ void __launch_bounds__(kCompactThreads) grm_compact_kernel(const int32_t* __restrict__ used, int nv,
                                                                      int32_t* __restrict__ inv, int* __restrict__ total) {
    __shared__ int part[kCompactThreads];
    const int tid = threadIdx.x;
    const int per = (nv + kCompactThreads - 1) / kCompactThreads;
    const int lo = min(nv, tid * per), hi = min(nv, lo + per);
    int c = 0;
    for (int v = lo; v < hi; ++v) c += used[v];
    part[tid] = c;
    __syncthreads();
    for (int off = 1; off < kCompactThreads; off <<= 1) {   // inclusive scan (Hillis-Steele)
        const int x = tid >= off ? part[tid - off] : 0;
        __syncthreads();
        part[tid] += x;
        __syncthreads();
    }
    int pos = part[tid] - c;
    for (int v = lo; v < hi; ++v)
        if (used[v]) inv[pos++] = v;
    if (tid == kCompactThreads - 1) *total = part[tid];
}

// Z[s][col0 + j] = tab[inv[j]][code of sample s in row inv[j]] for j < cnt, s < n.  Threads of a warp take consecutive
// columns, so the stores of a warp are one contiguous run of a Z row.
__global__ void grm_expand_kernel(const uint8_t* __restrict__ rows, int64_t stride, const int32_t* __restrict__ inv,
                                  const double* __restrict__ tab, int cnt, int n, double* __restrict__ Z, int ldz,
                                  int col0) {
    const int j = blockIdx.x * 32 + (threadIdx.x & 31);
    const int s = blockIdx.y * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (j >= cnt || s >= n) return;
    const int v = inv[j];
    const int code = (rows[(int64_t)v * stride + (s >> 2)] >> (2 * (s & 3))) & 3;
    Z[(int64_t)s * ldz + col0 + j] = tab[4 * (int64_t)v + code];
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// D += A B with A 16 x 16 (row), B 16 x 8 (col), FP64.  Lane l = 4 g + t holds A[g (+8)][t + 4i], B[t + 4i][g],
// D[g (+8)][2t (+1)].
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
        "{%12, %13, %14, %15}, {%0, %1, %2, %3};\n"
        : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
        : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
          "d"(b[2]), "d"(b[3]));
}

// 64 rows x kStageK doubles of Z (rows row0 .., columns k0 ..) into a padded stage; 16-byte copies, 8 per thread.
__device__ __forceinline__ void load_stage(double* __restrict__ st, const double* __restrict__ Z, int ldz, int row0, int k0) {
#pragma unroll
    for (int i = 0; i < kTile * kStageK / 2 / kSyrkThreads; ++i) {
        const int c = threadIdx.x + i * kSyrkThreads;
        const int r = c / (kStageK / 2), q = c % (kStageK / 2);
        cp_async16(st + r * kPitch + 2 * q, Z + (int64_t)(row0 + r) * ldz + k0 + 2 * q);
    }
}

// grid: one CTA per lower-triangle tile (ti >= tj), blockIdx.x = ti (ti + 1) / 2 + tj.  Z: npad rows of ldz doubles, zero
// on rows >= n and on columns >= the panel's fill.  C: n x n row-major; cells of the tile inside n get C += (Z Z^T).
__global__ void __launch_bounds__(kSyrkThreads) grm_syrk_kernel(const double* __restrict__ Z, int ldz, int kdim, int n,
                                                                double* __restrict__ C) {
    extern __shared__ __align__(16) double smem[];   // [stage][A | B]
    const int t = blockIdx.x;
    int ti = (int)((sqrt(8.0 * t + 1.0) - 1.0) * 0.5);
    while ((ti + 1) * (ti + 2) / 2 <= t) ++ti;
    while (ti * (ti + 1) / 2 > t) --ti;
    const int tj = t - ti * (ti + 1) / 2;
    const bool diag = ti == tj;
    const int rowA = ti * kTile, rowB = tj * kTile;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;   // the warp's 32 x 32 block of the tile
    const int g = lane >> 2, tg = lane & 3;
    double acc[2][4][4];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.0;

    const int nk = kdim / kStageK;
    auto issue = [&](int ks) {
        double* st = smem + (ks & 1) * 2 * kStageDoubles;
        load_stage(st, Z, ldz, rowA, ks * kStageK);
        if (!diag) load_stage(st + kStageDoubles, Z, ldz, rowB, ks * kStageK);
        cp_async_commit();
    };
    issue(0);
#pragma unroll 1
    for (int ks = 0; ks < nk; ++ks) {
        if (ks + 1 < nk) {
            issue(ks + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const double* sa = smem + (ks & 1) * 2 * kStageDoubles;
        const double* sb = diag ? sa : sa + kStageDoubles;
#pragma unroll
        for (int kk = 0; kk < kStageK; kk += 16) {
            double a[2][8], b[4][4];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    a[i][2 * q] = sa[(wm + 16 * i + g) * kPitch + kk + tg + 4 * q];
                    a[i][2 * q + 1] = sa[(wm + 16 * i + g + 8) * kPitch + kk + tg + 4 * q];
                }
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int q = 0; q < 4; ++q) b[j][q] = sb[(wn + 8 * j + g) * kPitch + kk + tg + 4 * q];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) dmma16816(acc[i][j], a[i], b[j]);
        }
        __syncthreads();   // the stage is refilled by the next iteration's issue
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int r = rowA + wm + 16 * i + g + (e >> 1) * 8;
                const int c = rowB + wn + 8 * j + 2 * tg + (e & 1);
                if (r < n && c < n) {
                    double* p = C + (int64_t)r * n + c;
                    *p = __dadd_rn(*p, acc[i][j][e]);
                }
            }
}

// C[i][j] = C[j][i] = C[i][j] / m for j <= i: the lower triangle divided once, then mirrored.
__global__ void grm_finish_kernel(double* __restrict__ C, int n, double m) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j > i) return;
    const double x = __ddiv_rn(C[(int64_t)i * n + j], m);
    C[(int64_t)i * n + j] = x;
    C[(int64_t)j * n + i] = x;
}

}  // namespace

int64_t grm_panel_rows(int n) { return ((int64_t)n + kTile - 1) / kTile * kTile; }

cudaError_t grm_tables(const int32_t* d_counts, int nv, double* d_tab, int32_t* d_used, int32_t* d_inv, int* d_total,
                       cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    grm_table_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(d_counts, nv, d_tab, d_used);
    grm_compact_kernel<<<1, kCompactThreads, 0, stream>>>(d_used, nv, d_inv, d_total);
    return cudaGetLastError();
}

cudaError_t grm_table(const int32_t* d_counts, int nv, double* d_tab, int32_t* d_used, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    grm_table_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(d_counts, nv, d_tab, d_used);
    return cudaGetLastError();
}

cudaError_t grm_expand(const uint8_t* d_rows, int64_t stride, const int32_t* d_inv, const double* d_tab, int cnt, int n,
                       double* d_Z, int col0, cudaStream_t stream) {
    if (cnt <= 0) return cudaSuccess;
    const dim3 grid((unsigned)((cnt + 31) / 32), (unsigned)((n + 7) / 8));
    grm_expand_kernel<<<grid, 256, 0, stream>>>(d_rows, stride, d_inv, d_tab, cnt, n, d_Z, kGrmPanelK, col0);
    return cudaGetLastError();
}

cudaError_t grm_syrk(const double* d_Z, int n, double* d_C, cudaStream_t stream) {
    static_assert(kGrmPanelK % kStageK == 0, "a panel is whole stages");
    const int nt = (int)(grm_panel_rows(n) / kTile);
    const size_t smem = 4 * (size_t)kStageDoubles * sizeof(double);
    cudaError_t e = cudaFuncSetAttribute(grm_syrk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    grm_syrk_kernel<<<(unsigned)((int64_t)nt * (nt + 1) / 2), kSyrkThreads, smem, stream>>>(d_Z, kGrmPanelK, kGrmPanelK,
                                                                                            n, d_C);
    return cudaGetLastError();
}

cudaError_t grm_finish(double* d_C, int n, int64_t m, cudaStream_t stream) {
    grm_finish_kernel<<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, stream>>>(d_C, n, (double)m);
    return cudaGetLastError();
}

}  // namespace vpca
