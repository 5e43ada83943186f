// Linear association tests (DESIGN.md 15): per .bed variant, the least-squares fit y = C gamma + beta g + e over the
// regression samples called at that variant, with the covariates C given to vpca_glm_begin as an orthonormal basis Q
// (n x q over the regression samples, zero elsewhere) and the residual phenotype y~ = y - Q Q^T y.
//
//   glm_count_kernel: one warp per variant, popcounts of the row under the regression mask: the exact integer sums
//     OBS_CT, sum g and sum g^2 of the counted allele's dosage g over the called regression samples A.
//   glm_sums_kernel: a thread owns VT variants and walks ALL samples in order 0 .. n-1 (grm_loadings_kernel's tiling: the
//     CTA's rows staged through shared memory in 32-byte tiles of 128 samples, Q and y~ in the same sample tiles).  Per
//     variant, one FMA chain per column: b_c = sum g' q_c (c < q) and b_q = sum g' y~ of the centred dosage g' = g - c
//     over A and 0 elsewhere, c in {0, 1, 2} the integer nearest the mean of g over A (glm_centre).
//   glm_solve_kernel: one warp (one CTA) per variant.  Over the fewer of the variant's missing and called regression
//     samples (in sample order, one FMA chain per entry) the packed lower triangle of [Q | y~]^T [Q | y~]; from it
//     P = Q_A^T Q_A, t = Q_A^T y~_A and y~_A^T y~_A over the called set A; Cholesky P = L L^T, u = L^-1 b, v = L^-1 t and
//     the Schur term s = sum g'^2 - u^T u, with the ERRCODEs that need no division.
//   glm_finish_kernel: one thread per variant: A1_FREQ, beta = (b_q - u^T v) / s,
//     RSS = y~_A^T y~_A - v^T v - (b_q - u^T v) beta, SE = sqrt(RSS / df / s), T_STAT = beta / SE and the two-sided
//     Student t p-value.
// Why g' and not g: q_0 is constant over the regression samples, so 1_A lies in the span of Q_A and replacing g by g - c
// over A changes neither s nor b_q - u^T v (nor beta, SE or the RSS) in exact arithmetic.  But with the raw dosage of an
// almost fixed allele, sum g^2 is about 4 OBS_CT while s is about the number of carriers of the other allele, and the
// rounding errors of the n-term chains in b, of size n u sum g^2, land on s whole.  With |mean(g')| <= 1/2 (and
// g'^2 >= |g'|), sum g'^2 <= 2 sum (g' - mean(g'))^2 = 2 VIF s: s cancels by at most a factor of 2 VIF.
// A variant's outputs depend on its row's codes, Q, y~, the mask and n only: not on the chunk split, the stride, the
// padding bits or bytes, or the call.  No floating-point atomics.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>
#include <type_traits>

#include "vpca_internal.h"

namespace vpca {
namespace {

// ---- integer sums --------------------------------------------------------------------------------------------------
// The centre of a variant's dosage: the integer in {0, 1, 2} nearest sum g / OBS_CT, a tie going to 1.  The tie rule
// makes the centre of 2 - g exactly 2 - c, so counting the other allele centres to -g' and negates BETA and T_STAT
// exactly.  Any c works for OBS_CT = 0 (TOO_FEW_OBS).
__device__ __forceinline__ int glm_centre(int obs, int sg) { return 2 * sg < obs ? 0 : 2 * sg > 3 * obs ? 2 : 1; }

// dosage of the counted allele by .bed code (00 HOM_A1, 01 missing, 10 HET, 11 HOM_A2), two bits each
constexpr uint32_t kLutA1 = 2u | 0u << 2 | 1u << 4 | 0u << 6;
constexpr uint32_t kLutA2 = 0u | 0u << 2 | 1u << 4 | 2u << 6;

constexpr int kCThreads = 256;

// grid ceil(nv / (kCThreads / 32)): warp w takes variant blockIdx.x kCThreads / 32 + w, lane l its bytes l, l + 32, ...
// With lo and hi the even and odd bits of a row byte under the byte's 4 mask bits spread to the even bits: MISSING
// lo & ~hi, HET hi & ~lo, HOM_A2 lo & hi, HOM_A1 ~(lo | hi).  Writes OBS_CT, sum g and sum g^2 (exact) under the mask
// to out[v * rec ..]: the linear path points out at the last three doubles of each record of sums (glm_sums_kernel leaves
// them there), the logistic path runs it twice, under the regression mask and under the case mask.
__global__ void __launch_bounds__(kCThreads) glm_count_kernel(const uint8_t* __restrict__ rows, int64_t stride, int nv,
                                                              int n, const uint8_t* __restrict__ mask, bool count_a2,
                                                              double* __restrict__ out, int rec) {
    const int lane = threadIdx.x & 31;
    const int v = blockIdx.x * (kCThreads / 32) + (threadIdx.x >> 5);
    if (v >= nv) return;   // the whole warp
    const uint8_t* row = rows + (int64_t)v * stride;
    const int nb = (n + 3) / 4;
    int obs = 0, hom = 0, het = 0;
    for (int b = lane; b < nb; b += 32) {
        uint32_t m = mask[b];
        m = (m | m << 2) & 0x33u;
        m = (m | m << 1) & 0x55u;
        const uint32_t by = row[b], lo = by & m, hi = (by >> 1) & m;
        obs += __popc(m) - __popc(lo & ~hi);
        het += __popc(hi & ~lo);
        hom += __popc(count_a2 ? lo & hi : m & ~(lo | hi));
    }
    obs = __reduce_add_sync(0xffffffffu, obs);
    het = __reduce_add_sync(0xffffffffu, het);
    hom = __reduce_add_sync(0xffffffffu, hom);
    if (lane == 0) {
        double* o = out + (int64_t)v * rec;
        o[0] = obs;
        o[1] = 2 * hom + het;
        o[2] = 4 * hom + het;
    }
}

// ---- sums ----------------------------------------------------------------------------------------------------------
constexpr int kSThreads = 128;
constexpr int kSTileBytes = 32;                 // row bytes per tile (128 samples)
constexpr int kSPitch = kSTileBytes / 4 + 1;    // words per staged row: odd, so 32 consecutive rows hit 32 banks
constexpr int kSTileS = 4 * kSTileBytes;        // samples per tile

// grid ceil(nv / (kSThreads VT)), after glm_count_kernel.  Qx: n rows of KMAX + 2 doubles, [q_0 .. q_{q-1}, y~, 0 ..,
// mask].  Samples >= n meet a zero tile row (mask 0, so g' = 0): fma(0, 0, a) = a for an accumulator that never holds -0,
// so they change no bit.  g' is an integer in [-2, 2], so every product g' x is exact.
template <int KMAX, int VT>
__global__ void __launch_bounds__(kSThreads) glm_sums_kernel(const uint8_t* __restrict__ rows, int64_t stride, int nv, int n,
                                                             const double* __restrict__ Qx, uint32_t lut,
                                                             double* __restrict__ sums) {
    constexpr int LD = KMAX + 2;
    constexpr int RB = kSThreads * VT;
    __shared__ uint32_t srow[RB * kSPitch];
    __shared__ __align__(16) double sq[kSTileS * LD];
    uint8_t* sb = reinterpret_cast<uint8_t*>(srow);
    const int v0 = blockIdx.x * RB;
    const int nb = (n + 3) / 4;
    double acc[VT][KMAX + 1];
    int cv[VT];   // the centre of each variant's dosage, from glm_count_kernel's OBS_CT and sum g
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int v = v0 + i * kSThreads + threadIdx.x;
        const double* rec = sums + (int64_t)min(v, nv - 1) * kGlmRec;
        cv[i] = glm_centre((int)rec[kGlmRec - 3], (int)rec[kGlmRec - 2]);
#pragma unroll
        for (int c = 0; c <= KMAX; ++c) acc[i][c] = 0.0;
    }
#pragma unroll 1
    for (int b0 = 0; b0 < nb; b0 += kSTileBytes) {
        __syncthreads();
        for (int t = threadIdx.x; t < RB * kSTileBytes; t += kSThreads) {
            const int r = t / kSTileBytes, j = t % kSTileBytes;
            const int v = v0 + r, b = b0 + j;
            sb[r * 4 * kSPitch + j] = (v < nv && b < nb) ? rows[(int64_t)v * stride + b] : 0;
        }
        const int s0 = 4 * b0;
        const int lim = min(kSTileS, n - s0) * LD;
        const double* src = Qx + (int64_t)s0 * LD;
        for (int t = threadIdx.x; t < kSTileS * LD; t += kSThreads) sq[t] = t < lim ? src[t] : 0.0;
        __syncthreads();
#pragma unroll 1
        for (int wd = 0; wd < kSTileBytes / 4; ++wd) {
            uint32_t word[VT];
#pragma unroll
            for (int i = 0; i < VT; ++i) word[i] = srow[(i * kSThreads + threadIdx.x) * kSPitch + wd];
#pragma unroll 2
            for (int j = 0; j < 16; ++j) {   // sample s0 + 16 wd + j is bits 2j, 2j + 1 of the word
                const double* x = sq + (wd * 16 + j) * LD;
                const bool in = x[KMAX + 1] != 0.0;
#pragma unroll
                for (int i = 0; i < VT; ++i) {
                    const uint32_t code = (word[i] >> (2 * j)) & 3u;
                    const double g = (in && code != 1u) ? (double)((int)((lut >> (2 * code)) & 3u) - cv[i]) : 0.0;
#pragma unroll
                    for (int c = 0; c <= KMAX; ++c) acc[i][c] = fma(g, x[c], acc[i][c]);
                }
            }
        }
    }
#pragma unroll
    for (int i = 0; i < VT; ++i) {
        const int v = v0 + i * kSThreads + threadIdx.x;
        if (v >= nv) continue;
        double* o = sums + (int64_t)v * kGlmRec;
#pragma unroll
        for (int c = 0; c <= KMAX; ++c) o[c] = acc[i][c];
    }
}

// ---- two-sided Student t p-value -------------------------------------------------------------------------------------
// ln B(a, 1/2).  From a = 10 up, ln G(a) - ln G(a + 1/2) by Stirling's series written so that nothing large cancels:
// -ln(a) / 2 + (1/2 - a log1p(1 / (2a))) + the difference of the 1/z series terms; below, lgamma directly (small values).
__device__ __forceinline__ double lbeta_half(double a) {
    const double lg_half = 0.57236494292470008707;   // ln G(1/2) = ln(pi) / 2
    if (a < 10.0) return lgamma(a) + lg_half - lgamma(a + 0.5);
    const double b = a + 0.5;
    auto corr = [](double z) {
        const double r = 1.0 / z, r2 = r * r;
        return r * (1.0 / 12.0 - r2 * (1.0 / 360.0 - r2 * (1.0 / 1260.0 - r2 * (1.0 / 1680.0))));
    };
    return lg_half - 0.5 * log(a) + (0.5 - a * log1p(0.5 / a)) + (corr(a) - corr(b));
}

// The continued fraction of I_x(a, b) (modified Lentz), converging fast for x < (a + 1) / (a + b + 2).
__device__ __forceinline__ double betacf(double a, double b, double x) {
    const double tiny = 1e-300, eps = 1e-16;
    double c = 1.0, d = 1.0 - (a + b) * x / (a + 1.0);
    if (fabs(d) < tiny) d = tiny;
    d = 1.0 / d;
    double h = d;
    for (int m = 1; m <= 100000; ++m) {
        const double m2 = 2.0 * m;
        double aa = m * (b - m) * x / ((a + m2 - 1.0) * (a + m2));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        h *= d * c;
        aa = -(a + m) * (a + b + m) * x / ((a + m2) * (a + m2 + 1.0));
        d = 1.0 + aa * d;
        if (fabs(d) < tiny) d = tiny;
        c = 1.0 + aa / c;
        if (fabs(c) < tiny) c = tiny;
        d = 1.0 / d;
        const double del = d * c;
        h *= del;
        if (fabs(del - 1.0) <= eps) break;
    }
    return h;
}

// P(|T_df| >= |t|) = I_x(df / 2, 1 / 2), x = df / (df + t^2), 1 - x = t^2 / (df + t^2) (never 1 - x by subtraction).  The
// continued fraction runs in whichever of x and 1 - x it converges for; a p below the double range comes back as 0.
__device__ __forceinline__ double t_pvalue(double t, double df) {
    const double t2 = t * t;
    const double a = 0.5 * df, b = 0.5;
    const double x = df / (df + t2), y = t2 / (df + t2);
    if (y == 0.0) return 1.0;
    const double lnx = -log1p(t2 / df), lny = log(y);
    const double front = exp(a * lnx + b * lny - lbeta_half(a));
    if (x < (a + 1.0) / (a + b + 2.0)) return fmin(1.0, front * betacf(a, b, x) / a);
    return fmax(0.0, 1.0 - front * betacf(b, a, y) / b);
}

// ---- solve ---------------------------------------------------------------------------------------------------------
// 1 / sqrt(d) for d > 0 in the normal float range (the linear solve's pivots lie in (1e-10, 1], the logistic Newton
// kernel's in (1e-10 H_jj, N]): the single-precision estimate and two Newton steps in FP64 (24 -> 48 -> ~53 bits), with
// no call into the slow paths of the FP64 division and square root (their calling convention makes the solve spill).
__device__ __forceinline__ double rsqrt_newton(double d) {
    double r = (double)__frsqrt_rn((float)d);
    r = r * fma(-0.5 * d * r, r, 1.5);
    r = r * fma(-0.5 * d * r, r, 1.5);
    return fma(r * fma(-d * r, r, 1.0), 0.5, r);
}

constexpr int kGWarps = 1;   // one warp per CTA: __syncthreads, which the compiler needs no divergence fallback for
constexpr double kPivotMin = 1e-10;   // P = Q_A^T Q_A has eigenvalues in [0, 1]: a smaller pivot is collinearity over A

// grid ceil(nv / kGWarps); warp w of CTA c takes variant c kGWarps + w.  mask: bit e of byte j = sample 4 j + e is a
// regression sample.  out[v * 6 ..] = OBS_CT, sum g, and for ERRCODE `.` the Schur term s, b_q - u^T v,
// y~_A^T y~_A - v^T v and y~_A^T y~_A, which glm_finish_kernel turns into the statistics; err[v] = VPCA_GLM_*.
// The lanes exchange values through shared memory and __syncthreads, not shuffles: every branch below is uniform over the
// warp, but the compiler cannot prove it, and its fallback for a shuffle it cannot prove converged spills.
template <int KMAX>
__global__ void __launch_bounds__(kGWarps * 32, KMAX >= 32 ? 8 : 16) glm_solve_kernel(const uint8_t* __restrict__ rows, int64_t stride, int nv,
                                                                 int n, int q, int n_reg, const double* __restrict__ Qx,
                                                                 const uint8_t* __restrict__ mask,
                                                                 const double* __restrict__ z0, double yty,
                                                                 const double* __restrict__ sums, double* __restrict__ out,
                                                                 int32_t* __restrict__ err) {
    constexpr int LD = KMAX + 2;
    constexpr int PL = KMAX + 1;                             // pitch of L: odd, so lanes reading a column hit distinct banks
    constexpr int NE = ((KMAX + 1) * (KMAX + 2) / 2 + 31) / 32;   // packed entries of [Q | y~]^T [Q | y~] per lane
    __shared__ double sL[kGWarps][KMAX * PL];
    __shared__ double sx[kGWarps][KMAX + 1];   // a sample's [q | y~], then t
    __shared__ double su[kGWarps][32], sv[kGWarps][32];
    __shared__ double sd[kGWarps][4];          // pivot, y~_A^T y~_A
    __shared__ uint32_t ssel[kGWarps][32];
    __shared__ int sc[kGWarps][4];             // OBS_CT, sum g, sum g^2, ERRCODE
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int v = blockIdx.x * kGWarps + w;
    if (v >= nv) return;   // the whole warp
    const double* rec = sums + (int64_t)v * kGlmRec;
    if (lane == 0) {
        const int obs = (int)rec[kGlmRec - 3], sg = (int)rec[kGlmRec - 2], gg = (int)rec[kGlmRec - 1];
        sc[w][0] = obs;
        sc[w][1] = sg;
        sc[w][2] = gg;
        sc[w][3] = obs - q - 1 < 1 ? VPCA_GLM_TOO_FEW_OBS
                   : (int64_t)obs * gg == (int64_t)sg * sg ? VPCA_GLM_CONST_ALLELE : VPCA_GLM_OK;
        double* o = out + (int64_t)v * 6;
        o[0] = obs;
        o[1] = sg;   // glm_finish_kernel divides
    }
    __syncthreads();
    if (sc[w][3] != VPCA_GLM_OK) {
        if (lane == 0) err[v] = sc[w][3];
        return;
    }
    // the missing-call terms over the fewer of the missing and the called regression samples
    const int obs = sc[w][0];
    const int E = (q + 1) * (q + 2) / 2;
    uint32_t eab[NE];   // (a << 8) | b of entry lane + 32 j: row a >= column b of the packed triangle
    double acc[NE];
#pragma unroll
    for (int j = 0; j < NE; ++j) {
        const int e = lane + 32 * j;
        int a = 0;
        while ((a + 1) * (a + 2) / 2 <= e) ++a;
        eab[j] = (uint32_t)a << 8 | (uint32_t)(e - a * (a + 1) / 2);
        acc[j] = 0.0;
    }
    const bool use_missing = n_reg - obs <= obs;
    if (use_missing ? n_reg > obs : obs > 0) {
        const uint8_t* row = rows + (int64_t)v * stride;
        const int nb = (n + 3) / 4;
        for (int b0 = 0; b0 < nb; b0 += 32) {
            const int b = b0 + lane;
            uint32_t sel = 0;
            if (b < nb) {
                const uint32_t by = row[b], mk = mask[b];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const bool miss = ((by >> (2 * e)) & 3u) == 1u;
                    if (((mk >> e) & 1u) && miss == use_missing) sel |= 1u << e;
                }
            }
            __syncthreads();   // the previous block's reads of ssel are done
            ssel[w][lane] = sel;
            __syncthreads();
            for (int src = 0; src < 32; ++src) {
                uint32_t sm = ssel[w][src];
                while (sm) {
                    const int e = __ffs(sm) - 1;
                    sm &= sm - 1;
                    const int64_t s = 4 * (int64_t)(b0 + src) + e;
                    for (int c = lane; c <= q; c += 32) sx[w][c] = Qx[s * LD + c];
                    __syncthreads();
#pragma unroll
                    for (int j = 0; j < NE; ++j)
                        if (lane + 32 * j < E) acc[j] = fma(sx[w][eab[j] >> 8], sx[w][eab[j] & 255u], acc[j]);
                    __syncthreads();
                }
            }
        }
    }
    // P (lower triangle) into sL, t into sx, y~_A^T y~_A into sd[1]
#pragma unroll
    for (int j = 0; j < NE; ++j) {
        if (lane + 32 * j >= E) continue;
        const int a = (int)(eab[j] >> 8), b = (int)(eab[j] & 255u);
        if (a < q) sL[w][a * PL + b] = use_missing ? (a == b ? 1.0 : 0.0) - acc[j] : acc[j];
        else if (b < q) sx[w][b] = use_missing ? z0[b] - acc[j] : acc[j];
        else sd[w][1] = use_missing ? yty - acc[j] : acc[j];
    }
    __syncthreads();
    // Cholesky P = L L^T, left-looking by column; lane i owns row i.  sr: 1 / L_jj, so the loops hold no division.
    double* sr = su[w];
    for (int j = 0; j < q; ++j) {
        if (lane == j) {
            double d = sL[w][j * PL + j];
            for (int k = 0; k < j; ++k) d = fma(-sL[w][j * PL + k], sL[w][j * PL + k], d);
            sd[w][0] = d;
            sr[j] = d > kPivotMin ? rsqrt_newton(d) : 0.0;
        }
        __syncthreads();
        if (!(sd[w][0] > kPivotMin)) {
            if (lane == 0) err[v] = VPCA_GLM_VIF_INFINITE;
            return;
        }
        if (lane > j && lane < q) {
            double x = sL[w][lane * PL + j];
            for (int k = 0; k < j; ++k) x = fma(-sL[w][lane * PL + k], sL[w][j * PL + k], x);
            sL[w][lane * PL + j] = x * sr[j];
        }
        __syncthreads();
    }
    // u = L^-1 b, v = L^-1 t by columns: lane i keeps the running right-hand sides of row i
    double wu = lane < q ? rec[lane] : 0.0, wv = lane < q ? sx[w][lane] : 0.0;
    for (int j = 0; j < q; ++j) {
        if (lane == j) {
            wu *= sr[j];
            wv *= sr[j];
            sv[w][j] = wu;
            sx[w][j] = wv;
        }
        __syncthreads();
        if (lane > j && lane < q) {
            const double lij = sL[w][lane * PL + j];
            wu = fma(-lij, sv[w][j], wu);
            wv = fma(-lij, sx[w][j], wv);
        }
    }
    __syncthreads();
    if (lane != 0) return;
    double uu = 0.0, uv = 0.0, vv = 0.0;
    for (int j = 0; j < q; ++j) {
        uu = fma(sv[w][j], sv[w][j], uu);
        uv = fma(sv[w][j], sx[w][j], uv);
        vv = fma(sx[w][j], sx[w][j], vv);
    }
    const int sg = sc[w][1], gg = sc[w][2];
    const int c = glm_centre(obs, sg);
    const double s = (double)((int64_t)gg - 2ll * c * sg + (int64_t)c * c * obs) - uu;   // sum g'^2 exactly, - u^T u
    double* o = out + (int64_t)v * 6;
    // s <= 1e-10 (sum g^2 - (sum g)^2 / OBS_CT), multiplied through by OBS_CT: the divisions wait for glm_finish_kernel.
    // The centred dosage has the same OBS_CT sum g'^2 - (sum g')^2, so the raw sums serve.
    if (!(s * obs > 1e-10 * (double)((int64_t)gg * obs - (int64_t)sg * sg))) {
        err[v] = VPCA_GLM_VIF_INFINITE;
        return;
    }
    const double yyA = sd[w][1];
    o[2] = s;
    o[3] = rec[q] - uv;
    o[4] = yyA - vv;
    o[5] = yyA;
    err[v] = VPCA_GLM_OK;
}

// From what glm_solve_kernel leaves in out[v * 6 ..] (OBS_CT, sum g, and for ERRCODE `.` the Schur term s, b_q - u^T v,
// y~_A^T y~_A - v^T v and y~_A^T y~_A): A1_FREQ, and for ERRCODE `.` BETA, the RSS check, SE, T_STAT and the two-sided p at
// df = OBS_CT - q - 1, one thread per variant; NaN where undefined.  The divisions and the p-value run here, apart from the
// solve's loops, so that none of the solve's registers has to survive their calls.
__global__ void glm_finish_kernel(int nv, int q, double* __restrict__ out, int32_t* __restrict__ err) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    double* o = out + (int64_t)v * 6;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const double obs = o[0];
    o[1] = obs > 0.0 ? o[1] / (2.0 * obs) : nan;
    if (err[v] != VPCA_GLM_OK) {
        o[2] = o[3] = o[4] = o[5] = nan;
        return;
    }
    const double s = o[2], num = o[3], rpre = o[4], yyA = o[5];
    const double beta = num / s;
    const double rss = rpre - num * beta;
    if (!(rss > 1e-12 * yyA)) {
        err[v] = VPCA_GLM_NO_RESIDUAL;
        o[2] = o[3] = o[4] = o[5] = nan;
        return;
    }
    const double df = obs - (double)(q + 1);
    const double se = sqrt(rss / df / s);
    const double t = beta / se;
    o[2] = beta;
    o[3] = se;
    o[4] = t;
    o[5] = t_pvalue(t, df);
}

template <int KMAX>
void launch(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, int n_reg, const double* d_Qx,
            const uint8_t* d_mask, const double* d_z0, double yty, uint32_t lut, double* d_sums, double* d_out,
            int32_t* d_err, cudaStream_t stream) {
    constexpr int VT = KMAX >= 32 ? 1 : 2;
    const unsigned grid = (unsigned)((nv + kSThreads * VT - 1) / (kSThreads * VT));
    glm_count_kernel<<<(unsigned)((nv + kCThreads / 32 - 1) / (kCThreads / 32)), kCThreads, 0, stream>>>(
        d_rows, stride, nv, n, d_mask, lut == kLutA2, d_sums + kGlmRec - 3, kGlmRec);
    glm_sums_kernel<KMAX, VT><<<grid, kSThreads, 0, stream>>>(d_rows, stride, nv, n, d_Qx, lut, d_sums);
    glm_solve_kernel<KMAX><<<(unsigned)((nv + kGWarps - 1) / kGWarps), kGWarps * 32, 0, stream>>>(
        d_rows, stride, nv, n, q, n_reg, d_Qx, d_mask, d_z0, yty, d_sums, d_out, d_err);
    glm_finish_kernel<<<(unsigned)((nv + 127) / 128), 128, 0, stream>>>(nv, q, d_out, d_err);
}

// ---- logistic regression (DESIGN.md 16) ------------------------------------------------------------------------------
// 1 / d for d in (1, 2]: the single-precision estimate and three Newton steps in FP64, with no call into the slow path of
// the FP64 division (as rsqrt_newton).
__device__ __forceinline__ double recip_newton(double d) {
    double r = (double)__frcp_rn((float)d);
    r = fma(r, fma(-d, r, 1.0), r);
    r = fma(r, fma(-d, r, 1.0), r);
    return fma(r, fma(-d, r, 1.0), r);
}

constexpr int kLWarps = 8;                 // variants in flight per CTA, all fed by each staged tile of Q and y
constexpr int kLPerCta = 4 * kLWarps;      // the contiguous range of variants a CTA owns
constexpr int kLTile = 32;                 // samples per staged tile: one per lane
constexpr int kLMaxPass = 25;              // passes (evaluations of l, its gradient and H) per variant
constexpr int kLMaxHalve = 8;              // step halvings in a row
constexpr double kLDelta2 = 1e-18;         // convergence: the Newton decrement squared, delta <= 1e-9
constexpr double kLFall = 1e-10;           // l fell: by more than this times |l| of the last accepted pass

// Shared memory of glm_logistic_kernel and glm_firth_kernel, in doubles.  LD: pitch of one staged sample, in the tile of
// Q and y [q_0 .. q_{KMAX-1}, y, mask, 0] and in a warp's tile U [w q_0 .. w q_{q-1}, w g', r, 0 .., g'] (u at
// 0 .. PMAX - 1, g' at PMAX).  PMAX = KMAX + 2 rows of the augmented lower triangle: H (p = q + 1 <= KMAX + 1 rows) and,
// in the logistic kernel, the gradient (row p; the Firth kernel's r is 0).  Once a pass is summed, H and then L (and the
// Firth kernel's L^-1) take the warp's U tile at pitch PH.  Per warp also theta, theta of the last accepted point, the
// step, the gradient or the Firth score (then L^-1 of it), 1 / L_jj, and NLANE arrays of one double per lane: the lanes'
// partial l, and the Firth kernel's u and g' of a tile (walk B).
template <int KMAX, int NLANE>
struct NewtonLayout {
    static constexpr int LD = KMAX + 3;
    static constexpr int PMAX = KMAX + 2;
    static constexpr int PH = KMAX + 1;
    static constexpr int NBK = PMAX / 2;                          // 2 x 2 blocks per side
    static constexpr int NB = (NBK * (NBK + 1) / 2 + 31) / 32;    // lower-triangle blocks per lane
    static constexpr int WARP = kLTile * LD + 5 * PMAX + NLANE * 32;
    static constexpr int TOTAL = kLTile * LD + kLWarps * WARP;
    static_assert(PH * PH <= kLTile * LD, "H must fit in the U tile it takes over");
};

// The pass boundary of both Newton kernels, once every warp's decision of the last pass is in sst[w] (variant, -1 for
// none; passes so far; backtracks in a row; centre of the dosage; the Firth kernel's walk).  Thread 0 gives each warp
// without a variant the CTA's next list position in [snext, end), in warp order: the variant idx[i], or i itself with
// idx == nullptr.  It writes OBS_CT and sum g from cnt[v * 6 ..] (OBS_CT, sum g, sum g^2 under the regression mask,
// then OBS_CT under the case mask) to out[v * 6 ..], and err[v] and passes[v] = 0 for the ERRCODEs that need no pass;
// firth[v], if firth is set, says whether a pass runs.  A warp that starts a variant starts from theta = (theta0, 0).
// Returns whether any warp holds a variant.
template <class Lo, int NST>
__device__ __forceinline__ bool newton_next_pass(int (*sst)[NST], int& snext, int& sany, int end, const int32_t* idx,
                                                 int q, const double* cnt, const double* theta0, double* th,
                                                 double* out, int32_t* err, int32_t* passes, uint8_t* firth) {
    __syncthreads();
    if (threadIdx.x == 0) {
        int any = 0;
        for (int ww = 0; ww < kLWarps; ++ww) {
            while (sst[ww][0] < 0 && snext < end) {
                const int v = idx ? idx[snext] : snext;
                ++snext;
                const double* c = cnt + (int64_t)v * 6;
                const int obs = (int)c[0], sg = (int)c[1], gg = (int)c[2], cases = (int)c[3];
                double* o = out + (int64_t)v * 6;
                o[0] = obs;
                o[1] = sg;   // glm_logistic_finish_kernel divides
                const int e = obs - q - 1 < 1                              ? VPCA_GLM_TOO_FEW_OBS
                              : (int64_t)obs * gg == (int64_t)sg * sg      ? VPCA_GLM_CONST_ALLELE
                              : cases == 0 || cases == obs                 ? VPCA_GLM_LOGISTIC_CONVERGE_FAIL
                                                                           : VPCA_GLM_OK;
                if (firth) firth[v] = e == VPCA_GLM_OK;
                if (e != VPCA_GLM_OK) {
                    err[v] = e;
                    passes[v] = 0;
                    continue;
                }
                sst[ww][0] = v;
                sst[ww][1] = 0;
                sst[ww][2] = 0;
                sst[ww][3] = glm_centre(obs, sg);
                if (NST > 4) sst[ww][4] = 0;
            }
            any |= sst[ww][0] >= 0;
        }
        sany = any;
    }
    __syncthreads();
    if (!sany) return false;
    const int w = threadIdx.x >> 5;
    if (sst[w][0] >= 0 && sst[w][1] == 0)
        for (int c = threadIdx.x & 31; c < Lo::PMAX; c += 32) th[c] = c < q ? theta0[c] : 0.0;
    __syncwarp();
    return true;
}

// Once every warp is done with the previous tile, the CTA stages samples [s0, s0 + kLTile) of Qx (n rows of KMAX + 2
// doubles; zero past n) into Qt at pitch LD.
template <class Lo>
__device__ __forceinline__ void newton_stage_tile(double* Qt, const double* __restrict__ Qx, int s0, int n) {
    constexpr int LD = Lo::LD, QLD = Lo::PMAX;
    __syncthreads();
    for (int i = threadIdx.x; i < kLTile * LD; i += kLWarps * 32) {
        const int r = i / LD, c = i - r * LD, s = s0 + r;
        Qt[i] = (c < QLD && s < n) ? Qx[(int64_t)s * QLD + c] : 0.0;
    }
    __syncthreads();
}

// This lane's 2 x 2 blocks of the lower triangle: rows ba, ba + 1 and columns bb, bb + 1; xo: the offset in the shared
// memory of each column's value of sample 0 (q_b in the tile of Q and y, g' in the warp's U tile at uoff, and past g'
// the tile's zero column).
template <class Lo>
__device__ __forceinline__ void newton_blocks(int lane, int q, int uoff, int (&ba)[Lo::NB], int (&bb)[Lo::NB],
                                              int (&xo)[Lo::NB][2]) {
#pragma unroll
    for (int j = 0; j < Lo::NB; ++j) {
        const int t = lane + 32 * j;
        int I = 0;
        while ((I + 1) * (I + 2) / 2 <= t) ++I;
        ba[j] = 2 * I;
        bb[j] = 2 * (t - I * (I + 1) / 2);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int b = bb[j] + e;
            xo[j][e] = b < q ? b : b == q ? uoff + Lo::PMAX : Lo::PMAX;
        }
    }
}

// The link at sample s of the warp's variant (x: its row of the staged tile): in says s is in A_v, g' the centred
// dosage (0 outside A_v), eta = x^T theta; inside A_v also e = exp(-|eta|), mu and the weight w = mu (1 - mu) (0
// outside).
struct NewtonLink {
    bool in;
    double g, eta, e, mu, wt;
};
template <class Lo>
__device__ __forceinline__ NewtonLink newton_link(const double* x, const uint8_t* row, int s, int n, int q, uint32_t lut,
                                                  int cen, const double* th) {
    NewtonLink k;
    const uint32_t code = s < n ? (row[s >> 2] >> (2 * (s & 3))) & 3u : 1u;
    k.in = x[Lo::PMAX - 1] != 0.0 && code != 1u;
    k.g = k.in ? (double)((int)((lut >> (2 * code)) & 3u) - cen) : 0.0;
    k.eta = 0.0;
    for (int c = 0; c < q; ++c) k.eta = fma(x[c], th[c], k.eta);
    k.eta = fma(th[q], k.g, k.eta);
    k.wt = k.mu = k.e = 0.0;
    if (k.in) {
        k.e = exp(-fabs(k.eta));
        const double rd = recip_newton(1.0 + k.e);
        k.mu = k.eta >= 0.0 ? rd : k.e * rd;
        k.wt = k.e * rd * rd;
    }
    return k;
}

// -l_s of a sample in A_v, from y, eta and e = exp(-|eta|): l_s = y eta - log(1 + e^eta) = -softplus(m).
__device__ __forceinline__ double newton_nll(double y, double eta, double e) {
    const double m = y != 0.0 ? -eta : eta;
    return fmax(m, 0.0) + log1p(e);
}

// One tile of the sums of H (and the gradient): lane l writes the row of U of sample s0 + l (x its row of the tile, r
// its gradient term), then every lane adds the 32 samples in order into its 2 x 2 blocks of the augmented triangle
// (4 shared loads feed 4 FMAs).  nblk: 2 x 2 blocks per side.
template <class Lo>
__device__ __forceinline__ void newton_tile_sums(const double* sm, double* U, int lane, const double* x, int q,
                                                 const NewtonLink& k, double r, int nblk, const int (&ba)[Lo::NB],
                                                 const int (&xo)[Lo::NB][2], double (&acc)[Lo::NB][4]) {
    constexpr int LD = Lo::LD;
    double* u = U + lane * LD;
    for (int c = 0; c < q; ++c) u[c] = k.wt * x[c];
    u[q] = k.wt * k.g;
    u[q + 1] = r;
    for (int c = q + 2; c < 2 * nblk; ++c) u[c] = 0.0;
    u[Lo::PMAX] = k.g;
    __syncwarp();
    const int nblocks = nblk * (nblk + 1) / 2;
#pragma unroll 2
    for (int s = 0; s < kLTile; ++s) {
        const double* ur = U + s * LD;
#pragma unroll
        for (int j = 0; j < Lo::NB; ++j) {
            if (lane + 32 * j >= nblocks) continue;
            const double u0 = ur[ba[j]], u1 = ur[ba[j] + 1];
            const double x0 = sm[xo[j][0] + s * LD], x1 = sm[xo[j][1] + s * LD];
            acc[j][0] = fma(u0, x0, acc[j][0]);
            acc[j][1] = fma(u0, x1, acc[j][1]);
            acc[j][2] = fma(u1, x0, acc[j][2]);
            acc[j][3] = fma(u1, x1, acc[j][3]);
        }
    }
}

// H (lower triangle, pitch PH, over the U tile) from the blocks, and with nrow = p + 1 the gradient (row p); each entry
// has one owner.
template <class Lo>
__device__ __forceinline__ void newton_unpack(double* H, double* grad, int p, int nrow, int lane, int nblk,
                                              const int (&ba)[Lo::NB], const int (&bb)[Lo::NB],
                                              const double (&acc)[Lo::NB][4]) {
    const int nblocks = nblk * (nblk + 1) / 2;
#pragma unroll
    for (int j = 0; j < Lo::NB; ++j) {
        if (lane + 32 * j >= nblocks) continue;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int a = ba[j] + (e >> 1), b = bb[j] + (e & 1);
            if (b >= p || a < b || a >= nrow) continue;
            if (a < p) H[a * Lo::PH + b] = acc[j][e];
            else grad[b] = acc[j][e];
        }
    }
}

// Cholesky H = L L^T over H (p x p, pitch PH), left-looking by column; lanes own rows j + 1 + lane, j + 33 + lane;
// sr[j] = 1 / L_jj.  First pass: a pivot <= kPivotMin H_jj sets flag (the warp's, in shared memory) to 3
// (VIF_INFINITE); later a pivot <= 0 sets it to 2; else it stays 0.  ldet, if set (lane 0): += sum log L_jj =
// sum log(pivot) / 2, in column order.
template <class Lo>
__device__ __forceinline__ void newton_cholesky(double* H, double* sr, int p, int lane, bool first, int& flag,
                                                double* ldet) {
    constexpr int PH = Lo::PH;
    for (int j = 0; j < p; ++j) {
        if (lane == 0) {
            const double hjj = H[j * PH + j];
            double d = hjj;
            for (int c = 0; c < j; ++c) d = fma(-H[j * PH + c], H[j * PH + c], d);
            const bool ok = first ? d > kPivotMin * hjj : d > 0.0;
            sr[j] = ok ? rsqrt_newton(d) : 0.0;
            if (ldet && ok) *ldet += 0.5 * log(d);
            flag = ok ? 0 : first ? 3 : 2;
        }
        __syncwarp();
        if (flag != 0) break;
        for (int i = j + 1 + lane; i < p; i += 32) {
            double x = H[i * PH + j];
            for (int c = 0; c < j; ++c) x = fma(-H[i * PH + c], H[j * PH + c], x);
            H[i * PH + j] = x * sr[j];
        }
        __syncwarp();
    }
}

// grid ceil(nv / kLPerCta); CTA c owns variants [c kLPerCta, min(nv, (c + 1) kLPerCta)).  cnt[v * 6 ..]: OBS_CT, sum g,
// sum g^2 under the regression mask, then OBS_CT under the case mask (glm_count_kernel).  Qx: n rows of KMAX + 2
// doubles [q_0 .. q_{q-1}, y, 0 .., mask] (y at column q); theta0: the null fit (q).  Per pass every warp holding a
// variant evaluates l, grad l and H = X^T W X at its theta over A_v, X = [Q | g'], while the CTA walks the sample tiles in
// order: lane l computes eta, mu, w and r of sample s0 + l and writes its row of U, then every lane adds the 32 samples
// in order into its 2 x 2 blocks of the augmented triangle (4 shared loads feed 4 FMAs).  Between passes the warp factors
// H and steps (DESIGN.md 16); a warp whose variant is done takes the CTA's next unstarted variant at the next pass
// boundary, in warp order.  Out: out[v * 6 ..] = OBS_CT, sum g, BETA, SE (glm_logistic_finish_kernel completes them),
// err[v], passes[v].  A sample outside A_v adds exactly 0 to every sum (u = 0, g' = 0, l untouched), so a variant's
// outputs depend on its row's codes, Q, y, theta0, the mask and n only.  No floating-point atomics.
template <int KMAX>
__global__ void __launch_bounds__(kLWarps * 32, 2) glm_logistic_kernel(const uint8_t* __restrict__ rows, int64_t stride,
                                                                      int nv, int n, int q, const double* __restrict__ Qx,
                                                                      const double* __restrict__ theta0, uint32_t lut,
                                                                      const double* __restrict__ cnt,
                                                                      double* __restrict__ out, int32_t* __restrict__ err,
                                                                      int32_t* __restrict__ passes) {
    using Lo = NewtonLayout<KMAX, 1>;
    constexpr int LD = Lo::LD, PMAX = Lo::PMAX, PH = Lo::PH, NB = Lo::NB;
    extern __shared__ __align__(16) double lsm[];
    __shared__ int sst[kLWarps][4];   // variant (-1: none), passes so far, halvings in a row, centre of the dosage
    __shared__ int sflag[kLWarps];
    __shared__ double slp[kLWarps][2];   // l of the last accepted pass, l of this pass
    __shared__ int snext, sany;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* const Qt = lsm;
    const int uoff = kLTile * LD + w * Lo::WARP;
    double* const U = lsm + uoff;
    double* const H = U;
    double* const th = U + kLTile * LD;
    double* const thp = th + PMAX;
    double* const del = thp + PMAX;
    double* const grad = del + PMAX;
    double* const sr = grad + PMAX;
    double* const lpart = sr + PMAX;
    const int p = q + 1;
    const int nblk = (p + 2) / 2;   // 2 x 2 blocks per side over rows 0 .. p
    int ba[NB], bb[NB], xo[NB][2];
    newton_blocks<Lo>(lane, q, uoff, ba, bb, xo);
    const int v_end = min(nv, (int)(blockIdx.x + 1) * kLPerCta);
    if (threadIdx.x == 0) snext = blockIdx.x * kLPerCta;
    if (lane == 0) sst[w][0] = -1;
    const int nt = (n + kLTile - 1) / kLTile;
    while (newton_next_pass<Lo>(sst, snext, sany, v_end, nullptr, q, cnt, theta0, th, out, err, passes, nullptr)) {
        const int v = sst[w][0];
        const bool act = v >= 0;   // uniform over the warp
        const uint8_t* row = rows + (int64_t)(act ? v : 0) * stride;
        const int cen = act ? sst[w][3] : 0;
        double acc[NB][4];
#pragma unroll
        for (int j = 0; j < NB; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
        double lsum = 0.0;
#pragma unroll 1
        for (int t = 0; t < nt; ++t) {
            const int s0 = t * kLTile;
            newton_stage_tile<Lo>(Qt, Qx, s0, n);
            if (!act) continue;
            const double* x = Qt + lane * LD;
            const NewtonLink k = newton_link<Lo>(x, row, s0 + lane, n, q, lut, cen, th);
            double r = 0.0;
            if (k.in) {
                r = x[q] - k.mu;
                lsum -= newton_nll(x[q], k.eta, k.e);
            }
            newton_tile_sums<Lo>(lsm, U, lane, x, q, k, r, nblk, ba, xo, acc);
            __syncwarp();
        }
        if (!act) continue;
        newton_unpack<Lo>(H, grad, p, p + 1, lane, nblk, ba, bb, acc);
        lpart[lane] = lsum;
        __syncwarp();
        if (lane == 0) {
            double l = 0.0;
            for (int i = 0; i < 32; ++i) l += lpart[i];
            const int k = ++sst[w][1];
            int fl = 0;   // 0: factor H; 1: the step was halved; 2: LOGISTIC_CONVERGE_FAIL
            if (!isfinite(l)) {
                fl = 2;
            } else if (k > 1 && l < slp[w][0] - kLFall * fabs(slp[w][0])) {
                if (sst[w][2] == kLMaxHalve || k == kLMaxPass) {
                    fl = 2;
                } else {
                    ++sst[w][2];
                    for (int c = 0; c < p; ++c) {
                        del[c] *= 0.5;
                        th[c] = thp[c] + del[c];
                    }
                    fl = 1;
                }
            }
            slp[w][1] = l;
            sflag[w] = fl;
        }
        __syncwarp();
        if (sflag[w] == 0) newton_cholesky<Lo>(H, sr, p, lane, sst[w][1] == 1, sflag[w], nullptr);
        if (lane == 0) {
            int fl = sflag[w];
            const int k = sst[w][1];
            bool done = false;
            if (fl == 0) {
                // z = L^-1 grad (over grad), delta^2 = z^T z, the step L^-T z
                double dd = 0.0;
                for (int i = 0; i < p; ++i) {
                    double z = grad[i];
                    for (int c = 0; c < i; ++c) z = fma(-H[i * PH + c], grad[c], z);
                    z *= sr[i];
                    grad[i] = z;
                    dd = fma(z, z, dd);
                }
                for (int i = p - 1; i >= 0; --i) {
                    double x = grad[i];
                    for (int c = i + 1; c < p; ++c) x = fma(-H[c * PH + i], del[c], x);
                    del[i] = x * sr[i];
                }
                if (!isfinite(dd)) {
                    fl = 2;
                } else if (dd <= kLDelta2) {
                    double* o = out + (int64_t)v * 6;
                    o[2] = th[q] + del[q];
                    o[3] = sr[q];   // sqrt([H^-1]_gg) = 1 / L_gg, g the last column
                    err[v] = VPCA_GLM_OK;
                    passes[v] = k;
                    done = true;
                } else if (k == kLMaxPass) {
                    fl = 2;
                } else {
                    slp[w][0] = slp[w][1];
                    sst[w][2] = 0;
                    for (int c = 0; c < p; ++c) {
                        thp[c] = th[c];
                        th[c] += del[c];
                    }
                }
            }
            if (fl >= 2) {
                err[v] = fl == 3 ? VPCA_GLM_VIF_INFINITE : VPCA_GLM_LOGISTIC_CONVERGE_FAIL;
                passes[v] = k;
                done = true;
            }
            if (done) sst[w][0] = -1;
        }
        __syncwarp();
    }
}

// From what glm_logistic_kernel leaves in out[v * 6 ..] (OBS_CT, sum g, and for ERRCODE `.` BETA and SE): A1_FREQ, and
// for ERRCODE `.` Z = BETA / SE and P = erfc(|Z| / sqrt(2)); NaN where undefined.  One thread per variant.
__global__ void glm_logistic_finish_kernel(int nv, double* __restrict__ out, const int32_t* __restrict__ err) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    double* o = out + (int64_t)v * 6;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const double obs = o[0];
    o[1] = obs > 0.0 ? o[1] / (2.0 * obs) : nan;
    if (err[v] != VPCA_GLM_OK) {
        o[2] = o[3] = o[4] = o[5] = nan;
        return;
    }
    const double z = o[2] / o[3];
    o[4] = z;
    o[5] = erfc(fabs(z) * 0.70710678118654752440);
}

// ---- Firth-penalized logistic regression (DESIGN.md 17) --------------------------------------------------------------
constexpr int kFMaxPass = 100;         // passes (walk A, and walk B unless A backtracks) per variant
constexpr int kFMaxBack = 30;          // backtracks in a row
constexpr double kFMaxDelta = 5.0;     // the first trial point of a step lies at most this Newton decrement away
constexpr double kFSecant = 0.45;      // the secant backtrack: U*^T Delta at the trial point < -kFSecant delta^2_prev

// grid ceil(nv / kLPerCta).  The variants to fit: list positions [0, nf) with nf = *d_nf (idx[i] the chunk's variant), or
// with idx == nullptr every variant of the chunk (nf = nv); CTA c owns positions [c kLPerCta, (c + 1) kLPerCta).  cnt,
// Qx, theta0 and out as glm_logistic_kernel.  Per variant, from (theta0, beta = 0), the passes of DESIGN.md 17: a warp is
// in walk A (l and H at theta: glm_logistic_kernel's walk without the gradient row) or in walk B (the Firth score U* with
// L^-1 in shared memory: lane l takes sample s0 + l, z = L^-1 x by independent FMA chains over the rows of L^-1, h =
// w z^T z and u = y - mu + h (1/2 - mu), then lanes own the score's entries and add the 32 samples in order).  All warps
// read the same staged tile whichever walk they are in; between walks a warp factors H, takes l* = l + sum log L_jj,
// inverts L in place, or backtracks / steps (lane 0).  Writes out[v * 6 + 2 ..] = BETA, SE for ERRCODE `.`, err[v],
// passes[v] and firth[v] = 1 where a pass ran, 0 where the ERRCODE came before any.  A sample outside A_v adds exactly 0
// to every sum, so a variant's outputs depend on its row's codes, Q, y, theta0, the mask and n only.
template <int KMAX>
__global__ void __launch_bounds__(kLWarps * 32, 2) glm_firth_kernel(const uint8_t* __restrict__ rows, int64_t stride,
                                                                   int nv, int n, int q, const double* __restrict__ Qx,
                                                                   const double* __restrict__ theta0, uint32_t lut,
                                                                   const double* __restrict__ cnt,
                                                                   const int32_t* __restrict__ idx,
                                                                   const int32_t* __restrict__ d_nf,
                                                                   double* __restrict__ out, int32_t* __restrict__ err,
                                                                   int32_t* __restrict__ passes,
                                                                   uint8_t* __restrict__ firth) {
    using Lo = NewtonLayout<KMAX, 3>;
    constexpr int LD = Lo::LD, PV = Lo::PMAX, PH = Lo::PH, NB = Lo::NB;
    extern __shared__ __align__(16) double fsm[];
    __shared__ int sst[kLWarps][5];      // variant (-1: none), passes so far, backtracks in a row, centre, walk (0 A, 1 B)
    __shared__ int sflag[kLWarps];
    __shared__ double sdp[kLWarps][4];   // l* of the last accepted point, l* of this point, s0 = its delta^2, t
    __shared__ int snext, sany;
    const int nf = idx ? *d_nf : nv;
    const int p0 = blockIdx.x * kLPerCta;
    if (p0 >= nf) return;   // the whole CTA
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double* const Qt = fsm;
    const int uoff = kLTile * LD + w * Lo::WARP;
    double* const U = fsm + uoff;
    double* const H = U;
    double* const th = U + kLTile * LD;
    double* const thp = th + PV;
    double* const del = thp + PV;
    double* const grad = del + PV;
    double* const sr = grad + PV;
    double* const lpart = sr + PV;
    double* const su = lpart + 32;
    double* const sg = su + 32;
    const int p = q + 1;
    const int nblk = (p + 1) / 2;   // 2 x 2 blocks per side over rows 0 .. p - 1
    int ba[NB], bb[NB], xo[NB][2];
    newton_blocks<Lo>(lane, q, uoff, ba, bb, xo);
    const int p_end = min(nf, p0 + kLPerCta);
    if (threadIdx.x == 0) snext = p0;
    if (lane == 0) sst[w][0] = -1;
    const int nt = (n + kLTile - 1) / kLTile;
    while (newton_next_pass<Lo>(sst, snext, sany, p_end, idx, q, cnt, theta0, th, out, err, passes, firth)) {
        const int v = sst[w][0];
        const bool act = v >= 0;   // uniform over the warp
        const bool walk_b = act && sst[w][4] == 1;
        const uint8_t* row = rows + (int64_t)(act ? v : 0) * stride;
        const int cen = act ? sst[w][3] : 0;
        double acc[NB][4];
#pragma unroll
        for (int j = 0; j < NB; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0;
        double gacc0 = 0.0, gacc1 = 0.0;   // walk B: score entries lane and lane + 32
        double lsum = 0.0;
#pragma unroll 1
        for (int t = 0; t < nt; ++t) {
            const int s0 = t * kLTile;
            newton_stage_tile<Lo>(Qt, Qx, s0, n);
            if (!act) continue;
            const double* x = Qt + lane * LD;
            const NewtonLink k = newton_link<Lo>(x, row, s0 + lane, n, q, lut, cen, th);
            if (!walk_b) {
                if (k.in) lsum -= newton_nll(x[q], k.eta, k.e);
                newton_tile_sums<Lo>(fsm, U, lane, x, q, k, 0.0, nblk, ba, xo, acc);
            } else {
                double uu = 0.0;
                if (k.in) {
                    // h = w ||L^-1 x||^2, one FMA chain per row of L^-1 (H holds L^-1)
                    double hh = 0.0;
                    for (int j = 0; j < q; ++j) {
                        const double* li = H + j * PH;
                        double z = 0.0;
                        for (int c = 0; c <= j; ++c) z = fma(li[c], x[c], z);
                        hh = fma(z, z, hh);
                    }
                    {
                        const double* li = H + q * PH;
                        double z = 0.0;
                        for (int c = 0; c < q; ++c) z = fma(li[c], x[c], z);
                        z = fma(li[q], k.g, z);
                        hh = fma(z, z, hh);
                    }
                    uu = fma(k.wt * hh, 0.5 - k.mu, x[q] - k.mu);
                }
                su[lane] = uu;
                sg[lane] = k.g;
                __syncwarp();
                const int c1 = lane + 32;
#pragma unroll 2
                for (int r = 0; r < kLTile; ++r) {
                    const double ur = su[r];
                    if (lane < p) gacc0 = fma(ur, lane < q ? Qt[r * LD + lane] : sg[r], gacc0);
                    if (c1 < p) gacc1 = fma(ur, c1 < q ? Qt[r * LD + c1] : sg[r], gacc1);
                }
            }
            __syncwarp();
        }
        if (!act) continue;
        if (!walk_b) {
            newton_unpack<Lo>(H, grad, p, p, lane, nblk, ba, bb, acc);
            lpart[lane] = lsum;
            __syncwarp();
            if (lane == 0) {
                double l = 0.0;
                for (int i = 0; i < 32; ++i) l += lpart[i];
                sdp[w][1] = l;
                ++sst[w][1];
                sflag[w] = isfinite(l) ? 0 : 2;   // 0: factor H; 2: not finite
            }
            __syncwarp();
            const int k = sst[w][1];
            const bool first = k == 1;
            double ldet = 0.0;   // lane 0: sum log L_jj
            // first pass: VIF_INFINITE (3); later a pivot <= 0 backtracks (2)
            if (sflag[w] == 0) newton_cholesky<Lo>(H, sr, p, lane, first, sflag[w], &ldet);
            if (lane == 0) {
                int fl = sflag[w];
                const double ls = sdp[w][1] + ldet;
                sdp[w][1] = ls;
                if (first) {
                    if (fl != 0) fl = fl == 3 ? 3 : 4;   // 4: FIRTH_CONVERGE_FAIL
                } else if (fl != 0 || ls < sdp[w][0] - kLFall * fabs(sdp[w][0])) {
                    // halve the step
                    if (sst[w][2] == kFMaxBack || k == kFMaxPass) {
                        fl = 4;
                    } else {
                        ++sst[w][2];
                        const double t = 0.5 * sdp[w][3];
                        sdp[w][3] = t;
                        for (int c = 0; c < p; ++c) th[c] = __dadd_rn(thp[c], __dmul_rn(t, del[c]));
                        fl = 1;
                    }
                }
                if (fl >= 3) {
                    err[v] = fl == 3 ? VPCA_GLM_VIF_INFINITE : VPCA_GLM_FIRTH_CONVERGE_FAIL;
                    passes[v] = k;
                    sst[w][0] = -1;
                } else if (fl == 0) {
                    sst[w][4] = 1;
                }
                sflag[w] = fl;
            }
            __syncwarp();
            if (sflag[w] == 0) {
                // L^-1 in place by rows: row i of L^-1 from row i of L and the rows of L^-1 above it
                for (int i = 0; i < p; ++i) {
                    double x = 0.0;
                    if (lane < i) {
                        for (int c = lane; c < i; ++c) x = fma(H[i * PH + c], H[c * PH + lane], x);
                        x = -x * sr[i];
                    }
                    __syncwarp();
                    if (lane < i) H[i * PH + lane] = x;
                    if (lane == (i & 31)) H[i * PH + i] = sr[i];
                    __syncwarp();
                }
            }
        } else {
            if (lane < p) grad[lane] = gacc0;
            if (lane + 32 < p) grad[lane + 32] = gacc1;
            __syncwarp();
            if (lane == 0) {
                const int k = sst[w][1];
                bool done = false;
                sst[w][4] = 0;
                double s1 = 0.0;
                if (k > 1)
                    for (int c = 0; c < p; ++c) s1 = fma(grad[c], del[c], s1);
                const double s0 = sdp[w][2];
                if (k > 1 && s1 < -kFSecant * s0) {
                    // the secant on the directional derivative of l* along the step
                    if (sst[w][2] == kFMaxBack || k == kFMaxPass) {
                        err[v] = VPCA_GLM_FIRTH_CONVERGE_FAIL;
                        passes[v] = k;
                        done = true;
                    } else {
                        ++sst[w][2];
                        const double t = sdp[w][3] * s0 / (s0 - s1);
                        sdp[w][3] = t;
                        for (int c = 0; c < p; ++c) th[c] = __dadd_rn(thp[c], __dmul_rn(t, del[c]));
                    }
                } else {
                    // z = L^-1 U* (over sr), delta^2 = z^T z, the step L^-T z
                    double dd = 0.0;
                    for (int i = 0; i < p; ++i) {
                        double z = 0.0;
                        for (int c = 0; c <= i; ++c) z = fma(H[i * PH + c], grad[c], z);
                        sr[i] = z;
                        dd = fma(z, z, dd);
                    }
                    for (int j = 0; j < p; ++j) {
                        double x = 0.0;
                        for (int i = j; i < p; ++i) x = fma(H[i * PH + j], sr[i], x);
                        del[j] = x;
                    }
                    if (!isfinite(dd) || (dd > kLDelta2 && k == kFMaxPass)) {
                        err[v] = VPCA_GLM_FIRTH_CONVERGE_FAIL;
                        passes[v] = k;
                        done = true;
                    } else if (dd <= kLDelta2) {
                        double* o = out + (int64_t)v * 6;
                        o[2] = th[q] + del[q];
                        o[3] = H[q * PH + q];   // 1 / L_gg
                        err[v] = VPCA_GLM_OK;
                        passes[v] = k;
                        done = true;
                    } else {
                        const double t = dd > kFMaxDelta * kFMaxDelta ? kFMaxDelta / sqrt(dd) : 1.0;
                        sdp[w][0] = sdp[w][1];
                        sdp[w][2] = dd;
                        sdp[w][3] = t;
                        sst[w][2] = 0;
                        for (int c = 0; c < p; ++c) {
                            thp[c] = th[c];
                            th[c] = __dadd_rn(thp[c], __dmul_rn(t, del[c]));
                        }
                    }
                }
                if (done) sst[w][0] = -1;
            }
        }
        __syncwarp();
    }
}

// The variants a fallback refits: those the maximum-likelihood kernel ended with LOGISTIC_CONVERGE_FAIL after at least
// one pass, into idx[0 .. *nf) (in any order: a variant's outputs do not depend on its place); firth[v] = 0 elsewhere.
__global__ void glm_firth_select_kernel(int nv, const int32_t* __restrict__ err, const int32_t* __restrict__ passes,
                                        uint8_t* __restrict__ firth, int32_t* __restrict__ idx, int32_t* __restrict__ nf) {
    const int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nv) return;
    const bool f = err[v] == VPCA_GLM_LOGISTIC_CONVERGE_FAIL && passes[v] > 0;
    firth[v] = f;
    if (f) idx[atomicAdd(nf, 1)] = v;
}

// firth_mode 0: the maximum-likelihood fit alone; VPCA_GLM_FIRTH_FALLBACK: then the Firth fit of the variants it could
// not fit; VPCA_GLM_FIRTH_ALWAYS: the Firth fit alone.  d_firth, d_idx, d_nf: unused in mode 0.
template <int KMAX>
cudaError_t launch_logistic(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, const double* d_Qx,
                            const uint8_t* d_mask, const uint8_t* d_case, const double* d_theta0, uint32_t lut,
                            double* d_cnt, double* d_out, int32_t* d_err, int32_t* d_passes, int firth_mode,
                            uint8_t* d_firth, int32_t* d_idx, int32_t* d_nf, cudaStream_t stream) {
    const unsigned cgrid = (unsigned)((nv + kCThreads / 32 - 1) / (kCThreads / 32));
    const unsigned lgrid = (unsigned)((nv + kLPerCta - 1) / kLPerCta);
    glm_count_kernel<<<cgrid, kCThreads, 0, stream>>>(d_rows, stride, nv, n, d_mask, lut == kLutA2, d_cnt, 6);
    glm_count_kernel<<<cgrid, kCThreads, 0, stream>>>(d_rows, stride, nv, n, d_case, lut == kLutA2, d_cnt + 3, 6);
    cudaError_t e = cudaSuccess;
    if (firth_mode != VPCA_GLM_FIRTH_ALWAYS) {
        const size_t smem = NewtonLayout<KMAX, 1>::TOTAL * sizeof(double);
        e = cudaFuncSetAttribute(glm_logistic_kernel<KMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        glm_logistic_kernel<KMAX><<<lgrid, kLWarps * 32, smem, stream>>>(d_rows, stride, nv, n, q, d_Qx, d_theta0, lut,
                                                                          d_cnt, d_out, d_err, d_passes);
    }
    if (firth_mode != 0) {
        const bool fallback = firth_mode == VPCA_GLM_FIRTH_FALLBACK;
        if (fallback) {
            e = cudaMemsetAsync(d_nf, 0, sizeof(int32_t), stream);
            if (e != cudaSuccess) return e;
            glm_firth_select_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(nv, d_err, d_passes, d_firth,
                                                                                      d_idx, d_nf);
        }
        const size_t smem = NewtonLayout<KMAX, 3>::TOTAL * sizeof(double);
        e = cudaFuncSetAttribute(glm_firth_kernel<KMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return e;
        glm_firth_kernel<KMAX><<<lgrid, kLWarps * 32, smem, stream>>>(d_rows, stride, nv, n, q, d_Qx, d_theta0, lut,
                                                                       d_cnt, fallback ? d_idx : nullptr, d_nf, d_out,
                                                                       d_err, d_passes, d_firth);
    }
    glm_logistic_finish_kernel<<<(unsigned)((nv + 127) / 128), 128, 0, stream>>>(nv, d_out, d_err);
    return cudaSuccess;
}

// Calls f(std::integral_constant<int, glm_kmax(q)>()): the one place a q picks the kernels' instantiation.
template <class F>
auto with_kmax(int q, F&& f) {
    switch (glm_kmax(q)) {
        case 2: return f(std::integral_constant<int, 2>());
        case 4: return f(std::integral_constant<int, 4>());
        case 8: return f(std::integral_constant<int, 8>());
        case 16: return f(std::integral_constant<int, 16>());
        default: return f(std::integral_constant<int, 32>());
    }
}

}  // namespace

int glm_kmax(int q) { return q <= 2 ? 2 : q <= 4 ? 4 : q <= 8 ? 8 : q <= 16 ? 16 : 32; }

cudaError_t glm_linear(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, int n_reg, const double* d_Qx,
                       const uint8_t* d_mask, const double* d_z0, double yty, int counted, double* d_sums, double* d_out,
                       int32_t* d_err, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    const uint32_t lut = counted == 2 ? kLutA2 : kLutA1;
    with_kmax(q, [&](auto K) {
        launch<decltype(K)::value>(d_rows, stride, nv, n, q, n_reg, d_Qx, d_mask, d_z0, yty, lut, d_sums, d_out, d_err,
                                   stream);
    });
    return cudaGetLastError();
}

cudaError_t glm_logistic(const uint8_t* d_rows, int64_t stride, int nv, int n, int q, const double* d_Qx,
                         const uint8_t* d_mask, const uint8_t* d_case, const double* d_theta0, int counted, double* d_cnt,
                         double* d_out, int32_t* d_err, int32_t* d_passes, int firth_mode, uint8_t* d_firth,
                         int32_t* d_idx, int32_t* d_nf, cudaStream_t stream) {
    if (nv <= 0) return cudaSuccess;
    const uint32_t lut = counted == 2 ? kLutA2 : kLutA1;
    const cudaError_t e = with_kmax(q, [&](auto K) {
        return launch_logistic<decltype(K)::value>(d_rows, stride, nv, n, q, d_Qx, d_mask, d_case, d_theta0, lut, d_cnt,
                                                   d_out, d_err, d_passes, firth_mode, d_firth, d_idx, d_nf, stream);
    });
    return e != cudaSuccess ? e : cudaGetLastError();
}

}  // namespace vpca
