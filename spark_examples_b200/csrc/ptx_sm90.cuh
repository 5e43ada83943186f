// Thin inline-PTX wrappers for the sm_90a features the Gram kernel uses: mbarrier, TMA (cp.async.bulk.tensor) and
// warpgroup MMA (wgmma).  Written for `nvcc -gencode arch=compute_90a,code=sm_90a` only.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace vpca {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%laneid;" : "=r"(r));
    return r;
}

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P1;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
    return ok != 0;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void prefetch_tensormap(const void* desc) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(desc)) : "memory");
}
// 3D variants (the genotype matrix is stored as panels: coordinate 2 selects the panel)
__device__ __forceinline__ void tma_load_3d(uint32_t smem_dst, const void* desc, uint32_t bar, int32_t c0, int32_t c1,
                                            int32_t c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(desc)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// ---------------------------------------------------------------- wgmma
// Warpgroup MMA, both operands K-major in shared memory (128-byte swizzle), 64 x 128 accumulator tile of the warpgroup
// in registers: d[4 i + {0, 1}] = (row r, columns 8 i + 2 (lane % 4) + {0, 1}), d[4 i + {2, 3}] = (row r + 8, same columns),
// r = 16 (warp % 4) + lane / 4.  The accumulator always adds (scale-d = 1): callers zero it before the first k-step.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma
__device__ __forceinline__ void wgmma_fence_acc(uint32_t (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+r"(d[i])::"memory");
}
__device__ __forceinline__ void wgmma_fence_acc(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// s32 += s8 x s8 (K = 32 bytes)
__device__ __forceinline__ void wgmma_s8(uint32_t (&d)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k32.s32.s8.s8 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p;\n\t}\n"
        : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]), "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]), "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]), "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]), "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]), "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]), "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]), "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
        : "l"(a_desc), "l"(b_desc));
}

// f32 += bf16 x bf16 (K = 16 elements = 32 bytes)
__device__ __forceinline__ void wgmma_bf16(float (&f)[64], uint64_t a_desc, uint64_t b_desc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(f[0]), "+f"(f[1]), "+f"(f[2]), "+f"(f[3]), "+f"(f[4]), "+f"(f[5]), "+f"(f[6]), "+f"(f[7]), "+f"(f[8]), "+f"(f[9]), "+f"(f[10]), "+f"(f[11]), "+f"(f[12]), "+f"(f[13]), "+f"(f[14]), "+f"(f[15]), "+f"(f[16]), "+f"(f[17]), "+f"(f[18]), "+f"(f[19]), "+f"(f[20]), "+f"(f[21]), "+f"(f[22]), "+f"(f[23]), "+f"(f[24]), "+f"(f[25]), "+f"(f[26]), "+f"(f[27]), "+f"(f[28]), "+f"(f[29]), "+f"(f[30]), "+f"(f[31]), "+f"(f[32]), "+f"(f[33]), "+f"(f[34]), "+f"(f[35]), "+f"(f[36]), "+f"(f[37]), "+f"(f[38]), "+f"(f[39]), "+f"(f[40]), "+f"(f[41]), "+f"(f[42]), "+f"(f[43]), "+f"(f[44]), "+f"(f[45]), "+f"(f[46]), "+f"(f[47]), "+f"(f[48]), "+f"(f[49]), "+f"(f[50]), "+f"(f[51]), "+f"(f[52]), "+f"(f[53]), "+f"(f[54]), "+f"(f[55]), "+f"(f[56]), "+f"(f[57]), "+f"(f[58]), "+f"(f[59]), "+f"(f[60]), "+f"(f[61]), "+f"(f[62]), "+f"(f[63])
        : "l"(a_desc), "l"(b_desc));
}

// Named barrier over `count` threads (the two consumer warpgroups of a CTA)
__device__ __forceinline__ void named_sync(uint32_t id, uint32_t count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

}  // namespace ptx
}  // namespace vpca
