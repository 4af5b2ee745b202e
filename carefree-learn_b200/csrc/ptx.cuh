// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with
// shared-memory descriptors), proxy fences.  Everything here is hand-written; no CUTLASS/CuTe types are used.
// Descriptor bit layouts follow the PTX ISA "matrix descriptor" table of the wgmma section.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

namespace b200 {

// ----------------------------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
    uint32_t pred = 0;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(pred));
    return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (launch fails with an error) instead of hanging the GPU.
// The wait must stay free of function calls: it sits between wgmma groups in the consumer k-loops, and any call there
// (printf is one) makes ptxas serialise every wgmma of the kernel (warning C7510; csrc/Makefile fails the build on it).
// B200_MBAR_TIMEOUT_PRINTF reports which block / thread timed out, for debugging builds only.
#ifndef B200_MBAR_TIMEOUT_CYCLES
#define B200_MBAR_TIMEOUT_CYCLES (4000000000ll)  // ~2 s at 1.98 GHz
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    long long t0 = clock64();
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3ffu) == 0u && (clock64() - t0) > B200_MBAR_TIMEOUT_CYCLES) {
#ifdef B200_MBAR_TIMEOUT_PRINTF
            printf("b200: mbarrier timeout block %d thread %d parity %u\n", blockIdx.x, threadIdx.x, parity);
#endif
            __trap();
        }
    }
}

// ----------------------------------------------------------------------------------------------
// proxy fences
// ----------------------------------------------------------------------------------------------
// generic-proxy smem writes -> visible to the async proxy (TMA store, wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
// 4-D box (channels, x, y, image) of a channels-last activation: coordinates may be NEGATIVE or past the end -- the
// out-of-bound part of the box is zero-filled, which is exactly the zero padding of a 3x3 convolution
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], "
        "[%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}
// Multicast load: the box lands at the SAME smem offset in every CTA of `cta_mask`, and each destination CTA's
// mbarrier (same offset) receives the complete_tx.
__device__ __forceinline__ void tma_load_2d_mcast(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1,
                                                  uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
        "[%0], [%1, {%3, %4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void tma_store_2d(const void* tmap, const void* smem_src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tmap)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_3d(const void* tmap, const void* smem_src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                     reinterpret_cast<uint64_t>(tmap)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// L2 prefetch of a tile (no smem destination): lets a later TMA load of the same bytes hit L2 instead of HBM
__device__ __forceinline__ void tma_prefetch_l2_3d(const void* tmap, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global.tile [%0, {%1, %2, %3}];" ::"l"(reinterpret_cast<uint64_t>(tmap)),
                 "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// L2 prefetch of a CONTIGUOUS byte range (16-byte aligned address and size): no smem destination, no completion to wait for
__device__ __forceinline__ void bulk_prefetch_l2(const void* gptr, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(reinterpret_cast<uint64_t>(gptr)), "r"(bytes) : "memory");
}
// wait until at most 1 committed bulk store still has to read its smem source (two staging buffers in rotation)
__device__ __forceinline__ void tma_store_wait_read1() {
    asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// wait until the smem source of all committed bulk stores has been read (buffer reusable)
__device__ __forceinline__ void tma_store_wait_read0() {
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
// wait until all committed bulk stores are complete (globally visible)
__device__ __forceinline__ void tma_store_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// wgmma (sm_90a warpgroup MMA): descriptors, fences, the instruction shapes the kernels use
// ----------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (64 bit, PTX ISA "matrix descriptor" for wgmma):
//   [0,14)  start address >> 4      [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset >> 4     [49,52) base offset = 0
//   [62,64) layout: 0 interleave, 1 SWIZZLE_128B, 2 SWIZZLE_64B, 3 SWIZZLE_32B
// K-major 128B-swizzled tile (rows of 64 bf16): SBO = 1024 (8-row group), LBO unused, +32 B per 16-element K step.
// MN-major 128B-swizzled tile (rows of 64 MN elements, one row per k): SBO = 1024 (8 k rows), LBO = distance between
// 64-element MN atoms, +2048 B per 16-row K step.
constexpr uint32_t kSwz128 = 1;
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes,
                                                   uint32_t layout) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3ffffu) >> 4);
    d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3fffu) << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3fffu) << 32;
    d |= static_cast<uint64_t>(layout & 3u) << 62;
    return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accumulator reads / writes across an asynchronous wgmma that is still in flight.
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D (+)= A * B, one warpgroup, fp32 accumulators in registers (m64nNk16; thread t of the warpgroup holds, for every
// n8 block j, rows 16 * (t / 32) + (t % 32) / 4 (+ 8) and columns 8 j + 2 (t % 4) (+ 1): d[4 j + {0, 1, 2, 3}]).
// _ss: A and B from shared memory (descriptors); t<A><B>: 1 = that operand is MN-major.
// _rs_tb: A from registers (the m16k16 fragment of mma.sync per warp), B MN-major from shared memory.
__device__ __forceinline__ void wgmma_m64n256k16_ss_t00(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n256k16_ss_t01(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 0, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n256k16_ss_t10(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 1, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n256k16_ss_t11(float (&d)[128], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %130, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n256k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
        "%128, %129, p, 1, 1, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "%32, %33, p, 1, 1, 0, 0;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(scale_d));
}

__device__ __forceinline__ void wgmma_m64n64k16_rs_tb(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t scale_d) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %37, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
        "{%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(scale_d));
}

// Register re-distribution between the warpgroups of a CTA (all 4 warps of a warpgroup execute it together)
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N));
}
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N));
}

// ----------------------------------------------------------------------------------------------
// numeric helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);  // .x = lo (low 16 bits), .y = hi
    return *reinterpret_cast<uint32_t*>(&t);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
__device__ __forceinline__ float bf16lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16hi(uint32_t u) { return __uint_as_float(u & 0xffff0000u); }

// exact-erf GELU, evaluated in fp32 like ATen's GeluCUDAKernelImpl ("none" approximation): libm reference versions
__device__ __forceinline__ float gelu_erf_libm(float x) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));
}
__device__ __forceinline__ float gelu_erf_grad_libm(float x) {
    const float kBeta = 0.39894228040143267794f;  // 1/sqrt(2*pi)   (M_2_SQRTPI * M_SQRT1_2 * 0.5)
    float cdf = 0.5f * (1.0f + erff(x * 0.70710678118654752440f));
    float pdf = expf(-0.5f * x * x) * kBeta;
    return cdf + x * pdf;
}
// Fast erf for the GEMM epilogues (libm erff costs ~30 issue slots / element and made the FF1 GEMM epilogue-bound).
// Measured against ATen's fp32 GELU on 4M bf16 inputs ~ N(0, 1.5): relative L2 difference of the bf16 results
// 3.4e-7 (1-ulp flips only where |gelu| is negligible); derivative max abs error 1.8e-7.
__device__ __forceinline__ float fast_rcp(float x) {
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_ex2(float x) {
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
// 1 + erf(z) without cancellation: erfc(|z|) = t exp(-z^2 + P(t)), t = 1 / (1 + |z| / 2)  (Chebyshev fit of
// Numerical Recipes' erfcc, fractional error < 1.2e-7 everywhere), then 1 + erf(z) = z >= 0 ? 2 - erfc : erfc.
__device__ __forceinline__ float one_plus_erf(float z) {
    const float az = fabsf(z);
    const float t = fast_rcp(fmaf(0.5f, az, 1.0f));
    float p = fmaf(0.17087277f, t, -0.82215223f);
    p = fmaf(p, t, 1.48851587f);
    p = fmaf(p, t, -1.13520398f);
    p = fmaf(p, t, 0.27886807f);
    p = fmaf(p, t, -0.18628806f);
    p = fmaf(p, t, 0.09678418f);
    p = fmaf(p, t, 0.37409196f);
    p = fmaf(p, t, 1.00002368f);
    p = fmaf(p, t, -1.26551223f);
    const float w = t * fast_ex2(fmaf(-az, az, p) * 1.4426950408889634f);
    return z >= 0.f ? 2.0f - w : w;
}
__device__ __forceinline__ float gelu_erf(float x) {
    return (0.5f * x) * one_plus_erf(x * 0.70710678118654752440f);
}
// d/dx gelu(x) = cdf + x * pdf, fp32, same formula as ATen's GeluBackwardCUDAKernelImpl
__device__ __forceinline__ float gelu_erf_grad(float x) {
    const float cdf = 0.5f * one_plus_erf(x * 0.70710678118654752440f);
    const float e = fast_ex2(x * x * (-0.5f * 1.4426950408889634f));  // exp(-x^2 / 2)
    return fmaf(x * 0.39894228040143267794f, e, cdf);
}
// ---- two-element versions ------------------------------------------------------------------------------------------
// The GELU epilogues evaluate two activations at a time.  sm_90 has no packed fp32x2 arithmetic, so a pair is two
// scalars: fma2 / mul2 round each lane exactly like fmaf / __fmul_rn.
struct f32x2_t {
    float x, y;
};
__device__ __forceinline__ f32x2_t pk2(float a, float b) { return f32x2_t{a, b}; }
__device__ __forceinline__ void upk2(f32x2_t v, float& a, float& b) {
    a = v.x;
    b = v.y;
}
__device__ __forceinline__ f32x2_t fma2(f32x2_t a, f32x2_t b, f32x2_t c) { return f32x2_t{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)}; }
__device__ __forceinline__ f32x2_t mul2(f32x2_t a, f32x2_t b) { return f32x2_t{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
// w = erfc(|x| / sqrt 2) for two values, ax = |x|, x2 = x^2 (packed).  erfc(z) = t exp(-z^2 + P(t)), t = 1 / (1 + z / 2):
// degree-6 minimax fit of P (max relative error 5.6e-6 in fp32), coefficients pre-multiplied by log2(e).
__device__ __forceinline__ void erfc_abs2(float x0, float x1, f32x2_t& w, f32x2_t& ax, f32x2_t& x2) {
    ax = pk2(fabsf(x0), fabsf(x1));
    float d0, d1;
    upk2(fma2(ax, pk2(0.35355339059327373f, 0.35355339059327373f), pk2(1.0f, 1.0f)), d0, d1);  // 1 + |x| / (2 sqrt 2)
    const f32x2_t t = pk2(fast_rcp(d0), fast_rcp(d1));
    constexpr float kL = 1.4426950408889634f;
    f32x2_t p = fma2(pk2(-0.0630452529f * kL, -0.0630452529f * kL), t, pk2(0.465173551f * kL, 0.465173551f * kL));
    p = fma2(p, t, pk2(-1.06472952f * kL, -1.06472952f * kL));
    p = fma2(p, t, pk2(0.747652742f * kL, 0.747652742f * kL));
    p = fma2(p, t, pk2(0.14202046f * kL, 0.14202046f * kL));
    p = fma2(p, t, pk2(1.04137768f * kL, 1.04137768f * kL));
    p = fma2(p, t, pk2(-1.26844758f * kL, -1.26844758f * kL));
    x2 = mul2(ax, ax);
    float g0, g1;
    upk2(fma2(x2, pk2(-0.5f * kL, -0.5f * kL), p), g0, g1);  // (-x^2/2 + P(t)) log2 e
    w = mul2(t, pk2(fast_ex2(g0), fast_ex2(g1)));
}
// gelu(x) = x Phi(x) = relu(x) - |x| erfc(|x| / sqrt 2) / 2   (exact identity; no sign-dependent select)
__device__ __forceinline__ void gelu_erf2(float x0, float x1, float& g0, float& g1) {
    f32x2_t w, ax, x2;
    erfc_abs2(x0, x1, w, ax, x2);
    upk2(fma2(mul2(ax, w), pk2(-0.5f, -0.5f), pk2(fmaxf(x0, 0.f), fmaxf(x1, 0.f))), g0, g1);
}
// gelu'(x) = Phi(x) + x phi(x),  Phi(x) = 1/2 + sign(x) (1/2 - erfc(|x| / sqrt 2) / 2),  phi(x) = exp(-x^2/2) / sqrt(2 pi).
// Here erfc(z) = t E Q(t) with E = exp(-z^2) = exp(-x^2/2) taken out of the fit (Q(t) = erfcx(z) / t, degree-6 fit on
// t in [0.2, 1], i.e. |x| <= 11.3, max relative error 9.3e-7; beyond that E < 2e-28 and Q stays in [0.28, 0.35]):
// the SAME exponential serves phi(x), so the derivative costs 2 MUFU ops per element (rcp, ex2) instead of 3 --
// the dGELU epilogue runs 32768 of these per tile against a 16-lane MUFU pipe.  Max abs error vs ATen 3e-7.
__device__ __forceinline__ void gelu_erf_grad2(float x0, float x1, float& g0, float& g1) {
    const f32x2_t ax = pk2(fabsf(x0), fabsf(x1));
    float d0, d1;
    upk2(fma2(ax, pk2(0.35355339059327373f, 0.35355339059327373f), pk2(1.0f, 1.0f)), d0, d1);  // 1 + |x| / (2 sqrt 2)
    const f32x2_t t = pk2(fast_rcp(d0), fast_rcp(d1));
    f32x2_t q = fma2(pk2(0.09331708401441574f, 0.09331708401441574f), t, pk2(-0.37464964389801025f, -0.37464964389801025f));
    q = fma2(q, t, pk2(0.4142274856567383f, 0.4142274856567383f));
    q = fma2(q, t, pk2(0.020182941108942032f, 0.020182941108942032f));
    q = fma2(q, t, pk2(0.2881791591644287f, 0.2881791591644287f));
    q = fma2(q, t, pk2(0.27631810307502747f, 0.27631810307502747f));
    q = fma2(q, t, pk2(0.28242501616477966f, 0.28242501616477966f));
    float n0, n1;
    upk2(mul2(mul2(ax, ax), pk2(-0.5f * 1.4426950408889634f, -0.5f * 1.4426950408889634f)), n0, n1);
    const f32x2_t e = pk2(fast_ex2(n0), fast_ex2(n1));  // exp(-x^2 / 2)
    float h0, h1;
    upk2(fma2(mul2(mul2(t, q), e), pk2(-0.5f, -0.5f), pk2(0.5f, 0.5f)), h0, h1);  // 1/2 - erfc(|x| / sqrt 2) / 2
    const f32x2_t cdf = pk2(0.5f + copysignf(h0, x0), 0.5f + copysignf(h1, x1));
    upk2(fma2(mul2(pk2(x0, x1), pk2(0.39894228040143267794f, 0.39894228040143267794f)), e, cdf), g0, g1);
}

// CLIP's QuickGELU (cflearn/modules/core/activations.py:151-153): `net * torch.sigmoid(1.702 * net)` on a bf16 tensor.
// Eager runs three elementwise kernels, each rounding its output to bf16; the same three roundings are made here.
__device__ __forceinline__ float fast_sigmoid(float x) {  // 1 / (1 + 2^(-x log2 e)); fp32 accuracy ~1e-7 relative
    return fast_rcp(1.0f + fast_ex2(-1.4426950408889634f * x));
}
__device__ __forceinline__ float quick_gelu_bf16(float x) {  // x: a bf16 value
    const float t = bf16_round(1.702f * x);
    const float sg = bf16_round(fast_sigmoid(t));
    return x * sg;  // (the caller rounds the product to bf16)
}
// autograd of the same three ops, with eager's bf16 rounding after every backward kernel (dy, x: bf16 values):
//   mul:      d_net1 = bf16(dy * s),  d_s = bf16(dy * x)            s = bf16(sigmoid(t)), t = bf16(1.702 x)
//   sigmoid:  d_t = bf16(bf16(d_s * bf16(1 - s)) * s)   -- ATen's CUDA sigmoid_backward evaluates `a * (1 - b) * b` in the
//             tensor's own type (c10::BFloat16 arithmetic rounds after every operator), unlike its opmath forward kernels
//   scale:    d_net2 = bf16(d_t * 1.702)
//   sum:      bf16(d_net1 + d_net2)   (the caller rounds the sum)
__device__ __forceinline__ float quick_gelu_bf16_grad(float x, float dy) {
    const float t = bf16_round(1.702f * x);
    const float sg = bf16_round(fast_sigmoid(t));
    const float d1 = bf16_round(dy * sg);
    const float ds = bf16_round(dy * x);
    const float dt = bf16_round(bf16_round(ds * bf16_round(1.0f - sg)) * sg);
    const float d2 = bf16_round(dt * 1.702f);
    return d1 + d2;
}

}  // namespace b200
