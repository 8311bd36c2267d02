// tc_ptx.cuh -- inline-PTX wrappers shared by the tensor-core kernels (sm_90a): mbarriers, TMA loads, wgmma
// shared-memory descriptors and the warpgroup fence / commit / wait around wgmma (wgmma.cuh).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace {

constexpr int BLOCK_M = 128;
constexpr int kRowBytes = 128;  // one swizzle row per pixel per K-step: 32 fp32 (tf32, K=8 per MMA)
                                // or 64 fp16 (f16, K=16 per MMA); four MMAs per K-step either way

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "r"(c2), "r"(c3)
        : "memory");
}
// TMA im2col load of a 4-D [C, W, H, N] tensor (map from cuTensorMapEncodeIm2col): the map's pixelsPerColumn pixels
// that follow (w, h, n) in (n, h, w) order inside the map's bounding box, each shifted by (off_w, off_h), c0.. of
// their channels; elements outside the tensor (the padding halo, pixels past the last image) are zero-filled and
// count toward complete_tx
__device__ __forceinline__ void tma_load_im2col_4d(const CUtensorMap* map, uint64_t* bar, void* smem, int c0, int w,
                                                   int h, int n, uint16_t off_w, uint16_t off_h) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.im2col.mbarrier::complete_tx::bytes"
        " [%0], [%1, {%3, %4, %5, %6}], [%2], {%7, %8};"
        ::"r"(smem_u32(smem)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(w), "r"(h),
        "r"(n), "h"(off_w), "h"(off_h)
        : "memory");
}
// TMA store of a shared-memory box, tracked by the issuing thread's bulk async-group
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t saddr, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(saddr), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the source shared memory of all but N committed groups has been read (it may be overwritten)
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
// all but N committed groups have completed (their global writes are done)
template <int N>
__device__ __forceinline__ void bulk_wait() {
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// barrier over `threads` threads (a multiple of 32) on hardware barrier `id` (0 is __syncthreads')
__device__ __forceinline__ void named_bar_sync(int id, int threads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// K-major, 128-byte swizzle wgmma shared-memory matrix descriptor (cute::GMMA::GmmaDescriptor):
// start>>4 [0,14) | LBO>>4 [16,30) (ignored for swizzled K-major, 1) | SBO>>4 [32,46) = 8 rows * 128 B
// | base offset [49,52) = 0 (stages are 1024-byte aligned) | layout SWIZZLE_128B = 1 [62,64)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ordering of register accesses around the asynchronous wgmma of a warpgroup
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of an accumulator register across the asynchronous MMAs
__device__ __forceinline__ void reg_fence(float& r) { asm volatile("" : "+f"(r)::"memory"); }

__device__ __forceinline__ void sts128u(uint32_t saddr, uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float2 lds64f(uint32_t saddr) {
    float2 v;
    asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr) : "memory");
    return v;
}
__device__ __forceinline__ void sts64f(uint32_t saddr, float x, float y) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(saddr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void sts32u(uint32_t saddr, uint32_t v) {
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(saddr), "r"(v) : "memory");
}
// byte offset inside a 1024-byte-aligned region written / read by TMA with 128-byte swizzle: 16-byte chunk
// (bits 4..6) XOR 128-byte row (bits 7..9)
__device__ __forceinline__ uint32_t swz128(uint32_t off) { return off ^ (((off >> 7) & 7u) << 4); }
// the same with 64-byte swizzle (512-byte aligned region): 16-byte chunk (bits 4..5) XOR bits 7..8
__device__ __forceinline__ uint32_t swz64(uint32_t off) { return off ^ (((off >> 7) & 3u) << 4); }

}  // namespace
