// ts_common.cuh — shared device-side helpers for the sm_90a chunk-transform kernels.
//
// The device headers are written in a restricted CUDA subset so that tests/simt/ (a TEST-ONLY fiber
// emulator, never linked into libtsgpu.so) can also compile them with g++ to check kernel logic on
// the GPU-less build box.  Everything inside `#ifdef TSGPU_SIMT` exists only for that test build.
#pragma once
#include <stdint.h>
#include <stddef.h>

#ifdef TSGPU_SIMT
#include "simt.h"
#define TS_DYN_SMEM(name) uint8_t* name = simt::g_blk->dyn_smem
#define TS_DEVICE_ASM 0
#define TS_NOINLINE __attribute__((noinline))
#else
#include <cuda_runtime.h>
#define TS_DYN_SMEM(name) extern __shared__ __align__(1024) uint8_t name[]
#define TS_DEVICE_ASM 1
#define TS_NOINLINE __noinline__
#endif

#define TS_FULL 0xffffffffu

namespace ts {

__device__ __forceinline__ uint32_t bswap32(uint32_t x) { return __byte_perm(x, 0, 0x0123); }
__device__ __forceinline__ uint4 xor4(uint4 a, uint4 b) { return make_uint4(a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w); }

// ---- unaligned little-endian reads from byte buffers (global or shared) --------------------------------
__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {
    // two aligned words + funnel shift: no byte loops on the hot paths
    uintptr_t a = (uintptr_t)p;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    uint32_t sh = (uint32_t)(a & 3) * 8;
    uint32_t lo = w[0];
    if (sh == 0) return lo;
    return __funnelshift_r(lo, w[1], sh);
}

// ---- 128-bit streaming global accesses -----------------------------------------------------------------
__device__ __forceinline__ uint4 ldg128_stream(const uint4* p) {
#if TS_DEVICE_ASM
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
#else
    return *p;
#endif
}
__device__ __forceinline__ void stg128_stream(uint4* p, uint4 v) {
#if TS_DEVICE_ASM
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#else
    *p = v;
#endif
}

// ---- TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP) ------------------------
// Used to stage read-only tables (GHASH H-power table, FSE/Huffman tables) and input blocks.
#if TS_DEVICE_ASM
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_1d(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "TS_WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra TS_DONE_%=;\n"
        "bra TS_WAIT_%=;\n"
        "TS_DONE_%=:\n"
        "}\n" :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
#endif

// Block-cooperative copy of `bytes` (multiple of 16, both sides 16-byte aligned) global -> shared.
// One elected thread issues TMA bulk copies (<= 64 KiB is fine in one instruction; we split at 32 KiB).
// Caller must __syncthreads() before (bar init visibility) — handled inside.
__device__ __forceinline__ void block_bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes,
                                                uint64_t* bar, uint32_t parity) {
#if TS_DEVICE_ASM
    if (threadIdx.x == 0) {
        mbar_expect_tx(bar, bytes);
        uint32_t off = 0;
        while (off < bytes) {
            uint32_t n = bytes - off > 32768u ? 32768u : bytes - off;
            tma_load_1d((uint8_t*)dst_smem + off, (const uint8_t*)src_gmem + off, n, bar);
            off += n;
        }
    }
    mbar_wait(bar, parity);
#else
    (void)bar; (void)parity;
    for (uint32_t i = threadIdx.x * 16; i < bytes; i += blockDim.x * 16)
        *(uint4*)((uint8_t*)dst_smem + i) = *(const uint4*)((const uint8_t*)src_gmem + i);
    __syncthreads();
#endif
}

}  // namespace ts
