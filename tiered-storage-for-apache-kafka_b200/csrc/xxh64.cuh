// xxh64.cuh — XXH64 (seed 0) of a byte range, computed by one warp: the Content_Checksum of RFC 8878 §3.1.1 (its low 32 bits,
// little-endian after the last block).  The compressor writes it when asked to (TSGPU_FLAG_ZSTD_CHECKSUM) and the decoder
// verifies it whenever a frame announces one; both use xxh64_warp_low32.
//
// XXH64 is serial within its input: four accumulators, each taking one 8-byte word of every 32-byte stripe, n/32 dependent
// rounds each.  Those four chains are the cost, so everything else stays off them:
//   * all 32 lanes stage the next XXH_BATCH stripes with 128-bit loads, issued before the chain lanes start on the current
//     batch, so the load latency hides behind the chains;
//   * the staging lanes multiply each word by P2 as they store it (the multiply does not depend on the accumulator);
//   * lanes 0-3 (the chains) only add the staged product, rotate and multiply by P1.
#pragma once
#include "ts_common.cuh"

namespace ts {

constexpr uint64_t XXH_P1 = 11400714785074694791ull, XXH_P2 = 14029467366897019727ull, XXH_P3 = 1609587929392839161ull,
                   XXH_P4 = 9650029242287828579ull, XXH_P5 = 2870177450012600261ull;
constexpr uint32_t XXH_BATCH = 64;                           // stripes staged per round trip
constexpr uint32_t XXH_STAGE_BYTES = XXH_BATCH * 32;         // shared memory per hashing warp (16-byte aligned)
constexpr uint32_t XXH_LOADS = XXH_STAGE_BYTES / (32 * 16);  // 128-bit loads per lane per batch
constexpr uint32_t XXH64_EMPTY_LOW32 = 0x51D8E999u;          // XXH64("", 0) = 0xEF46DB3751D8E999

__device__ __forceinline__ uint64_t xxh_rotl(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
__device__ __forceinline__ uint64_t xxh_round(uint64_t acc, uint64_t in) { return xxh_rotl(acc + in * XXH_P2, 31) * XXH_P1; }
__device__ __forceinline__ uint64_t xxh_rd64(const uint8_t* p) {    // little-endian, any alignment, no byte past p + 7
    if ((((uintptr_t)p) & 7) == 0) return *(const uint64_t*)p;
    uint64_t v = 0;
    for (int k = 0; k < 8; k++) v |= (uint64_t)p[k] << (8 * k);
    return v;
}
struct alignas(16) XxhPair { uint64_t a, b; };

// 16 input bytes at p; `al`: p is 16-byte aligned
__device__ __forceinline__ uint4 xxh_ld16(const uint8_t* p, bool al) {
    if (al) return *(const uint4*)p;
    return make_uint4(ld_u32_unaligned(p), ld_u32_unaligned(p + 4), ld_u32_unaligned(p + 8), ld_u32_unaligned(p + 12));
}
// batch starting at byte b0: lane l loads the 16-byte words l, l + 32, ... of it (coalesced), nothing at or beyond `body`
__device__ __forceinline__ void xxh_load(uint4 (&r)[XXH_LOADS], const uint8_t* d, uint32_t b0, uint32_t body, bool al, uint32_t lane) {
    _Pragma("unroll")
    for (uint32_t k = 0; k < XXH_LOADS; k++) {
        const uint32_t o = b0 + (k * 32 + lane) * 16;
        r[k] = o < body ? xxh_ld16(d + o, al) : make_uint4(0, 0, 0, 0);
    }
}

// Low 32 bits of XXH64(d[0, n), seed 0), on every lane.  Called by a whole, converged warp.  stage: XXH_STAGE_BYTES of shared
// memory owned by this warp, 16-byte aligned.  `d` may be written earlier in the same kernel by the same warp (plain loads).
__device__ TS_NOINLINE uint32_t xxh64_warp_low32(const uint8_t* d, uint32_t n, uint64_t* stage, uint32_t lane) {
    uint64_t v = lane == 0 ? XXH_P1 + XXH_P2 : lane == 1 ? XXH_P2 : lane == 2 ? 0ull : 0ull - XXH_P1;
    const uint32_t body = n / 32 * 32;                       // the stripes; the tail (< 32 bytes) is folded in below
    const bool al = (((uintptr_t)d) & 15) == 0;
    uint4 r[XXH_LOADS];
    xxh_load(r, d, 0, body, al, lane);
    for (uint32_t b0 = 0; b0 < body; b0 += XXH_STAGE_BYTES) {
        __syncwarp();                                        // the chains are done with the previous batch
        _Pragma("unroll")
        for (uint32_t k = 0; k < XXH_LOADS; k++) {           // 16-byte word i of the batch = stripe i / 2, words 2 (i & 1) and + 1
            const uint32_t i = k * 32 + lane;
            const uint64_t lo = (uint64_t)r[k].x | ((uint64_t)r[k].y << 32), hi = (uint64_t)r[k].z | ((uint64_t)r[k].w << 32);
            ((XxhPair*)stage)[i] = XxhPair{lo * XXH_P2, hi * XXH_P2};
        }
        __syncwarp();
        if (b0 + XXH_STAGE_BYTES < body) xxh_load(r, d, b0 + XXH_STAGE_BYTES, body, al, lane);   // in flight during the chains
        if (lane < 4) {
            const uint32_t cnt = min(XXH_BATCH, (body - b0) / 32);
            const uint64_t* s = stage + lane;
            _Pragma("unroll 8")
            for (uint32_t i = 0; i < cnt; i++) v = xxh_rotl(v + s[4 * i], 31) * XXH_P1;
        }
    }
    __syncwarp();
    const uint64_t v1 = __shfl_sync(TS_FULL, v, 0), v2 = __shfl_sync(TS_FULL, v, 1), v3 = __shfl_sync(TS_FULL, v, 2),
                   v4 = __shfl_sync(TS_FULL, v, 3);
    uint64_t h;
    if (n >= 32) {
        h = xxh_rotl(v1, 1) + xxh_rotl(v2, 7) + xxh_rotl(v3, 12) + xxh_rotl(v4, 18);
        h = (h ^ xxh_round(0, v1)) * XXH_P1 + XXH_P4;
        h = (h ^ xxh_round(0, v2)) * XXH_P1 + XXH_P4;
        h = (h ^ xxh_round(0, v3)) * XXH_P1 + XXH_P4;
        h = (h ^ xxh_round(0, v4)) * XXH_P1 + XXH_P4;
    } else h = XXH_P5;
    h += n;
    uint32_t at = body;                                      // the tail: every lane computes the same value
    for (; at + 8 <= n; at += 8) { h ^= xxh_round(0, xxh_rd64(d + at)); h = xxh_rotl(h, 27) * XXH_P1 + XXH_P4; }
    if (at + 4 <= n) {
        const uint32_t w = d[at] | (d[at + 1] << 8) | (d[at + 2] << 16) | ((uint32_t)d[at + 3] << 24);
        h ^= (uint64_t)w * XXH_P1; h = xxh_rotl(h, 23) * XXH_P2 + XXH_P3; at += 4;
    }
    for (; at < n; at++) { h ^= (uint64_t)d[at] * XXH_P5; h = xxh_rotl(h, 11) * XXH_P1; }
    h ^= h >> 33; h *= XXH_P2; h ^= h >> 29; h *= XXH_P3; h ^= h >> 32;
    return (uint32_t)h;
}

}  // namespace ts
