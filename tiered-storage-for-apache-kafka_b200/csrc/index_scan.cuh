// index_scan.cuh — K5: exclusive prefix sum of transformed chunk sizes -> transformed positions.
// Replaces the serial loop of AbstractChunkIndex.materializeChunks
// (<reference>/core/src/main/java/io/aiven/kafka/tieredstorage/manifest/index/AbstractChunkIndex.java:52-72).
// One warp; 32 sizes per step through a shuffle scan with a 64-bit running carry (n = 256 for a 1 GiB segment).
#pragma once
#include "ts_common.cuh"

namespace ts {

__device__ __forceinline__ uint64_t warp_inclusive_scan_u64(uint64_t v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t u = __shfl_up_sync(TS_FULL, v, o);
        if ((int)lane >= o) v += u;
    }
    return v;
}
__device__ __forceinline__ uint32_t warp_inclusive_scan_u32(uint32_t v, uint32_t lane) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        uint32_t u = __shfl_up_sync(TS_FULL, v, o);
        if ((int)lane >= o) v += u;
    }
    return v;
}

// positions[i] = sum_{k<i} sizes[k]; positions[n] = total
__global__ void __launch_bounds__(32) chunk_index_scan_kernel(const uint32_t* __restrict__ sizes, uint32_t n,
                                                              uint64_t* __restrict__ positions) {
    const uint32_t lane = threadIdx.x;
    uint64_t carry = 0;
    for (uint32_t base = 0; base < n; base += 32) {
        uint32_t i = base + lane;
        uint64_t v = i < n ? sizes[i] : 0;
        uint64_t inc = warp_inclusive_scan_u64(v, lane);
        if (i < n) positions[i] = carry + inc - v;
        carry += __shfl_sync(TS_FULL, inc, 31);
    }
    if (lane == 0) positions[n] = carry;
}

}  // namespace ts
