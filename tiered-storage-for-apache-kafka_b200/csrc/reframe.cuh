// reframe.cuh — TSGPU_FLAG_REFRAME of tsgpu_rewrite_object: the source frames of a batch, already accepted by the decoder and
// sitting in their 16-byte aligned d_frames slots, are sealed with their Content_Checksum in place, or replaced by a smaller
// dense frame of the same chunk.
//
// Sealing (RFC 8878 3.1.1): Frame_Header_Descriptor bit 2 is set (the header keeps its length) and the low 32 bits of XXH64 of
// the chunk's decoded bytes go, little-endian, right after the last block; skippable frames that followed the frame in the chunk
// move 4 bytes on.  That is byte for byte what libzstd writes for the same blocks with ZSTD_c_checksumFlag, and clearing the bit
// and dropping the 4 bytes gives the old frame back.
//
// Writes stay inside the frame's own bytes plus 4 and inside its slot: `room` bounds every chunk, and a chunk whose frame the
// walk does not accept, or that would not fit, is left as it is -- the decoder has refused it, and its batch fails at the drain.
#pragma once
#include "ts_common.cuh"
#include "xxh64.cuh"
#include "zstd_dec.cuh"

namespace ts {

constexpr int RF_WPB = 4;                        // chunks (warps) per CTA of the seal kernel

struct ReframeArgs {
    uint8_t* frames; const uint64_t* f_off; uint32_t* f_len;       // the frame slots (b_off / b_len); f_len is updated
    const uint8_t* orig; const uint64_t* o_off; const uint32_t* o_len;   // the chunks' decoded bytes (d_orig, by the chunk index)
    const uint8_t* cand; const uint32_t* cand_len;                  // pick: the dense frames, at f_off in their own area
    uint32_t n;                                                     // chunks of the batch
    uint32_t room;                                                  // bytes of a frame slot
};

// End of the last block of the frame at p[0, n), 0 when the frame is not one the walk accepts.  One thread.
__device__ __forceinline__ uint32_t rf_blocks_end(const uint8_t* p, uint32_t n) {
    uint64_t fcs;
    uint32_t pos = zd_frame_header(p, n, &fcs);
    if (!pos) return 0;
    while (pos + 3 <= n) {
        const uint32_t bh = p[pos] | (p[pos + 1] << 8) | ((uint32_t)p[pos + 2] << 16);
        const uint32_t type = (bh >> 1) & 3, body = type == 1 ? 1u : bh >> 3;
        pos += 3;
        if (type == 3 || body > n - pos) return 0;
        pos += body;
        if (bh & 1) return pos;
    }
    return 0;
}

// One warp per chunk: the frame gets its Content_Checksum unless it has one (the source decode verified that one).
__global__ void __launch_bounds__(RF_WPB * 32) reframe_seal_kernel(const __grid_constant__ ReframeArgs A) {
    __shared__ uint4 stage[RF_WPB][XXH_STAGE_BYTES / 16];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * RF_WPB + warp;
    if (chunk >= A.n) return;                                        // whole warp
    uint8_t* f = A.frames + A.f_off[chunk];
    const uint32_t n = A.f_len[chunk];
    uint32_t end = 0;
    if (lane == 0 && n <= A.room - 4) end = rf_blocks_end(f, n);
    end = __shfl_sync(TS_FULL, end, 0);
    if (end == 0 || (f[4] & 0x04)) return;                           // damaged, or sealed already: as it is
    const uint32_t h = xxh64_warp_low32(A.orig + A.o_off[chunk], A.o_len[chunk], (uint64_t*)stage[warp], lane);
    // the skippable frames after the last block move 4 bytes on, 32 bytes at a time from the back: a window is read whole
    // before it is written, and the windows below it only write bytes that have been read
    for (uint32_t hi = n; hi > end;) {
        const uint32_t lo = hi - end > 32 ? hi - 32 : end;
        const uint32_t at = lo + lane;
        const uint8_t b = at < hi ? f[at] : 0;
        __syncwarp();
        if (at < hi) f[at + 4] = b;
        __syncwarp();
        hi = lo;
    }
    if (lane < 4) f[end + lane] = (uint8_t)(h >> (8 * lane));
    if (lane == 0) { f[4] |= 0x04; A.f_len[chunk] = n + 4; }
}

constexpr int RF_PICK_T = 256;

// One CTA per chunk: the dense frame replaces the frame in the slot when it is strictly smaller.
__global__ void __launch_bounds__(RF_PICK_T) reframe_pick_kernel(const __grid_constant__ ReframeArgs A) {
    const uint32_t chunk = blockIdx.x, tid = threadIdx.x;
    const uint32_t old = A.f_len[chunk], m = A.cand_len[chunk];
    __syncthreads();                                                 // every thread has read f_len before it changes
    if (m >= old || m > A.room) return;
    uint4* d = (uint4*)(A.frames + A.f_off[chunk]);
    const uint4* s = (const uint4*)(A.cand + A.f_off[chunk]);
    for (uint32_t i = tid; i < (m + 15) / 16; i += RF_PICK_T) d[i] = s[i];
    if (tid == 0) A.f_len[chunk] = m;
}

}  // namespace ts
