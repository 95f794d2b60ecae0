// frame_walk.cuh — tsgpu_encrypt_object on a compressed object: every chunk's zstd frame is checked the way the decoder's index
// stage (zstd_dec_index_kernel) checks it, and nothing is decoded.  The frame header must carry the magic number, no Dictionary_ID
// and a Frame_Content_Size; the block walk must end at a last block without a reserved type and inside the chunk; after the frame
// come only the announced Content_Checksum and skippable frames (zd_frame_tail_ok).  The Content_Checksum itself is not verified:
// that needs the decoded bytes.
//
// The walk is a serial chain of dependent 3-byte header loads, one thread per chunk: a speed-mode 4 MiB frame has 512 blocks, a
// libzstd level-3 frame about 32.  The chunks were copied in just before, so the headers are read from L2.  The verdict only
// gates the batch's release on the host: the encryption runs regardless, and a refused batch never leaves the GPU.
#pragma once
#include "ts_common.cuh"
#include "zstd_dec.cuh"

namespace ts {

constexpr int FW_T = 128;

struct FrameWalkArgs {
    const uint8_t* base; const uint64_t* off; const uint32_t* len;   // chunk i: len[i] bytes at base + off[i]
    uint32_t* status;        // per chunk: ZD_ST_OK, or ZD_ST_CORRUPT for a frame the index stage would refuse
    uint32_t* fcs;           // per chunk: its Frame_Content_Size (clamped to 32 bits); 0 for an empty chunk or a refused frame
    uint32_t n;              // chunks of the batch
};

__global__ void __launch_bounds__(FW_T) frame_walk_kernel(const __grid_constant__ FrameWalkArgs A) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const uint8_t* p = A.base + A.off[i];
    const uint32_t n = A.len[i];
    uint32_t st = ZD_ST_OK, size = 0;
    if (n) {
        uint64_t fcs = 0;
        uint32_t pos = zd_frame_header(p, n, &fcs);
        bool ok = pos != 0 && fcs != 0xffffffffffffffffull, last = false;
        while (ok && !last) {
            if (pos + 3 > n) { ok = false; break; }
            const ZdBlkHdr bh = zd_block_header(p + pos);
            if (bh.type == 3) { ok = false; break; }
            last = bh.last;
            pos += 3 + (bh.type == 1 ? 1 : bh.size);
            if (pos > n) ok = false;
        }
        if (ok && !zd_frame_tail_ok(p, n, pos)) ok = false;
        if (ok) size = fcs > 0xffffffffull ? 0xffffffffu : (uint32_t)fcs;
        else st = ZD_ST_CORRUPT;
    }
    A.status[i] = st;
    A.fcs[i] = size;
}

}  // namespace ts
