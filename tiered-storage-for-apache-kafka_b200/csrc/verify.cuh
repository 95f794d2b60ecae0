// verify.cuh — read-back check of a transform batch (TSGPU_FLAG_VERIFY): the chunks the detransform stages decoded from the
// batch's own output, compared with the original chunks still in HBM.  One CTA per (64 KiB piece, chunk); the read-back side
// sits in 16-byte aligned slots and is read with 128-bit loads, the original side may start anywhere (ragged calls) and is
// read by funnel shift as in pack.cuh.  Each chunk ends with its first differing byte offset (atomicMin) or a size code.
#pragma once
#include "ts_common.cuh"

namespace ts {

constexpr uint32_t VERIFY_PIECE = 64 * 1024;     // bytes of one chunk a CTA compares
constexpr int VERIFY_T = 256;
constexpr uint32_t VERIFY_ST_SIZE = 3;           // status code next to the read-back stages' 1 (tag) and 2 (frame)
constexpr uint32_t VERIFY_NO_DIFF = 0xffffffffu;

struct VerifyArgs {
    const uint8_t* orig; const uint64_t* orig_off; const uint32_t* orig_len;   // the batch's input chunks
    const uint8_t* back; const uint64_t* back_off; const uint32_t* back_len;   // read back; back + back_off[i] is 16-byte aligned
    uint32_t* status;    // in: 0, or 1 / 2 from the decrypt / decode stage (the chunk is skipped); out: VERIFY_ST_SIZE
    uint32_t* diff;      // out: first differing byte offset per chunk; the caller presets VERIFY_NO_DIFF
};

__device__ __forceinline__ uint32_t first_diff_byte(uint4 a, uint4 b) {      // a != b; little-endian byte index 0..15
    const uint32_t w[4] = {a.x ^ b.x, a.y ^ b.y, a.z ^ b.z, a.w ^ b.w};
    for (uint32_t k = 0; k < 4; k++)
        if (w[k]) return 4 * k + ((uint32_t)(__ffs((int)w[k]) - 1) >> 3);
    return 16;
}

__global__ void __launch_bounds__(VERIFY_T) verify_compare_kernel(const __grid_constant__ VerifyArgs A) {
    const uint32_t tid = threadIdx.x;
    const uint32_t chunk = blockIdx.y, piece = blockIdx.x;
    if (A.status[chunk] != 0) return;                        // tag / frame failure: reported as such, nothing to compare
    const uint32_t n = A.orig_len[chunk];
    if (A.back_len[chunk] != n) {
        if (piece == 0 && tid == 0) A.status[chunk] = VERIFY_ST_SIZE;
        return;
    }
    const uint32_t lo = piece * VERIFY_PIECE;
    if (lo >= n) return;                                     // whole CTA
    const uint32_t cnt = min(n, lo + VERIFY_PIECE) - lo;
    const uint8_t* o = A.orig + A.orig_off[chunk] + lo;
    const uint8_t* b = A.back + A.back_off[chunk] + lo;
    const bool o_aligned = ((uintptr_t)o & 15) == 0;
    const uint32_t vecs = cnt >> 4;
    for (uint32_t i = tid; i < vecs; i += VERIFY_T) {
        const uint4 bv = ldg128_stream((const uint4*)b + i);
        const uint8_t* q = o + 16 * (size_t)i;
        const uint4 ov = o_aligned ? ldg128_stream((const uint4*)q)
                                   : make_uint4(ld_u32_unaligned(q), ld_u32_unaligned(q + 4), ld_u32_unaligned(q + 8), ld_u32_unaligned(q + 12));
        if (ov.x != bv.x || ov.y != bv.y || ov.z != bv.z || ov.w != bv.w) {
            atomicMin(&A.diff[chunk], lo + 16 * i + first_diff_byte(ov, bv));
            break;                                           // this thread's later vectors lie further in
        }
    }
    const uint32_t done = 16 * vecs;
    if (tid < cnt - done && o[done + tid] != b[done + tid]) atomicMin(&A.diff[chunk], lo + done + tid);
}

}  // namespace ts
