// part_crc.cuh — CRC-32C or CRC-64/NVME of the upload parts of a transformed object (tsgpu_transform_parts and its _crc64 twin),
// hashed from the bytes in HBM that one D2H per batch takes home (the slot's d_pack: the batch's transformed chunks back to back).
// Everything here is generic over the CRC word W (crc32.cuh): uint32_t for CRC-32C, uint64_t for CRC-64/NVME.
//
// Per batch of L packed bytes, two kernels:
//   pcrc_tiles  (compute stream, after pack_chunks) one thread per 256-byte piece: its raw CRC by slice-by-8 (eight tables of 256
//               words in shared memory: 8 KiB for CRC-32C, 16 KiB for CRC-64; 128-bit loads), and the inclusive prefix over the 128
//               pieces of a 32 KiB tile (GF(2) shifts by x^(8*256*2^r)).  The last CTA to finish turns the tile CRCs into
//               exclusive prefixes over the batch.
//   pcrc_cuts   (out_stream, at the drain, when the batch's object offset is known) one thread per part boundary inside the
//               batch and one for its end: the raw CRC of [0, x) of the batch from a tile prefix, a piece prefix and at most 256
//               bytes.  The host turns consecutive prefixes into the raw CRCs of the part pieces (crc32.cuh) and combines them, in
//               batch order, into the part CRCs and the object CRC.
// With SLOTS (tsgpu_check_object) both kernels read the batch's chunks in place instead of packed: chunk i at b + off[i], as
// the fetched object sits in its transformed slots.  The bytes hashed are the same, the chunks taken back to back.
#pragma once
#include <type_traits>
#include "crc32.cuh"

namespace ts {

constexpr uint32_t PCRC_PIECE = 256;                   // bytes per thread in pcrc_tiles
constexpr uint32_t PCRC_T = 128;                       // threads per CTA
constexpr uint32_t PCRC_TILE = PCRC_PIECE * PCRC_T;    // 32 KiB
constexpr uint32_t PCRC_GRID = 264;                    // pcrc_tiles CTAs at most (they stride over the tiles)
constexpr uint32_t PCRC_CUTS_T = 128;

template <typename W> struct PcrcArgs {
    const uint8_t* b;                // the batch's packed transformed bytes (256-byte aligned)
    const uint32_t* len; uint32_t nb;   // the batch's transformed chunk sizes (device): L = their sum
    W* pin;                          // [npieces] raw CRC of [tile start, end of piece q)
    W* ttot;                         // [ntiles]  raw CRC of each tile, then (after the last CTA) of [0, tile start)
    uint32_t* done;                  // CTAs of pcrc_tiles that have finished (the last one resets it to 0)
};
template <typename W> struct PcrcSlotsArgs : PcrcArgs<W> {
    const uint64_t* off;             // chunk i starts at b + off[i] (device)
};
template <typename W, bool SLOTS> using PcrcIn = typename std::conditional<SLOTS, PcrcSlotsArgs<W>, PcrcArgs<W>>::type;

// Slice-by-8 tables: T[k][i] is the raw CRC of byte i followed by k zero bytes.  Block-cooperative.
template <typename W>
__device__ __forceinline__ void pcrc_tables(W (*T)[256]) {
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) T[0][i] = crc_table_entry(i, crc_poly<W>(0));
    __syncthreads();
    for (int k = 1; k < 8; k++) {
        for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) { const W p = T[k - 1][i]; T[k][i] = (p >> 8) ^ T[0][p & 0xffu]; }
        __syncthreads();
    }
}
// 8 bytes, little-endian words: the register's low 32 bits meet lo, and a 64-bit register's high 32 bits meet hi
template <typename W>
__device__ __forceinline__ W pcrc_8(const W (*T)[256], W c, uint32_t lo, uint32_t hi) {
    if constexpr (sizeof(W) == 8) { lo ^= (uint32_t)c; hi ^= (uint32_t)(c >> 32); }
    else lo ^= c;
    return T[7][lo & 0xffu] ^ T[6][(lo >> 8) & 0xffu] ^ T[5][(lo >> 16) & 0xffu] ^ T[4][lo >> 24] ^
           T[3][hi & 0xffu] ^ T[2][(hi >> 8) & 0xffu] ^ T[1][(hi >> 16) & 0xffu] ^ T[0][hi >> 24];
}
// The batch's packed length, from its chunk sizes (every thread).
template <typename W>
__device__ __forceinline__ uint32_t pcrc_len(const PcrcArgs<W>& A) {
    uint32_t L = 0;
    for (uint32_t i = 0; i < A.nb; i++) L += A.len[i];
    return L;
}

// SLOTS: raw CRC update by bytes [lo, hi) of the batch's chunks taken back to back, each read where it sits.
template <typename W>
__device__ __forceinline__ W pcrc_slots_bytes(const W* T, W c, const PcrcSlotsArgs<W>& A, uint32_t lo, uint32_t hi) {
    uint32_t start = 0;
    for (uint32_t i = 0; i < A.nb && lo < hi; i++) {
        const uint32_t end = start + A.len[i];
        if (lo < end) {
            const uint32_t n = min(hi, end) - lo;
            c = crc_bytes(T, c, A.b + A.off[i] + (lo - start), n);
            lo += n;
        }
        start = end;
    }
    return c;
}
// SLOTS: raw CRC of the piece [lo, hi).  A full piece inside one chunk is read as aligned words joined by funnel shifts (a chunk
// starts 4 bytes into its slot, and a piece anywhere in it); the word after the piece is still inside the slot, whose stride leaves
// at least 16 bytes after the largest chunk it accepts.  Pieces across a chunk end and the batch's last piece go byte by byte.
template <typename W>
__device__ __forceinline__ W pcrc_slots_piece(const W (*T)[256], const PcrcSlotsArgs<W>& A, uint32_t lo, uint32_t hi) {
    uint32_t i = 0, start = 0;
    while (i + 1 < A.nb && start + A.len[i] <= lo) start += A.len[i++];
    if (hi - lo != PCRC_PIECE || hi > start + A.len[i]) return pcrc_slots_bytes(T[0], W(0), A, lo, hi);
    const uint8_t* p = A.b + A.off[i] + (lo - start);
    const uint32_t* V = (const uint32_t*)((uintptr_t)p & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)((uintptr_t)p & 3) * 8;
    W c = 0;
    uint32_t prev = __ldg(V);
#pragma unroll 4
    for (uint32_t k = 1; k <= PCRC_PIECE / 4; k += 2) {
        const uint32_t w1 = __ldg(V + k), w2 = __ldg(V + k + 1);
        c = pcrc_8(T, c, __funnelshift_r(prev, w1, sh), __funnelshift_r(w1, w2, sh));
        prev = w2;
    }
    return c;
}

// ---------------------------------------------------------------------------------------------------- pcrc_tiles
template <typename W, bool SLOTS>
__global__ void __launch_bounds__(PCRC_T) pcrc_tiles_kernel(const __grid_constant__ PcrcIn<W, SLOTS> A) {
    __shared__ W T[8][256];
    __shared__ W s[PCRC_T];
    __shared__ uint32_t last;
    pcrc_tables(T);
    const uint32_t tid = threadIdx.x, L = pcrc_len(A);
    const uint32_t ntiles = (L + PCRC_TILE - 1) / PCRC_TILE, npieces = (L + PCRC_PIECE - 1) / PCRC_PIECE;
    for (uint32_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        const uint32_t q = t * PCRC_T + tid;
        const uint64_t lo64 = (uint64_t)q * PCRC_PIECE;
        const uint32_t lo = lo64 < L ? (uint32_t)lo64 : L, hi = min(L, lo + PCRC_PIECE);
        W c = 0;
        if constexpr (SLOTS) {
            c = pcrc_slots_piece(T, A, lo, hi);
        } else if (hi - lo == PCRC_PIECE) {
            const uint4* v = (const uint4*)(A.b + lo);
#pragma unroll 4
            for (uint32_t i = 0; i < PCRC_PIECE / 16; i++) {
                const uint4 w = ldg128_stream(v + i);
                c = pcrc_8(T, c, w.x, w.y);
                c = pcrc_8(T, c, w.z, w.w);
            }
        } else {
            c = crc_bytes(T[0], W(0), A.b + lo, hi - lo);
        }
        // tile-local inclusive prefix: after round r a thread at tid >= 2^r holds 2^r full pieces on its right
        s[tid] = c;
        __syncthreads();
        for (uint32_t r = 0, d = 1; d < PCRC_T; r++, d <<= 1) {
            const W a = tid >= d ? s[tid - d] : 0;
            __syncthreads();
            if (a) c ^= crc_mult(crc_x2n<W>(0, 11 + r), a, crc_poly<W>(0));
            s[tid] = c;
            __syncthreads();
        }
        if (q < npieces) A.pin[q] = c;
        if (tid == PCRC_T - 1) A.ttot[t] = c;
        __syncthreads();                                   // s is reused by the next tile
    }
    // the last CTA to finish: exclusive prefixes of the tiles (all full but the batch's last), in place
    __threadfence();
    __syncthreads();
    if (tid == 0) last = atomicAdd(A.done, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return;
    __threadfence();
    volatile W* tt = A.ttot;
    const uint32_t per = (ntiles + PCRC_T - 1) / PCRC_T;
    const uint32_t t0 = min(ntiles, tid * per), t1 = min(ntiles, t0 + per);
    W e = 0;
    for (uint32_t t = t0; t < t1; t++) e = crc_mult(crc_x2n<W>(0, 18), e, crc_poly<W>(0)) ^ tt[t];   // this thread's tiles together
    s[tid] = e;
    __syncthreads();
    for (uint32_t d = 1; d < PCRC_T; d <<= 1) {
        const W a = tid >= d ? s[tid - d] : 0;
        __syncthreads();
        if (tid >= d) e ^= crc_shift(a, (uint64_t)d * per * PCRC_TILE, 0);   // the right operand covers d threads' tiles
        s[tid] = e;
        __syncthreads();
    }
    W x = tid ? s[tid - 1] : 0;                            // raw CRC of [0, first tile of this thread)
    for (uint32_t t = t0; t < t1; t++) {
        const W own = tt[t];
        tt[t] = x;
        x = crc_mult(crc_x2n<W>(0, 18), x, crc_poly<W>(0)) ^ own;
    }
    if (tid == 0) *A.done = 0;
}

// ---------------------------------------------------------------------------------------------------- pcrc_cuts
// out[k] = raw CRC of [0, x_k) of the batch, x_k = first + k * step for k < m, x_m = L.
template <typename W, bool SLOTS>
__global__ void __launch_bounds__(PCRC_CUTS_T) pcrc_cuts_kernel(const __grid_constant__ PcrcIn<W, SLOTS> A, uint32_t L, uint32_t first,
                                                                uint64_t step, uint32_t m, W* out) {
    __shared__ W T[256];
    for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) T[i] = crc_table_entry(i, crc_poly<W>(0));
    __syncthreads();
    const uint32_t k = blockIdx.x * PCRC_CUTS_T + threadIdx.x;
    if (k > m) return;
    const uint32_t u = k < m ? (uint32_t)(first + k * step) : L;
    W c = 0;
    if (u) {
        const uint32_t q = (u - 1) / PCRC_PIECE, t = q / PCRC_T, lq = q % PCRC_T;     // the piece holding byte u - 1
        c = A.ttot[t];
        if (lq) c = crc_shift(c, (uint64_t)lq * PCRC_PIECE, 0) ^ A.pin[q - 1];
        if constexpr (SLOTS) c = pcrc_slots_bytes(T, c, A, q * PCRC_PIECE, u);
        else c = crc_bytes(T, c, A.b + (uint64_t)q * PCRC_PIECE, u - q * PCRC_PIECE);
    }
    out[k] = c;
}

}  // namespace ts
