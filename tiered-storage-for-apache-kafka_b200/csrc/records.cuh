// records.cuh — validation of the Kafka log entries of a segment (TSGPU_FLAG_VALIDATE_RECORDS), on the original bytes of a
// host-buffer transform batch that are already in HBM for compression.
//
// A segment is a sequence of entries `offset i64 | size i32 | ...`, each 12 + size bytes, ending exactly at the segment's end:
//   magic 2 at +16: size >= 49, CRC-32C (Castagnoli) at +17 over [+21, end)        (DefaultRecordBatch.ensureValid)
//   magic 0/1:      size >= 14, CRC-32 (IEEE) at +12 over [+16, end)                (legacy message sets)
// Nothing inside a batch is parsed.  Polynomial index 0 is CRC-32C (magic 2), 1 is CRC-32 (magic 0/1); the GF(2) arithmetic is crc32.cuh.
//
// The work does not follow the length chain hop by hop (a dependent load per entry).  Per batch of L bytes:
//   rec_scan    one thread per 256-byte piece: raw CRC-32C and CRC-32 of the piece (tables in shared memory, 128-bit loads),
//               a tile-local prefix over the 128 pieces of a 32 KiB tile (GF(2) shifts by x^(8*256*2^r)), and the number of
//               candidates in the tile.  A candidate is a position whose header is plausible: magic in {0,1,2}, size at least
//               the minimum, header inside the batch.
//   rec_tiles   one CTA: prefix CRCs of the tiles and exclusive sums of the candidate counts.
//   rec_place   candidate positions, compacted in order.
//   rec_link    per candidate: its entry's CRC (combined from the prefixes when it is long), and its successor, found by binary
//               search; an entry that reaches the batch end or whose successor is not a candidate is a terminal.  Each node
//               holds (next, first failing position on the way).
//   rec_jump    pointer jumping, REC_JUMPS hops per thread per launch, in place: every node ends at its terminal with the first
//               failure of its orbit.  False candidates cost gathers only: just the orbit of the true entry counts.
//   rec_resolve at the drain of the batch, in order: takes the carry of the previous batch (or call), finishes a straddling
//               entry (header bytes, running CRC), looks the entry position up in the orbit table and leaves the verdict and
//               the next carry.  One thread, a few hundred bytes of CRC at most outside the prefixes.
#pragma once
#include "crc32.cuh"

namespace ts {

constexpr uint32_t REC_PIECE = 256;                 // bytes per thread in rec_scan
constexpr uint32_t REC_T = 128;                     // threads per tile CTA
constexpr uint32_t REC_TILE = REC_PIECE * REC_T;    // 32 KiB
constexpr uint32_t REC_TILES_T = 1024;
constexpr uint32_t REC_LINK_T = 256;
constexpr uint32_t REC_JUMPS = 16;                  // hops per node per rec_jump launch: coverage grows 17x per launch
constexpr uint32_t REC_NONE = 0xffffffffu;
constexpr uint32_t REC_TERM = 0x80000000u;          // node index flag: terminal
constexpr uint32_t REC_HDR = 21;                    // header bytes up to the end of the v2 CRC field

enum RecKind : uint32_t { REC_OK = 0, REC_LENGTH = 1, REC_MAGIC = 2, REC_CRC = 3, REC_INTERNAL = 4 };

// The state of a segment between batches and between calls: the public tsgpu_records_cursor (64 bytes, zero = start).
struct RecCarry {
    uint64_t base;       // segment position of the next byte
    uint64_t start;      // open entry: where it starts
    uint64_t end;        // open entry with its whole header: where it ends
    uint32_t run;        // open entry with its whole header: raw CRC of [start + crc_from, base)
    uint32_t stored;     //   ... and the CRC its header stores
    uint8_t open;        // an entry started before `base` and has not ended
    uint8_t hlen;        // header bytes held (REC_HDR: complete)
    uint8_t magic;
    uint8_t pad0;
    uint8_t hdr[REC_HDR];
    uint8_t pad1[3];
};
static_assert(sizeof(RecCarry) == 64, "RecCarry is tsgpu_records_cursor");

struct RecOut {
    uint64_t fail;       // segment position of the first invalid entry, or ~0
    uint32_t kind;       // RecKind
    uint32_t stored, computed;
    int32_t size;
    uint32_t magic, pad;
    RecCarry carry;      // the state after this batch (valid when kind == REC_OK)
};

struct RecArgs {
    const uint8_t* b; uint32_t L;    // the batch's original bytes (256-byte aligned) and their count, L < 2^31
    uint32_t* pin;                   // [2][npieces] raw CRC of [tile start, end of piece q)
    uint32_t* ttot;                  // [2][ntiles]  raw CRC of each tile
    uint32_t* tex;                   // [2][ntiles]  raw CRC of [0, tile start)
    uint32_t* cnt;                   // [ntiles]     candidates per tile
    uint32_t* tbase;                 // [ntiles + 1] exclusive sums of cnt; tbase[ntiles] = number of candidates K
    uint32_t* cpos;                  // [K] candidate positions, ascending
    unsigned long long* node;        // [K] (next index | REC_TERM) low, first failing position high
    uint32_t npieces, ntiles;
};

__device__ __forceinline__ uint32_t rec_be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
// A plausible header at x: what a candidate is.  Needs x + REC_HDR <= L.
__device__ __forceinline__ bool rec_plausible(const uint8_t* b, uint32_t x) {
    const uint32_t m = b[x + 16];
    if (m > 2) return false;
    const int32_t size = (int32_t)rec_be32(b + x + 8);
    return size >= (m == 2 ? 49 : 14);
}

// ---------------------------------------------------------------------------------------------------- rec_scan
__global__ void __launch_bounds__(REC_T) rec_scan_kernel(const __grid_constant__ RecArgs A) {
    __shared__ uint32_t T[2][256];
    __shared__ uint32_t s0[REC_T], s1[REC_T], sc[REC_T];
    crc_tables(T);
    const uint32_t tid = threadIdx.x, q = blockIdx.x * REC_T + tid;
    const uint64_t lo64 = (uint64_t)q * REC_PIECE;
    const uint32_t lo = lo64 < A.L ? (uint32_t)lo64 : A.L, hi = min(A.L, lo + REC_PIECE);
    uint32_t c0 = 0, c1 = 0, n = 0;
    if (hi - lo == REC_PIECE) {
        const uint4* v = (const uint4*)(A.b + lo);
        for (uint32_t i = 0; i < REC_PIECE / 16; i++) {
            const uint4 w = ldg128_stream(v + i);
            const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
            for (int k = 0; k < 4; k++)
                for (int j = 0; j < 4; j++) {
                    const uint32_t byte = (ws[k] >> (8 * j)) & 0xffu;
                    c0 = crc_upd(T[0], c0, byte); c1 = crc_upd(T[1], c1, byte);
                }
        }
    } else {
        for (uint32_t x = lo; x < hi; x++) { c0 = crc_upd(T[0], c0, A.b[x]); c1 = crc_upd(T[1], c1, A.b[x]); }
    }
    const uint32_t last = A.L >= REC_HDR ? A.L - REC_HDR : 0;       // candidates x <= last
    if (A.L >= REC_HDR) for (uint32_t x = lo; x < hi && x <= last; x++) n += rec_plausible(A.b, x) ? 1u : 0u;
    // tile-local inclusive prefix: after round r a thread at tid >= 2^r holds exactly 2^r full pieces on its right
    s0[tid] = c0; s1[tid] = c1; sc[tid] = n;
    __syncthreads();
    for (uint32_t r = 0, d = 1; d < REC_T; r++, d <<= 1) {
        uint32_t a0 = 0, a1 = 0, an = 0;
        if (tid >= d) { a0 = s0[tid - d]; a1 = s1[tid - d]; an = sc[tid - d]; }
        __syncthreads();
        if (tid >= d) {
            c0 ^= a0 ? crc_mult(crc_x2n(0, 11 + r), a0, crc_poly(0)) : 0;
            c1 ^= a1 ? crc_mult(crc_x2n(1, 11 + r), a1, crc_poly(1)) : 0;
            n += an;
        }
        s0[tid] = c0; s1[tid] = c1; sc[tid] = n;
        __syncthreads();
    }
    if (q < A.npieces) { A.pin[q] = c0; A.pin[A.npieces + q] = c1; }
    if (tid == REC_T - 1) {
        A.ttot[blockIdx.x] = c0; A.ttot[A.ntiles + blockIdx.x] = c1;
        A.cnt[blockIdx.x] = n;
    }
}

// ---------------------------------------------------------------------------------------------------- rec_tiles
__global__ void __launch_bounds__(REC_TILES_T) rec_tiles_kernel(const __grid_constant__ RecArgs A) {
    __shared__ uint32_t s0[REC_TILES_T], s1[REC_TILES_T], sc[REC_TILES_T];
    const uint32_t tid = threadIdx.x, nt = A.ntiles;
    const uint32_t per = (nt + REC_TILES_T - 1) / REC_TILES_T;
    const uint32_t t0 = min(nt, tid * per), t1 = min(nt, t0 + per);
    uint32_t e0 = 0, e1 = 0, en = 0;
    for (uint32_t t = t0; t < t1; t++) {              // thread-local exclusive prefix over its tiles (all full but the batch's last)
        A.tex[t] = e0; A.tex[nt + t] = e1; A.tbase[t] = en;
        e0 = crc_mult(crc_x2n(0, 18), e0, crc_poly(0)) ^ A.ttot[t];
        e1 = crc_mult(crc_x2n(1, 18), e1, crc_poly(1)) ^ A.ttot[nt + t];
        en += A.cnt[t];
    }
    s0[tid] = e0; s1[tid] = e1; sc[tid] = en;
    __syncthreads();
    for (uint32_t d = 1; d < REC_TILES_T; d <<= 1) {
        uint32_t a0 = 0, a1 = 0, an = 0;
        if (tid >= d) { a0 = s0[tid - d]; a1 = s1[tid - d]; an = sc[tid - d]; }
        __syncthreads();
        if (tid >= d) {                                // the right operand covers d threads' tiles
            const uint64_t bytes = (uint64_t)d * per * REC_TILE;
            e0 ^= crc_shift(a0, bytes, 0); e1 ^= crc_shift(a1, bytes, 1); en += an;
        }
        s0[tid] = e0; s1[tid] = e1; sc[tid] = en;
        __syncthreads();
    }
    const uint32_t x0 = tid ? s0[tid - 1] : 0, x1 = tid ? s1[tid - 1] : 0, xn = tid ? sc[tid - 1] : 0;
    for (uint32_t t = t0; t < t1; t++) {
        const uint64_t bytes = (uint64_t)(t - t0) * REC_TILE;
        A.tex[t] ^= crc_shift(x0, bytes, 0); A.tex[nt + t] ^= crc_shift(x1, bytes, 1); A.tbase[t] += xn;
    }
    if (tid == REC_TILES_T - 1) A.tbase[nt] = sc[tid];
}

// ---------------------------------------------------------------------------------------------------- rec_place
__global__ void __launch_bounds__(REC_T) rec_place_kernel(const __grid_constant__ RecArgs A) {
    __shared__ uint32_t sc[REC_T];
    const uint32_t tid = threadIdx.x, q = blockIdx.x * REC_T + tid;
    const uint64_t lo64 = (uint64_t)q * REC_PIECE;
    const uint32_t lo = lo64 < A.L ? (uint32_t)lo64 : A.L, hi = min(A.L, lo + REC_PIECE);
    const uint32_t last = A.L >= REC_HDR ? A.L - REC_HDR : 0;
    uint32_t n = 0;
    if (A.L >= REC_HDR) for (uint32_t x = lo; x < hi && x <= last; x++) n += rec_plausible(A.b, x) ? 1u : 0u;
    sc[tid] = n;
    __syncthreads();
    uint32_t incl = n;
    for (uint32_t d = 1; d < REC_T; d <<= 1) {
        const uint32_t a = tid >= d ? sc[tid - d] : 0;
        __syncthreads();
        incl += a; sc[tid] = incl;
        __syncthreads();
    }
    uint32_t k = A.tbase[blockIdx.x] + incl - n;
    if (n) for (uint32_t x = lo; x < hi && x <= last; x++) if (rec_plausible(A.b, x)) A.cpos[k++] = x;
}

// ---------------------------------------------------------------------------------------------------- CRC of a range
// Raw CRC of [0, u) of the batch: the prefix at the start of the piece holding byte u - 1, then at most 256 bytes.
__device__ __forceinline__ uint32_t rec_prefix(const RecArgs& A, const uint32_t* T, int pi, uint32_t u) {
    if (u == 0) return 0;
    const uint32_t q = (u - 1) / REC_PIECE, t = q / REC_T, lq = q % REC_T;     // the piece holding byte u - 1
    uint32_t c = A.tex[pi * A.ntiles + t];
    if (lq) c = crc_shift(c, (uint64_t)lq * REC_PIECE, pi) ^ A.pin[pi * A.npieces + q - 1];
    return crc_bytes(T, c, A.b + (uint64_t)q * REC_PIECE, u - q * REC_PIECE);
}
// Raw CRC (register starting at 0) of [u, v) of the batch.
__device__ __forceinline__ uint32_t rec_raw(const RecArgs& A, const uint32_t* T, int pi, uint32_t u, uint32_t v) {
    if (v - u <= 2 * REC_PIECE) return crc_bytes(T, 0, A.b + u, v - u);
    return rec_prefix(A, T, pi, v) ^ crc_shift(rec_prefix(A, T, pi, u), v - u, pi);
}
// The CRC an entry of magic m at x (ending at e <= L) stores and the one its bytes have.
__device__ __forceinline__ void rec_entry_crc(const RecArgs& A, const uint32_t (*T)[256], uint32_t x, uint32_t e, uint32_t* stored,
                                              uint32_t* computed) {
    const uint32_t m = A.b[x + 16];
    const int pi = m == 2 ? 0 : 1;
    const uint32_t from = x + (m == 2 ? 21 : 16);
    *stored = rec_be32(A.b + x + (m == 2 ? 17 : 12));
    *computed = ~(rec_raw(A, T[pi], pi, from, e) ^ crc_shift(0xffffffffu, e - from, pi));
}

// ---------------------------------------------------------------------------------------------------- rec_link
__global__ void __launch_bounds__(REC_LINK_T) rec_link_kernel(const __grid_constant__ RecArgs A) {
    __shared__ uint32_t T[2][256];
    crc_tables(T);
    const uint32_t K = A.tbase[A.ntiles];
    for (uint32_t k = blockIdx.x * REC_LINK_T + threadIdx.x; k < K; k += gridDim.x * REC_LINK_T) {
        const uint32_t x = A.cpos[k];
        const uint64_t e = (uint64_t)x + 12 + (uint32_t)(int32_t)rec_be32(A.b + x + 8);
        uint32_t fail = REC_NONE;
        if (e <= A.L) {
            uint32_t st, co;
            rec_entry_crc(A, T, x, (uint32_t)e, &st, &co);
            if (st != co) fail = x;
        }
        uint32_t next = k | REC_TERM;                  // reaches the batch end (or its successor's header is cut by it)
        if (e + REC_HDR <= A.L) {
            uint32_t lo = k + 1, hi = K;               // successors lie further on
            while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (A.cpos[mid] < (uint32_t)e) lo = mid + 1; else hi = mid; }
            if (lo < K && A.cpos[lo] == (uint32_t)e) next = lo;
            else fail = min(fail, (uint32_t)e);        // the orbit breaks at e: its header is not plausible
        }
        A.node[k] = (unsigned long long)fail << 32 | next;
    }
}

// ---------------------------------------------------------------------------------------------------- rec_jump
// In place: a node always holds (a node on its orbit, first failure between them), so reading a neighbour that has already
// moved on only helps.  After launch r every node covers at least (REC_JUMPS + 1)^r nodes of its orbit or has reached its end.
__global__ void __launch_bounds__(REC_LINK_T) rec_jump_kernel(const __grid_constant__ RecArgs A) {
    const uint32_t K = A.tbase[A.ntiles];
    for (uint32_t k = blockIdx.x * REC_LINK_T + threadIdx.x; k < K; k += gridDim.x * REC_LINK_T) {
        unsigned long long v = A.node[k];
        uint32_t next = (uint32_t)v, fail = (uint32_t)(v >> 32);
        if (next & REC_TERM) continue;
        for (uint32_t j = 0; j < REC_JUMPS && !(next & REC_TERM); j++) {
            const unsigned long long w = A.node[next];
            next = (uint32_t)w; fail = min(fail, (uint32_t)(w >> 32));
        }
        A.node[k] = (unsigned long long)fail << 32 | next;
    }
}

// ---------------------------------------------------------------------------------------------------- rec_resolve
__device__ __forceinline__ void rec_fail(RecOut& o, uint64_t at, uint32_t kind, const uint8_t* hdr, uint32_t hlen) {
    o.fail = at; o.kind = kind;
    o.magic = hlen > 16 ? hdr[16] : 0xffffffffu;
    o.size = hlen >= 12 ? (int32_t)rec_be32(hdr + 8) : 0;
}
// Classifies an invalid entry at x of the batch (header inside it): magic, size, else its CRC.
__device__ __forceinline__ void rec_fail_at(const RecArgs& A, const uint32_t (*T)[256], RecOut& o, uint64_t base, uint32_t x) {
    const uint8_t* h = A.b + x;
    const uint32_t m = h[16];
    const int32_t size = (int32_t)rec_be32(h + 8);
    rec_fail(o, base + x, REC_CRC, h, REC_HDR);
    if (m > 2) o.kind = REC_MAGIC;
    else if (size < (m == 2 ? 49 : 14) || (uint64_t)x + 12 + (uint32_t)size > A.L) o.kind = REC_LENGTH;
    else rec_entry_crc(A, T, x, x + 12 + (uint32_t)size, &o.stored, &o.computed);
}
// An entry starts at x of the batch: open it in the carry if it reaches past the batch (with as much header as there is).
__device__ __forceinline__ void rec_open(const RecArgs& A, const uint32_t (*T)[256], RecCarry& c, uint32_t x) {
    c.open = 1; c.start = c.base + x;
    c.hlen = (uint8_t)(A.L - x < REC_HDR ? A.L - x : REC_HDR);
    for (uint32_t i = 0; i < c.hlen; i++) c.hdr[i] = A.b[x + i];
    if (c.hlen == REC_HDR) {
        const uint32_t m = c.hdr[16];
        const int pi = m == 2 ? 0 : 1;
        const uint32_t from = x + (m == 2 ? 21 : 16);
        c.magic = (uint8_t)m;
        c.end = c.start + 12 + (uint32_t)(int32_t)rec_be32(c.hdr + 8);
        c.stored = rec_be32(c.hdr + (m == 2 ? 17 : 12));
        c.run = rec_raw(A, T[pi], pi, from, A.L);
    }
}

__global__ void __launch_bounds__(32) rec_resolve_kernel(const __grid_constant__ RecArgs A, const RecCarry in, RecOut* out) {
    __shared__ uint32_t T[2][256];
    crc_tables(T);
    if (threadIdx.x != 0) return;
    RecOut o{};
    o.fail = ~0ull; o.kind = REC_OK;
    RecCarry c = in;
    const uint32_t L = A.L;
    uint32_t p = 0;                                           // where the next entry starts in this batch
    if (c.open) {
        if (c.hlen < REC_HDR) {                               // the header was cut: complete it
            const uint32_t had = c.hlen, take = REC_HDR - had < L ? REC_HDR - had : L;
            for (uint32_t i = 0; i < take; i++) c.hdr[had + i] = A.b[i];
            c.hlen = (uint8_t)(had + take);
            if (c.hlen < REC_HDR) { c.base += L; o.carry = c; *out = o; return; }
            const uint32_t m = c.hdr[16];
            const int32_t size = (int32_t)rec_be32(c.hdr + 8);
            if (m > 2) { rec_fail(o, c.start, REC_MAGIC, c.hdr, REC_HDR); *out = o; return; }
            if (size < (m == 2 ? 49 : 14)) { rec_fail(o, c.start, REC_LENGTH, c.hdr, REC_HDR); *out = o; return; }
            c.magic = (uint8_t)m;
            c.end = c.start + 12 + (uint32_t)size;
            c.stored = rec_be32(c.hdr + (m == 2 ? 17 : 12));
            const uint32_t from = m == 2 ? 21 : 16;            // covered header bytes that came before this batch
            c.run = had > from ? crc_bytes(T[m == 2 ? 0 : 1], 0, c.hdr + from, had - from) : 0;
        }
        const int pi = c.magic == 2 ? 0 : 1;
        const uint64_t crc_from = c.start + (c.magic == 2 ? 21 : 16);
        const uint32_t from = crc_from > c.base ? (uint32_t)(crc_from - c.base) : 0;
        const uint32_t to = c.end - c.base < L ? (uint32_t)(c.end - c.base) : L;
        if (to > from) c.run = crc_shift(c.run, to - from, pi) ^ rec_raw(A, T[pi], pi, from, to);
        if (c.end - c.base > L) { c.base += L; o.carry = c; *out = o; return; }
        const uint32_t computed = ~(c.run ^ crc_shift(0xffffffffu, c.end - crc_from, pi));
        if (computed != c.stored) {
            rec_fail(o, c.start, REC_CRC, c.hdr, REC_HDR); o.stored = c.stored; o.computed = computed;
            *out = o; return;
        }
        c.open = 0;
        p = (uint32_t)(c.end - c.base);
    }
    if (p + REC_HDR > L) {                                    // the batch ends at p or inside the next header
        if (p < L) rec_open(A, T, c, p);
        c.base += L; o.carry = c; *out = o; return;
    }
    const uint32_t K = A.tbase[A.ntiles];
    uint32_t lo = 0, hi = K;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (A.cpos[mid] < p) lo = mid + 1; else hi = mid; }
    if (lo == K || A.cpos[lo] != p) { rec_fail_at(A, T, o, c.base, p); *out = o; return; }
    const unsigned long long v = A.node[lo];
    const uint32_t root = (uint32_t)v, fail = (uint32_t)(v >> 32);
    if (!(root & REC_TERM)) { o.fail = c.base + p; o.kind = REC_INTERNAL; *out = o; return; }
    if (fail != REC_NONE) { rec_fail_at(A, T, o, c.base, fail); *out = o; return; }
    const uint32_t x = A.cpos[root & ~REC_TERM];
    const uint64_t e = (uint64_t)x + 12 + (uint32_t)(int32_t)rec_be32(A.b + x + 8);
    if (e > L) rec_open(A, T, c, x);
    else if (e < L) rec_open(A, T, c, (uint32_t)e);
    c.base += L; o.carry = c; *out = o;
}

}  // namespace ts
