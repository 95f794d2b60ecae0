// zstd_dec.cuh — batched Zstandard decompression for sm_90a (kernel K2 of SURVEY.md §2a).
//
// Replaces Zstd.decompressedSize + Zstd.decompress as called per chunk from
//   core/M/transform/DecompressionChunkEnumeration.java:38-46
// (Frame_Content_Size is mandatory there: a frame without it is "Invalid decompressed size").
// Must read frames written by libzstd level 3 (the reference's writer): Raw/RLE/Compressed blocks,
// Huffman literals (1 or 4 streams, direct or FSE-compressed weights, treeless reuse), FSE sequences in
// Predefined/RLE/Compressed/Repeat modes, repeat offsets, matches reaching into earlier blocks.
//
// Three kernels per batch:
//   zstd_dec_index_kernel    one warp per chunk: frame header, Frame_Content_Size, block offsets; marks frames
//                            whose block structure matches this library's writer (ceil(FCS / ZB), ZB = 8 KiB blocks)
//   zstd_dec_blocks_kernel   fast path, one warp PER BLOCK of such frames (131,072 independent units per GiB);
//                            every assumption (block regenerates exactly ZB bytes, no offset before the block, no
//                            repeat offsets/tables carried in) is verified while decoding, and a violation only
//                            flags the frame for the general path — correctness never depends on the guess
//   zstd_dec_frames_kernel   general path, one warp per frame walking its blocks in order (what libzstd frames need)
// Inside a block: lane 0 parses headers and builds tables in shared memory, lanes 0-3 decode the Huffman
// streams, lane 0 decodes sequences 32 at a time into shared memory, all 32 lanes execute them.
#pragma once
#include "ts_common.cuh"
#include "rt.h"
#include "launch_prof.h"
#include "zstd_format.h"
#include "zstd_enc.cuh"
#include "zstd_enc_blk.cuh"

namespace ts {

constexpr int ZD_WPB = 4;
constexpr uint32_t ZD_ST_OK = 0, ZD_ST_CORRUPT = 2;
constexpr uint32_t ZD_LIT_GENERAL = zf::BLOCK_MAX + 64;

struct ZdWarpCtx {                        // per-warp shared-memory working set (~16 KiB)
    uint16_t huf[1 << zf::HUF_MAX_LOG];   // symbol | nbits << 8
    zf::FseDEntry ll[1 << zf::LL_MAX_LOG];
    zf::FseDEntry ml[1 << zf::ML_MAX_LOG];
    zf::FseDEntry of[1 << zf::OF_MAX_LOG];
    uint32_t s_ll[32], s_ml[32], s_off[32];
    uint8_t symbol_of[512];
    uint16_t next[64];
    int16_t norm[64];
    int16_t norm3[3][64];                 // FSE_Compressed tables waiting for the warp-parallel build
    uint32_t pend_log[3], pend_nsym[3];
    uint32_t cum[65];
    uint16_t hstart[256];                 // first table cell of each Huffman symbol (filled by all lanes)
    uint32_t huf_nw;
    uint8_t weights[256];
    zf::FseDEntry wt[1 << zf::HUFW_MAX_LOG];
    uint32_t rank_start[16];
    uint32_t huf_log, ll_log, ml_log, of_log;
    uint32_t huf_valid, ll_valid, ml_valid, of_valid;
    uint32_t rep[3];
    int32_t err;                          // 0 ok, <0 corrupt, >0 "needs the general path"
    uint32_t tmp[8];
    static constexpr int kTabLogCap = 9;  // largest FSE table this context holds
};

struct ZstdDecScratch {
    uint32_t* blk_off = nullptr;     // n_chunks * (blocks_per_chunk + 1)
    uint32_t* info = nullptr;        // n_chunks * 8: fcs, nblk, eligible, need_general, first_block_off, ...
    uint8_t* lits_general = nullptr; // n_chunks * ZD_LIT_GENERAL
    uint64_t* pos_tmp = nullptr;     // n_chunks + 1
    uint32_t blocks_per_chunk = 0, max_batch = 0, chunk_cap = 0;
    // per-block results of the entropy stage + per-frame arenas
    uint8_t* par_meta = nullptr;     // n_chunks * blocks_per_chunk * sizeof(ZdBlkMeta)
    uint8_t* par_lits = nullptr;     // n_chunks * par_lit_cap
    uint64_t* par_seqs = nullptr;    // n_chunks * par_seq_cap
    uint32_t par_lit_cap = 0, par_seq_cap = 0;
    unsigned long long* stats = nullptr;   // [0] regions executed in shared memory, [1] frames sent to the frame executor after a
                                           // region / block refused, [2] frames executed whole (libzstd-shaped), [3] frames on the serial
                                           // kernel, [4] independent blocks executed by a warp each
};

struct ZstdDecArgs {
    const uint8_t* in_base; const uint64_t* in_off; const uint32_t* in_len;
    uint8_t* out_base; const uint64_t* out_off; uint32_t* out_len; uint32_t* status;
    uint32_t* blk_off; uint32_t* info; uint8_t* lits_general;
    uint32_t blocks_per_chunk, chunk_cap, n_chunks;
    uint32_t in_cap;                 // bytes a frame can occupy in its input slot: a longer in_len (device-resident, untrusted) is corrupt
    uint8_t* par_meta; uint8_t* par_lits; uint64_t* par_seqs; uint32_t par_lit_cap, par_seq_cap;
    unsigned long long* stats;
};
constexpr int ZD_INFO = 12;    // fcs, nblk, region-path eligible, state bits (1 executor refused -> frame executor, 2 failed, 4 independent-
                               // block entropy stage refused), header size, parallel-general, literal bump, sequence bump, [8] independent-block guess

// ------------------------------------------------------------------------------------------ bit readers
__device__ __forceinline__ uint64_t zd_ld64(const uint8_t* p) {          // unaligned little-endian 64-bit window
    uintptr_t a = (uintptr_t)p;
    const uint32_t* w = (const uint32_t*)(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3) * 8;
    const uint32_t w0 = w[0], w1 = w[1];
    if (sh == 0) return (uint64_t)w1 << 32 | w0;
    const uint32_t w2 = w[2];
    return (uint64_t)__funnelshift_r(w1, w2, sh) << 32 | __funnelshift_r(w0, w1, sh);
}
// Backward stream (FSE / Huffman): `bits` unread bits remain below the end mark.  A 64-bit window of the stream
// (bits [cbase, cbase+64), cbase a multiple of 8) is cached in registers and refilled about once per 57 bits.
struct ZdBack { const uint8_t* p; int32_t bits; uint64_t C; int32_t cbase; };
__device__ __forceinline__ bool zd_back_init(ZdBack& b, const uint8_t* p, uint32_t size) {
    b.p = p; b.bits = 0; b.C = 0; b.cbase = 0x3fffffff;
    if (size == 0) return false;
    const uint32_t last = p[size - 1];
    if (last == 0) return false;
    b.bits = (int32_t)(size - 1) * 8 + zf::highbit32(last);
    return true;
}
// peek nb (<= 32) bits below the cursor without consuming; zero-extends past the start of the stream
__device__ __forceinline__ uint32_t zd_back_peek(ZdBack& b, uint32_t nb) {
    if (nb == 0) return 0;
    const int32_t lo = b.bits - (int32_t)nb;
    if (lo >= 0) {
        if (lo < b.cbase || b.bits > b.cbase + 64) {
            b.cbase = max(0, ((b.bits + 7) & ~7) - 64);
            b.C = zd_ld64(b.p + (b.cbase >> 3));
        }
        return (uint32_t)(b.C >> (lo - b.cbase)) & (uint32_t)((1ull << nb) - 1);
    }
    if (b.bits <= 0) return 0;
    const uint32_t have = (uint32_t)b.bits;
    const uint32_t v = (uint32_t)zd_ld64(b.p) & (uint32_t)((1ull << have) - 1);
    return v << (nb - have);
}
__device__ __forceinline__ uint32_t zd_back_read(ZdBack& b, uint32_t nb) {
    const uint32_t v = zd_back_peek(b, nb);
    b.bits -= (int32_t)nb;
    return v;
}
// stateless: bits [end - nb, end) of a backward stream, nb <= 32, end - nb >= 0
__device__ __forceinline__ uint32_t zd_bits_at(const uint8_t* p, int32_t end, uint32_t nb) {
    if (nb == 0) return 0;
    const int32_t base = max(0, ((end + 7) & ~7) - 64);
    const uint64_t C = zd_ld64(p + (base >> 3));
    return (uint32_t)(C >> (end - (int32_t)nb - base)) & (uint32_t)((1ull << nb) - 1);
}
// Forward LSB-first reader for FSE table descriptions
struct ZdFwd { const uint8_t* p; uint32_t size; uint32_t bit; };
__device__ __forceinline__ uint32_t zd_fwd_peek(const ZdFwd& f, uint32_t nb) {
    const uint32_t byte = f.bit >> 3;
    uint64_t v = 0;
    for (uint32_t k = 0; k < 5; k++) if (byte + k < f.size) v |= (uint64_t)f.p[byte + k] << (8 * k);
    return (uint32_t)(v >> (f.bit & 7)) & (uint32_t)((1ull << nb) - 1);
}

// ------------------------------------------------------------------------------------------ table readers (one lane)
// FSE_readNCount: normalized counts of an FSE table description.  Returns bytes consumed, 0 on error.
__device__ TS_NOINLINE uint32_t zd_read_ncount(const uint8_t* src, uint32_t size, int16_t* norm, int max_sym, int max_log,
                                               uint32_t* out_log, int* out_nsym) {
    if (size < 1) return 0;
    ZdFwd f{src, size, 0};
    const int log = (int)zd_fwd_peek(f, 4) + 5; f.bit += 4;
    if (log > max_log) return 0;
    int remaining = (1 << log) + 1, threshold = 1 << log, nb = log + 1;
    int sym = 0;
    bool prev0 = false;
    while (remaining > 1 && sym <= max_sym) {
        if (prev0) {
            int n0 = sym;
            while (true) {
                const uint32_t r = zd_fwd_peek(f, 2); f.bit += 2;
                n0 += (int)r;
                if (r != 3) break;
                if (f.bit > size * 8) return 0;
            }
            if (n0 > max_sym + 1) return 0;
            while (sym < n0) norm[sym++] = 0;
            if (sym > max_sym) break;
        }
        const int mx = (2 * threshold - 1) - remaining;
        int count;
        const uint32_t bitsv = zd_fwd_peek(f, (uint32_t)nb);
        if ((int)(bitsv & (uint32_t)(threshold - 1)) < mx) { count = (int)(bitsv & (uint32_t)(threshold - 1)); f.bit += (uint32_t)(nb - 1); }
        else { count = (int)(bitsv & (uint32_t)(2 * threshold - 1)); if (count >= threshold) count -= mx; f.bit += (uint32_t)nb; }
        count--;
        remaining -= count < 0 ? -count : count;
        norm[sym++] = (int16_t)count;
        prev0 = count == 0;
        while (remaining < threshold) { nb--; threshold >>= 1; }
        if (f.bit > size * 8 + 7) return 0;
    }
    if (remaining != 1 || sym > max_sym + 1) return 0;
    *out_log = (uint32_t)log; *out_nsym = sym;
    const uint32_t used = (f.bit + 7) >> 3;
    return used <= size ? used : 0;
}

// Huffman tree description -> decoding table.  Returns bytes consumed, 0 on error.  One lane.
template <class CX> __device__ TS_NOINLINE uint32_t zd_read_huf_table(const uint8_t* src, uint32_t size, CX* cx) {
    if (size < 1) return 0;
    const uint32_t hb = src[0];
    uint32_t nw = 0, used = 0;
    uint8_t* W = cx->weights;
    if (hb >= 128) {                                    // direct 4-bit weights
        nw = hb - 127;
        used = 1 + (nw + 1) / 2;
        if (used > size) return 0;
        for (uint32_t i = 0; i < nw; i++) W[i] = (i & 1) ? (src[1 + i / 2] & 15) : (src[1 + i / 2] >> 4);
    } else {                                            // FSE-compressed weights, two interleaved states
        if (hb == 0 || 1 + hb > size) return 0;
        used = 1 + hb;
        uint32_t log; int nsym;
        const uint32_t h = zd_read_ncount(src + 1, hb, cx->norm, 12, zf::HUFW_MAX_LOG, &log, &nsym);
        if (!h) return 0;
        // weight-decoding table: next_base / nb_bits / symbol in nb_extra
        zf::fse_spread(cx->norm, nsym, (int)log, cx->symbol_of, cx->next);
        zf::FseDEntry* T = cx->wt;
        for (uint32_t u = 0; u < (1u << log); u++) {
            const int s = cx->symbol_of[u];
            const uint32_t ns = cx->next[s]++;
            const int nb = (int)log - zf::highbit32(ns);
            zf::FseDEntry e{};
            e.nb_bits = (uint32_t)nb; e.next_base = (ns << nb) - (1u << log); e.nb_extra = (uint32_t)s;
            T[u] = e;
        }
        ZdBack b;
        if (!zd_back_init(b, src + 1 + h, hb - h)) return 0;
        uint32_t s1 = zd_back_read(b, log), s2 = zd_back_read(b, log);
        if (b.bits < 0) return 0;
        while (true) {
            if (nw >= 254) return 0;
            W[nw++] = T[s1].nb_extra;
            if ((int32_t)T[s1].nb_bits > b.bits) { W[nw++] = T[s2].nb_extra; break; }
            s1 = T[s1].next_base + zd_back_read(b, T[s1].nb_bits);
            if (nw >= 254) return 0;
            W[nw++] = T[s2].nb_extra;
            if ((int32_t)T[s2].nb_bits > b.bits) { W[nw++] = T[s1].nb_extra; break; }
            s2 = T[s2].next_base + zd_back_read(b, T[s2].nb_bits);
        }
    }
    // implied last weight
    uint32_t total = 0;
    for (uint32_t i = 0; i < nw; i++) { if (W[i] > zf::HUF_MAX_LOG) return 0; total += W[i] ? 1u << (W[i] - 1) : 0; }
    if (total == 0) return 0;
    const uint32_t max_bits = (uint32_t)zf::highbit32(total) + 1;
    if (max_bits > zf::HUF_MAX_LOG) return 0;
    const uint32_t rest = (1u << max_bits) - total;
    if (rest & (rest - 1)) return 0;                    // must be a power of two
    W[nw++] = (uint8_t)(zf::highbit32(rest) + 1);
    // rank starts: weight-w symbols occupy 2^(w-1) consecutive cells each, lowest weights first
    uint32_t cnt[16];
    for (int w = 0; w < 16; w++) cnt[w] = 0;
    for (uint32_t i = 0; i < nw; i++) cnt[W[i]]++;
    if (cnt[1] < 2 || (cnt[1] & 1)) return 0;
    uint32_t start = 0;
    for (uint32_t w = 1; w <= max_bits; w++) { cx->rank_start[w] = start; start += cnt[w] << (w - 1); }
    if (start != (1u << max_bits)) return 0;
    for (uint32_t s = 0; s < nw; s++) {
        const uint32_t w = W[s];
        if (!w) continue;
        cx->hstart[s] = (uint16_t)cx->rank_start[w];
        cx->rank_start[w] += 1u << (w - 1);
    }
    cx->huf_log = max_bits; cx->huf_valid = 1; cx->huf_nw = nw;
    return used;
}
// All lanes: fill the decoding table from the per-symbol start cells computed above.
template <class CX> __device__ __forceinline__ void zd_fill_huf_warp(CX* cx, uint32_t lane) {
    const uint32_t nw = cx->huf_nw, max_bits = cx->huf_log;
    for (uint32_t s = 0; s < nw; s++) {
        const uint32_t w = cx->weights[s];
        if (!w) continue;
        const uint32_t len = 1u << (w - 1), at = cx->hstart[s];
        const uint16_t e = (uint16_t)(s | ((max_bits + 1 - w) << 8));
        for (uint32_t k = lane; k < len; k += 32) cx->huf[at + k] = e;
    }
    __syncwarp();
}

// One Huffman stream: `count` symbols from src[0..size) into dst.  Any lane; returns false on corruption.
__device__ __forceinline__ bool zd_huf_stream(const uint16_t* __restrict__ huf, uint32_t log, const uint8_t* src, uint32_t size,
                                              uint8_t* dst, uint32_t count) {
    ZdBack b;
    if (!zd_back_init(b, src, size)) return false;
    for (uint32_t i = 0; i < count; i++) {
        const uint16_t e = huf[zd_back_peek(b, log)];
        dst[i] = (uint8_t)e;
        b.bits -= (int32_t)(e >> 8);
        if (b.bits < 0) return false;
    }
    return b.bits == 0;
}

// Sequence table of one kind according to its compression mode.  Lane 0.  Returns bytes consumed, -1 on error.
// Warp-parallel build of a sequence decoding table whose distribution has no "less than one" symbols (what this
// library's writer emits): the spread then has the closed form pos(i) = i*step & mask, a cell's symbol is found by
// binary search in the cumulative counts, and cells of a symbol are numbered in position order with match_any.
template <class CX> __device__ __forceinline__ void zd_build_dtable_warp(int kind, CX* cx, uint32_t lane) {
    zf::FseDEntry* T = kind == 0 ? cx->ll : kind == 1 ? cx->of : cx->ml;
    const int16_t* nm = cx->norm3[kind];
    const uint32_t log = cx->pend_log[kind], nsym = cx->pend_nsym[kind];
    const uint32_t size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    const uint32_t p0 = lane < nsym ? (uint32_t)nm[lane] : 0u, p1 = lane + 32 < nsym ? (uint32_t)nm[lane + 32] : 0u;
    const uint32_t inc0 = warp_inclusive_scan_u32(p0, lane);
    const uint32_t inc1 = warp_inclusive_scan_u32(p1, lane) + __shfl_sync(TS_FULL, inc0, 31);
    cx->cum[lane] = inc0 - p0; cx->cum[32 + lane] = inc1 - p1;
    if (lane == 0) cx->cum[64] = size;
    cx->next[lane] = (uint16_t)p0; cx->next[32 + lane] = (uint16_t)p1;
    __syncwarp();
    for (uint32_t i = lane; i < size; i += 32) {
        uint32_t lo = 0, hi = 64;
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (cx->cum[mid] <= i) lo = mid; else hi = mid; }
        cx->symbol_of[(i * step) & mask] = (uint8_t)lo;
    }
    __syncwarp();
    for (uint32_t u0 = 0; u0 < size; u0 += 32) {
        const uint32_t u = u0 + lane;
        const uint32_t sym = cx->symbol_of[u];
        const uint32_t same = __match_any_sync(TS_FULL, sym);
        const uint32_t rank = (uint32_t)__popc(same & ((1u << lane) - 1));
        const uint32_t base = cx->next[sym];
        const uint32_t ns = base + rank;
        const int nb = (int)log - zf::highbit32(ns);
        zf::FseDEntry e{};
        e.nb_bits = (uint32_t)nb;
        e.next_base = (ns << nb) - size;
        e.sym = sym;
        e.nb_extra = kind == 0 ? g_seq_tables.ll_bits[sym] : kind == 2 ? g_seq_tables.ml_bits[sym] : sym;
        T[u] = e;
        __syncwarp();
        if (rank == 0) cx->next[sym] = (uint16_t)(base + (uint32_t)__popc(same));
        __syncwarp();
    }
}

template <class CX> __device__ TS_NOINLINE int32_t zd_seq_table(uint32_t mode, int kind, const uint8_t* src, uint32_t size, CX* cx, bool fast_nonfirst, uint32_t* pending) {
    zf::FseDEntry* T = kind == 0 ? cx->ll : kind == 1 ? cx->of : cx->ml;
    uint32_t* logp = kind == 0 ? &cx->ll_log : kind == 1 ? &cx->of_log : &cx->ml_log;
    uint32_t* validp = kind == 0 ? &cx->ll_valid : kind == 1 ? &cx->of_valid : &cx->ml_valid;
    const int max_sym = kind == 0 ? 35 : kind == 1 ? 31 : 52;
    const int fmt_log = kind == 0 ? zf::LL_MAX_LOG : kind == 1 ? zf::OF_MAX_LOG : zf::ML_MAX_LOG;
    const int max_log = fmt_log < CX::kTabLogCap ? fmt_log : CX::kTabLogCap;      // (a lean context refuses larger tables)
    if (mode == 0) {                                    // Predefined_Mode
        const int16_t* nm = kind == 0 ? g_seq_tables.ll_norm : kind == 1 ? g_seq_tables.of_norm : g_seq_tables.ml_norm;
        const int ns = kind == 0 ? 36 : kind == 1 ? 29 : 53;
        const int lg = kind == 0 ? zf::LL_DEFAULT_LOG : kind == 1 ? zf::OF_DEFAULT_LOG : zf::ML_DEFAULT_LOG;
        zf::fse_build_dtable(nm, ns, lg, kind, g_seq_tables, T, cx->symbol_of, cx->next);
        *logp = (uint32_t)lg; *validp = 1;
        return 0;
    }
    if (mode == 1) {                                    // RLE_Mode
        if (size < 1 || src[0] > max_sym) return -1;
        zf::fse_build_rle(src[0], kind, g_seq_tables, T);
        *logp = 0; *validp = 1;
        return 1;
    }
    if (mode == 2) {                                    // FSE_Compressed_Mode
        uint32_t lg; int ns;
        int16_t* nm = cx->norm3[kind];
        const uint32_t h = zd_read_ncount(src, size, nm, max_sym, max_log, &lg, &ns);
        if (!h) return -1;
        bool low = false;
        for (int q = 0; q < ns; q++) low |= nm[q] < 0;
        if (low) zf::fse_build_dtable(nm, ns, (int)lg, kind, g_seq_tables, T, cx->symbol_of, cx->next);   // libzstd-style table: serial
        else { cx->pend_log[kind] = lg; cx->pend_nsym[kind] = (uint32_t)ns; *pending |= 1u << kind; }  // built by all lanes later
        *logp = lg; *validp = 1;
        return (int32_t)h;
    }
    // Repeat_Mode: the previous block's table of this kind
    if (fast_nonfirst) { cx->err = 1; return 0; }
    return *validp ? 0 : -1;
}

// 3-byte Block_Header (RFC 8878 §3.1.1.2).
struct ZdBlkHdr { uint32_t last, type, size; };
__device__ __forceinline__ ZdBlkHdr zd_block_header(const uint8_t* p) {
    const uint32_t h = p[0] | (p[1] << 8) | ((uint32_t)p[2] << 16);
    return ZdBlkHdr{h & 1, (h >> 1) & 3, h >> 3};
}

// Literals section of a Compressed_Block: type, header size, Regenerated_Size, Compressed_Size (Raw: the bytes, RLE: 1,
// Compressed / Treeless: the streams, a Huffman tree description included), streams, tree-description bytes.
struct ZdLitSec { uint32_t type, hs, regen, comp, streams, tree; };
// Field decode of the Literals_Section_Header (tree = 0).  hs = 0: the block is too short to hold the header.
__device__ __forceinline__ ZdLitSec zd_lit_section(const uint8_t* blk, uint32_t bsize) {
    ZdLitSec L{0, 0, 0, 0, 1, 0};
    if (bsize < 2) return L;                            // Compressed_Block needs at least literals header + seq header
    const uint32_t b0 = blk[0], sf = (b0 >> 2) & 3;
    L.type = b0 & 3;
    if (L.type < 2) {
        if ((sf & 1) == 0) { L.hs = 1; L.regen = b0 >> 3; }
        else if (sf == 1) { L.hs = 2; L.regen = (b0 >> 4) | ((uint32_t)blk[1] << 4); }
        else { if (bsize < 3) return L; L.hs = 3; L.regen = (b0 >> 4) | ((uint32_t)blk[1] << 4) | ((uint32_t)blk[2] << 12); }
        L.comp = L.type == 0 ? L.regen : 1;
    } else {
        if (bsize < 5) return L;
        const uint32_t h = blk[0] | ((uint32_t)blk[1] << 8) | ((uint32_t)blk[2] << 16) | ((uint32_t)blk[3] << 24);
        if (sf <= 1) { L.hs = 3; L.regen = (h >> 4) & 0x3ff; L.comp = (h >> 14) & 0x3ff; L.streams = sf == 0 ? 1 : 4; }
        else if (sf == 2) { L.hs = 4; L.regen = (h >> 4) & 0x3fff; L.comp = h >> 18; L.streams = 4; }
        else { L.hs = 5; L.regen = (h >> 4) & 0x3ffff; L.comp = (h >> 22) | ((uint32_t)blk[4] << 10); L.streams = 4; }
    }
    return L;
}

// Literals_Section_Header of a Compressed_Block, one lane; a Huffman tree description is read into cx.  false: malformed.
// Treeless literals with no_inherit set cx->err = 1 ("needs the general path") and still return true.
template <class CX> __device__ __forceinline__ bool zd_parse_lit_header(const uint8_t* blk, uint32_t bsize, uint32_t limit, uint32_t litcap,
                                                                        bool no_inherit, CX* cx, ZdLitSec& L) {
    L = zd_lit_section(blk, bsize);
    if (!L.hs || L.hs + L.comp > bsize || L.regen > limit || L.regen > zf::BLOCK_MAX) return false;
    if (L.type >= 2 && L.regen > litcap) return false;
    if (L.type == 2) {
        L.tree = zd_read_huf_table(blk + L.hs, L.comp, cx);
        if (!L.tree) return false;
    } else if (L.type == 3) {
        if (no_inherit) { cx->err = 1; }
        else if (!cx->huf_valid) return false;
    }
    return true;
}

// Stream k (0..3) of a 4-stream Huffman literals section src[0..size) of `regen` symbols: where its bytes start (past the
// 6-byte jump table), how many there are, its first symbol and its symbol count.  false: the jump table does not fit.
struct ZdHufStream { uint32_t off, size, first, count; };
__device__ __forceinline__ bool zd_huf4_stream(const uint8_t* src, uint32_t size, uint32_t regen, uint32_t k, ZdHufStream& s) {
    if (size < 10) return false;
    const uint32_t s1 = src[0] | (src[1] << 8), s2 = src[2] | (src[3] << 8), s3 = src[4] | (src[5] << 8);
    if (6 + s1 + s2 + s3 > size) return false;
    const uint32_t s4 = size - 6 - s1 - s2 - s3;
    const uint32_t per = (regen + 3) / 4;
    s.off = 6 + (k == 0 ? 0 : k == 1 ? s1 : k == 2 ? s1 + s2 : s1 + s2 + s3);
    s.size = k == 0 ? s1 : k == 1 ? s2 : k == 2 ? s3 : s4;
    s.first = k * per;
    if (s.first > regen || (k == 3 && 3 * per > regen)) return false;
    s.count = k < 3 ? min(per, regen - s.first) : regen - s.first;
    return true;
}

// Sequences_Section_Header, one lane: Number_of_Sequences, the modes byte and the three tables (serial builds happen here,
// FSE_Compressed tables without "less than one" symbols are left pending for the warp).  out: nseq, bytes before the bit
// stream, pending mask.  false: malformed.  Repeat_Mode with no_inherit sets cx->err = 1.
template <class CX> __device__ __forceinline__ bool zd_parse_seq_header(const uint8_t* sp, uint32_t ssize, bool no_inherit, CX* cx, uint32_t* out) {
    if (ssize < 1) return false;
    uint32_t nseq = sp[0], hs = 1;
    if (nseq >= 128) {
        if (nseq == 255) { if (ssize < 3) return false; nseq = sp[1] + ((uint32_t)sp[2] << 8) + 0x7f00; hs = 3; }
        else { if (ssize < 2) return false; nseq = ((nseq - 128) << 8) + sp[1]; hs = 2; }
    }
    uint32_t pos = hs, pend = 0;
    if (nseq) {
        if (ssize < hs + 1) return false;
        const uint32_t modes = sp[hs];
        if (modes & 3) return false;                    // reserved bits
        pos = hs + 1;
        const uint32_t m3[3] = { modes >> 6, (modes >> 4) & 3, (modes >> 2) & 3 };   // LL, OF, ML
        for (int k = 0; k < 3; k++) {
            const int32_t used = zd_seq_table(m3[k], k, sp + pos, ssize - pos, cx, no_inherit, &pend);
            if (used < 0) return false;
            pos += (uint32_t)used;
        }
        if (pos > ssize) return false;
    }
    out[0] = nseq; out[1] = pos; out[2] = pend;
    return true;
}

// ------------------------------------------------------------------------------------------ sequence words of the arenas
// Sequence word of the arenas: bits 0..29 offset field, 30..46 literal length, 47..63 match length - 3.
// Offset field: a concrete offset (< 2^29), or — when the sequence used a repeat offset that reaches back to the state the
// block STARTED with, which the entropy stage cannot know — bit 29 set, bits 27..28 = which of the three initial repeat
// offsets (1..3), bits 0..26 = how much was subtracted from it (the "rep1 - 1" form, RFC 8878 §3.1.1.5).
constexpr uint32_t ZD_OFF_SYM = 1u << 29;
constexpr uint32_t ZD_SYM_D = (1u << 27) - 1;
// Does a sequence (offset value ofv as decoded: <= 3 a repeat code) fit the word?
__device__ __forceinline__ bool zd_seq_fits(uint32_t ofv, uint32_t ll, uint32_t ml) {
    return (ofv <= 3 || ofv - 3 < ZD_OFF_SYM) && ll < (1u << 17) && ml - 3 < (1u << 17);
}
__device__ __forceinline__ uint64_t zd_seq_pack(uint32_t of, uint32_t ll, uint32_t ml) {
    return (uint64_t)of | ((uint64_t)ll << 30) | ((uint64_t)(ml - 3) << 47);
}
__device__ __forceinline__ void zd_seq_unpack(uint64_t v, uint32_t& of, uint32_t& ll, uint32_t& ml) {
    of = (uint32_t)v & (2 * ZD_OFF_SYM - 1);
    ll = (uint32_t)(v >> 30) & 0x1ffffu; ml = (uint32_t)(v >> 47) + 3;
}
// The repeat offset k (1..3) a block starts with, as a symbol.
__device__ __forceinline__ uint32_t zd_sym_rep(uint32_t k) { return ZD_OFF_SYM | (k << 27); }
// A symbolic offset field against the repeat offsets R0..R2 its block started with: returns the one it names, *d what was
// subtracted from it.  The offset is that minus *d, which only exists when it is larger than *d.
__device__ __forceinline__ uint32_t zd_sym_base(uint32_t of, uint32_t R0, uint32_t R1, uint32_t R2, uint32_t* d) {
    const uint32_t k = (of >> 27) & 3;
    *d = of & ZD_SYM_D;
    return k == 1 ? R0 : k == 2 ? R1 : R2;
}
__device__ __forceinline__ uint32_t zd_rep_sub1(uint32_t v) {            // "rep1 - 1" on an offset field; 0 = invalid
    if (v & ZD_OFF_SYM) return (v & ZD_SYM_D) == ZD_SYM_D ? 0u : v + 1;   // symbolic: one more subtracted
    return v - 1;                                                        // concrete: 0 when the offset was 1 (corrupt)
}

// ------------------------------------------------------------------------------------------ stages of a compressed block
// Warp-uniform.  Each stage returns false where the block cannot go on: cx->err is then set (<0 corrupt, >0 needs another
// path), the warp agrees on it and the caller returns.

// Literals section header (lane 0 parses, the warp shares it through cx->tmp); a Huffman tree description is read into cx.
__device__ __forceinline__ bool zd_stage_lit_header(const uint8_t* blk, uint32_t bsize, uint32_t limit, ZdWarpCtx* cx, uint32_t lane,
                                                    ZdLitSec& L) {
    if (lane == 0) {
        ZdLitSec h;
        if (zd_parse_lit_header(blk, bsize, limit, zf::BLOCK_MAX, false, cx, h)) {
            cx->tmp[1] = h.type; cx->tmp[2] = h.hs; cx->tmp[3] = h.regen; cx->tmp[4] = h.comp; cx->tmp[5] = h.streams; cx->tmp[6] = h.tree;
            cx->tmp[0] = 1u;
        } else cx->tmp[0] = 0u;
    }
    __syncwarp();
    if (!cx->tmp[0]) { if (lane == 0 && cx->err == 0) cx->err = -1; __syncwarp(); return false; }
    if (cx->err) return false;
    L = ZdLitSec{cx->tmp[1], cx->tmp[2], cx->tmp[3], cx->tmp[4], cx->tmp[5], cx->tmp[6]};
    return true;
}

// Where the literals come from: bytes (Raw in the block, Huffman decoded into litbuf by lanes 0-3) or a single RLE byte.
struct ZdLitSrc { const uint8_t* lit; uint32_t rle_lit; };      // rle_lit 0x100: not RLE
__device__ __forceinline__ bool zd_stage_lit_source(const uint8_t* blk, const ZdLitSec& L, ZdWarpCtx* cx, uint8_t* litbuf,
                                                    uint32_t lane, ZdLitSrc& src) {
    src.lit = nullptr; src.rle_lit = 0x100;
    if (L.type == 0) src.lit = blk + L.hs;
    else if (L.type == 1) src.rle_lit = blk[L.hs];
    else {
        if (L.type == 2) zd_fill_huf_warp(cx, lane);
        const uint8_t* hsrc = blk + L.hs + L.tree;
        const uint32_t hsize = L.comp - L.tree;
        bool ok = true;
        if (L.streams == 1) {
            if (lane == 0) ok = zd_huf_stream(cx->huf, cx->huf_log, hsrc, hsize, litbuf, L.regen);
        } else if (lane < 4) {
            ZdHufStream s;
            ok = zd_huf4_stream(hsrc, hsize, L.regen, lane, s) &&
                 zd_huf_stream(cx->huf, cx->huf_log, hsrc + s.off, s.size, litbuf + s.first, s.count);
        }
        if (!__all_sync(TS_FULL, ok)) { if (lane == 0) cx->err = -1; __syncwarp(); return false; }
        src.lit = litbuf;
        __threadfence_block();
    }
    __syncwarp();
    return true;
}

// Sequences section header and the three FSE tables (lane 0 reads, the warp builds).  bs: the bit stream.
struct ZdSeqSec { uint32_t nseq; const uint8_t* bs; uint32_t bs_size; };
__device__ __forceinline__ bool zd_stage_seq_header(const uint8_t* blk, uint32_t bsize, const ZdLitSec& L, ZdWarpCtx* cx, uint32_t lane,
                                                    ZdSeqSec& S) {
    const uint8_t* sp = blk + L.hs + L.comp;
    const uint32_t ssize = bsize - L.hs - L.comp;
    if (lane == 0) cx->tmp[0] = zd_parse_seq_header(sp, ssize, false, cx, cx->tmp + 1) ? 1u : 0u;
    __syncwarp();
    if (!cx->tmp[0]) { if (lane == 0 && cx->err == 0) cx->err = -1; __syncwarp(); return false; }
    if (cx->err) return false;
    S.nseq = cx->tmp[1];
    {
        const uint32_t pend = cx->tmp[3];
        for (int k = 0; k < 3; k++) if (pend & (1u << k)) zd_build_dtable_warp(k, cx, lane);
        __syncwarp();
    }
    S.bs = sp + cx->tmp[2];
    S.bs_size = ssize - cx->tmp[2];
    return true;
}

// Position in the sequence bit stream: the backward reader and the three FSE states (lane 0's are the real ones).
struct ZdSeqCursor { ZdBack br; uint32_t st_ll, st_of, st_ml; };
__device__ __forceinline__ bool zd_stage_seq_init(const ZdSeqSec& S, ZdWarpCtx* cx, uint32_t lane, ZdSeqCursor& c) {
    c.br.p = S.bs; c.br.bits = 0; c.br.C = 0; c.br.cbase = 0x3fffffff;
    c.st_ll = 0; c.st_of = 0; c.st_ml = 0;
    if (S.nseq) {
        if (lane == 0) {
            bool ok = zd_back_init(c.br, S.bs, S.bs_size);
            if (ok) {
                c.st_ll = zd_back_read(c.br, cx->ll_log); c.st_of = zd_back_read(c.br, cx->of_log); c.st_ml = zd_back_read(c.br, cx->ml_log);
                if (c.br.bits < 0) ok = false;
            }
            if (!ok) cx->err = -1;
        }
        __syncwarp();
        if (cx->err) return false;
    }
    return true;
}

// One decoded sequence per lane of a batch: lane < cnt (mine), literal / match length, offset value as coded (<= 3: a repeat
// code) and the offset (ofv - 3 until repeat codes are resolved).
struct ZdSeq { bool mine; uint32_t ll, ml, ofv, off; };
// Sequences s0 .. s0 + cnt - 1: (1) lane 0 walks the FSE state chain, (2) every lane cuts its own sequence's offset value /
// match length / literal length out of the stream.
__device__ __forceinline__ bool zd_decode_batch(const ZdSeqSec& S, uint32_t s0, uint32_t cnt, ZdWarpCtx* cx, ZdSeqCursor& c,
                                                uint32_t lane, ZdSeq& q) {
    // (1) lane 0 walks ONLY the state chain: per sequence three table entries, the bit count, three state updates.
    //     It records where each sequence's bits end and which states it was decoded from.
    if (lane == 0) {
        const uint32_t* tof = (const uint32_t*)cx->of; const uint32_t* tml = (const uint32_t*)cx->ml; const uint32_t* tll = (const uint32_t*)cx->ll;
        const uint32_t n_upd = min(cnt, S.nseq - 1 - s0);          // sequences of this batch that are followed by another one
        int32_t bits = c.br.bits;
        bool bad = false;
        uint32_t i = 0;
        for (; i < n_upd; i++) {
            // Bits of one sequence, first read first: offset extra, match-length extra, literal-length extra, then the
            // LL, ML, OF state updates (<= 27 bits: one cached window).
            const uint32_t eo = tof[c.st_of], em = tml[c.st_ml], el = tll[c.st_ll];
            cx->s_ll[i] = c.st_of | (c.st_ml << 10) | (c.st_ll << 20);
            cx->s_ml[i] = (uint32_t)bits;
            const uint32_t t = eo + em + el;                         // bits 0..5: state-update bits, bits 6..11: extra bits
            bits -= (int32_t)((t >> 6) & 63);
            const int32_t lo = bits - (int32_t)(t & 63);
            if (lo < 0) { bad = true; break; }
            if (lo < c.br.cbase || bits > c.br.cbase + 64) {
                c.br.cbase = max(0, ((bits + 7) & ~7) - 64);
                c.br.C = zd_ld64(c.br.p + (c.br.cbase >> 3));
            }
            uint32_t W = (uint32_t)(c.br.C >> (lo - c.br.cbase));
            const uint32_t u_of = eo & 63, u_ml = em & 63, u_ll = el & 63;
            c.st_of = (eo >> 18) + (W & ((1u << u_of) - 1)); W >>= u_of;
            c.st_ml = (em >> 18) + (W & ((1u << u_ml) - 1)); W >>= u_ml;
            c.st_ll = (el >> 18) + (W & ((1u << u_ll) - 1));
            bits = lo;
        }
        if (!bad && i < cnt) {                                   // the block's last sequence: values only
            const uint32_t t = tof[c.st_of] + tml[c.st_ml] + tll[c.st_ll];
            cx->s_ll[i] = c.st_of | (c.st_ml << 10) | (c.st_ll << 20);
            cx->s_ml[i] = (uint32_t)bits;
            bits -= (int32_t)((t >> 6) & 63);
            if (bits < 0) bad = true;
        }
        c.br.bits = bits;
        if (bad) cx->err = -1;
    }
    __syncwarp();
    if (cx->err) return false;
    // (2) every lane cuts the three values of its own sequence out of the stream
    q.mine = lane < cnt;
    q.ll = 0; q.ml = 0; q.off = 1; q.ofv = 4;
    if (q.mine) {
        const uint32_t st = cx->s_ll[lane];
        const int32_t end = (int32_t)cx->s_ml[lane];
        const zf::FseDEntry eo = cx->of[st & 1023], em = cx->ml[(st >> 10) & 1023], el = cx->ll[st >> 20];
        q.ofv = (1u << eo.sym) + zd_bits_at(S.bs, end, eo.nb_extra);
        const uint32_t v = zd_bits_at(S.bs, end - (int32_t)eo.nb_extra, (uint32_t)em.nb_extra + el.nb_extra);
        q.ml = g_seq_tables.ml_base[em.sym] + (v >> el.nb_extra);
        q.ll = g_seq_tables.ll_base[el.sym] + (v & ((1u << el.nb_extra) - 1));
        q.off = q.ofv - 3;
    }
    return true;
}

// Repeat offsets after a batch of cnt (1..32) sequences without a repeat code: its last three offsets, shifted in.  All lanes
// shuffle; lanes with `upd` update r0..r2.
__device__ __forceinline__ void zd_shift_in(uint32_t off, uint32_t cnt, bool upd, uint32_t& r0, uint32_t& r1, uint32_t& r2) {
    const uint32_t o1 = __shfl_sync(TS_FULL, off, cnt - 1), o2 = __shfl_sync(TS_FULL, off, cnt >= 2 ? cnt - 2 : 0),
                   o3 = __shfl_sync(TS_FULL, off, cnt >= 3 ? cnt - 3 : 0);
    if (upd) {
        const uint32_t q0 = r0, q1 = r1;
        r2 = cnt >= 3 ? o3 : cnt == 2 ? q0 : q1;
        r1 = cnt >= 2 ? o2 : q0;
        r0 = o1;
    }
}

// Repeat offsets of a batch (RFC 8878 §3.1.1.5), state in cx->rep: batches without a repeat code (all of this library's) only
// shift in, others are resolved serially by lane 0 and q.off becomes the offset used.  SYM: offsets may be symbolic (see
// ZD_OFF_SYM), "rep1 - 1" by zd_rep_sub1; otherwise they are concrete and may reach bit 29, so "rep1 - 1" is r0 - 1.
template <bool SYM> __device__ __forceinline__ bool zd_resolve_reps(ZdSeq& q, uint32_t cnt, ZdWarpCtx* cx, uint32_t lane) {
    const uint32_t rep_mask = __ballot_sync(TS_FULL, q.mine && q.ofv <= 3);
    if (rep_mask == 0) {
        zd_shift_in(q.off, cnt, lane == 0, cx->rep[0], cx->rep[1], cx->rep[2]);
        return true;
    }
    __syncwarp();
    cx->s_off[lane] = q.ofv; cx->s_ml[lane] = q.ll;
    __syncwarp();
    if (lane == 0) {
        uint32_t r0 = cx->rep[0], r1 = cx->rep[1], r2 = cx->rep[2];
        for (uint32_t i = 0; i < cnt; i++) {
            const uint32_t v = cx->s_off[i];
            uint32_t o;
            if (v > 3) { o = v - 3; r2 = r1; r1 = r0; r0 = o; }
            else {
                const uint32_t idx = v - 1 + (cx->s_ml[i] == 0 ? 1 : 0);     // 0: rep1, 1: rep2, 2: rep3, 3: rep1 - 1
                if (idx == 0) o = r0;
                else {
                    const uint32_t t = idx == 1 ? r1 : idx == 2 ? r2 : SYM ? zd_rep_sub1(r0) : r0 - 1;
                    if (t == 0) { cx->err = -1; break; }
                    if (idx != 1) r2 = r1;
                    r1 = r0; r0 = t; o = t;
                }
            }
            cx->s_off[i] = o;
        }
        cx->rep[0] = r0; cx->rep[1] = r1; cx->rep[2] = r2;
    }
    __syncwarp();
    if (cx->err) return false;
    q.off = q.mine ? cx->s_off[lane] : 1;
    return true;
}

// Executes a resolved batch into dst: lane i owns sequence i.  Output/literal positions come from shuffle prefix sums;
// literal runs are independent; a match may start once its source range lies inside the completed prefix (multi-round
// resolution: far matches of a batch all copy at once, so their memory latency overlaps).  `hist` bytes before dst may be
// referenced, at most `limit` produced; advances op / lp.
__device__ __forceinline__ bool zd_exec_batch(const ZdSeq& q, const ZdLitSrc& src, uint32_t regen, uint8_t* dst, uint64_t hist,
                                              uint32_t limit, ZdWarpCtx* cx, uint32_t lane, uint32_t& op, uint32_t& lp) {
    const bool mine = q.mine;
    const uint32_t ll = q.ll, ml = q.ml, off = q.off;
    const uint8_t* lit = src.lit;
    const uint32_t rle_lit = src.rle_lit;
    __syncwarp();
    const uint32_t inc_o = warp_inclusive_scan_u32(ll + ml, lane), inc_l = warp_inclusive_scan_u32(ll, lane);
    const uint32_t tot_o = __shfl_sync(TS_FULL, inc_o, 31), tot_l = __shfl_sync(TS_FULL, inc_l, 31);
    const uint32_t o_start = op + inc_o - ll - ml, l_start = lp + inc_l - ll, m_start = o_start + ll;
    const bool bad_off = mine && (uint64_t)off > hist + m_start;
    const uint32_t any_bad = __ballot_sync(TS_FULL, bad_off);
    if (lp + tot_l > regen || (uint64_t)op + tot_o > limit || any_bad) {
        if (lane == 0) cx->err = -1;
        __syncwarp();
        return false;
    }
    // literals: short runs by their own lane, long runs by the whole warp
    {
        const uint32_t quick = min(ll, 32u);
        if (rle_lit < 0x100) { for (uint32_t k = 0; k < quick; k++) dst[o_start + k] = (uint8_t)rle_lit; }
        else {                                       // four loads in flight per step (lit and dst never alias)
            const uint8_t* ls = lit + l_start; uint8_t* ld = dst + o_start;
            uint32_t k = 0;
            for (; k + 4 <= quick; k += 4) {
                const uint8_t b0 = ls[k], b1 = ls[k + 1], b2 = ls[k + 2], b3 = ls[k + 3];
                ld[k] = b0; ld[k + 1] = b1; ld[k + 2] = b2; ld[k + 3] = b3;
            }
            for (; k < quick; k++) ld[k] = ls[k];
        }
        uint32_t longs = __ballot_sync(TS_FULL, ll > 32);
        while (longs) {
            const uint32_t f = (uint32_t)__ffs((int)longs) - 1;
            longs &= longs - 1;
            const uint32_t fo = __shfl_sync(TS_FULL, o_start, f), fl = __shfl_sync(TS_FULL, l_start, f), fn = __shfl_sync(TS_FULL, ll, f);
            if (rle_lit < 0x100) { for (uint32_t k = 32 + lane; k < fn; k += 32) dst[fo + k] = (uint8_t)rle_lit; }
            else { for (uint32_t k = 32 + lane; k < fn; k += 32) dst[fo + k] = lit[fl + k]; }
        }
    }
    __syncwarp();
    // matches
    bool done = !mine || ml == 0;
    const int64_t src_end = (int64_t)m_start - (int64_t)off + (int64_t)ml;      // relative to dst
    while (true) {
        const uint32_t pending = __ballot_sync(TS_FULL, !done);
        if (!pending) break;
        const uint32_t first = (uint32_t)__ffs((int)pending) - 1;
        const uint32_t frontier = __shfl_sync(TS_FULL, m_start, first);
        const bool ready = !done && (lane == first || src_end <= (int64_t)frontier);
        uint8_t* d = dst + m_start;
        const uint8_t* m = d - off;
        if (ready && ml <= 64) {
            uint32_t k = 0;
            if (off >= 4) {                              // the four source bytes of a step all precede its first store
                for (; k + 4 <= ml; k += 4) {
                    const uint8_t b0 = m[k], b1 = m[k + 1], b2 = m[k + 2], b3 = m[k + 3];
                    d[k] = b0; d[k + 1] = b1; d[k + 2] = b2; d[k + 3] = b3;
                }
            }
            for (; k < ml; k++) d[k] = m[k];             // byte-serial: overlap (off < ml) is fine
            done = true;
        }
        uint32_t big = __ballot_sync(TS_FULL, ready && ml > 64);
        while (big) {                                                            // long matches: 32 lanes per match
            const uint32_t f = (uint32_t)__ffs((int)big) - 1;
            big &= big - 1;
            const uint32_t fm = __shfl_sync(TS_FULL, m_start, f), fl = __shfl_sync(TS_FULL, ml, f), fo = __shfl_sync(TS_FULL, off, f);
            uint8_t* dd = dst + fm;
            const uint8_t* mm = dd - fo;
            if (fo >= 32) {
                for (uint32_t k0 = 0; k0 < fl; k0 += 32) {
                    const uint32_t k = k0 + lane;
                    if (k < fl) dd[k] = mm[k];
                    if (fo < fl) __syncwarp();                                   // later strides may read what this one wrote
                }
            } else {
                for (uint32_t k = lane; k < fl; k += 32) dd[k] = mm[k % fo];     // periodic source entirely before dd
            }
            if (lane == f) done = true;
        }
        __syncwarp();
    }
    op += tot_o; lp += tot_l;
    return true;
}

// The literals after the last sequence.
__device__ __forceinline__ bool zd_trailing_literals(const ZdLitSrc& src, uint32_t regen, uint32_t lp, uint8_t* dst, uint32_t limit,
                                                     ZdWarpCtx* cx, uint32_t lane, uint32_t& op) {
    const uint32_t ll = regen - lp;
    if ((uint64_t)op + ll > limit) { if (lane == 0) cx->err = -1; __syncwarp(); return false; }
    if (src.rle_lit < 0x100) { for (uint32_t k = lane; k < ll; k += 32) dst[op + k] = (uint8_t)src.rle_lit; }
    else { for (uint32_t k = lane; k < ll; k += 32) dst[op + k] = src.lit[lp + k]; }
    op += ll;
    return true;
}

// ------------------------------------------------------------------------------------------ one compressed block
// Warp-uniform.  Decodes the Compressed_Block at blk[0..bsize) and appends its output at dst[0..); `hist` bytes
// before dst belong to this frame and may be referenced; at most `limit` bytes may be produced.
// Returns the number of bytes produced; cx->err != 0 on failure.
__device__ __forceinline__ uint32_t zd_compressed_block(const uint8_t* blk, uint32_t bsize, uint8_t* dst, uint64_t hist,
                                                        uint32_t limit, ZdWarpCtx* cx, uint8_t* litbuf, uint32_t lane) {
    ZdLitSec L;
    ZdLitSrc src;
    ZdSeqSec S;
    ZdSeqCursor c;
    if (!zd_stage_lit_header(blk, bsize, limit, cx, lane, L) || !zd_stage_lit_source(blk, L, cx, litbuf, lane, src) ||
        !zd_stage_seq_header(blk, bsize, L, cx, lane, S) || !zd_stage_seq_init(S, cx, lane, c)) return 0;
    uint32_t op = 0, lp = 0;                            // output / literal cursors (uniform)
    for (uint32_t s0 = 0; s0 < S.nseq; s0 += 32) {
        const uint32_t cnt = min(32u, S.nseq - s0);
        ZdSeq q;
        if (!zd_decode_batch(S, s0, cnt, cx, c, lane, q) || !zd_resolve_reps<false>(q, cnt, cx, lane) ||
            !zd_exec_batch(q, src, L.regen, dst, hist, limit, cx, lane, op, lp)) return 0;
    }
    if (!zd_trailing_literals(src, L.regen, lp, dst, limit, cx, lane, op)) return 0;
    __syncwarp();
    return op;
}

// ------------------------------------------------------------------------------------------ parallel general path
// (The general decode path of the product; round 1 had it behind TSGPU_DEC_PARALLEL=1.)  Frames written by libzstd have few,
// large blocks that inherit tables and repeat offsets from each other, so the per-block fast path does not apply and one
// warp per frame is slow for a lone frame.  Here every block's ENTROPY decoding (Huffman literals, FSE sequences) runs on its own warp into global scratch:
// tables a block inherits (treeless literals, Repeat_Mode) are rebuilt by replaying the table definitions of the blocks
// before it; offsets stay unresolved offset VALUES.  One warp per frame then resolves repeat offsets and executes the
// sequences in order.  The stages are the same functions the serial decoder is made of.
struct ZdBlkMeta {
    uint32_t status;                 // 1 decoded, 2 failed, 3 = needs the serial path (a field does not fit the sequence word)
    uint32_t lit_kind, lit_off, regen, nseq, seq_off;      // lit_kind 0 arena, 1 in the block, 2 RLE
    uint32_t rep[3];                 // repeat offsets after the block, in the offset-field encoding (ZD_OFF_SYM)
    uint32_t pad[3];
};
struct ZdParIO { uint8_t* lit_arena; uint32_t lit_cap; uint32_t* lit_bump; uint64_t* seq_arena; uint32_t seq_cap; uint32_t* seq_bump; };

// Only the Huffman tree of a Compressed_Block with Compressed_Literals (what treeless blocks after it inherit).
__device__ __forceinline__ bool zd_block_huf_only(const uint8_t* blk, uint32_t bsize, ZdWarpCtx* cx, uint32_t lane, ZdLitSec& L) {
    if (!zd_stage_lit_header(blk, bsize, zf::BLOCK_MAX, cx, lane, L)) return false;
    if (L.type == 2) zd_fill_huf_warp(cx, lane);
    __syncwarp();
    return true;
}

// Table definitions of one Compressed_Block only (Huffman tree, the three FSE tables): what a later block may inherit.
__device__ __forceinline__ void zd_block_tables(const uint8_t* blk, uint32_t bsize, ZdWarpCtx* cx, uint32_t lane) {
    ZdLitSec L;
    ZdSeqSec S;
    if (zd_block_huf_only(blk, bsize, cx, lane, L)) zd_stage_seq_header(blk, bsize, L, cx, lane, S);
}

// What a Compressed_Block inherits and what it defines.  Lane 0 parses, the warp gets the answer as a mask:
//   bit 0  literals are treeless (the Huffman tree comes from an earlier block)
//   bit 1  at least one FSE table is in Repeat_Mode
//   bit 2  the block has no sequences (its sequences section defines no table)
//   bit 3  the block carries a Huffman tree (Compressed_Literals)
// Malformed headers answer "inherits everything": the replay or the block's own decode then reports the error.
__device__ __forceinline__ uint32_t zd_block_inherits(const uint8_t* blk, uint32_t bsize, uint32_t lane) {
    uint32_t r = 3;
    if (lane == 0) {
        do {
            const ZdLitSec L = zd_lit_section(blk, bsize);
            if (!L.hs) break;
            if ((uint64_t)L.hs + L.comp + 1 > bsize) break;
            const uint8_t* sp = blk + L.hs + L.comp;
            const uint32_t ssize = bsize - L.hs - L.comp;
            uint32_t nseq = sp[0], sh = 1;
            if (nseq >= 128) { sh = nseq == 255 ? 3 : 2; if (ssize < sh) break; nseq = 1; }
            const uint32_t huf = (L.type == 3 ? 1u : 0u) | (L.type == 2 ? 8u : 0u);
            if (nseq == 0) { r = huf | 4u; break; }
            if (ssize < sh + 1) break;
            const uint32_t modes = sp[sh];
            r = huf | (((modes >> 6) == 3 || ((modes >> 4) & 3) == 3 || ((modes >> 2) & 3) == 3) ? 2u : 0u);
        } while (false);
    }
    return __shfl_sync(TS_FULL, r, 0);
}

// Entropy stage of one Compressed_Block: literals into the frame's literal arena (unless Raw / RLE), sequences as
// packed words (see ZD_OFF_SYM) into the frame's sequence arena.  Repeat offsets are resolved HERE, per block and in
// parallel across blocks: the three repeat offsets a block starts with are unknown to it, so they are carried as symbols
// (initial offset k, minus d) until real offsets have pushed them out; the execution stage substitutes them.
__device__ __forceinline__ void zd_block_entropy(const uint8_t* blk, uint32_t bsize, ZdWarpCtx* cx, const ZdParIO& io,
                                                 ZdBlkMeta* meta, uint32_t lane) {
    ZdLitSec L;
    if (!zd_stage_lit_header(blk, bsize, zf::BLOCK_MAX, cx, lane, L)) return;
    uint8_t* litbuf = nullptr;
    uint32_t lit_at = 0;
    if (L.type >= 2) {
        if (lane == 0) {
            const uint32_t o = atomicAdd(io.lit_bump, (L.regen + 15) & ~15u);
            cx->tmp[7] = o;
            if ((uint64_t)o + L.regen + 16 > io.lit_cap) cx->err = -1;
        }
        __syncwarp();
        if (cx->err) return;
        lit_at = cx->tmp[7];
        litbuf = io.lit_arena + lit_at;
    }
    ZdLitSrc src;
    ZdSeqSec S;
    if (!zd_stage_lit_source(blk, L, cx, litbuf, lane, src) || !zd_stage_seq_header(blk, bsize, L, cx, lane, S)) return;
    if (lane == 0) {
        const uint32_t o = atomicAdd(io.seq_bump, S.nseq);
        cx->tmp[7] = o;
        if ((uint64_t)o + S.nseq > io.seq_cap) cx->err = -1;
        cx->rep[0] = zd_sym_rep(1); cx->rep[1] = zd_sym_rep(2); cx->rep[2] = zd_sym_rep(3);
    }
    __syncwarp();
    if (cx->err) return;
    const uint32_t seq_at = cx->tmp[7];
    uint64_t* sq = io.seq_arena + seq_at;
    ZdSeqCursor c;
    if (!zd_stage_seq_init(S, cx, lane, c)) return;
    for (uint32_t s0 = 0; s0 < S.nseq; s0 += 32) {
        const uint32_t cnt = min(32u, S.nseq - s0);
        ZdSeq q;
        if (!zd_decode_batch(S, s0, cnt, cx, c, lane, q)) return;
        const bool wide = q.mine && !zd_seq_fits(q.ofv, q.ll, q.ml);
        if (__ballot_sync(TS_FULL, wide)) { if (lane == 0) cx->err = 2; __syncwarp(); return; }    // does not fit the word: serial path
        if (!zd_resolve_reps<true>(q, cnt, cx, lane)) return;
        if (q.mine) sq[s0 + lane] = zd_seq_pack(q.off, q.ll, q.ml);
        __syncwarp();
    }
    if (lane == 0) {
        meta->lit_kind = L.type == 0 ? 1u : L.type == 1 ? 2u : 0u;
        meta->lit_off = L.type == 0 ? L.hs : L.type == 1 ? src.rle_lit : lit_at;
        meta->regen = L.regen; meta->nseq = S.nseq; meta->seq_off = seq_at;
        if (S.nseq) { meta->rep[0] = cx->rep[0]; meta->rep[1] = cx->rep[1]; meta->rep[2] = cx->rep[2]; }
        else { meta->rep[0] = zd_sym_rep(1); meta->rep[1] = zd_sym_rep(2); meta->rep[2] = zd_sym_rep(3); }
    }
}

// ------------------------------------------------------------------------------------------ execution stage, one CTA
// Executes the sequences the entropy stage left in the arenas, blocks [b_first, b_last) in order.  Output is assembled in a
// shared-memory WINDOW (`win`, holding frame positions [win_pos0, win_pos0 + win_cap)) and flushed to HBM by the caller
// (regions: once, 64 KiB) or here after every block (whole frames: the window is the current block, <= 128 KiB; matches that
// reach before it read the flushed bytes from `far`).  ZX_T sequences are taken per step:
//   * positions by a CTA-wide prefix sum of literal and match lengths,
//   * every literal run copied at once (they depend on nothing),
//   * matches by EXACT dependency tracking without barriers: the sequences whose output covers a match's source are found
//     by binary search in the step's positions; a match spins on their done bits (one 32-bit word per warp, written only by
//     that warp) and copies as soon as they are set.  Text compressed against its nearest earlier occurrence makes chains
//     of dozens of dependent matches inside one step: a hop along such a chain costs a shared-memory poll, not a barrier.
constexpr int ZX_T = 512;                 // threads of the region executor; the frame executor runs ZX_TF
constexpr int ZX_TF = 1024;
template <int T> struct ZxShared {
    uint32_t ostart[T + 1];               // output position of each sequence of the step (+ end)
    uint32_t mlen[T], moff[T];         // match length / offset of each sequence of the step (source forwarding)
    uint32_t dbits[T / 32];               // done bit per sequence of the step; word w is written by warp w only
    uint64_t wsum[T / 32];
    uint64_t tot;
    uint32_t rep[3];
    int32_t err;
};

// T == 32: the "CTA" is one warp among several of its thread block, so barriers are warp barriers.
template <int T> __device__ __forceinline__ void zx_barrier() { if (T == 32) __syncwarp(); else __syncthreads(); }
template <int T> __device__ __forceinline__ bool zx_barrier_or(bool p) {
    if (T == 32) return __any_sync(TS_FULL, p) != 0;
    return __syncthreads_or(p) != 0;
}
template <int T> __device__ __forceinline__ uint32_t zx_barrier_count(bool p) {
    if (T == 32) return (uint32_t)__popc(__ballot_sync(TS_FULL, p));
    return (uint32_t)__syncthreads_count(p);
}
template <int T> __device__ __forceinline__ uint64_t zx_block_scan(uint64_t v, uint32_t tid, ZxShared<T>* sh, uint64_t* total) {
    const uint32_t lane = tid & 31, w = tid >> 5;
    uint64_t inc = warp_inclusive_scan_u64(v, lane);
    if (T == 32) { *total = __shfl_sync(TS_FULL, inc, 31); return inc; }
    if (lane == 31) sh->wsum[w] = inc;
    __syncthreads();
    if (w == 0) {
        const uint64_t x = lane < T / 32 ? sh->wsum[lane] : 0;
        const uint64_t xi = warp_inclusive_scan_u64(x, lane);
        if (lane < T / 32) sh->wsum[lane] = xi - x;
        if (lane == T / 32 - 1) sh->tot = xi;
    }
    __syncthreads();
    inc += sh->wsum[w];
    *total = sh->tot;
    return inc;
}

__device__ __forceinline__ uint32_t zx_ld_volatile(const uint32_t* p) { return *(const volatile uint32_t*)p; }

// are all sequences [ja, jb] of the step done?  (bits of words ja/32 .. jb/32)
__device__ __forceinline__ bool zx_all_done(const uint32_t* dbits, uint32_t ja, uint32_t jb) {
    const uint32_t wa = ja >> 5, wb = jb >> 5;
    for (uint32_t w = wa; w <= wb; w++) {
        uint32_t need = 0xffffffffu;
        if (w == wa) need &= 0xffffffffu << (ja & 31);
        if (w == wb) need &= 0xffffffffu >> (31 - (jb & 31));
        if ((zx_ld_volatile(&dbits[w]) & need) != need) return false;
    }
    return true;
}

// Copy n (<= 64) bytes from HBM to the window by ONE thread: the loads of a 16-byte piece are issued together (one memory
// latency per piece instead of one per byte — a byte loop through generic pointers waits for every load before the next).
__device__ __forceinline__ void zx_copy_from_hbm(uint8_t* d, const uint8_t* s, uint32_t n) {
    uint32_t k = 0;
    for (; k + 16 <= n; k += 16) {
        const uint32_t w0 = ld_u32_unaligned(s + k), w1 = ld_u32_unaligned(s + k + 4), w2 = ld_u32_unaligned(s + k + 8), w3 = ld_u32_unaligned(s + k + 12);
        _Pragma("unroll")
        for (int q = 0; q < 4; q++) { d[k + q] = (uint8_t)(w0 >> (8 * q)); d[k + 4 + q] = (uint8_t)(w1 >> (8 * q)); d[k + 8 + q] = (uint8_t)(w2 >> (8 * q)); d[k + 12 + q] = (uint8_t)(w3 >> (8 * q)); }
    }
    if (k < n) {                                         // tail: up to 15 bytes, loads first (reads at most 3 bytes past the end of the source's last word)
        const uint32_t r = n - k;
        const uint32_t w0 = ld_u32_unaligned(s + k);
        uint32_t w1 = 0, w2 = 0, w3 = 0;
        if (r > 4) w1 = ld_u32_unaligned(s + k + 4);
        if (r > 8) w2 = ld_u32_unaligned(s + k + 8);
        if (r > 12) w3 = ld_u32_unaligned(s + k + 12);
        uint32_t q = 0;
        for (; q + 4 <= r; q += 4) {
            const uint32_t w = q == 0 ? w0 : q == 4 ? w1 : w2;
            d[k + q] = (uint8_t)w; d[k + q + 1] = (uint8_t)(w >> 8); d[k + q + 2] = (uint8_t)(w >> 16); d[k + q + 3] = (uint8_t)(w >> 24);
        }
        uint32_t w = q == 0 ? w0 : q == 4 ? w1 : q == 8 ? w2 : w3;
        for (; q < r; q++) { d[k + q] = (uint8_t)w; w >>= 8; }
    }
}

// Flush win[0..n) to dst (HBM), 128-bit stores when the destination allows.  All threads; no barrier inside.
template <int T> __device__ __forceinline__ void zx_flush(uint8_t* dst, const uint8_t* win, uint32_t n, uint32_t tid) {
    if ((((uintptr_t)dst) & 15) == 0) {
        for (uint32_t k = tid * 16; k + 16 <= n; k += T * 16) stg128_stream((uint4*)(dst + k), *(const uint4*)(win + k));
        for (uint32_t k = (n & ~15u) + tid; k < n; k += T) dst[k] = win[k];
    } else {
        for (uint32_t k = tid; k < n; k += T) dst[k] = win[k];
    }
}

// Returns the new output position (bytes produced since position 0 of the caller's numbering) or sets sh->err
// (<0 corrupt / contract violated, 3 = a block needs the serial path).
//   win / win_cap   shared-memory window
//   far             HBM image of the output, position 0 at far[0] (nullptr: nothing before the window may be referenced)
//   per_block       true: the window restarts at every block and is flushed to `far` after it (whole frames)
//                   false: one window for all blocks, the caller flushes (regions)
//   PJ / pj         false: matches of a step resolve by exact dependency tracking (done bits, see above);
//                   true: by POINTER JUMPING over the step's bytes.  pj[r] (r relative to the step's first byte; identity on entry
//                   and on exit) names the byte that byte r is a copy of; bytes copied from before the step, and literals, are
//                   roots.  Every thread then replaces pj[r] by pj[pj[r]] for its bytes until all of them point at roots — a
//                   chain of d dependent copies (text matched against its nearest earlier occurrence makes d ~ 50..100 per
//                   1024 sequences) resolves in log2 d sweeps with one barrier each, not in d hand-overs — and fetches the
//                   bytes.  A step is cut so that it spans at most 32 * T bytes (32 bytes per thread, one mask word).
template <int T, bool PJ = false>
__device__ __forceinline__ uint32_t zx_execute_blocks(const uint8_t* frame, const uint32_t* bo, const ZdBlkMeta* meta,
                                                      uint32_t b_first, uint32_t b_last, uint8_t* win, uint32_t win_cap,
                                                      uint8_t* far, bool per_block, uint32_t out_cap,
                                                      const uint8_t* lit_arena, const uint64_t* seq_arena, uint32_t frame_len,
                                                      ZxShared<T>* sh, uint32_t tid, bool no_carried_reps, uint16_t* pj = nullptr) {
    const uint32_t lane = tid & 31, w = tid >> 5;
    uint32_t op = 0;
    uint32_t win_pos0 = 0;                               // frame position of win[0]
    if (tid == 0) { sh->rep[0] = 1; sh->rep[1] = 4; sh->rep[2] = 8; sh->err = 0; }
    zx_barrier<T>();
    for (uint32_t b = b_first; b < b_last; b++) {
        const uint32_t pos = bo[b];
        const ZdBlkHdr bh = zd_block_header(frame + pos);
        const uint32_t type = bh.type, bsz = bh.size;
        if (per_block) win_pos0 = op;
        const uint32_t room = min(min((uint32_t)zf::BLOCK_MAX, out_cap - op), win_cap - (op - win_pos0));
        uint8_t* wout = win - win_pos0;                  // wout[position] for positions inside the window
        if (type == 0 || type == 1) {                    // Raw_Block / RLE_Block
            if (bsz > room || pos + 3 + (type == 0 ? bsz : 1) > frame_len) { if (tid == 0) sh->err = -1; zx_barrier<T>(); return op; }
            const uint8_t v = frame[pos + 3];
            if (type == 0) { for (uint32_t k = tid; k < bsz; k += T) wout[op + k] = frame[pos + 3 + k]; }
            else { for (uint32_t k = tid; k < bsz; k += T) wout[op + k] = v; }
            zx_barrier<T>();
            if (per_block) { zx_flush<T>(far + op, win, bsz, tid); zx_barrier<T>(); }
            op += bsz;
            continue;
        }
        const ZdBlkMeta m = meta[b];
        if (m.status != 1) { if (tid == 0) sh->err = m.status == 3 ? 3 : -1; zx_barrier<T>(); return op; }
        const uint8_t* blk = frame + pos + 3;
        const uint8_t* lit = nullptr;
        uint32_t rle_lit = 0x100;
        if (m.lit_kind == 1) lit = blk + m.lit_off;
        else if (m.lit_kind == 2) rle_lit = m.lit_off & 0xff;
        else lit = lit_arena + m.lit_off;
        const uint64_t* sq = seq_arena + m.seq_off;
        const uint32_t N = m.nseq, regen = m.regen;
        const uint32_t R0 = sh->rep[0], R1 = sh->rep[1], R2 = sh->rep[2];     // repeat offsets at the start of the block
        const uint32_t blk_op0 = op;
        uint32_t lp = 0;
        uint32_t n_take = T;                                  // sequences a step consumed (PJ: a step may be cut short)
        for (uint32_t base = 0; base < N; base += n_take) {
            const uint32_t i = base + tid;
            bool mine = i < N;
            uint32_t ll = 0, ml = 0, off = 1;
            bool bad = false;
            if (mine) {
                uint32_t of;
                zd_seq_unpack(sq[i], of, ll, ml);
                if (of & ZD_OFF_SYM) {
                    uint32_t d;
                    const uint32_t r = zd_sym_base(of, R0, R1, R2, &d);
                    if (r <= d || no_carried_reps) bad = true; else off = r - d;      // a region cannot know what earlier regions left behind
                } else off = of;
                if (off == 0) bad = true;
            }
            uint64_t tot;
            uint64_t inc = zx_block_scan<T>(((uint64_t)(ll + ml) << 32) | ll, tid, sh, &tot);
            n_take = T;
            if (PJ && (uint32_t)(tot >> 32) > 32u * T) {                  // cut the step after the last sequence that ends inside the span
                const uint32_t fit = zx_barrier_count<T>(mine && (uint32_t)(inc >> 32) <= 32u * T);
                if (fit == 0) {
                    // one sequence larger than the span: literal run and match by the whole CTA, then on with the next sequence
                    if (tid == 0) { sh->ostart[0] = ll; sh->mlen[0] = ml; sh->moff[0] = off; sh->dbits[0] = bad ? 1u : 0u; }
                    zx_barrier<T>();
                    const uint32_t gl = sh->ostart[0], gm = sh->mlen[0], go = sh->moff[0];
                    const bool gbad = sh->dbits[0] != 0 || lp + gl > regen || (uint64_t)(op - blk_op0) + gl + gm > room ||
                                      go > op + gl || (!far && go > op + gl - win_pos0);
                    zx_barrier<T>();
                    if (gbad) { if (tid == 0) sh->err = -1; zx_barrier<T>(); return op; }
                    if (rle_lit < 0x100) { for (uint32_t k = tid; k < gl; k += T) wout[op + k] = (uint8_t)rle_lit; }
                    else { for (uint32_t k = tid; k < gl; k += T) wout[op + k] = lit[lp + k]; }
                    zx_barrier<T>();
                    const uint32_t gs = op + gl;                          // match start
                    if (go < T) {                                         // periodic source: the go bytes before the match, all written
                        for (uint32_t k = tid; k < gm; k += T) { const uint32_t q = gs - go + k % go; wout[gs + k] = q < win_pos0 ? far[q] : wout[q]; }
                    } else {
                        for (uint32_t k0 = 0; k0 < gm; k0 += T) {         // T <= go bytes per round never read what the round writes
                            const uint32_t k = k0 + tid;
                            if (k < gm) { const uint32_t q = gs - go + k; wout[gs + k] = q < win_pos0 ? far[q] : wout[q]; }
                            zx_barrier<T>();
                        }
                    }
                    zx_barrier<T>();
                    op += gl + gm; lp += gl; n_take = 1;
                    continue;
                }
                n_take = fit;
                if (tid >= fit) { mine = false; ll = 0; ml = 0; off = 1; bad = false; }
                inc = zx_block_scan<T>(((uint64_t)(ll + ml) << 32) | ll, tid, sh, &tot);
            }
            const uint32_t tot_o = (uint32_t)(tot >> 32), tot_l = (uint32_t)tot;
            const uint32_t o_start = op + (uint32_t)(inc >> 32) - ll - ml, l_start = lp + (uint32_t)inc - ll, m_start = o_start + ll;
            if (mine && (off > m_start || (!far && off > m_start - win_pos0))) bad = true;
            sh->ostart[tid] = mine ? o_start : op + tot_o;
            sh->mlen[tid] = mine ? ml : 0; sh->moff[tid] = off;
            const uint32_t preset = __ballot_sync(TS_FULL, !mine || ml == 0);         // nothing to wait for on these
            if (lane == 0) sh->dbits[w] = preset;
            if (tid == 0) sh->ostart[T] = op + tot_o;
            const bool any_bad = zx_barrier_or<T>(bad);
            if (any_bad || lp + tot_l > regen || (uint64_t)(op - blk_op0) + tot_o > room) {
                if (tid == 0) sh->err = -1;
                zx_barrier<T>();
                return op;
            }
            // ---- literal runs: short ones by their own thread, long ones by the warp
            {
                const uint32_t quick = min(ll, 32u);
                uint8_t* ld = wout + o_start;
                if (rle_lit < 0x100) { for (uint32_t k = 0; k < quick; k++) ld[k] = (uint8_t)rle_lit; }
                else zx_copy_from_hbm(ld, lit + l_start, quick);
                uint32_t longs = __ballot_sync(TS_FULL, ll > 32);
                while (longs) {
                    const uint32_t f = (uint32_t)__ffs((int)longs) - 1;
                    longs &= longs - 1;
                    const uint32_t fo = __shfl_sync(TS_FULL, o_start, f), fl = __shfl_sync(TS_FULL, l_start, f), fn = __shfl_sync(TS_FULL, ll, f);
                    if (rle_lit < 0x100) { for (uint32_t k = 32 + lane; k < fn; k += 32) wout[fo + k] = (uint8_t)rle_lit; }
                    else { for (uint32_t k = 32 + lane; k < fn; k += 32) wout[fo + k] = lit[fl + k]; }
                }
            }
            zx_barrier<T>();                                              // literals, ostart, mlen, moff, dbits visible to everyone
            if (PJ) {
                // ---- matches by pointer jumping
                const uint32_t s_lo = m_start - off;
                const uint32_t s_hi = min(s_lo + ml, m_start);            // one past the last source byte somebody else wrote
                const bool has = mine && ml != 0;
                const bool inside = has && s_hi > op;                     // reads bytes of this step
                uint8_t* d = wout + m_start;
                if (has && !inside && ml <= 64) {                         // complete before the step: copy now, these bytes are roots
                    if (s_hi <= win_pos0) zx_copy_from_hbm(d, far + s_lo, ml);
                    else if (s_lo < win_pos0) { for (uint32_t k = 0; k < ml; k++) { const uint32_t q = s_lo + k; d[k] = q < win_pos0 ? far[q] : wout[q]; } }
                    else { const uint8_t* ms = d - off; for (uint32_t k = 0; k < ml; k++) d[k] = ms[k]; }
                }
                if (inside && ml <= 64) {
                    for (uint32_t k = 0; k < ml; k++) {
                        const uint32_t q = m_start + k, sq_ = q - off;
                        if (sq_ < op) d[k] = sq_ < win_pos0 ? far[sq_] : wout[sq_];
                        else pj[q - op] = (uint16_t)(sq_ - op);
                    }
                }
                uint32_t big = __ballot_sync(TS_FULL, has && ml > 64);
                while (big) {                                             // long matches: 32 lanes per match
                    const uint32_t f = (uint32_t)__ffs((int)big) - 1;
                    big &= big - 1;
                    const uint32_t fm = __shfl_sync(TS_FULL, m_start, f), fl = __shfl_sync(TS_FULL, ml, f), fo = __shfl_sync(TS_FULL, off, f);
                    for (uint32_t k = lane; k < fl; k += 32) {
                        const uint32_t q = fm + k;
                        const uint32_t sq_ = q - fo;
                        if (sq_ >= op) pj[q - op] = (uint16_t)(sq_ - op);  // (includes every byte of an overlapping match past its first period)
                        else wout[q] = sq_ < win_pos0 ? far[sq_] : wout[sq_];
                    }
                }
                zx_barrier<T>();                                          // pointers and roots are in place
                uint32_t nonroot = 0;
                for (uint32_t j = 0; j * T + tid < tot_o; j++) { const uint32_t r = j * T + tid; if (pj[r] != r) nonroot |= 1u << j; }
                uint32_t pend = nonroot;
                while (true) {
                    bool changed = false;
                    uint32_t m = pend;
                    while (m) {
                        const uint32_t j = (uint32_t)__ffs((int)m) - 1;
                        m &= m - 1;
                        const uint32_t r = j * T + tid;
                        const uint32_t s1 = *(volatile uint16_t*)&pj[r];
                        const uint32_t s2 = *(volatile uint16_t*)&pj[s1];
                        if (s2 != s1) { *(volatile uint16_t*)&pj[r] = (uint16_t)s2; changed = true; }
                        else pend &= ~(1u << j);                          // points at a root
                    }
                    if (!zx_barrier_or<T>(changed)) break;
                }
                for (uint32_t m = nonroot; m; m &= m - 1) {
                    const uint32_t r = ((uint32_t)__ffs((int)m) - 1) * T + tid;
                    wout[op + r] = wout[op + pj[r]];                      // roots are final and nobody writes them here
                    pj[r] = (uint16_t)r;
                }
            } else {
                // ---- producers of this match inside the step: sequences [ja, jb] cover the part of its source other sequences write.
                // Source forwarding first: text matched against its nearest earlier occurrence makes chains of dozens of matches
                // inside one step, each copying what the previous one wrote.  When a source lies entirely inside ONE earlier match
                // of the step, the bytes are, by the definition of an LZ copy, the bytes that match itself copies — so this match
                // can read THEM instead (offset += that match's offset) and no longer depends on it.  A few hops shorten the
                // chains to what really is a partial overlap.
                uint32_t s_lo = m_start - off;                                // first source byte
                uint32_t s_hi = min(s_lo + ml, m_start);                      // one past the last source byte written by someone else
                uint32_t ja = 0, jb = 0;
                bool inside = false;                                          // does the source reach into this step's output?
                if (mine && ml) {
                    uint32_t top = tid;                                       // producers are searched below this index
                    for (uint32_t hop = 0; ; hop++) {
                        inside = false;
                        if (s_hi <= op) break;                                // everything it reads was complete before the step
                        inside = true;
                        uint32_t lo = 0, hi = top;                            // ja: last j <= top with ostart[j] <= x
                        const uint32_t x = max(s_lo, op);
                        while (hi - lo > 0) { const uint32_t mid = (lo + hi + 1) >> 1; if (sh->ostart[mid] <= x) lo = mid; else hi = mid - 1; }
                        ja = lo;
                        const uint32_t pend_ = sh->ostart[ja + 1];            // end of sequence ja's output = end of its match
                        if (ja < tid && s_hi <= pend_ && s_lo >= op) {        // the whole source lies in ONE earlier sequence of the step
                            jb = ja;
                            const uint32_t pst = pend_ - sh->mlen[ja];        // its match bytes are [pst, pend_)
                            if (s_hi <= pst) { inside = false; break; }       // only its literals: written already
                            if (s_lo >= pst && off >= ml && hop < 12) {       // inside its match: read what IT reads
                                const uint32_t po = sh->moff[ja];
                                off += po; s_lo -= po; s_hi -= po;
                                top = ja;
                                continue;
                            }
                            break;
                        }
                        lo = ja; hi = tid;                                    // jb: last j <= tid with ostart[j] < s_hi
                        while (hi - lo > 0) { const uint32_t mid = (lo + hi + 1) >> 1; if (sh->ostart[mid] < s_hi) lo = mid; else hi = mid - 1; }
                        jb = lo;
                        if (jb == tid) { if (tid == 0 || ja == tid) inside = false; else jb = tid - 1; }   // own literals precede the match: never a producer
                        break;
                    }
                }
                // ---- matches: every warp runs its own loop; a lane copies once the done bits of its producers are set
                {
                    bool done = !mine || ml == 0;
                    const bool from_far = s_hi <= win_pos0 && ml != 0;        // whole source before the window: flushed long ago
                    const bool straddle = !from_far && s_lo < win_pos0;       // (only with off >= ml, else s_hi would be m_start)
                    uint8_t* d = wout + m_start;
                    uint32_t pend = __ballot_sync(TS_FULL, !done);
                    while (pend) {
                        bool ready = false;
                        if (!done) ready = !inside || zx_all_done(sh->dbits, ja, jb);
                        if (ready) __threadfence_block();                      // acquire: the producers' bytes are visible
                        if (ready && ml <= 64) {
                            if (from_far) zx_copy_from_hbm(d, far + s_lo, ml);
                            else if (straddle) { for (uint32_t k = 0; k < ml; k++) { const uint32_t q = s_lo + k; d[k] = q < win_pos0 ? far[q] : wout[q]; } }
                            else {
                                const uint8_t* ms = d - off;
                                uint32_t k = 0;
                                if (off >= 4) {
                                    for (; k + 4 <= ml; k += 4) {
                                        const uint8_t b0 = ms[k], b1 = ms[k + 1], b2 = ms[k + 2], b3 = ms[k + 3];
                                        d[k] = b0; d[k + 1] = b1; d[k + 2] = b2; d[k + 3] = b3;
                                    }
                                }
                                for (; k < ml; k++) d[k] = ms[k];             // byte-serial: overlap (off < ml) is fine
                            }
                        }
                        uint32_t big = __ballot_sync(TS_FULL, ready && ml > 64);
                        while (big) {                                         // long matches: 32 lanes per match
                            const uint32_t f = (uint32_t)__ffs((int)big) - 1;
                            big &= big - 1;
                            const uint32_t fm = __shfl_sync(TS_FULL, m_start, f), fl = __shfl_sync(TS_FULL, ml, f), fo = __shfl_sync(TS_FULL, off, f);
                            uint8_t* dd = wout + fm;
                            const uint32_t fs = fm - fo;                      // source position
                            if (fo >= 32) {
                                for (uint32_t k0 = 0; k0 < fl; k0 += 32) {
                                    const uint32_t k = k0 + lane;
                                    if (k < fl) { const uint32_t q = fs + k; dd[k] = q < win_pos0 ? far[q] : wout[q]; }
                                    if (fo < fl) __syncwarp();               // later strides may read what this one wrote
                                }
                            } else {
                                // periodic source: the fo bytes before the destination, all of them already written
                                for (uint32_t k = lane; k < fl; k += 32) { const uint32_t q = fs + k % fo; dd[k] = q < win_pos0 ? far[q] : wout[q]; }
                            }
                        }
                        __syncwarp();                                         // the warp's copies of this round are ordered before ...
                        if (ready) done = true;
                        const uint32_t now = __ballot_sync(TS_FULL, !done);
                        if (now != pend) {                                    // ... the release of their done bits
                            if (lane == 0) { __threadfence_block(); *(volatile uint32_t*)&sh->dbits[w] = ~now; }
                            pend = now;
                        }
                    }
                }
            }
            zx_barrier<T>();                                              // the step is complete
            op += tot_o; lp += tot_l;
        }
        // trailing literals of the block
        {
            if (lp > regen || (uint64_t)(op - blk_op0) + (regen - lp) > room) {
                if (tid == 0) sh->err = -1;
                zx_barrier<T>();
                return op;
            }
            const uint32_t ll = regen - lp;
            if (rle_lit < 0x100) { for (uint32_t k = tid; k < ll; k += T) wout[op + k] = (uint8_t)rle_lit; }
            else { for (uint32_t k = tid; k < ll; k += T) wout[op + k] = lit[lp + k]; }
            op += ll;
        }
        zx_barrier<T>();
        if (per_block) { zx_flush<T>(far + blk_op0, win, op - blk_op0, tid); }
        if (tid == 0) {                                                   // repeat offsets after the block
            uint32_t nr[3];
            for (int k = 0; k < 3; k++) {                                 // an offset that underflowed is only an error if it is used
                const uint32_t of = m.rep[k];
                if (of & ZD_OFF_SYM) {
                    uint32_t d;
                    const uint32_t r = zd_sym_base(of, R0, R1, R2, &d);
                    nr[k] = r > d ? r - d : 0;
                } else nr[k] = of;
            }
            sh->rep[0] = nr[0]; sh->rep[1] = nr[1]; sh->rep[2] = nr[2];
        }
        zx_barrier<T>();                                                  // (also: the flushed bytes are visible before the next block reads `far`)
        if (sh->err) return op;
    }
    return op;
}

// ------------------------------------------------------------------------------------------ frame header
// Returns header size (0 on error); fcs = 0xffffffffffffffff when absent.
__device__ __forceinline__ uint32_t zd_frame_header(const uint8_t* p, uint32_t n, uint64_t* fcs) {
    if (n < 6) return 0;
    if ((p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24)) != zf::MAGIC) return 0;
    const uint32_t fhd = p[4];
    const uint32_t fcs_flag = fhd >> 6, single = (fhd >> 5) & 1, dict = fhd & 3;
    if (fhd & 0x08) return 0;                            // reserved bit
    uint32_t pos = 5;
    if (!single) {                                       // Window_Descriptor (the window is the whole output buffer here);
        if ((uint32_t)(p[5] >> 3) + 10 > 31) return 0;   // libzstd refuses a windowLog above ZSTD_WINDOWLOG_MAX (31)
        pos += 1;
    }
    const uint32_t dl = dict == 0 ? 0 : dict == 1 ? 1 : dict == 2 ? 2 : 4;
    const uint32_t fl = fcs_flag == 0 ? (single ? 1 : 0) : fcs_flag == 1 ? 2 : fcs_flag == 2 ? 4 : 8;
    if (pos + dl + fl > n) return 0;
    for (uint32_t k = 0; k < dl; k++) if (p[pos + k]) return 0;   // a Dictionary_ID other than 0: the reader has no dictionary ("Dictionary mismatch" in libzstd)
    pos += dl;
    uint64_t v = 0xffffffffffffffffull;
    if (fl) {
        v = 0;
        for (uint32_t k = 0; k < fl; k++) v |= (uint64_t)p[pos + k] << (8 * k);
        if (fl == 2) v += 256;
    }
    *fcs = v;
    return pos + fl;
}

// What may follow the last block of the frame inside the chunk: the 4-byte Content_Checksum when the frame header announces one
// (verified by xxh64_warp_low32 in the last kernel of the batch), then only skippable
// frames (ZSTD_decompress steps over those).  Anything else — trailing bytes, a second frame — is what zstd-jni's
// Zstd.decompress(chunk, size) rejects ("Src size is incorrect" / "Destination buffer is too small"), so it is corrupt here too.
__device__ __forceinline__ bool zd_frame_tail_ok(const uint8_t* p, uint32_t n, uint32_t pos) {
    if (p[4] & 0x04) { if (pos + 4 > n) return false; pos += 4; }
    while (pos < n) {
        if (pos + 8 > n) return false;
        const uint32_t magic = p[pos] | (p[pos + 1] << 8) | (p[pos + 2] << 16) | ((uint32_t)p[pos + 3] << 24);
        const uint32_t size = p[pos + 4] | (p[pos + 5] << 8) | (p[pos + 6] << 16) | ((uint32_t)p[pos + 7] << 24);
        if ((magic & 0xfffffff0u) != 0x184D2A50u || size > n - pos - 8) return false;
        pos += 8 + size;
    }
    return true;
}

// Content_Checksum (RFC 8878 3.1.1): the low 32 bits of XXH64(content, seed 0), little-endian after the last block.  libzstd —
// hence zstd-jni's Zstd.decompress, DecompressionChunkEnumeration.java:41-45 — verifies it when the header announces one, and so
// does this decoder: frames of this library's writer carry one with TSGPU_FLAG_ZSTD_CHECKSUM.  xxh64_warp_low32 (xxh64.cuh)
// stages the decoded bytes through the warp's shared-memory working set, which is free by then.
static_assert(sizeof(ZdWarpCtx) % 16 == 0 && sizeof(ZdWarpCtx) >= XXH_STAGE_BYTES, "checksum staging aliases a warp's working set");

// ------------------------------------------------------------------------------------------ kernel 1: index
__global__ void __launch_bounds__(128) zstd_dec_index_kernel(const __grid_constant__ ZstdDecArgs A) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t chunk = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (chunk >= A.n_chunks) return;
    if (lane != 0) return;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t n = A.in_len[chunk];
    uint64_t fcs = 0;
    for (int k = 0; k < ZD_INFO; k++) info[k] = 0;
    if (A.status[chunk] != 0) { A.out_len[chunk] = 0; info[3] = 2; return; }      // e.g. tag mismatch upstream: nothing to decode
    if (n > A.in_cap) { A.status[chunk] = ZD_ST_CORRUPT; A.out_len[chunk] = 0; info[3] = 2; return; }
    const uint32_t hs = zd_frame_header(p, n, &fcs);
    // "Invalid decompressed size" (DecompressionChunkEnumeration.java:41-44): no FCS, or larger than a chunk can be
    if (!hs || fcs == 0xffffffffffffffffull || fcs > A.chunk_cap) { A.status[chunk] = ZD_ST_CORRUPT; A.out_len[chunk] = 0; info[3] = 2; return; }
    A.out_len[chunk] = (uint32_t)fcs;
    info[0] = (uint32_t)fcs; info[4] = hs;
    // walk the block headers; the frame is "ours" when it has exactly ceil(FCS / ZB) blocks
    const uint32_t want = fcs ? (uint32_t)((fcs + ZB - 1) / ZB) : 1;
    uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
    uint32_t pos = hs, nblk = 0;
    bool ok = true, last = false;
    while (!last) {
        if (pos + 3 > n) { ok = false; break; }
        const ZdBlkHdr bh = zd_block_header(p + pos);
        last = bh.last;
        const uint32_t type = bh.type, bsz = bh.size;
        if (type == 3) { ok = false; break; }
        if (nblk < A.blocks_per_chunk) bo[nblk] = pos;
        nblk++;
        pos += 3 + (type == 1 ? 1 : bsz);
        if (pos > n || nblk > want + 1) { if (pos > n) ok = false; break; }
    }
    if (ok && last && !zd_frame_tail_ok(p, n, pos)) ok = false;
    if (ok && last && (p[4] & 0x04)) info[9] = pos;                               // Content_Checksum at pos: verified by the last kernel of the batch
    if (!ok) { A.status[chunk] = ZD_ST_CORRUPT; info[3] = 2; return; }
    info[1] = nblk;
    // Frames whose blocks look like this library's (ceil(FCS / 8 KiB) blocks) are first tried region by region (64 KiB of
    // output per CTA, assembled in shared memory); every assumption is verified while executing and a violation only sends
    // the frame to the frame-level executor.
    info[2] = (last && nblk == want && nblk <= A.blocks_per_chunk) ? 1 : 0;
    info[5] = (last && nblk <= A.blocks_per_chunk) ? 1 : 0;                       // entropy stage per block + CTA executors (else: serial kernel)
    // Speed-mode frames of this library have self-contained blocks (own tables, no match leaves the block): guessed from the
    // second block — it inherits nothing — and verified by the kernels that rely on it (a wrong guess costs time, never bytes).
    if (info[2]) {
        uint32_t indep = 1;
        if (nblk >= 2) {
            const uint32_t p1 = bo[1];
            const ZdBlkHdr h1 = zd_block_header(p + p1);
            if (h1.type == 2 && h1.size >= 2) {
                const uint32_t t1 = p[p1 + 3] & 3;
                if (t1 == 3) indep = 0;                                           // Treeless literals
                // (Repeat_Mode tables behind Raw / RLE literals are found by the entropy stage itself)
            }
        }
        info[8] = indep;
    }
}

// ------------------------------------------------------------------------------------------ kernel 4: serial fallback
// One warp per frame, blocks in order.  Only frames the parallel stages hand back (a sequence field too wide for the packed
// sequence word, more blocks than the index holds) come here.
__global__ void __launch_bounds__(ZD_WPB * 32) zstd_dec_frames_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(smem);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.x * ZD_WPB + warp;
    if (chunk >= A.n_chunks) return;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (info[3] & 2) return;                             // already failed in the index pass
    if (info[5]) {                                       // the parallel stages own this frame; this kernel runs after them (stream order)
        if (info[9] && A.status[chunk] == 0) {           // ... so a Content_Checksum, if the frame carries one, can be verified here
            const uint8_t* f = A.in_base + A.in_off[chunk] + info[9];
            const uint32_t want = f[0] | (f[1] << 8) | (f[2] << 16) | ((uint32_t)f[3] << 24);
            uint64_t* stage = (uint64_t*)(smem + (size_t)warp * sizeof(ZdWarpCtx));
            const uint32_t got = xxh64_warp_low32(A.out_base + A.out_off[chunk], info[0], stage, lane);
            if (lane == 0 && got != want) { A.status[chunk] = ZD_ST_CORRUPT; A.out_len[chunk] = 0; }
        }
        return;
    }
    if (lane == 0) atomicAdd(&A.stats[3], 1ull);
    ZdWarpCtx* cx = (ZdWarpCtx*)(smem + (size_t)warp * sizeof(ZdWarpCtx));
    const uint32_t fcs = info[0];
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t n = A.in_len[chunk];
    uint8_t* dst = A.out_base + A.out_off[chunk];
    uint8_t* litbuf = A.lits_general + (size_t)chunk * ZD_LIT_GENERAL;
    if (lane == 0) {
        cx->err = 0; cx->huf_valid = 0; cx->ll_valid = 0; cx->ml_valid = 0; cx->of_valid = 0;
        cx->rep[0] = 1; cx->rep[1] = 4; cx->rep[2] = 8;
    }
    __syncwarp();
    uint32_t pos = info[4];
    uint64_t op = 0;
    bool last = false, bad = false;
    while (!last && !bad) {
        if (pos + 3 > n) { bad = true; break; }
        const ZdBlkHdr bh = zd_block_header(p + pos);
        last = bh.last;
        const uint32_t type = bh.type, bsz = bh.size;
        const uint32_t room = (uint32_t)min((uint64_t)zf::BLOCK_MAX, (uint64_t)fcs - op);
        if (type == 0) {
            if (bsz > room || pos + 3 + bsz > n) { bad = true; break; }
            for (uint32_t k = lane; k < bsz; k += 32) dst[op + k] = p[pos + 3 + k];
            op += bsz; pos += 3 + bsz;
        } else if (type == 1) {
            if (bsz > room || pos + 4 > n) { bad = true; break; }
            const uint8_t v = p[pos + 3];
            for (uint32_t k = lane; k < bsz; k += 32) dst[op + k] = v;
            op += bsz; pos += 4;
        } else if (type == 2) {
            if (pos + 3 + bsz > n || bsz > zf::BLOCK_MAX) { bad = true; break; }
            const uint32_t made = zd_compressed_block(p + pos + 3, bsz, dst + op, op, room, cx, litbuf, lane);
            if (cx->err) { bad = true; break; }
            op += made; pos += 3 + bsz;
        } else { bad = true; break; }
        __syncwarp();
        __threadfence_block();
    }
    bool sum_bad = false;
    if (!bad && op == fcs && (p[4] & 0x04) && pos + 4 <= n) {
        __syncwarp();
        __threadfence_block();
        const uint32_t want = p[pos] | (p[pos + 1] << 8) | (p[pos + 2] << 16) | ((uint32_t)p[pos + 3] << 24);
        sum_bad = xxh64_warp_low32(dst, (uint32_t)fcs, (uint64_t*)cx, lane) != want;   // (the block walk is done with cx)
    }
    if (lane == 0) {
        if (bad || op != fcs || sum_bad || !zd_frame_tail_ok(p, n, pos)) { A.status[chunk] = ZD_ST_CORRUPT; A.out_len[chunk] = 0; }
    }
}

// ------------------------------------------------------------------------------------------ kernels 3a / 3b: parallel general path
// 3a: one WARP per block — entropy stage.  Tables a block inherits are rebuilt by replaying table definitions, starting
// at the nearest earlier block that defines all three FSE tables itself (and, for treeless literals, after loading the
// latest Huffman tree): libzstd frames inherit the tree in nearly every block, frames of this library's compressor inherit
// everything from the first block of their 64 KiB region.
__device__ __forceinline__ bool zd_blk_hdr(const uint8_t* p, const uint32_t* bo, uint32_t j, uint32_t* pos, uint32_t* type, uint32_t* bsz) {
    const uint32_t pj = bo[j];
    const ZdBlkHdr h = zd_block_header(p + pj);
    *pos = pj; *type = h.type; *bsz = h.size;
    return *type == 2 && *bsz <= zf::BLOCK_MAX;
}

__global__ void __launch_bounds__(ZD_WPB * 32) zstd_dec_par_entropy_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(smem);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.y, b = blockIdx.x * ZD_WPB + warp;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || b >= info[1]) return;
    if (info[8] && !(info[3] & 4)) return;                                // the independent-block entropy stage did this frame
    ZdWarpCtx* cx = (ZdWarpCtx*)(smem + (size_t)warp * sizeof(ZdWarpCtx));
    ZdBlkMeta* meta = (ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk + b;
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t n = A.in_len[chunk];
    const uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
    uint32_t pos, type, bsz;
    const bool comp = zd_blk_hdr(p, bo, b, &pos, &type, &bsz);
    if (type != 2) { if (lane == 0) meta->status = 1; return; }           // Raw / RLE blocks need no entropy stage
    if (!comp || pos + 3 + bsz > n) { if (lane == 0) meta->status = 2; return; }
    if (lane == 0) { cx->err = 0; cx->huf_valid = 0; cx->ll_valid = 0; cx->ml_valid = 0; cx->of_valid = 0; }
    __syncwarp();
    const uint32_t inherits = zd_block_inherits(p + pos + 3, bsz, lane);
    if (inherits & 3) {
        ZdLitSec L;                                                       // (what the tree loads parse; not needed here)
        // j0: where the replay of FSE definitions has to start (none needed: j0 = b)
        uint32_t j0 = b;
        bool tree_in_replay = false;
        if (inherits & 2) {
            bool found = false;
            while (j0 > 0 && !found) {
                j0--;
                uint32_t pj, tj, bj;
                if (!zd_blk_hdr(p, bo, j0, &pj, &tj, &bj)) continue;
                const uint32_t r = zd_block_inherits(p + pj + 3, bj, lane);
                if ((r & 6) == 0) { found = true; tree_in_replay = (r & 8) != 0; }   // defines LL, OF and ML itself
            }
            if (!found) { if (lane == 0) cx->err = -1; __syncwarp(); }   // Repeat_Mode without any definition before it
        }
        // the Huffman tree: the latest block with Compressed_Literals before the replay range — unless the replay range
        // starts with one (every treeless block inside it is then served by the replay itself)
        if (!cx->err && !tree_in_replay && ((inherits & 1) || j0 < b)) {
            bool found = false;
            for (uint32_t j = j0; j-- > 0 && !found; ) {
                uint32_t pj, tj, bj;
                if (!zd_blk_hdr(p, bo, j, &pj, &tj, &bj) || bj < 1 || (p[pj + 3] & 3) != 2) continue;
                found = true;
                zd_block_huf_only(p + pj + 3, bj, cx, lane, L);
                __syncwarp();
            }
            // not found: fine as long as nothing treeless shows up before a tree (the decode reports it otherwise)
        }
        for (uint32_t j = j0; j < b && !cx->err; j++) {
            uint32_t pj, tj, bj;
            if (!zd_blk_hdr(p, bo, j, &pj, &tj, &bj)) continue;
            if ((inherits & 2) || (p[pj + 3] & 3) == 2) {                 // FSE replay, or at least the trees on the way
                if (inherits & 2) zd_block_tables(p + pj + 3, bj, cx, lane);
                else zd_block_huf_only(p + pj + 3, bj, cx, lane, L);
            }
            __syncwarp();
        }
    }
    if (!cx->err) {
        ZdParIO io;
        io.lit_arena = A.par_lits + (size_t)chunk * A.par_lit_cap; io.lit_cap = A.par_lit_cap; io.lit_bump = info + 6;
        io.seq_arena = A.par_seqs + (size_t)chunk * A.par_seq_cap; io.seq_cap = A.par_seq_cap; io.seq_bump = info + 7;
        zd_block_entropy(p + pos + 3, bsz, cx, io, meta, lane);
    }
    __syncwarp();
    if (lane == 0) meta->status = cx->err == 0 ? 1u : cx->err == 2 ? 3u : 2u;
}

// 3b: one CTA per 64 KiB REGION of frames that look like this library's: the region's 8 blocks are executed into shared
// memory (matches never leave the region, so every dependent copy is a shared-memory access) and flushed with 128-bit
// stores.  Anything unexpected — an offset reaching before the region, a repeat offset carried in from an earlier region,
// a region that does not regenerate exactly its share — sends the whole frame to the frame-level executor below.
constexpr uint32_t ZX_REGION_SMEM = ZR;
__global__ void __launch_bounds__(ZX_T, 2) zstd_dec_regions_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(obuf);
    __shared__ ZxShared<ZX_T> sh;
    const uint32_t tid = threadIdx.x;
    const uint32_t chunk = blockIdx.y, region = blockIdx.x;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || !info[2] || (info[3] & 2)) return;
    if (info[8] && !(info[3] & 4)) return;                                // executed block by block (or handed to the frame executor)
    const uint32_t fcs = info[0], nblk = info[1];
    if ((uint64_t)region * ZR >= fcs) return;
    const uint32_t want = min(ZR, fcs - region * ZR);
    const uint32_t b0 = region * ZR_SLICES, b1 = min(nblk, b0 + ZR_SLICES);
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
    const ZdBlkMeta* meta = (const ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk;
    const uint32_t made = zx_execute_blocks<ZX_T>(p, bo, meta, b0, b1, obuf, ZR, nullptr, false, want,
                                            A.par_lits + (size_t)chunk * A.par_lit_cap, A.par_seqs + (size_t)chunk * A.par_seq_cap,
                                            A.in_len[chunk], &sh, tid, region != 0);
    if (sh.err || made != want) {
        if (tid == 0) {
            if (sh.err == 3) info[5] = 0;                                 // a field too wide for the sequence word: serial kernel
            else atomicOr(&info[3], 1u);                                  // not regional after all (or corrupt): the frame executor decides
        }
        return;
    }
    if (tid == 0) atomicAdd(&A.stats[0], 1ull);
    zx_flush<ZX_T>(A.out_base + A.out_off[chunk] + (size_t)region * ZR, obuf, made, tid);
}

// 3c: one CTA per frame — execution stage straight into the frame's output in HBM (what libzstd-written frames need: their
// matches reach back up to the whole window).
constexpr uint32_t ZX_FRAME_SMEM = zf::BLOCK_MAX + 32 * ZX_TF * 2;      // the window is the current block; + the pointer array of a step
__global__ void __launch_bounds__(ZX_TF, 1) zstd_dec_par_execute_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(wbuf);
    __shared__ ZxShared<ZX_TF> sh;
    const uint32_t tid = threadIdx.x;
    const uint32_t chunk = blockIdx.x;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || (info[3] & 2)) return;
    if (info[2] && !(info[3] & 1)) return;                                // the region / block executors finished this frame
    if (tid == 0) atomicAdd(&A.stats[info[2] ? 1 : 2], 1ull);
    const uint32_t fcs = info[0], nblk = info[1];
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
    const ZdBlkMeta* meta = (const ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk;
    uint16_t* pj = (uint16_t*)(wbuf + zf::BLOCK_MAX);
    for (uint32_t r = tid; r < 32u * ZX_TF; r += ZX_TF) pj[r] = (uint16_t)r;
    __syncthreads();
    const uint32_t made = zx_execute_blocks<ZX_TF, true>(p, bo, meta, 0, nblk, wbuf, zf::BLOCK_MAX, A.out_base + A.out_off[chunk], true, fcs,
                                            A.par_lits + (size_t)chunk * A.par_lit_cap, A.par_seqs + (size_t)chunk * A.par_seq_cap,
                                            A.in_len[chunk], &sh, tid, false, pj);
    if (tid == 0) {
        if (sh.err == 3) info[5] = 0;                                     // a field too wide for the sequence word: the serial kernel decodes this frame
        else if (sh.err || made != fcs) { A.status[chunk] = ZD_ST_CORRUPT; A.out_len[chunk] = 0; }
    }
}


// ------------------------------------------------------------------------------------------ kernels 2a / 2b / 2c: independent blocks
// Frames of this library's SPEED mode: every 8 KiB block carries its own tables and no match leaves it.  The serial parts of a
// block's entropy stage (header parsing, table descriptions, the FSE state chain: one lane, ~55 instructions per sequence)
// then no longer need a warp each — one warp takes EIGHT blocks, four lanes per block:
//   * lane 4g (the leader of block g) parses headers and walks block g's state chain, all eight chains at once;
//   * lanes 4g..4g+3 decode the four Huffman streams of block g, 32 streams at once;
//   * table fills and the per-sequence value extraction stay warp-wide, block after block.
// Such a warp is latency-bound, so what matters is how many fit on an SM, i.e. shared memory per block: literals and
// sequences are two kernels with lean contexts (literals: the 4 KiB Huffman table, 5 warps per SM; sequences: three tables of
// at most 2^7 cells — what the speed-mode writer emits — 9 warps = 72 chains per SM), and no serial loop waits for HBM:
// the bytes a stream is about to consume are staged in shared memory, 64 / 128 at a time, by loads issued together.
// Literals and sequences go to FIXED slots of the frame's arenas (block b: literals at b * ZB, sequences at b * ZB / 3), in
// the format of the general entropy stage, so every executor can consume them.  Anything a self-contained speed-mode block
// does not contain (Treeless literals, Repeat_Mode, a repeat-offset code, larger tables, more than ZB bytes) makes these
// kernels REFUSE the frame: the general entropy stage then redoes it — they never declare a frame corrupt themselves.
constexpr int ZDI_G = 8;                                  // blocks per warp
constexpr uint32_t ZDI_SEQ_SLOT = ZB / 3;                 // most sequences ZB bytes of output can come from (minimum match 3)

struct ZdLitCtx {                                         // literal phase of one block
    uint16_t huf[1 << zf::HUF_MAX_LOG];
    uint16_t hstart[256];
    uint8_t weights[256];
    zf::FseDEntry wt[1 << zf::HUFW_MAX_LOG];
    uint32_t rank_start[16];
    uint8_t symbol_of[1 << zf::HUFW_MAX_LOG];
    uint16_t next[16];
    int16_t norm[16];
    uint32_t huf_nw, huf_log, huf_valid;
    int32_t err;
    static constexpr int kTabLogCap = 0;
};
struct ZdSeqCtx {                                         // sequence phase of one block
    static constexpr int kTabLogCap = 7;
    zf::FseDEntry ll[1 << kTabLogCap], ml[1 << kTabLogCap], of[1 << kTabLogCap];
    int16_t norm3[3][64];
    uint32_t cum[65];
    uint8_t symbol_of[1 << kTabLogCap];
    uint16_t next[64];
    uint32_t s_ll[32], s_ml[32];
    uint32_t stage[36];                                   // 128 bytes of the bit stream below the cursor (+ padding for the funnel shift)
    uint32_t pend_log[3], pend_nsym[3];
    uint32_t ll_log, ml_log, of_log, ll_valid, ml_valid, of_valid;
    int32_t err;
};
constexpr uint32_t ZDL_STAGE_WORDS = 17;                  // per lane: 64 bytes of its Huffman stream (+ one word for the funnel shift)
constexpr uint32_t ZDL_SMEM_BYTES = ZDI_G * sizeof(ZdLitCtx) + 32 * ZDL_STAGE_WORDS * 4;
constexpr uint32_t ZDS_SMEM_BYTES = ZDI_G * sizeof(ZdSeqCtx);
static_assert(5 * (ZDL_SMEM_BYTES + 1024) <= 228 * 1024, "five literal warps per SM");
static_assert(9 * (ZDS_SMEM_BYTES + 1024) <= 228 * 1024, "nine sequence warps per SM");

// Table fill for the lean literal kernel: symbols with few cells by a lane each, symbols with many cells by the warp.
__device__ __forceinline__ void zd_fill_huf_lean(ZdLitCtx* cx, uint32_t lane) {
    const uint32_t nw = cx->huf_nw, max_bits = cx->huf_log;
    for (uint32_t s0 = 0; s0 < nw; s0 += 32) {
        const uint32_t sy = s0 + lane;
        const uint32_t w = sy < nw ? cx->weights[sy] : 0u;
        const uint32_t len = w ? 1u << (w - 1) : 0u, at = w ? cx->hstart[sy] : 0u;
        const uint16_t e = (uint16_t)(sy | ((max_bits + 1 - w) << 8));
        if (len && len < 16) for (uint32_t k = 0; k < len; k++) cx->huf[at + k] = e;
        uint32_t big = __ballot_sync(TS_FULL, len >= 16);
        while (big) {
            const uint32_t f = (uint32_t)__ffs((int)big) - 1;
            big &= big - 1;
            const uint32_t fa = __shfl_sync(TS_FULL, at, f), fl = __shfl_sync(TS_FULL, len, f), fe = __shfl_sync(TS_FULL, (uint32_t)e, f);
            uint32_t* t2 = (uint32_t*)(cx->huf + fa);                     // fa is a multiple of fl >= 16: word aligned
            for (uint32_t k = lane; k < fl / 2; k += 32) t2[k] = fe | (fe << 16);
        }
    }
    __syncwarp();
}

// One Huffman stream by one lane, destination in global memory.  The 64 bytes below the cursor are staged in the lane's
// column of `stg` (word j at stg[32 * j]: conflict-free) by 16 loads issued together; ten groups of four symbols (<= 440
// bits) are decoded per staging, each leaving as one 32-bit store.  The first symbols (until the destination is aligned) and
// the last ones (fewer than 44 bits left: peeks zero-extend past the start of the stream) take the generic reader.
// `base` / `lim`: 4-byte aligned bounds of the frame's buffer — staging never reads outside them.
__device__ __forceinline__ bool zd_huf_stream_staged(const uint16_t* __restrict__ huf, uint32_t log, const uint8_t* src, uint32_t size,
                                                     uint8_t* dst, uint32_t count, uint32_t* stg, const uint8_t* base, const uint8_t* lim) {
    ZdBack b;
    if (!zd_back_init(b, src, size)) return false;
    uint32_t i = 0;
    const uint32_t head = min(count, (4u - (uint32_t)((uintptr_t)dst & 3)) & 3u);
    for (; i < head; i++) {
        const uint16_t e = huf[zd_back_peek(b, log)];
        dst[i] = (uint8_t)e;
        b.bits -= (int32_t)(e >> 8);
    }
    if (b.bits < 0) return false;
    const uint32_t mask = (1u << log) - 1;
    int32_t bits = b.bits;
    while (i + 4 <= count && bits >= 44) {
        const int32_t tb = (bits + 7) >> 3;
        const uint8_t* a0 = (const uint8_t*)(((uintptr_t)(src + tb) - 60) & ~(uintptr_t)3);
        if (a0 < base) a0 = base;
        const int32_t sbit0 = (int32_t)(a0 - src) * 8;                   // stream bit index of stg word 0, bit 0 (may be negative)
        uint32_t t[16];                                                  // all sixteen loads in flight before the first store
        _Pragma("unroll")
        for (int j = 0; j < 16; j++) { const uint8_t* q = a0 + 4 * j; t[j] = q < lim ? __ldg((const uint32_t*)q) : 0u; }
        _Pragma("unroll")
        for (int j = 0; j < 16; j++) stg[32 * j] = t[j];
        for (int r = 0; r < 10 && i + 4 <= count && bits >= 44; r++) {
            uint32_t out = 0;
            _Pragma("unroll")
            for (int k = 0; k < 4; k++) {
                const uint32_t rel = (uint32_t)(bits - (int32_t)log - sbit0);
                const uint32_t v = __funnelshift_r(stg[32 * (rel >> 5)], stg[32 * ((rel >> 5) + 1)], rel & 31) & mask;
                const uint16_t e = huf[v];
                out |= (uint32_t)(e & 0xff) << (8 * k);
                bits -= (int32_t)(e >> 8);
            }
            *(uint32_t*)(dst + i) = out;
            i += 4;
        }
    }
    b.bits = bits; b.cbase = 0x3fffffff;
    for (; i < count; i++) {
        const uint16_t e = huf[zd_back_peek(b, log)];
        dst[i] = (uint8_t)e;
        b.bits -= (int32_t)(e >> 8);
        if (b.bits < 0) return false;
    }
    return b.bits == 0;
}

// Common prologue: which block this group of four lanes owns.  live: a Compressed_Block to decode; refuse: malformed framing.
struct ZdiBlock { uint32_t b, blk_off, bsize; bool live; uint32_t refuse; };
__device__ __forceinline__ ZdiBlock zdi_block(const ZstdDecArgs& A, uint32_t chunk, uint32_t nblk, uint32_t g) {
    ZdiBlock r; r.b = blockIdx.x * ZDI_G + g; r.blk_off = 0; r.bsize = 0; r.live = false; r.refuse = 0;
    if (r.b < nblk) {
        const uint8_t* p = A.in_base + A.in_off[chunk];
        const uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
        uint32_t pos, type, bsz;
        const bool comp = zd_blk_hdr(p, bo, r.b, &pos, &type, &bsz);
        if (type == 2) {
            if (!comp || pos + 3 + bsz > A.in_len[chunk]) r.refuse = 1;
            else { r.live = true; r.blk_off = pos + 3; r.bsize = bsz; }
        }
    }
    return r;
}

// 2a: literals.
__global__ void __launch_bounds__(32) zstd_dec_blk_literals_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(smem);
    const uint32_t lane = threadIdx.x, g = lane >> 2, sub = lane & 3, lead = lane & ~3u;
    const uint32_t chunk = blockIdx.y;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || !info[8] || (info[3] & 6)) return;                     // (bit 4 set by another warp of this launch: nothing left to win)
    const uint32_t nblk = info[1];
    if (blockIdx.x * ZDI_G >= nblk) return;
    ZdLitCtx* ctx = (ZdLitCtx*)smem;
    ZdLitCtx* cx = ctx + g;
    uint32_t* stg = (uint32_t*)(smem + ZDI_G * sizeof(ZdLitCtx)) + lane;
    stg[32 * 16] = 0;
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint8_t* base = (const uint8_t*)((uintptr_t)p & ~(uintptr_t)3);
    const uint8_t* lim = (const uint8_t*)(((uintptr_t)p + A.in_len[chunk] + 3) & ~(uintptr_t)3);
    ZdiBlock B = zdi_block(A, chunk, nblk, g);
    const uint8_t* blk = p + B.blk_off;
    ZdBlkMeta* meta = (ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk + B.b;
    uint8_t* litbuf = A.par_lits + (size_t)chunk * A.par_lit_cap + (size_t)B.b * ZB;
    bool live = B.live;
    uint32_t refuse = B.refuse;

    // header + tree description (leaders), table fill (warp), streams (4 lanes per block)
    ZdLitSec L{0, 0, 0, 0, 1, 0};
    if (live && sub == 0) {
        cx->err = 0; cx->huf_valid = 0;
        ZdLitSec h;
        if (!zd_parse_lit_header(blk, B.bsize, ZB, ZB, true, cx, h) || cx->err) refuse = 1;
        else L = h;
    }
    const uint32_t ltype = __shfl_sync(TS_FULL, L.type, lead), lhs = __shfl_sync(TS_FULL, L.hs, lead), regen = __shfl_sync(TS_FULL, L.regen, lead);
    const uint32_t lcomp = __shfl_sync(TS_FULL, L.comp, lead), streams = __shfl_sync(TS_FULL, L.streams, lead), tree = __shfl_sync(TS_FULL, L.tree, lead);
    refuse = __shfl_sync(TS_FULL, refuse, lead);
    live = live && !refuse;
    for (uint32_t gg = 0; gg < ZDI_G; gg++) {
        if (__shfl_sync(TS_FULL, (uint32_t)(live && ltype == 2), gg * 4)) zd_fill_huf_lean(ctx + gg, lane);
    }
    __syncwarp();
    if (live && ltype == 2) {
        const uint8_t* hsrc = blk + lhs + tree;
        const uint32_t hsize = lcomp - tree;
        bool ok = true;
        if (streams == 1) {
            if (sub == 0) ok = zd_huf_stream_staged(cx->huf, cx->huf_log, hsrc, hsize, litbuf, regen, stg, base, lim);
        } else {
            ZdHufStream s;
            ok = zd_huf4_stream(hsrc, hsize, regen, sub, s) &&
                 zd_huf_stream_staged(cx->huf, cx->huf_log, hsrc + s.off, s.size, litbuf + s.first, s.count, stg, base, lim);
        }
        if (!ok) refuse = 1;
    }
    {   // a group's verdict is the OR of its four lanes
        const uint32_t bad = __ballot_sync(TS_FULL, refuse != 0);
        refuse = (bad >> lead) & 15u ? 1u : 0u;
    }
    if (B.b < nblk && sub == 0) {
        if (refuse) atomicOr(&info[3], 4u);
        else if (live) {
            meta->lit_kind = ltype == 0 ? 1u : ltype == 1 ? 2u : 0u;
            meta->lit_off = ltype == 0 ? lhs : ltype == 1 ? (uint32_t)blk[lhs] : B.b * ZB;
            meta->regen = regen;
        }
    }
}

// 2b: sequences.
__global__ void __launch_bounds__(32) zstd_dec_blk_sequences_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(smem);
    const uint32_t lane = threadIdx.x, g = lane >> 2, sub = lane & 3, lead = lane & ~3u;
    const uint32_t chunk = blockIdx.y;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || !info[8] || (info[3] & 6)) return;
    const uint32_t nblk = info[1];
    if (blockIdx.x * ZDI_G >= nblk) return;
    ZdSeqCtx* ctx = (ZdSeqCtx*)smem;
    ZdSeqCtx* cx = ctx + g;
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint8_t* base = (const uint8_t*)((uintptr_t)p & ~(uintptr_t)3);
    const uint8_t* lim = (const uint8_t*)(((uintptr_t)p + A.in_len[chunk] + 3) & ~(uintptr_t)3);
    ZdiBlock B = zdi_block(A, chunk, nblk, g);
    const uint8_t* blk = p + B.blk_off;
    ZdBlkMeta* meta = (ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk + B.b;
    uint64_t* sq_base = A.par_seqs + (size_t)chunk * A.par_seq_cap + (size_t)blockIdx.x * ZDI_G * ZDI_SEQ_SLOT;
    bool live = B.live;
    uint32_t refuse = B.refuse;
    if (B.b < nblk && !live && !refuse && sub == 0) meta->status = 1;      // Raw / RLE blocks need no entropy stage

    // ---- header + table descriptions (leaders), table builds (warp)
    uint32_t nseq = 0, bs_off = 0, pend = 0, lsec = 0;
    if (live && sub == 0) {
        cx->err = 0; cx->ll_valid = 0; cx->ml_valid = 0; cx->of_valid = 0;
        uint32_t h[3];
        const ZdLitSec L = zd_lit_section(blk, B.bsize);
        if (!L.hs || (uint64_t)L.hs + L.comp > B.bsize) refuse = 1;
        else {
            lsec = L.hs + L.comp;                                         // where the sequences section starts
            if (!zd_parse_seq_header(blk + lsec, B.bsize - lsec, true, cx, h) || cx->err || h[0] > ZDI_SEQ_SLOT) refuse = 1;
            else { nseq = h[0]; bs_off = h[1]; pend = h[2]; }
        }
    }
    refuse = __shfl_sync(TS_FULL, refuse, lead);
    live = live && !refuse;
    for (uint32_t gg = 0; gg < ZDI_G; gg++) {
        const uint32_t pg = __shfl_sync(TS_FULL, live ? pend : 0u, gg * 4);
        for (int k = 0; k < 3; k++) if (pg & (1u << k)) zd_build_dtable_warp(k, ctx + gg, lane);
    }
    __syncwarp();
    const uint32_t bs_frame_off = __shfl_sync(TS_FULL, B.blk_off + lsec + bs_off, lead);      // the bit stream, relative to the frame
    const uint8_t* bs = p + bs_frame_off;
    int32_t bits = 0;                                                     // unread bits of the stream (leaders; shared per round)
    uint32_t st_ll = 0, st_of = 0, st_ml = 0;
    if (live && sub == 0 && nseq) {
        ZdBack br;
        bool ok = zd_back_init(br, bs, B.bsize - lsec - bs_off);
        if (ok) {
            st_ll = zd_back_read(br, cx->ll_log); st_of = zd_back_read(br, cx->of_log); st_ml = zd_back_read(br, cx->ml_log);
            if (br.bits < 0) ok = false;
        }
        if (!ok) refuse = 1;
        bits = br.bits;
    }
    // ---- rounds of up to 32 sequences per block: the group stages the 128 bytes below the cursor, the leaders walk their
    // chains (a chain stops early when it would leave the staged bytes), then the warp cuts the values out, block after block
    uint32_t s0 = 0;
    uint32_t r0 = zd_sym_rep(1), r1 = zd_sym_rep(2), r2 = zd_sym_rep(3);   // repeat offsets after the block
    while (true) {
        const bool more = live && !refuse && sub == 0 && s0 < nseq;
        const uint32_t more_mask = __ballot_sync(TS_FULL, more);
        if (!more_mask) break;
        // stage: bytes [a0, a0 + 128) with a0 + 128 > the byte holding the cursor
        const int32_t gbits = __shfl_sync(TS_FULL, bits, lead);
        const bool gmore = (more_mask >> lead) & 1u;
        const int32_t tb = (gbits + 7) >> 3;
        const uint8_t* a0 = (const uint8_t*)(((uintptr_t)(bs + tb) - 124) & ~(uintptr_t)3);
        if (a0 < base) a0 = base;
        const int32_t sbit0 = (int32_t)(a0 - bs) * 8;
        if (gmore) {
            uint32_t t[8];                                               // all eight loads in flight before the first store
            _Pragma("unroll")
            for (int j = 0; j < 8; j++) { const uint8_t* q = a0 + 4 * (sub * 8 + j); t[j] = q < lim ? __ldg((const uint32_t*)q) : 0u; }
            _Pragma("unroll")
            for (int j = 0; j < 8; j++) cx->stage[sub * 8 + j] = t[j];
        }
        __syncwarp();
        uint32_t cnt = 0;
        if (more) {
            const uint32_t want = min(32u, nseq - s0);
            const uint32_t* tof = (const uint32_t*)cx->of; const uint32_t* tml = (const uint32_t*)cx->ml; const uint32_t* tll = (const uint32_t*)cx->ll;
            const uint32_t n_upd = min(want, nseq - 1 - s0);             // sequences of this round that are followed by another one
            bool bad = false;
            uint32_t i = 0;
            for (; i < n_upd; i++) {
                const uint32_t eo = tof[st_of], em = tml[st_ml], el = tll[st_ll];
                const uint32_t t = eo + em + el;                         // bits 0..5: state-update bits, bits 6..11: extra bits
                const int32_t hi = bits - (int32_t)((t >> 6) & 63);
                const int32_t lo = hi - (int32_t)(t & 63);
                if (lo < sbit0) { if (lo < 0) bad = true; break; }       // leaves the staged bytes (or the stream: corrupt)
                cx->s_ll[i] = st_of | (st_ml << 10) | (st_ll << 20);
                cx->s_ml[i] = (uint32_t)(bits - sbit0);
                const uint32_t rel = (uint32_t)(lo - sbit0);
                uint32_t W = __funnelshift_r(cx->stage[rel >> 5], cx->stage[(rel >> 5) + 1], rel & 31);
                const uint32_t u_of = eo & 63, u_ml = em & 63, u_ll = el & 63;
                st_of = (eo >> 18) + (W & ((1u << u_of) - 1)); W >>= u_of;
                st_ml = (em >> 18) + (W & ((1u << u_ml) - 1)); W >>= u_ml;
                st_ll = (el >> 18) + (W & ((1u << u_ll) - 1));
                bits = lo;
            }
            if (!bad && i == n_upd && i < want) {                        // the block's last sequence: values only
                const uint32_t t = tof[st_of] + tml[st_ml] + tll[st_ll];
                const int32_t hi = bits - (int32_t)((t >> 6) & 63);
                if (hi >= sbit0 || hi < 0) {
                    cx->s_ll[i] = st_of | (st_ml << 10) | (st_ll << 20);
                    cx->s_ml[i] = (uint32_t)(bits - sbit0);
                    bits = hi;
                    if (bits != 0) bad = true;                           // the stream ends exactly with the last sequence's bits
                    i++;
                }
            }
            cnt = i;
            if (bad) { refuse = 1; cnt = 0; }
        }
        __syncwarp();
        for (uint32_t gg = 0; gg < ZDI_G; gg++) {
            const uint32_t c = __shfl_sync(TS_FULL, cnt, gg * 4);
            if (!c) continue;
            const uint32_t sbase = __shfl_sync(TS_FULL, s0, gg * 4);
            const ZdSeqCtx* cg = ctx + gg;
            const bool mine = lane < c;
            uint32_t ll = 0, ml = 3, ofv = 4;
            if (mine) {
                const uint32_t st = cg->s_ll[lane];
                const uint32_t end = cg->s_ml[lane];                     // staged bit index just above this sequence's bits
                const zf::FseDEntry eo = cg->of[st & 1023], em = cg->ml[(st >> 10) & 1023], el = cg->ll[st >> 20];
                const uint32_t nbo = eo.nb_extra, nbv = (uint32_t)em.nb_extra + el.nb_extra;
                const uint32_t ro = end - nbo, rv = ro - nbv;
                const uint32_t xo = __funnelshift_r(cg->stage[ro >> 5], cg->stage[(ro >> 5) + 1], ro & 31) & (uint32_t)((1ull << nbo) - 1);
                const uint32_t v = __funnelshift_r(cg->stage[rv >> 5], cg->stage[(rv >> 5) + 1], rv & 31) & (uint32_t)((1ull << nbv) - 1);
                ofv = (1u << eo.sym) + xo;
                ml = g_seq_tables.ml_base[em.sym] + (v >> el.nb_extra);
                ll = g_seq_tables.ll_base[el.sym] + (v & ((1u << el.nb_extra) - 1));
            }
            // a repeat-offset code, or a field the sequence word cannot hold: not a block of this kind
            const bool odd = mine && (ofv <= 3 || !zd_seq_fits(ofv, ll, ml));
            const uint32_t any_odd = __ballot_sync(TS_FULL, odd);
            const uint32_t of = ofv - 3;
            if (mine && !any_odd) sq_base[(size_t)gg * ZDI_SEQ_SLOT + sbase + lane] = zd_seq_pack(of, ll, ml);
            if (g == gg && any_odd) refuse = 1;
            zd_shift_in(of, c, g == gg, r0, r1, r2);
        }
        s0 += cnt;
        __syncwarp();                                    // stage / s_ll / s_ml are rewritten by the next round
    }
    refuse = __shfl_sync(TS_FULL, refuse, lead);
    if (B.b < nblk && sub == 0 && (live || refuse)) {
        if (refuse) { atomicOr(&info[3], 4u); meta->status = 2; }
        else {
            meta->nseq = nseq; meta->seq_off = B.b * ZDI_SEQ_SLOT;
            meta->rep[0] = r0; meta->rep[1] = r1; meta->rep[2] = r2;
            meta->status = 1;
        }
    }
}

// 2c: one WARP per block of such frames — the executor above with a "CTA" of 32: the block is assembled in 8 KiB of shared
// memory and flushed with 128-bit stores.  A match that reaches before its block, or a block that does not regenerate exactly
// its share, hands the frame to the frame executor (which consumes the same arenas).
constexpr int ZXB_WPB = 4;
constexpr uint32_t ZXB_SMEM_BYTES = ZXB_WPB * ZB;
__global__ void __launch_bounds__(ZXB_WPB * 32, 6) zstd_dec_indep_execute_kernel(const __grid_constant__ ZstdDecArgs A) {
    TS_DYN_SMEM(wins);
    __shared__ ZxShared<32> shs[ZXB_WPB];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t chunk = blockIdx.y, b = blockIdx.x * ZXB_WPB + warp;
    uint32_t* info = A.info + (size_t)chunk * ZD_INFO;
    if (!info[5] || !info[8] || (info[3] & 6)) return;
    const uint32_t fcs = info[0], nblk = info[1];
    if (b >= nblk) return;
    const uint32_t want = (uint64_t)b * ZB >= fcs ? 0u : min(ZB, fcs - b * ZB);
    const uint8_t* p = A.in_base + A.in_off[chunk];
    const uint32_t* bo = A.blk_off + (size_t)chunk * (A.blocks_per_chunk + 1);
    const ZdBlkMeta* meta = (const ZdBlkMeta*)A.par_meta + (size_t)chunk * A.blocks_per_chunk;
    uint8_t* win = wins + (size_t)warp * ZB;
    ZxShared<32>* sh = &shs[warp];
    const uint32_t made = zx_execute_blocks<32>(p, bo, meta, b, b + 1, win, ZB, nullptr, false, want,
                                                A.par_lits + (size_t)chunk * A.par_lit_cap, A.par_seqs + (size_t)chunk * A.par_seq_cap,
                                                A.in_len[chunk], sh, lane, true);
    __syncwarp();
    if (sh->err || made != want) { if (lane == 0) atomicOr(&info[3], 1u); return; }
    if (lane == 0) atomicAdd(&A.stats[4], 1ull);
    zx_flush<32>(A.out_base + A.out_off[chunk] + (size_t)b * ZB, win, made, lane);
}

// ------------------------------------------------------------------------------------------ host side
inline const char* zstd_dec_scratch_alloc(ZstdDecScratch& s, uint32_t chunk_cap, uint32_t max_batch) {
    s.blocks_per_chunk = ((chunk_cap + ZR - 1) / ZR) * ZR_SLICES;        // whole regions of 8 KiB blocks
    if (s.blocks_per_chunk == 0) s.blocks_per_chunk = ZR_SLICES;
    s.max_batch = max_batch; s.chunk_cap = chunk_cap;
    const char* e;
    if ((e = rt::malloc_device((void**)&s.blk_off, (size_t)max_batch * (s.blocks_per_chunk + 1) * 4 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.info, (size_t)max_batch * ZD_INFO * 4 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.lits_general, (size_t)max_batch * ZD_LIT_GENERAL + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.pos_tmp, (size_t)(max_batch + 1) * 8 + 256))) return e;
    // the independent-block stage uses fixed slots: block b's literals at b * ZB (<= ZB bytes), its sequences at b * ZB / 3
    const uint64_t zb_blocks = ((uint64_t)chunk_cap + ZB - 1) / ZB ? ((uint64_t)chunk_cap + ZB - 1) / ZB : 1;
    s.par_lit_cap = (uint32_t)((zb_blocks * ZB + 16ull * (s.blocks_per_chunk + 1) + 4096 + 15) & ~15ull);
    s.par_seq_cap = (uint32_t)std::max<uint64_t>(chunk_cap / 3 + 64, zb_blocks * (ZB / 3) + 64);
    if ((e = rt::malloc_device((void**)&s.par_meta, (size_t)max_batch * s.blocks_per_chunk * sizeof(ZdBlkMeta) + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.par_lits, (size_t)max_batch * s.par_lit_cap + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.par_seqs, (size_t)max_batch * s.par_seq_cap * 8 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.stats, 64))) return e;
    if ((e = rt::memset_async(s.stats, 0, 64, nullptr))) return e;
    if ((e = rt::device_sync())) return e;                   // the work streams do not order themselves behind the null stream
    return nullptr;
}
inline void zstd_dec_scratch_free(ZstdDecScratch& s) {
    rt::free_device(s.blk_off); rt::free_device(s.info); rt::free_device(s.lits_general);
    rt::free_device(s.pos_tmp); rt::free_device(s.par_meta); rt::free_device(s.par_lits); rt::free_device(s.par_seqs);
    rt::free_device(s.stats);
    s = ZstdDecScratch{};
}

constexpr uint32_t ZD_SMEM_BYTES = ZD_WPB * sizeof(ZdWarpCtx);

inline const char* zstd_kernels_configure() {
    const char* e;
    if ((e = rt::allow_smem(zstd_enc_regions_kernel, ZE_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_enc_blocks_kernel, ZB_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_frames_kernel, ZD_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_par_entropy_kernel, ZD_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_regions_kernel, ZX_REGION_SMEM))) return e;
    if ((e = rt::allow_smem(zstd_dec_blk_literals_kernel, ZDL_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_blk_sequences_kernel, ZDS_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_indep_execute_kernel, ZXB_SMEM_BYTES))) return e;
    if ((e = rt::allow_smem(zstd_dec_par_execute_kernel, ZX_FRAME_SMEM))) return e;
    return nullptr;
}

// out_off: when compute_offsets, written on the device as the exclusive scan of the frames' content sizes
// (chunks packed back to back); otherwise read as given.
inline int zstd_decompress_batch(ZstdDecScratch& s, rt::stream_t st, const uint8_t* in_base, const uint64_t* d_in_off,
                                 const uint32_t* d_in_len, uint32_t n_chunks, uint32_t chunk_cap, uint8_t* out_base,
                                 uint64_t* d_out_off, uint32_t* d_out_len, uint32_t* d_status, bool compute_offsets,
                                 LaunchProf& prof, uint32_t in_cap = 0xffffffffu) {
    if (n_chunks > s.max_batch) { g_zstd_err = "batch larger than the context"; return -1; }
    if (chunk_cap > s.chunk_cap) { g_zstd_err = "chunk larger than the context"; return -1; }
    ZstdDecArgs A;
    A.in_base = in_base; A.in_off = d_in_off; A.in_len = d_in_len;
    A.out_base = out_base; A.out_off = d_out_off; A.out_len = d_out_len; A.status = d_status;
    A.blk_off = s.blk_off; A.info = s.info; A.lits_general = s.lits_general;
    A.blocks_per_chunk = s.blocks_per_chunk; A.chunk_cap = chunk_cap; A.n_chunks = n_chunks; A.in_cap = in_cap;
    A.par_meta = s.par_meta; A.par_lits = s.par_lits; A.par_seqs = s.par_seqs;
    A.par_lit_cap = s.par_lit_cap; A.par_seq_cap = s.par_seq_cap; A.stats = s.stats;
    const char* e;
    TS_LAUNCH_P(prof, "zstd_dec_index", zstd_dec_index_kernel, dim3((n_chunks + 3) / 4), dim3(128), 0, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    if (compute_offsets) {
        TS_LAUNCH_P(prof, "chunk_index_scan", chunk_index_scan_kernel, dim3(1), dim3(32), 0, st, d_out_len, n_chunks, s.pos_tmp);
        if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
        if ((e = rt::d2d(d_out_off, s.pos_tmp, 8ull * n_chunks, st))) { g_zstd_err = e; return -7; }
    }
    const uint32_t rpc = (chunk_cap + ZR - 1) / ZR ? (chunk_cap + ZR - 1) / ZR : 1;
    const uint32_t bpc = rpc * ZR_SLICES;
    TS_LAUNCH_P(prof, "zstd_dec_blk_literals", zstd_dec_blk_literals_kernel, dim3((bpc + ZDI_G - 1) / ZDI_G, n_chunks), dim3(32), ZDL_SMEM_BYTES, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_blk_sequences", zstd_dec_blk_sequences_kernel, dim3((bpc + ZDI_G - 1) / ZDI_G, n_chunks), dim3(32), ZDS_SMEM_BYTES, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_entropy", zstd_dec_par_entropy_kernel, dim3((bpc + ZD_WPB - 1) / ZD_WPB, n_chunks), dim3(ZD_WPB * 32),
                ZD_SMEM_BYTES, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_blk_exec", zstd_dec_indep_execute_kernel, dim3((bpc + ZXB_WPB - 1) / ZXB_WPB, n_chunks), dim3(ZXB_WPB * 32), ZXB_SMEM_BYTES, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_regions", zstd_dec_regions_kernel, dim3(rpc, n_chunks), dim3(ZX_T), ZX_REGION_SMEM, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_frame_exec", zstd_dec_par_execute_kernel, dim3(n_chunks), dim3(ZX_TF), ZX_FRAME_SMEM, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_dec_serial", zstd_dec_frames_kernel, dim3((n_chunks + ZD_WPB - 1) / ZD_WPB), dim3(ZD_WPB * 32),
                ZD_SMEM_BYTES, st, A);
    if ((e = rt::last_error())) { g_zstd_err = e; return -7; }
    return 0;
}

}  // namespace ts
