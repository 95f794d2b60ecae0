// zstd_enc.cuh — batched Zstandard compression for sm_90a (kernel K1 of SURVEY.md §2a).
//
// Replaces ZstdCompressCtx.compress as called per chunk from
//   core/M/transform/CompressionChunkEnumeration.java:49-62 (new ctx, default level, setPledgedSrcSize,
//   setContentSize(true)): one independent RFC 8878 frame WITH Frame_Content_Size per chunk.
// Parity bar (SURVEY.md §8c): libzstd decodes every frame to the original bytes and
// ZSTD_getFrameContentSize(frame) == original size.  Compressed bytes are not expected to equal libzstd's.
//
// GPU-first decomposition: a chunk is cut into REGIONS of 64 KiB that never reference each other, one CTA (8 warps) per
// region; a region is 8 zstd blocks of 8 KiB, one warp each.  A 1 GiB segment is 16,384 independent regions / 131,072
// warps instead of 256 sequential frames.  Inside a region
//   * matches reach back across the whole region (one 64 KiB window in shared memory): every slice has its own running
//     hash table (nearest earlier occurrence inside the slice) plus a history table = last occurrence in all EARLIER
//     slices, built by a hashing pre-pass + an in-place cumulative merge, so that the 8 slices are parsed concurrently
//     and the result does not depend on warp timing (hash-slot winners are the highest position, deterministically);
//   * ONE Huffman tree and ONE set of FSE tables serve the region: the first block that needs them carries the
//     descriptions, the others are Treeless / Repeat_Mode blocks (the statistics of 64 KiB instead of 8 KiB, table
//     construction amortised 8x, ~100 bytes of descriptions saved per block);
//   * the region claims its place in the frame by a look-back over the previous regions' sizes and writes its blocks
//     straight into the frame — no assemble launch, no second pass over the compressed bytes.
// Everything is integer/byte work on the ALU and shared-memory pipes; there is no dense contraction to put on tensor cores.
#pragma once
#include "ts_common.cuh"
#include "rt.h"
#include "launch_prof.h"
#include "zstd_format.h"
#include "index_scan.cuh"
#include "xxh64.cuh"

namespace ts {

constexpr uint32_t ZB = 8192;                  // bytes of original data per zstd block (= per warp)
constexpr uint32_t ZR_SLICES = 8;              // blocks per region (= warps per CTA)
constexpr uint32_t ZR = ZB * ZR_SLICES;        // 64 KiB region
// the ZE_TUNE_* macros exist for parameter studies on the emulator (-DZE_TUNE_...=v); the defaults are the product
#ifndef ZE_TUNE_HLOG
#define ZE_TUNE_HLOG 10
#endif
#ifndef ZE_TUNE_HLOG_H
#define ZE_TUNE_HLOG_H 11
#endif
#ifndef ZE_TUNE_DET      // 0: plain hash-table stores (whichever lane wins) — A/B runs only: what determinism costs
#define ZE_TUNE_DET 1
#endif
#ifndef ZE_TUNE_HIST     // 0: no history tables (matches stay inside their 8 KiB slice) — A/B runs only: what the 64 KiB window costs
#define ZE_TUNE_HIST 1
#endif
constexpr int ZE_HLOG = ZE_TUNE_HLOG;          // per-slice running tables: 2^10 x u16 (region-relative position)
constexpr uint32_t ZE_HSIZE = 1u << ZE_HLOG;
constexpr int ZE_HLOG_H = ZE_TUNE_HLOG_H;      // history tables (last occurrence in all earlier slices): 7 of them
constexpr uint32_t ZE_HSIZE_H = 1u << ZE_HLOG_H;
constexpr uint32_t ZE_EMPTY = 0xffffu;         // no position: 65535 cannot start a 4-byte match in a 64 KiB region
constexpr uint32_t ZE_MAXSEQ = ZB / 8;         // sequences kept per block; beyond that the rest goes out as literals
constexpr uint32_t ZE_MIN_MATCH = 5;           // a 4-byte match costs more bits than four Huffman-coded literals (libzstd level 3 also uses 5); candidates are verified on 5 bytes
constexpr uint32_t ZE_THREADS = ZR_SLICES * 32;
static_assert(ZR <= 65536 && ZE_MAXSEQ <= 1024, "16-bit hash slots / sequence fields assume 64 KiB regions of 8 KiB blocks");

// ---- shared-memory map of one CTA ----
// parse phases:   [buf: region bytes + pad][ht_run: 8 x 2 KiB][ht_fin: 8 x 2 KiB][ctl]
// entropy phases: [8 x per-warp staging (ZE_STAGE bytes) over buf][shared tables over ht_run][tree / table scratch over ht_fin][ctl]
constexpr uint32_t ZE_STAGE = ZB + 448;                         // per-warp staging: literal streams, then the sequence bit stream + tile scratch
constexpr uint32_t ZE_BUF_BYTES = ZR_SLICES * ZE_STAGE + 64;    // region bytes (65536) + zero pad for over-reads
constexpr uint32_t ZE_HT_BYTES = ZR_SLICES * ZE_HSIZE * 2;
constexpr uint32_t ZE_HTH_BYTES = (ZR_SLICES - 1) * ZE_HSIZE_H * 2 < 12288 ? 12288 : (ZR_SLICES - 1) * ZE_HSIZE_H * 2;   // also the entropy phases' scratch
constexpr uint32_t ZE_OFF_RUN = ZE_BUF_BYTES;
constexpr uint32_t ZE_OFF_FIN = ZE_OFF_RUN + ZE_HT_BYTES;
constexpr uint32_t ZE_OFF_CTL = ZE_OFF_FIN + ZE_HTH_BYTES;
constexpr uint32_t ZE_SMEM_BYTES = ZE_OFF_CTL + 512;
// per-tile FSE scratch lives in the tail of a warp's staging area: the sequence bit stream staged there is at most
// ZE_MAXSEQ * 58 bits, which ends below this offset.  Per tile of 32 sequences and per kind (OF, ML, LL): the symbols'
// transforms (8 bytes each) going in, the state bits (value | count << 16) coming out of the chains.
constexpr uint32_t ZE_SEQ_AUX_OFF = 7456;
static_assert(ZE_MAXSEQ * 58 / 8 + 16 <= ZE_SEQ_AUX_OFF && ZE_SEQ_AUX_OFF % 8 == 0, "sequence bit stream would overlap the FSE tile scratch");
static_assert(ZE_SEQ_AUX_OFF + 3 * 32 * 8 + 3 * 32 * 4 <= ZE_STAGE, "FSE tile scratch must fit the staging area");

__constant__ zf::SeqTables g_seq_tables = zf::make_seq_tables();
__constant__ zf::PredefinedCTables g_pre_ctables = zf::make_predefined_ctables();

// Per-block scratch in HBM (L2-resident in practice: written and read back by the same CTA within microseconds).
constexpr uint32_t ZE_SLOT_A = ZB + 64;        // literal streams (or nothing for Raw / RLE literals)
constexpr uint32_t ZE_SLOT_B = ZB;             // sequence bit stream
struct ZstdEncScratch {
    uint2* seqs = nullptr;           // blocks * ZE_MAXSEQ
    uint8_t* lits = nullptr;         // blocks * ZB            literals in order
    uint8_t* slot_a = nullptr;       // blocks * ZE_SLOT_A
    uint8_t* slot_b = nullptr;       // blocks * ZE_SLOT_B
    unsigned long long* reg_state = nullptr;   // chunks * regions_per_chunk: look-back words (ready bit 63 | inclusive frame bytes)
    unsigned long long* ck_state = nullptr;    // chunks: Content_Checksum hand-over words (ze_hash_warp)
    uint32_t blocks_per_chunk = 0, regions_per_chunk = 0;
    uint32_t max_batch = 0;
};

struct ZstdEncArgs {
    const uint8_t* in_base; const uint64_t* in_off; const uint32_t* in_len;
    uint2* seqs; uint8_t* lits; uint8_t* slot_a; uint8_t* slot_b; unsigned long long* reg_state;
    uint32_t blocks_per_chunk, regions_per_chunk;
    uint8_t* out_base; const uint64_t* out_off; uint32_t* out_len;
    unsigned long long* ck_state;    // null: no Content_Checksum; else one hand-over word per chunk, zeroed before the launch
    uint32_t hash_rows, n_chunks;    // grid rows of hashing CTAs in front of the chunks' rows (0 without the checksum)
};

// ------------------------------------------------------------------------------------------ small helpers
__device__ __forceinline__ uint32_t ze_hash(uint32_t v) { return (v * 2654435761u) >> (32 - ZE_HLOG); }
__device__ __forceinline__ uint32_t ze_hash_h(uint32_t v) { return (v * 2654435761u) >> (32 - ZE_HLOG_H); }


// number of equal leading bytes (0..4) of two words given their XOR
__device__ __forceinline__ uint32_t ze_common_bytes(uint32_t x) { return (uint32_t)__clz((int)__brev(x)) >> 3; }

// OR a bit field (val, nb <= 58 bits) into a zeroed little-endian word buffer at bit offset `o` (shared memory)
__device__ __forceinline__ void ze_put_bits(uint32_t* words, uint32_t o, uint64_t val, uint32_t nb) {
    if (nb == 0) return;
    const uint32_t w = o >> 5, sh = o & 31;
    atomicOr(&words[w], (uint32_t)(val << sh));
    if (sh + nb > 32) atomicOr(&words[w + 1], (uint32_t)(val >> (32 - sh)));
    if (sh + nb > 64) atomicOr(&words[w + 2], (uint32_t)(val >> (64 - sh)));
}

// Hash-table insert where the HIGHEST position of the warp's step wins a shared slot — the hardware would keep an
// arbitrary one, which made frames differ between runs; retried uploads must produce identical objects.  Lanes re-store
// until no lower position is left in a slot: one round when the step has no slot collision, one more per extra peer.
// (match.any would find the peers in one instruction but serialises on the number of distinct values, which is slow on
// random data; 32-bit slots would allow atomicMax but halve the table at equal shared memory: -1.7 % ratio.)
#ifdef TSGPU_SIMT
static inline unsigned __match_any_sync(unsigned, unsigned v) {
    simt::Warp& w = simt::g_blk->warps[simt::g_cur->warp];
    w.buf[simt::g_cur->lane] = v;
    simt::warp_barrier();
    unsigned r = 0;
    for (int i = 0; i < 32; i++) if (w.buf[i] == v) r |= 1u << i;
    simt::warp_barrier();
    return r;
}
#endif

__device__ __forceinline__ void ze_insert_max(uint16_t* ht, uint32_t h, uint32_t p, bool valid) {
    if (valid) ht[h] = (uint16_t)p;
    while (ZE_TUNE_DET) {
        __syncwarp();
        const bool lost = valid && ht[h] < p;            // a lower position of this step sits in the slot
        if (!__any_sync(TS_FULL, lost)) break;
        if (lost) ht[h] = (uint16_t)p;
    }
    if (!ZE_TUNE_DET) __syncwarp();
}

}  // namespace ts

#include "zstd_fse_enc.cuh"
#include "zstd_huf_enc.cuh"

namespace ts {

// ------------------------------------------------------------------------------------------ region-wide state (shared memory)
struct ZeRegion {                    // lives in the ctl area
    uint32_t nseq[ZR_SLICES], nlit[ZR_SLICES];
    ZeLitBlock lit[ZR_SLICES];
    uint32_t seq_bytes[ZR_SLICES];   // bytes of the sequence bit stream of each block
    uint32_t frame_base;             // where this region's first block goes in the frame
    ZeKind kll, kof, kml;
    uint32_t desc_bytes;             // FSE table descriptions (without the modes byte)
};
static_assert(sizeof(ZeRegion) <= 512, "ctl area");

// Code tables of the sequence fields in shared memory (the constant-memory originals serialise on divergent indices).
struct ZeCodeTabs { uint8_t ll_code[64], ml_code[128], ll_bits[36], ml_bits[53], pad[3]; };
__device__ __forceinline__ uint32_t ze_ll_code_s(const ZeCodeTabs* t, uint32_t ll) { return ll < 64 ? t->ll_code[ll] : (uint32_t)zf::highbit32(ll) + 19; }
__device__ __forceinline__ uint32_t ze_ml_code_s(const ZeCodeTabs* t, uint32_t mlbase) { return mlbase < 128 ? t->ml_code[mlbase] : (uint32_t)zf::highbit32(mlbase) + 36; }

struct ZeShared {                    // over the ht_run area during the entropy phases
    uint32_t hist[256];              // literal histogram of the region
    uint32_t ctab[256];              // Huffman codes
    uint32_t cnt[ZE_NSYM_LL + ZE_NSYM_ML + ZE_NSYM_OF + 7];   // sequence code histograms, then normalised counts
    ZeCTab ct;
    ZeHuf huf;
    uint8_t desc[3][96];             // FSE table descriptions LL, OF, ML
    uint32_t desc_len[3];
    ZeCodeTabs tabs;
};
static_assert(sizeof(ZeShared) <= ZE_HT_BYTES, "shared tables must fit the running-hash-table area");
constexpr uint32_t ZE_KIND_SCRATCH = 1024;     // per FSE kind in the ht_fin area (ze_build_kind needs >= 784 bytes)
static_assert(8192 + 3 * ZE_KIND_SCRATCH <= ZE_HTH_BYTES, "tree scratch (7.5 KiB) + three table scratches must fit the history-table area");

// ------------------------------------------------------------------------------------------ sequences of one block
// Code histograms of one block's sequences, added to cnt (LL, ML, OF back to back; shared-memory atomics).
__device__ __forceinline__ void ze_seq_hist(const uint2* __restrict__ seqs, uint32_t N, uint32_t* cnt, const ZeCodeTabs* tabs, uint32_t lane) {
    uint2 pre = lane < N ? seqs[lane] : make_uint2(0, 0);
    for (uint32_t t0 = 0; t0 < N; t0 += 32) {
        const uint32_t j = t0 + lane;
        const uint2 s = pre;
        if (j + 32 < N) pre = seqs[j + 32];                  // next tile in flight while this one is counted
        if (j < N) {
            atomicAdd(&cnt[ze_ll_code_s(tabs, s.x & 0xffff)], 1u);
            atomicAdd(&cnt[ZE_NSYM_LL + ze_ml_code_s(tabs, s.x >> 16)], 1u);
            atomicAdd(&cnt[ZE_NSYM_LL + ZE_NSYM_ML + (uint32_t)zf::highbit32(s.y + 3)], 1u);
        }
    }
}

// ze_build_kind for one sequence code, k = 0 LL, 1 OF, 2 ML (the order of the descriptions in the stream), from the histograms
// in cnt (LL, ML, OF back to back) with the predefined tables as the Predefined_Mode choice.  CT: ZeCTab or a smaller table
// set with the same members.
template <class CT>
__device__ __forceinline__ uint32_t ze_build_seq_kind(uint32_t k, uint32_t* cnt, uint32_t N, CT* ct, uint8_t* scratch, uint8_t* desc,
                                                      ZeKind* kind, uint32_t lane) {
    const zf::PredefinedCTables& pre = g_pre_ctables;
    if (k == 0) return ze_build_kind(cnt, ZE_NSYM_LL, N, zf::LL_MAX_LOG, zf::LL_DEFAULT_LOG, pre.ll.state, pre.ll.sym,
                                     ct->st_ll, ct->sy_ll, scratch, desc, kind, true, lane);
    if (k == 1) return ze_build_kind(cnt + ZE_NSYM_LL + ZE_NSYM_ML, ZE_NSYM_OF, N, zf::OF_MAX_LOG, zf::OF_DEFAULT_LOG, pre.of.state,
                                     pre.of.sym, ct->st_of, ct->sy_of, scratch, desc, kind, true, lane);
    return ze_build_kind(cnt + ZE_NSYM_LL, ZE_NSYM_ML, N, zf::ML_MAX_LOG, zf::ML_DEFAULT_LOG, pre.ml.state, pre.ml.sym,
                         ct->st_ml, ct->sy_ml, scratch, desc, kind, true, lane);
}

// Number_of_Sequences field: its size, and the field itself (one lane; returns the size)
__device__ __forceinline__ uint32_t ze_nseq_size(uint32_t n) { return n < 128 ? 1u : n < 0x7f00 ? 2u : 3u; }
__device__ __forceinline__ uint32_t ze_write_nseq(uint8_t* p, uint32_t n) {
    if (n < 128) p[0] = (uint8_t)n;
    else if (n < 0x7f00) { p[0] = (uint8_t)((n >> 8) + 0x80); p[1] = (uint8_t)n; }
    else { p[0] = 0xff; p[1] = (uint8_t)(n - 0x7f00); p[2] = (uint8_t)((n - 0x7f00) >> 8); }
    return ze_nseq_size(n);
}

// Bit stream of one block's sequences, staged in the word buffer `bits` (shared, zeroed by the caller), with the per-tile
// scratch at ZE_SEQ_AUX_OFF.  Returns its size in bytes.  Warp-uniform, N >= 1.  Per tile of 32 sequences every lane looks
// up the transforms of its sequence's three codes; lanes 0-2 then walk the three state chains (the only serial part: one
// 8-byte load, the bit count, one store, one table load per symbol) and every lane packs its own field.  CT: as above.
template <class CT>
__device__ __forceinline__ uint32_t ze_encode_seq_bits(const uint2* __restrict__ seqs, uint32_t N, uint32_t* bits, const CT* ct,
                                                       const ZeCodeTabs* tabs, const ZeKind kll, const ZeKind kof, const ZeKind kml,
                                                       uint32_t lane) {
    uint2* pk = (uint2*)((uint8_t*)bits + ZE_SEQ_AUX_OFF);   // [3][32] transforms going in (OF, ML, LL)
    uint32_t* sb = (uint32_t*)(pk + 96);                     // [3][32] state bits coming out: value | count << 16
    uint32_t bitpos = 0;
    uint32_t state = 0;                              // lanes 0..2: OF, ML, LL chains
    const uint16_t* st_tab = lane == 0 ? ct->st_of : lane == 1 ? ct->st_ml : ct->st_ll;
    const bool rle = (lane == 0 ? kof.mode : lane == 1 ? kml.mode : kll.mode) == 1;
    const uint2* mypk = pk + (lane < 3 ? lane : 0) * 32;
    uint32_t* mysb = sb + (lane < 3 ? lane : 0) * 32;
    uint2 pre = lane < N ? seqs[N - 1 - lane] : make_uint2(0, 0);
    for (uint32_t t0 = 0; t0 < N; t0 += 32) {
        const uint32_t j = t0 + lane;                // stream order: j = 0 is the LAST sequence
        const bool have = j < N;
        uint32_t ll = 0, mlb = 0, offb = 0, llc = 0, mlc = 0, ofc = 0;
        const uint2 s = pre;
        if (j + 32 < N) pre = seqs[N - 1 - (j + 32)];
        if (have) {
            ll = s.x & 0xffff; mlb = s.x >> 16; offb = s.y + 3;       // mlb = matchLength - 3, offb = offset + 3 (no repcodes)
            llc = ze_ll_code_s(tabs, ll); mlc = ze_ml_code_s(tabs, mlb); ofc = (uint32_t)zf::highbit32(offb);
            const zf::FseCSym a = ct->sy_of[ofc], b = ct->sy_ml[mlc], c = ct->sy_ll[llc];
            pk[lane] = make_uint2((uint32_t)a.delta_nb_bits, (uint32_t)a.delta_find_state);
            pk[32 + lane] = make_uint2((uint32_t)b.delta_nb_bits, (uint32_t)b.delta_find_state);
            pk[64 + lane] = make_uint2((uint32_t)c.delta_nb_bits, (uint32_t)c.delta_find_state);
        }
        __syncwarp();
        if (lane < 3) {
            const uint32_t cnt = min(32u, N - t0);
            if (rle) {
                for (uint32_t i = 0; i < cnt; i++) mysb[i] = 0;
            } else {
                uint32_t i = 0;
                if (t0 == 0) {                       // FSE_initCState2 with the last sequence's symbol
                    const uint2 c = mypk[0];
                    const uint32_t nb = (uint32_t)((int32_t)c.x + (1 << 15)) >> 16;
                    const uint32_t v = (nb << 16) - c.x;
                    state = st_tab[(int32_t)(v >> nb) + (int32_t)c.y];
                    mysb[0] = 0;
                    i = 1;
                }
                _Pragma("unroll 4")
                for (; i < cnt; i++) {               // FSE_encodeSymbol
                    const uint2 c = mypk[i];
                    const uint32_t nb = (state + c.x) >> 16;
                    mysb[i] = (state & ((1u << nb) - 1)) | (nb << 16);
                    state = st_tab[(int32_t)(state >> nb) + (int32_t)c.y];
                }
            }
        }
        __syncwarp();
        uint64_t field = 0; uint32_t nb = 0;
        if (have) {
            const uint32_t llb = tabs->ll_bits[llc], mlbits = tabs->ml_bits[mlc];
            // order inside a field (first written = lowest bits): OF state, ML state, LL state, LL extra, ML extra, OF extra
            const uint32_t b0 = sb[lane], b1 = sb[32 + lane], b2 = sb[64 + lane];
            field = b0 & 0xffff; nb = b0 >> 16;
            field |= (uint64_t)(b1 & 0xffff) << nb; nb += b1 >> 16;
            field |= (uint64_t)(b2 & 0xffff) << nb; nb += b2 >> 16;
            field |= (uint64_t)(ll & ((1u << llb) - 1)) << nb; nb += llb;
            field |= (uint64_t)(mlb & ((1u << mlbits) - 1)) << nb; nb += mlbits;
            field |= (uint64_t)(offb & ((1u << ofc) - 1)) << nb; nb += ofc;
        }
        const uint32_t inc = warp_inclusive_scan_u32(nb, lane);
        ze_put_bits(bits, bitpos + inc - nb, field, nb);
        bitpos += __shfl_sync(TS_FULL, inc, 31);
        __syncwarp();
    }
    // FSE_flushCState x3 (ML, OF, LL) then the closing 1 bit
    const uint32_t st_of = __shfl_sync(TS_FULL, state, 0), st_ml = __shfl_sync(TS_FULL, state, 1),
                   st_ll = __shfl_sync(TS_FULL, state, 2);
    if (lane == 0) {
        uint64_t f = st_ml & ((1u << kml.log) - 1);
        uint32_t nb = kml.log;
        f |= (uint64_t)(st_of & ((1u << kof.log) - 1)) << nb; nb += kof.log;
        f |= (uint64_t)(st_ll & ((1u << kll.log) - 1)) << nb; nb += kll.log;
        f |= 1ull << nb; nb += 1;
        ze_put_bits(bits, bitpos, f, nb);
    }
    bitpos += kml.log + kof.log + kll.log + 1;
    __syncwarp();
    return (bitpos + 7) >> 3;
}

// warp copy of n bytes, any alignment on either side: aligned 32-bit stores in the middle, source words by funnel shift
__device__ TS_NOINLINE void ze_warp_copy(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint32_t n, uint32_t lane) {
    const uint32_t head = min(n, (uint32_t)((4 - ((uintptr_t)dst & 3)) & 3));
    if (lane < head) dst[lane] = src[lane];
    const uint32_t words = (n - head) >> 2;
    uint32_t* d32 = (uint32_t*)(dst + head);
    const uint8_t* s = src + head;
    for (uint32_t i = lane; i < words; i += 32) d32[i] = ld_u32_unaligned(s + 4 * i);
    const uint32_t done = head + 4 * words;
    if (lane < n - done) dst[done + lane] = src[done + lane];
}

// ------------------------------------------------------------------------------------------ frame header
// checksum: Content_Checksum_flag (Frame_Header_Descriptor bit 2); the frame then ends with 4 more bytes (ze_hash_warp)
__device__ __forceinline__ uint32_t ze_frame_header(uint8_t* h, uint32_t n, bool checksum) {     // see tshost::zstdFrameHeader
    uint32_t p = 0;
    const uint8_t ck = checksum ? 0x04 : 0x00;
    h[p++] = 0x28; h[p++] = 0xB5; h[p++] = 0x2F; h[p++] = 0xFD;
    if (n <= (1u << 21)) {
        if (n < 256) { h[p++] = 0x20 | ck; h[p++] = (uint8_t)n; }
        else if (n < 65536 + 256) { h[p++] = 0x60 | ck; h[p++] = (uint8_t)(n - 256); h[p++] = (uint8_t)((n - 256) >> 8); }
        else { h[p++] = 0xA0 | ck; h[p++] = (uint8_t)n; h[p++] = (uint8_t)(n >> 8); h[p++] = (uint8_t)(n >> 16); h[p++] = (uint8_t)(n >> 24); }
    } else {
        h[p++] = 0x80 | ck; h[p++] = 0x58;
        h[p++] = (uint8_t)n; h[p++] = (uint8_t)(n >> 8); h[p++] = (uint8_t)(n >> 16); h[p++] = (uint8_t)(n >> 24);
    }
    return p;
}
__device__ __forceinline__ uint32_t ze_frame_header_size(uint32_t n) {
    return n <= (1u << 21) ? (n < 256 ? 6u : n < 65536 + 256 ? 7u : 9u) : 10u;
}
// The frame of an empty chunk: header, one empty last Raw block [, the checksum of no bytes].  Returns its size.
__device__ __forceinline__ uint32_t ze_empty_frame(uint8_t* frame, bool checksum) {
    uint32_t p = ze_frame_header(frame, 0, checksum);
    frame[p++] = 1; frame[p++] = 0; frame[p++] = 0;
    if (checksum) { for (int k = 0; k < 4; k++) frame[p++] = (uint8_t)(XXH64_EMPTY_LOW32 >> (8 * k)); }
    return p;
}

// ------------------------------------------------------------------------------------------ Content_Checksum
// With TSGPU_FLAG_ZSTD_CHECKSUM the compressor's grid gains `hash_rows` rows of CTAs IN FRONT of the chunks' rows: they have the
// lowest block indices, so they are dispatched first and hash while the other CTAs compress.  Warp k of those CTAs, counted
// across the rows, hashes chunk k (xxh64.cuh: the chunk's four XXH64 chains take ~n/32 dependent rounds, milliseconds for a
// 4 MiB chunk, which the compression of the other chunks hides).  The 4 bytes go right after the chunk's last block and are
// written by whichever finishes second -- the hash warp, or the unit (region / block) that placed the last block -- decided by
// one word per chunk: both add 1 << 32 to it, the hash warp adds its hash too.  Neither ever waits for the other.
__device__ __forceinline__ void ze_put_u32le(uint8_t* p, uint32_t v) {
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}
__device__ TS_NOINLINE void ze_hash_warp(const uint8_t* in_base, const uint64_t* in_off, const uint32_t* in_len, uint8_t* out_base,
                                         const uint64_t* out_off, const uint32_t* out_len, unsigned long long* ck_state,
                                         uint32_t n_chunks, uint32_t chunk, uint64_t* stage, uint32_t lane) {
    if (chunk >= n_chunks) return;
    const uint32_t clen = in_len[chunk];
    if (clen == 0) return;                                   // ze_empty_frame carries the checksum of no bytes
    const uint32_t h = xxh64_warp_low32(in_base + in_off[chunk], clen, stage, lane);
    if (lane == 0) {
        const unsigned long long old = atomicAdd(&ck_state[chunk], (1ull << 32) | h);
        if (old >> 32) {                                     // the last block is placed, and out_len (its end + 4) published
            __threadfence();
            const uint32_t end = *(const volatile uint32_t*)&out_len[chunk];
            ze_put_u32le(out_base + out_off[chunk] + end - 4, h);
        }
    }
}
// The unit that placed the chunk's last block, which ends at `at`, after publishing out_len (one lane).
__device__ __forceinline__ void ze_ck_unit_done(unsigned long long* ck, uint8_t* at) {
    __threadfence();                                         // out_len before the hand-over word
    const unsigned long long old = atomicAdd(ck, 1ull << 32);
    if (old >> 32) ze_put_u32le(at, (uint32_t)old);          // the hash warp was first: its hash is in the word
}

// ------------------------------------------------------------------------------------------ look-back words
// Where a unit (a region, or a block in the speed mode) goes in its frame = frame header + the sizes of all units before it.
// Decoupled look-back (Merrill & Garland's single-pass scan): a unit publishes its own SIZE as soon as it is known, then
// walks back over its predecessors' words, 32 at a time, adding sizes until it meets one that already carries an inclusive
// PREFIX; then it publishes its own prefix.  Nothing waits for a chain of prefixes to propagate unit by unit — a first
// version did (each unit waited for its predecessor's prefix) and the 512-hop chain per chunk nearly doubled the kernel's time.
// Word: bits 62-63 = 0 empty / 1 size / 2 inclusive prefix, bits 0-61 the value.  Called by a whole warp.
constexpr unsigned long long ZE_LB_SIZE = 1ull << 62, ZE_LB_PREFIX = 2ull << 62, ZE_LB_VALUE = (1ull << 62) - 1;
__device__ __forceinline__ unsigned long long ze_lb_load(const unsigned long long* w) {
#ifdef TSGPU_SIMT
    return *(const volatile unsigned long long*)w;
#else
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(w) : "memory");
    return v;
#endif
}
__device__ __forceinline__ void ze_lb_store(unsigned long long* w, unsigned long long v) {
#ifdef TSGPU_SIMT
    *(volatile unsigned long long*)w = v;
#else
    asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(w), "l"(v) : "memory");
#endif
}
// st: the chunk's words; idx: this unit; size: its bytes; head: what precedes unit 0 (the frame header).  Returns the
// unit's offset in the frame (warp-uniform).  `last` units do not publish (nobody looks back at them).
#ifndef ZE_TUNE_LB_BACKOFF   // 1: exponential back-off (100 ns .. 1.6 us) while a predecessor has not published its size yet
#define ZE_TUNE_LB_BACKOFF 0
#endif
__device__ __forceinline__ uint32_t ze_lookback(unsigned long long* st, uint32_t idx, uint32_t size, uint32_t head, bool last, uint32_t lane) {
    if (lane == 0 && !last) ze_lb_store(&st[idx], ZE_LB_SIZE | size);
    uint64_t excl = 0;
    int32_t hi = (int32_t)idx - 1;                           // the window is units hi, hi-1, ..., hi-31 (lane 0 = nearest)
#if ZE_TUNE_LB_BACKOFF
    uint32_t pause = 100;                                    // doubles per failed probe: a waiting warp should not eat issue slots
#endif
    while (true) {
        const int32_t i = hi - (int32_t)lane;
        unsigned long long v = i >= 0 ? ze_lb_load(&st[i]) : (i == -1 ? (ZE_LB_PREFIX | head) : 0ull);
        const uint32_t flag = (uint32_t)(v >> 62);
        const uint32_t pref = __ballot_sync(TS_FULL, flag == 2);
        const uint32_t empty = __ballot_sync(TS_FULL, flag == 0);
        const uint32_t first = pref ? (uint32_t)__ffs((int)pref) - 1 : 32u;
        const uint32_t need = first >= 31 ? 0xffffffffu : (1u << (first + 1)) - 1;     // everything up to (and including) the first prefix
        if (empty & need) {                                  // a predecessor has not finished encoding yet
#ifdef TSGPU_SIMT
            simt::yield();
#elif ZE_TUNE_LB_BACKOFF
            __nanosleep(pause);
            pause = min(pause * 2, 1600u);
#else
            __nanosleep(200);
#endif
            continue;
        }
        uint64_t part = ((need >> lane) & 1) ? (uint64_t)(v & ZE_LB_VALUE) : 0ull;
        for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(TS_FULL, part, o);
        excl += part;
        if (first < 32) break;
        hi -= 32;
    }
    if (lane == 0 && !last) ze_lb_store(&st[idx], ZE_LB_PREFIX | (excl + size));
    return (uint32_t)excl;
}

// ------------------------------------------------------------------------------------------ the region kernel
__global__ void __launch_bounds__(ZE_THREADS, 2) zstd_enc_regions_kernel(const __grid_constant__ ZstdEncArgs A) {
    TS_DYN_SMEM(smem);
    const uint32_t tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    if (blockIdx.y < A.hash_rows) {                      // a hashing CTA: one chunk per warp (Content_Checksum)
        ze_hash_warp(A.in_base, A.in_off, A.in_len, A.out_base, A.out_off, A.out_len, A.ck_state, A.n_chunks,
                     (blockIdx.y * gridDim.x + blockIdx.x) * ZR_SLICES + w, (uint64_t*)(smem + w * XXH_STAGE_BYTES), lane);
        return;
    }
    const uint32_t chunk = blockIdx.y - A.hash_rows, region = blockIdx.x;
    const uint32_t clen = A.in_len[chunk];
    uint8_t* frame = A.out_base + A.out_off[chunk];
    const bool checksum = A.ck_state != nullptr;
    if (clen == 0) {                                     // empty chunk: header + empty last raw block
        if (region == 0 && tid == 0) A.out_len[chunk] = ze_empty_frame(frame, checksum);
        return;
    }
    if ((uint64_t)region * ZR >= clen) return;           // whole CTA
    const uint32_t rn = min(ZR, clen - region * ZR);     // bytes of this region
    const uint32_t nreg = (clen + ZR - 1) / ZR;
    const uint32_t nslice = (rn + ZB - 1) / ZB;
    const uint8_t* src = A.in_base + A.in_off[chunk] + (size_t)region * ZR;
    const size_t gblk = (size_t)chunk * A.blocks_per_chunk + (size_t)region * ZR_SLICES + w;
    uint2* seqs = A.seqs + gblk * ZE_MAXSEQ;
    uint8_t* lits = A.lits + gblk * ZB;

    uint8_t* buf = smem;
    uint16_t* ht_run = (uint16_t*)(smem + ZE_OFF_RUN) + w * ZE_HSIZE;
    uint16_t* ht_fin_all = (uint16_t*)(smem + ZE_OFF_FIN);
    ZeRegion* R = (ZeRegion*)(smem + ZE_OFF_CTL);

    // ---- phase 0: stage the region (128-bit loads when the source is aligned), zero the pad, reset the tables
    if ((((uintptr_t)src) & 15) == 0) {
        for (uint32_t i = tid * 16; i < rn; i += ZE_THREADS * 16) {
            if (i + 16 <= rn) *(uint4*)(buf + i) = ldg128_stream((const uint4*)(src + i));
            else for (uint32_t k = i; k < rn; k++) buf[k] = src[k];
        }
    } else {
        for (uint32_t i = tid; i < rn; i += ZE_THREADS) buf[i] = src[i];
    }
    for (uint32_t i = rn + tid; i < ZE_BUF_BYTES; i += ZE_THREADS) buf[i] = 0;
    for (uint32_t i = tid; i < (ZE_HT_BYTES + ZE_HTH_BYTES) / 4; i += ZE_THREADS) ((uint32_t*)(smem + ZE_OFF_RUN))[i] = 0xffffffffu;
    __syncthreads();

    const uint32_t s0 = w * ZB;                          // this warp's slice [s0, s1) of the region
    const uint32_t s1 = min(s0 + ZB, rn);
    const bool have_slice = s0 < rn;

    // ---- phase 1: history tables.  Pre-pass: last occurrence of every hash inside each slice ...
    if (ZE_TUNE_HIST && have_slice && nslice > 1 && w + 1 < nslice) {    // the last slice's table would serve nobody
        uint16_t* fin = ht_fin_all + w * ZE_HSIZE_H;
        for (uint32_t cur = s0; cur < s1; cur += 32) {
            const uint32_t p = cur + lane;
            const bool valid = p < s1 && p + 4 <= rn;            // as a SOURCE a position may run over the slice end
            const uint32_t v = ld_u32_unaligned(buf + p);
            ze_insert_max(fin, ze_hash_h(v), p, valid);
        }
    }
    __syncthreads();
    // ... then an in-place cumulative merge: table j becomes "last occurrence in slices 0..j"; slice j+1 consults table j
    for (uint32_t j = 1; j + 1 < nslice; j++) {
        uint32_t* cur32 = (uint32_t*)(ht_fin_all + j * ZE_HSIZE_H);
        const uint32_t* prev32 = (const uint32_t*)(ht_fin_all + (j - 1) * ZE_HSIZE_H);
        for (uint32_t i = tid; i < ZE_HSIZE_H / 2; i += ZE_THREADS) {
            const uint32_t c = cur32[i], p = prev32[i];
            const uint32_t lo = (c & 0xffffu) != ZE_EMPTY ? (c & 0xffffu) : (p & 0xffffu);
            const uint32_t hi = (c >> 16) != ZE_EMPTY ? (c >> 16) : (p >> 16);
            cur32[i] = lo | (hi << 16);
        }
        __syncthreads();
    }
    const uint16_t* ht_hist = (ZE_TUNE_HIST && w > 0) ? ht_fin_all + (w - 1) * ZE_HSIZE_H : nullptr;

    // ---- phase 2: greedy LZ parse of the slice, 32 positions per step
    // Straight-line work per lane (no loops, no divergence worth the name): hash, look up, verify the candidate on 4 bytes,
    // measure the next 4 forwards and the 4 before it backwards.  The verified candidates are then walked left to right —
    // the only serial part: a match that ran through all 8 measured bytes is extended by the whole warp (128 bytes per
    // probe), every taken match grows backwards over the literals before it (libzstd's "catch up", up to 4 bytes).
    // Sequences are written by their own lanes afterwards; the step's literals leave in the same step.
    uint32_t nseq = 0, nlit = 0;
    if (have_slice) {
        uint32_t anchor = s0, cur = s0;
        while (cur + 4 <= s1 && nseq + 8 <= ZE_MAXSEQ) {                // a step adds at most 8 sequences (min match 4)
            const uint32_t p = cur + lane;
            const bool valid = p + ZE_MIN_MATCH <= s1;
            // 12 bytes around the position as aligned words: [p-4, p+8)
            const uint32_t* wp = (const uint32_t*)(buf + (p & ~3u));
            const uint32_t shp = (p & 3) * 8;
            const uint32_t am = p >= 4 ? wp[-1] : 0u, a0 = wp[0], a1 = wp[1], a2 = wp[2];
            const uint32_t v = __funnelshift_r(a0, a1, shp);
            const uint32_t h = ze_hash(v);
            const uint32_t slot = valid ? ht_run[h] : ZE_EMPTY;
            __syncwarp();
            ze_insert_max(ht_run, h, p, valid);                        // the highest position of the step wins a shared slot
            uint32_t cand = slot != ZE_EMPTY ? slot : 0u;
            const uint32_t* wc = (const uint32_t*)(buf + (cand & ~3u));
            uint32_t shc = (cand & 3) * 8;
            uint32_t cm = cand >= 4 ? wc[-1] : 0u, c0 = wc[0], c1 = wc[1], c2 = wc[2];
            bool ok = slot != ZE_EMPTY && __funnelshift_r(c0, c1, shc) == v;
            if (ht_hist) {                                            // nothing (or a collision) in this slice: the earlier slices
                const uint32_t hs = (valid && !ok) ? ht_hist[ze_hash_h(v)] : ZE_EMPTY;
                if (hs != ZE_EMPTY) {
                    const uint32_t* wh = (const uint32_t*)(buf + (hs & ~3u));
                    const uint32_t shh = (hs & 3) * 8;
                    const uint32_t h0 = wh[0], h1 = wh[1];
                    if (__funnelshift_r(h0, h1, shh) == v) { ok = true; cand = hs; shc = shh; cm = hs >= 4 ? wh[-1] : 0u; c0 = h0; c1 = h1; c2 = wh[2]; }
                }
            }
            // forwards: bytes 4..7; backwards: how many of the 4 bytes before the position match (never past the candidate's start)
            uint32_t len = 4 + ze_common_bytes(__funnelshift_r(a1, a2, shp) ^ __funnelshift_r(c1, c2, shc));
            len = min(len, s1 - p);
            ok = ok && valid && len >= ZE_MIN_MATCH;
            const uint32_t xb = __funnelshift_r(am, a0, shp) ^ __funnelshift_r(cm, c0, shc);
            const uint32_t bkr = min((uint32_t)__clz((int)xb) >> 3, min(cand, 4u));
            const uint32_t packed = len | (bkr << 8);
            const uint32_t mask = __ballot_sync(TS_FULL, ok);
            // walk the candidates
            uint32_t taken = 0, cov = 0;
            uint32_t my_ll = 0, my_ml = 0;                             // sequence of this lane, if it is taken
            uint32_t prev_end = anchor;
            uint32_t f = mask ? (uint32_t)__ffs((int)mask) - 1 : 32u;
            while (f < 32) {
                const uint32_t pf = cur + f;
                const uint32_t info = __shfl_sync(TS_FULL, packed, f);
                uint32_t L = info & 0xffu;
                if (L == 8 && pf + 8 < s1) {                           // ran through the measured bytes: lane l compares the 4 bytes at +8 + 4l
                    const uint32_t cf = __shfl_sync(TS_FULL, cand, f);
                    while (true) {
                        const uint32_t q = pf + L + 4 * lane;
                        uint32_t c = 0;
                        if (q < s1) {
                            c = ze_common_bytes(ld_u32_unaligned(buf + q) ^ ld_u32_unaligned(buf + (q - pf + cf)));
                            c = min(c, s1 - q);
                        }
                        const uint32_t stop = __ballot_sync(TS_FULL, c < 4);
                        if (stop) {
                            const uint32_t fl = (uint32_t)__ffs((int)stop) - 1;
                            L += 4 * fl + __shfl_sync(TS_FULL, c, fl);
                            break;
                        }
                        L += 128;
                    }
                }
                const uint32_t bk = min(info >> 8, pf - max(prev_end, cur));     // backwards only over this step's literals
                const uint32_t start = f - bk, tl = L + bk;            // in lanes of this step
                if (lane == f) { my_ll = pf - bk - prev_end; my_ml = tl; }
                taken |= 1u << f;
                cov |= (tl >= 32 - start ? 0xffffffffu : (1u << tl) - 1) << start;
                prev_end = pf + L;
                const uint32_t end = f + L;
                const uint32_t rest = end < 32 ? mask & (0xffffffffu << end) : 0u;
                f = rest ? (uint32_t)__ffs((int)rest) - 1 : 32u;
            }
            if (taken) {
                if ((taken >> lane) & 1)
                    seqs[nseq + (uint32_t)__popc(taken & ((1u << lane) - 1))] = make_uint2(my_ll | ((my_ml - 3) << 16), p - cand);
                nseq += (uint32_t)__popc(taken);
                anchor = prev_end;
            }
            // literals of the step, in order: one byte per uncovered position below the end of the slice
            {
                const uint32_t inside = s1 - cur >= 32 ? 0xffffffffu : (1u << (s1 - cur)) - 1;
                const uint32_t lm = ~cov & inside;
                if ((lm >> lane) & 1) lits[nlit + (uint32_t)__popc(lm & ((1u << lane) - 1))] = (uint8_t)v;
                nlit += (uint32_t)__popc(lm);
            }
            cur = max(cur + 32, anchor);
        }
        // the rest of the slice (after the last step, or after the sequence budget ran out) is literals
        if (cur < s1) {
            const uint32_t ll = s1 - cur;
            for (uint32_t k = lane; k < ll; k += 32) lits[nlit + k] = buf[cur + k];
            nlit += ll;
        }
        __syncwarp();
        __threadfence_block();
    }
    if (lane == 0) { R->nseq[w] = nseq; R->nlit[w] = nlit; }
    __syncthreads();                                                   // ---- the region's bytes and hash tables are dead from here on

    // ---- phase 3: region statistics
    ZeShared* S = (ZeShared*)(smem + ZE_OFF_RUN);
    for (uint32_t i = tid; i < sizeof(ZeShared) / 4; i += ZE_THREADS) ((uint32_t*)S)[i] = 0;
    __syncthreads();
    if (tid < 64) S->tabs.ll_code[tid] = g_seq_tables.ll_code[tid];
    if (tid < 128) S->tabs.ml_code[tid] = g_seq_tables.ml_code[tid];
    if (tid < 36) S->tabs.ll_bits[tid] = g_seq_tables.ll_bits[tid];
    if (tid >= 64 && tid < 64 + 53) S->tabs.ml_bits[tid - 64] = g_seq_tables.ml_bits[tid - 64];
    __syncthreads();
    if (have_slice) {
        _Pragma("unroll 2")
        for (uint32_t i = lane; i < nlit; i += 32) atomicAdd(&S->hist[lits[i]], 1u);
        ze_seq_hist(seqs, nseq, S->cnt, &S->tabs, lane);
    }
    __syncthreads();
    uint32_t nseq_total = 0, nlit_total = 0;
    for (uint32_t k = 0; k < ZR_SLICES; k++) { nseq_total += R->nseq[k]; nlit_total += R->nlit[k]; }

    // ---- phase 4: one Huffman tree (warp 0) and the three FSE tables (warps 1-3), concurrently
    {
        uint8_t* fin_area = smem + ZE_OFF_FIN;
        if (w == 0) {
            ze_huf_build(S->hist, S->ctab, (uint32_t*)fin_area, nlit_total, &S->huf, lane);
        } else if (w <= 3 && nseq_total) {
            ZeKind k;
            const uint32_t dn = ze_build_seq_kind(w - 1, S->cnt, nseq_total, &S->ct, fin_area + 8192 + (w - 1) * ZE_KIND_SCRATCH,
                                                  S->desc[w - 1], &k, lane);
            if (lane == 0) {
                S->desc_len[w - 1] = dn;
                if (w == 1) R->kll = k; else if (w == 2) R->kof = k; else R->kml = k;
            }
        }
    }
    __syncthreads();

    // ---- phase 5: every warp encodes its block's literal streams and sequence bits (sizes first, nothing placed yet)
    uint8_t* stage = smem + w * ZE_STAGE;
    uint8_t* slot_a = A.slot_a + gblk * ZE_SLOT_A;
    uint8_t* slot_b = A.slot_b + gblk * ZE_SLOT_B;
    if (have_slice) {
        ze_huf_plan_block(lits, nlit, S->ctab, &S->huf, &R->lit[w], lane);
        const ZeLitBlock lb = R->lit[w];
        if (lb.kind == 2) {
            ze_huf_encode_block(lits, nlit, S->ctab, lb.stream_bytes, (uint32_t*)stage, lane);
            ze_warp_copy(slot_a, stage, lb.stream_bytes, lane);
        }
        __syncwarp();
        uint32_t sbytes = 0;
        if (nseq) {
            for (uint32_t i = lane; i < ZE_STAGE / 4; i += 32) ((uint32_t*)stage)[i] = 0;
            __syncwarp();
            sbytes = ze_encode_seq_bits(seqs, nseq, (uint32_t*)stage, &S->ct, &S->tabs, R->kll, R->kof, R->kml, lane);
            ze_warp_copy(slot_b, stage, sbytes, lane);
        }
        if (lane == 0) R->seq_bytes[w] = sbytes;
    }
    __syncthreads();

    // ---- phase 6: who carries the descriptions, what each block weighs, where the region goes
    // (every thread computes the same small table from shared memory: 8 entries)
    uint32_t my_off = 0, my_size = 0, my_lit_type = 0, total = 0;
    bool my_raw = false, my_seq_owner = false;
    const uint32_t desc_total = nseq_total ? ((R->kll.mode == 0 ? 0 : S->desc_len[0]) + (R->kof.mode == 0 ? 0 : S->desc_len[1]) +
                                              (R->kml.mode == 0 ? 0 : S->desc_len[2])) : 0;
    {
        bool tree_given = false, desc_given = false;
        for (uint32_t k = 0; k < nslice; k++) {
            const uint32_t bn = min(ZB, rn - k * ZB);
            const ZeLitBlock lb = R->lit[k];
            const uint32_t nsq = R->nseq[k];
            const bool tree_here = lb.kind == 2 && !tree_given;
            const bool desc_here = nsq != 0 && !desc_given;
            uint32_t lit_sz;
            if (lb.kind == 0) lit_sz = 3 + lb.n;
            else if (lb.kind == 1) lit_sz = 3 + 1;
            else {
                const uint32_t comp = (tree_here ? S->huf.tree_bytes : 0) + 6 + lb.stream_bytes;
                lit_sz = ze_lit_header_huf_size(lb.n, comp) + comp;
            }
            const uint32_t shdr = ze_nseq_size(nsq) + (nsq ? 1u : 0u);            // Number_of_Sequences (+ modes byte)
            const uint32_t payload = lit_sz + shdr + (desc_here ? desc_total : 0) + R->seq_bytes[k];
            const bool raw = payload >= bn;                                  // would not shrink (with its duties): Raw_Block, state untouched
            const uint32_t bsize = 3 + (raw ? bn : payload);
            if (!raw) { tree_given |= lb.kind == 2; desc_given |= nsq != 0; }
            if (k == w) { my_off = total; my_size = bsize; my_raw = raw; my_lit_type = lb.kind == 2 ? (tree_here ? 2u : 3u) : lb.kind; my_seq_owner = desc_here; }
            total += bsize;
        }
    }
    if (w == 0) {
        unsigned long long* rs = A.reg_state + (size_t)chunk * A.regions_per_chunk;
        const uint32_t hl = ze_frame_header_size(clen);
        if (region == 0 && lane == 0) ze_frame_header(frame, clen, checksum);
        const uint32_t base = ze_lookback(rs, region, total, hl, region + 1 == nreg, lane);
        if (lane == 0) {
            R->frame_base = base;
            if (region + 1 == nreg) {
                A.out_len[chunk] = base + total + (checksum ? 4u : 0u);
                if (checksum) ze_ck_unit_done(A.ck_state + chunk, frame + base + total);
            }
        }
    }
    __syncthreads();

    // ---- phase 7: every warp writes its block into the frame
    if (have_slice) {
        const uint32_t bn = s1 - s0;
        uint8_t* out = frame + R->frame_base + my_off;
        const bool last_block = region + 1 == nreg && w + 1 == nslice;
        if (lane == 0) {
            const uint32_t hdr = (last_block ? 1u : 0u) | ((my_raw ? 0u : 2u) << 1) | ((my_size - 3) << 3);
            out[0] = (uint8_t)hdr; out[1] = (uint8_t)(hdr >> 8); out[2] = (uint8_t)(hdr >> 16);
        }
        if (my_raw) {
            ze_warp_copy(out + 3, src + s0, bn, lane);
        } else {
            const ZeLitBlock lb = R->lit[w];
            uint8_t* body = out + 3;
            uint32_t at = 0;
            if (lb.kind == 0) {
                if (lane == 0) ze_lit_header_raw(body, 0, lb.n);
                ze_warp_copy(body + 3, lits, lb.n, lane);
                at = 3 + lb.n;
            } else if (lb.kind == 1) {
                if (lane == 0) { ze_lit_header_raw(body, 1, lb.n); body[3] = (uint8_t)lb.rle_byte; }
                at = 4;
            } else {
                const uint32_t tb = my_lit_type == 2 ? S->huf.tree_bytes : 0;
                const uint32_t comp = tb + 6 + lb.stream_bytes;
                const uint32_t hsz = ze_lit_header_huf_size(lb.n, comp);
                if (lane == 0) {
                    ze_lit_header_huf(body, my_lit_type, lb.n, comp);
                    ze_lit_jump_table(body + hsz + tb, lb.ssz[0] | (lb.ssz[1] << 16) | ((uint64_t)lb.ssz[2] << 32));
                }
                for (uint32_t i = lane; i < tb; i += 32) body[hsz + i] = S->huf.desc[i];
                ze_warp_copy(body + hsz + tb + 6, slot_a, lb.stream_bytes, lane);
                at = hsz + comp;
            }
            uint8_t* sp = body + at;
            const uint32_t shdr = ze_nseq_size(nseq);
            if (lane == 0) ze_write_nseq(sp, nseq);                    // 0: the sequences section ends here
            if (nseq) {
                uint32_t dn = 0;
                if (lane == 0) {
                    // owner: the real modes + descriptions; the others repeat them (Predefined_Mode costs nothing to restate)
                    const uint32_t mll = R->kll.mode, mof = R->kof.mode, mml = R->kml.mode;
                    const uint32_t rll = mll == 0 ? 0u : 3u, rof = mof == 0 ? 0u : 3u, rml = mml == 0 ? 0u : 3u;
                    sp[shdr] = my_seq_owner ? (uint8_t)((mll << 6) | (mof << 4) | (mml << 2)) : (uint8_t)((rll << 6) | (rof << 4) | (rml << 2));
                }
                if (my_seq_owner) {
                    uint8_t* d = sp + shdr + 1;
                    const uint32_t order[3] = {0, 1, 2};               // stream order LL, OF, ML = desc[0], desc[1], desc[2]
                    for (uint32_t q = 0; q < 3; q++) {
                        const uint32_t kmode = q == 0 ? R->kll.mode : q == 1 ? R->kof.mode : R->kml.mode;
                        if (kmode == 0) continue;
                        const uint32_t len = S->desc_len[order[q]];
                        for (uint32_t i = lane; i < len; i += 32) d[dn + i] = S->desc[order[q]][i];
                        dn += len;
                    }
                }
                ze_warp_copy(sp + shdr + 1 + dn, slot_b, R->seq_bytes[w], lane);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ host side
static thread_local const char* g_zstd_err = "";
inline const char* zstd_last_error() { return g_zstd_err; }

inline const char* zstd_enc_scratch_alloc(ZstdEncScratch& s, uint32_t chunk_cap, uint32_t max_batch) {
    s.regions_per_chunk = (chunk_cap + ZR - 1) / ZR;
    if (s.regions_per_chunk == 0) s.regions_per_chunk = 1;
    s.blocks_per_chunk = s.regions_per_chunk * ZR_SLICES;
    s.max_batch = max_batch;
    const size_t nblk = (size_t)s.blocks_per_chunk * max_batch;
    const char* e;
    if ((e = rt::malloc_device((void**)&s.seqs, nblk * ZE_MAXSEQ * sizeof(uint2) + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.lits, nblk * ZB + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.slot_a, nblk * ZE_SLOT_A + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.slot_b, nblk * ZE_SLOT_B + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.reg_state, (size_t)s.regions_per_chunk * max_batch * 8 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.ck_state, (size_t)max_batch * 8 + 256))) return e;
    return nullptr;
}
inline void zstd_enc_scratch_free(ZstdEncScratch& s) {
    rt::free_device(s.seqs); rt::free_device(s.lits); rt::free_device(s.slot_a); rt::free_device(s.slot_b); rt::free_device(s.reg_state);
    rt::free_device(s.ck_state);
    s = ZstdEncScratch{};
}

// checksum: end every frame with its Content_Checksum, hashed by extra CTAs of the same launch (ze_hash_warp)
inline int zstd_compress_batch(ZstdEncScratch& s, rt::stream_t st, const uint8_t* in_base, const uint64_t* d_in_off,
                               const uint32_t* d_in_len, uint32_t n_chunks, uint32_t chunk_size, bool checksum,
                               uint8_t* out_base, const uint64_t* d_out_off, uint32_t* d_out_len, LaunchProf& prof) {
    if (n_chunks > s.max_batch) { g_zstd_err = "batch larger than the context"; return -1; }
    uint32_t rpc = (chunk_size + ZR - 1) / ZR;
    if (rpc > s.regions_per_chunk) { g_zstd_err = "chunk larger than the context"; return -1; }
    if (rpc == 0) rpc = 1;                                   // empty chunks still get their frame
    ZstdEncArgs A;
    A.in_base = in_base; A.in_off = d_in_off; A.in_len = d_in_len;
    A.seqs = s.seqs; A.lits = s.lits; A.slot_a = s.slot_a; A.slot_b = s.slot_b; A.reg_state = s.reg_state;
    A.blocks_per_chunk = s.blocks_per_chunk; A.regions_per_chunk = s.regions_per_chunk;
    A.out_base = out_base; A.out_off = d_out_off; A.out_len = d_out_len;
    A.ck_state = checksum ? s.ck_state : nullptr;
    A.n_chunks = n_chunks;
    A.hash_rows = checksum ? ((n_chunks + ZR_SLICES - 1) / ZR_SLICES + rpc - 1) / rpc : 0;    // one warp per chunk
    const char* e = rt::memset_async(s.reg_state, 0, (size_t)s.regions_per_chunk * n_chunks * 8, st);
    if (!e && checksum) e = rt::memset_async(s.ck_state, 0, (size_t)n_chunks * 8, st);
    if (e) { g_zstd_err = e; return -7; }
    static_assert(ZE_SMEM_BYTES >= ZR_SLICES * XXH_STAGE_BYTES, "hashing warps stage in the region buffer");
    TS_LAUNCH_P(prof, "zstd_enc_regions", zstd_enc_regions_kernel, dim3(rpc, n_chunks + A.hash_rows), dim3(ZE_THREADS), ZE_SMEM_BYTES, st, A);
    e = rt::last_error();
    if (e) { g_zstd_err = e; return -7; }
    return 0;
}

}  // namespace ts
