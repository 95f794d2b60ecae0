// zstd_enc_blk.cuh — the SPEED mode of the compressor: one warp per independent 8 KiB zstd block.
//
// Same contract as zstd_enc.cuh (one RFC 8878 frame with Frame_Content_Size per chunk, CompressionChunkEnumeration.java:49-62),
// different trade: every 8 KiB block is self-contained (own Huffman tree, own FSE tables, no match leaves the block), so a
// 1 GiB segment is 131,072 independent warps with no barrier between them, 20 warps per SM.  That is the round-1 kernel with
// the streamlined FSE chains and the backwards growth of taken matches ("catch up"); it compresses the K corpus ~3.1 : 1 at
// ~14.9 ms per GiB on an H100, where the region kernel of zstd_enc.cuh reaches ~3.5 : 1 at about twice the time (one 64 KiB
// window and one set of tables per 8 blocks).  TSGPU_FLAG_ZSTD picks this kernel, TSGPU_FLAG_ZSTD | TSGPU_FLAG_ZSTD_DENSE the region kernel;
// the decoder reads both through the same region path (zstd_dec.cuh).
//   zstd_enc_blocks_kernel    one WARP per block: block staged in shared memory; 32 positions hashed and verified per step
//                             against a per-warp hash table, greedy left-to-right selection by ballot/ffs, match extension
//                             per lane then warp-wide; literals (Raw / RLE / Huffman) + sequences (per-block FSE tables)
//                             placement: look-back over the previous blocks' sizes, the block copies itself into the frame
// Hash-slot winners inside a step are whichever lane the hardware keeps (every outcome is a valid parse: candidates are
// verified before use), so frames of this mode may differ between runs in bytes, never in what they decode to; the region
// kernel is deterministic.
#pragma once
#include "zstd_enc.cuh"

namespace ts {

constexpr int ZB_HLOG = 10;                    // per-warp hash table: 2^10 x u16 (position + 1)
constexpr uint32_t ZB_HSIZE = 1u << ZB_HLOG;
// ZB_TUNE_* exist for A/B runs on the GPU (scripts/ab_variants.sh builds one library per setting); the defaults are the product
#ifndef ZB_TUNE_WPB       // H100: 8 warps per CTA 19.0 ms per GiB, 4 warps 16.6, 2 warps 16.5 (within noise of 4)
#define ZB_TUNE_WPB 4
#endif
#ifndef ZB_TUNE_LANE_EXT
#define ZB_TUNE_LANE_EXT 12
#endif
#ifndef ZB_TUNE_BACK      // 1: taken matches grow backwards over up to 4 literals ("catch up"): +3.6 % ratio for ~0.5 ms per GiB (H100)
#define ZB_TUNE_BACK 1
#endif
#ifndef ZB_TUNE_STRAIGHT  // 1: per-lane match extension as straight-line code over 12 bytes instead of a divergent loop:
#define ZB_TUNE_STRAIGHT 1 //   18.1 -> 16.6 ms per GiB on an H100
#endif
#ifndef ZB_TUNE_EXTLDS    // 1: the warp-wide extension of long matches reads shared memory with LDS word pairs instead of generic loads
#define ZB_TUNE_EXTLDS 0  //    (H100: within 1 % of the generic loads, 16.5 vs 16.6 ms per GiB — off)
#endif
#ifndef ZB_TUNE_PHASES    // 1: every warp stamps clock64() at its block's phase boundaries into g_zb_phases, read back through
#define ZB_TUNE_PHASES 0  //    tsgpu_zb_phases (scripts/enc_phases.py); measurement builds only, never the product
#endif
#ifndef ZB_TUNE_PAD       // N > 0: N extra FFMAs per parse step in 4 independent chains, off the step's dependent chain: if the
#define ZB_TUNE_PAD 0     //    kernel time grows with N as issue slots predict, the parse is issue-bound (measurement builds only)
#endif
constexpr int ZB_WPB = ZB_TUNE_WPB;            // warps (= blocks in flight) per CTA
constexpr uint32_t ZB_LANE_EXT = ZB_TUNE_LANE_EXT;   // bytes a lane extends its own match beyond the first 4
constexpr uint32_t ZB_BUF_PAD = 416;           // zero pad for over-reads; its tail also holds the FSE tile scratch
constexpr uint32_t ZB_SLOT = ZB + 512;         // per-block output slot: 3-byte header + payload
constexpr uint32_t ZB_SMEM_WARP = ZB + ZB_BUF_PAD + ZB_HSIZE * 2;   // buf, ht
constexpr uint32_t ZB_SMEM_WARP_AL = (ZB_SMEM_WARP + 15) & ~15u;
// the sequence bit stream is staged in `buf`, its per-tile FSE scratch at ZE_SEQ_AUX_OFF in the tail
static_assert(ZE_SEQ_AUX_OFF + 3 * 32 * 8 + 3 * 32 * 4 <= ZB + ZB_BUF_PAD, "FSE tile scratch must fit the block buffer");
struct ZbCTab {                                // per-warp FSE encoding tables (logs <= 7 for <= 1024 sequences); aliases the hash-table area
    uint16_t st_ll[128], st_ml[128], st_of[128];
    zf::FseCSym sy_ll[ZE_NSYM_LL], sy_ml[ZE_NSYM_ML], sy_of[ZE_NSYM_OF];
};
static_assert(sizeof(ZbCTab) + sizeof(ZeCodeTabs) <= ZB_HSIZE * 2 && 2048 <= ZB_HSIZE * 2,
              "FSE tables + sequence code tables, and the 2 KiB Huffman scratch, alias the hash-table area");

#if ZB_TUNE_PHASES
// t[0] start, then the end of: 1 staging, 2 parse, 3 Huffman code table, 4 literals section, 5 FSE tables, 6 sequence
// bit stream, 7 look-back, 8 copy into the frame.  A phase the block skips (raw literals, no sequences) keeps t = 0.
struct ZbPhases { unsigned long long t[9]; uint32_t nseq, nlit, nsym, pad; };
constexpr uint32_t ZB_PHASES_MAX = 1u << 17;   // blocks of one launch recorded (chunk * blocks_per_chunk + block): 1 GiB
__device__ ZbPhases g_zb_phases[ZB_PHASES_MAX];
#define ZB_PH_PARAM , ZbPhases* ph
#define ZB_PH_ARG , ph
#define ZB_MARK(k) do { if (lane == 0 && ph) ph->t[k] = clock64(); } while (0)
#define ZB_NOTE(f, v) do { if (lane == 0 && ph) ph->f = (v); } while (0)
#else
#define ZB_PH_PARAM
#define ZB_PH_ARG
#define ZB_MARK(k) do {} while (0)
#define ZB_NOTE(f, v) do {} while (0)
#endif

__device__ __forceinline__ uint32_t zb_hash(uint32_t v) { return (v * 2654435761u) >> (32 - ZB_HLOG); }
// the pointer unchanged, but opaque to the compiler, which would otherwise rebuild it from its parts at every use
template <class T> __device__ __forceinline__ T* zb_opaque(T* p) {
#if TS_DEVICE_ASM
    asm("mov.b64 %0, %0;" : "+l"(p));
#endif
    return p;
}
// 0xffffffff << n, 0 for every n >= 32: one SHF on the GPU (PTX clamps shift counts), spelt out for the emulator
__device__ __forceinline__ uint32_t zb_ones_from(uint32_t n) {
#if TS_DEVICE_ASM
    uint32_t r;
    asm("shl.b32 %0, %1, %2;" : "=r"(r) : "r"(0xffffffffu), "r"(n));
    return r;
#else
    return n >= 32 ? 0u : 0xffffffffu << n;
#endif
}

struct ZstdBlkScratch {
    uint8_t* blk_out = nullptr;      // blocks * ZB_SLOT
    uint32_t* blk_size = nullptr;    // blocks
    uint2* seqs = nullptr;           // blocks * ZE_MAXSEQ
    uint8_t* lits = nullptr;         // blocks * ZB
    unsigned long long* blk_state = nullptr;   // blocks: look-back words (ready bit 63 | inclusive frame bytes)
    unsigned long long* ck_state = nullptr;    // chunks: Content_Checksum hand-over words (ze_hash_warp)
    uint32_t blocks_per_chunk = 0, max_batch = 0;
};
struct ZstdBlkArgs {
    const uint8_t* in_base; const uint64_t* in_off; const uint32_t* in_len;
    uint8_t* blk_out; uint32_t* blk_size; uint2* seqs; uint8_t* lits; unsigned long long* blk_state;
    uint32_t blocks_per_chunk;
    uint8_t* out_base; const uint64_t* out_off; uint32_t* out_len;
    unsigned long long* ck_state;    // as in ZstdEncArgs: null without the Content_Checksum
    uint32_t hash_rows, n_chunks;
};

// Raw_Literals_Block with the 3-byte header (Size_Format 11: 20-bit Regenerated_Size).
__device__ TS_NOINLINE uint32_t zb_raw_literals(const uint8_t* __restrict__ lits, uint32_t n, uint8_t* body, uint32_t lane) {
    if (lane == 0) ze_lit_header_raw(body, 0, n);
    for (uint32_t i = lane; i < n; i += 32) body[3 + i] = lits[i];
    return 3 + n;
}


// Returns the bytes written at `body`.  `work`: >= ZB + 160 bytes of shared memory (tree scratch, then the
// stream staging area); `aux16`: 2 KiB of shared memory (histogram + code table).
__device__ __forceinline__ uint32_t zb_encode_literals(const uint8_t* __restrict__ lits, uint32_t n, uint8_t* body,
                                                       uint32_t* work, uint16_t* aux16, uint32_t lane ZB_PH_PARAM) {
    if (n < ZE_HUF_MIN) return zb_raw_literals(lits, n, body, lane);
    uint32_t* hist = (uint32_t*)aux16;         // [256]
    uint32_t* ctab = hist + 256;               // [256] code | len << 16

    for (uint32_t i = lane; i < 256; i += 32) { hist[i] = 0; ctab[i] = 0; }
    __syncwarp();
    {   // 16 literals per load: the block's literal slot is 16-byte aligned and ZB bytes long
        const uint4* l16 = (const uint4*)lits;
        _Pragma("unroll 2")
        for (uint32_t i = lane; i * 16 < n; i += 32) {
            const uint4 q = l16[i];
            const uint32_t w4[4] = {q.x, q.y, q.z, q.w};
            _Pragma("unroll")
            for (uint32_t k = 0; k < 16; k++)
                if (i * 16 + k < n) atomicAdd(&hist[(w4[k >> 2] >> (8 * (k & 3))) & 0xff], 1u);
        }
    }
    __syncwarp();

    bool pays;
    const uint32_t m = ze_huf_symbols(hist, n, work, &pays, lane);
    ZB_NOTE(nsym, m);
    if (m == 1) {                                                         // RLE literals
        if (lane == 0) { ze_lit_header_raw(body, 1, n); body[3] = (uint8_t)work[1280]; }
        return 4;
    }
    if (!pays) return zb_raw_literals(lits, n, body, lane);
    const uint32_t last_sym = work[1280 + m - 1] & 0xff;
    uint32_t total_bits;
    const uint32_t max_len = ze_huf_codes(hist, m, last_sym, 16, ctab, work, &total_bits, lane);
    if (max_len > (uint32_t)zf::HUF_MAX_LOG) return zb_raw_literals(lits, n, body, lane);
    ZB_MARK(3);
    uint8_t* desc = (uint8_t*)hist;                                       // the histogram is dead
    const uint32_t tree_bytes = ze_huf_tree_desc(ctab, last_sym, max_len, desc, work, lane);   // symbols 0 .. last_sym-1 are listed
    if (tree_bytes == ZE_NO_TREE) return zb_raw_literals(lits, n, body, lane);
    const uint32_t est = tree_bytes + 6 + (total_bits >> 3) + 8;
    if (est + 5 >= n) return zb_raw_literals(lits, n, body, lane);        // Huffman would not pay

    // ---- the four streams, staged in `work` (cleared first; tree scratch is dead from here on)
    const uint32_t seg = (n + 3) / 4;
    __syncwarp();
    for (uint32_t i = lane; i < (ZB + 128) / 4; i += 32) work[i] = 0;
    __syncwarp();
    // this lane's run [ra, rb) of each stream (32 runs per stream, symbols written last-to-first: the offset of a run is the
    // number of bits of all LATER runs); the loads of the four runs go out together, once to size them and once to encode
    uint32_t ra[4], rb[4], rbits[4];
    _Pragma("unroll")
    for (uint32_t st = 0; st < 4; st++) {
        const uint32_t s0 = st * seg, s1 = st < 3 ? min(n, s0 + seg) : n;
        const uint32_t cnt = s1 > s0 ? s1 - s0 : 0;
        const uint32_t per = (cnt + 31) / 32;
        ra[st] = s0 + min(cnt, lane * per); rb[st] = s0 + min(cnt, lane * per + per); rbits[st] = 0;
    }
    const uint32_t per0 = (seg + 31) / 32;                                // the longest run (stream 0 is full)
    _Pragma("unroll 2")
    for (uint32_t k = 0; k < per0; k++) {
        _Pragma("unroll")
        for (uint32_t st = 0; st < 4; st++) if (ra[st] + k < rb[st]) rbits[st] += ctab[lits[ra[st] + k]] >> 16;
    }
    uint32_t off[4];
    uint32_t byte_pos = 0;
    uint64_t ssz_all = 0;                                                 // four 16-bit stream sizes
    _Pragma("unroll")
    for (uint32_t st = 0; st < 4; st++) {
        const uint32_t incb = warp_inclusive_scan_u32(rbits[st], lane);
        const uint32_t total = __shfl_sync(TS_FULL, incb, 31);
        off[st] = byte_pos * 8 + (total - incb);
        if (lane == 0) {                                                  // end mark
            const uint32_t o = byte_pos * 8 + total;
            atomicOr(&work[o >> 5], 1u << (o & 31));
        }
        const uint32_t sz = (total + 1 + 7) >> 3;
        ssz_all |= (uint64_t)sz << (16 * st);
        byte_pos += sz;
    }
    _Pragma("unroll 2")
    for (uint32_t k = 0; k < per0; k++) {
        _Pragma("unroll")
        for (uint32_t st = 0; st < 4; st++) {
            if (ra[st] + k < rb[st]) {
                const uint32_t c = ctab[lits[rb[st] - 1 - k]];
                const uint32_t len = c >> 16, code = c & 0xffff;
                const uint32_t w = off[st] >> 5, sh = off[st] & 31;
                atomicOr(&work[w], code << sh);
                if (sh + len > 32) atomicOr(&work[w + 1], code >> (32 - sh));
                off[st] += len;
            }
        }
    }
    __syncwarp();
    const uint32_t comp = tree_bytes + 6 + byte_pos;
    const uint32_t hsz = ze_lit_header_huf_size(n, comp);
    if (hsz + comp >= 3 + n) return zb_raw_literals(lits, n, body, lane);
    if (lane == 0) {
        ze_lit_header_huf(body, 2, n, comp);
        ze_lit_jump_table(body + hsz + tree_bytes, ssz_all);
    }
    for (uint32_t i = lane; i < tree_bytes; i += 32) body[hsz + i] = desc[i];
    uint8_t* sp = body + hsz + tree_bytes + 6;
    const uint8_t* wb = (const uint8_t*)work;
    _Pragma("unroll 2")
    for (uint32_t i = lane; i < byte_pos; i += 32) sp[i] = wb[i];
    __syncwarp();
    return hsz + comp;
}


// Encodes the sequences section (everything after the Number_of_Sequences field): the modes byte and table
// descriptions go straight to `hdr_out` (global), the bit stream is staged in the word buffer `bits` (shared).
// Returns the bit-stream bytes; *desc_bytes = 1 (modes byte) + table descriptions.  Warp-uniform, N >= 1.
__device__ __forceinline__ uint32_t zb_encode_sequences(const uint2* __restrict__ seqs, uint32_t N, uint32_t* bits, ZbCTab* ct,
                                                        const ZeCodeTabs* tabs, uint8_t* hdr_out, uint32_t* desc_bytes,
                                                        uint32_t lane ZB_PH_PARAM) {
    // code histograms (then normalised counts), in the word buffer beyond ze_build_kind's own scratch
    uint32_t* cnt = bits + 256;
    for (uint32_t i = lane; i < ZE_NSYM_LL + ZE_NSYM_ML + ZE_NSYM_OF; i += 32) cnt[i] = 0;
    __syncwarp();
    ze_seq_hist(seqs, N, cnt, tabs, lane);
    __syncwarp();
    // tables (descriptions in stream order LL, OF, ML); `bits` doubles as scratch until it is cleared
    ZeKind kll, kof, kml;
    uint8_t* desc = hdr_out + 1;
    uint32_t dn = ze_build_seq_kind(0, cnt, N, ct, (uint8_t*)bits, desc, &kll, lane);
    dn += ze_build_seq_kind(1, cnt, N, ct, (uint8_t*)bits, desc + dn, &kof, lane);
    dn += ze_build_seq_kind(2, cnt, N, ct, (uint8_t*)bits, desc + dn, &kml, lane);
    if (lane == 0) hdr_out[0] = (uint8_t)((kll.mode << 6) | (kof.mode << 4) | (kml.mode << 2));
    *desc_bytes = 1 + dn;
    __syncwarp();
    for (uint32_t i = lane; i < (ZB + ZB_BUF_PAD) / 4; i += 32) bits[i] = 0;
    __syncwarp();
    ZB_MARK(5);
    return ze_encode_seq_bits(seqs, N, bits, ct, tabs, kll, kof, kml, lane);
}

__global__ void __launch_bounds__(ZB_WPB * 32, 5) zstd_enc_blocks_kernel(const __grid_constant__ ZstdBlkArgs A) {
    // which block this warp owns, its scratch slots and its shared-memory window
    TS_DYN_SMEM(smem);
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (blockIdx.y < A.hash_rows) {                               // a hashing CTA: one chunk per warp (Content_Checksum)
        ze_hash_warp(A.in_base, A.in_off, A.in_len, A.out_base, A.out_off, A.out_len, A.ck_state, A.n_chunks,
                     (blockIdx.y * gridDim.x + blockIdx.x) * ZB_WPB + warp, (uint64_t*)(smem + warp * XXH_STAGE_BYTES), lane);
        return;
    }

    const uint32_t chunk = blockIdx.y - A.hash_rows;
    const uint32_t blk = blockIdx.x * ZB_WPB + warp;
    const uint32_t clen = A.in_len[chunk];
    if (clen == 0 && blk == 0) {                                  // empty chunk: header + empty last raw block
        if (lane == 0) A.out_len[chunk] = ze_empty_frame(A.out_base + A.out_off[chunk], A.ck_state != nullptr);
        return;
    }
    if ((uint64_t)blk * ZB >= clen) return;                       // whole warp
    const uint32_t bn = min(ZB, clen - blk * ZB);
    const bool last_block = (uint64_t)(blk + 1) * ZB >= clen;
    const uint8_t* src = A.in_base + A.in_off[chunk] + (size_t)blk * ZB;
    const size_t gblk = (size_t)chunk * A.blocks_per_chunk + blk;
    uint8_t* out = A.blk_out + gblk * ZB_SLOT;
    // per-block bases kept in registers: the parse step indexes them with 32-bit counts instead of redoing gblk's math
    uint2* const seqs = zb_opaque(A.seqs + gblk * ZE_MAXSEQ);
    uint8_t* const lits = zb_opaque(A.lits + gblk * ZB);

    uint8_t* wbase = smem + warp * ZB_SMEM_WARP_AL;
    uint8_t* buf = wbase;
    uint16_t* ht = (uint16_t*)(wbase + ZB + ZB_BUF_PAD);
#if ZB_TUNE_PHASES
    ZbPhases* ph = gblk < ZB_PHASES_MAX ? &g_zb_phases[gblk] : nullptr;
    if (lane == 0 && ph) { *ph = ZbPhases{}; ph->t[0] = clock64(); }
#endif
    // ---- stage the block in shared memory (128-bit loads when the source is aligned), zero the pad, reset the table
    if ((((uintptr_t)src) & 15) == 0) {
        for (uint32_t i = lane * 16; i < bn; i += 512) {
            if (i + 16 <= bn) *(uint4*)(buf + i) = ldg128_stream((const uint4*)(src + i));
            else for (uint32_t k = i; k < bn; k++) buf[k] = src[k];
        }
    } else {
        _Pragma("unroll 2")
        for (uint32_t i = lane; i < bn; i += 32) buf[i] = src[i];
    }
    _Pragma("unroll 1")
    for (uint32_t i = bn + lane; i < ZB + ZB_BUF_PAD; i += 32) buf[i] = 0;
    for (uint32_t i = lane; i < ZB_HSIZE / 2; i += 32) ((uint32_t*)ht)[i] = 0;
    __syncwarp();
    ZB_MARK(1);

    // ---- phase A: greedy LZ parse, 32 positions per step
    // Selection (which of the 32 candidate matches survive, left to right) is the only serial part and costs a
    // handful of instructions per taken match; sequences are then written by their own lanes in parallel and
    // the step's literals (the positions no taken match covers) leave in the same step.  The step is bound by instruction
    // issue (ZB_TUNE_PAD, DESIGN.md §8), so it is written for few instructions; the `step:` markers split the loop body
    // into the parts whose static instructions scripts/parse_step_sass.py counts.
#if ZB_TUNE_PAD
    float pad[4] = {(float)lane, 1.f, 2.f, 3.f};
#endif
    const uint32_t lanes_below = (1u << lane) - 1;
    uint32_t anchor = 0, cur = 0, nseq = 0, nlit = 0;
    while (cur + 4 <= bn && nseq + 8 <= ZE_MAXSEQ) {                // a step adds at most 8 sequences (min match 4)
        // step: probe
        const uint32_t p = cur + lane;
        const bool valid = p + 4 <= bn;
        // unaligned 4-byte reads as a rolling pair of aligned words per stream: one new LDS per stream and step
        const uint32_t* wp = (const uint32_t*)(buf + (p & ~3u));
        const uint32_t shp = (p & 3) * 8;
        uint32_t a0 = wp[0], a1 = wp[1];
        const uint32_t v = __funnelshift_r(a0, a1, shp);
        const uint32_t h = zb_hash(v);
        const uint32_t slot = valid ? ht[h] : 0u;                  // position + 1, 0 = empty
        __syncwarp();
        // Lanes of this step that share a slot all store; the CUDA model lets any one of them win.  Every outcome is a
        // valid parse (candidates are verified before use), so frames may differ in bytes, never in what they decode to.
        if (valid) ht[h] = (uint16_t)(p + 1);
        __syncwarp();
        const uint32_t cand = slot ? slot - 1 : 0u;
        const uint32_t* wc = (const uint32_t*)(buf + (cand & ~3u));
        const uint32_t shc = (cand & 3) * 8;
        uint32_t c0 = wc[0], c1 = wc[1];
        const bool ok = slot != 0 && __funnelshift_r(c0, c1, shc) == v;
#if ZB_TUNE_BACK
        // how many of the 4 bytes before the position also match (straight-line, all lanes: two loads, two funnel shifts):
        // a taken match grows backwards over the literals before it, libzstd's "catch up".  (A first version did this in a
        // branch of the lanes with a verified candidate, through ld_u32_unaligned, and was slower.)
        const uint32_t am = p >= 4 ? wp[-1] : 0u, cm = cand >= 4 ? wc[-1] : 0u;
        const uint32_t bkr = min((uint32_t)__clz((int)(__funnelshift_r(am, a0, shp) ^ __funnelshift_r(cm, c0, shc))) >> 3, min(cand, 4u));
#else
        const uint32_t bkr = 0;
#endif
        uint32_t len = 0;
#if ZB_TUNE_STRAIGHT
        {   // the 12 bytes after the verified 4, straight-line on all lanes (three more words per stream): no divergent loop
            static_assert(ZB_TUNE_LANE_EXT == 12, "the straight-line extension measures exactly 12 bytes");
            const uint32_t a2 = wp[2], a3 = wp[3], a4 = wp[4], c2 = wc[2], c3 = wc[3], c4 = wc[4];
            const uint32_t x1 = __funnelshift_r(a1, a2, shp) ^ __funnelshift_r(c1, c2, shc);
            const uint32_t x2 = __funnelshift_r(a2, a3, shp) ^ __funnelshift_r(c2, c3, shc);
            const uint32_t x3 = __funnelshift_r(a3, a4, shp) ^ __funnelshift_r(c3, c4, shc);
            // the equal bytes end in the first word that differs (all 12 are equal when none does): one count, not three
            const uint32_t e = (x1 ? 0u : x2 ? 4u : 8u) + ze_common_bytes(x1 ? x1 : x2 ? x2 : x3);
            len = ok ? min(4 + e, min(bn - p, 4 + ZB_LANE_EXT)) : 0u;
        }
#else
        if (ok) {
            len = 4;
            const uint32_t lim = min(bn - p, 4 + ZB_LANE_EXT);
            for (uint32_t k = 2; len < lim; k++) {
                a0 = a1; a1 = wp[k]; c0 = c1; c1 = wc[k];
                const uint32_t c = ze_common_bytes(__funnelshift_r(a0, a1, shp) ^ __funnelshift_r(c0, c1, shc));
                len += c;
                if (c < 4) break;
            }
            len = min(len, lim);
        }
#endif
#if ZB_TUNE_PAD
        {
            const float pv = __uint_as_float((v & 0x007fffffu) | 0x3f000000u);   // in [0.5, 1)
            _Pragma("unroll")
            for (int k = 0; k < ZB_TUNE_PAD; k++) asm volatile("fma.rn.f32 %0, %0, %1, %2;" : "+f"(pad[k & 3]) : "f"(pv), "f"(0.25f));
        }
#endif
        // step: select
        const uint32_t mask = __ballot_sync(TS_FULL, ok && len >= ZE_MIN_MATCH);
        // Greedy selection, left to right.  Every lane precomputes where its match would end and which candidate would
        // come next, so one shuffle per taken match walks the chain (the only serial part of the parse).
        const uint32_t e = lane + len;
        const uint32_t nxt = (uint32_t)__clz((int)__brev(mask & zb_ones_from(e)));       // 32: none
        const bool capped = ok && len == 4 + ZB_LANE_EXT && p + len < bn;
        const uint32_t packed = e | (capped ? 1u << 8 : 0u) | (nxt << 16);
        // The walk also hands every taken lane where the match before it ends (`my_prev`, relative to `cur`; the step's
        // first match gets `anchor`, at or before `cur`), so the sequences need no shuffle after the walk.
        uint32_t taken = 0, prev = anchor - cur, my_prev = 0;
        uint32_t f = (uint32_t)__clz((int)__brev(mask));
        // step: walk
        while (f < 32) {
            const uint32_t info = __shfl_sync(TS_FULL, packed, f);
            uint32_t end = info & 0xffu, nf = info >> 16;
            if (info & (1u << 8)) {                                // warp-wide extension of a long match
                // step: long
                uint32_t L = 4 + ZB_LANE_EXT;
                const uint32_t off = __shfl_sync(TS_FULL, p - cand, f);
                const uint32_t mpos = cur + f;
                while (true) {
                    const uint32_t q = mpos + L + 4 * lane;
                    uint32_t c = 0;
                    if (q < bn) {
#if ZB_TUNE_EXTLDS      // shared-memory word pairs + funnel shifts (ld_u32_unaligned goes through a generic pointer: LD.E, not LDS)
                        const uint32_t r = q - off;
                        const uint32_t* wq = (const uint32_t*)(buf + (q & ~3u));
                        const uint32_t* wr = (const uint32_t*)(buf + (r & ~3u));
                        c = ze_common_bytes(__funnelshift_r(wq[0], wq[1], (q & 3) * 8) ^ __funnelshift_r(wr[0], wr[1], (r & 3) * 8));
#else
                        c = ze_common_bytes(ld_u32_unaligned(buf + q) ^ ld_u32_unaligned(buf + q - off));
#endif
                        c = min(c, bn - q);
                    }
                    const uint32_t stop = __ballot_sync(TS_FULL, c < 4);
                    if (stop) {
                        const uint32_t fl = (uint32_t)__ffs((int)stop) - 1;
                        L += 4 * fl + __shfl_sync(TS_FULL, c, fl);
                        break;
                    }
                    L += 128;
                }
                if (lane == f) len = L;
                end = f + L;
                nf = (uint32_t)__clz((int)__brev(mask & zb_ones_from(end)));
                // step: walk
            }
            taken |= 1u << f;
            if (lane == f) my_prev = prev;
            prev = end;
            f = nf;
        }
        // step: tail
        uint32_t cov = 0;                                          // positions of this step covered by a taken match
        if (taken) {
            const bool mine = (taken >> lane) & 1;
            const uint32_t pe = cur + my_prev;                     // where the match before this lane's ends
            const uint32_t bk = mine ? min(bkr, p - max(pe, cur)) : 0u;   // "catch up" over this step's literals, never into the previous match
            if (mine)
                seqs[nseq + (uint32_t)__popc(taken & lanes_below)] = make_uint2((p - bk - pe) | ((len + bk - 3) << 16), p - cand);
            nseq += (uint32_t)__popc(taken);
            // Two warp syncs stand where the previous end was shuffled: the test emulator runs the lanes in an order that
            // follows the warp's rendezvous count, and its frames (tests/golden/speed_frames.json) pin that order.
            __syncwarp();
            __syncwarp();
            cov = __reduce_or_sync(TS_FULL, mine ? zb_ones_from(lane - bk) & ~zb_ones_from(lane + len) : 0u);
        }
        anchor = cur + prev;
        // step: literals
        // the step's literals, in order: one byte per position of the block no taken match covers
        {
            const uint32_t lm = ~(cov | zb_ones_from(bn - cur));       // (positions at or past bn are no literals)
            if ((lm >> lane) & 1) lits[nlit + (uint32_t)__popc(lm & lanes_below)] = (uint8_t)v;
            nlit += (uint32_t)__popc(lm);
        }
        cur = max(cur + 32, anchor);
        // step: end
    }
#if ZB_TUNE_PAD
    if (nlit == 0xffffffffu) lits[0] = (uint8_t)__float_as_uint(pad[0] + pad[1] + pad[2] + pad[3]);   // keeps the chains live
#endif
    if (cur < bn) {                                                // the rest of the block is literals
        const uint32_t ll = bn - cur;
        for (uint32_t k = lane; k < ll; k += 32) lits[nlit + k] = buf[cur + k];
        nlit += ll;
    }
    __syncwarp();
    __threadfence_block();
    ZB_MARK(2);
    ZB_NOTE(nseq, nseq);
    ZB_NOTE(nlit, nlit);

    // ---- phase B: entropy stage into the (now free) shared block buffer and hash table, then emit
    uint32_t payload = 0xffffffffu;                                // "not compressible"
    {
        // literals section first (into `out` directly), then the sequences bit stream staged in `buf`
        uint8_t* body = out + 3;
        const uint32_t lit_bytes = zb_encode_literals(lits, nlit, body, (uint32_t*)buf, ht, lane ZB_PH_ARG);   // header + payload
        __syncwarp();
        ZB_MARK(4);
        if (nseq == 0) {
            // no match at all: the block may still be worth a compressed block with entropy-coded literals and zero sequences
            if (lit_bytes + 1 < bn) {
                if (lane == 0) body[lit_bytes] = 0;                // Number_of_Sequences = 0: the sequences section ends here
                payload = lit_bytes + 1;
            }
        } else {
            const uint32_t shdr = ze_nseq_size(nseq);
            uint8_t* sp = body + lit_bytes;
            uint32_t desc_bytes = 0;
            // the code tables of the sequence fields go next to the FSE tables, over the (now dead) Huffman scratch
            ZeCodeTabs* tabs = (ZeCodeTabs*)((uint8_t*)ht + sizeof(ZbCTab));
            for (uint32_t i = lane; i < 128; i += 32) {
                if (i < 64) tabs->ll_code[i] = g_seq_tables.ll_code[i];
                tabs->ml_code[i] = g_seq_tables.ml_code[i];
                if (i < 36) tabs->ll_bits[i] = g_seq_tables.ll_bits[i];
                if (i < 53) tabs->ml_bits[i] = g_seq_tables.ml_bits[i];
            }
            __syncwarp();
            const uint32_t sbytes = zb_encode_sequences(seqs, nseq, (uint32_t*)buf, (ZbCTab*)ht, tabs, sp + shdr, &desc_bytes, lane ZB_PH_ARG);
            ZB_MARK(6);
            const uint32_t total = lit_bytes + shdr + desc_bytes + sbytes;
            if (total < bn) {
                if (lane == 0) ze_write_nseq(sp, nseq);
                _Pragma("unroll 2")
                for (uint32_t i = lane; i < sbytes; i += 32) sp[shdr + desc_bytes + i] = buf[i];
                payload = total;
            }
        }
    }
    if (payload == 0xffffffffu) {                                  // Raw_Block
        ze_warp_copy(out + 3, src, bn, lane);
    }
    if (lane == 0) {
        const uint32_t type = payload == 0xffffffffu ? 0u : 2u;
        const uint32_t bsize = payload == 0xffffffffu ? bn : payload;
        const uint32_t hdr = (last_block ? 1u : 0u) | (type << 1) | (bsize << 3);
        out[0] = (uint8_t)hdr; out[1] = (uint8_t)(hdr >> 8); out[2] = (uint8_t)(hdr >> 16);
        A.blk_size[gblk] = 3 + bsize;
    }
    // ---- placement: the block claims its place in the frame by a decoupled look-back over the sizes of the blocks before
    // it (ze_lookback; they were launched earlier — CTAs start in grid order — so a wait is for work in flight, never for
    // work not yet scheduled) and copies itself there while it is still hot in L2: no assemble launch, no second pass.
    {
        const uint32_t bsize_all = 3 + (payload == 0xffffffffu ? bn : payload);
        unsigned long long* st = A.blk_state + (size_t)chunk * A.blocks_per_chunk;
        uint8_t* frame = A.out_base + A.out_off[chunk];
        if (blk == 0 && lane == 0) ze_frame_header(frame, clen, A.ck_state != nullptr);
        __threadfence();                                           // (the slot's bytes are this warp's own: ordered by the warp sync below)
        const uint32_t base = ze_lookback(st, blk, bsize_all, ze_frame_header_size(clen), last_block, lane);
        if (last_block && lane == 0) {
            A.out_len[chunk] = base + bsize_all + (A.ck_state ? 4u : 0u);
            if (A.ck_state) ze_ck_unit_done(A.ck_state + chunk, frame + base + bsize_all);
        }
        __syncwarp();
        ZB_MARK(7);
        ze_warp_copy(frame + base, out, bsize_all, lane);
        ZB_MARK(8);
    }
}

// ------------------------------------------------------------------------------------------ host side
inline const char* zstd_blk_scratch_alloc(ZstdBlkScratch& s, uint32_t chunk_cap, uint32_t max_batch) {
    s.blocks_per_chunk = (chunk_cap + ZB - 1) / ZB;
    s.max_batch = max_batch;
    const size_t nblk = (size_t)s.blocks_per_chunk * max_batch;
    const char* e;
    if ((e = rt::malloc_device((void**)&s.blk_out, nblk * ZB_SLOT + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.blk_size, nblk * 4 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.seqs, nblk * ZE_MAXSEQ * sizeof(uint2) + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.lits, nblk * ZB + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.blk_state, nblk * 8 + 256))) return e;
    if ((e = rt::malloc_device((void**)&s.ck_state, (size_t)max_batch * 8 + 256))) return e;
    return nullptr;
}
inline void zstd_blk_scratch_free(ZstdBlkScratch& s) {
    rt::free_device(s.blk_out); rt::free_device(s.blk_size); rt::free_device(s.seqs); rt::free_device(s.lits); rt::free_device(s.blk_state);
    rt::free_device(s.ck_state);
    s = ZstdBlkScratch{};
}
constexpr uint32_t ZB_SMEM_BYTES = ZB_WPB * ZB_SMEM_WARP_AL;
static_assert(ZB_SMEM_BYTES >= ZB_WPB * XXH_STAGE_BYTES && ZB_SMEM_WARP_AL % 16 == 0, "hashing warps stage in the block buffers");

inline int zstd_compress_batch_blocks(ZstdBlkScratch& s, rt::stream_t st, const uint8_t* in_base, const uint64_t* d_in_off,
                                      const uint32_t* d_in_len, uint32_t n_chunks, uint32_t chunk_size, bool checksum,
                                      uint8_t* out_base, const uint64_t* d_out_off, uint32_t* d_out_len, LaunchProf& prof) {
    if (n_chunks > s.max_batch) { g_zstd_err = "batch larger than the context"; return -1; }
    const uint32_t bpc = (chunk_size + ZB - 1) / ZB;
    if (bpc > s.blocks_per_chunk) { g_zstd_err = "chunk larger than the context"; return -1; }
    ZstdBlkArgs A;
    A.in_base = in_base; A.in_off = d_in_off; A.in_len = d_in_len;
    A.blk_out = s.blk_out; A.blk_size = s.blk_size; A.seqs = s.seqs; A.lits = s.lits; A.blk_state = s.blk_state;
    A.blocks_per_chunk = s.blocks_per_chunk;
    A.out_base = out_base; A.out_off = d_out_off; A.out_len = d_out_len;
    const uint32_t gx = bpc ? (bpc + ZB_WPB - 1) / ZB_WPB : 1;   // (empty chunks still get their frame from block 0)
    A.ck_state = checksum ? s.ck_state : nullptr;
    A.n_chunks = n_chunks;
    A.hash_rows = checksum ? ((n_chunks + ZB_WPB - 1) / ZB_WPB + gx - 1) / gx : 0;     // one warp per chunk (ze_hash_warp)
    const char* e = rt::memset_async(s.blk_state, 0, (size_t)s.blocks_per_chunk * n_chunks * 8, st);
    if (!e && checksum) e = rt::memset_async(s.ck_state, 0, (size_t)n_chunks * 8, st);
    if (e) { g_zstd_err = e; return -7; }
    TS_LAUNCH_P(prof, "zstd_enc_blocks", zstd_enc_blocks_kernel, dim3(gx, n_chunks + A.hash_rows), dim3(ZB_WPB * 32), ZB_SMEM_BYTES, st, A);
    e = rt::last_error();
    if (e) { g_zstd_err = e; return -7; }
    return 0;
}

}  // namespace ts
