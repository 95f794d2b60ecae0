// zstd_huf_enc.cuh — literals section of a compressed block (RFC 8878 §3.1.1.3.1, §4.2): Raw, RLE, or Huffman-compressed with
// ONE tree per 64 KiB region: the first block of the region that uses it carries the tree description
// (Compressed_Literals_Block), the later ones are Treeless_Literals_Blocks.
//   ze_huf_build          one warp, once per region: region histogram -> rank sort of the used symbols -> two-queue Huffman
//                         merge on lane 0 (depth limited to 11 by halving counts and rebuilding) -> canonical codes in the
//                         order the decoder's table is filled (weight ascending, symbol ascending) -> tree description
//                         (direct 4-bit weights, or FSE-compressed weights when byte values above 128 occur)
//   ze_huf_encode_block   one warp per block: exact size first (sum of code lengths per stream), then the four streams
//                         packed by all lanes with a shuffle suffix-scan of code lengths and atomicOr into a zeroed staging
//                         buffer in shared memory
#pragma once
#include "ts_common.cuh"
#include "zstd_format.h"
#include "index_scan.cuh"
#include "zstd_fse_enc.cuh"

namespace ts {

constexpr uint32_t ZE_HUF_MIN = 64;            // below this many literals in a block Huffman streams cannot pay for their 6-byte jump table
constexpr uint32_t ZE_HUF_REGION_MIN = 256;    // below this many literals in a region a tree cannot pay for itself
// FSE-compressed weights shave ~1.5 % off text-like data at 8 KiB granularity; with one tree per 64 KiB region the tree is
// < 0.5 % of the output, so they are used only where direct weights cannot describe the tree (symbols > 128).
constexpr bool ZE_FSE_WEIGHTS_ALWAYS = false;

struct ZeHuf {                                 // region-wide result of ze_huf_build (shared memory)
    uint32_t ok;                               // 0: no usable tree (blocks write Raw / RLE literals)
    uint32_t tree_bytes;                       // size of the description in `desc`
    uint32_t max_len;
    uint8_t desc[132];                         // header byte + weights (direct: <= 1 + 64; FSE-compressed: <= 1 + 127)
};

// Code lengths and canonical codes of a Huffman tree over the m >= 2 used symbols, one warp.  keys[] (at work + 1280: count << 8 |
// symbol for each used symbol, distinct) is rewritten with halved counts while the tree is deeper than 11 levels, at most
// `max_rounds` times.  On success ctab[s] = code | len << 16 for every used symbol (ctab must be zero on entry), *total_bits =
// sum of len * hist[s], and the result is max_len <= HUF_MAX_LOG; otherwise the result is larger and ctab is untouched.
//   rank sort of the keys (lane-parallel) -> two-queue merge on lane 0 (queue heads in registers; ties take the leaf, which
//   the format of the frames depends on) -> depths by pointer jumping over parent[] (ceil(log2(m - 1)) warp rounds) ->
//   canonical codes, weight ascending then symbol ascending: the first code of each weight class from a scan of the class
//   sizes, then 32 symbols per step, each taking its class's next code plus its rank among the step's symbols of its class.
// work: >= 1296 words of shared memory.
__device__ __forceinline__ uint32_t ze_huf_codes(const uint32_t* hist, uint32_t m, uint32_t last_sym, uint32_t max_rounds,
                                                 uint32_t* ctab, uint32_t* work, uint32_t* total_bits, uint32_t lane) {
    uint32_t* keys = work + 1280;              // [256]
    uint32_t* sorted = work;                   // [256]
    uint32_t* nodew = work + 256;              // [512] node weights while merging
    uint16_t* anc1 = (uint16_t*)(work + 256);  // [512] then (dead weights) the second buffer of the pointer jumping
    uint8_t* dep1 = (uint8_t*)(work + 512);    // [512]
    uint16_t* anc0 = (uint16_t*)(work + 768);  // [512] parent[], then the first buffer
    uint8_t* dep0 = (uint8_t*)(work + 1024);   // [512]
    uint32_t* wcnt = work + 1200;              // [16] symbols per weight class
    const uint32_t root = 2 * m - 2;
    const uint32_t jumps = m <= 2 ? 0u : 32u - (uint32_t)__clz((int)(m - 2));   // 2^jumps >= m - 1 >= any depth
    uint32_t max_len = 0xffu;
    const uint8_t* depth = dep0;
    for (uint32_t round = 0; round < max_rounds; round++) {
        for (uint32_t e = lane; e < m; e += 32) {                         // rank sort (keys are distinct)
            const uint32_t key = keys[e];
            uint32_t r = 0;
            _Pragma("unroll 2")
            for (uint32_t j = 0; j < m; j++) r += keys[j] < key ? 1u : 0u;
            sorted[r] = key;
            nodew[r] = key >> 8;
        }
        __syncwarp();
        if (lane == 0) {
            uint32_t li = 0, ii = m, ni = m;
            uint32_t wl = nodew[0], wi = 0;                               // heads of the leaf and internal-node queues
            _Pragma("unroll 1")
            for (uint32_t k = 0; k + 1 < m; k++) {
                uint32_t a, b, wa, wb;
                if (li < m && (ii >= ni || wl <= wi)) { a = li++; wa = wl; wl = nodew[li]; } else { a = ii++; wa = wi; wi = nodew[ii]; }
                if (li < m && (ii >= ni || wl <= wi)) { b = li++; wb = wl; wl = nodew[li]; } else { b = ii++; wb = wi; wi = nodew[ii]; }
                nodew[ni] = wa + wb;
                anc0[a] = (uint16_t)ni; anc0[b] = (uint16_t)ni;
                if (ii == ni) wi = wa + wb;                               // the new node heads an empty queue
                ni++;
            }
            anc0[root] = (uint16_t)root;
        }
        __syncwarp();
        // depth = edges to the root: dep holds the distance to anc, both double each round until every anc is the root
        for (uint32_t e = lane; e <= root; e += 32) dep0[e] = e == root ? 0 : 1;
        __syncwarp();
        const uint16_t* ai = anc0; const uint8_t* di = dep0;
        uint16_t* ao = anc1; uint8_t* dn = dep1;
        for (uint32_t j = 0; j < jumps; j++) {
            for (uint32_t e = lane; e <= root; e += 32) { const uint32_t a = ai[e]; dn[e] = (uint8_t)(di[e] + di[a]); ao[e] = ai[a]; }
            __syncwarp();
            const uint16_t* ta = ai; const uint8_t* td = di;
            ai = ao; di = dn; ao = (uint16_t*)ta; dn = (uint8_t*)td;
        }
        depth = di;
        uint32_t mx = 0;
        for (uint32_t e = lane; e < m; e += 32) mx = max(mx, (uint32_t)di[e]);
        max_len = __reduce_max_sync(TS_FULL, mx);
        if (max_len <= (uint32_t)zf::HUF_MAX_LOG) break;
        for (uint32_t e = lane; e < m; e += 32) {                         // flatten the distribution and retry
            const uint32_t key = keys[e];
            keys[e] = ((((key >> 8) + 1) >> 1) << 8) | (key & 0xff);
        }
        __syncwarp();
    }
    if (max_len > (uint32_t)zf::HUF_MAX_LOG) return max_len;

    // ---- canonical codes: weight w = max_len + 1 - len; cells are dealt weight-ascending, symbol-ascending
    if (lane < 16) wcnt[lane] = 0;
    __syncwarp();
    uint32_t tb = 0;
    for (uint32_t i = lane; i < m; i += 32) {
        const uint32_t s = sorted[i] & 0xff, len = depth[i];
        ctab[s] = len << 16;                                              // park the length
        atomicAdd(&wcnt[max_len + 1 - len], 1u);
        tb += len * hist[s];
    }
    *total_bits = __reduce_add_sync(TS_FULL, tb);
    __syncwarp();
    // lane w (1 .. max_len) keeps the next code of weight class w
    const bool cls = lane >= 1 && lane <= max_len;
    const uint32_t cells = cls ? wcnt[lane] << (lane - 1) : 0u;
    const uint32_t inc = warp_inclusive_scan_u32(cells, lane);
    uint32_t next = cls ? (inc - cells) >> (lane - 1) : 0u;
    const uint32_t lt = (1u << lane) - 1;
    for (uint32_t s0 = 0; s0 <= last_sym; s0 += 32) {
        const uint32_t s = s0 + lane;
        const uint32_t len = ctab[s] >> 16;
        const uint32_t w = len ? max_len + 1 - len : 0u;
        const uint32_t first = __shfl_sync(TS_FULL, next, w);
        uint32_t rank = 0;
        for (uint32_t c = 1; c <= max_len; c++) {
            const uint32_t bm = __ballot_sync(TS_FULL, w == c);
            if (w == c) rank = (uint32_t)__popc(bm & lt);
            if (lane == c) next += (uint32_t)__popc(bm);
        }
        if (len) ctab[s] = (first + rank) | (len << 16);
    }
    __syncwarp();
    return max_len;
}

// Compacts the used symbols of hist[256] into keys at work + 1280 (count << 8 | symbol, ascending symbol order, where
// ze_huf_codes reads them; counts must stay below 2^24) and returns their number m.  *pays: the Shannon estimate of the
// Huffman-coded size (in 1/16 bits: sum c * (log2(n) - log2(c)), log2 by leading zeros + a linear fraction) leaves room
// to beat the n literals stored raw.  One warp.
__device__ __forceinline__ uint32_t ze_huf_symbols(const uint32_t* hist, uint32_t n, uint32_t* work, bool* pays, uint32_t lane) {
    uint32_t* keys = work + 1280;
    uint32_t mine = 0;                                                    // 8 symbols per lane
    for (uint32_t k = 0; k < 8; k++) mine += hist[lane * 8 + k] ? 1u : 0u;
    const uint32_t inc = warp_inclusive_scan_u32(mine, lane);
    const uint32_t m = __shfl_sync(TS_FULL, inc, 31);
    uint32_t at = inc - mine, cost = 0;
    const uint32_t hn = (uint32_t)zf::highbit32(n);
    const uint32_t lgn = (hn << 4) + (((n << (31 - hn)) >> 27) & 15) + 1;
    for (uint32_t k = 0; k < 8; k++) {
        const uint32_t s = lane * 8 + k, c = hist[s];
        if (c) {
            keys[at++] = (c << 8) | s;
            const uint32_t hb = (uint32_t)zf::highbit32(c);
            const uint32_t lg16 = (hb << 4) + (((c << (31 - hb)) >> 27) & 15);       // ~ 16 * log2(c)
            cost += c * (lgn - lg16);
        }
    }
    const uint32_t bits16 = __reduce_add_sync(TS_FULL, cost);
    *pays = (bits16 >> 7) + m / 2 + 16 < n;                               // else >= n bytes even before rounding losses
    __syncwarp();
    return m;
}

constexpr uint32_t ZE_NO_TREE = 0xffffffffu;

// Tree description of the codes in ctab (RFC 8878 §4.2.1) for the weights of symbols 0 .. nweights-1: direct 4-bit weights
// (at most 128 of them) or FSE-compressed weights, the shorter form.  The FSE form is what lets alphabets above byte value
// 128 (binary payloads) be Huffman-coded.  Written to desc (shared memory, never more than 128 bytes); returns its size, or
// ZE_NO_TREE when neither form can describe the tree.  work: the scratch given to ze_huf_codes (bytes 6144 .. 7504 are
// used here).  One warp.
__device__ __forceinline__ uint32_t ze_huf_tree_desc(const uint32_t* ctab, uint32_t nweights, uint32_t max_len, uint8_t* desc,
                                                     uint32_t* work, uint32_t lane) {
    uint8_t* wts = (uint8_t*)(work + 1536);                               // weights, then FSE tables, in dead tree scratch
    uint32_t* wcnt = (uint32_t*)(wts + 256);                              // [16]
    uint16_t* wst = (uint16_t*)(wcnt + 16);                               // [64]
    zf::FseCSym* wsy = (zf::FseCSym*)(wst + 64);                          // [16]
    uint8_t* wscratch = (uint8_t*)(wsy + 16);                             // >= 784 bytes
    if (lane < 16) wcnt[lane] = 0;
    __syncwarp();
    for (uint32_t s = lane; s < nweights; s += 32) {
        const uint32_t l = ctab[s] >> 16;
        const uint32_t w = l ? max_len + 1 - l : 0;
        wts[s] = (uint8_t)w;
        atomicAdd(&wcnt[w], 1u);
    }
    __syncwarp();
    uint32_t tree_bytes = nweights <= 128 ? 1 + (nweights + 1) / 2 : ZE_NO_TREE;
    if (nweights >= 2 && (ZE_FSE_WEIGHTS_ALWAYS || nweights > 128)) {
        const uint32_t wr = ze_build_kind(wcnt, 13, nweights, zf::HUFW_MAX_LOG, zf::HUFW_MAX_LOG, nullptr, nullptr, wst, wsy,
                                          wscratch, desc + 1, false, lane);
        const uint32_t dsz = ze_kind_bytes(wr);
        const ZeKind wk = ze_kind_of(wr);
        if (wk.mode == 2) {
            uint32_t fsz = 0;
            if (lane == 0) {                                              // two interleaved states, last weight first
                uint8_t* o = desc + 1 + dsz;
                const uint32_t cap = 127 - dsz;                           // bytes left for the stream in 128
                uint64_t acc = 0; uint32_t nb = 0, ob = 0;
                uint32_t st_even = 0, st_odd = 0;                         // the chains of the even and the odd weights
                for (uint32_t q = 0; q < 2; q++) {                        // FSE_initCState2 for the two last weights
                    const uint32_t i = nweights - 1 - q;
                    const zf::FseCSym c = wsy[wts[i]];
                    const uint32_t nbo = (uint32_t)(c.delta_nb_bits + (1 << 15)) >> 16;
                    const uint32_t v = (nbo << 16) - (uint32_t)c.delta_nb_bits;
                    const uint32_t s0 = wst[(int32_t)(v >> nbo) + c.delta_find_state];
                    if (i & 1) st_odd = s0; else st_even = s0;
                }
                // a full buffer stops the walk: the flush below then cannot finish and the form is rejected
                for (int32_t i = (int32_t)nweights - 3; i >= 0 && ob < cap; i--) {
                    const zf::FseCSym c = wsy[wts[i]];
                    const uint32_t sv = (i & 1) ? st_odd : st_even;
                    const uint32_t nbo = (sv + (uint32_t)c.delta_nb_bits) >> 16;
                    acc |= (uint64_t)(sv & ((1u << nbo) - 1)) << nb; nb += nbo;
                    const uint32_t s1 = wst[(int32_t)(sv >> nbo) + c.delta_find_state];
                    if (i & 1) st_odd = s1; else st_even = s1;
                    while (nb >= 8) { o[ob++] = (uint8_t)acc; acc >>= 8; nb -= 8; }       // nb <= 13: one byte at most
                }
                acc |= (uint64_t)(st_odd & ((1u << wk.log) - 1)) << nb; nb += wk.log;     // flush odd chain, then even chain
                acc |= (uint64_t)(st_even & ((1u << wk.log) - 1)) << nb; nb += wk.log;
                acc |= 1ull << nb; nb += 1;                                                // end mark
                while (nb > 0 && ob < cap) { o[ob++] = (uint8_t)acc; acc >>= 8; nb = nb >= 8 ? nb - 8 : 0; }
                fsz = nb ? ZE_NO_TREE : dsz + ob;                         // did not fit 127 bytes: unusable
            }
            fsz = __shfl_sync(TS_FULL, fsz, 0);
            if (fsz < 128 && 1 + fsz < tree_bytes) {
                if (lane == 0) desc[0] = (uint8_t)fsz;
                tree_bytes = 1 + fsz;
                __syncwarp();
                return tree_bytes;
            }
        }
    }
    if (tree_bytes != ZE_NO_TREE) {
        if (lane == 0) {                           // (one lane: a warp-wide loop costs the speed kernel 6 registers)
            desc[0] = (uint8_t)(127 + nweights);
            for (uint32_t i = 0; 2 * i < nweights; i++)
                desc[1 + i] = (uint8_t)((wts[2 * i] << 4) | (2 * i + 1 < nweights ? wts[2 * i + 1] : 0u));
        }
    }
    __syncwarp();
    return tree_bytes;
}

// Region-wide tree.  hist[256] (counts), ctab[256] out (code | len << 16, 0 = unused symbol), work: >= 7.5 KiB of
// shared-memory scratch, n = literals in the region.  One warp.
__device__ TS_NOINLINE void ze_huf_build(uint32_t* hist, uint32_t* ctab, uint32_t* work, uint32_t n, ZeHuf* hf, uint32_t lane) {
    if (lane == 0) { hf->ok = 0; hf->tree_bytes = 0; hf->max_len = 0; }
    for (uint32_t i = lane; i < 256; i += 32) ctab[i] = 0;
    __syncwarp();
    if (n < ZE_HUF_REGION_MIN) return;
    bool pays;
    const uint32_t m = ze_huf_symbols(hist, n, work, &pays, lane);
    if (m < 2 || !pays) return;                // a single symbol: every block of the region is an RLE literals block
    const uint32_t last_sym = work[1280 + m - 1] & 0xff;
    uint32_t total_bits;
    const uint32_t max_len = ze_huf_codes(hist, m, last_sym, 20, ctab, work, &total_bits, lane);
    if (max_len > (uint32_t)zf::HUF_MAX_LOG) return;
    const uint32_t tree_bytes = ze_huf_tree_desc(ctab, last_sym, max_len, hf->desc, work, lane);   // symbols 0 .. last_sym-1 are listed
    if (tree_bytes == ZE_NO_TREE) return;
    if (lane == 0) { hf->ok = 1; hf->tree_bytes = tree_bytes; hf->max_len = max_len; }
    __syncwarp();
}

struct ZeLitBlock {                  // what a block's literals section will consist of (decided before anything is written)
    uint32_t kind;                   // 0 Raw, 1 RLE, 2 Huffman (tree or treeless decided later)
    uint32_t n;                      // regenerated size
    uint32_t stream_bytes;           // Huffman: bytes of the four streams
    uint32_t ssz[3];                 // Huffman: sizes of streams 1-3 (jump table)
    uint32_t rle_byte;
};

// Exact sizes of the four Huffman streams of this block (no output).  Returns false when a literal has no code.
__device__ __forceinline__ void ze_huf_plan_block(const uint8_t* __restrict__ lits, uint32_t n, const uint32_t* ctab, const ZeHuf* hf,
                                                  ZeLitBlock* lb, uint32_t lane) {
    uint32_t kind = 0, stream_bytes = 0, s1 = 0, s2 = 0, s3 = 0, rle = 0;
    if (n >= 1) {                                                         // RLE: all literals equal
        const uint8_t first = lits[0];
        bool same = true;
        for (uint32_t i = lane; i < n; i += 32) same = same && lits[i] == first;
        if (__all_sync(TS_FULL, same)) { kind = 1; rle = first; }
    }
    if (kind == 0 && hf->ok && n >= ZE_HUF_MIN) {
        const uint32_t seg = (n + 3) / 4;
        uint32_t tot[4];
        bool coded = true;
        for (uint32_t st = 0; st < 4; st++) {
            const uint32_t a = st * seg, b = st < 3 ? min(n, a + seg) : n;
            uint32_t bits = 0;
            for (uint32_t i = a + lane; i < b; i += 32) { const uint32_t l = ctab[lits[i]] >> 16; coded = coded && l != 0; bits += l; }
            tot[st] = __reduce_add_sync(TS_FULL, bits);
        }
        if (__all_sync(TS_FULL, coded)) {
            s1 = (tot[0] + 8) >> 3; s2 = (tot[1] + 8) >> 3; s3 = (tot[2] + 8) >> 3;         // + end mark, rounded up
            const uint32_t s4 = (tot[3] + 8) >> 3;
            stream_bytes = s1 + s2 + s3 + s4;
            if (stream_bytes + 6 + 2 < n && s1 < 65536 && s2 < 65536 && s3 < 65536) kind = 2;   // must beat Raw (3-byte header vs up to 5)
        }
    }
    if (lane == 0) { lb->kind = kind; lb->n = n; lb->stream_bytes = stream_bytes; lb->ssz[0] = s1; lb->ssz[1] = s2; lb->ssz[2] = s3; lb->rle_byte = rle; }
    __syncwarp();
}

// The four streams of this block into `work` (shared-memory words, >= stream_bytes + 8 bytes).  Layout: streams back to back.
__device__ __forceinline__ void ze_huf_encode_block(const uint8_t* __restrict__ lits, uint32_t n, const uint32_t* ctab, uint32_t stream_bytes,
                                                    uint32_t* work, uint32_t lane) {
    for (uint32_t i = lane; i < (stream_bytes + 11) / 4; i += 32) work[i] = 0;
    __syncwarp();
    const uint32_t seg = (n + 3) / 4;
    uint32_t byte_pos = 0;
    _Pragma("unroll 1")
    for (uint32_t st = 0; st < 4; st++) {
        const uint32_t s0 = st * seg, s1 = st < 3 ? min(n, s0 + seg) : n;
        const uint32_t cnt = s1 > s0 ? s1 - s0 : 0;
        const uint32_t per = (cnt + 31) / 32;
        const uint32_t a = min(cnt, lane * per), b = min(cnt, a + per);   // this lane's run [a, b) of the stream
        uint32_t mybits = 0;
        _Pragma("unroll 2")
        for (uint32_t i = a; i < b; i++) mybits += ctab[lits[s0 + i]] >> 16;
        // symbols are written last-to-first: the offset of a run is the number of bits of all LATER runs
        const uint32_t incb = warp_inclusive_scan_u32(mybits, lane);
        const uint32_t total = __shfl_sync(TS_FULL, incb, 31);
        uint32_t off = byte_pos * 8 + (total - incb);
        for (uint32_t i = b; i > a; i--) {
            const uint32_t c = ctab[lits[s0 + i - 1]];
            const uint32_t len = c >> 16, code = c & 0xffff;
            const uint32_t w = off >> 5, sh = off & 31;
            atomicOr(&work[w], code << sh);
            if (sh + len > 32) atomicOr(&work[w + 1], code >> (32 - sh));
            off += len;
        }
        if (lane == 0) {                                                  // end mark
            const uint32_t o = byte_pos * 8 + total;
            atomicOr(&work[o >> 5], 1u << (o & 31));
        }
        byte_pos += (total + 1 + 7) >> 3;
        __syncwarp();
    }
}

// Literals_Section_Header for a Raw / RLE literals block (always the 3-byte form) — one lane.
__device__ __forceinline__ uint32_t ze_lit_header_raw(uint8_t* body, uint32_t type, uint32_t n) {
    body[0] = (uint8_t)(type | (3u << 2) | ((n & 0xf) << 4));
    body[1] = (uint8_t)(n >> 4);
    body[2] = (uint8_t)(n >> 12);
    return 3;
}
// ... and for a Compressed (type 2) / Treeless (type 3) block with four streams; comp = tree + jump table + streams.
__device__ __forceinline__ uint32_t ze_lit_header_huf_size(uint32_t n, uint32_t comp) {
    return (n < 1024 && comp < 1024) ? 3u : (n < 16384 && comp < 16384) ? 4u : 5u;
}
__device__ __forceinline__ uint32_t ze_lit_header_huf(uint8_t* body, uint32_t type, uint32_t n, uint32_t comp) {
    const uint32_t hsz = ze_lit_header_huf_size(n, comp);
    const uint32_t sf = hsz - 2;                                          // 1, 2, 3: all with four streams
    uint64_t h;
    if (hsz == 3) h = type | (sf << 2) | ((uint64_t)n << 4) | ((uint64_t)comp << 14);
    else if (hsz == 4) h = type | (sf << 2) | ((uint64_t)n << 4) | ((uint64_t)comp << 18);
    else h = type | (sf << 2) | ((uint64_t)n << 4) | ((uint64_t)comp << 22);
    for (uint32_t k = 0; k < hsz; k++) body[k] = (uint8_t)(h >> (8 * k));
    return hsz;
}
// Jump table of a four-stream literals section: the sizes of streams 1-3, packed 16 bits each in `sizes` — one lane.
__device__ __forceinline__ void ze_lit_jump_table(uint8_t* j, uint64_t sizes) {
    for (uint32_t k = 0; k < 6; k++) j[k] = (uint8_t)(sizes >> (8 * k));
}

}  // namespace ts
