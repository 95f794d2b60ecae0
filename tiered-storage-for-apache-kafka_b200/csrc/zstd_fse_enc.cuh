// zstd_fse_enc.cuh — sequences section of a compressed block (RFC 8878 §3.1.1.3.2) with per-block FSE tables.
//
// One warp per block.  For each of literal-length / offset / match-length codes the block picks
//   RLE_Mode            when a single code occurs,
//   Predefined_Mode     for blocks with few sequences (a table description would not pay),
//   FSE_Compressed_Mode otherwise: counts -> normalised distribution (every present code >= 1 cell, so the
//                       spread has the closed form pos(i) = i*step & mask and can be built by all lanes),
//                       table description written in libzstd's FSE_writeNCount format, encoding tables
//                       (state table + per-symbol transform) built in shared memory.
// Encoding: code / extra bits per lane, the three state chains on lanes 0-2 (the only serial part), fields packed
// by all lanes through a shuffle prefix sum and shared-memory atomicOr.
#pragma once
#include "ts_common.cuh"
#include "zstd_format.h"
#include "index_scan.cuh"

namespace ts {

constexpr uint32_t ZE_NSYM_LL = 36, ZE_NSYM_ML = 53, ZE_NSYM_OF = 32;
constexpr uint32_t ZE_PREDEF_BELOW = 64;          // fewer sequences than this: Predefined_Mode

// One set of tables per 64 KiB region (up to 8192 sequences): table logs as FSE_optimalTableLog picks them, i.e. up to the
// format's maxima 9 / 9 / 8 (LL / ML / OF); the predefined tables are 6 / 6 / 5 bits.
constexpr uint32_t ZE_MAX_TLOG = 9;
struct ZeCTab {                                   // per region, in the (free) hash-table area during the entropy phases
    uint16_t st_ll[1 << zf::LL_MAX_LOG], st_ml[1 << zf::ML_MAX_LOG], st_of[1 << zf::OF_MAX_LOG];
    zf::FseCSym sy_ll[ZE_NSYM_LL], sy_ml[ZE_NSYM_ML], sy_of[ZE_NSYM_OF];
};
static_assert(sizeof(ZeCTab) <= 4096, "ZeCTab must fit its slot of the hash-table area");

struct ZeKind {                                   // uniform per-kind parameters after table selection
    uint32_t mode;                                // 0 predefined, 1 RLE, 2 FSE compressed
    uint32_t log;                                 // table log (0 for RLE)
};
// ze_build_kind's result in one register (no stack frame for an out-parameter of the non-inlined call):
// description bytes | mode << 8 | log << 12 | largest present code << 16
__device__ __forceinline__ uint32_t ze_kind_bytes(uint32_t r) { return r & 0xff; }
__device__ __forceinline__ ZeKind ze_kind_of(uint32_t r) { return ZeKind{(r >> 8) & 3, (r >> 12) & 15}; }
__device__ __forceinline__ uint32_t ze_kind_max_sym(uint32_t r) { return r >> 16; }

// ---- table description, libzstd FSE_writeNCount layout.  One lane.  Returns bytes written.
__device__ TS_NOINLINE uint32_t ze_write_ncount(uint8_t* out, const uint32_t* norm, uint32_t alphabet, uint32_t log) {
    const int table_size = 1 << log;
    uint64_t bit_stream = log - 5;
    int bit_count = 4;
    int remaining = table_size + 1, threshold = table_size, nb_bits = (int)log + 1;
    uint32_t symbol = 0, o = 0;
    bool prev0 = false;
    while (symbol < alphabet && remaining > 1) {
        if (prev0) {
            uint32_t start = symbol;
            while (symbol < alphabet && !norm[symbol]) symbol++;
            if (symbol == alphabet) break;
            while (symbol >= start + 24) {
                start += 24;
                bit_stream += 0xFFFFull << bit_count; bit_count += 16;
                while (bit_count >= 16) { out[o++] = (uint8_t)bit_stream; out[o++] = (uint8_t)(bit_stream >> 8); bit_stream >>= 16; bit_count -= 16; }
            }
            while (symbol >= start + 3) { start += 3; bit_stream += 3ull << bit_count; bit_count += 2; }
            bit_stream += (uint64_t)(symbol - start) << bit_count; bit_count += 2;
            while (bit_count > 16) { out[o++] = (uint8_t)bit_stream; out[o++] = (uint8_t)(bit_stream >> 8); bit_stream >>= 16; bit_count -= 16; }
        }
        int count = (int)norm[symbol++];
        const int mx = (2 * threshold - 1) - remaining;
        remaining -= count;
        count++;                                             // +1 for extra accuracy
        if (count >= threshold) count += mx;
        bit_stream += (uint64_t)count << bit_count;
        bit_count += nb_bits;
        bit_count -= (count < mx) ? 1 : 0;
        prev0 = (count == 1);
        while (remaining < threshold) { nb_bits--; threshold >>= 1; }
        while (bit_count > 16) { out[o++] = (uint8_t)bit_stream; out[o++] = (uint8_t)(bit_stream >> 8); bit_stream >>= 16; bit_count -= 16; }
    }
    out[o] = (uint8_t)bit_stream; out[o + 1] = (uint8_t)(bit_stream >> 8);
    return o + (uint32_t)((bit_count + 7) / 8);
}

// ---- choose the mode of one kind and build its encoding tables.  Warp-uniform.
// cnt[alphabet]: histogram on entry, normalised counts on exit (FSE mode).  scratch: >= 512 + 4*68 bytes of shared memory.
// Writes the table description at desc (the RLE byte, or FSE_writeNCount on lane 0) unless desc is null, when the caller
// writes it.  Returns the packed result above.
__device__ TS_NOINLINE uint32_t ze_build_kind(uint32_t* cnt, uint32_t alphabet, uint32_t N, uint32_t max_log, uint32_t default_log,
                                                  const uint16_t* pre_state, const zf::FseCSym* pre_sym, uint16_t* st, zf::FseCSym* sy,
                                                  uint8_t* scratch, uint8_t* desc, bool allow_predefined, uint32_t lane) {
    const uint32_t c0 = lane < alphabet ? cnt[lane] : 0, c1 = lane + 32 < alphabet ? cnt[lane + 32] : 0;
    const uint32_t used0 = __ballot_sync(TS_FULL, c0 != 0), used1 = __ballot_sync(TS_FULL, c1 != 0);
    const uint32_t nused = (uint32_t)__popc(used0) + (uint32_t)__popc(used1);
    const uint32_t max_sym = used1 ? 32 + (31 - (uint32_t)__clz((int)used1)) : 31 - (uint32_t)__clz((int)used0);
    if (nused == 1) {                                        // RLE_Mode: one byte, states carry no bits
        if (lane == 0 && desc) desc[0] = (uint8_t)max_sym;
        return 1u | 1u << 8 | max_sym << 16;
    }
    if (allow_predefined && N < ZE_PREDEF_BELOW) {           // Predefined_Mode
        const uint32_t size = 1u << default_log;
        for (uint32_t i = lane; i < size; i += 32) st[i] = pre_state[i];
        for (uint32_t i = lane; i < alphabet; i += 32) sy[i] = pre_sym[i];
        __syncwarp();
        return default_log << 12 | max_sym << 16;
    }
    // ---- FSE_Compressed_Mode.  Table log as FSE_optimalTableLog picks it.
    uint32_t log = max_log;
    const uint32_t max_bits_src = (uint32_t)zf::highbit32(N - 1) - 2;
    const uint32_t min_bits = min((uint32_t)zf::highbit32(N) + 1, (uint32_t)zf::highbit32(max_sym) + 2);
    if (max_bits_src < log) log = max_bits_src;
    if (min_bits > log) log = min_bits;
    if (log < 5) log = 5;
    if (log > max_log) log = max_log;
    if (log > ZE_MAX_TLOG) log = ZE_MAX_TLOG;                // cannot bind (max_log <= 9); keeps the tables in bounds regardless
    const uint32_t size = 1u << log;
    // normalise: floor share, at least one cell per present code, remainder to (or excess from) the largest codes
    uint32_t p0 = c0 ? max(1u, (uint32_t)(((uint64_t)c0 << log) / N)) : 0u;
    uint32_t p1 = c1 ? max(1u, (uint32_t)(((uint64_t)c1 << log) / N)) : 0u;
    int32_t diff = (int32_t)size - (int32_t)__reduce_add_sync(TS_FULL, p0 + p1);
    while (diff != 0) {
        const uint32_t best = __reduce_max_sync(TS_FULL, max(p0 << 6 | (63 - lane), p1 ? (p1 << 6 | (31 - lane)) : 0u));
        const uint32_t who = best & 63, val = best >> 6;     // largest normalised count; ties -> lowest symbol
        int32_t delta = diff > 0 ? diff : -min((int32_t)val - 1, -diff);
        if (delta == 0) break;                               // cannot shrink further (cannot happen: size >= nused)
        if (who >= 32) { if (lane == 63 - who) p0 = (uint32_t)((int32_t)p0 + delta); }
        else { if (lane == 31 - who) p1 = (uint32_t)((int32_t)p1 + delta); }
        diff -= delta;
    }
    if (lane < alphabet) cnt[lane] = p0;
    if (lane + 32 < alphabet) cnt[lane + 32] = p1;
    // cumulative starts (exclusive scan over symbols) -> scratch cum[0..64]
    uint32_t* cum = (uint32_t*)(scratch + 512);
    const uint32_t inc0 = warp_inclusive_scan_u32(p0, lane);
    const uint32_t tot0 = __shfl_sync(TS_FULL, inc0, 31);
    const uint32_t inc1 = warp_inclusive_scan_u32(p1, lane) + tot0;
    cum[lane] = inc0 - p0; cum[32 + lane] = inc1 - p1;
    if (lane == 0) cum[64] = size;
    __syncwarp();
    // per-symbol transform (FSE_buildCTable symbolTT)
    for (uint32_t s = lane; s < alphabet; s += 32) {
        const uint32_t n = cnt[s];
        zf::FseCSym e;
        if (n == 0) { e.delta_nb_bits = (int32_t)(((log + 1) << 16) - size); e.delta_find_state = 0; }
        else if (n == 1) { e.delta_nb_bits = (int32_t)((log << 16) - size); e.delta_find_state = (int32_t)cum[s] - 1; }
        else {
            const uint32_t max_bits_out = log - (uint32_t)zf::highbit32(n - 1);
            e.delta_nb_bits = (int32_t)((max_bits_out << 16) - (n << max_bits_out));
            e.delta_find_state = (int32_t)cum[s] - (int32_t)n;
        }
        sy[s] = e;
    }
    // spread: cell i of the emission order lands at (i * step) & mask; find its symbol by binary search in cum
    uint8_t* symbol_of = scratch;
    const uint32_t mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    for (uint32_t i = lane; i < size; i += 32) {
        uint32_t lo = 0, hi = 64;                            // largest s with cum[s] <= i
        while (hi - lo > 1) { const uint32_t mid = (lo + hi) >> 1; if (cum[mid] <= i) lo = mid; else hi = mid; }
        symbol_of[(i * step) & mask] = (uint8_t)lo;
    }
    __syncwarp();
    // state table: cells of a symbol, in increasing position, get consecutive slots starting at cum[symbol]
    for (uint32_t u0 = 0; u0 < size; u0 += 32) {
        const uint32_t u = u0 + lane;
        const uint32_t s = symbol_of[u];
        const uint32_t same = __match_any_sync(TS_FULL, s);
        const uint32_t rank = (uint32_t)__popc(same & ((1u << lane) - 1));
        const uint32_t base = cum[s];
        st[base + rank] = (uint16_t)(size + u);
        __syncwarp();
        if (rank == 0) cum[s] = base + (uint32_t)__popc(same);
        __syncwarp();
    }
    uint32_t bytes = 0;
    if (desc) {
        if (lane == 0) bytes = ze_write_ncount(desc, cnt, max_sym + 1, log);
        bytes = __shfl_sync(TS_FULL, bytes, 0);
    }
    __syncwarp();
    return bytes | 2u << 8 | log << 12 | max_sym << 16;
}

}  // namespace ts
