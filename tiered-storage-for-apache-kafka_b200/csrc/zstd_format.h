// zstd_format.h — RFC 8878 constants and FSE table construction shared by the compressor and decompressor.
//
// The reference reaches this format through com.github.luben:zstd-jni:1.5.6-9 (libzstd 1.5.6), which is not in
// the reference repository; the call sites are core/M/transform/CompressionChunkEnumeration.java:52-61 and
// core/M/transform/DecompressionChunkEnumeration.java:41-45.  Everything here restates the published format
// (RFC 8878 §3.1.1.3-§3.1.1.5, §4.1): code tables, default distributions, FSE spread/state tables.
#pragma once
#include <stdint.h>

#ifndef __CUDACC__
#ifndef __host__
#define __host__
#endif
#ifndef __device__
#define __device__
#endif
#endif

namespace ts {
namespace zf {

constexpr uint32_t MAGIC = 0xFD2FB528u;
constexpr uint32_t BLOCK_MAX = 128 * 1024;        // Block_Maximum_Size upper bound
constexpr int LL_MAX_LOG = 9, ML_MAX_LOG = 9, OF_MAX_LOG = 8, HUF_MAX_LOG = 11, HUFW_MAX_LOG = 6;
constexpr int LL_NSYM = 36, ML_NSYM = 53, OF_NSYM_DEFAULT = 29, OF_NSYM = 32;
constexpr int LL_DEFAULT_LOG = 6, ML_DEFAULT_LOG = 6, OF_DEFAULT_LOG = 5;

// ---- sequence code tables (RFC 8878 §3.1.1.3.2.1.1) ----
struct SeqTables {
    uint8_t ll_bits[36]; uint32_t ll_base[36];
    uint8_t ml_bits[53]; uint32_t ml_base[53];
    uint8_t ll_code[64]; uint8_t ml_code[128];
    int16_t ll_norm[36]; int16_t ml_norm[53]; int16_t of_norm[29];
};

constexpr SeqTables make_seq_tables() {
    SeqTables t{};
    const uint8_t llb[36] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0, 1,1,1,1,2,2,3,3,4,6,7,8,9,10,11,12,13,14,15,16};
    const uint8_t mlb[53] = {0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,0,
                             1,1,1,1,2,2,3,3,4,4,5,7,8,9,10,11,12,13,14,15,16};
    uint32_t b = 0;
    for (int i = 0; i < 36; i++) { t.ll_bits[i] = llb[i]; t.ll_base[i] = b; b += 1u << llb[i]; }
    b = 3;
    for (int i = 0; i < 53; i++) { t.ml_bits[i] = mlb[i]; t.ml_base[i] = b; b += 1u << mlb[i]; }
    for (int v = 0; v < 64; v++) { int c = 0; for (int i = 0; i < 36; i++) if (t.ll_base[i] <= (uint32_t)v) c = i; t.ll_code[v] = (uint8_t)c; }
    for (int v = 0; v < 128; v++) { int c = 0; for (int i = 0; i < 53; i++) if (t.ml_base[i] <= (uint32_t)v + 3) c = i; t.ml_code[v] = (uint8_t)c; }
    const int16_t lln[36] = {4,3,2,2,2,2,2,2,2,2,2,2,2,1,1,1,2,2,2,2,2,2,2,2,2,3,2,1,1,1,1,1,-1,-1,-1,-1};
    const int16_t mln[53] = {1,4,3,2,2,2,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,
                             1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1,-1,-1};
    const int16_t ofn[29] = {1,1,1,1,1,1,2,2,2,1,1,1,1,1,1,1,1,1,1,1,1,1,1,1,-1,-1,-1,-1,-1};
    for (int i = 0; i < 36; i++) t.ll_norm[i] = lln[i];
    for (int i = 0; i < 53; i++) t.ml_norm[i] = mln[i];
    for (int i = 0; i < 29; i++) t.of_norm[i] = ofn[i];
    return t;
}

__host__ __device__ inline int highbit32(uint32_t v) {       // v != 0
#if defined(__CUDA_ARCH__)
    return 31 - __clz((int)v);
#else
    return 31 - __builtin_clz(v);
#endif
}

// ---- FSE decoding table entry (sequence flavour: carries the code's base value and extra-bit count) ----
// One 32-bit word per cell: the state chain needs next_base / nb_bits / nb_extra only; the code's base value is looked
// up from `sym` by whoever cuts the extra bits out of the stream (ll_base / ml_base / 1 << ofCode).
struct FseDEntry {              // field order is the bit layout (LSB first) the decoder's state chain relies on:
    uint32_t nb_bits : 6;       //   the sum of three cells' words carries sum(nb_bits) in bits 0..5 (<= 27) and
    uint32_t nb_extra : 6;      //   sum(nb_extra) in bits 6..11 (<= 63); next_base needs no mask (word >> 18)
    uint32_t sym : 6;           // the code itself; nb_extra = additional bits of the code (LL_bits / ML_bits / offset code)
    uint32_t next_base : 10;    // new state = next_base + read(nb_bits)
    uint32_t pad : 4;
};
static_assert(sizeof(FseDEntry) == 4, "FSE decoding cell is one word");

// Spread + state assignment of RFC 8878 §4.1.1 (same procedure libzstd's FSE_buildDTable follows).
// symbol_of[] is scratch of table_size bytes; next[] scratch of nsym uint16.
__host__ __device__ inline void fse_spread(const int16_t* norm, int nsym, int log, uint8_t* symbol_of, uint16_t* next) {
    const uint32_t size = 1u << log, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    uint32_t high = size - 1;
    for (int s = 0; s < nsym; s++) {
        if (norm[s] == -1) { symbol_of[high--] = (uint8_t)s; next[s] = 1; }
        else next[s] = (uint16_t)norm[s];
    }
    uint32_t pos = 0;
    for (int s = 0; s < nsym; s++) {
        for (int i = 0; i < norm[s]; i++) {
            symbol_of[pos] = (uint8_t)s;
            pos = (pos + step) & mask;
            while (pos > high) pos = (pos + step) & mask;
        }
    }
}

// kind: 0 = literal lengths, 1 = offsets, 2 = match lengths (selects base / extra-bit tables)
__host__ __device__ inline void fse_build_dtable(const int16_t* norm, int nsym, int log, int kind, const SeqTables& st,
                                                 FseDEntry* table, uint8_t* symbol_of, uint16_t* next) {
    fse_spread(norm, nsym, log, symbol_of, next);
    const uint32_t size = 1u << log;
    for (uint32_t u = 0; u < size; u++) {
        const int s = symbol_of[u];
        const uint32_t ns = next[s]++;
        const int nb = log - highbit32(ns);
        FseDEntry e{};
        e.nb_bits = (uint32_t)nb;
        e.next_base = (ns << nb) - size;
        e.sym = (uint32_t)s;
        e.nb_extra = kind == 0 ? st.ll_bits[s] : kind == 2 ? st.ml_bits[s] : (uint32_t)s;
        table[u] = e;
    }
}
// RLE mode: a single-entry table
__host__ __device__ inline void fse_build_rle(int sym, int kind, const SeqTables& st, FseDEntry* table) {
    FseDEntry e{};
    e.sym = (uint32_t)sym;
    e.nb_extra = kind == 0 ? st.ll_bits[sym] : kind == 2 ? st.ml_bits[sym] : (uint32_t)sym;
    table[0] = e;
}

// ---- FSE encoding table (libzstd's FSE_buildCTable layout: state table + per-symbol transform) ----
struct FseCSym { int32_t delta_nb_bits; int32_t delta_find_state; };
template <int LOG, int NSYM> struct FseCTable {
    uint16_t state[1 << LOG];
    FseCSym sym[NSYM];
};
template <int LOG, int NSYM>
constexpr FseCTable<LOG, NSYM> make_fse_ctable(const int16_t* norm, int nsym_used) {
    FseCTable<LOG, NSYM> ct{};
    constexpr uint32_t size = 1u << LOG, mask = size - 1, step = (size >> 1) + (size >> 3) + 3;
    uint8_t symbol_of[size] = {};
    uint32_t cumul[NSYM + 2] = {};
    uint32_t high = size - 1;
    for (int u = 1; u <= nsym_used; u++) {
        if (norm[u - 1] == -1) { cumul[u] = cumul[u - 1] + 1; symbol_of[high--] = (uint8_t)(u - 1); }
        else cumul[u] = cumul[u - 1] + (uint32_t)norm[u - 1];
    }
    cumul[nsym_used + 1] = size + 1;
    uint32_t pos = 0;
    for (int s = 0; s < nsym_used; s++) {
        for (int i = 0; i < norm[s]; i++) {
            symbol_of[pos] = (uint8_t)s;
            pos = (pos + step) & mask;
            while (pos > high) pos = (pos + step) & mask;
        }
    }
    for (uint32_t u = 0; u < size; u++) { uint8_t s = symbol_of[u]; ct.state[cumul[s]++] = (uint16_t)(size + u); }
    int total = 0;
    for (int s = 0; s < NSYM; s++) {
        int n = s < nsym_used ? norm[s] : 0;
        if (n == 0) { ct.sym[s].delta_nb_bits = ((LOG + 1) << 16) - (1 << LOG); ct.sym[s].delta_find_state = 0; }
        else if (n == -1 || n == 1) { ct.sym[s].delta_nb_bits = (LOG << 16) - (1 << LOG); ct.sym[s].delta_find_state = total - 1; total++; }
        else {
            int hb = 0; for (uint32_t v = (uint32_t)(n - 1); v > 1; v >>= 1) hb++;       // highbit32(n-1), n >= 2
            if (n - 1 == 0) hb = 0;
            int max_bits_out = LOG - hb;
            int min_state_plus = n << max_bits_out;
            ct.sym[s].delta_nb_bits = (max_bits_out << 16) - min_state_plus;
            ct.sym[s].delta_find_state = total - n;
            total += n;
        }
    }
    return ct;
}

struct PredefinedCTables {
    FseCTable<LL_DEFAULT_LOG, LL_NSYM> ll;
    FseCTable<OF_DEFAULT_LOG, OF_NSYM> of;
    FseCTable<ML_DEFAULT_LOG, ML_NSYM> ml;
};
constexpr PredefinedCTables make_predefined_ctables() {
    PredefinedCTables p{};
    SeqTables st = make_seq_tables();
    p.ll = make_fse_ctable<LL_DEFAULT_LOG, LL_NSYM>(st.ll_norm, 36);
    p.of = make_fse_ctable<OF_DEFAULT_LOG, OF_NSYM>(st.of_norm, 29);
    p.ml = make_fse_ctable<ML_DEFAULT_LOG, ML_NSYM>(st.ml_norm, 53);
    return p;
}

}  // namespace zf
}  // namespace ts
