// host_index.hpp — host-side ChunkIndex plumbing of libtsgpu (integer-only, a few hundred bytes per segment).
// Mirrors, under the same names, the reference's
//   ChunkSizesBinaryCodec            core/M/manifest/index/serde/ChunkSizesBinaryCodec.java:104-202
//   TransformedChunksSerializer      core/M/manifest/index/serde/TransformedChunksSerializer.java:30-52
//   Fixed/VariableSizeChunkIndex JSON core/M/manifest/index/{FixedSizeChunkIndex,VariableSizeChunkIndex}.java,
//                                    type tag core/M/manifest/index/ChunkIndex.java:36-42
// (core/M = <reference>/core/src/main/java/io/aiven/kafka/tieredstorage).
#pragma once
#include <stdint.h>
#include <string>
#include <vector>

namespace tshost {

struct Error { int code; std::string msg; };
#define TSH_FAIL(c, m) do { err.code = (c); err.msg = (m); return false; } while (0)

// ------------------------------------------------------------------ ChunkSizesBinaryCodec
struct ChunkSizesBinaryCodec {
    static int bytesNeeded(int32_t v) { return v <= 0xFF ? 1 : v <= 0xFFFF ? 2 : v <= 0xFFFFFF ? 3 : 4; }
    static void putInt(std::vector<uint8_t>& b, uint32_t v) {
        b.push_back((uint8_t)(v >> 24)); b.push_back((uint8_t)(v >> 16)); b.push_back((uint8_t)(v >> 8)); b.push_back((uint8_t)v);
    }
    static uint32_t getInt(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }

    static bool encode(const int32_t* values, uint32_t count, std::vector<uint8_t>& out, Error& err) {
        out.clear();
        if (count == 0) { putInt(out, 0); return true; }
        const int32_t lastValue = values[count - 1];
        if (count == 1) {
            if (lastValue < 0) TSH_FAIL(-1, "Values cannot be negative");
            putInt(out, 1); putInt(out, (uint32_t)lastValue); return true;
        }
        int32_t min = values[0];
        for (uint32_t i = 1; i + 1 < count; i++) if (values[i] < min) min = values[i];
        if (min < 0 || lastValue < 0) TSH_FAIL(-1, "Values cannot be negative");
        int bytesPerValue = 1;
        for (uint32_t i = 0; i + 1 < count; i++) { int b = bytesNeeded(values[i] - min); if (b > bytesPerValue) bytesPerValue = b; }
        putInt(out, count); putInt(out, (uint32_t)min); out.push_back((uint8_t)bytesPerValue);
        for (uint32_t i = 0; i + 1 < count; i++) {
            uint32_t onBase = (uint32_t)(values[i] - min);
            for (int k = bytesPerValue - 1; k >= 0; k--) out.push_back((uint8_t)(onBase >> (8 * k)));
        }
        putInt(out, (uint32_t)lastValue);
        return true;
    }
    static bool decode(const uint8_t* in, size_t n, std::vector<int32_t>& out, Error& err) {
        out.clear();
        if (n < 4) TSH_FAIL(-4, "BufferUnderflowException");
        int32_t count = (int32_t)getInt(in);
        if (count == 0) return true;
        if (count < 0) TSH_FAIL(-4, "negative count");
        if (count == 1) { if (n < 8) TSH_FAIL(-4, "BufferUnderflowException"); out.push_back((int32_t)getInt(in + 4)); return true; }
        if (n < 9) TSH_FAIL(-4, "BufferUnderflowException");
        int32_t base = (int32_t)getInt(in + 4);
        int bpv = in[8];
        if (bpv < 1 || bpv > 4 || n < 9 + (size_t)(count - 1) * bpv + 4) TSH_FAIL(-4, "BufferUnderflowException");
        const uint8_t* p = in + 9;
        for (int32_t i = 0; i + 1 < count; i++) {
            uint32_t x = 0;
            for (int k = 0; k < bpv; k++) x = x << 8 | *p++;
            out.push_back((int32_t)x + base);
        }
        out.push_back((int32_t)getInt(p));
        return true;
    }
};

// ------------------------------------------------------------------ java.util.Base64 (basic alphabet, padded)
inline std::string base64Encode(const uint8_t* in, size_t n) {
    static const char A[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string o;
    for (size_t i = 0; i < n; i += 3) {
        uint32_t v = (uint32_t)in[i] << 16 | (i + 1 < n ? (uint32_t)in[i + 1] << 8 : 0) | (i + 2 < n ? in[i + 2] : 0);
        o += A[v >> 18]; o += A[(v >> 12) & 63];
        o += i + 1 < n ? A[(v >> 6) & 63] : '=';
        o += i + 2 < n ? A[v & 63] : '=';
    }
    return o;
}
inline bool base64Decode(const char* s, std::vector<uint8_t>& out, Error& err) {
    out.clear();
    uint32_t acc = 0; int bits = 0;
    for (; *s && *s != '='; s++) {
        int c = *s, v;
        if (c >= 'A' && c <= 'Z') v = c - 'A'; else if (c >= 'a' && c <= 'z') v = c - 'a' + 26;
        else if (c >= '0' && c <= '9') v = c - '0' + 52; else if (c == '+') v = 62; else if (c == '/') v = 63;
        else TSH_FAIL(-4, "Illegal base64 character");
        acc = acc << 6 | (uint32_t)v; bits += 6;
        if (bits >= 8) { bits -= 8; out.push_back((uint8_t)(acc >> bits)); }
    }
    return true;
}

// ------------------------------------------------------------------ zstd frame header (RFC 8878 §3.1.1), as libzstd sizes it
// Header choice mirrors what libzstd emits for a pledged source size at level 3 (windowLog 21):
// Single_Segment with the smallest Frame_Content_Size field while the content fits the window, otherwise
// FHD 0x80 + Window_Descriptor 0x58 (2 MiB) + 4-byte FCS.  (Golden vector ENCODED_CHUNKS: 28 B5 2F FD 20 0F.)
inline size_t zstdFrameHeader(uint8_t* out, uint64_t contentSize) {
    size_t p = 0;
    out[p++] = 0x28; out[p++] = 0xB5; out[p++] = 0x2F; out[p++] = 0xFD;
    const uint64_t windowSize = 1ull << 21;
    if (contentSize <= windowSize) {
        if (contentSize < 256) { out[p++] = 0x20; out[p++] = (uint8_t)contentSize; }
        else if (contentSize < 65536 + 256) { out[p++] = 0x60; uint32_t v = (uint32_t)contentSize - 256; out[p++] = (uint8_t)v; out[p++] = (uint8_t)(v >> 8); }
        else { out[p++] = 0xA0; for (int k = 0; k < 4; k++) out[p++] = (uint8_t)(contentSize >> (8 * k)); }
    } else {
        out[p++] = 0x80; out[p++] = 0x58;
        for (int k = 0; k < 4; k++) out[p++] = (uint8_t)(contentSize >> (8 * k));
    }
    return p;
}

}  // namespace tshost
