// TEST-ONLY CPU oracle of TSGPU_FLAG_VALIDATE_RECORDS (tests/records_util.py loads it): the restatement of the Kafka log
// format in host/segment_upload.hpp (its CRC-32C / CRC-32 definitions), extended from the first batch to every entry.
//   rec_walk  the first invalid entry of a segment, walked entry by entry in the order the checks are made:
//             fewer than 17 bytes left -> length; magic not 0/1/2 -> magic; size below 49 (v2) / 14 (v0/1) -> length;
//             entry past the end -> length; stored CRC != computed CRC -> crc.
//   rec_seal  writes the right CRC into every entry of a generated segment (sizes and magics are trusted).
//   rec_starts  the start of every entry of a valid segment.
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_upload.hpp"

namespace {
struct Tables {
    uint32_t t[2][256];
    Tables() {
        for (uint32_t i = 0; i < 256; i++) {
            t[0][i] = tieredstorage::detail::crcTableEntry(i, 0x82F63B78u);     // the restatement's polynomials
            t[1][i] = tieredstorage::detail::crcTableEntry(i, 0xEDB88320u);
        }
    }
};
const Tables g_tab;
uint32_t crc(int pi, const uint8_t* p, uint64_t n) {          // tieredstorage::crc32c / crc32, with the table built once
    uint32_t c = 0xffffffffu;
    for (uint64_t i = 0; i < n; i++) c = g_tab.t[pi][(c ^ p[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
}  // namespace

extern "C" int64_t rec_walk(const uint8_t* p, uint64_t n, int* kind, uint32_t* stored, uint32_t* computed) {
    using tieredstorage::detail::be32;
    uint64_t x = 0;
    *kind = 0;
    while (x < n) {
        if (n - x < 17) { *kind = 1; return (int64_t)x; }
        const uint8_t m = p[x + 16];
        if (m > 2) { *kind = 2; return (int64_t)x; }
        const int32_t size = (int32_t)be32(p + x + 8);
        if (size < (m == 2 ? 49 : 14) || x + 12 + (uint64_t)size > n) { *kind = 1; return (int64_t)x; }
        const uint64_t from = m == 2 ? 21 : 16, len = 12 + (uint64_t)size;
        *stored = be32(p + x + (m == 2 ? 17 : 12));
        *computed = crc(m == 2 ? 0 : 1, p + x + from, len - from);
        if (*stored != *computed) { *kind = 3; return (int64_t)x; }
        x += len;
    }
    return -1;
}

extern "C" void rec_seal(uint8_t* p, uint64_t n) {
    uint64_t x = 0;
    while (x + 21 <= n) {
        const uint8_t m = p[x + 16];
        const uint64_t len = 12 + (uint64_t)tieredstorage::detail::be32(p + x + 8), from = m == 2 ? 21 : 16;
        if (x + len > n) return;
        const uint32_t c = crc(m == 2 ? 0 : 1, p + x + from, len - from);
        uint8_t* at = p + x + (m == 2 ? 17 : 12);
        at[0] = (uint8_t)(c >> 24); at[1] = (uint8_t)(c >> 16); at[2] = (uint8_t)(c >> 8); at[3] = (uint8_t)c;
        x += len;
    }
}

extern "C" uint64_t rec_starts(const uint8_t* p, uint64_t n, uint64_t* out, uint64_t cap) {
    uint64_t x = 0, k = 0;
    while (x + 12 <= n) {
        if (k < cap) out[k] = x;
        k++;
        x += 12 + (uint64_t)tieredstorage::detail::be32(p + x + 8);
    }
    return k;
}
