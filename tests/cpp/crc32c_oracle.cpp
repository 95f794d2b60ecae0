// CPU oracle of the upload-part checksums (tests/part_crc_util.py): the CRC-32C restatement of host/segment_upload.hpp
// (tieredstorage::detail::crcTableEntry, bit-reflected Castagnoli, init and xorout 0xFFFFFFFF), one byte at a time, applied to
// every part of an object and to the whole object separately.  Shares no code with the library's GF(2) combination.
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_upload.hpp"

namespace {
uint32_t table[256];
bool ready = false;
uint32_t crc(const uint8_t* p, uint64_t n) {
    if (!ready) { for (uint32_t i = 0; i < 256; i++) table[i] = tieredstorage::detail::crcTableEntry(i, 0x82F63B78u); ready = true; }
    uint32_t c = 0xffffffffu;
    for (uint64_t i = 0; i < n; i++) c = table[(c ^ p[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
}  // namespace

extern "C" uint32_t pc_crc32c(const uint8_t* p, uint64_t n) { return crc(p, n); }
// out[k] = CRC-32C of bytes [k * part, min((k + 1) * part, n)); returns the number of parts
extern "C" uint64_t pc_parts(const uint8_t* p, uint64_t n, uint64_t part, uint32_t* out) {
    uint64_t k = 0;
    for (uint64_t off = 0; off < n; off += part) out[k++] = crc(p + off, std::min(part, n - off));
    return k;
}
