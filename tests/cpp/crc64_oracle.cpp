// CPU oracle of the CRC-64/NVME checksums (tests/crc64_util.py): the catalogue definition -- reflected polynomial
// 0x9A6C9329AC4BC9B5, init and xorout all ones -- one byte at a time from a table built bit by bit here, applied to every part of
// an object and to the whole object separately.  Shares no code with the library's slice-by-8 kernels or GF(2) combination.
#include <algorithm>
#include <cstdint>

namespace {
uint64_t table[256];
bool ready = false;
uint64_t crc(const uint8_t* p, uint64_t n) {
    if (!ready) {
        for (uint32_t i = 0; i < 256; i++) {
            uint64_t c = i;
            for (int k = 0; k < 8; k++) c = (c & 1) ? (c >> 1) ^ 0x9A6C9329AC4BC9B5ull : c >> 1;
            table[i] = c;
        }
        ready = true;
    }
    uint64_t c = ~0ull;
    for (uint64_t i = 0; i < n; i++) c = table[(c ^ p[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
}  // namespace

extern "C" uint64_t pc_crc64nvme(const uint8_t* p, uint64_t n) { return crc(p, n); }
// out[k] = CRC-64/NVME of bytes [k * part, min((k + 1) * part, n)); returns the number of parts
extern "C" uint64_t pc_parts64(const uint8_t* p, uint64_t n, uint64_t part, uint64_t* out) {
    uint64_t k = 0;
    for (uint64_t off = 0; off < n; off += part) out[k++] = crc(p + off, std::min(part, n - off));
    return k;
}
