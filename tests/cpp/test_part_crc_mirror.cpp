// Host mirror with part checksums (SegmentLogUploader::partChecksums, tsgpu_transform_parts): every UploadPart handed to the
// sink carries the CRC-32C of exactly its bytes, the upload carries the object's, both equal the host restatement
// tieredstorage::crc32c; without the switch no part carries one.  Compressed and encrypted segments, several part sizes, with
// and without record validation.  Links the test-only SIMT build (`--device`) or the product library.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_upload.hpp"

using namespace tieredstorage;
static int checks = 0, failures = 0;
#define CHECK(c) do { checks++; if (!(c)) { failures++; printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); } } while (0)

static void be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
// A segment of valid v2 record batches (uncompressed attribute bits) with text payloads.
static Bytes segment(size_t target, std::mt19937& rng) {
    Bytes s;
    for (int i = 0; s.size() < target; i++) {
        const uint32_t len = 61 + rng() % 3000;
        Bytes e(len);
        for (uint32_t j = 21; j < len; j++) e[j] = (uint8_t)"topic-partition-offset "[(j + i) % 23];
        be32(e.data() + 4, (uint32_t)i); be32(e.data() + 8, len - 12);
        e[16] = 2; e[21] = 0; e[22] = 0;
        be32(e.data() + 17, crc32c(e.data() + 21, len - 21));
        s.insert(s.end(), e.begin(), e.end());
    }
    return s;
}

int main(int argc, char** argv) {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(11);
    const Bytes seg = segment(70000, rng);
    const int cs = 8192;
    const int nch = (int)((seg.size() + cs - 1) / cs);
    DataKeyAndAAD km; km.dataKey.resize(32); km.aad.resize(32);
    for (auto& b : km.dataKey) b = (uint8_t)rng();
    for (auto& b : km.aad) b = (uint8_t)rng();
    Bytes ivs(12 * nch); for (auto& b : ivs) b = (uint8_t)rng();
    for (int compress = 0; compress < 2; compress++) for (int enc = 0; enc < 2; enc++) for (uint64_t part : {1000ull, 8220ull, 16384ull, 1ull << 30})
    for (int validate = 0; validate < 2; validate++) for (int on = 0; on < 2; on++) {
        if (!compress && !enc && on) continue;                    // a plain copy: no byte reaches the GPU
        SegmentLogUploader up(ctx, cs, compress != 0, /*heuristic=*/false, enc != 0, part);
        up.validateRecords = validate != 0;
        up.partChecksums = on != 0;
        Bytes object; bool crcs = true, any = false;
        auto res = up.upload(seg.data(), seg.size(), enc ? &km : nullptr, enc ? ivs.data() : nullptr, [&](const UploadPart& p, const uint8_t* d) {
            any = any || p.crc32c.has_value();
            if (on) crcs = crcs && p.crc32c && *p.crc32c == crc32c(d, p.size) && p.size <= part && p.offset == object.size();
            object.insert(object.end(), d, d + p.size);
        });
        CHECK(object.size() == res.objectBytes);
        if (on) {
            CHECK(crcs && any);
            CHECK(res.objectCrc32c && *res.objectCrc32c == crc32c(object.data(), object.size()));
        } else {
            CHECK(!any && !res.objectCrc32c);
        }
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
