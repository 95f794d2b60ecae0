// Host mirror with CRC-64/NVME: SegmentLogUploader::crc64Parts hands every part to the sink with the CRC-64/NVME of exactly its
// bytes (and no CRC-32C), the upload carries the object's, and the object is byte for byte the one partChecksums alone gives;
// RemoteSegmentChecker::check64 gives the CRC-64/NVME of the object and of the segment in windows of 1, 3 and 64 chunks; and
// RemoteSegmentRewriter::crc64 hands every new part over with its CRC-64/NVME and returns the 64-bit source, object and segment
// words.  Compressed and encrypted segments, several part sizes.  The reference CRC is a bitwise restatement of the catalogue
// definition here.  Links the test-only SIMT build.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_check.hpp"
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_rewrite.hpp"

using namespace tieredstorage;
static int checks = 0, failures = 0;
#define CHECK(c) do { checks++; if (!(c)) { failures++; printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); } } while (0)

static uint64_t crc64nvme(const uint8_t* p, size_t n) {
    uint64_t c = ~0ull;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x9A6C9329AC4BC9B5ull & (0ull - (c & 1))); }
    return ~c;
}
static void be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
static Bytes segment(size_t target, std::mt19937& rng) {      // valid v2 record batches with text payloads
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

int main() {
    CHECK(crc64nvme((const uint8_t*)"123456789", 9) == 0xAE8B14860A799888ull);
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(29);
    const Bytes seg = segment(60000, rng);
    const int cs = 8192;
    const int nch = (int)((seg.size() + cs - 1) / cs);
    DataKeyAndAAD km; km.dataKey.resize(32); km.aad.resize(32);
    for (auto& b : km.dataKey) b = (uint8_t)rng();
    for (auto& b : km.aad) b = (uint8_t)rng();
    Bytes ivs(12 * nch); for (auto& b : ivs) b = (uint8_t)rng();
    for (int compress = 0; compress < 2; compress++) for (int enc = 0; enc < 2; enc++) for (uint64_t part : {1000ull, 8220ull, 1ull << 30}) {
        if (!compress && !enc) continue;                              // a plain copy: no byte reaches the GPU
        // 1. upload with CRC-64/NVME parts, and the same upload with CRC-32C parts
        SegmentLogUploader up(ctx, cs, compress != 0, /*heuristic=*/false, enc != 0, part);
        up.partChecksums = true; up.crc64Parts = true; up.validateRecords = true;
        Bytes object, object32;
        bool ok = true;
        auto res = up.upload(seg.data(), seg.size(), enc ? &km : nullptr, enc ? ivs.data() : nullptr, [&](const UploadPart& p, const uint8_t* d) {
            ok = ok && !p.crc32c && p.crc64nvme && *p.crc64nvme == crc64nvme(d, p.size) && p.size <= part && p.offset == object.size();
            object.insert(object.end(), d, d + p.size);
        });
        CHECK(ok && object.size() == res.objectBytes && !res.objectCrc32c);
        CHECK(res.objectCrc64nvme && *res.objectCrc64nvme == crc64nvme(object.data(), object.size()));
        if (!compress) {                                              // the deterministic writer: the bytes of the CRC-32C upload
            up.crc64Parts = false;
            auto r32 = up.upload(seg.data(), seg.size(), enc ? &km : nullptr, enc ? ivs.data() : nullptr,
                                 [&](const UploadPart& p, const uint8_t* d) { object32.insert(object32.end(), d, d + p.size); });
            CHECK(object32 == object && r32.objectCrc32c && !r32.objectCrc64nvme);
        }
        // 2. the check, with 64-bit words
        const SegmentManifestV1 manifest = parseSegmentManifestV1(
            segmentManifestV1Json(*res.chunkIndex, SegmentIndexesV1{}, res.compressed, std::nullopt, enc ? &km.aad : nullptr,
                                  RemoteLogSegmentMetadataJson{}), ctx);
        auto fetch = [&](const BytesRange& r) { return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };
        for (uint32_t window : {1u, 3u, 64u}) {
            RemoteSegmentChecker checker(ctx, window);
            checker.validateRecords = true;
            const ObjectCheck64 got = checker.check64(manifest, fetch, enc ? &km : nullptr);
            CHECK(got.objectCrc64nvme == crc64nvme(object.data(), object.size()));
            CHECK(got.segmentCrc64nvme == crc64nvme(seg.data(), seg.size()));
        }
        // 3. the rewrite to Zstd+AES under a new key, with 64-bit words
        if (part != 8220) continue;
        DataKeyAndAAD nk; nk.dataKey.resize(32); nk.aad.resize(32);
        for (auto& b : nk.dataKey) b = (uint8_t)rng();
        for (auto& b : nk.aad) b = (uint8_t)rng();
        Bytes nivs(12 * nch), indexIvs(12 * 5);
        for (auto& b : nivs) b = (uint8_t)rng();
        for (auto& b : indexIvs) b = (uint8_t)rng();
        RemoteSegmentRewriter rw(ctx, true, true, 5000, 3);
        rw.crc64 = true;
        Bytes neo;
        bool parts = true;
        const SegmentRewrite got = rw.rewrite(manifest, fetch, Bytes(), enc ? &km : nullptr, &nk, nivs.data(), indexIvs.data(),
            [&](const UploadPart& p, const uint8_t* d) {
                parts = parts && !p.crc32c && p.crc64nvme && *p.crc64nvme == crc64nvme(d, p.size) && p.offset == neo.size();
                neo.insert(neo.end(), d, d + p.size);
            });
        CHECK(parts && neo.size() == got.objectBytes);
        CHECK(got.sourceCrc64nvme == crc64nvme(object.data(), object.size()));
        CHECK(got.objectCrc64nvme == crc64nvme(neo.data(), neo.size()));
        CHECK(got.segmentCrc64nvme == crc64nvme(seg.data(), seg.size()));
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
