// Host mirror of tsgpu_check_object (RemoteSegmentChecker): segments uploaded by SegmentLogUploader (plain, compressed,
// encrypted, both) are checked from their manifest JSON through a ranged-GET fetcher in windows of 1, 3 and 64 chunks; the CRCs
// equal the host restatement tieredstorage::crc32c of the object and of the segment.  A flipped object byte throws
// std::runtime_error, a bad record batch InvalidRecordBatchException, each with the library's message.  Links the test-only SIMT
// build.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_check.hpp"

using namespace tieredstorage;
static int checks = 0, failures = 0;
#define CHECK(c) do { checks++; if (!(c)) { failures++; printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); } } while (0)

static void be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
// A segment of valid v2 record batches with text payloads.
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

int main() {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(17);
    Bytes seg = segment(60000, rng);
    const int cs = 8192;
    const int nch = (int)((seg.size() + cs - 1) / cs);
    DataKeyAndAAD km; km.dataKey.resize(32); km.aad.resize(32);
    for (auto& b : km.dataKey) b = (uint8_t)rng();
    for (auto& b : km.aad) b = (uint8_t)rng();
    Bytes ivs(12 * nch); for (auto& b : ivs) b = (uint8_t)rng();
    Bytes bad = seg;
    bad[seg.size() / 2 + 5] ^= 1;                                       // inside some batch: its CRC no longer matches
    for (int compress = 0; compress < 2; compress++) for (int enc = 0; enc < 2; enc++) for (int damaged = 0; damaged < 2; damaged++) {
        const Bytes& s = damaged ? bad : seg;
        SegmentLogUploader up(ctx, cs, compress != 0, /*heuristic=*/false, enc != 0, 1 << 20);
        Bytes object;
        auto res = up.upload(s.data(), s.size(), enc ? &km : nullptr, enc ? ivs.data() : nullptr,
                             [&](const UploadPart& p, const uint8_t* d) { object.insert(object.end(), d, d + p.size); });
        const std::string json = segmentManifestV1Json(*res.chunkIndex, SegmentIndexesV1{}, res.compressed, std::nullopt,
                                                       enc ? &km.aad : nullptr, RemoteLogSegmentMetadataJson{});
        const SegmentManifestV1 manifest = parseSegmentManifestV1(json, ctx);
        int gets = 0;
        auto fetch = [&](const BytesRange& r) { gets++; return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };
        for (uint32_t window : {1u, 3u, 64u}) {
            RemoteSegmentChecker checker(ctx, window);
            gets = 0;
            const ObjectCheck got = checker.check(manifest, fetch, enc ? &km : nullptr);
            CHECK(got.objectCrc32c == crc32c(object.data(), object.size()));
            CHECK(got.segmentCrc32c == crc32c(s.data(), s.size()));
            CHECK(gets == (nch + (int)window - 1) / (int)window);
            checker.validateRecords = true;
            bool threw = false;
            try { checker.check(manifest, fetch, enc ? &km : nullptr); }
            catch (const InvalidRecordBatchException& e) { threw = strstr(e.what(), "(check: crc)") != nullptr; }
            CHECK(threw == (damaged != 0));
        }
        if (compress || enc) {
            Bytes flipped = object;
            flipped[flipped.size() / 3] ^= 0x10;
            auto fetchFlipped = [&](const BytesRange& r) { return Bytes(flipped.begin() + r.from, flipped.begin() + r.to + 1); };
            bool threw = false;
            try { RemoteSegmentChecker(ctx, 2).check(manifest, fetchFlipped, enc ? &km : nullptr); }
            catch (const InvalidRecordBatchException&) {}
            catch (const std::runtime_error& e) { threw = strstr(e.what(), "chunk") != nullptr; }
            CHECK(threw || !enc);                                       // zstd alone may still decode a flipped literal
        }
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
