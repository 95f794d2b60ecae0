// Host mirror of tsgpu_rewrite_object (RemoteSegmentRewriter): a segment and its indexes uploaded with compression and
// encryption off (SegmentLogUploader, uploadIndexes) are rewritten to Zstd+AES under a new key in windows of 1, 3 and 64 chunks,
// with and without record validation and VERIFY; the new manifest is written and parsed again.  FetchChunkEnumeration over a
// grid of ranges returns the segment's bytes with the new key, fetchIndexBytes returns the index blobs, and the old key fails
// on both; the parts reach the sink in order with the CRC-32C of their bytes, and the three CRCs equal the host restatement
// tieredstorage::crc32c.  A second rewrite, Zstd+AES to Zstd+AES under another key, keeps the frames.  Links the test-only SIMT
// build.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_rewrite.hpp"

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
static DataKeyAndAAD keyMaterial(std::mt19937& rng) {
    DataKeyAndAAD km; km.dataKey.resize(32); km.aad.resize(32);
    for (auto& b : km.dataKey) b = (uint8_t)rng();
    for (auto& b : km.aad) b = (uint8_t)rng();
    return km;
}
static Bytes random(size_t n, std::mt19937& rng) { Bytes b(n); for (auto& x : b) x = (uint8_t)rng(); return b; }

int main() {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(23);
    const Bytes seg = segment(60000, rng);
    const int cs = 8192;
    const int nch = (int)((seg.size() + cs - 1) / cs);
    const std::vector<std::pair<IndexType, Bytes>> blobs{
        {IndexType::OFFSET, random(800, rng)}, {IndexType::TIMESTAMP, random(1200, rng)}, {IndexType::PRODUCER_SNAPSHOT, Bytes()},
        {IndexType::LEADER_EPOCH, random(40, rng)}, {IndexType::TRANSACTION, random(100, rng)}};

    // 1. upload, compression and encryption off
    SegmentLogUploader up(ctx, cs, false, false, false, 1 << 20);
    Bytes object;
    auto res = up.upload(seg.data(), seg.size(), nullptr, nullptr,
                         [&](const UploadPart& p, const uint8_t* d) { object.insert(object.end(), d, d + p.size); });
    const SegmentIndexesUpload ix = uploadIndexes(ctx, blobs, false, nullptr, nullptr);
    const SegmentManifestV1 manifest = parseSegmentManifestV1(
        segmentManifestV1Json(*res.chunkIndex, ix.segmentIndexes, false, std::nullopt, nullptr, RemoteLogSegmentMetadataJson{}), ctx);
    auto fetchOld = [&](const BytesRange& r) { return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };

    const DataKeyAndAAD oldKey = keyMaterial(rng), newKey = keyMaterial(rng);
    const Bytes ivs = random(12 * nch, rng), indexIvs = random(12 * 5, rng);
    for (uint32_t window : {1u, 3u, 64u}) for (int flags = 0; flags < 2; flags++) {
        // 2. rewrite to Zstd+AES under a new key
        const uint64_t partSize = 5000;
        RemoteSegmentRewriter rw(ctx, true, true, partSize, window);
        rw.validateRecords = flags != 0; rw.verify = flags != 0;
        Bytes neo;
        bool inOrder = true, crcsMatch = true;
        const SegmentRewrite got = rw.rewrite(manifest, fetchOld, ix.object, nullptr, &newKey, ivs.data(), indexIvs.data(),
            [&](const UploadPart& p, const uint8_t* d) {
                inOrder &= p.offset == neo.size() && p.partNumber == (int)(neo.size() / partSize) + 1;
                crcsMatch &= p.crc32c && *p.crc32c == crc32c(d, p.size);
                neo.insert(neo.end(), d, d + p.size);
            });
        CHECK(inOrder && crcsMatch && neo.size() == got.objectBytes);
        CHECK(got.sourceCrc32c == crc32c(object.data(), object.size()));
        CHECK(got.objectCrc32c == crc32c(neo.data(), neo.size()));
        CHECK(got.segmentCrc32c == crc32c(seg.data(), seg.size()));
        // 3. the new manifest, written and parsed again
        const SegmentManifestV1 m2 = parseSegmentManifestV1(
            segmentManifestV1Json(*got.chunkIndex, got.segmentIndexes, true, std::string("key-2:AAAA"), &newKey.aad,
                                  RemoteLogSegmentMetadataJson{}), ctx);
        CHECK(m2.compression && m2.aad && *m2.aad == newKey.aad && m2.chunkIndex->chunks().size() == (size_t)nch);
        auto fetchNew = [&](const BytesRange& r) { return Bytes(neo.begin() + r.from, neo.begin() + r.to + 1); };
        const int n = (int)seg.size();
        for (int from : {0, 1, cs - 1, cs, 3 * cs + 17, n - 1}) for (int len : {1, 100, cs, 3 * cs + 5, n}) {
            const int to = std::min(n - 1, from + len - 1);
            FetchChunkEnumeration fe(ctx, *m2.chunkIndex, BytesRange::of(from, to), fetchNew, true, &newKey, 4);
            const Bytes b = fe.readAll();
            CHECK(b == Bytes(seg.begin() + from, seg.begin() + to + 1));
        }
        for (const auto& bl : blobs) {
            const SegmentIndexesV1& si = m2.segmentIndexes;
            const SegmentIndexV1 idx[5] = {si.offset, si.timestamp, si.producerSnapshot, si.leaderEpoch,
                                           si.transaction ? *si.transaction : SegmentIndexV1{0, 0}};
            CHECK(fetchIndexBytes(ctx, got.indexesObject, idx[(int)bl.first], &newKey) == bl.second);
        }
        // the old key fails on both objects
        bool threw = false;
        try { FetchChunkEnumeration(ctx, *m2.chunkIndex, BytesRange::of(0, n - 1), fetchNew, true, &oldKey, 4).readAll(); }
        catch (const std::runtime_error&) { threw = true; }
        CHECK(threw);
        threw = false;
        try { fetchIndexBytes(ctx, got.indexesObject, m2.segmentIndexes.offset, &oldKey); }
        catch (const std::runtime_error&) { threw = true; }
        CHECK(threw);

        // Zstd+AES to Zstd+AES under another key: the frames are kept, the IVs must be new
        if (window == 3 && flags == 0) {
            const DataKeyAndAAD key3 = keyMaterial(rng);
            const Bytes ivs3 = random(12 * nch, rng), indexIvs3 = random(12 * 5, rng);
            Bytes third;
            const SegmentRewrite r3 = RemoteSegmentRewriter(ctx, true, true, 1 << 30, 2).rewrite(
                m2, fetchNew, got.indexesObject, &newKey, &key3, ivs3.data(), indexIvs3.data(),
                [&](const UploadPart&, const uint8_t* d) { (void)d; });
            CHECK(r3.segmentCrc32c == got.segmentCrc32c && r3.sourceCrc32c == got.objectCrc32c && r3.objectBytes == got.objectBytes);
            bool refused = false;                                       // the same key with the old object's IVs
            try { RemoteSegmentRewriter(ctx, true, true, 1 << 30, 2).rewrite(m2, fetchNew, got.indexesObject, &newKey, &newKey,
                                                                             ivs.data(), indexIvs3.data(), [](const UploadPart&, const uint8_t*) {}); }
            catch (const IllegalArgumentException& e) { refused = strstr(e.what(), "repeats the IV") != nullptr; }
            CHECK(refused);
        }
    }
    // a damaged old object fails with the library's message
    Bytes bad = object;
    bad[seg.size() / 2 + 5] ^= 1;
    auto fetchBad = [&](const BytesRange& r) { return Bytes(bad.begin() + r.from, bad.begin() + r.to + 1); };
    RemoteSegmentRewriter rw(ctx, true, true, 1 << 20, 3);
    rw.validateRecords = true;
    bool threw = false;
    try { rw.rewrite(manifest, fetchBad, ix.object, nullptr, &newKey, ivs.data(), indexIvs.data(), [](const UploadPart&, const uint8_t*) {}); }
    catch (const InvalidRecordBatchException& e) { threw = strstr(e.what(), "(check: crc)") != nullptr; }
    CHECK(threw);
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
