// Host mirror of key rotation (RemoteSegmentRekeyer, tsgpu_rekey_object): a Zstd+AES `.log` object the oracle wrote (libzstd level
// 3 + OpenSSL: what the Java plugin wrote) and its `.indexes` object with an empty producer-snapshot blob are re-encrypted under a
// new key, the `.log` object in windows of 1, 3 and 64 chunks.  Both new objects decrypt under the new key with the oracle to the
// old plaintexts and fail under the old key; the parts reach the sink in order with the CRC of their bytes; the chunk index and
// SegmentIndexesV1 are unchanged and the manifest JSON differs only in its encryption fields.  The CRC-64/NVME form writes the
// same bytes.  A manifest without encryption is refused.  Links the test-only SIMT build and the oracle.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_rekey.hpp"
#include "../../oracle/tsoracle.h"

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

static uint64_t crc64nvme(const uint8_t* p, size_t n) {
    uint64_t c = ~0ull;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x9A6C9329AC4BC9B5ull & (0ull - (c & 1ull))); }
    return ~c;
}
// Chunk `size` bytes at `pos` of `obj` decrypted with `key`; false when its tag fails.
static bool decrypts(const Bytes& obj, size_t pos, size_t size, const DataKeyAndAAD& key, Bytes& pt) {
    pt.assign(size >= 28 ? size - 28 : 0, 0);
    return size >= 28 && ora_aesgcm_decrypt_chunk(key.dataKey.data(), key.aad.data(), key.aad.size(), obj.data() + pos, size, pt.data()) == 0;
}
// The encryption object of a manifest JSON cut out: what must stay the same across a key rotation.
static std::string withoutEncryption(const std::string& s) {
    const size_t a = s.find(",\"encryption\":{");
    const size_t b = s.find('}', a);
    return a == std::string::npos ? s : s.substr(0, a) + s.substr(b + 1);
}

int main() {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(31);
    const Bytes seg = segment(60000, rng);
    const int cs = 8192, n = (int)seg.size();
    const int nch = (n + cs - 1) / cs;
    const std::vector<std::pair<IndexType, Bytes>> blobs{
        {IndexType::OFFSET, random(800, rng)}, {IndexType::TIMESTAMP, random(1200, rng)}, {IndexType::PRODUCER_SNAPSHOT, Bytes()},
        {IndexType::LEADER_EPOCH, random(40, rng)}, {IndexType::TRANSACTION, random(100, rng)}};
    const DataKeyAndAAD oldKey = keyMaterial(rng), newKey = keyMaterial(rng);
    const Bytes oldIvs = random(12 * nch, rng), ivs = random(12 * nch, rng), indexIvs = random(12 * 4, rng), oldIndexIvs = random(12 * 5, rng);

    Bytes object(ora_transform_bound(TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES, n, cs) + 64);
    std::vector<uint32_t> sizes(nch + 1);
    uint32_t got_n = (uint32_t)sizes.size();
    CHECK(ora_transform_segment(TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES, seg.data(), n, cs, oldKey.dataKey.data(), oldKey.aad.data(),
                                (uint32_t)oldKey.aad.size(), oldIvs.data(), object.data(), object.size(), sizes.data(), &got_n) == 0);
    CHECK(got_n == (uint32_t)nch);
    std::vector<int32_t> isz(sizes.begin(), sizes.begin() + nch);
    size_t total = 0;
    for (int32_t s : isz) total += (size_t)s;
    object.resize(total);
    SegmentManifestV1 manifest;
    manifest.chunkIndex = std::make_shared<VariableSizeChunkIndex>(cs, n, isz);
    manifest.compression = true;
    manifest.aad = oldKey.aad;
    manifest.wrappedDataKey = std::string("old-key:AAAA");
    const SegmentIndexesUpload ix = uploadIndexes(ctx, blobs, true, &oldKey, oldIndexIvs.data());
    manifest.segmentIndexes = ix.segmentIndexes;
    CHECK(ix.segmentIndexes.producerSnapshot.size == 0);
    auto fetchOld = [&](const BytesRange& r) { return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };
    RemoteLogSegmentMetadataJson meta{"topic-id", "topic", 3, "segment-id", 0, 99, 1234, 1, 5678, {{0, 0}}};
    const std::string oldJson = segmentManifestV1Json(*manifest.chunkIndex, manifest.segmentIndexes, true, manifest.wrappedDataKey,
                                                      &oldKey.aad, meta);

    Bytes first;
    for (int wide = 0; wide < 2; wide++) for (uint32_t window : {1u, 3u, 64u}) {
        const uint64_t partSize = 5000;
        RemoteSegmentRekeyer rk(ctx, partSize, window);
        rk.verify = window == 3;
        rk.crc64 = wide != 0;
        Bytes neo;
        bool inOrder = true, crcsMatch = true;
        const SegmentRekey got = rk.rekey(manifest, fetchOld, ix.object, &oldKey, &newKey, ivs.data(), indexIvs.data(),
            [&](const UploadPart& p, const uint8_t* d) {
                inOrder &= p.offset == neo.size() && p.partNumber == (int)(neo.size() / partSize) + 1;
                crcsMatch &= wide ? (p.crc64nvme && *p.crc64nvme == crc64nvme(d, p.size)) : (p.crc32c && *p.crc32c == crc32c(d, p.size));
                neo.insert(neo.end(), d, d + p.size);
            });
        CHECK(inOrder && crcsMatch);
        CHECK(neo.size() == object.size() && got.objectBytes == object.size());
        if (first.empty()) first = neo;
        CHECK(neo == first);                                           // every window and both widths write the same bytes
        // the .log object: every chunk decrypts under the new key to the old frame, and no more under the old key
        bool same = true, oldFails = true;
        for (const Chunk& c : manifest.chunkIndex->chunks()) {
            Bytes a, b;
            same &= decrypts(object, c.transformedPosition, c.transformedSize, oldKey, a) &&
                    decrypts(neo, c.transformedPosition, c.transformedSize, newKey, b) && a == b;
            oldFails &= !decrypts(neo, c.transformedPosition, c.transformedSize, oldKey, b);
        }
        CHECK(same && oldFails);
        Bytes back(n);
        CHECK(ora_detransform_chunks(TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES, neo.data(), sizes.data(), nch, newKey.dataKey.data(),
                                     newKey.aad.data(), newKey.aad.size(), back.data(), back.size(), nullptr) == 0 && back == seg);
        // the .indexes object: every blob at its unchanged position and size, under the new key
        CHECK(got.indexesObject.size() == ix.object.size());
        const SegmentIndexesV1& si = got.segmentIndexes;
        const SegmentIndexV1 all[5] = {si.offset, si.timestamp, si.producerSnapshot, si.leaderEpoch, *si.transaction};
        const SegmentIndexV1 was[5] = {ix.segmentIndexes.offset, ix.segmentIndexes.timestamp, ix.segmentIndexes.producerSnapshot,
                                       ix.segmentIndexes.leaderEpoch, *ix.segmentIndexes.transaction};
        for (int i = 0; i < 5; i++) {
            CHECK(all[i].position == was[i].position && all[i].size == was[i].size);
            Bytes pt;
            if (all[i].size == 0) continue;
            CHECK(decrypts(got.indexesObject, all[i].position, all[i].size, newKey, pt) && pt == blobs[i].second);
            CHECK(!decrypts(got.indexesObject, all[i].position, all[i].size, oldKey, pt));
        }
        // the checksums of both objects
        if (wide) {
            CHECK(got.sourceCrc64nvme == crc64nvme(object.data(), object.size()) && got.objectCrc64nvme == crc64nvme(neo.data(), neo.size()));
            CHECK(got.indexesSourceCrc64nvme == crc64nvme(ix.object.data(), ix.object.size()));
            CHECK(got.indexesObjectCrc64nvme == crc64nvme(got.indexesObject.data(), got.indexesObject.size()));
        } else {
            CHECK(got.sourceCrc32c == crc32c(object.data(), object.size()) && got.objectCrc32c == crc32c(neo.data(), neo.size()));
            CHECK(got.indexesSourceCrc32c == crc32c(ix.object.data(), ix.object.size()));
            CHECK(got.indexesObjectCrc32c == crc32c(got.indexesObject.data(), got.indexesObject.size()));
        }
        CHECK(got.indexesPartCrcs.size() == (ix.object.size() + partSize - 1) / partSize);
        // the chunk index is the same object and the manifest changes only in its encryption fields
        CHECK(got.chunkIndex == manifest.chunkIndex);
        const std::string newJson = segmentManifestV1Json(*got.chunkIndex, got.segmentIndexes, true, std::string("new-key:BBBB"),
                                                          &newKey.aad, meta);
        CHECK(newJson != oldJson && withoutEncryption(newJson) == withoutEncryption(oldJson));
        CHECK(newJson.find(base64Std(newKey.aad.data(), newKey.aad.size())) != std::string::npos);
    }
    // a segment stored without encryption has no key to rotate
    {
        SegmentManifestV1 plain = manifest;
        plain.aad.reset();
        bool refused = false;
        try {
            RemoteSegmentRekeyer(ctx, 5000).rekey(plain, fetchOld, ix.object, &oldKey, &newKey, ivs.data(), indexIvs.data(),
                                                  [](const UploadPart&, const uint8_t*) {});
        } catch (const IllegalArgumentException& e) {
            refused = strstr(e.what(), "not encrypted") != nullptr;
        }
        CHECK(refused);
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
