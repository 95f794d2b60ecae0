// Host mirror of encryption after the fact (RemoteSegmentEncryptor, tsgpu_encrypt_object): a Zstd-only `.log` object the oracle
// wrote (libzstd level 3: what the Java plugin wrote) and a plain one, each with an unencrypted `.indexes` object holding an empty
// producer-snapshot blob, are encrypted, the `.log` object in windows of 1, 3 and 64 chunks.  The new chunk index is the one
// TransformFinisher builds with encryption on (variable for the compressed object, fixed with transformedChunkSize = ocs + 28 for the
// plain one), the new objects detransform through the oracle to the segment and the index blobs, the SegmentIndexesV1 positions
// follow the new sizes (non-empty blobs 28 bytes longer, the empty one empty), the parts reach the sink in order with the CRC of
// their bytes, and the CRC-64/NVME form writes the same bytes.  A manifest that already has encryption is refused.  Links the
// test-only SIMT build and the oracle.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_encrypt.hpp"
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
static Bytes random(size_t n, std::mt19937& rng) { Bytes b(n); for (auto& x : b) x = (uint8_t)rng(); return b; }
static uint64_t crc64nvme(const uint8_t* p, size_t n) {
    uint64_t c = ~0ull;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x9A6C9329AC4BC9B5ull & (0ull - (c & 1ull))); }
    return ~c;
}

int main() {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(37);
    const Bytes seg = segment(60000, rng);
    const int cs = 8192, n = (int)seg.size();
    const int nch = (n + cs - 1) / cs;
    const std::vector<std::pair<IndexType, Bytes>> blobs{
        {IndexType::OFFSET, random(800, rng)}, {IndexType::TIMESTAMP, random(1200, rng)}, {IndexType::PRODUCER_SNAPSHOT, Bytes()},
        {IndexType::LEADER_EPOCH, random(40, rng)}, {IndexType::TRANSACTION, random(100, rng)}};
    DataKeyAndAAD key; key.dataKey = random(32, rng); key.aad = random(32, rng);
    const Bytes ivs = random(12 * nch, rng), indexIvs = random(12 * 4, rng), zeros(12 * nch, 0);
    const SegmentIndexesUpload ix = uploadIndexes(ctx, blobs, false, nullptr, nullptr);         // stored unencrypted
    RemoteLogSegmentMetadataJson meta{"topic-id", "topic", 3, "segment-id", 0, 99, 1234, 1, 5678, {{0, 0}}};

    for (int compressed = 0; compressed < 2; compressed++) {
        Bytes object;
        std::vector<int32_t> isz;
        if (compressed) {
            object.resize(ora_transform_bound(TSGPU_FLAG_ZSTD, n, cs) + 64);
            std::vector<uint32_t> sizes(nch + 1);
            uint32_t got_n = (uint32_t)sizes.size();
            CHECK(ora_transform_segment(TSGPU_FLAG_ZSTD, seg.data(), n, cs, nullptr, nullptr, 0, zeros.data(), object.data(),
                                        object.size(), sizes.data(), &got_n) == 0 && got_n == (uint32_t)nch);
            isz.assign(sizes.begin(), sizes.begin() + nch);
        } else {
            object = seg;
            for (int i = 0; i < nch; i++) isz.push_back(std::min(cs, n - i * cs));
        }
        size_t total = 0;
        for (int32_t s : isz) total += (size_t)s;
        object.resize(total);
        SegmentManifestV1 manifest;
        const std::vector<uint32_t> usz(isz.begin(), isz.end());
        manifest.chunkIndex = finisherChunkIndex(cs, n, compressed != 0, false, usz.data(), (uint32_t)nch);   // as uploaded
        manifest.compression = compressed != 0;
        manifest.segmentIndexes = ix.segmentIndexes;
        auto fetchOld = [&](const BytesRange& r) { return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };
        // what TransformFinisher builds for these original sizes with encryption on
        std::vector<uint32_t> want(isz.begin(), isz.end());
        for (uint32_t& s : want) s += 28;
        const std::string wantIndex = finisherChunkIndex(cs, n, compressed != 0, true, want.data(), (uint32_t)want.size())->toJson();
        Bytes first;
        for (int wide = 0; wide < 2; wide++) for (uint32_t window : {1u, 3u, 64u}) {
            const uint64_t partSize = 5000;
            RemoteSegmentEncryptor en(ctx, partSize, window);
            en.verify = window == 3;
            en.crc64 = wide != 0;
            Bytes neo;
            bool inOrder = true, crcsMatch = true;
            const SegmentEncrypt got = en.encrypt(manifest, fetchOld, ix.object, &key, ivs.data(), indexIvs.data(),
                [&](const UploadPart& p, const uint8_t* d) {
                    inOrder &= p.offset == neo.size() && p.partNumber == (int)(neo.size() / partSize) + 1;
                    crcsMatch &= wide ? (p.crc64nvme && *p.crc64nvme == crc64nvme(d, p.size)) : (p.crc32c && *p.crc32c == crc32c(d, p.size));
                    neo.insert(neo.end(), d, d + p.size);
                });
            CHECK(inOrder && crcsMatch);
            CHECK(neo.size() == total + 28ull * nch && got.objectBytes == neo.size());
            if (first.empty() || wide + window == 1) first = neo;
            CHECK(neo == first);                                           // every window and both widths write the same bytes
            // the chunk index: TransformFinisher's, of the type it picks
            CHECK(got.chunkIndex->toJson() == wantIndex);
            CHECK(compressed ? dynamic_cast<const VariableSizeChunkIndex*>(got.chunkIndex.get()) != nullptr
                             : dynamic_cast<const FixedSizeChunkIndex*>(got.chunkIndex.get()) != nullptr);
            std::vector<uint32_t> nsz;
            for (const Chunk& c : got.chunkIndex->chunks()) nsz.push_back((uint32_t)c.transformedSize);
            CHECK(nsz == want);
            const uint32_t fl = TSGPU_FLAG_AES | (compressed ? TSGPU_FLAG_ZSTD : 0u);
            Bytes back(n);
            CHECK(ora_detransform_chunks(fl, neo.data(), nsz.data(), nch, key.dataKey.data(), key.aad.data(), key.aad.size(),
                                         back.data(), back.size(), nullptr) == 0 && back == seg);
            // the .indexes object: non-empty blobs 28 bytes longer at positions that follow the new sizes, the empty one empty
            const SegmentIndexesV1& si = got.segmentIndexes;
            const SegmentIndexV1 all[5] = {si.offset, si.timestamp, si.producerSnapshot, si.leaderEpoch, *si.transaction};
            int pos = 0;
            for (int i = 0; i < 5; i++) {
                const int size = blobs[i].second.empty() ? 0 : (int)blobs[i].second.size() + 28;
                CHECK(all[i].position == pos && all[i].size == size);
                pos += size;
                CHECK(fetchIndexBytes(ctx, got.indexesObject, all[i], &key) == blobs[i].second);
            }
            CHECK((int)got.indexesObject.size() == pos);
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
            CHECK(got.indexesPartCrcs.size() == (got.indexesObject.size() + partSize - 1) / partSize);
            // the manifest the caller writes: encryption on, the new index fields
            const std::string json = segmentManifestV1Json(*got.chunkIndex, got.segmentIndexes, compressed != 0,
                                                           std::string("new-key:BBBB"), &key.aad, meta);
            CHECK(json.find(base64Std(key.aad.data(), key.aad.size())) != std::string::npos);
        }
        // a segment stored with encryption already has a key: rotating it is another call
        {
            SegmentManifestV1 enc = manifest;
            enc.aad = key.aad;
            enc.wrappedDataKey = std::string("old-key:AAAA");
            bool refused = false;
            try {
                RemoteSegmentEncryptor(ctx, 5000).encrypt(enc, fetchOld, ix.object, &key, ivs.data(), indexIvs.data(),
                                                          [](const UploadPart&, const uint8_t*) {});
            } catch (const IllegalArgumentException& e) {
                refused = strstr(e.what(), "already encrypted") != nullptr;
            }
            CHECK(refused);
        }
        // a chunk index that does not match the object: the library's refusal
        {
            SegmentManifestV1 wrong = manifest;
            if (compressed) wrong.chunkIndex = std::make_shared<VariableSizeChunkIndex>(cs, n + 1, isz);
            bool refused = !compressed;
            try {
                if (compressed) RemoteSegmentEncryptor(ctx, 5000).encrypt(wrong, fetchOld, ix.object, &key, ivs.data(), indexIvs.data(),
                                                                          [](const UploadPart&, const uint8_t*) {});
            } catch (const std::runtime_error& e) {
                refused = strstr(e.what(), "the chunk index gives") != nullptr;
            }
            CHECK(refused);
        }
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
