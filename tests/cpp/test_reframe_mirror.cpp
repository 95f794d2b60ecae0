// Host mirror of TSGPU_FLAG_REFRAME (RemoteSegmentRewriter::addChecksums and ::denseFrames): a Zstd+AES object the oracle wrote
// (libzstd level 3 + OpenSSL, no Content_Checksum: what the Java plugin wrote) is rewritten under a new key in windows of 1, 3 and
// 64 chunks.  With addChecksums every new frame is libzstd's checksummed frame of the chunk and 4 bytes longer; with denseFrames
// too, no chunk grows by more than 4 bytes and every frame carries its checksum.  The new ChunkIndex takes the new sizes, the
// parts reach the sink in order with the CRC-32C of their bytes, and the new object, under a manifest with that index, passes
// RemoteSegmentChecker with the segment CRC of the old one.  A plain source is compressed with the two modifiers instead, and
// without compressionEnabled the options change nothing.  Links the test-only SIMT build and the oracle.
#include <cstdio>
#include <cstring>
#include <random>
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_rewrite.hpp"
#include "../../tiered-storage-for-apache-kafka_b200/host/segment_check.hpp"
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

// The chunks of an object by its index, decrypted with `key` when it has one.
static std::vector<Bytes> frames(const Bytes& obj, const ChunkIndex& index, const DataKeyAndAAD* key) {
    std::vector<Bytes> out;
    for (const Chunk& c : index.chunks()) {
        Bytes ch(obj.begin() + c.transformedPosition, obj.begin() + c.transformedPosition + c.transformedSize);
        if (key) {
            Bytes pt(ch.size() - 28);
            if (ora_aesgcm_decrypt_chunk(key->dataKey.data(), key->aad.data(), key->aad.size(), ch.data(), ch.size(), pt.data())) pt.clear();
            ch = pt;
        }
        out.push_back(ch);
    }
    return out;
}

int main() {
    tsgpu_ctx* ctx = nullptr;
    if (tsgpu_create(nullptr, 0, 1 << 16, 2, &ctx)) { printf("tsgpu_create failed: %s\n", tsgpu_last_error()); return 2; }
    std::mt19937 rng(29);
    const Bytes seg = segment(60000, rng);
    const int cs = 8192, n = (int)seg.size();
    const int nch = (n + cs - 1) / cs;
    const std::vector<std::pair<IndexType, Bytes>> blobs{
        {IndexType::OFFSET, random(800, rng)}, {IndexType::TIMESTAMP, random(1200, rng)}, {IndexType::PRODUCER_SNAPSHOT, Bytes()},
        {IndexType::LEADER_EPOCH, random(40, rng)}, {IndexType::TRANSACTION, random(100, rng)}};
    const DataKeyAndAAD oldKey = keyMaterial(rng), newKey = keyMaterial(rng);
    const Bytes oldIvs = random(12 * nch, rng), ivs = random(12 * nch, rng), indexIvs = random(12 * 5, rng), oldIndexIvs = random(12 * 5, rng);

    // the oracle's Zstd+AES object and a manifest for it
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
    const SegmentIndexesUpload ix = uploadIndexes(ctx, blobs, true, &oldKey, oldIndexIvs.data());
    manifest.segmentIndexes = ix.segmentIndexes;
    auto fetchOld = [&](const BytesRange& r) { return Bytes(object.begin() + r.from, object.begin() + r.to + 1); };
    const std::vector<Bytes> oldFrames = frames(object, *manifest.chunkIndex, &oldKey);
    std::vector<Bytes> sealed;                                         // libzstd's level-3 frames with their checksum
    for (int i = 0; i < nch; i++) {
        const int len = std::min(cs, n - i * cs);
        Bytes f(ora_zstd_bound(len) + 8);
        const int64_t m = ora_zstd_compress_checksum(seg.data() + (size_t)i * cs, len, f.data(), f.size(), 3);
        f.resize(m > 0 ? (size_t)m : 0);
        sealed.push_back(f);
    }

    for (int dense = 0; dense < 2; dense++) for (uint32_t window : {1u, 3u, 64u}) {
        const uint64_t partSize = 5000;
        RemoteSegmentRewriter rw(ctx, true, true, partSize, window);
        rw.validateRecords = true;
        rw.addChecksums = true;
        rw.denseFrames = dense != 0;
        Bytes neo;
        bool inOrder = true, crcsMatch = true;
        const SegmentRewrite got = rw.rewrite(manifest, fetchOld, ix.object, &oldKey, &newKey, ivs.data(), indexIvs.data(),
            [&](const UploadPart& p, const uint8_t* d) {
                inOrder &= p.offset == neo.size() && p.partNumber == (int)(neo.size() / partSize) + 1;
                crcsMatch &= p.crc32c && *p.crc32c == crc32c(d, p.size);
                neo.insert(neo.end(), d, d + p.size);
            });
        CHECK(inOrder && crcsMatch && neo.size() == got.objectBytes);
        CHECK(got.sourceCrc32c == crc32c(object.data(), object.size()));
        CHECK(got.objectCrc32c == crc32c(neo.data(), neo.size()));
        CHECK(got.segmentCrc32c == crc32c(seg.data(), seg.size()));
        // the new index: the new sizes, each chunk at most 4 bytes longer (exactly 4 when sealed), the object's length in all
        const std::vector<Chunk>& nc = got.chunkIndex->chunks();
        CHECK(nc.size() == (size_t)nch && got.chunkIndex->originalChunkSize == cs && got.chunkIndex->originalFileSize == n);
        uint64_t sum = 0;
        for (int i = 0; i < nch; i++) {
            sum += (uint64_t)nc[i].transformedSize;
            CHECK(nc[i].transformedSize <= isz[i] + 4);
            if (!dense) CHECK(nc[i].transformedSize == isz[i] + 4);
        }
        CHECK(sum == neo.size());
        const std::vector<Bytes> nf = frames(neo, *got.chunkIndex, &newKey);
        for (int i = 0; i < nch; i++) {
            const int len = std::min(cs, n - i * cs);
            CHECK(nf[i].size() > 4 && (nf[i][4] & 0x04));
            if (!dense) CHECK(nf[i] == sealed[i]);
            Bytes back(len + 16);
            CHECK(ora_zstd_decompress_chunk(nf[i].data(), nf[i].size(), back.data(), back.size()) == len);   // verifies the checksum
            CHECK(memcmp(back.data(), seg.data() + (size_t)i * cs, len) == 0);
        }
        // a manifest with the new index: the new object passes the check with the old object's segment CRC
        SegmentManifestV1 m2 = manifest;
        m2.chunkIndex = got.chunkIndex;
        m2.aad = newKey.aad;
        m2.segmentIndexes = got.segmentIndexes;
        auto fetchNew = [&](const BytesRange& r) { return Bytes(neo.begin() + r.from, neo.begin() + r.to + 1); };
        RemoteSegmentChecker ck(ctx, 3);
        ck.validateRecords = true;
        const ObjectCheck oc = ck.check(m2, fetchNew, &newKey);
        CHECK(oc.objectCrc32c == got.objectCrc32c && oc.segmentCrc32c == got.segmentCrc32c);
        CHECK(fetchIndexBytes(ctx, got.indexesObject, m2.segmentIndexes.offset, &newKey) == blobs[0].second);
    }

    // a plain source: compressed with the modifiers (no REFRAME, which needs compressed frames)
    SegmentLogUploader up(ctx, cs, false, false, false, 1 << 20);
    Bytes plain;
    auto res = up.upload(seg.data(), seg.size(), nullptr, nullptr,
                         [&](const UploadPart& p, const uint8_t* d) { plain.insert(plain.end(), d, d + p.size); });
    const SegmentIndexesUpload pix = uploadIndexes(ctx, blobs, false, nullptr, nullptr);
    SegmentManifestV1 pm;
    pm.chunkIndex = res.chunkIndex;
    pm.segmentIndexes = pix.segmentIndexes;
    auto fetchPlain = [&](const BytesRange& r) { return Bytes(plain.begin() + r.from, plain.begin() + r.to + 1); };
    {
        RemoteSegmentRewriter rw(ctx, true, false, 1 << 30, 3);
        rw.addChecksums = true;
        rw.denseFrames = true;
        Bytes neo;
        const SegmentRewrite got = rw.rewrite(pm, fetchPlain, pix.object, nullptr, nullptr, nullptr, nullptr,
                                              [&](const UploadPart& p, const uint8_t* d) { neo.insert(neo.end(), d, d + p.size); });
        const std::vector<Bytes> nf = frames(neo, *got.chunkIndex, nullptr);
        Bytes dense(tsgpu_transform_bound(TSGPU_FLAG_ZSTD, n, cs));
        std::vector<uint32_t> dsz(nch + 1);
        uint32_t dn = (uint32_t)dsz.size();
        CHECK(tsgpu_transform(ctx, TSGPU_FLAG_ZSTD | TSGPU_FLAG_ZSTD_DENSE | TSGPU_FLAG_ZSTD_CHECKSUM, seg.data(), n, cs, nullptr,
                              nullptr, 0, nullptr, dense.data(), dense.size(), dsz.data(), &dn) == 0);
        size_t at = 0;
        for (int i = 0; i < nch; i++) {
            CHECK(nf[i] == Bytes(dense.begin() + at, dense.begin() + at + dsz[i]));                  // tsgpu_transform's dense frames
            at += dsz[i];
        }
        CHECK(got.segmentCrc32c == crc32c(seg.data(), seg.size()));
    }
    // without compressionEnabled the options change nothing: an encrypted-only object, identical to one rewritten without them
    {
        Bytes a, b;
        RemoteSegmentRewriter rw(ctx, false, true, 1 << 30, 3);
        rw.rewrite(manifest, fetchOld, ix.object, &oldKey, &newKey, ivs.data(), indexIvs.data(),
                   [&](const UploadPart& p, const uint8_t* d) { a.insert(a.end(), d, d + p.size); });
        rw.addChecksums = true;
        rw.denseFrames = true;
        rw.rewrite(manifest, fetchOld, ix.object, &oldKey, &newKey, ivs.data(), indexIvs.data(),
                   [&](const UploadPart& p, const uint8_t* d) { b.insert(b.end(), d, d + p.size); });
        CHECK(!a.empty() && a == b);
    }
    tsgpu_destroy(ctx);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
