// segment_rewrite.hpp — a stored segment rewritten under a new data key, or with compression or encryption added, host-only C++
// over tsgpu_rewrite_object.
//
// An operator tool reads the segment's manifest (parseSegmentManifestV1), fetches the `.log` object in windows of chunks with
// ranged GETs (as FetchChunkEnumeration fetches a range) and has the GPU check every chunk as RemoteSegmentChecker does and
// transform it for the new object; the segment's plaintext never reaches host memory.  The new object goes to the part sink in
// upload parts of partSize bytes, each with its CRC-32C.  The five index blobs of the `.indexes` object are small and carry no
// record payloads: they are decrypted with the old key and encrypted with the new one on the host (fetchIndexBytes,
// uploadIndexes), so their plaintext does pass through host memory.  The caller writes the new manifest with
// segmentManifestV1Json from the result, after the new `.log` and `.indexes` objects are uploaded (INTEGRATION.md).
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include "segment_upload.hpp"

namespace tieredstorage {

struct SegmentRewrite {
    std::shared_ptr<ChunkIndex> chunkIndex;      // the new object's, built as SegmentLogUploader builds it
    bool compressed = false;
    uint64_t objectBytes = 0;
    Bytes indexesObject;                         // the new `.indexes` object
    SegmentIndexesV1 segmentIndexes{};
    uint32_t sourceCrc32c = 0;                   // CRC-32C of the old `.log` object (compare with the store's checksum of it)
    uint32_t objectCrc32c = 0;                   // CRC-32C of the new `.log` object (S3 FULL_OBJECT, GCS crc32c)
    uint32_t segmentCrc32c = 0;                  // CRC-32C of the decoded segment (the same for both objects)
    // With RemoteSegmentRewriter::crc64 the three words are CRC-64/NVME (S3 CRC64NVME) here instead, and the 32-bit ones stay 0.
    uint64_t sourceCrc64nvme = 0, objectCrc64nvme = 0, segmentCrc64nvme = 0;
};

class RemoteSegmentRewriter {
public:
    using RangeFetcher = FetchChunkEnumeration::RangeFetcher;       // ObjectFetcher.fetch(key, range) on the old .log object
    using PartSink = SegmentLogUploader::PartSink;
    // The new object's compression and encryption; at least one must be on (the plain object is what a fetch gives).
    RemoteSegmentRewriter(tsgpu_ctx* ctx, bool compressionEnabled, bool encryptionEnabled, uint64_t partSize, uint32_t windowChunks = 32)
        : ctx(ctx), compressionEnabled(compressionEnabled), encryptionEnabled(encryptionEnabled), partSize(partSize),
          window(windowChunks ? windowChunks : 1) {
        if (!ctx) throw NullPointerException("ctx cannot be null");
        if (!compressionEnabled && !encryptionEnabled) throw IllegalArgumentException("the new object needs compression or encryption");
        if (partSize == 0) throw IllegalArgumentException("partSize must be positive");
    }
    bool validateRecords = false;        // also check every record batch of the decoded segment (TSGPU_FLAG_VALIDATE_RECORDS)
    bool verify = false;                 // read every new batch back on the GPU before it leaves (TSGPU_FLAG_VERIFY)
    // With compressionEnabled: every new frame carries its Content_Checksum (addChecksums), or comes from the dense compressor
    // when that makes it smaller (denseFrames).  A compressed source's frames are sealed or re-encoded (TSGPU_FLAG_REFRAME, which
    // also reads every new chunk back); a plain source is compressed with the ZSTD_CHECKSUM and ZSTD_DENSE modifiers.
    bool addChecksums = false;
    bool denseFrames = false;
    // CRC-64/NVME instead of CRC-32C (tsgpu_rewrite_object_crc64): every part reaches the sink with crc64nvme, and the result
    // carries the 64-bit words.  The new object's bytes are the same.
    bool crc64 = false;

    // `oldKey`: the old manifest's unwrapped data key and AAD, or null when it has no encryption.  `newKey`: the new data key
    // (DataKeyAndAAD) when encryptionEnabled; `ivs`: 12 random bytes per chunk of the segment and `indexIvs` 12 per non-empty
    // index blob, under newKey.  Throws InvalidRecordBatchException for a bad record batch, IllegalArgumentException for
    // arguments the library refuses (among them an IV of the old object reused under the same key), and std::runtime_error for a
    // failed tag, a bad frame, a size that disagrees with the index, a new chunk that did not read back or a short fetch; the
    // message is the library's.  Parts already handed to the sink belong to an upload the caller then aborts.
    SegmentRewrite rewrite(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const Bytes& indexesObject,
                           const DataKeyAndAAD* oldKey, const DataKeyAndAAD* newKey, const uint8_t* ivs, const uint8_t* indexIvs,
                           const PartSink& sink) const {
        if (!fetcher) throw NullPointerException("objectKey cannot be null");
        if (!manifest.chunkIndex) throw NullPointerException("chunkIndex cannot be null");
        const bool encrypted = manifest.aad.has_value();
        if (encrypted && !oldKey) throw NullPointerException("dataKey cannot be null");
        if (encrypted && oldKey->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        if (encryptionEnabled && (!newKey || !ivs || !indexIvs)) throw NullPointerException("cipherSupplier cannot be null");
        if (encryptionEnabled && newKey->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        const uint32_t from = (manifest.compression ? TSGPU_FLAG_ZSTD : 0u) | (encrypted ? TSGPU_FLAG_AES : 0u) |
                              (validateRecords ? TSGPU_FLAG_VALIDATE_RECORDS : 0u);
        const uint32_t modifiers = compressionEnabled ? (addChecksums ? TSGPU_FLAG_ZSTD_CHECKSUM : 0u) |
                                                        (denseFrames ? TSGPU_FLAG_ZSTD_DENSE : 0u) : 0u;
        const uint32_t to = (compressionEnabled ? TSGPU_FLAG_ZSTD : 0u) | (encryptionEnabled ? TSGPU_FLAG_AES : 0u) |
                            (verify ? TSGPU_FLAG_VERIFY : 0u) | modifiers |
                            (modifiers && manifest.compression ? TSGPU_FLAG_REFRAME : 0u);
        const ChunkIndex& index = *manifest.chunkIndex;
        const std::vector<Chunk>& chunks = index.chunks();
        const uint32_t ocs = (uint32_t)index.originalChunkSize;
        tsgpu_rewrite_cursor cursor{};
        SegmentRewrite r;
        r.compressed = compressionEnabled;
        std::vector<int32_t> sizes;                  // the new object's chunk sizes
        Bytes pending;                               // bytes of the open part
        std::vector<uint64_t> crcs;                  // CRCs of the parts not yet handed to the sink
        int partNumber = 0;
        uint64_t sent = 0;
        auto emit = [&](uint64_t n, uint64_t crc) {
            UploadPart p{++partNumber, sent, n};
            if (crc64) p.crc64nvme = crc;
            else p.crc32c = (uint32_t)crc;
            sink(p, pending.data());
            pending.erase(pending.begin(), pending.begin() + (ptrdiff_t)n);
            sent += n;
        };
        for (size_t k = 0;; k += window) {
            const size_t e = std::min(chunks.size(), k + window);
            const bool end = e == chunks.size();
            std::vector<uint32_t> tsz;
            Bytes bytes;
            uint64_t oneWindow = 0;
            if (k < e) {
                const std::vector<Chunk> part(chunks.begin() + k, chunks.begin() + e);
                for (const Chunk& c : part) { tsz.push_back((uint32_t)c.transformedSize); oneWindow += (uint64_t)c.originalSize; }
                const BytesRange range = transformedRange(part);
                if (!range.isEmpty()) bytes = fetcher(range);
            }
            // room for every new chunk, kept frames included (a frame plus IV and tag per chunk, and 4 bytes for a sealed frame)
            const uint64_t cap = std::max<uint64_t>(tsgpu_transform_bound(to | TSGPU_FLAG_ZSTD, oneWindow, ocs),
                                                    (uint64_t)bytes.size() + 28 * tsz.size()) + 28 * tsz.size() + 64;
            Bytes out(cap);
            std::vector<uint32_t> nsz(std::max<size_t>(tsz.size(), 1));
            const size_t partCap = (pending.size() + cap) / partSize + 2;
            std::vector<uint32_t> windowCrcs(crc64 ? 0 : partCap);
            std::vector<uint64_t> windowCrcs64(crc64 ? partCap : 0);
            uint32_t nParts = 0, src = 0, obj = 0, seg = 0;
            uint64_t src64 = 0, obj64 = 0, seg64 = 0;
            const int rc = crc64
                ? tsgpu_rewrite_object_crc64(ctx, from, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(), ocs,
                                             (uint64_t)index.originalFileSize, encrypted ? oldKey->dataKey.data() : nullptr,
                                             encrypted ? oldKey->aad.data() : nullptr, encrypted ? (uint32_t)oldKey->aad.size() : 0u,
                                             to, encryptionEnabled ? newKey->dataKey.data() : nullptr,
                                             encryptionEnabled ? newKey->aad.data() : nullptr,
                                             encryptionEnabled ? (uint32_t)newKey->aad.size() : 0u,
                                             encryptionEnabled ? ivs + 12 * k : nullptr, out.data(), out.size(), nsz.data(),
                                             partSize, windowCrcs64.data(), (uint32_t)partCap, &nParts, &cursor,
                                             end ? 1 : 0, &src64, &obj64, &seg64)
                : tsgpu_rewrite_object(ctx, from, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(), ocs,
                                                (uint64_t)index.originalFileSize, encrypted ? oldKey->dataKey.data() : nullptr,
                                                encrypted ? oldKey->aad.data() : nullptr, encrypted ? (uint32_t)oldKey->aad.size() : 0u,
                                                to, encryptionEnabled ? newKey->dataKey.data() : nullptr,
                                                encryptionEnabled ? newKey->aad.data() : nullptr,
                                                encryptionEnabled ? (uint32_t)newKey->aad.size() : 0u,
                                                encryptionEnabled ? ivs + 12 * k : nullptr, out.data(), out.size(), nsz.data(),
                                                partSize, windowCrcs.data(), (uint32_t)windowCrcs.size(), &nParts, &cursor,
                                                end ? 1 : 0, &src, &obj, &seg);
            if (rc == TSGPU_E_RECORDS) throw InvalidRecordBatchException(tsgpu_last_error());
            if (rc == TSGPU_E_ARG) throw IllegalArgumentException(tsgpu_last_error());
            if (rc) throw std::runtime_error(tsgpu_last_error());
            uint64_t produced = 0;
            for (size_t i = 0; i < tsz.size(); i++) { sizes.push_back((int32_t)nsz[i]); produced += nsz[i]; }
            pending.insert(pending.end(), out.begin(), out.begin() + (ptrdiff_t)produced);
            r.objectBytes += produced;
            if (crc64) crcs.insert(crcs.end(), windowCrcs64.begin(), windowCrcs64.begin() + nParts);
            else crcs.insert(crcs.end(), windowCrcs.begin(), windowCrcs.begin() + nParts);
            size_t c = 0;
            for (; c < crcs.size() && pending.size() >= partSize; c++) emit(partSize, crcs[c]);
            if (end && !pending.empty() && c < crcs.size()) emit(pending.size(), crcs[c++]);
            crcs.erase(crcs.begin(), crcs.begin() + (ptrdiff_t)c);
            if (end) {
                if (!pending.empty() || !crcs.empty()) throw std::runtime_error("part checksums do not match the new object");
                r.sourceCrc32c = src; r.objectCrc32c = obj; r.segmentCrc32c = seg;
                r.sourceCrc64nvme = src64; r.objectCrc64nvme = obj64; r.segmentCrc64nvme = seg64;
                break;
            }
        }
        const int ofs = (int)index.originalFileSize;
        if (sizes.empty()) {
            r.chunkIndex = FixedSizeChunkIndexBuilder((int)ocs, ofs, (int)ocs).finish(0);
        } else if (compressionEnabled) {
            VariableSizeChunkIndexBuilder b((int)ocs, ofs);
            for (size_t i = 0; i + 1 < sizes.size(); i++) b.addChunk(sizes[i]);
            r.chunkIndex = b.finish(sizes.back());
        } else {
            FixedSizeChunkIndexBuilder b((int)ocs, ofs, (int)ocs + 28);
            for (size_t i = 0; i + 1 < sizes.size(); i++) b.addChunk(sizes[i]);
            r.chunkIndex = b.finish(sizes.back());
        }
        // the index blobs: plaintext on the host, as fetchIndexBytes and uploadIndexes handle them
        const SegmentIndexesV1& si = manifest.segmentIndexes;
        const DataKeyAndAAD* dec = encrypted ? oldKey : nullptr;
        std::vector<std::pair<IndexType, Bytes>> blobs{
            {IndexType::OFFSET, fetchIndexBytes(ctx, indexesObject, si.offset, dec)},
            {IndexType::TIMESTAMP, fetchIndexBytes(ctx, indexesObject, si.timestamp, dec)},
            {IndexType::PRODUCER_SNAPSHOT, fetchIndexBytes(ctx, indexesObject, si.producerSnapshot, dec)},
            {IndexType::LEADER_EPOCH, fetchIndexBytes(ctx, indexesObject, si.leaderEpoch, dec)}};
        if (si.transaction) blobs.push_back({IndexType::TRANSACTION, fetchIndexBytes(ctx, indexesObject, *si.transaction, dec)});
        SegmentIndexesUpload ix = uploadIndexes(ctx, blobs, encryptionEnabled, newKey, indexIvs);
        r.indexesObject = std::move(ix.object);
        r.segmentIndexes = ix.segmentIndexes;
        return r;
    }

private:
    tsgpu_ctx* ctx;
    bool compressionEnabled, encryptionEnabled;
    uint64_t partSize;
    uint32_t window;
};

}  // namespace tieredstorage
