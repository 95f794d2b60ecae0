// segment_encrypt.hpp — a stored unencrypted segment encrypted with AES-GCM, host-only C++ over tsgpu_encrypt_object.
//
// An operator tool that turns encryption on for segments already in the bucket reads a segment's manifest
// (parseSegmentManifestV1), fetches the `.log` object in windows of chunks with ranged GETs (as FetchChunkEnumeration fetches a
// range) and has the GPU encrypt every chunk as it is stored, frame or plain chunk, with nothing decoded: chunk i becomes
// IV || AES-GCM(chunk i) || TAG, 28 bytes longer.  The new `.log` object goes to the part sink in upload parts of partSize bytes,
// each with its CRC-32C.  The `.indexes` object is encrypted in one call whose chunks are its index blobs at their SegmentIndexV1
// positions and sizes; an empty blob stays empty, as transformIndex leaves it.  The result carries the chunk index and
// SegmentIndexesV1 the new objects need, exactly what TransformFinisher and uploadIndexes build for an encrypted upload: the
// caller writes the new manifest with segmentManifestV1Json, after both new objects are uploaded (INTEGRATION.md).
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include "segment_upload.hpp"

namespace tieredstorage {

struct SegmentEncrypt {
    std::shared_ptr<ChunkIndex> chunkIndex;      // of the new `.log` object
    SegmentIndexesV1 segmentIndexes{};           // of the new `.indexes` object
    uint64_t objectBytes = 0;                    // of the new `.log` object
    Bytes indexesObject;                         // the new `.indexes` object
    // CRC-32C of the old and the new `.log` object (the parts went to the sink), and of the old and the new `.indexes` object with
    // the CRC-32C of its upload parts of partSize bytes.  With RemoteSegmentEncryptor::crc64 these are CRC-64/NVME (S3 CRC64NVME)
    // in the 64-bit fields instead, and the 32-bit ones stay 0.
    uint32_t sourceCrc32c = 0, objectCrc32c = 0, indexesSourceCrc32c = 0, indexesObjectCrc32c = 0;
    uint64_t sourceCrc64nvme = 0, objectCrc64nvme = 0, indexesSourceCrc64nvme = 0, indexesObjectCrc64nvme = 0;
    std::vector<uint64_t> indexesPartCrcs;
};

class RemoteSegmentEncryptor {
public:
    using RangeFetcher = FetchChunkEnumeration::RangeFetcher;       // ObjectFetcher.fetch(key, range) on the old .log object
    using PartSink = SegmentLogUploader::PartSink;
    RemoteSegmentEncryptor(tsgpu_ctx* ctx, uint64_t partSize, uint32_t windowChunks = 32)
        : ctx(ctx), partSize(partSize), window(windowChunks ? windowChunks : 1) {
        if (!ctx) throw NullPointerException("ctx cannot be null");
        if (partSize == 0) throw IllegalArgumentException("partSize must be positive");
    }
    bool verify = false;                 // decrypt every batch again on the GPU and compare it with its source (TSGPU_FLAG_VERIFY)
    // CRC-64/NVME instead of CRC-32C (tsgpu_encrypt_object_crc64): every part reaches the sink with crc64nvme, and the result
    // carries the 64-bit words.  The new objects' bytes are the same.
    bool crc64 = false;

    // `newKey`: the data key and AAD to encrypt with.  `ivs`: 12 random bytes per chunk of the segment and `indexIvs` 12 per
    // non-empty index blob, in SegmentIndexesV1 order (offset, timestamp, producer snapshot, leader epoch, transaction).  Throws
    // IllegalArgumentException for a manifest that already has encryption and for arguments the library refuses (among them a
    // reused IV), and std::runtime_error for a chunk that does not match the chunk index, a frame the decoder would refuse, a new
    // chunk that did not read back or a short fetch; the message is the library's.  Parts already handed to the sink belong to an
    // upload the caller then aborts.
    SegmentEncrypt encrypt(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const Bytes& indexesObject,
                           const DataKeyAndAAD* newKey, const uint8_t* ivs, const uint8_t* indexIvs, const PartSink& sink) const {
        if (manifest.aad.has_value() || manifest.wrappedDataKey.has_value())
            throw IllegalArgumentException("the segment is already encrypted: rotate its data key with tsgpu_rekey_object instead");
        if (!fetcher) throw NullPointerException("objectKey cannot be null");
        if (!manifest.chunkIndex) throw NullPointerException("chunkIndex cannot be null");
        if (!newKey) throw NullPointerException("dataKey cannot be null");
        if (newKey->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        if (!ivs || !indexIvs) throw NullPointerException("ivs cannot be null");
        const ChunkIndex& index = *manifest.chunkIndex;
        const uint32_t flags = (manifest.compression ? TSGPU_FLAG_ZSTD : 0u) | (verify ? TSGPU_FLAG_VERIFY : 0u);
        const std::vector<Chunk>& chunks = index.chunks();
        SegmentEncrypt r;
        // the .log object, in windows of chunks
        tsgpu_encrypt_cursor cursor{};
        std::vector<uint32_t> newSizes;
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
            if (k < e) {
                const std::vector<Chunk> part(chunks.begin() + k, chunks.begin() + e);
                for (const Chunk& c : part) tsz.push_back((uint32_t)c.transformedSize);
                const BytesRange range = transformedRange(part);
                if (!range.isEmpty()) bytes = fetcher(range);
            }
            std::vector<uint64_t> windowCrcs;
            std::vector<uint32_t> sizes;
            uint64_t src = 0, obj = 0;
            const Bytes out = call(flags, bytes, tsz, index.originalChunkSize, index.originalFileSize, newKey, ivs + 12 * k, &cursor,
                                   end, sizes, windowCrcs, src, obj, pending.size());
            newSizes.insert(newSizes.end(), sizes.begin(), sizes.end());
            pending.insert(pending.end(), out.begin(), out.end());
            r.objectBytes += out.size();
            crcs.insert(crcs.end(), windowCrcs.begin(), windowCrcs.end());
            size_t c = 0;
            for (; c < crcs.size() && pending.size() >= partSize; c++) emit(partSize, crcs[c]);
            if (end && !pending.empty() && c < crcs.size()) emit(pending.size(), crcs[c++]);
            crcs.erase(crcs.begin(), crcs.begin() + (ptrdiff_t)c);
            if (end) {
                if (!pending.empty() || !crcs.empty()) throw std::runtime_error("part checksums do not match the new object");
                if (crc64) { r.sourceCrc64nvme = src; r.objectCrc64nvme = obj; }
                else { r.sourceCrc32c = (uint32_t)src; r.objectCrc32c = (uint32_t)obj; }
                break;
            }
        }
        r.chunkIndex = finisherChunkIndex(index.originalChunkSize, index.originalFileSize, manifest.compression, true, newSizes.data(),
                                          (uint32_t)newSizes.size());
        // the .indexes object: one call whose chunks are its blobs in object order, back to back from its start (as uploadIndexes
        // lays them out)
        const SegmentIndexesV1& si = manifest.segmentIndexes;
        std::vector<std::pair<IndexType, SegmentIndexV1>> blobs{{IndexType::OFFSET, si.offset}, {IndexType::TIMESTAMP, si.timestamp},
            {IndexType::PRODUCER_SNAPSHOT, si.producerSnapshot}, {IndexType::LEADER_EPOCH, si.leaderEpoch}};
        if (si.transaction) blobs.push_back({IndexType::TRANSACTION, *si.transaction});
        Bytes orderedIvs;
        std::vector<uint32_t> tsz;
        uint64_t at = 0;
        for (size_t i = 0, next = 0; i < blobs.size(); i++) {
            const SegmentIndexV1& b = blobs[i].second;
            if (b.position < 0 || b.size < 0 || (uint64_t)b.position != at)
                throw IllegalArgumentException("the index blobs of SegmentIndexesV1 do not lie back to back from the start of the "
                                               ".indexes object: a blob at " + std::to_string(b.position) + ", " +
                                               std::to_string(at) + " expected");
            at += (uint64_t)b.size;
            Bytes iv(12, 0);                         // an empty blob takes no IV: its 12 bytes are not read
            if (b.size > 0) { std::copy(indexIvs + 12 * next, indexIvs + 12 * (next + 1), iv.begin()); next++; }
            orderedIvs.insert(orderedIvs.end(), iv.begin(), iv.end());
            tsz.push_back((uint32_t)b.size);
        }
        if (at != indexesObject.size())
            throw IllegalArgumentException("the index blobs of SegmentIndexesV1 hold " + std::to_string(at) + " bytes, the .indexes "
                                           "object " + std::to_string(indexesObject.size()));
        tsgpu_encrypt_cursor icur{};
        std::vector<uint32_t> isz;
        uint64_t isrc = 0, iobj = 0;
        r.indexesObject = call(flags & TSGPU_FLAG_VERIFY, indexesObject, tsz, 0, 0, newKey, orderedIvs.data(), &icur, true, isz,
                               r.indexesPartCrcs, isrc, iobj, 0);
        SegmentIndexesV1Builder builder;                 // transformIndex: the new sizes, positions back to back
        for (size_t i = 0; i < blobs.size(); i++) builder.add(blobs[i].first, (int)isz[i]);
        r.segmentIndexes = builder.build();
        if (crc64) { r.indexesSourceCrc64nvme = isrc; r.indexesObjectCrc64nvme = iobj; }
        else { r.indexesSourceCrc32c = (uint32_t)isrc; r.indexesObjectCrc32c = (uint32_t)iobj; }
        return r;
    }

private:
    // One window through tsgpu_encrypt_object[_crc64]: returns the new chunks, `sizes` their sizes, `partCrcs` the CRCs of the
    // parts it completes after `carried` bytes of the open part; src / obj the object words at the end.
    Bytes call(uint32_t flags, const Bytes& bytes, const std::vector<uint32_t>& tsz, int ocs, int ofs, const DataKeyAndAAD* key,
               const uint8_t* ivs, tsgpu_encrypt_cursor* cursor, bool end, std::vector<uint32_t>& sizes,
               std::vector<uint64_t>& partCrcs, uint64_t& src, uint64_t& obj, uint64_t carried) const {
        uint64_t total = 0;
        for (uint32_t t : tsz) total += t ? t + 28 : 0;
        Bytes out(total);
        sizes.assign(tsz.size(), 0);
        const size_t partCap = (carried % partSize + total) / partSize + 1;
        uint32_t nParts = 0;
        int rc;
        if (crc64) {
            partCrcs.assign(partCap, 0);
            rc = tsgpu_encrypt_object_crc64(ctx, flags, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(), (uint32_t)ocs,
                                            (uint64_t)ofs, key->dataKey.data(), key->aad.data(), (uint32_t)key->aad.size(), ivs,
                                            out.data(), out.size(), sizes.data(), partSize, partCrcs.data(), (uint32_t)partCap, &nParts,
                                            cursor, end ? 1 : 0, &src, &obj);
        } else {
            std::vector<uint32_t> c32(partCap);
            uint32_t s32 = 0, o32 = 0;
            rc = tsgpu_encrypt_object(ctx, flags, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(), (uint32_t)ocs,
                                      (uint64_t)ofs, key->dataKey.data(), key->aad.data(), (uint32_t)key->aad.size(), ivs, out.data(),
                                      out.size(), sizes.data(), partSize, c32.data(), (uint32_t)partCap, &nParts, cursor, end ? 1 : 0,
                                      &s32, &o32);
            partCrcs.assign(c32.begin(), c32.end());
            src = s32; obj = o32;
        }
        if (rc == TSGPU_E_ARG) throw IllegalArgumentException(tsgpu_last_error());
        if (rc) throw std::runtime_error(tsgpu_last_error());
        partCrcs.resize(nParts);
        return out;
    }

    tsgpu_ctx* ctx;
    uint64_t partSize;
    uint32_t window;
};

}  // namespace tieredstorage
