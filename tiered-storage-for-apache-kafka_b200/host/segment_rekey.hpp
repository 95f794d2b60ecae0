// segment_rekey.hpp — a stored encrypted segment re-encrypted under a new data key, host-only C++ over tsgpu_rekey_object.
//
// An operator tool that must replace an exposed data key reads the segment's manifest (parseSegmentManifestV1), fetches the `.log`
// object in windows of chunks with ranged GETs (as FetchChunkEnumeration fetches a range) and has the GPU check every chunk's old
// tag and re-encrypt it under the new key, with nothing decoded: neither the segment nor an index blob is ever plaintext in host
// memory.  The new `.log` object goes to the part sink in upload parts of partSize bytes, each with its CRC-32C.  The `.indexes`
// object is rekeyed in one call whose chunks are its index blobs at their SegmentIndexV1 positions and sizes.  Every chunk keeps
// its size, so the chunk index and SegmentIndexesV1 are returned unchanged: the caller writes the new manifest with
// segmentManifestV1Json and the new key's encryption metadata, after both new objects are uploaded (INTEGRATION.md).
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include "segment_upload.hpp"

namespace tieredstorage {

struct SegmentRekey {
    std::shared_ptr<ChunkIndex> chunkIndex;      // the manifest's, unchanged
    SegmentIndexesV1 segmentIndexes{};           // the manifest's, unchanged
    uint64_t objectBytes = 0;                    // of the new `.log` object (the old one's)
    Bytes indexesObject;                         // the new `.indexes` object, the old one's size
    // CRC-32C of the old and the new `.log` object (the parts went to the sink), and of the old and the new `.indexes` object with
    // the CRC-32C of its upload parts of partSize bytes.  With RemoteSegmentRekeyer::crc64 these are CRC-64/NVME (S3 CRC64NVME)
    // in the 64-bit fields instead, and the 32-bit ones stay 0.
    uint32_t sourceCrc32c = 0, objectCrc32c = 0, indexesSourceCrc32c = 0, indexesObjectCrc32c = 0;
    uint64_t sourceCrc64nvme = 0, objectCrc64nvme = 0, indexesSourceCrc64nvme = 0, indexesObjectCrc64nvme = 0;
    std::vector<uint64_t> indexesPartCrcs;
};

class RemoteSegmentRekeyer {
public:
    using RangeFetcher = FetchChunkEnumeration::RangeFetcher;       // ObjectFetcher.fetch(key, range) on the old .log object
    using PartSink = SegmentLogUploader::PartSink;
    RemoteSegmentRekeyer(tsgpu_ctx* ctx, uint64_t partSize, uint32_t windowChunks = 32)
        : ctx(ctx), partSize(partSize), window(windowChunks ? windowChunks : 1) {
        if (!ctx) throw NullPointerException("ctx cannot be null");
        if (partSize == 0) throw IllegalArgumentException("partSize must be positive");
    }
    bool verify = false;                 // decrypt every batch again under both keys on the GPU and compare (TSGPU_FLAG_VERIFY)
    // CRC-64/NVME instead of CRC-32C (tsgpu_rekey_object_crc64): every part reaches the sink with crc64nvme, and the result
    // carries the 64-bit words.  The new objects' bytes are the same.
    bool crc64 = false;

    // `oldKey`: the manifest's unwrapped data key and AAD; `newKey`: the new ones.  `ivs`: 12 random bytes per chunk of the
    // segment and `indexIvs` 12 per non-empty index blob, in SegmentIndexesV1 order (offset, timestamp, producer snapshot, leader
    // epoch, transaction), under newKey.  Throws IllegalArgumentException for a manifest without encryption and for arguments the
    // library refuses (among them an IV of the old object reused when newKey is oldKey), and std::runtime_error for a failed tag,
    // a new chunk that did not read back or a short fetch; the message is the library's.  Parts already handed to the sink
    // belong to an upload the caller then aborts.
    SegmentRekey rekey(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const Bytes& indexesObject,
                       const DataKeyAndAAD* oldKey, const DataKeyAndAAD* newKey, const uint8_t* ivs, const uint8_t* indexIvs,
                       const PartSink& sink) const {
        if (!manifest.aad.has_value()) throw IllegalArgumentException("the segment is not encrypted: there is no data key to rotate");
        if (!fetcher) throw NullPointerException("objectKey cannot be null");
        if (!manifest.chunkIndex) throw NullPointerException("chunkIndex cannot be null");
        if (!oldKey || !newKey) throw NullPointerException("dataKey cannot be null");
        if (oldKey->dataKey.size() != 32 || newKey->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        if (!ivs || !indexIvs) throw NullPointerException("ivs cannot be null");
        const uint32_t flags = verify ? TSGPU_FLAG_VERIFY : 0u;
        const std::vector<Chunk>& chunks = manifest.chunkIndex->chunks();
        SegmentRekey r;
        r.chunkIndex = manifest.chunkIndex;
        r.segmentIndexes = manifest.segmentIndexes;
        // the .log object, in windows of chunks
        tsgpu_rekey_cursor cursor{};
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
            Bytes out(bytes.size());
            std::vector<uint64_t> windowCrcs;
            uint64_t src = 0, obj = 0;
            call(flags, bytes, tsz, oldKey, newKey, ivs + 12 * k, out, &cursor, end, windowCrcs, src, obj, pending.size());
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
        // the .indexes object: one call whose chunks are its blobs in object order, back to back from its start (as uploadIndexes
        // lays them out)
        const SegmentIndexesV1& si = manifest.segmentIndexes;
        std::vector<SegmentIndexV1> blobs{si.offset, si.timestamp, si.producerSnapshot, si.leaderEpoch};
        if (si.transaction) blobs.push_back(*si.transaction);
        Bytes blobIvs(12 * blobs.size(), 0);        // an empty blob takes no IV: its 12 bytes are not read
        for (size_t i = 0, next = 0; i < blobs.size(); i++)
            if (blobs[i].size > 0) { std::copy(indexIvs + 12 * next, indexIvs + 12 * (next + 1), blobIvs.begin() + 12 * i); next++; }
        std::vector<size_t> order(blobs.size());
        for (size_t i = 0; i < order.size(); i++) order[i] = i;
        std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return blobs[a].position < blobs[b].position; });
        Bytes orderedIvs;
        std::vector<uint32_t> tsz;
        uint64_t at = 0;
        for (size_t i : order) {
            if (blobs[i].position < 0 || blobs[i].size < 0 || (uint64_t)blobs[i].position != at)
                throw IllegalArgumentException("the index blobs of SegmentIndexesV1 do not lie back to back from the start of the "
                                               ".indexes object: a blob at " + std::to_string(blobs[i].position) + ", " +
                                               std::to_string(at) + " expected");
            at += (uint64_t)blobs[i].size;
            orderedIvs.insert(orderedIvs.end(), blobIvs.begin() + 12 * i, blobIvs.begin() + 12 * (i + 1));
            tsz.push_back((uint32_t)blobs[i].size);
        }
        if (at != indexesObject.size())
            throw IllegalArgumentException("the index blobs of SegmentIndexesV1 hold " + std::to_string(at) + " bytes, the .indexes "
                                           "object " + std::to_string(indexesObject.size()));
        r.indexesObject.assign(indexesObject.size(), 0);
        tsgpu_rekey_cursor icur{};
        uint64_t isrc = 0, iobj = 0;
        call(flags, indexesObject, tsz, oldKey, newKey, orderedIvs.data(), r.indexesObject, &icur, true, r.indexesPartCrcs, isrc, iobj, 0);
        if (crc64) { r.indexesSourceCrc64nvme = isrc; r.indexesObjectCrc64nvme = iobj; }
        else { r.indexesSourceCrc32c = (uint32_t)isrc; r.indexesObjectCrc32c = (uint32_t)iobj; }
        return r;
    }

private:
    // One window through tsgpu_rekey_object[_crc64]: `out` (bytes.size() bytes) receives the new chunks, `partCrcs` the CRCs of the
    // parts it completes after `carried` bytes of the open part; src / obj the object words at the end.
    void call(uint32_t flags, const Bytes& bytes, const std::vector<uint32_t>& tsz, const DataKeyAndAAD* oldKey,
              const DataKeyAndAAD* newKey, const uint8_t* ivs, Bytes& out, tsgpu_rekey_cursor* cursor, bool end,
              std::vector<uint64_t>& partCrcs, uint64_t& src, uint64_t& obj, uint64_t carried) const {
        const size_t partCap = (carried % partSize + bytes.size()) / partSize + 1;
        uint32_t nParts = 0;
        int rc;
        if (crc64) {
            partCrcs.assign(partCap, 0);
            rc = tsgpu_rekey_object_crc64(ctx, flags, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(),
                                          oldKey->dataKey.data(), oldKey->aad.data(), (uint32_t)oldKey->aad.size(), newKey->dataKey.data(),
                                          newKey->aad.data(), (uint32_t)newKey->aad.size(), ivs, out.data(), out.size(), partSize,
                                          partCrcs.data(), (uint32_t)partCap, &nParts, cursor, end ? 1 : 0, &src, &obj);
        } else {
            std::vector<uint32_t> c32(partCap);
            uint32_t s32 = 0, o32 = 0;
            rc = tsgpu_rekey_object(ctx, flags, bytes.data(), bytes.size(), tsz.data(), (uint32_t)tsz.size(), oldKey->dataKey.data(),
                                    oldKey->aad.data(), (uint32_t)oldKey->aad.size(), newKey->dataKey.data(), newKey->aad.data(),
                                    (uint32_t)newKey->aad.size(), ivs, out.data(), out.size(), partSize, c32.data(), (uint32_t)partCap,
                                    &nParts, cursor, end ? 1 : 0, &s32, &o32);
            partCrcs.assign(c32.begin(), c32.end());
            src = s32; obj = o32;
        }
        if (rc == TSGPU_E_ARG) throw IllegalArgumentException(tsgpu_last_error());
        if (rc) throw std::runtime_error(tsgpu_last_error());
        partCrcs.resize(nParts);
    }

    tsgpu_ctx* ctx;
    uint64_t partSize;
    uint32_t window;
};

}  // namespace tieredstorage
