// segment_check.hpp — proof that a stored .log object still decodes to a valid segment, host-only C++ over tsgpu_check_object.
//
// An operator tool or a background job reads the segment's manifest (parseSegmentManifestV1), fetches the object in windows of
// chunks with ranged GETs (as FetchChunkEnumeration fetches a range) and has the GPU check every chunk against the manifest's
// chunk index: GCM tag, zstd frame and Content_Checksum, decoded size, and with validateRecords every record batch.  No plaintext
// comes back to the host; check() returns the CRC-32C of the object (compare with the object store's full-object checksum or the
// one recorded at upload) and of the decoded segment (compare with the local segment file before it is deleted).
#pragma once
#include <algorithm>
#include <cstdint>
#include <stdexcept>
#include <vector>

#include "segment_upload.hpp"

namespace tieredstorage {

struct ObjectCheck { uint32_t objectCrc32c, segmentCrc32c; };
struct ObjectCheck64 { uint64_t objectCrc64nvme, segmentCrc64nvme; };     // check64: CRC-64/NVME (S3 CRC64NVME)

class RemoteSegmentChecker {
public:
    using RangeFetcher = FetchChunkEnumeration::RangeFetcher;       // ObjectFetcher.fetch(key, range) on the .log object
    RemoteSegmentChecker(tsgpu_ctx* ctx, uint32_t windowChunks = 32) : ctx(ctx), window(windowChunks ? windowChunks : 1) {
        if (!ctx) throw NullPointerException("ctx cannot be null");
    }
    bool validateRecords = false;        // also check every record batch of the decoded segment (TSGPU_FLAG_VALIDATE_RECORDS)

    // `key`: the manifest's unwrapped data key and AAD, or null when the manifest has no encryption.  Throws
    // InvalidRecordBatchException for a bad record batch, IllegalArgumentException for arguments the library refuses, and
    // std::runtime_error (RuntimeException in the reference) for a failed tag, a bad frame, a size that disagrees with the index
    // or a short fetch; the message is the library's.
    ObjectCheck check(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const DataKeyAndAAD* key) const {
        ObjectCheck out{0, 0};
        run(manifest, fetcher, key, tsgpu_check_object, &out.objectCrc32c, &out.segmentCrc32c);
        return out;
    }
    // check with the CRC-64/NVME of the object and of the decoded segment (tsgpu_check_object_crc64).
    ObjectCheck64 check64(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const DataKeyAndAAD* key) const {
        ObjectCheck64 out{0, 0};
        run(manifest, fetcher, key, tsgpu_check_object_crc64, &out.objectCrc64nvme, &out.segmentCrc64nvme);
        return out;
    }

private:
    template <typename W, typename Call>
    void run(const SegmentManifestV1& manifest, const RangeFetcher& fetcher, const DataKeyAndAAD* key, Call call, W* objectCrc,
             W* segmentCrc) const {
        if (!fetcher) throw NullPointerException("objectKey cannot be null");
        if (!manifest.chunkIndex) throw NullPointerException("chunkIndex cannot be null");
        const bool encrypted = manifest.aad.has_value();
        if (encrypted && !key) throw NullPointerException("dataKey cannot be null");
        if (encrypted && key->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        const uint32_t flags = (manifest.compression ? TSGPU_FLAG_ZSTD : 0u) | (encrypted ? TSGPU_FLAG_AES : 0u) |
                               (validateRecords ? TSGPU_FLAG_VALIDATE_RECORDS : 0u);
        const ChunkIndex& index = *manifest.chunkIndex;
        const std::vector<Chunk>& chunks = index.chunks();
        tsgpu_check_cursor cursor{};
        for (size_t k = 0;; k += window) {
            const size_t e = std::min(chunks.size(), k + window);
            const bool end = e == chunks.size();
            std::vector<uint32_t> sizes;
            Bytes bytes;
            if (k < e) {
                const std::vector<Chunk> part(chunks.begin() + k, chunks.begin() + e);
                for (const Chunk& c : part) sizes.push_back((uint32_t)c.transformedSize);
                const BytesRange range = transformedRange(part);
                if (!range.isEmpty()) bytes = fetcher(range);
            }
            const int rc = call(ctx, flags, bytes.data(), bytes.size(), sizes.data(), (uint32_t)sizes.size(),
                                              (uint32_t)index.originalChunkSize, (uint64_t)index.originalFileSize,
                                              encrypted ? key->dataKey.data() : nullptr, encrypted ? key->aad.data() : nullptr,
                                              encrypted ? (uint32_t)key->aad.size() : 0u, &cursor, end ? 1 : 0,
                                              objectCrc, segmentCrc);
            if (rc == TSGPU_E_RECORDS) throw InvalidRecordBatchException(tsgpu_last_error());
            if (rc == TSGPU_E_ARG) throw IllegalArgumentException(tsgpu_last_error());
            if (rc) throw std::runtime_error(tsgpu_last_error());
            if (end) return;
        }
    }

    tsgpu_ctx* ctx;
    uint32_t window;
};

}  // namespace tieredstorage
