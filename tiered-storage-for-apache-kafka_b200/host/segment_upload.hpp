// segment_upload.hpp — the caller side of the copy path (SURVEY.md §8f.4), host-only C++ over the C-ABI.
//
// Mirrors, with the reference's names, argument meaning and error behaviour:
//   core/M/SegmentCompressionChecker.java:37-56      is the first record batch of a log segment compressed?
//   core/M/RemoteStorageManager.java:381-398         requiresCompression (the "compression heuristic")
//   core/M/transform/RateLimitedInputStream.java:36-84   token bucket: capacity = rate, greedy refill of rate tokens/s
//   core/M/RemoteStorageManager.java:401-432         uploadSegmentLog: transform -> rate-limited stream -> uploader
//   storage/s3/M/s3/S3MultiPartOutputStream.java:51-125  fixed-size parts, the last one may be short
// (M = src/main/java/io/aiven/kafka/tieredstorage.)
//
// The record-batch layout and its checksums live in kafka-clients 3.6.0 (build.gradle:110), which is not vendored in
// the reference repository; they are restated here from the published Kafka message format:
//   v2:  baseOffset i64 | batchLength i32 | partitionLeaderEpoch i32 | magic i8 (=2) | crc u32 (CRC-32C of everything
//        after it) | attributes i16 (bits 0-2 = compression codec) | ... 61 bytes of header in all
//   v0/v1: offset i64 | size i32 | crc u32 (CRC-32 of everything after it) | magic i8 | attributes i8 (bits 0-2) | ...
// SegmentCompressionChecker below is plain CPU code and checks the first batch only, as the reference does.  With
// SegmentLogUploader::validateRecords every entry of the segment is checked on the GPU inside the transform call
// (TSGPU_FLAG_VALIDATE_RECORDS, csrc/records.cuh), against the same layout and checksums.
#pragma once
#include <chrono>
#include <cstdint>
#include <cstring>
#include <fstream>
#include <functional>
#include <mutex>
#include <stdexcept>
#include <string>
#include <thread>
#include <vector>

#include "chunk_transform.hpp"

namespace tieredstorage {

struct InvalidRecordBatchException : std::runtime_error { using std::runtime_error::runtime_error; };

namespace detail {
inline uint32_t crcTableEntry(uint32_t i, uint32_t poly) { for (int k = 0; k < 8; k++) i = (i >> 1) ^ (poly & (0u - (i & 1u))); return i; }
inline uint32_t crcReflected(const uint8_t* p, size_t n, uint32_t poly) {
    uint32_t table[256];
    for (uint32_t i = 0; i < 256; i++) table[i] = crcTableEntry(i, poly);
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; i++) c = table[(c ^ p[i]) & 0xff] ^ (c >> 8);
    return ~c;
}
inline uint32_t be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
}  // namespace detail

inline uint32_t crc32c(const uint8_t* p, size_t n) { return detail::crcReflected(p, n, 0x82F63B78u); }   // Castagnoli (record batch v2)
inline uint32_t crc32(const uint8_t* p, size_t n) { return detail::crcReflected(p, n, 0xEDB88320u); }    // IEEE (legacy records)

class SegmentCompressionChecker {
public:
    // `log` = the first bytes of the segment file (the whole first batch must be inside [log, log+n) unless the file
    // itself ends there).  true = compressed.  FileRecords.firstBatch() returns null for a file without one complete
    // batch -> "Record batch is null"; ensureValid() failures -> "Failed to read and validate first batch".
    static bool check(const uint8_t* log, size_t n) {
        constexpr size_t LOG_OVERHEAD = 12, HEADER_UP_TO_MAGIC = 17, RECORD_OVERHEAD_V0 = 14, BATCH_OVERHEAD_V2 = 61;
        if (n < HEADER_UP_TO_MAGIC) throw InvalidRecordBatchException("Record batch is null");
        const int32_t size = (int32_t)detail::be32(log + 8);
        if (size < (int32_t)RECORD_OVERHEAD_V0) throw InvalidRecordBatchException("Failed to read and validate first batch");
        if (n < LOG_OVERHEAD + (size_t)size) throw InvalidRecordBatchException("Record batch is null");     // partial batch at the end
        const size_t total = LOG_OVERHEAD + (size_t)size;
        const int8_t magic = (int8_t)log[16];
        if (magic < 0 || magic > 2) throw InvalidRecordBatchException("Failed to read and validate first batch");
        if (magic == 2) {
            if (total < BATCH_OVERHEAD_V2 || detail::be32(log + 17) != crc32c(log + 21, total - 21))
                throw InvalidRecordBatchException("Failed to read and validate first batch");
            return (log[22] & 0x07) != 0;                    // attributes i16 at 21: the codec is in the low byte
        }
        // magic 0 / 1: crc at 12 over [16, end), attributes at 17
        if (total < LOG_OVERHEAD + RECORD_OVERHEAD_V0 || detail::be32(log + 12) != crc32(log + 16, total - 16))
            throw InvalidRecordBatchException("Failed to read and validate first batch");
        return (log[17] & 0x07) != 0;
    }
    static bool check(const std::string& path) {
        std::ifstream f(path, std::ios::binary);
        if (!f) throw InvalidRecordBatchException("Failed to read and validate first batch");
        std::vector<uint8_t> head(17);
        f.read((char*)head.data(), 17);
        if ((size_t)f.gcount() < 17) throw InvalidRecordBatchException("Record batch is null");
        const int32_t size = (int32_t)detail::be32(head.data() + 8);
        if (size >= 14 && size <= (1 << 30)) {
            head.resize(12 + (size_t)size);
            f.read((char*)head.data() + 17, (std::streamsize)(head.size() - 17));
            head.resize(17 + (size_t)f.gcount());
        }
        return check(head.data(), head.size());
    }
};

// RemoteStorageManager.requiresCompression: a segment whose first batch cannot be validated is uploaded UNcompressed
// (the reference logs a warning and leaves the flag false).
inline bool requiresCompression(bool compressionEnabled, bool compressionHeuristic, const uint8_t* log, size_t n) {
    if (!compressionEnabled) return false;
    if (!compressionHeuristic) return true;
    try { return !SegmentCompressionChecker::check(log, n); } catch (const InvalidRecordBatchException&) { return false; }
}

// Token bucket with Bucket4j's semantics as the reference configures it (rateLimitBucket): capacity `rate` tokens, full at
// start, greedy refill of `rate` tokens per second; a blocking consume RESERVES the tokens (the balance may go negative)
// and sleeps for the deficit; forceAddTokens ignores the capacity.  Clock and sleep are injectable for tests.
class RateLimitBucket {
public:
    static constexpr int MIN_RATE = 16384;                   // RateLimitedInputStream.MIN_RATE on JDK >= 21 (8192 before)
    using Clock = std::function<int64_t()>;                  // nanoseconds, monotonic
    using Sleep = std::function<void(int64_t)>;              // nanoseconds
    explicit RateLimitBucket(int uploadRate, Clock clock = {}, Sleep sleep = {})
        : rate_(std::max(uploadRate, MIN_RATE)), clock_(clock ? clock : Clock(&RateLimitBucket::steadyNanos)),
          sleep_(sleep ? sleep : Sleep(&RateLimitBucket::sleepNanos)), tokens_((double)rate_), last_(clock_()) {}
    int64_t capacity() const { return rate_; }
    // returns the nanoseconds it had to wait
    int64_t consume(int64_t n) {
        if (n <= 0) return 0;
        int64_t wait = 0;
        {
            std::lock_guard<std::mutex> g(mu_);
            refill();
            tokens_ -= (double)n;
            if (tokens_ < 0) wait = (int64_t)(-tokens_ * 1e9 / (double)rate_);
        }
        if (wait > 0) sleep_(wait);
        return wait;
    }
    void forceAddTokens(int64_t n) { std::lock_guard<std::mutex> g(mu_); refill(); tokens_ += (double)n; }
    double availableTokens() { std::lock_guard<std::mutex> g(mu_); refill(); return tokens_; }

private:
    static int64_t steadyNanos() { return std::chrono::duration_cast<std::chrono::nanoseconds>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
    static void sleepNanos(int64_t ns) { std::this_thread::sleep_for(std::chrono::nanoseconds(ns)); }
    void refill() {
        const int64_t now = clock_();
        if (now > last_) {
            // refill never lifts the balance above the capacity, but tokens forced in above it stay
            const double cap = std::max(tokens_, (double)rate_);
            tokens_ = std::min(cap, tokens_ + (double)(now - last_) * (double)rate_ / 1e9);
            last_ = now;
        }
    }
    const int64_t rate_;
    Clock clock_;
    Sleep sleep_;
    std::mutex mu_;
    double tokens_;
    int64_t last_;
};

// S3MultiPartOutputStream: the object goes out in parts of exactly partSize bytes, the last one may be shorter.  With
// SegmentLogUploader::partChecksums a part carries the CRC-32C of its bytes, computed on the GPU (tsgpu_transform_parts).
// With SegmentLogUploader::crc64Parts the part carries the CRC-64/NVME of its bytes instead (tsgpu_transform_parts_crc64).
struct UploadPart {
    int partNumber; uint64_t offset; uint64_t size;
    std::optional<uint32_t> crc32c = std::nullopt;
    std::optional<uint64_t> crc64nvme = std::nullopt;
};
inline std::vector<UploadPart> multipartPlan(uint64_t objectBytes, uint64_t partSize) {
    if (partSize == 0) throw IllegalArgumentException("partSize must be positive");
    std::vector<UploadPart> parts;
    for (uint64_t off = 0; off < objectBytes; off += partSize)
        parts.push_back({(int)parts.size() + 1, off, std::min(partSize, objectBytes - off)});
    return parts;
}

// RemoteStorageManager.uploadSegmentLog, GPU shape: the whole segment goes through ONE tsgpu_transform call (batches are
// pipelined inside), the packed object lands in a pinned buffer, and the uploader is handed finished parts of that
// buffer — it never pulls a stream through the transform.  The rate limiter is charged per part, as the reference's
// stream is charged per read(buf, off, len).
struct SegmentLogUpload {
    std::shared_ptr<ChunkIndex> chunkIndex;
    uint64_t objectBytes = 0;
    bool compressed = false;
    std::vector<int32_t> transformedSizes;
    std::optional<uint32_t> objectCrc32c;                // with partChecksums: CRC-32C of the whole object (S3 FULL_OBJECT, GCS crc32c)
    std::optional<uint64_t> objectCrc64nvme;             // with partChecksums and crc64Parts: CRC-64/NVME of the whole object (S3 CRC64NVME)
};
// The chunk index TransformFinisher builds for a segment of n original bytes in chunks of ocs whose `got` transformed sizes are
// `sizes`: fixed when every chunk has the same known transformed size (ocs, or ocs + 28 encrypted), variable after compression.
inline std::shared_ptr<ChunkIndex> finisherChunkIndex(int ocs, int n, bool compressed, bool encrypted, const uint32_t* sizes,
                                                      uint32_t got) {
    if (got == 0) {                                      // nothing went through the finisher (TransformFinisher.java:112-132)
        if (compressed || encrypted) throw IllegalStateException("Chunk index was not built, was finisher used?");
        return FixedSizeChunkIndexBuilder(ocs, n, ocs).finish(0);
    }
    if (compressed) {
        VariableSizeChunkIndexBuilder b(ocs, n);
        for (uint32_t i = 0; i + 1 < got; i++) b.addChunk((int)sizes[i]);
        return b.finish((int)sizes[got - 1]);
    }
    FixedSizeChunkIndexBuilder b(ocs, n, encrypted ? ocs + 28 : ocs);
    for (uint32_t i = 0; i + 1 < got; i++) b.addChunk((int)sizes[i]);
    return b.finish((int)sizes[got - 1]);
}

class SegmentLogUploader {
public:
    using PartSink = std::function<void(const UploadPart&, const uint8_t* data)>;
    SegmentLogUploader(tsgpu_ctx* ctx, int chunkSize, bool compressionEnabled, bool compressionHeuristic, bool encryptionEnabled,
                       uint64_t partSize, RateLimitBucket* bucket = nullptr)
        : ctx(ctx), chunkSize(chunkSize), compressionEnabled(compressionEnabled), compressionHeuristic(compressionHeuristic),
          encryptionEnabled(encryptionEnabled), partSize(partSize), bucket(bucket) {
        if (!ctx) throw NullPointerException("ctx cannot be null");
        if (chunkSize < 0) throw IllegalArgumentException("originalChunkSize must be non-negative, " + std::to_string(chunkSize) + " given");
    }
    // Check every record batch of the segment before it is uploaded (TSGPU_FLAG_VALIDATE_RECORDS): a damaged batch fails the
    // upload with InvalidRecordBatchException, so the copy is retried and the local segment kept.  It applies when the segment
    // is compressed or encrypted: otherwise the transform is a plain copy on the host and no byte reaches the GPU.
    bool validateRecords = false;
    // Hand every part to the sink with the CRC-32C of its bytes, and the object's CRC-32C in the result, both computed on the GPU
    // from the bytes it copied out (tsgpu_transform_parts with this uploader's partSize): the storage client sends them with the
    // part (S3 x-amz-checksum-crc32c, GCS crc32c; INTEGRATION.md), so damage on any later hop is refused by the object store.
    // Like validateRecords it applies when the segment is compressed or encrypted; otherwise no byte reaches the GPU.
    bool partChecksums = false;
    // With partChecksums: CRC-64/NVME instead of CRC-32C (tsgpu_transform_parts_crc64), for S3's CRC64NVME and, unverified,
    // Azure's x-ms-content-crc64: the parts carry crc64nvme and the result objectCrc64nvme.  The object's bytes are the same.
    bool crc64Parts = false;
    // `log`/`n`: the segment file (ideally in memory from tsgpu_host_alloc); `ivs`: 12 bytes per chunk when encrypting.
    SegmentLogUpload upload(const uint8_t* log, uint64_t n, const DataKeyAndAAD* key, const uint8_t* ivs, const PartSink& sink) {
        if (n > 0x7fffffffull) throw IllegalArgumentException("originalFileSize must fit an int");
        SegmentLogUpload r;
        r.compressed = requiresCompression(compressionEnabled, compressionHeuristic, log, (size_t)n);
        uint32_t flags = (r.compressed ? TSGPU_FLAG_ZSTD : 0u) | (encryptionEnabled ? TSGPU_FLAG_AES : 0u);
        const uint32_t callFlags = flags | (validateRecords && flags ? TSGPU_FLAG_VALIDATE_RECORDS : 0u);
        if (encryptionEnabled) {
            if (!key || !ivs) throw NullPointerException("cipherSupplier cannot be null");
            if (key->dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        }
        const uint32_t cs = (uint32_t)chunkSize;
        const uint64_t bound = tsgpu_transform_bound(flags, n, cs);
        uint8_t* dst = (uint8_t*)tsgpu_host_alloc(bound ? bound : 1);
        if (!dst) throw std::runtime_error("tsgpu_host_alloc failed");
        struct Free { uint8_t* p; ~Free() { tsgpu_host_free(p); } } guard{dst};
        const uint64_t per = cs ? cs : (n ? n : 1);
        uint32_t nChunks = (uint32_t)((n + per - 1) / per);
        std::vector<uint32_t> sizes(nChunks ? nChunks : 1);
        uint32_t got = (uint32_t)sizes.size();
        const bool checksums = partChecksums && flags;
        std::vector<uint32_t> partCrcs;
        std::vector<uint64_t> partCrcs64;
        uint32_t objectCrc = 0;
        uint64_t objectCrc64 = 0;
        int rc;
        if (checksums) {
            if (partSize == 0) throw IllegalArgumentException("partSize must be positive");
            tsgpu_records_cursor records{};
            tsgpu_parts_cursor parts{};
            uint32_t nParts = 0;
            if (crc64Parts) {
                partCrcs64.resize(bound / partSize + 2);
                rc = tsgpu_transform_parts_crc64(ctx, callFlags, log, n, cs, key ? key->dataKey.data() : nullptr,
                                                 key ? key->aad.data() : nullptr, key ? (uint32_t)key->aad.size() : 0u, ivs, dst, bound,
                                                 sizes.data(), &got, &records, 1, partSize, &parts, partCrcs64.data(),
                                                 (uint32_t)partCrcs64.size(), &nParts, &objectCrc64);
                partCrcs64.resize(rc ? 0 : nParts);
            } else {
                partCrcs.resize(bound / partSize + 2);
                rc = tsgpu_transform_parts(ctx, callFlags, log, n, cs, key ? key->dataKey.data() : nullptr, key ? key->aad.data() : nullptr,
                                           key ? (uint32_t)key->aad.size() : 0u, ivs, dst, bound, sizes.data(), &got, &records, 1,
                                           partSize, &parts, partCrcs.data(), (uint32_t)partCrcs.size(), &nParts, &objectCrc);
                partCrcs.resize(rc ? 0 : nParts);
            }
        } else {
            rc = tsgpu_transform(ctx, callFlags, log, n, cs, key ? key->dataKey.data() : nullptr, key ? key->aad.data() : nullptr,
                                 key ? (uint32_t)key->aad.size() : 0u, ivs, dst, bound, sizes.data(), &got);
        }
        if (rc == TSGPU_E_RECORDS) throw InvalidRecordBatchException(tsgpu_last_error());
        if (rc) throw std::runtime_error(tsgpu_last_error());            // RuntimeException in the reference
        const int ocs = chunkSize ? chunkSize : (int)n;
        for (uint32_t i = 0; i < got; i++) { r.transformedSizes.push_back((int32_t)sizes[i]); r.objectBytes += sizes[i]; }
        r.chunkIndex = finisherChunkIndex(ocs, (int)n, r.compressed, encryptionEnabled, sizes.data(), got);
        std::vector<UploadPart> plan = multipartPlan(r.objectBytes, partSize);
        if (checksums && crc64Parts) {
            if (partCrcs64.size() != plan.size()) throw std::runtime_error("part checksums do not match the multipart plan");
            for (size_t i = 0; i < plan.size(); i++) plan[i].crc64nvme = partCrcs64[i];
            r.objectCrc64nvme = objectCrc64;
        } else if (checksums) {
            if (partCrcs.size() != plan.size()) throw std::runtime_error("part checksums do not match the multipart plan");
            for (size_t i = 0; i < plan.size(); i++) plan[i].crc32c = partCrcs[i];
            r.objectCrc32c = objectCrc;
        }
        for (const UploadPart& p : plan) {
            if (bucket) bucket->consume((int64_t)p.size);
            sink(p, dst + p.offset);
        }
        return r;
    }

private:
    tsgpu_ctx* ctx;
    int chunkSize;
    bool compressionEnabled, compressionHeuristic, encryptionEnabled;
    uint64_t partSize;
    RateLimitBucket* bucket;
};

// ------------------------------------------------------------------ index files (SURVEY.md §8f.3)
// RemoteStorageManager.uploadIndexes / transformIndex (RemoteStorageManager.java:287-354, :455-490): every Kafka index is
// ONE chunk (chunking disabled), encryption only; the `.indexes` object is their concatenation in the order OFFSET,
// TIMESTAMP, PRODUCER_SNAPSHOT, LEADER_EPOCH, [TRANSACTION] and SegmentIndexesV1 records (position, size) of each
// transformed blob.  Here the non-empty blobs of a segment ride ONE ragged AES batch (tsgpu_transform_chunks).
enum class IndexType { OFFSET, TIMESTAMP, PRODUCER_SNAPSHOT, LEADER_EPOCH, TRANSACTION };
inline const char* indexTypeName(IndexType t) {
    static const char* N[] = {"OFFSET", "TIMESTAMP", "PRODUCER_SNAPSHOT", "LEADER_EPOCH", "TRANSACTION"};
    return N[(int)t];
}
class SegmentIndexesV1Builder {                      // core/M/manifest/SegmentIndexesV1Builder.java:27-64
public:
    SegmentIndexesV1Builder& add(IndexType type, int size) {
        if (have[(int)type]) throw IllegalStateException(std::string("Index ") + indexTypeName(type) + " is already added");
        have[(int)type] = true; idx[(int)type] = SegmentIndexV1{currentPosition, size};
        currentPosition += size;
        return *this;
    }
    std::string indexes() const {                    // sorted by enum order, like the reference's list
        std::string s = "[";
        for (int t = 0; t < 5; t++) if (have[t]) { if (s.size() > 1) s += ", "; s += indexTypeName((IndexType)t); }
        return s + "]";
    }
    SegmentIndexesV1 build() const {
        int n = 0; for (bool h : have) n += h ? 1 : 0;
        if (n < 4) throw IllegalStateException("Not enough indexes have been added; at least 4 required. Indexes included: " + indexes());
        if (n == 4 && have[(int)IndexType::TRANSACTION]) throw IllegalStateException("OFFSET, TIMESTAMP, PRODUCER_SNAPSHOT, and LEADER_EPOCH indexes are required");
        SegmentIndexesV1 r{idx[0], idx[1], idx[2], idx[3], std::nullopt};
        if (have[4]) r.transaction = idx[4];
        return r;
    }
private:
    bool have[5] = {false, false, false, false, false};
    SegmentIndexV1 idx[5] = {};
    int currentPosition = 0;
};

struct SegmentIndexesUpload { Bytes object; SegmentIndexesV1 segmentIndexes; };
// `blobs`: the index files in the reference's order (the transaction index may be absent); `ivs`: 12 bytes per NON-EMPTY blob.
inline SegmentIndexesUpload uploadIndexes(tsgpu_ctx* ctx, const std::vector<std::pair<IndexType, Bytes>>& blobs, bool encryptionEnabled,
                                          const DataKeyAndAAD* key, const uint8_t* ivs) {
    if (!ctx) throw NullPointerException("ctx cannot be null");
    if (encryptionEnabled && (!key || !ivs)) throw NullPointerException("cipherSupplier cannot be null");
    SegmentIndexesV1Builder builder;
    SegmentIndexesUpload r;
    Bytes src; std::vector<uint32_t> lens;
    for (auto& b : blobs) if (!b.second.empty()) { src.insert(src.end(), b.second.begin(), b.second.end()); lens.push_back((uint32_t)b.second.size()); }
    std::vector<uint32_t> tsz(lens.size());
    if (encryptionEnabled && !lens.empty()) {
        r.object.resize(src.size() + 28 * lens.size());
        const int rc = tsgpu_transform_chunks(ctx, TSGPU_FLAG_AES, src.data(), lens.data(), (uint32_t)lens.size(), key->dataKey.data(), key->aad.data(),
                                              (uint32_t)key->aad.size(), ivs, r.object.data(), r.object.size(), tsz.data());
        if (rc) throw std::runtime_error(tsgpu_last_error());
    } else { r.object = src; tsz = lens; }
    size_t k = 0;
    for (auto& b : blobs) builder.add(b.first, b.second.empty() ? 0 : (int)tsz[k++]);     // transformIndex: size 0 -> empty stream, size 0
    r.segmentIndexes = builder.build();
    return r;
}
// RemoteStorageManager.fetchIndexBytes (:624-652): the index's transformed range of the `.indexes` object, decrypted.
inline Bytes fetchIndexBytes(tsgpu_ctx* ctx, const Bytes& indexesObject, const SegmentIndexV1& index, const DataKeyAndAAD* decryptWith) {
    if (index.size == 0) return Bytes();
    if ((size_t)index.position + (size_t)index.size > indexesObject.size()) throw std::runtime_error("Error fetching index from remote storage");
    const uint8_t* p = indexesObject.data() + index.position;
    if (!decryptWith) return Bytes(p, p + index.size);
    const uint32_t t = (uint32_t)index.size;
    Bytes out((size_t)index.size + 64); uint32_t osz = 0;
    const int rc = tsgpu_detransform(ctx, TSGPU_FLAG_AES, p, t, &t, 1, decryptWith->dataKey.data(), decryptWith->aad.data(), (uint32_t)decryptWith->aad.size(),
                                     out.data(), out.size(), &osz);
    if (rc) throw std::runtime_error(std::string("Error reading de-transformed index bytes: ") + tsgpu_last_error());
    out.resize(osz);
    return out;
}

}  // namespace tieredstorage
