// chunk_transform.hpp — host side above the C-ABI: a C++ mirror of the reference's operator surface for this path
// (the reference is Java and there is no JVM in the build image; the JNI binding of the same C-ABI is in jni/).
// Same names, argument meaning and error behaviour as
//   core/M/transform/{BaseTransform,Compression,Encryption}ChunkEnumeration.java, TransformFinisher.java,
//   core/M/transform/{BaseDetransform,Decryption,Decompression}ChunkEnumeration.java, DetransformFinisher.java,
//   core/M/manifest/index/{AbstractChunkIndexBuilder,FixedSizeChunkIndexBuilder,VariableSizeChunkIndexBuilder}.java,
//   core/M/manifest/index/{AbstractChunkIndex,FixedSizeChunkIndex,VariableSizeChunkIndex}.java, core/M/Chunk.java,
//   core/M/fetch/FetchChunkEnumeration.java
// (core/M = <reference>/core/src/main/java/io/aiven/kafka/tieredstorage).
//
// Difference that makes it GPU-native: the reference pulls ONE chunk through the decorator chain per
// nextElement(); here the outermost enumeration pulls a BATCH of original chunks from the base enumeration,
// hands the whole batch to tsgpu_transform / tsgpu_detransform once, and then serves the results one at a time.
// The decorators only contribute their flag, key material and transformedChunkSize() arithmetic.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <functional>
#include <sstream>
#include <istream>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/tsgpu.h"

namespace tieredstorage {

using Bytes = std::vector<uint8_t>;
struct NoSuchElementException : std::runtime_error { NoSuchElementException() : std::runtime_error("NoSuchElementException") {} };
struct IllegalArgumentException : std::invalid_argument { using std::invalid_argument::invalid_argument; };
struct IllegalStateException : std::logic_error { using std::logic_error::logic_error; };
struct NullPointerException : std::invalid_argument { using std::invalid_argument::invalid_argument; };

// ------------------------------------------------------------------ core/M/Chunk.java:21-36
struct Chunk {
    int id, originalPosition, originalSize, transformedPosition, transformedSize;
    bool operator==(const Chunk& o) const {
        return id == o.id && originalPosition == o.originalPosition && originalSize == o.originalSize &&
               transformedPosition == o.transformedPosition && transformedSize == o.transformedSize;
    }
    // Chunk.range(): inclusive byte range of the transformed chunk inside the object
    std::pair<int, int> range() const { return {transformedPosition, transformedPosition + transformedSize - 1}; }
};

// ------------------------------------------------------------------ AbstractChunkIndex.java:27-152
class ChunkIndex {
public:
    virtual ~ChunkIndex() = default;
    const std::vector<Chunk>& chunks() const { return chunks_; }
    // findChunkForOriginalOffset :75-110 — nullopt is the reference's `null`
    std::optional<Chunk> findChunkForOriginalOffset(int offset) const {
        if (offset < 0) throw IllegalArgumentException("Offset must be non-negative, " + std::to_string(offset) + " given");
        if (offset >= originalFileSize) return std::nullopt;
        int chunkI = 0, op = 0, tp = 0;
        for (; chunkI < chunkCount; chunkI++) {
            const long long beyond = (long long)(chunkI + 1) * originalChunkSize;
            if (offset < beyond) break;
            op += originalChunkSizeAt(chunkI); tp += transformedChunkSizeAt(chunkI);
        }
        return Chunk{chunkI, op, originalChunkSizeAt(chunkI), tp, transformedChunkSizeAt(chunkI)};
    }
    // chunksForRange :113-123 (BytesRange is inclusive on both ends)
    std::vector<Chunk> chunksForRange(int first, int last) const {
        std::vector<Chunk> r;
        Chunk cur{};
        for (long long i = first; i <= last && i < originalFileSize; i += cur.originalSize) {
            cur = *findChunkForOriginalOffset((int)i);
            r.push_back(cur);
        }
        return r;
    }
    // ctx != nullptr: a variable index's transformedChunks is compressed like the reference compresses it
    // (TransformedChunksSerializer.java:40-48; tsgpu_chunk_index_json_ctx) instead of framed as a Raw block
    virtual std::string toJson(tsgpu_ctx* ctx = nullptr) const = 0;
    const int originalChunkSize, originalFileSize, finalTransformedChunkSize, chunkCount;

protected:
    ChunkIndex(int ocs, int ofs, int ftcs, int count)
        : originalChunkSize(checkPositive(ocs, "Original chunk size")), originalFileSize(checkNonNeg(ofs, "Original file size")),
          finalTransformedChunkSize(checkNonNeg(ftcs, "Final transformed chunk size")), chunkCount(count) {}
    static int checkNonNeg(int v, const char* name) {
        if (v < 0) throw IllegalArgumentException(std::string(name) + " must be non-negative, " + std::to_string(v) + " given");
        return v;
    }
    static int checkPositive(int v, const char* name) {
        if (v <= 0) throw IllegalArgumentException(std::string(name) + " must be positive, " + std::to_string(v) + " given");
        return v;
    }
    int originalChunkSizeAt(int i) const { return i == chunkCount - 1 ? originalFileSize - (chunkCount - 1) * originalChunkSize : originalChunkSize; }
    virtual int transformedChunkSizeAt(int i) const = 0;
    void materializeChunks() {       // :52-72
        chunks_.clear();
        if (chunkCount == 0) { chunks_.push_back(Chunk{0, 0, 0, 0, 0}); return; }
        int op = 0, tp = 0;
        for (int i = 0; i < chunkCount; i++) {
            Chunk c{i, op, originalChunkSizeAt(i), tp, transformedChunkSizeAt(i)};
            chunks_.push_back(c);
            op += c.originalSize; tp += c.transformedSize;
        }
    }
    std::vector<Chunk> chunks_;
};

inline std::string jsonFromAbi(int ocs, int ofs, int tcs, int ftcs, const std::vector<int32_t>* sizes, tsgpu_ctx* ctx = nullptr) {
    std::vector<char> buf(1024 + (sizes ? sizes->size() * 8 : 0));
    uint32_t n = (uint32_t)buf.size();
    const int32_t* sp = sizes ? sizes->data() : nullptr;
    const uint32_t sn = sizes ? (uint32_t)sizes->size() : 0;
    int rc = ctx ? tsgpu_chunk_index_json_ctx(ctx, ocs, ofs, tcs, ftcs, sp, sn, buf.data(), &n)
                 : tsgpu_chunk_index_json(ocs, ofs, tcs, ftcs, sp, sn, buf.data(), &n);
    if (rc) throw IllegalArgumentException(tsgpu_last_error());
    return std::string(buf.data(), n);
}

class FixedSizeChunkIndex : public ChunkIndex {       // FixedSizeChunkIndex.java:45-120
public:
    FixedSizeChunkIndex(int ocs, int ofs, int tcs, int ftcs)
        : ChunkIndex(ocs, ofs, ftcs, count(ocs, ofs)), transformedChunkSize(checkNonNeg(tcs, "Transformed chunk size")) { materializeChunks(); }
    const int transformedChunkSize;
    std::string toJson(tsgpu_ctx* = nullptr) const override { return jsonFromAbi(originalChunkSize, originalFileSize, transformedChunkSize, finalTransformedChunkSize, nullptr); }
protected:
    int transformedChunkSizeAt(int i) const override { return i == chunkCount - 1 ? finalTransformedChunkSize : transformedChunkSize; }
private:
    static int count(int ocs, int ofs) { checkPositive(ocs, "Original chunk size"); return ofs % ocs == 0 ? ofs / ocs : ofs / ocs + 1; }
};

class VariableSizeChunkIndex : public ChunkIndex {    // VariableSizeChunkIndex.java:49-110
public:
    VariableSizeChunkIndex(int ocs, int ofs, std::vector<int32_t> sizes)
        : ChunkIndex(ocs, ofs, last(sizes), (int)sizes.size()), transformedChunks(std::move(sizes)) { materializeChunks(); }
    const std::vector<int32_t> transformedChunks;
    std::string toJson(tsgpu_ctx* ctx = nullptr) const override { return jsonFromAbi(originalChunkSize, originalFileSize, -1, 0, &transformedChunks, ctx); }
protected:
    int transformedChunkSizeAt(int i) const override { return transformedChunks[i]; }
private:
    static int last(const std::vector<int32_t>& s) { if (s.empty()) throw NullPointerException("transformedChunks cannot be null"); return s.back(); }
};

// ------------------------------------------------------------------ AbstractChunkIndexBuilder.java:19-97
class AbstractChunkIndexBuilder {
public:
    virtual ~AbstractChunkIndexBuilder() = default;
    void addChunk(int transformedChunkSize) {
        if (finished) throw IllegalStateException("Cannot add chunk to already finished index");
        checkSize(transformedChunkSize, "Transformed chunk size");
        if (remainOfOriginalFileSize() <= originalChunkSize) throw IllegalStateException("This must be final chunk. Call `finish` instead.");
        addChunk0(transformedChunkSize);
        chunksAdded += 1;
    }
    std::shared_ptr<ChunkIndex> finish(int finalTransformedChunkSize) {
        if (finished) throw IllegalStateException("Cannot finish already finished index");
        checkSize(finalTransformedChunkSize, "Transformed chunk size");
        if (remainOfOriginalFileSize() > originalChunkSize)
            throw IllegalStateException("This cannot be final chunk: not enough chunks to cover original file. Call `addChunk` instead.");
        auto r = finish0(finalTransformedChunkSize);
        chunksAdded += 1; finished = true;
        return r;
    }
protected:
    AbstractChunkIndexBuilder(int ocs, int ofs) : originalChunkSize(checkSize(ocs, "Original chunk size")), originalFileSize(checkSize(ofs, "Original file size")) {}
    virtual void addChunk0(int) = 0;
    virtual std::shared_ptr<ChunkIndex> finish0(int) = 0;
    static int checkSize(int v, const char* name) {
        if (v < 0) throw IllegalArgumentException(std::string(name) + " must be non-negative, " + std::to_string(v) + " given");
        return v;
    }
    int remainOfOriginalFileSize() const { return originalFileSize - chunksAdded * originalChunkSize; }
    const int originalChunkSize, originalFileSize;
private:
    int chunksAdded = 0;
    bool finished = false;
};
class FixedSizeChunkIndexBuilder : public AbstractChunkIndexBuilder {     // FixedSizeChunkIndexBuilder.java:19-45
public:
    FixedSizeChunkIndexBuilder(int ocs, int ofs, int tcs) : AbstractChunkIndexBuilder(ocs, ofs), transformedChunkSize(checkSize(tcs, "Transformed chunk size")) {}
protected:
    void addChunk0(int t) override {
        if (t != transformedChunkSize)
            throw IllegalArgumentException("Non-final chunk must be of size " + std::to_string(transformedChunkSize) + ", but " + std::to_string(t) + " given");
    }
    std::shared_ptr<ChunkIndex> finish0(int ft) override { return std::make_shared<FixedSizeChunkIndex>(originalChunkSize, originalFileSize, transformedChunkSize, ft); }
private:
    const int transformedChunkSize;
};
class VariableSizeChunkIndexBuilder : public AbstractChunkIndexBuilder {  // VariableSizeChunkIndexBuilder.java:21-43
public:
    VariableSizeChunkIndexBuilder(int ocs, int ofs) : AbstractChunkIndexBuilder(ocs, ofs) {}
protected:
    void addChunk0(int t) override { sizes.push_back(t); }
    std::shared_ptr<ChunkIndex> finish0(int ft) override { sizes.push_back(ft); return std::make_shared<VariableSizeChunkIndex>(originalChunkSize, originalFileSize, sizes); }
private:
    std::vector<int32_t> sizes;
};

// ------------------------------------------------------------------ key material (AesEncryptionProvider.java:52-75)
struct DataKeyAndAAD { Bytes dataKey /*32*/; Bytes aad; };
// The reference draws a fresh 12-byte IV per chunk from SecureRandom.getInstanceStrong(); the host supplies it.
using IvSupplier = std::function<void(uint8_t iv[TSGPU_IV_SIZE])>;

// ------------------------------------------------------------------ TransformChunkEnumeration.java:28-42
class TransformChunkEnumeration {
public:
    virtual ~TransformChunkEnumeration() = default;
    virtual int originalChunkSize() const = 0;
    virtual std::optional<int> transformedChunkSize() const = 0;     // nullopt = variable (Java null)
    virtual bool hasMoreElements() = 0;
    virtual Bytes nextElement() = 0;
    // --- batching plumbing (not in the reference)
    virtual TransformChunkEnumeration* innerEnumeration() { return nullptr; }
    virtual uint32_t flag() const { return 0; }
    virtual const DataKeyAndAAD* keyMaterial() const { return nullptr; }
    virtual const IvSupplier* ivSupplier() const { return nullptr; }
};

// BaseTransformChunkEnumeration.java:29-98
class BaseTransformChunkEnumeration : public TransformChunkEnumeration {
public:
    BaseTransformChunkEnumeration(std::istream* inputStream, int originalChunkSize) : in(inputStream), ocs(originalChunkSize) {
        if (!inputStream) throw NullPointerException("inputStream cannot be null");
        if (originalChunkSize < 0) throw IllegalArgumentException("originalChunkSize must be non-negative, " + std::to_string(originalChunkSize) + " given");
    }
    int originalChunkSize() const override { return ocs; }
    std::optional<int> transformedChunkSize() const override { return ocs; }
    bool hasMoreElements() override { fill(); return !chunk->empty(); }
    Bytes nextElement() override {
        fill();
        if (chunk->empty()) throw NoSuchElementException();
        Bytes r = std::move(*chunk); chunk.reset(); return r;
    }
private:
    void fill() {
        if (chunk) return;
        chunk = Bytes();
        if (ocs != 0) { chunk->resize((size_t)ocs); in->read((char*)chunk->data(), ocs); chunk->resize((size_t)in->gcount()); }
        else { char buf[65536]; while (in->read(buf, sizeof buf) || in->gcount()) chunk->insert(chunk->end(), buf, buf + in->gcount()); }
    }
    std::istream* in; int ocs; std::optional<Bytes> chunk;
};

// Shared batching core of the decorators.
class GpuBatchingEnumeration : public TransformChunkEnumeration {
public:
    bool hasMoreElements() override { return !ready.empty() || base()->hasMoreElements(); }
    Bytes nextElement() override {
        if (ready.empty()) pump();
        if (ready.empty()) throw NoSuchElementException();
        Bytes r = std::move(ready.front()); ready.erase(ready.begin()); return r;
    }
    TransformChunkEnumeration* innerEnumeration() override { return inner; }
    int originalChunkSize() const override { return inner->originalChunkSize(); }
protected:
    GpuBatchingEnumeration(tsgpu_ctx* c, TransformChunkEnumeration* in, uint32_t batchChunks) : ctx(c), inner(in), batch(batchChunks ? batchChunks : 1) {
        if (!in) throw NullPointerException("inner cannot be null");
    }
    tsgpu_ctx* ctx; TransformChunkEnumeration* inner; uint32_t batch;
private:
    TransformChunkEnumeration* base() { TransformChunkEnumeration* e = this; while (e->innerEnumeration()) e = e->innerEnumeration(); return e; }
    void pump() {
        uint32_t flags = 0; const DataKeyAndAAD* km = nullptr; const IvSupplier* ivs = nullptr;
        for (TransformChunkEnumeration* e = this; e; e = e->innerEnumeration()) {
            flags |= e->flag();
            if (e->keyMaterial()) km = e->keyMaterial();
            if (e->ivSupplier()) ivs = e->ivSupplier();
        }
        TransformChunkEnumeration* b = base();
        Bytes src; std::vector<uint32_t> lens;
        while (lens.size() < batch && b->hasMoreElements()) { Bytes c = b->nextElement(); lens.push_back((uint32_t)c.size()); src.insert(src.end(), c.begin(), c.end()); }
        if (lens.empty()) return;
        const uint32_t cs = lens.front();                  // every non-final chunk has the base chunk size
        Bytes iv(lens.size() * TSGPU_IV_SIZE);
        if (flags & TSGPU_FLAG_AES) for (size_t i = 0; i < lens.size(); i++) (*ivs)(iv.data() + i * TSGPU_IV_SIZE);
        Bytes dst((size_t)tsgpu_transform_bound(flags, src.size(), cs) + 64);
        std::vector<uint32_t> sizes(lens.size());
        uint32_t n = (uint32_t)sizes.size();
        int rc = tsgpu_transform(ctx, flags, src.data(), src.size(), cs, km ? km->dataKey.data() : nullptr, km ? km->aad.data() : nullptr,
                                 km ? (uint32_t)km->aad.size() : 0, iv.data(), dst.data(), dst.size(), sizes.data(), &n);
        if (rc) throw std::runtime_error(tsgpu_last_error());      // RuntimeException in the reference
        size_t pos = 0;
        for (uint32_t i = 0; i < n; i++) { ready.emplace_back(dst.begin() + pos, dst.begin() + pos + sizes[i]); pos += sizes[i]; }
    }
    std::vector<Bytes> ready;
};

// CompressionChunkEnumeration.java:26-63
class CompressionChunkEnumeration : public GpuBatchingEnumeration {
public:
    CompressionChunkEnumeration(tsgpu_ctx* ctx, TransformChunkEnumeration* inner, uint32_t batchChunks = 32) : GpuBatchingEnumeration(ctx, inner, batchChunks) {}
    std::optional<int> transformedChunkSize() const override { return std::nullopt; }   // variable
    uint32_t flag() const override { return TSGPU_FLAG_ZSTD; }
};

// EncryptionChunkEnumeration.java:30-85
class EncryptionChunkEnumeration : public GpuBatchingEnumeration {
public:
    EncryptionChunkEnumeration(tsgpu_ctx* ctx, TransformChunkEnumeration* inner, DataKeyAndAAD keyAndAad, IvSupplier ivSupplier, uint32_t batchChunks = 32)
        : GpuBatchingEnumeration(ctx, inner, batchChunks), km(std::move(keyAndAad)), ivs(std::move(ivSupplier)) {
        if (!ivs) throw NullPointerException("cipherSupplier cannot be null");
        if (km.dataKey.size() != 32) throw IllegalArgumentException("dataKey must be 32 bytes");
        auto in = inner->transformedChunkSize();
        if (in) tcs = TSGPU_IV_SIZE + *in + TSGPU_TAG_SIZE;          // encryptedChunkSize :82-84 (ivSize + getOutputSize(n))
    }
    std::optional<int> transformedChunkSize() const override { return tcs; }
    uint32_t flag() const override { return TSGPU_FLAG_AES; }
    const DataKeyAndAAD* keyMaterial() const override { return &km; }
    const IvSupplier* ivSupplier() const override { return &ivs; }
private:
    DataKeyAndAAD km; IvSupplier ivs; std::optional<int> tcs;
};

// TransformFinisher.java:47-199 (without the rate limiter, which wraps the resulting stream in the reference)
class TransformFinisher {
public:
    TransformFinisher(TransformChunkEnumeration* inner, int originalFileSize, bool chunkingEnabled = true) : inner(inner), originalFileSize(originalFileSize) {
        if (!inner) throw NullPointerException("inner cannot be null");
        if (originalFileSize < 0) throw IllegalArgumentException("originalFileSize must be non-negative, " + std::to_string(originalFileSize) + " given");
        const int ocs = chunkingEnabled ? inner->originalChunkSize() : originalFileSize;
        auto t = inner->transformedChunkSize();
        if (!t) builder = std::make_unique<VariableSizeChunkIndexBuilder>(ocs, originalFileSize);
        else builder = std::make_unique<FixedSizeChunkIndexBuilder>(ocs, originalFileSize, *t);
    }
    bool hasMoreElements() { return inner->hasMoreElements(); }
    Bytes nextElement() {                                    // :101-110
        Bytes chunk = inner->nextElement();
        if (hasMoreElements()) builder->addChunk((int)chunk.size());
        else index = builder->finish((int)chunk.size());
        return chunk;
    }
    std::shared_ptr<ChunkIndex> chunkIndex() {               // :112-132
        if (!index) {
            if (dynamic_cast<BaseTransformChunkEnumeration*>(inner)) {
                const int cs = *inner->transformedChunkSize();
                int size = originalFileSize;
                while (size > cs) { builder->addChunk(cs); size -= cs; }
                index = builder->finish(size);
            } else throw IllegalStateException("Chunk index was not built, was finisher used?");
        }
        return index;
    }
    Bytes readAll() { Bytes all; while (hasMoreElements()) { Bytes c = nextElement(); all.insert(all.end(), c.begin(), c.end()); } return all; }   // SequenceInputStream
private:
    TransformChunkEnumeration* inner; int originalFileSize;
    std::unique_ptr<AbstractChunkIndexBuilder> builder; std::shared_ptr<ChunkIndex> index;
};

// ------------------------------------------------------------------ detransform side
// DefaultChunkManager.getChunk (DefaultChunkManager.java:50-70) generalised to a list of consecutive chunks:
// BaseDetransform (cut at transformedSize; "Stream has fewer bytes than expected") -> Decryption -> Decompression.
class DetransformChunkEnumeration {
public:
    DetransformChunkEnumeration(tsgpu_ctx* ctx, std::istream* inputStream, std::vector<Chunk> chunks, bool decompress,
                                const DataKeyAndAAD* decryptWith, uint32_t maxOriginalChunkSize, uint32_t batchChunks = 32)
        : ctx(ctx), in(inputStream), chunks(std::move(chunks)), flags((decompress ? TSGPU_FLAG_ZSTD : 0) | (decryptWith ? TSGPU_FLAG_AES : 0)),
          ocs(maxOriginalChunkSize), batch(batchChunks ? batchChunks : 1) {
        if (!inputStream) throw NullPointerException("inputStream cannot be null");
        if (decryptWith) km = *decryptWith;
    }
    bool hasMoreElements() { return !ready.empty() || next < chunks.size(); }
    Bytes nextElement() {
        if (ready.empty()) pump();
        if (ready.empty()) throw NoSuchElementException();
        Bytes r = std::move(ready.front()); ready.erase(ready.begin()); return r;
    }
private:
    void pump() {
        std::vector<uint32_t> ts;
        Bytes src;
        while (ts.size() < batch && next < chunks.size()) {
            const uint32_t t = (uint32_t)chunks[next++].transformedSize;
            const size_t at = src.size();
            src.resize(at + t);
            in->read((char*)src.data() + at, t);
            if ((uint32_t)in->gcount() < t) throw std::runtime_error("Stream has fewer bytes than expected");
            ts.push_back(t);
        }
        if (ts.empty()) return;
        Bytes dst((size_t)ocs * ts.size() + 64);
        std::vector<uint32_t> osz(ts.size());
        int rc = tsgpu_detransform(ctx, flags, src.data(), src.size(), ts.data(), (uint32_t)ts.size(), km.dataKey.empty() ? nullptr : km.dataKey.data(),
                                   km.aad.data(), (uint32_t)km.aad.size(), dst.data(), dst.size(), osz.data());
        if (rc) throw std::runtime_error(tsgpu_last_error());
        size_t pos = 0;
        for (size_t i = 0; i < ts.size(); i++) { ready.emplace_back(dst.begin() + pos, dst.begin() + pos + osz[i]); pos += osz[i]; }
    }
    tsgpu_ctx* ctx; std::istream* in; std::vector<Chunk> chunks; uint32_t flags; uint32_t ocs; uint32_t batch; size_t next = 0;
    DataKeyAndAAD km; std::vector<Bytes> ready;
};

// DetransformFinisher.java:30-55: the enumeration of byte[] as ONE stream of original bytes (the reference concatenates
// ByteArrayInputStreams in a SequenceInputStream; with no transform at all the input stream is passed through untouched).
class DetransformFinisher {
public:
    explicit DetransformFinisher(DetransformChunkEnumeration* inner) : inner(inner) {
        if (!inner) throw NullPointerException("inner cannot be null");
    }
    bool hasMoreElements() { return inner->hasMoreElements(); }
    Bytes nextElement() { return inner->nextElement(); }
    Bytes readAll() { Bytes all; while (hasMoreElements()) { Bytes c = nextElement(); all.insert(all.end(), c.begin(), c.end()); } return all; }
private:
    DetransformChunkEnumeration* inner;
};

// storage/core/src/main/java/io/aiven/kafka/tieredstorage/storage/BytesRange.java:26-113: inclusive on both ends, `to == -1`
// is the empty range.
struct BytesRange {
    int from, to;
    static BytesRange of(int from, int to) {
        if (from < 0) throw IllegalArgumentException("from cannot be negative, " + std::to_string(from) + " given");
        if (to != -1 && to < from)
            throw IllegalArgumentException("to cannot be less than from, from=" + std::to_string(from) + ", to=" + std::to_string(to) + " given");
        return BytesRange{from, to};
    }
    static BytesRange empty(int from) { return of(from, -1); }
    static BytesRange ofFromPositionAndSize(int from, int size) { return size == 0 ? empty(from) : of(from, from + size - 1); }
    int firstPosition() const { return from; }
    bool isEmpty() const { return to == -1; }
    int lastPosition() const { if (isEmpty()) throw IllegalStateException("No last position, range is empty"); return to; }
    int size() const { return isEmpty() ? 0 : to - from + 1; }
    bool operator==(const BytesRange& o) const { return from == o.from && to == o.to; }
    std::string toString() const { return "BytesRange{position=" + std::to_string(from) + ", size=" + std::to_string(size()) + "}"; }
};
// The ONE ranged GET that covers consecutive chunks (what a batched DefaultChunkManager issues, SURVEY.md §8f.1): from the
// first chunk's transformed position to the last chunk's last transformed byte (Chunk.range(), core/M/Chunk.java:21-36).
inline BytesRange transformedRange(const std::vector<Chunk>& consecutive) {
    if (consecutive.empty()) throw IllegalArgumentException("no chunks");
    const Chunk& a = consecutive.front(); const Chunk& b = consecutive.back();
    return BytesRange::of(a.transformedPosition, b.transformedPosition + b.transformedSize - 1);
}

// FetchChunkEnumeration.java:54-138: which chunks cover [from, to] and how much of the first / last one to keep.
struct FetchPiece { int chunkId, skip, take; };
inline std::vector<FetchPiece> fetchPlan(const ChunkIndex& index, int from, int to) {
    if (to < from) throw IllegalArgumentException("range cannot be empty");
    auto first = index.findChunkForOriginalOffset(from);
    if (!first) throw IllegalArgumentException("Invalid start position " + std::to_string(from) + " in segment path");
    auto lastOpt = index.findChunkForOriginalOffset(to);
    const Chunk last = lastOpt ? *lastOpt : index.chunks().back();
    std::vector<FetchPiece> plan;
    for (int id = first->id; id <= last.id; id++) {
        const Chunk& c = index.chunks()[id];
        int skip = 0, take = c.originalSize;
        const bool atFirst = id == first->id, atLast = id == last.id;
        if (atFirst && atLast) { skip = from - c.originalPosition; take = std::min(c.originalSize - skip, to - from + 1); }
        else {
            if (atFirst) { skip = from - c.originalPosition; take = c.originalSize - skip; }
            if (atLast) take = std::min(c.originalSize, to - c.originalPosition + 1);
        }
        plan.push_back({id, skip, take});
    }
    return plan;
}

// FetchChunkEnumeration + DefaultChunkManager, batched (SURVEY.md §8f.1): the reference asks its ChunkManager for one chunk
// at a time (one ranged GET and one detransform each, DefaultChunkManager.java:50-70); here the chunks the range touches
// are fetched with ONE ranged GET and detransformed in batches, then served with the reference's skip / bound rules.
class FetchChunkEnumeration {
public:
    using RangeFetcher = std::function<Bytes(const BytesRange&)>;       // ObjectFetcher.fetch(key, range)
    FetchChunkEnumeration(tsgpu_ctx* ctx, const ChunkIndex& index, const BytesRange& range, RangeFetcher fetcher, bool decompress,
                          const DataKeyAndAAD* decryptWith, uint32_t batchChunks = 32)
        : ctx(ctx), decompress(decompress), batch(batchChunks ? batchChunks : 1) {
        if (!ctx) throw NullPointerException("chunkManager cannot be null");
        if (!fetcher) throw NullPointerException("objectKey cannot be null");
        if (range.isEmpty()) throw IllegalArgumentException("range cannot be empty");
        if (decryptWith) { km = *decryptWith; decrypt = true; }
        plan = fetchPlan(index, range.firstPosition(), range.lastPosition());
        uint32_t maxOriginal = 1;
        for (const FetchPiece& pc : plan) {
            chunks.push_back(index.chunks()[pc.chunkId]);
            maxOriginal = std::max<uint32_t>(maxOriginal, (uint32_t)chunks.back().originalSize);
        }
        object = fetcher(transformedRange(chunks));
        if (object.size() != (size_t)transformedRange(chunks).size()) throw std::runtime_error("Stream has fewer bytes than expected");
        stream = std::make_unique<std::istringstream>(std::string((const char*)object.data(), object.size()));
        inner = std::make_unique<DetransformChunkEnumeration>(ctx, stream.get(), chunks, decompress, decrypt ? &km : nullptr, maxOriginal, batch);
    }
    bool hasMoreElements() const { return next < plan.size(); }
    Bytes nextElement() {
        if (!hasMoreElements()) throw NoSuchElementException();
        Bytes chunk = inner->nextElement();
        const FetchPiece& pc = plan[next++];
        if ((size_t)pc.skip > chunk.size()) return Bytes();
        const size_t take = std::min<size_t>((size_t)pc.take, chunk.size() - (size_t)pc.skip);
        return Bytes(chunk.begin() + pc.skip, chunk.begin() + pc.skip + take);
    }
    Bytes readAll() { Bytes all; while (hasMoreElements()) { Bytes c = nextElement(); all.insert(all.end(), c.begin(), c.end()); } return all; }
    size_t chunkCount() const { return plan.size(); }
private:
    tsgpu_ctx* ctx; bool decompress, decrypt = false; uint32_t batch;
    DataKeyAndAAD km; std::vector<FetchPiece> plan; std::vector<Chunk> chunks; Bytes object;
    std::unique_ptr<std::istringstream> stream; std::unique_ptr<DetransformChunkEnumeration> inner; size_t next = 0;
};

// ------------------------------------------------------------------ SegmentManifestV1 JSON (SURVEY.md §8f.2)
// Writer for the exact on-disk form of core/M/manifest/SegmentManifestV1.java:37-91 with the property order Jackson
// produces (golden strings: core/T/manifest/SegmentManifestV1SerdeTest.java:82-133).  The wrapped data key string
// "<keyId>:<base64 RSA-OAEP(dek)>" is produced by the host's RsaEncryptionProvider and passed through untouched.
struct SegmentIndexV1 { int position, size; };
struct SegmentIndexesV1 {                            // core/M/manifest/SegmentIndexesV1.java, builder :27-60
    SegmentIndexV1 offset, timestamp, producerSnapshot, leaderEpoch;
    std::optional<SegmentIndexV1> transaction;
};
struct RemoteLogSegmentMetadataJson {                // the mixin of core/M/manifest/serde/KafkaTypeSerdeModule.java:63-115
    std::string topicId, topic; int partition; std::string id;
    long long startOffset, endOffset, maxTimestampMs; int brokerId; long long eventTimestampMs;
    std::vector<std::pair<int, long long>> segmentLeaderEpochs;
};
inline std::string base64Std(const uint8_t* in, size_t n) {
    static const char A[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
    std::string o;
    for (size_t i = 0; i < n; i += 3) {
        const uint32_t v = (uint32_t)in[i] << 16 | (i + 1 < n ? (uint32_t)in[i + 1] << 8 : 0) | (i + 2 < n ? in[i + 2] : 0);
        o += A[v >> 18]; o += A[(v >> 12) & 63]; o += i + 1 < n ? A[(v >> 6) & 63] : '='; o += i + 2 < n ? A[v & 63] : '=';
    }
    return o;
}
inline std::string segmentManifestV1Json(const ChunkIndex& chunkIndex, const SegmentIndexesV1& idx, bool compression,
                                         const std::optional<std::string>& wrappedDataKey, const Bytes* aad,
                                         const RemoteLogSegmentMetadataJson& m, tsgpu_ctx* ctx = nullptr) {
    auto one = [](const char* name, const SegmentIndexV1& i) {
        return std::string("\"") + name + "\":{\"position\":" + std::to_string(i.position) + ",\"size\":" + std::to_string(i.size) + "}";
    };
    std::string s = "{\"version\":\"1\",\"chunkIndex\":" + chunkIndex.toJson(ctx) + ",\"segmentIndexes\":{";
    s += one("offset", idx.offset) + "," + one("timestamp", idx.timestamp) + "," + one("producerSnapshot", idx.producerSnapshot) + "," +
         one("leaderEpoch", idx.leaderEpoch) + ",";
    s += idx.transaction ? one("transaction", *idx.transaction) : std::string("\"transaction\":null");
    s += std::string("},\"compression\":") + (compression ? "true" : "false");
    if (aad) {                                       // SegmentEncryptionMetadataV1.java:35-61
        s += ",\"encryption\":{";
        if (wrappedDataKey) s += "\"dataKey\":\"" + *wrappedDataKey + "\",";
        s += "\"aad\":\"" + base64Std(aad->data(), aad->size()) + "\"}";
    }
    s += ",\"remoteLogSegmentMetadata\":{\"remoteLogSegmentId\":{\"topicIdPartition\":{\"topicId\":\"" + m.topicId +
         "\",\"topicPartition\":{\"topic\":\"" + m.topic + "\",\"partition\":" + std::to_string(m.partition) + "}},\"id\":\"" + m.id + "\"}," +
         "\"startOffset\":" + std::to_string(m.startOffset) + ",\"endOffset\":" + std::to_string(m.endOffset) +
         ",\"maxTimestampMs\":" + std::to_string(m.maxTimestampMs) + ",\"brokerId\":" + std::to_string(m.brokerId) +
         ",\"eventTimestampMs\":" + std::to_string(m.eventTimestampMs) + ",\"segmentLeaderEpochs\":{";
    for (size_t i = 0; i < m.segmentLeaderEpochs.size(); i++)
        s += (i ? "," : "") + std::string("\"") + std::to_string(m.segmentLeaderEpochs[i].first) + "\":" + std::to_string(m.segmentLeaderEpochs[i].second);
    return s + "}}}";
}

// Reader for the same form (the reference reads it with Jackson; a C++ fetch-side consumer needs the chunk index, the
// compression flag, the AAD and the wrapped data key — unwrapping the key stays with the host's RsaEncryptionProvider).
// Unknown properties are an error, as with the reference's ObjectMapper (FAIL_ON_UNKNOWN_PROPERTIES is Jackson's default).
namespace json {
struct Value {
    enum Kind { Null, Bool, Number, String, Object, Array } kind = Null;
    bool b = false; long long num = 0; std::string str;
    std::vector<std::pair<std::string, Value>> obj; std::vector<Value> arr;
    const Value* get(const std::string& k) const { for (auto& kv : obj) if (kv.first == k) return &kv.second; return nullptr; }
};
struct Parser {
    const std::string& s; size_t p = 0;
    explicit Parser(const std::string& s) : s(s) {}
    [[noreturn]] void fail(const char* what) const { throw IllegalArgumentException(std::string("manifest JSON: ") + what + " at " + std::to_string(p)); }
    void ws() { while (p < s.size() && (s[p] == ' ' || s[p] == '\n' || s[p] == '\t' || s[p] == '\r')) p++; }
    bool eat(char c) { ws(); if (p < s.size() && s[p] == c) { p++; return true; } return false; }
    std::string string() {
        if (!eat('"')) fail("string expected");
        std::string o;
        while (p < s.size() && s[p] != '"') {
            if (s[p] == '\\') {
                if (++p >= s.size()) fail("bad escape");
                const char c = s[p++];
                if (c == 'n') o += '\n'; else if (c == 't') o += '\t'; else if (c == 'r') o += '\r'; else if (c == 'b') o += '\b'; else if (c == 'f') o += '\f';
                else if (c == 'u') { if (p + 4 > s.size()) fail("bad \\u"); o += (char)std::stoi(s.substr(p, 4), nullptr, 16); p += 4; }
                else o += c;
            } else o += s[p++];
        }
        if (p >= s.size()) fail("unterminated string");
        p++;
        return o;
    }
    Value value() {
        ws();
        Value v;
        if (p >= s.size()) fail("value expected");
        const char c = s[p];
        if (c == '{') {
            p++; v.kind = Value::Object;
            if (eat('}')) return v;
            do { std::string k = string(); if (!eat(':')) fail("':' expected"); v.obj.emplace_back(std::move(k), value()); } while (eat(','));
            if (!eat('}')) fail("'}' expected");
        } else if (c == '[') {
            p++; v.kind = Value::Array;
            if (eat(']')) return v;
            do { v.arr.push_back(value()); } while (eat(','));
            if (!eat(']')) fail("']' expected");
        } else if (c == '"') { v.kind = Value::String; v.str = string(); }
        else if (s.compare(p, 4, "true") == 0) { v.kind = Value::Bool; v.b = true; p += 4; }
        else if (s.compare(p, 5, "false") == 0) { v.kind = Value::Bool; p += 5; }
        else if (s.compare(p, 4, "null") == 0) { p += 4; }
        else {
            size_t q = p; if (q < s.size() && s[q] == '-') q++;
            while (q < s.size() && s[q] >= '0' && s[q] <= '9') q++;
            if (q == p || (q == p + 1 && s[p] == '-')) fail("unexpected character");
            v.kind = Value::Number; v.num = std::stoll(s.substr(p, q - p)); p = q;
        }
        return v;
    }
};
}  // namespace json

inline Bytes base64StdDecode(const std::string& in) {
    Bytes o; uint32_t acc = 0; int bits = 0;
    for (char c : in) {
        int v = c >= 'A' && c <= 'Z' ? c - 'A' : c >= 'a' && c <= 'z' ? c - 'a' + 26 : c >= '0' && c <= '9' ? c - '0' + 52 : c == '+' ? 62 : c == '/' ? 63 : -1;
        if (c == '=') break;
        if (v < 0) throw IllegalArgumentException("Illegal base64 character");
        acc = acc << 6 | (uint32_t)v; bits += 6;
        if (bits >= 8) { bits -= 8; o.push_back((uint8_t)(acc >> bits)); }
    }
    return o;
}

struct SegmentManifestV1 {
    std::shared_ptr<ChunkIndex> chunkIndex;
    SegmentIndexesV1 segmentIndexes{};
    bool compression = false;
    std::optional<std::string> wrappedDataKey;       // "<keyId>:<base64>" as written; unwrapping is the host's business
    std::optional<Bytes> aad;
    RemoteLogSegmentMetadataJson remoteLogSegmentMetadata{};
};
// `ctx` is needed for variable indexes: the size list is a zstd frame (possibly libzstd-compressed) decoded on the device.
inline SegmentManifestV1 parseSegmentManifestV1(const std::string& text, tsgpu_ctx* ctx) {
    using json::Value;
    json::Parser ps(text);
    const Value root = ps.value();
    ps.ws();
    if (ps.p != text.size() || root.kind != Value::Object) throw IllegalArgumentException("manifest JSON: one object expected");
    auto need = [](const Value& o, const char* k, Value::Kind kind) -> const Value& {
        const Value* v = o.get(k);
        if (!v || v->kind != kind) throw IllegalArgumentException(std::string("manifest JSON: missing or mistyped property '") + k + "'");
        return *v;
    };
    auto only = [](const Value& o, std::initializer_list<const char*> allowed) {
        for (auto& kv : o.obj) { bool ok = false; for (const char* a : allowed) ok = ok || kv.first == a; if (!ok) throw IllegalArgumentException("manifest JSON: unknown property '" + kv.first + "'"); }
    };
    only(root, {"version", "chunkIndex", "segmentIndexes", "compression", "encryption", "remoteLogSegmentMetadata"});
    if (need(root, "version", Value::String).str != "1") throw IllegalArgumentException("manifest JSON: unsupported version");
    SegmentManifestV1 m;
    const Value& ci = need(root, "chunkIndex", Value::Object);
    const std::string type = need(ci, "type", Value::String).str;
    const int ocs = (int)need(ci, "originalChunkSize", Value::Number).num, ofs = (int)need(ci, "originalFileSize", Value::Number).num;
    if (type == "fixed") {
        only(ci, {"type", "originalChunkSize", "originalFileSize", "transformedChunkSize", "finalTransformedChunkSize"});
        m.chunkIndex = std::make_shared<FixedSizeChunkIndex>(ocs, ofs, (int)need(ci, "transformedChunkSize", Value::Number).num,
                                                             (int)need(ci, "finalTransformedChunkSize", Value::Number).num);
    } else if (type == "variable") {
        only(ci, {"type", "originalChunkSize", "originalFileSize", "transformedChunks"});
        const std::string& b64 = need(ci, "transformedChunks", Value::String).str;
        std::vector<int32_t> sizes(b64.size() * 2 + 1024);          // every size takes >= 1 byte of the decoded frame, Base64 inflates by 4/3
        uint32_t n = (uint32_t)sizes.size();
        int rc = tsgpu_transformed_chunks_deserialize(ctx, b64.c_str(), sizes.data(), &n);
        if (rc == TSGPU_E_SHORT) { sizes.resize((size_t)ofs / std::max(1, ocs) + 2); n = (uint32_t)sizes.size(); rc = tsgpu_transformed_chunks_deserialize(ctx, b64.c_str(), sizes.data(), &n); }
        if (rc) throw IllegalArgumentException(tsgpu_last_error());
        sizes.resize(n);
        m.chunkIndex = std::make_shared<VariableSizeChunkIndex>(ocs, ofs, sizes);
    } else throw IllegalArgumentException("manifest JSON: unknown chunk index type '" + type + "'");
    const Value& si = need(root, "segmentIndexes", Value::Object);
    only(si, {"offset", "timestamp", "producerSnapshot", "leaderEpoch", "transaction"});
    auto one = [&](const char* k) { const Value& v = need(si, k, Value::Object); return SegmentIndexV1{(int)need(v, "position", Value::Number).num, (int)need(v, "size", Value::Number).num}; };
    m.segmentIndexes.offset = one("offset"); m.segmentIndexes.timestamp = one("timestamp");
    m.segmentIndexes.producerSnapshot = one("producerSnapshot"); m.segmentIndexes.leaderEpoch = one("leaderEpoch");
    if (const Value* t = si.get("transaction")) if (t->kind == Value::Object) m.segmentIndexes.transaction = one("transaction");
    m.compression = need(root, "compression", Value::Bool).b;
    if (const Value* e = root.get("encryption")) if (e->kind == Value::Object) {
        only(*e, {"dataKey", "aad"});
        if (const Value* k = e->get("dataKey")) if (k->kind == Value::String) m.wrappedDataKey = k->str;
        m.aad = base64StdDecode(need(*e, "aad", Value::String).str);
    }
    if (const Value* r = root.get("remoteLogSegmentMetadata")) if (r->kind == Value::Object) {
        auto& o = m.remoteLogSegmentMetadata;
        const Value& id = need(*r, "remoteLogSegmentId", Value::Object);
        const Value& tip = need(id, "topicIdPartition", Value::Object);
        const Value& tp = need(tip, "topicPartition", Value::Object);
        o.topicId = need(tip, "topicId", Value::String).str; o.topic = need(tp, "topic", Value::String).str;
        o.partition = (int)need(tp, "partition", Value::Number).num; o.id = need(id, "id", Value::String).str;
        o.startOffset = need(*r, "startOffset", Value::Number).num; o.endOffset = need(*r, "endOffset", Value::Number).num;
        o.maxTimestampMs = need(*r, "maxTimestampMs", Value::Number).num; o.brokerId = (int)need(*r, "brokerId", Value::Number).num;
        o.eventTimestampMs = need(*r, "eventTimestampMs", Value::Number).num;
        for (auto& kv : need(*r, "segmentLeaderEpochs", Value::Object).obj) o.segmentLeaderEpochs.emplace_back(std::stoi(kv.first), kv.second.num);
    }
    return m;
}

// Object keys (core/M/ObjectKeyFactory.java:43-53, 81-124): "<prefix><topic>-<topicId>/<partition>/<startOffset %020d>-<segmentId>.<suffix>"
enum class Suffix { LOG, INDEXES, MANIFEST };
inline std::string objectKey(const std::string& prefix, const RemoteLogSegmentMetadataJson& m, Suffix suffix) {
    char off[32];
    snprintf(off, sizeof off, "%020lld", m.startOffset);
    const char* sfx = suffix == Suffix::LOG ? "log" : suffix == Suffix::INDEXES ? "indexes" : "rsm-manifest";
    return prefix + m.topic + "-" + m.topicId + "/" + std::to_string(m.partition) + "/" + off + "-" + m.id + "." + sfx;
}

}  // namespace tieredstorage
