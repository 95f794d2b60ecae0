/*
 * tsgpu.h — C-ABI of libtsgpu.so: the H100-native (sm_90a) chunk-transform pipeline behind Aiven's
 * tiered-storage RemoteStorageManager operator surface.
 *
 * The reference has no FFI of its own (pure Java); its boundary for this path is the pair of Java interfaces
 *   TransformChunkEnumeration    core/M/transform/TransformChunkEnumeration.java:28-42
 *   DetransformChunkEnumeration  core/M/transform/DetransformChunkEnumeration.java:28-29
 * (core/M = <reference>/core/src/main/java/io/aiven/kafka/tieredstorage).  A thin JNI class (jni/, see
 * INTEGRATION.md) implements those interfaces by handing a *batch* of chunks to the calls below and serving
 * one byte[] per nextElement().  Each entry point names the reference code it replaces.
 *
 * Conventions: plain pointers and sizes only; return 0 (TSGPU_OK) or a negative error code; never throws or
 * aborts; the caller owns every buffer and the library keeps no pointer after a call returns; a context may
 * be used from several threads at once (a host-buffer call claims work slots — stream pair, arenas, pinned descriptor
 * block — and concurrent calls overlap on the GPU; only the slot bookkeeping is under the context mutex); there is NO
 * CPU fallback — without a CUDA device tsgpu_create fails with TSGPU_E_NODEVICE.
 */
#ifndef TSGPU_H
#define TSGPU_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TSGPU_FLAG_ZSTD 1u     /* compression.enabled  (RemoteStorageManagerConfig.java:132-138) */
#define TSGPU_FLAG_AES  2u     /* encryption.enabled   (RemoteStorageManagerConfig.java:147-153) */
/* Modifier of TSGPU_FLAG_ZSTD on the transform side (ignored by detransform): compress for size rather than for speed.
 * Default: independent 8 KiB blocks, ~3.1 : 1 on Kafka-like text, about twice as fast as dense.  Dense: 64 KiB regions
 * sharing one window and one set of entropy tables, ~3.5 : 1 and
 * byte-identical frames on every run.  Both are plain zstd frames with Frame_Content_Size; libzstd and this library read both.
 * TSGPU_ZSTD_MODE=dense in the environment makes dense the default of a context. */
#define TSGPU_FLAG_ZSTD_DENSE 4u
/* Read-back check of the host-buffer transform calls (tsgpu_transform, tsgpu_transform_chunks; any mix of ZSTD / ZSTD_DENSE /
 * AES): each batch is detransformed on the device and compared byte for byte with its input before any of its bytes are
 * copied to dst.  A chunk that does not read back fails the call with TSGPU_E_VERIFY.  Opt-in, like RocksDB's
 * verify_compression: with 4 MiB chunks it adds the device decrypt / decode of every batch (cost: DESIGN.md §8).
 * The check decodes with this library's own decoder.  It catches runtime faults of the writer -- races, memory errors,
 * silent data corruption -- but not a misreading of the format that the writer and the reader share; the libzstd and
 * OpenSSL cross-tests of the test suite remain the guard for that.  Its decodes count in tsgpu_decode_path_stats.
 * TSGPU_VERIFY=1 in the environment makes the flag the default of a context's host-buffer transform calls.  The
 * device-resident calls refuse the bit (TSGPU_E_ARG): they have no status output on the transform side. */
#define TSGPU_FLAG_VERIFY 8u
/* Modifier of TSGPU_FLAG_ZSTD on the transform side (ignored by detransform), for tsgpu_transform, tsgpu_transform_chunks and
 * tsgpu_transform_device; combines with ZSTD_DENSE, AES and VERIFY.  Every frame ends with its Content_Checksum (RFC 8878
 * 3.1.1: the low 32 bits of XXH64 of the chunk, seed 0, little-endian after the last block; Frame_Header_Descriptor bit 2 set).
 * Otherwise the frame is exactly the one written without the flag, so it is 4 bytes longer and transformed_sizes count them;
 * tsgpu_transform_bound and tsgpu_slot_stride already leave room.  Every zstd reader -- libzstd and zstd-jni, `zstd -t`, this
 * library's decoder -- then verifies the content, so a damaged byte in a Raw block or a Huffman literal stream, which would
 * otherwise decode to a different byte without an error, fails the read (TSGPU_E_CORRUPT here).  The checksum is computed
 * from the original bytes by code that shares nothing with the compressor's stages, so with TSGPU_FLAG_VERIFY it also catches a
 * misreading of the format that the writer and this library's reader share.  The hash runs in the compressor's own launch,
 * beside the compression (cost: DESIGN.md §8).  TSGPU_ZSTD_CHECKSUM=1 in the environment makes the flag the default of a
 * context's transform calls. */
#define TSGPU_FLAG_ZSTD_CHECKSUM 16u
/* Validation of the Kafka log segment given to tsgpu_transform / tsgpu_transform_cursor, on the GPU, before any of its bytes are
 * uploaded: every entry `offset i64 | size i32 | ...` (12 + size bytes; the entries must end exactly at the end of the segment;
 * an empty segment is valid) is checked as DefaultRecordBatch.ensureValid() checks a batch -- magic 2: size >= 49 and the
 * CRC-32C at +17 over [+21, end); magic 0/1 (legacy message sets): size >= 14 and the CRC-32 at +12 over [+16, end); any other
 * magic fails.  Records inside a batch are not parsed.  The first invalid entry fails the call with TSGPU_E_RECORDS.  The check
 * reads the bytes the transform already copied to HBM and adds no copy; the transformed bytes are exactly those written without
 * the flag.  It combines with ZSTD, ZSTD_DENSE, ZSTD_CHECKSUM, AES and VERIFY and needs ZSTD or AES (TSGPU_E_ARG without: with
 * flags 0 the transform is a host memcpy and no byte reaches the GPU).  tsgpu_transform_chunks and the device-resident calls
 * refuse it (TSGPU_E_ARG: index blobs are not record batches, and the device calls have no status output on the transform side);
 * detransform ignores it.  TSGPU_VALIDATE_RECORDS=1 in the environment makes the flag the default of a context's
 * tsgpu_transform_cursor calls that have ZSTD or AES: those callers say where their segment ends, and the JNI enumeration
 * transforms every window of a segment that way.  It does not reach tsgpu_transform, which a caller may also use for one
 * window of a segment (a window checked as a whole segment would fail where an entry crosses its end).  Cost and memory:
 * DESIGN.md §3 and §8. */
#define TSGPU_FLAG_VALIDATE_RECORDS 32u
/* to_flags of tsgpu_rewrite_object and tsgpu_rewrite_object_crc64 only (every other call refuses it as an unknown bit): when
 * from_flags and to_flags both have TSGPU_FLAG_ZSTD, the ZSTD_CHECKSUM and ZSTD_DENSE bits of to_flags act on the source frames
 * instead of being refused.  It needs ZSTD on both sides and one of the two bits, else TSGPU_E_ARG.
 *   REFRAME | ZSTD_CHECKSUM (seal): every source frame is kept byte for byte, except that Frame_Header_Descriptor bit 2 is set
 *     and the 4-byte Content_Checksum of the chunk is inserted after its last block; skippable frames that followed it in the
 *     chunk move 4 bytes on.  That is the frame libzstd writes for the same blocks with its checksum flag, so objects the Java
 *     plugin wrote keep their level-3 density.  A frame that already has a checksum (verified by the source decode) is kept as
 *     it is.  Clearing the bit and dropping the 4 bytes gives back the old frame.
 *   REFRAME | ZSTD_DENSE [| ZSTD_CHECKSUM] (re-encode): every chunk is also compressed anew by the dense compressor, with a
 *     checksum if asked, and the new frame replaces the old one only when it is strictly smaller than what the old frame
 *     becomes (sealed with CHECKSUM, else unchanged).  No chunk grows by more than the 4 checksum bytes.  Without
 *     ZSTD_CHECKSUM a dense frame carries no checksum, so it can replace a frame that had one: add ZSTD_CHECKSUM when the source
 *     may hold checksummed frames.
 * Only the bits given count: the context's TSGPU_ZSTD_MODE=dense and TSGPU_ZSTD_CHECKSUM=1 do not add to them.  REFRAME turns
 * TSGPU_FLAG_VERIFY on, so every new chunk is decoded again, and its new checksum checked, before its batch leaves: a chunk the
 * first decode misread by chance fails the call with TSGPU_E_VERIFY instead of being sealed with the checksum of wrong bytes.
 * A misread that repeats is caught by TSGPU_FLAG_VALIDATE_RECORDS on the source, which a caller sealing objects should set.
 * The part_cap bound and dst grow by 4 bytes per chunk with ZSTD_CHECKSUM, and a chunk whose sealed frame would not fit the
 * context's frame slot (tsgpu_transform_bound of max_chunk_bytes) fails with TSGPU_E_ARG before any GPU work.  Cost: DESIGN.md §8. */
#define TSGPU_FLAG_REFRAME 64u

#define TSGPU_IV_SIZE   12     /* SegmentEncryptionMetadataV1.java:30 */
#define TSGPU_TAG_SIZE  16     /* AesEncryptionProvider.java:38 (128-bit tag) */

#define TSGPU_OK            0
#define TSGPU_E_ARG        -1  /* IllegalArgumentException / NullPointerException in the reference */
#define TSGPU_E_STATE      -2  /* IllegalStateException */
#define TSGPU_E_AUTH       -3  /* AEADBadTagException wrapped in RuntimeException (DecryptionChunkEnumeration.java:59-61) */
#define TSGPU_E_CORRUPT    -4  /* "Invalid decompressed size" / malformed zstd frame (DecompressionChunkEnumeration.java:42-44) */
#define TSGPU_E_SHORT      -5  /* destination too small / "Stream has fewer bytes than expected" (BaseDetransformChunkEnumeration.java:106-108) */
#define TSGPU_E_NODEVICE   -6  /* no usable CUDA device: the product path does not fall back to the CPU */
#define TSGPU_E_CUDA       -7  /* a CUDA call or kernel failed; message in tsgpu_last_error() */
#define TSGPU_E_NOMEM      -8
/* TSGPU_FLAG_VERIFY: a transformed chunk did not read back.  The message names the chunk and the check that failed: tag,
 * frame, size, or the first byte offset that differs.  No byte of the failing batch reaches dst; earlier batches may
 * already be there, and the caller discards the whole result as with any error. */
#define TSGPU_E_VERIFY     -9
/* TSGPU_FLAG_VALIDATE_RECORDS: a record batch failed validation.  The message names the segment byte position of the first
 * invalid entry and the check that failed -- "Record batch is corrupt (check: length)" / "(check: magic)", or "Record is corrupt
 * (stored crc = S, computed crc = C) (check: crc)".  No byte of the failing batch reaches dst; earlier batches may already be
 * there, as with TSGPU_E_VERIFY. */
#define TSGPU_E_RECORDS   -10

typedef struct tsgpu_ctx tsgpu_ctx;

/* Thread-local message for the last failing call on this thread (maps to the Java exception message). */
const char* tsgpu_last_error(void);
const char* tsgpu_version(void);

/* ---------------------------------------------------------------------------------------------------------
 * Context: owns, per listed device, streams, device arenas and pinned staging sized for `max_batch` chunks of
 * `max_chunk_bytes` original bytes (= chunk.size, RemoteStorageManagerConfig.java:123-130).
 * Batches are dealt round-robin to the devices (BASELINE.json north_star: segments shard by chunk batch).
 * A host-buffer call (tsgpu_transform / tsgpu_detransform) cuts its chunks into batches of `max_batch` and keeps up to
 * 8 of them in flight per device (work slots, allocated on first use; each has a compute stream and a copy-out stream).
 * With 4 MiB chunks `max_batch = 4` measured best through PCIe; device-resident callers pass whole segments.
 * Environment (read once by tsgpu_create): TSGPU_SLOTS=1..16 slots per device, TSGPU_ZSTD_MODE=dense makes
 * TSGPU_FLAG_ZSTD_DENSE the context's default (both tuning only), TSGPU_VERIFY=1 turns TSGPU_FLAG_VERIFY on for the
 * context's host-buffer transform calls (not for the device-resident calls), TSGPU_ZSTD_CHECKSUM=1 turns
 * TSGPU_FLAG_ZSTD_CHECKSUM on for all of the context's compressing transform calls, TSGPU_VALIDATE_RECORDS=1 turns
 * TSGPU_FLAG_VALIDATE_RECORDS on for the context's tsgpu_transform_cursor calls with ZSTD or AES.
 * --------------------------------------------------------------------------------------------------------- */
int  tsgpu_create(const int* device_ids, int n_devices, uint32_t max_chunk_bytes, uint32_t max_batch,
                  tsgpu_ctx** out);
void tsgpu_destroy(tsgpu_ctx* ctx);

/* Pinned host memory for the caller's staging (JNI: NewDirectByteBuffer over it).  Optional: pageable
 * buffers are accepted everywhere, they are just slower to copy. */
void* tsgpu_host_alloc(size_t bytes);
void  tsgpu_host_free(void* p);

/* Upper bound of the transformed size of a segment: sum over chunks of (zstd bound) + 28 if encrypted. */
uint64_t tsgpu_transform_bound(uint32_t flags, uint64_t src_len, uint32_t chunk_size);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_transform — the upload chain of RemoteStorageManager.transformation (RemoteStorageManager.java:434-453):
 *   BaseTransformChunkEnumeration (split src into chunk_size pieces; 0 = no chunking; BaseTransform…java:61-93)
 *   -> [CompressionChunkEnumeration: one zstd frame with Frame_Content_Size per chunk; Compression…java:49-62]
 *   -> [EncryptionChunkEnumeration: IV(12) || AES-256-GCM(ct) || TAG(16); Encryption…java:65-84]
 * plus the size bookkeeping TransformFinisher.nextElement feeds to the ChunkIndex builder (TransformFinisher.java:101-110).
 *
 *   src/src_len   original segment bytes (host memory)
 *   key[32], aad  per-segment DataKeyAndAAD (AesEncryptionProvider.java:52-58); ignored without TSGPU_FLAG_AES
 *   ivs           12 bytes per chunk, generated by the HOST (SecureRandom in Java, AesEncryptionProvider.java:70)
 *   dst/dst_cap   receives the transformed chunks back to back, i.e. exactly the bytes of the uploaded .log object
 *   transformed_sizes[n]  one entry per chunk (input of AbstractChunkIndexBuilder.addChunk/finish)
 *   n_chunks      in: capacity of transformed_sizes; out: number of chunks (0 for an empty segment)
 * --------------------------------------------------------------------------------------------------------- */
int tsgpu_transform(tsgpu_ctx* ctx, uint32_t flags,
                    const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                    const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                    uint8_t* dst, uint64_t dst_cap,
                    uint32_t* transformed_sizes, uint32_t* n_chunks);

/* A segment transformed in several calls (windows of chunks, as a streaming caller reads it) with
 * TSGPU_FLAG_VALIDATE_RECORDS: entries cross the calls, so the validation state goes from one call to the next in a cursor.  A
 * zeroed cursor is the start of a segment; each call continues at the byte after the previous call's last one and updates the
 * cursor on success (after a failure it is meaningless).  The cursor holds what an entry that straddles the end of the call
 * needs: its start, its end, the running CRC with its kind and the stored value, and up to 21 header bytes when the call ends
 * inside its header.  segment_ends_here != 0 marks the last call (a short or empty window): a segment that ends inside an entry
 * then fails with check "length".  Without the flag (or its environment default) the cursor is not used and may be NULL.
 * With the flag, tsgpu_transform is tsgpu_transform_cursor with a zeroed cursor and segment_ends_here = 1. */
typedef struct tsgpu_records_cursor { uint64_t opaque[8]; } tsgpu_records_cursor;
int tsgpu_transform_cursor(tsgpu_ctx* ctx, uint32_t flags,
                           const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                           const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                           uint8_t* dst, uint64_t dst_cap,
                           uint32_t* transformed_sizes, uint32_t* n_chunks,
                           tsgpu_records_cursor* cursor, int segment_ends_here);

/* tsgpu_transform_cursor plus the CRC-32C of the object's upload parts, computed on the GPU from the bytes it copies to dst.
 * The object is what dst receives, call after call, for one segment (the transformed chunks back to back: the .log object);
 * part k is its bytes [k * part_size, min((k + 1) * part_size, object length)), as a multipart upload cuts it.  CRC-32C is the
 * Castagnoli CRC (reflected polynomial 0x82F63B78, init and xorout 0xFFFFFFFF; crc32c("123456789") = 0xE3069283): what S3
 * UploadPart takes as x-amz-checksum-crc32c and GCS as the object's crc32c (wiring: INTEGRATION.md).  It covers the bytes as
 * they were in HBM when the library copied them out, so a part damaged on any later hop -- pinned buffer, JVM copies, the
 * storage client's part buffer -- is refused by the object store while the local segment still exists.
 *
 *   part_size      >= 1 and the same for every call of a segment (TSGPU_E_ARG otherwise); no minimum is imposed
 *   parts          32-byte cursor, zeroed at the start of the object; carries the open part and the object CRC between calls
 *   part_crc32c    receives, in part order, the CRC of every part whose last byte this call produced; *n_parts is their count
 *   part_cap       capacity of part_crc32c.  It must be at least
 *                    floor((carried + tsgpu_transform_bound(flags, src_len, chunk_size)) / part_size) + (segment_ends_here ? 1 : 0)
 *                  where carried is the open part's length (object bytes so far mod part_size; 0 for a new object, and the
 *                  bound is 0 when src_len is 0); a smaller part_cap is refused with TSGPU_E_SHORT before any GPU work
 *   object_crc32c  with segment_ends_here: the open part is emitted too and *object_crc32c is the CRC-32C of the whole object
 *                  (S3's FULL_OBJECT checksum, GCS's object crc32c).  An empty object has no part and CRC 0.  Without
 *                  segment_ends_here it is not written.
 * flags must include ZSTD or AES (TSGPU_E_ARG: with flags 0 no byte reaches the GPU); the call combines with ZSTD_DENSE,
 * ZSTD_CHECKSUM, VERIFY and VALIDATE_RECORDS, and `records` may be NULL without VALIDATE_RECORDS.  dst, transformed_sizes and
 * every error are those of tsgpu_transform_cursor with the same arguments.  A failed call writes no part CRC and no object CRC --
 * not even those of batches before a batch that failed VERIFY or VALIDATE_RECORDS, whose bytes may already be in dst -- and leaves
 * both cursors without a defined value: the caller discards the object, as with any error.  Cost and memory: DESIGN.md §3, §8. */
typedef struct tsgpu_parts_cursor { uint64_t opaque[4]; } tsgpu_parts_cursor;
int tsgpu_transform_parts(tsgpu_ctx* ctx, uint32_t flags,
                          const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                          const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                          uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                          tsgpu_records_cursor* records, int segment_ends_here,
                          uint64_t part_size, tsgpu_parts_cursor* parts,
                          uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts, uint32_t* object_crc32c);

/* Ragged variant of tsgpu_transform: chunk i is the next chunk_lens[i] bytes of src (no fixed chunk size).
 * Replaces the per-index chains of RemoteStorageManager.transformIndex (RemoteStorageManager.java:455-490; each Kafka
 * index file is ONE chunk, chunking disabled, encryption only) so the five index blobs of a segment go through one batch. */
int tsgpu_transform_chunks(tsgpu_ctx* ctx, uint32_t flags,
                           const uint8_t* src, const uint32_t* chunk_lens, uint32_t n_chunks,
                           const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                           uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_detransform — the fetch chain of DefaultChunkManager.getChunk (DefaultChunkManager.java:50-70):
 *   BaseDetransformChunkEnumeration (cut src at transformed_sizes; BaseDetransform…java:47-120)
 *   -> [DecryptionChunkEnumeration: IV from the chunk head, tag verified; Decryption…java:53-62]
 *   -> [DecompressionChunkEnumeration: Frame_Content_Size mandatory; Decompression…java:38-46]
 * for n_chunks consecutive chunks at once (the reference does one chunk per call; batching is what makes
 * ranged fetches fast, SURVEY.md §8f.1).
 *
 *   src            transformed chunks back to back (bytes [first.transformedPosition, last.end) of the object)
 *   src_len        bytes available at src; fewer than sum(transformed_sizes) => TSGPU_E_SHORT
 *   original_sizes[n]  out: bytes produced per chunk (may be NULL)
 *   dst/dst_cap    receives the original bytes of the chunks back to back
 * Returns TSGPU_E_AUTH if any tag fails (no plaintext of that batch is released: dst is zeroed),
 * TSGPU_E_CORRUPT for malformed frames — a compressed chunk must be exactly one zstd frame with Frame_Content_Size (skippable
 * frames may follow it); bytes after the frame are refused like Zstd.decompress(chunk, size) refuses them.
 * --------------------------------------------------------------------------------------------------------- */
int tsgpu_detransform(tsgpu_ctx* ctx, uint32_t flags,
                      const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                      const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                      uint8_t* dst, uint64_t dst_cap, uint32_t* original_sizes);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_check_object — proof that a stored .log object still decodes to a valid segment, without its plaintext leaving the GPU.
 * It reads what tsgpu_detransform reads and runs the same stages, but copies nothing back except sizes, statuses, record verdicts
 * and CRC words: for an object that is the only copy of its segment (after local.retention), one moved between buckets or
 * providers, or one written by the Java plugin before the broker used this library.  Every chunk is checked, in object order:
 *   1. its GCM tag (AES);  2. its zstd frame, and the frame's Content_Checksum when it carries one (ZSTD);
 *   3. its decoded size against the manifest's chunk index (AbstractChunkIndex.materializeChunks): ceil(original_file_size /
 *      original_chunk_size) chunks, each of original_chunk_size bytes but the last, which holds the remainder; an empty segment
 *      has no chunk (or the index's one chunk of 0 transformed bytes, which a caller may pass);
 *   4. with TSGPU_FLAG_VALIDATE_RECORDS: every record batch of the decoded segment, with the rules and messages of that flag on
 *      the upload side (a segment that ends inside an entry fails with check "length").
 *
 *   flags          the manifest's compression (TSGPU_FLAG_ZSTD; ZSTD_DENSE and ZSTD_CHECKSUM are accepted and ignored) and
 *                  encryption (TSGPU_FLAG_AES), plus TSGPU_FLAG_VALIDATE_RECORDS; any other bit fails with TSGPU_E_ARG.  Flags 0
 *                  is a plain object: it is the segment, and only the size, record and CRC checks apply.
 *   src, transformed_sizes, n_chunks, key, aad   one window of the object, as tsgpu_detransform takes it (n_chunks may be 0)
 *   original_chunk_size, original_file_size      the manifest's chunk index (original_chunk_size <= the context's max_chunk_bytes)
 *   cursor         128 bytes, zeroed at the start of the object; a caller checks an object in windows of chunks, in order,
 *                  passing the same cursor (chunks and bytes so far, the two running CRCs, the record-validation state).  It is
 *                  updated on success; after a failure it has no defined value.
 *   object_ends_here  != 0 on the last window (which may be empty): the chunk count must then match the index, and
 *                  *object_crc32c receives the CRC-32C of the object's bytes (compare with S3's FULL_OBJECT checksum, GCS's crc32c
 *                  or the object CRC of tsgpu_transform_parts recorded at upload) and *segment_crc32c that of the decoded segment
 *                  (compare with the local segment file before it is deleted).  Neither is written before the end or on failure.
 * Returns the first failure in object order: TSGPU_E_AUTH (a tag), TSGPU_E_CORRUPT (a frame, a Content_Checksum, or a decoded
 * size or chunk count that disagrees with the index; the message names the chunk and both sizes -- a frame that would decode to
 * more than original_chunk_size bytes is refused as an invalid frame), TSGPU_E_RECORDS (the message
 * names the segment position), TSGPU_E_SHORT (src_len below the sum of transformed_sizes).  Within a batch of chunks, a tag, frame
 * or size failure is reported before the batch's record verdict.  TSGPU_E_ARG as tsgpu_detransform for sizes beyond the
 * context's capacity.  Cost and memory: DESIGN.md §3, §8.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct tsgpu_check_cursor { uint64_t opaque[16]; } tsgpu_check_cursor;
int tsgpu_check_object(tsgpu_ctx* ctx, uint32_t flags,
                       const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                       uint32_t original_chunk_size, uint64_t original_file_size,
                       const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                       tsgpu_check_cursor* cursor, int object_ends_here,
                       uint32_t* object_crc32c, uint32_t* segment_crc32c);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_rewrite_object — a stored .log object rewritten on the GPU under a new data key, or with compression or encryption
 * added, without its plaintext leaving the GPU: for encryption or compression turned on after the fact, a data key that must be
 * replaced because it was exposed, or a migration between buckets, regions or providers that copies every object anyway.  Each
 * window is checked exactly as tsgpu_check_object checks it, then transformed as tsgpu_transform_parts transforms a segment,
 * batch by batch in HBM; the host sees only the old and the new transformed bytes.
 *
 * Source side: from_flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, from_key, from_aad,
 *   the cursor walk and the empty-segment rule are those of tsgpu_check_object (flags 0 is a plain object; VALIDATE_RECORDS
 *   checks every record batch).  Every source chunk passes all of that call's checks before any byte of its batch is released.
 * Target side:
 *   to_flags       TSGPU_FLAG_ZSTD, ZSTD_DENSE, ZSTD_CHECKSUM, AES, VERIFY and REFRAME; it must contain ZSTD or AES (the plain object is
 *                  what tsgpu_detransform gives).  Any other bit fails with TSGPU_E_ARG.  New chunk i holds the same original
 *                  bytes as old chunk i: the chunk size and the file size do not change.
 *                  When both from_flags and to_flags have ZSTD, every source frame goes into the new object byte for byte (it
 *                  is still decoded, for the size, record and segment-CRC checks, but not re-encoded: objects the Java plugin
 *                  wrote are libzstd level 3, denser than this library's speed mode).  ZSTD_DENSE or ZSTD_CHECKSUM then fail with
 *                  TSGPU_E_ARG, having nothing to act on, unless TSGPU_FLAG_REFRAME is set: it seals or re-encodes the frames.  Only a source without ZSTD is compressed, by the selected compressor.
 *                  The context's TSGPU_ZSTD_MODE=dense and TSGPU_ZSTD_CHECKSUM=1 act where a chunk is compressed, and
 *                  TSGPU_VERIFY=1 turns on VERIFY, as for tsgpu_transform_parts.
 *   to_key, to_aad, to_ivs   with AES: the new data key, AAD and one 12-byte IV per chunk of the window.  One GCM key must never
 *                  encrypt two plaintexts under one IV, so before any GPU work the call fails with TSGPU_E_ARG when two entries of
 *                  to_ivs are equal, or, with AES on both sides and to_key equal to from_key, when an entry equals the IV of any
 *                  source chunk of the window (its first 12 bytes).  IVs of other windows are not seen: a caller draws them at
 *                  random (or never reuses to_key for another object).
 *   dst, dst_cap, new_transformed_sizes   the window's new chunks back to back and their sizes (n_chunks entries; the empty
 *                  segment's one empty chunk gets size 0), as tsgpu_transform_parts gives them.
 *   part_size, part_crc32c, part_cap, n_parts   as tsgpu_transform_parts, with the bound's src_len taken from the chunk index:
 *                  part_cap >= floor((carried + B) / part_size) + (object_ends_here ? 1 : 0), B = tsgpu_transform_bound(to_flags,
 *                  L, original_chunk_size) with L the window's original bytes by the index -- or, when the frames are kept, the
 *                  window's exact new length (its frames, plus 28 bytes each with AES), which is no more for frames within the
 *                  zstd bound; 4 bytes more per frame that TSGPU_FLAG_REFRAME seals.  A smaller part_cap fails with TSGPU_E_SHORT before any GPU work.  A caller that uploads in one
 *                  PUT passes a part_size no smaller than the object's bound.
 *   cursor         192 bytes, zeroed at the start of the object, passed to every window in order; updated on success, without a
 *                  defined value after a failure.
 *   object_ends_here  != 0 on the last window (which may be empty): the chunk count must match the index, and then
 *                  *source_crc32c is the CRC-32C of the old object (compare with the store's checksum of what was read),
 *                  *object_crc32c that of the new object (FULL_OBJECT) and *segment_crc32c that of the decoded segment (equal
 *                  to the segment CRC of tsgpu_check_object over either object).  None is written before the end or on failure.
 * Returns the first failure in object order; within a batch: the source's tag, frame and size (TSGPU_E_AUTH, TSGPU_E_CORRUPT, as
 * tsgpu_check_object names them), then its records (TSGPU_E_RECORDS), then VERIFY of the new chunks (TSGPU_E_VERIFY).  No byte of
 * a failing batch reaches dst; earlier batches may already be there.  A failed call writes no CRC.  TSGPU_E_SHORT for a short src
 * or dst.  Buffers and cost: DESIGN.md §3, §8.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct tsgpu_rewrite_cursor { uint64_t opaque[24]; } tsgpu_rewrite_cursor;
int tsgpu_rewrite_object(tsgpu_ctx* ctx,
                         uint32_t from_flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                         uint32_t original_chunk_size, uint64_t original_file_size,
                         const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                         uint32_t to_flags, const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs,
                         uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                         uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts,
                         tsgpu_rewrite_cursor* cursor, int object_ends_here,
                         uint32_t* source_crc32c, uint32_t* object_crc32c, uint32_t* segment_crc32c);

/* ---------------------------------------------------------------------------------------------------------
 * CRC-64/NVME twins of tsgpu_transform_parts, tsgpu_check_object and tsgpu_rewrite_object.  Each takes the arguments, rules,
 * errors and part_cap bound of its CRC-32C twin, and writes the same transformed bytes, transformed_sizes and
 * new_transformed_sizes for the same arguments; only the checksum outputs differ, as uint64_t.  A failed call writes no
 * checksum, as in the CRC-32C calls.
 *
 * CRC-64/NVME: width 64, polynomial 0xAD93D23594C93659 (reflected 0x9A6C9329AC4BC9B5), init and xorout all ones, reflected
 * input and output; crc64nvme("123456789") = 0xAE8B14860A799888, and 0 for no bytes.  The stores take it as 8 big-endian
 * bytes, Base64-encoded (wiring: INTEGRATION.md):
 *   - S3: CRC64NVME as a part checksum (x-amz-checksum-crc64nvme on UploadPart) and as the FULL_OBJECT checksum of a multipart
 *     upload.  S3 is understood to store a CRC64NVME full-object checksum for objects uploaded without a client checksum, so
 *     object_crc64 of tsgpu_check_object_crc64 is what such an object is compared with -- unverified here.
 *   - Azure Blob: x-ms-content-crc64 on Put Block is understood to be this CRC -- unverified here (INTEGRATION.md).
 *
 * The cursors keep their sizes and hold the 64-bit words in place of the 32-bit ones.  A cursor carries one width: continuing
 * a cursor with the twin of the call that started it gives wrong checksums.  The call does not detect this; the object store
 * then refuses the upload, so the failure is safe.
 * --------------------------------------------------------------------------------------------------------- */
int tsgpu_transform_parts_crc64(tsgpu_ctx* ctx, uint32_t flags,
                                const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                                const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                                tsgpu_records_cursor* records, int segment_ends_here,
                                uint64_t part_size, tsgpu_parts_cursor* parts,
                                uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts, uint64_t* object_crc64);
int tsgpu_check_object_crc64(tsgpu_ctx* ctx, uint32_t flags,
                             const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                             uint32_t original_chunk_size, uint64_t original_file_size,
                             const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                             tsgpu_check_cursor* cursor, int object_ends_here,
                             uint64_t* object_crc64, uint64_t* segment_crc64);
int tsgpu_rewrite_object_crc64(tsgpu_ctx* ctx,
                               uint32_t from_flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                               uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size,
                               const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                               uint32_t to_flags, const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len,
                               const uint8_t* to_ivs, uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                               uint64_t part_size, uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts,
                               tsgpu_rewrite_cursor* cursor, int object_ends_here,
                               uint64_t* source_crc64, uint64_t* object_crc64, uint64_t* segment_crc64);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_rekey_object — the AES-GCM chunks of a stored object re-encrypted under a new data key with nothing decoded: for replacing
 * an exposed key.  Each chunk (IV || CT || TAG) is read once; one GPU pass computes CT ^ E_old(ctr) ^ E_new(ctr), checks the old
 * tag and writes the new IV and tag.  The plaintext exists only in registers.  The call serves both objects of an encrypted
 * segment: the .log object (its chunks by the chunk index) and the .indexes object (its blobs at their SegmentIndexesV1 positions
 * and sizes).  Sizes do not change, so the chunk index and SegmentIndexesV1 stay as they are and only the manifest's encryption
 * metadata changes.  Unlike tsgpu_rewrite_object this proves only that every chunk is authentic under the old key: nothing checks
 * that the object decodes to a valid segment.
 *
 *   flags          TSGPU_FLAG_VERIFY only; any other bit fails with TSGPU_E_ARG.  TSGPU_VERIFY=1 turns VERIFY on.  With VERIFY every
 *                  batch is decrypted again by the separate decrypt kernels, the source under the old key and the output under
 *                  the new one, and the two plaintexts are compared on the GPU before any byte of the batch is released; a
 *                  difference fails with TSGPU_E_VERIFY naming the chunk and the first differing byte.
 *   src, src_len, transformed_sizes, n_chunks   the window's chunks back to back.  A chunk of 0 bytes passes through as 0 bytes
 *                  (an empty index blob, the empty segment's one chunk) and takes no IV; a chunk of 1 to 27 bytes fails its tag
 *                  (TSGPU_E_AUTH); a chunk larger than the context's transformed slot (what tsgpu_detransform takes) fails with
 *                  TSGPU_E_ARG before any GPU work.
 *   from_key, from_aad   the old data key and AAD; to_key, to_aad, to_ivs   the new ones and one 12-byte IV per chunk.  The IV
 *                  rules and messages are those of tsgpu_rewrite_object: no two non-empty chunks of the window may get the same
 *                  IV, and when to_key equals from_key no new IV may equal a source chunk's IV (TSGPU_E_ARG, before any GPU work).
 *   dst, dst_cap   receive exactly sum(transformed_sizes) bytes: chunk i keeps its size and gets to_ivs[i].  A smaller dst_cap
 *                  fails with TSGPU_E_SHORT before any GPU work.
 *   part_size, part_crc32c, part_cap, n_parts   as tsgpu_transform_parts, with an exact bound: part_cap >= floor((carried +
 *                  sum(transformed_sizes)) / part_size) + (object_ends_here ? 1 : 0); a smaller part_cap fails with TSGPU_E_SHORT
 *                  before any GPU work.
 *   cursor         64 bytes, zeroed at the start of the object, passed to every window in order: the parts cursor, the source
 *                  object's running CRC and length, and the chunk count (messages name a chunk by its number in the object).
 *                  Updated on success, without a defined value after a failure.
 *   object_ends_here  != 0 on the last window (which may be empty): then *source_crc32c is the CRC-32C of the old object and
 *                  *object_crc32c that of the new object (FULL_OBJECT).  Neither is written before the end or on failure.
 * Returns the first failure in object order; within a batch: the first bad tag (TSGPU_E_AUTH, "Tag mismatch in chunk <k>"), then
 * VERIFY (TSGPU_E_VERIFY).  No byte of a failing batch reaches dst; earlier batches may already be there.  A failed call writes no
 * CRC.  Buffers and cost: DESIGN.md §3, §4.1, §8.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct tsgpu_rekey_cursor { uint64_t opaque[8]; } tsgpu_rekey_cursor;
int tsgpu_rekey_object(tsgpu_ctx* ctx, uint32_t flags,
                       const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                       const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                       const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs,
                       uint8_t* dst, uint64_t dst_cap,
                       uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts,
                       tsgpu_rekey_cursor* cursor, int object_ends_here,
                       uint32_t* source_crc32c, uint32_t* object_crc32c);
/* The CRC-64/NVME twin: the same arguments, rules, errors and output bytes, with 64-bit part, source and object words. */
int tsgpu_rekey_object_crc64(tsgpu_ctx* ctx, uint32_t flags,
                             const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes, uint32_t n_chunks,
                             const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                             const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs,
                             uint8_t* dst, uint64_t dst_cap,
                             uint64_t part_size, uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts,
                             tsgpu_rekey_cursor* cursor, int object_ends_here,
                             uint64_t* source_crc64, uint64_t* object_crc64);

/* ---------------------------------------------------------------------------------------------------------
 * tsgpu_encrypt_object — the chunks of a stored unencrypted object encrypted with AES-GCM and nothing decoded: for turning
 * encryption on for a segment already in the bucket.  A stored chunk, compressed or plain, is exactly the plaintext that
 * EncryptionChunkEnumeration encrypts, so the new chunk i is IV_i || AES-256-GCM(key, IV_i, aad, chunk i) || TAG, 28 bytes longer,
 * and the frames stay byte for byte what they were (a Content_Checksum they carry included): the new object decodes to the same
 * segment.  One GCM pass per byte; no decoder runs.  The call serves both objects of a segment: the .log object (its chunks by the
 * chunk index) and the .indexes object (its blobs at their SegmentIndexesV1 positions and sizes).
 *
 *   flags          TSGPU_FLAG_ZSTD when the object is compressed (the manifest's `compression`), and TSGPU_FLAG_VERIFY; any other
 *                  bit fails with TSGPU_E_ARG, TSGPU_FLAG_AES with a message that points at tsgpu_rekey_object (the object is
 *                  already encrypted).  TSGPU_VERIFY=1 turns VERIFY on; TSGPU_ZSTD_MODE and TSGPU_ZSTD_CHECKSUM have nothing to act
 *                  on.  With VERIFY every new chunk of a batch is decrypted again by the separate decrypt kernels and compared
 *                  with its source chunk on the GPU before any byte of the batch is released; a difference fails with
 *                  TSGPU_E_VERIFY naming the chunk and the first differing byte.
 *   src, src_len, chunk_sizes, n_chunks   the window's chunks back to back.
 *   original_chunk_size, original_file_size   the chunk index of a .log object (> 0): the chunks are walked as tsgpu_check_object
 *                  walks them, chunk k holding the size the index gives it, and at object_ends_here the chunk count must be the
 *                  index's (an empty segment's object is its one chunk of 0 bytes).  Without ZSTD each chunk's size must be its
 *                  index size.  With ZSTD each non-empty chunk must be one frame that the decoder's index stage accepts: the magic
 *                  number, no Dictionary_ID, a Frame_Content_Size equal to the index size, a block walk that ends at a last block
 *                  without a reserved type inside the chunk, and after the frame only the announced Content_Checksum and
 *                  skippable frames.  The Content_Checksum is not verified: that needs the decoded bytes.  A failure is
 *                  TSGPU_E_CORRUPT with tsgpu_check_object's messages ("Invalid zstd frame in chunk <k> (code 2)", "chunk <k>
 *                  decoded to <n> bytes, the chunk index gives <m>": for a frame, n is its Frame_Content_Size).
 *                  0 for an .indexes object: its chunks are the index blobs, only the size bound below applies, and ZSTD fails
 *                  with TSGPU_E_ARG.
 *   key, aad, ivs  the data key and AAD, and one 12-byte IV per chunk.  No two non-empty chunks of the window may get the same IV
 *                  (TSGPU_E_ARG, before any GPU work: tsgpu_rewrite_object's message).
 *   dst, dst_cap, new_transformed_sizes   receive exactly the sum of the new sizes: new_transformed_sizes[i] = chunk_sizes[i] + 28,
 *                  or 0 for a chunk of 0 bytes, which passes through as 0 bytes and takes no IV (an empty index blob, the empty
 *                  segment's chunk: what transformIndex writes for an empty index).  A smaller dst_cap fails with TSGPU_E_SHORT,
 *                  and a chunk whose new size does not fit the context's transformed slot (what tsgpu_detransform takes) with
 *                  TSGPU_E_ARG, both before any GPU work.
 *   part_size, part_crc32c, part_cap, n_parts   as tsgpu_transform_parts, with an exact bound: part_cap >= floor((carried +
 *                  sum(new sizes)) / part_size) + (object_ends_here ? 1 : 0); a smaller part_cap fails with TSGPU_E_SHORT before any
 *                  GPU work.
 *   cursor         64 bytes, zeroed at the start of the object, passed to every window in order: the parts cursor, the source
 *                  object's running CRC and length, and the chunk count (messages name a chunk by its number in the object).
 *                  Updated on success, without a defined value after a failure.
 *   object_ends_here  != 0 on the last window (which may be empty): then *source_crc32c is the CRC-32C of the old object and
 *                  *object_crc32c that of the new object (FULL_OBJECT).  Neither is written before the end or on failure.
 * Returns the first failure in object order; within a batch: the frame and size checks (TSGPU_E_CORRUPT), then VERIFY
 * (TSGPU_E_VERIFY).  No byte of a failing batch reaches dst; earlier batches may already be there.  A failed call writes no CRC.
 * Buffers and cost: DESIGN.md §3, §8.
 * --------------------------------------------------------------------------------------------------------- */
typedef struct tsgpu_encrypt_cursor { uint64_t opaque[8]; } tsgpu_encrypt_cursor;
int tsgpu_encrypt_object(tsgpu_ctx* ctx, uint32_t flags,
                         const uint8_t* src, uint64_t src_len, const uint32_t* chunk_sizes, uint32_t n_chunks,
                         uint32_t original_chunk_size, uint64_t original_file_size,
                         const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                         uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                         uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts,
                         tsgpu_encrypt_cursor* cursor, int object_ends_here,
                         uint32_t* source_crc32c, uint32_t* object_crc32c);
/* The CRC-64/NVME twin: the same arguments, rules, errors and output bytes, with 64-bit part, source and object words. */
int tsgpu_encrypt_object_crc64(tsgpu_ctx* ctx, uint32_t flags,
                               const uint8_t* src, uint64_t src_len, const uint32_t* chunk_sizes, uint32_t n_chunks,
                               uint32_t original_chunk_size, uint64_t original_file_size,
                               const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                               uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                               uint64_t part_size, uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts,
                               tsgpu_encrypt_cursor* cursor, int object_ends_here,
                               uint64_t* source_crc64, uint64_t* object_crc64);

/* ---------------------------------------------------------------------------------------------------------
 * Device-resident variants (inputs and outputs already in HBM of device `device_index` of the context; used by
 * bench.py for the kernel-side throughput and by callers that keep segments on the GPU).  Layouts:
 *   original side     contiguous, chunk i at i * chunk_size
 *   transformed side  one slot per chunk, slot i at i * slot_stride; the chunk's bytes start at
 *                     slot + TSGPU_SLOT_HEAD so that the ciphertext / frame body is 16-byte aligned
 * All pointers are device pointers except key/aad/ivs (host).  `stream` is a cudaStream_t (0 = default).
 * The calls enqueue work and return without synchronising; sizes/status land in device memory.  Consecutive device
 * calls on one context may use different streams: the library orders each call behind the previous one with events
 * (they share one descriptor block and scratch arena per device), so they execute back to back, never concurrently.
 * Sizes read from device memory are untrusted: a chunk larger than its slot / destination is reported in d_status
 * (1 for the AES stage, 2 for zstd) and nothing is written for it.
 * --------------------------------------------------------------------------------------------------------- */
#define TSGPU_SLOT_HEAD 4
uint64_t tsgpu_slot_stride(uint32_t flags, uint32_t chunk_size);
int tsgpu_transform_device(tsgpu_ctx* ctx, int device_index, uint32_t flags,
                           const uint8_t* d_src, uint64_t src_len, uint32_t chunk_size,
                           const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                           uint8_t* d_slots, uint64_t slot_stride, uint32_t* d_transformed_sizes,
                           void* stream);
int tsgpu_detransform_device(tsgpu_ctx* ctx, int device_index, uint32_t flags,
                             const uint8_t* d_slots, uint64_t slot_stride, const uint32_t* d_transformed_sizes,
                             uint32_t n_chunks, uint32_t chunk_size,
                             const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                             uint8_t* d_dst, uint32_t* d_original_sizes, uint32_t* d_status,
                             void* stream);
/* Number of kernels this context has launched so far (bench.py reports it as gpu_launches). */
uint64_t tsgpu_launch_count(const tsgpu_ctx* ctx);
/* Which decode path zstd frames took so far on this context: out[0] 64 KiB regions executed in shared memory (dense-mode frames
 * of this library's writer), out[1] frames handed from a region / block to the frame executor, out[2] frames executed whole
 * (frames written by libzstd, i.e. by the reference), out[3] frames on the serial fallback kernel, out[4] self-contained 8 KiB
 * blocks executed by a warp each (speed-mode frames of this library's writer), out[5..7] reserved (0).
 * The read-back decodes of TSGPU_FLAG_VERIFY count here like any other decode.
 * Synchronises the context's devices. */
int tsgpu_decode_path_stats(tsgpu_ctx* ctx, uint64_t out[8]);
/* Optional per-kernel timing with CUDA events recorded on the launching stream (bench.py's roofline numbers).
 * report: JSON {"kernel": {"launches": n, "ms": total}, ...}; synchronises the context's devices. */
int tsgpu_profile_enable(tsgpu_ctx* ctx, int on);
int tsgpu_profile_report(tsgpu_ctx* ctx, char* out, uint32_t* out_len);

/* ---------------------------------------------------------------------------------------------------------
 * ChunkIndex plumbing (host side; tiny, integer only).
 *   tsgpu_chunk_positions      exclusive prefix sums of AbstractChunkIndex.materializeChunks (AbstractChunkIndex.java:52-72);
 *                              runs the warp-shuffle scan kernel (K5) on device 0 of the context.  `positions` receives
 *                              n + 1 values: positions[i] = start of chunk i, positions[n] = total — allocate n + 1 entries
 *   tsgpu_chunk_sizes_encode / decode   ChunkSizesBinaryCodec.encode/decode (ChunkSizesBinaryCodec.java:104-202)
 *   tsgpu_transformed_chunks_serialize / deserialize   TransformedChunksSerializer / Deserializer (:30-52 / :36-49)
 *   tsgpu_chunk_index_json     Jackson form of Fixed/VariableSizeChunkIndex (ChunkIndexSerializationTest.java:63-74)
 * --------------------------------------------------------------------------------------------------------- */
int tsgpu_chunk_positions(tsgpu_ctx* ctx, const uint32_t* sizes, uint32_t n, uint64_t* positions);
int tsgpu_chunk_sizes_encode(const int32_t* v, uint32_t n, uint8_t* out, uint32_t* out_len);
int tsgpu_chunk_sizes_decode(const uint8_t* in, uint32_t in_len, int32_t* out, uint32_t* n);
int tsgpu_transformed_chunks_serialize(const int32_t* v, uint32_t n, char* out, uint32_t* out_len);
/* Same field, compressed like the reference compresses it (TransformedChunksSerializer.java:40-48 runs libzstd over the codec
 * bytes): the codec bytes go through this library's dense compressor as one chunk and the shorter of {that frame, the Raw-block
 * frame of the ctx-less call} is kept — lists that repeat or cluster shrink as they do in the reference's manifests.  Frames of
 * both calls are read by TransformedChunksDeserializer.java:36-49 and by tsgpu_transformed_chunks_deserialize. */
int tsgpu_transformed_chunks_serialize_ctx(tsgpu_ctx* ctx, const int32_t* v, uint32_t n, char* out, uint32_t* out_len);
/* deserialize needs a context: frames written by the reference are libzstd-compressed and are decoded on the GPU */
int tsgpu_transformed_chunks_deserialize(tsgpu_ctx* ctx, const char* b64, int32_t* out, uint32_t* n);
/* transformed_chunk_size < 0 => variable index built from sizes[0..n); else fixed (sizes may be NULL) */
int tsgpu_chunk_index_json(int32_t original_chunk_size, int32_t original_file_size,
                           int32_t transformed_chunk_size, int32_t final_transformed_chunk_size,
                           const int32_t* sizes, uint32_t n, char* out, uint32_t* out_len);

/* tsgpu_chunk_index_json with the variable index's transformedChunks compressed (tsgpu_transformed_chunks_serialize_ctx). */
int tsgpu_chunk_index_json_ctx(tsgpu_ctx* ctx, int32_t original_chunk_size, int32_t original_file_size,
                               int32_t transformed_chunk_size, int32_t final_transformed_chunk_size,
                               const int32_t* sizes, uint32_t n, char* out, uint32_t* out_len);

#ifdef __cplusplus
}
#endif
#endif
