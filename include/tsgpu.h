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
 * Environment (read once by tsgpu_create; tuning only): TSGPU_SLOTS=1..16 slots per device, TSGPU_ZSTD_MODE=dense makes
 * TSGPU_FLAG_ZSTD_DENSE the context's default.
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
