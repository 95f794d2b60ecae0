/*
 * tsoracle.h — CPU ORACLE for the chunk-transform hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg may
 * load this library.  The product (libtsgpu.so) never links, loads or calls anything in oracle/.
 *
 * What it restates (reference paths relative to <reference>/core/src/main/java/io/aiven/kafka/tieredstorage/):
 *   - transform/CompressionChunkEnumeration.java:49-62   one zstd frame per chunk, level 3, contentSize=true,
 *                                                        pledgedSrcSize, fresh ctx per chunk
 *   - transform/EncryptionChunkEnumeration.java:65-84    IV(12) || AES-256-GCM(ct) || TAG(16), AAD per segment
 *   - transform/DecryptionChunkEnumeration.java:53-62, transform/DecompressionChunkEnumeration.java:38-46
 *   - transform/TransformFinisher.java:75-132            index-builder choice + no-transform fast path
 *   - manifest/index/AbstractChunkIndexBuilder.java:39-96, Fixed/VariableSizeChunkIndexBuilder.java
 *   - manifest/index/AbstractChunkIndex.java:52-123      prefix sums, offset lookup, chunksForRange
 *   - manifest/index/serde/ChunkSizesBinaryCodec.java:104-202, TransformedChunksSerializer.java:30-52
 *   - fetch/FetchChunkEnumeration.java:68-138            ranged-fetch chunk selection / skip / bound
 *
 * The byte-level algorithms live in un-vendored third-party code (SURVEY.md §8c):
 *   - com.github.luben:zstd-jni:1.5.6-9 (libzstd 1.5.6)  -> stand-in: system libzstd 1.5.5 via dlopen
 *   - JDK SunJCE "AES/GCM/NoPadding"                      -> stand-in: OpenSSL EVP aes-256-gcm, AND a
 *     plain-C restatement of NIST SP 800-38D (ora_aesgcm_plain) pinned on the GCM-spec AES-256 test cases.
 * Pinning: tests/test_oracle_golden.py checks this oracle against every golden vector the reference's
 * tests hold for the path (ENCODED_CHUNKS, ChunkIndex JSON, codec layouts, Chunk tuples, builder errors).
 * Compressed bytes of real chunks and ciphertexts are "parity unpinned" in the reference itself
 * (its tests are round-trip only); AES-GCM is pinned here by NIST KATs, zstd by cross-decoding.
 */
#ifndef TSORACLE_H
#define TSORACLE_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORA_FLAG_ZSTD 1u
#define ORA_FLAG_AES  2u
#define ORA_IV_SIZE   12
#define ORA_TAG_SIZE  16

#define ORA_OK            0
#define ORA_E_ARG        -1
#define ORA_E_STATE      -2   /* IllegalStateException in the reference */
#define ORA_E_AUTH       -3   /* AEADBadTagException */
#define ORA_E_CORRUPT    -4
#define ORA_E_SHORT      -5   /* destination too small / stream has fewer bytes than expected */
#define ORA_E_NOLIB      -6

const char* ora_last_error(void);
const char* ora_zstd_version(void);

/* ---- zstd (CompressionChunkEnumeration / DecompressionChunkEnumeration) ---- */
size_t  ora_zstd_bound(size_t n);
int64_t ora_zstd_compress_chunk(const uint8_t* src, size_t n, uint8_t* dst, size_t cap);    /* <0 error */
int64_t ora_zstd_compress_level(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int level);      /* test coverage only */
int64_t ora_zstd_compress_checksum(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int level);   /* + Content_Checksum; test coverage only */
int64_t ora_zstd_content_size(const uint8_t* frame, size_t n);                               /* <0: unknown/err */
int64_t ora_zstd_decompress_chunk(const uint8_t* frame, size_t n, uint8_t* dst, size_t cap);

/* ---- AES-256-GCM (EncryptionChunkEnumeration / DecryptionChunkEnumeration) ---- */
/* out = IV || CT || TAG, n + 28 bytes */
int ora_aesgcm_encrypt_chunk(const uint8_t key[32], const uint8_t iv[12], const uint8_t* aad, size_t aad_len,
                             const uint8_t* pt, size_t n, uint8_t* out);
/* in = IV || CT || TAG (m bytes), out = m - 28 bytes; ORA_E_AUTH on tag mismatch */
int ora_aesgcm_decrypt_chunk(const uint8_t key[32], const uint8_t* aad, size_t aad_len,
                             const uint8_t* in, size_t m, uint8_t* out);
/* plain-C NIST SP 800-38D restatement (no OpenSSL), same layouts */
int ora_aesgcm_plain_encrypt(const uint8_t key[32], const uint8_t iv[12], const uint8_t* aad, size_t aad_len,
                             const uint8_t* pt, size_t n, uint8_t* ct, uint8_t tag[16]);
void ora_aes256_encrypt_block(const uint8_t key[32], const uint8_t in[16], uint8_t out[16]);

/* ---- whole-segment transform / detransform (the decorator chains of RemoteStorageManager.java:434-453
 *      and DefaultChunkManager.java:50-70) ---- */
uint64_t ora_transform_bound(uint32_t flags, uint64_t src_len, uint32_t chunk_size);
int ora_transform_segment(uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                          const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                          uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks);
int ora_detransform_chunks(uint32_t flags, const uint8_t* src, const uint32_t* transformed_sizes,
                           uint32_t n_chunks, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                           uint8_t* dst, uint64_t dst_cap, uint32_t* original_sizes);

/* ---- ChunkIndex builders (AbstractChunkIndexBuilder state machine) ---- */
typedef struct ora_index_builder ora_index_builder;
typedef struct {
    int32_t id, original_position, original_size, transformed_position, transformed_size;
} ora_chunk;
typedef struct {
    int is_variable;               /* 0 = fixed, 1 = variable */
    int32_t original_chunk_size, original_file_size;
    int32_t transformed_chunk_size;        /* fixed only */
    int32_t final_transformed_chunk_size;
    int32_t chunk_count;
    int32_t* transformed_chunks;   /* variable only, chunk_count entries (malloc'd) */
} ora_chunk_index;

/* transformed_chunk_size < 0 => variable (TransformChunkEnumeration.transformedChunkSize()==null) */
ora_index_builder* ora_builder_new(int32_t original_chunk_size, int32_t original_file_size,
                                   int32_t transformed_chunk_size);
int  ora_builder_add_chunk(ora_index_builder*, int32_t transformed_chunk_size);
int  ora_builder_finish(ora_index_builder*, int32_t final_transformed_chunk_size, ora_chunk_index** out);
void ora_builder_free(ora_index_builder*);

int  ora_index_new_fixed(int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, ora_chunk_index** out);
int  ora_index_new_variable(int32_t ocs, int32_t ofs, const int32_t* sizes, int32_t n, ora_chunk_index** out);
void ora_index_free(ora_chunk_index*);
int32_t ora_index_materialized_count(const ora_chunk_index*);         /* max(1, chunk_count) */
int  ora_index_chunks(const ora_chunk_index*, ora_chunk* out);        /* materializeChunks */
/* returns 1 found, 0 "null" (offset >= file size), <0 error */
int  ora_index_find(const ora_chunk_index*, int32_t offset, ora_chunk* out);
int  ora_index_chunks_for_range(const ora_chunk_index*, int32_t from, int32_t to, ora_chunk* out, int32_t cap);
/* JSON exactly as Jackson writes it (ChunkIndexSerializationTest.java:63-74) */
int  ora_index_to_json(const ora_chunk_index*, char* out, size_t cap);

/* ---- ChunkSizesBinaryCodec + TransformedChunksSerializer ---- */
int64_t ora_codec_encode(const int32_t* v, int32_t n, uint8_t* out, size_t cap);
int32_t ora_codec_decode(const uint8_t* in, size_t n, int32_t* out, int32_t cap);
int64_t ora_transformed_chunks_serialize(const int32_t* v, int32_t n, char* out, size_t cap);   /* base64(zstd(codec)) */
int32_t ora_transformed_chunks_deserialize(const char* b64, int32_t* out, int32_t cap);
int64_t ora_base64_encode(const uint8_t* in, size_t n, char* out, size_t cap);
int64_t ora_base64_decode(const char* in, uint8_t* out, size_t cap);

/* ---- FetchChunkEnumeration range math: chunk ids + skip/bound for [from, to] inclusive ---- */
typedef struct { int32_t chunk_id, skip, take; } ora_fetch_piece;
int ora_fetch_plan(const ora_chunk_index*, int32_t from, int32_t to, ora_fetch_piece* out, int32_t cap);

#ifdef __cplusplus
}
#endif
#endif
