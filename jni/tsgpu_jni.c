/*
 * tsgpu_jni.c — JNI glue between the reference's Java operator surface and the C-ABI of include/tsgpu.h.
 * There is no JDK in this repository's build image: the tests compile this file against a test-only stand-in for
 * <jni.h> and drive it through a fake JNIEnv (tests/cpp/test_jni_shim.c).  Build on the broker host with
 *   gcc -shared -fPIC -I$JAVA_HOME/include -I$JAVA_HOME/include/linux -Iinclude jni/tsgpu_jni.c -L<pkg> -ltsgpu -o libtsgpu_jni.so
 * Java side: jni/io/aiven/kafka/tieredstorage/transform/gpu/{TsGpu,RecordsCursor,PartsCursor,CheckCursor,RewriteCursor,RekeyCursor,EncryptCursor,Crc64,PinnedPool,GpuTransformChunkEnumeration,GpuDetransformChunkEnumeration}.java
 * (implement TransformChunkEnumeration / DetransformChunkEnumeration of the reference, core/M/transform/TransformChunkEnumeration.java:28-42,
 * DetransformChunkEnumeration.java:28-29) and jni/io/aiven/kafka/tieredstorage/fetch/gpu/GpuChunkManager.java (ChunkManager, fetch/ChunkManager.java).
 *
 * Buffers are direct ByteBuffers (ideally over tsgpu_host_alloc'ed pinned memory, see allocPinned), so there is no
 * JNI array copy on the data path.  Errors become RuntimeException(tsgpu_last_error()), which is what the
 * reference's operators throw and RemoteStorageManager converts (RemoteStorageManager.java:258-267, :566-575).
 */
#include <jni.h>
#include <stdint.h>
#include "tsgpu.h"

#define CLS "io/aiven/kafka/tieredstorage/transform/gpu/TsGpu"

static void throw_rt(JNIEnv* env, int rc) {
    jclass ex = (*env)->FindClass(env, rc == TSGPU_E_ARG ? "java/lang/IllegalArgumentException" : "java/lang/RuntimeException");
    (*env)->ThrowNew(env, ex, tsgpu_last_error());
}
static void throw_arg(JNIEnv* env, const char* msg) {
    (*env)->ThrowNew(env, (*env)->FindClass(env, "java/lang/IllegalArgumentException"), msg);
}
/* A direct ByteBuffer's address and capacity, or NULL with an IllegalArgumentException pending: a heap buffer has no
 * address (GetDirectBufferAddress gives NULL, the capacity -1) and `need` bytes must fit. */
static uint8_t* direct(JNIEnv* env, jobject buf, jlong need, jlong* cap, const char* what) {
    if (!buf) { throw_arg(env, what); return NULL; }
    uint8_t* p = (uint8_t*)(*env)->GetDirectBufferAddress(env, buf);
    const jlong c = (*env)->GetDirectBufferCapacity(env, buf);
    if (!p || c < 0) { throw_arg(env, what); return NULL; }
    if (need < 0 || need > c) { throw_arg(env, "length exceeds the direct buffer's capacity"); return NULL; }
    if (cap) *cap = c;
    return p;
}

JNIEXPORT jlong JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_create(JNIEnv* env, jclass c, jintArray devices,
                                                                                     jint maxChunkBytes, jint maxBatch) {
    tsgpu_ctx* ctx = NULL;
    jint n = devices ? (*env)->GetArrayLength(env, devices) : 0;
    jint* ids = n ? (*env)->GetIntArrayElements(env, devices, NULL) : NULL;
    int rc = tsgpu_create((const int*)ids, n, (uint32_t)maxChunkBytes, (uint32_t)maxBatch, &ctx);
    if (ids) (*env)->ReleaseIntArrayElements(env, devices, ids, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return 0; }
    return (jlong)(intptr_t)ctx;
}
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_destroy(JNIEnv* env, jclass c, jlong h) {
    tsgpu_destroy((tsgpu_ctx*)(intptr_t)h);
}
JNIEXPORT jobject JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_allocPinned(JNIEnv* env, jclass c, jlong bytes) {
    void* p = tsgpu_host_alloc((size_t)bytes);
    return p ? (*env)->NewDirectByteBuffer(env, p, bytes) : NULL;
}
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_freePinned(JNIEnv* env, jclass c, jobject buf) {
    if (buf) tsgpu_host_free((*env)->GetDirectBufferAddress(env, buf));
}
JNIEXPORT jlong JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_transformBound(JNIEnv* env, jclass c, jint flags,
                                                                                             jlong srcLen, jint chunkSize) {
    return (jlong)tsgpu_transform_bound((uint32_t)flags, (uint64_t)srcLen, (uint32_t)chunkSize);
}
/* The part-checksum arguments of tsgpu_transform_parts (PartsCursor.transformParts), or with crcs64 of
 * tsgpu_transform_parts_crc64 (Crc64.transformParts). */
typedef struct {
    uint64_t part_size; tsgpu_parts_cursor* cursor;
    uint32_t* crcs; uint32_t cap; uint32_t n; uint32_t object_crc;
    uint64_t* crcs64; uint64_t object_crc64;
} parts_args;
/* tsgpu_transform, tsgpu_transform_cursor when `cursor` is given, or tsgpu_transform_parts[_crc64] when `parts` is; returns the
 * number of chunks, or -1 with an exception pending.  transformedSizes (int[]) receives one entry per chunk. */
static jint transform_call(JNIEnv* env, jlong h, jint flags, jobject src, jlong srcLen, jint chunkSize, jbyteArray key, jbyteArray aad,
                           jbyteArray ivs, jobject dst, jintArray transformedSizes, tsgpu_records_cursor* cursor, int segmentEndsHere,
                           parts_args* parts) {
    jlong dcap = 0;
    uint8_t* s = direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer");
    if (!s) return -1;
    uint8_t* d = direct(env, dst, 0, &dcap, "dst must be a direct ByteBuffer");
    if (!d) return -1;
    if (!transformedSizes) { throw_arg(env, "transformedSizes cannot be null"); return -1; }
    if ((flags & TSGPU_FLAG_AES) && key && (*env)->GetArrayLength(env, key) != 32) { throw_arg(env, "data key must be 32 bytes"); return -1; }
    jbyte* k = key ? (*env)->GetByteArrayElements(env, key, NULL) : NULL;
    jbyte* a = aad ? (*env)->GetByteArrayElements(env, aad, NULL) : NULL;
    jbyte* iv = ivs ? (*env)->GetByteArrayElements(env, ivs, NULL) : NULL;
    jint alen = aad ? (*env)->GetArrayLength(env, aad) : 0;
    uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    if ((flags & TSGPU_FLAG_AES) && iv && chunkSize > 0 &&
        (jlong)(*env)->GetArrayLength(env, ivs) < TSGPU_IV_SIZE * ((srcLen + chunkSize - 1) / chunkSize)) {
        if (k) (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
        if (a) (*env)->ReleaseByteArrayElements(env, aad, a, JNI_ABORT);
        (*env)->ReleaseByteArrayElements(env, ivs, iv, JNI_ABORT);
        throw_arg(env, "ivs holds fewer than 12 bytes per chunk");
        return -1;
    }
    jint* sizes = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    int rc = parts && parts->crcs64
        ? tsgpu_transform_parts_crc64((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (uint32_t)chunkSize, (const uint8_t*)k,
                                      (const uint8_t*)a, (uint32_t)alen, (const uint8_t*)iv, d, (uint64_t)dcap, (uint32_t*)sizes, &n,
                                      cursor, segmentEndsHere, parts->part_size, parts->cursor, parts->crcs64, parts->cap, &parts->n,
                                      &parts->object_crc64)
        : parts
        ? tsgpu_transform_parts((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (uint32_t)chunkSize, (const uint8_t*)k,
                                (const uint8_t*)a, (uint32_t)alen, (const uint8_t*)iv, d, (uint64_t)dcap, (uint32_t*)sizes, &n,
                                cursor, segmentEndsHere, parts->part_size, parts->cursor, parts->crcs, parts->cap, &parts->n,
                                &parts->object_crc)
        : cursor
        ? tsgpu_transform_cursor((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (uint32_t)chunkSize, (const uint8_t*)k,
                                 (const uint8_t*)a, (uint32_t)alen, (const uint8_t*)iv, d, (uint64_t)dcap, (uint32_t*)sizes, &n,
                                 cursor, segmentEndsHere)
        : tsgpu_transform((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (uint32_t)chunkSize, (const uint8_t*)k,
                          (const uint8_t*)a, (uint32_t)alen, (const uint8_t*)iv, d, (uint64_t)dcap, (uint32_t*)sizes, &n);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, sizes, 0);
    if (k) (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
    if (a) (*env)->ReleaseByteArrayElements(env, aad, a, JNI_ABORT);
    if (iv) (*env)->ReleaseByteArrayElements(env, ivs, iv, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return -1; }           /* TSGPU_E_RECORDS too: a RuntimeException, the copy is retried */
    return (jint)n;
}
JNIEXPORT jint JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_transform(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jint chunkSize, jbyteArray key, jbyteArray aad,
    jbyteArray ivs, jobject dst, jintArray transformedSizes) {
    return transform_call(env, h, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, NULL, 0, NULL);
}
/* One window of a segment (RecordsCursor.transformCursor): `cursor` is a direct ByteBuffer of at least 64 bytes holding the
 * tsgpu_records_cursor (zeros at the start of the segment), updated in place; segmentEndsHere marks the segment's last window. */
JNIEXPORT jint JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_RecordsCursor_transformCursor(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jint chunkSize, jbyteArray key, jbyteArray aad,
    jbyteArray ivs, jobject dst, jintArray transformedSizes, jobject cursor, jboolean segmentEndsHere) {
    jlong ccap = 0;
    tsgpu_records_cursor* cur = (tsgpu_records_cursor*)direct(env, cursor, 0, &ccap, "cursor must be a direct ByteBuffer of 64 bytes");
    if (!cur) return -1;
    if (ccap < (jlong)sizeof(tsgpu_records_cursor)) { throw_arg(env, "cursor must be a direct ByteBuffer of 64 bytes"); return -1; }
    return transform_call(env, h, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, cur, segmentEndsHere ? 1 : 0, NULL);
}
/* One window of a segment with the CRC-32C of its upload parts (PartsCursor.transformParts): `recordsCursor` as transformCursor
 * takes it (64 bytes), `partsCursor` a direct ByteBuffer of at least 32 bytes holding the tsgpu_parts_cursor (zeros at the start
 * of the object), both updated in place.  partCrc32c (int[]) receives the CRCs of the parts the window completed, in part order;
 * partsOut (int[2]) receives their count and, on the segment's last window, the object's CRC-32C. */
JNIEXPORT jint JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_PartsCursor_transformParts(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jint chunkSize, jbyteArray key, jbyteArray aad,
    jbyteArray ivs, jobject dst, jintArray transformedSizes, jobject recordsCursor, jboolean segmentEndsHere, jlong partSize,
    jobject partsCursor, jintArray partCrc32c, jintArray partsOut) {
    jlong rcap = 0, pcap = 0;
    tsgpu_records_cursor* rcur = (tsgpu_records_cursor*)direct(env, recordsCursor, 0, &rcap, "records cursor must be a direct ByteBuffer of 64 bytes");
    if (!rcur) return -1;
    if (rcap < (jlong)sizeof(tsgpu_records_cursor)) { throw_arg(env, "records cursor must be a direct ByteBuffer of 64 bytes"); return -1; }
    tsgpu_parts_cursor* pcur = (tsgpu_parts_cursor*)direct(env, partsCursor, 0, &pcap, "parts cursor must be a direct ByteBuffer of 32 bytes");
    if (!pcur) return -1;
    if (pcap < (jlong)sizeof(tsgpu_parts_cursor)) { throw_arg(env, "parts cursor must be a direct ByteBuffer of 32 bytes"); return -1; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return -1; }
    if (!partCrc32c || !partsOut) { throw_arg(env, "partCrc32c and partsOut cannot be null"); return -1; }
    if ((*env)->GetArrayLength(env, partsOut) < 2) { throw_arg(env, "partsOut must hold 2 ints"); return -1; }
    parts_args pa = {(uint64_t)partSize, pcur, NULL, (uint32_t)(*env)->GetArrayLength(env, partCrc32c), 0, 0, NULL, 0};
    jint* crcs = (*env)->GetIntArrayElements(env, partCrc32c, NULL);
    pa.crcs = (uint32_t*)crcs;
    const jint n = transform_call(env, h, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, rcur,
                                  segmentEndsHere ? 1 : 0, &pa);
    (*env)->ReleaseIntArrayElements(env, partCrc32c, crcs, n < 0 ? JNI_ABORT : 0);
    if (n < 0) return -1;
    jint* out = (*env)->GetIntArrayElements(env, partsOut, NULL);
    out[0] = (jint)pa.n; out[1] = (jint)pa.object_crc;
    (*env)->ReleaseIntArrayElements(env, partsOut, out, 0);
    return n;
}
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_detransform(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray transformedSizes, jbyteArray key, jbyteArray aad,
    jobject dst, jintArray originalSizes) {
    jlong dcap = 0;
    uint8_t* s = direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer");
    if (!s) return;
    uint8_t* d = direct(env, dst, 0, &dcap, "dst must be a direct ByteBuffer");
    if (!d) return;
    if (!transformedSizes || !originalSizes) { throw_arg(env, "chunks cannot be null"); return; }
    if ((*env)->GetArrayLength(env, originalSizes) < (*env)->GetArrayLength(env, transformedSizes)) { throw_arg(env, "originalSizes is shorter than transformedSizes"); return; }
    if ((flags & TSGPU_FLAG_AES) && key && (*env)->GetArrayLength(env, key) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    jbyte* k = key ? (*env)->GetByteArrayElements(env, key, NULL) : NULL;
    jbyte* a = aad ? (*env)->GetByteArrayElements(env, aad, NULL) : NULL;
    jint alen = aad ? (*env)->GetArrayLength(env, aad) : 0;
    uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    jint* ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    jint* os = (*env)->GetIntArrayElements(env, originalSizes, NULL);
    int rc = tsgpu_detransform((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (const uint32_t*)ts, n, (const uint8_t*)k,
                               (const uint8_t*)a, (uint32_t)alen, d, (uint64_t)dcap, (uint32_t*)os);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, ts, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, originalSizes, os, 0);
    if (k) (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
    if (a) (*env)->ReleaseByteArrayElements(env, aad, a, JNI_ABORT);
    if (rc) throw_rt(env, rc);
}

/* One window of a stored object checked against its chunk index (CheckCursor.checkObject, tsgpu_check_object): `cursor` a direct
 * ByteBuffer of at least 128 bytes holding the tsgpu_check_cursor (zeros at the start of the object), updated in place;
 * crcsOut (int[2]) receives, on the object's last window, the CRC-32C of the object and of the decoded segment. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_CheckCursor_checkObject(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray transformedSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray key, jbyteArray aad, jobject cursor, jboolean objectEndsHere, jintArray crcsOut) {
    jlong ccap = 0;
    uint8_t* s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !s) return;
    tsgpu_check_cursor* cur = (tsgpu_check_cursor*)direct(env, cursor, 0, &ccap, "check cursor must be a direct ByteBuffer of 128 bytes");
    if (!cur) return;
    if (ccap < (jlong)sizeof(tsgpu_check_cursor)) { throw_arg(env, "check cursor must be a direct ByteBuffer of 128 bytes"); return; }
    if (!transformedSizes) { throw_arg(env, "chunks cannot be null"); return; }
    if (!crcsOut || (*env)->GetArrayLength(env, crcsOut) < 2) { throw_arg(env, "crcsOut must hold 2 ints"); return; }
    if (originalChunkSize < 1) { throw_arg(env, "Original chunk size must be positive"); return; }
    if (originalFileSize < 0) { throw_arg(env, "Original file size must be non-negative"); return; }
    if ((flags & TSGPU_FLAG_AES) && key && (*env)->GetArrayLength(env, key) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    jbyte* k = key ? (*env)->GetByteArrayElements(env, key, NULL) : NULL;
    jbyte* a = aad ? (*env)->GetByteArrayElements(env, aad, NULL) : NULL;
    jint alen = aad ? (*env)->GetArrayLength(env, aad) : 0;
    uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    jint* ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    uint32_t crcs[2] = {0, 0};
    int rc = tsgpu_check_object((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (const uint32_t*)ts, n,
                                (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)k, (const uint8_t*)a,
                                (uint32_t)alen, cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1]);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, ts, JNI_ABORT);
    if (k) (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
    if (a) (*env)->ReleaseByteArrayElements(env, aad, a, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    if (objectEndsHere) {
        jint* out = (*env)->GetIntArrayElements(env, crcsOut, NULL);
        out[0] = (jint)crcs[0]; out[1] = (jint)crcs[1];
        (*env)->ReleaseIntArrayElements(env, crcsOut, out, 0);
    }
}

/* One window of a stored object rewritten under a new key or with compression or encryption added (RewriteCursor.rewriteObject,
 * tsgpu_rewrite_object): `cursor` a direct ByteBuffer of at least 192 bytes holding the tsgpu_rewrite_cursor (zeros at the start
 * of the object), updated in place; dst a direct ByteBuffer receiving the window's new chunks, newTransformedSizes their sizes
 * (one per chunk of the window), partCrcs the CRC-32C of every upload part the window completes (its length is part_cap) and
 * nPartsOut[0] their count; crcsOut (int[3]) receives, on the object's last window, the CRC-32C of the old object, of the new
 * object and of the decoded segment.  toIvs: 12 bytes per chunk of the window when toFlags has AES. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_RewriteCursor_rewriteObject(
    JNIEnv* env, jclass c, jlong h, jint fromFlags, jobject src, jlong srcLen, jintArray transformedSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray fromKey, jbyteArray fromAad, jint toFlags, jbyteArray toKey, jbyteArray toAad,
    jbyteArray toIvs, jobject dst, jlong dstCap, jintArray newTransformedSizes, jlong partSize, jintArray partCrcs,
    jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jintArray crcsOut) {
    jlong ccap = 0;
    uint8_t* s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !s) return;
    uint8_t* d = dstCap ? direct(env, dst, dstCap, NULL, "dst must be a direct ByteBuffer") : NULL;
    if (dstCap && !d) return;
    tsgpu_rewrite_cursor* cur = (tsgpu_rewrite_cursor*)direct(env, cursor, 0, &ccap, "rewrite cursor must be a direct ByteBuffer of 192 bytes");
    if (!cur) return;
    if (ccap < (jlong)sizeof(tsgpu_rewrite_cursor)) { throw_arg(env, "rewrite cursor must be a direct ByteBuffer of 192 bytes"); return; }
    if (!transformedSizes) { throw_arg(env, "chunks cannot be null"); return; }
    const uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    if (!newTransformedSizes || (uint32_t)(*env)->GetArrayLength(env, newTransformedSizes) < n) {
        throw_arg(env, "newTransformedSizes must hold one int per chunk"); return;
    }
    if (!partCrcs) { throw_arg(env, "partCrcs cannot be null"); return; }
    if (!nPartsOut || (*env)->GetArrayLength(env, nPartsOut) < 1) { throw_arg(env, "nPartsOut must hold 1 int"); return; }
    if (!crcsOut || (*env)->GetArrayLength(env, crcsOut) < 3) { throw_arg(env, "crcsOut must hold 3 ints"); return; }
    if (originalChunkSize < 1) { throw_arg(env, "Original chunk size must be positive"); return; }
    if (originalFileSize < 0) { throw_arg(env, "Original file size must be non-negative"); return; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return; }
    if ((fromFlags & TSGPU_FLAG_AES) && fromKey && (*env)->GetArrayLength(env, fromKey) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    if ((toFlags & TSGPU_FLAG_AES) && toKey && (*env)->GetArrayLength(env, toKey) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    if ((toFlags & TSGPU_FLAG_AES) && n && (!toIvs || (uint32_t)(*env)->GetArrayLength(env, toIvs) < 12 * n)) {
        throw_arg(env, "toIvs must hold 12 bytes per chunk"); return;
    }
    jbyte* fk = fromKey ? (*env)->GetByteArrayElements(env, fromKey, NULL) : NULL;
    jbyte* fa = fromAad ? (*env)->GetByteArrayElements(env, fromAad, NULL) : NULL;
    jint falen = fromAad ? (*env)->GetArrayLength(env, fromAad) : 0;
    jbyte* tk = toKey ? (*env)->GetByteArrayElements(env, toKey, NULL) : NULL;
    jbyte* ta = toAad ? (*env)->GetByteArrayElements(env, toAad, NULL) : NULL;
    jint talen = toAad ? (*env)->GetArrayLength(env, toAad) : 0;
    jbyte* iv = toIvs ? (*env)->GetByteArrayElements(env, toIvs, NULL) : NULL;
    jint* ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    jint* nts = (*env)->GetIntArrayElements(env, newTransformedSizes, NULL);
    const uint32_t cap = (uint32_t)(*env)->GetArrayLength(env, partCrcs);
    jint* pc = (*env)->GetIntArrayElements(env, partCrcs, NULL);
    uint32_t nParts = 0, crcs[3] = {0, 0, 0};
    int rc = tsgpu_rewrite_object((tsgpu_ctx*)(intptr_t)h, (uint32_t)fromFlags, s, (uint64_t)srcLen, (const uint32_t*)ts, n,
                                  (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)fk, (const uint8_t*)fa,
                                  (uint32_t)falen, (uint32_t)toFlags, (const uint8_t*)tk, (const uint8_t*)ta, (uint32_t)talen,
                                  (const uint8_t*)iv, d, (uint64_t)dstCap, (uint32_t*)nts, (uint64_t)partSize, (uint32_t*)pc, cap,
                                  &nParts, cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1], &crcs[2]);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, ts, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, newTransformedSizes, nts, rc ? JNI_ABORT : 0);
    (*env)->ReleaseIntArrayElements(env, partCrcs, pc, rc ? JNI_ABORT : 0);
    if (fk) (*env)->ReleaseByteArrayElements(env, fromKey, fk, JNI_ABORT);
    if (fa) (*env)->ReleaseByteArrayElements(env, fromAad, fa, JNI_ABORT);
    if (tk) (*env)->ReleaseByteArrayElements(env, toKey, tk, JNI_ABORT);
    if (ta) (*env)->ReleaseByteArrayElements(env, toAad, ta, JNI_ABORT);
    if (iv) (*env)->ReleaseByteArrayElements(env, toIvs, iv, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    jint* np = (*env)->GetIntArrayElements(env, nPartsOut, NULL);
    np[0] = (jint)nParts;
    (*env)->ReleaseIntArrayElements(env, nPartsOut, np, 0);
    if (objectEndsHere) {
        jint* out = (*env)->GetIntArrayElements(env, crcsOut, NULL);
        out[0] = (jint)crcs[0]; out[1] = (jint)crcs[1]; out[2] = (jint)crcs[2];
        (*env)->ReleaseIntArrayElements(env, crcsOut, out, 0);
    }
}

/* ---------------------------------------------------------------------------------------------------------------------------
 * CRC-64/NVME twins (Crc64.java).  Each takes the arguments of its CRC-32C twin above; the 64-bit checksums come back in direct
 * ByteBuffers, one 8-byte word each in the platform's byte order (ByteOrder.nativeOrder() on the Java side). */

/* The cursors of a parts call, checked as PartsCursor.transformParts checks them; NULL with an exception pending. */
static int parts_cursors(JNIEnv* env, jobject recordsCursor, jobject partsCursor, jlong partSize, tsgpu_records_cursor** rcur,
                         tsgpu_parts_cursor** pcur) {
    jlong rcap = 0, pcap = 0;
    *rcur = (tsgpu_records_cursor*)direct(env, recordsCursor, 0, &rcap, "records cursor must be a direct ByteBuffer of 64 bytes");
    if (!*rcur) return -1;
    if (rcap < (jlong)sizeof(tsgpu_records_cursor)) { throw_arg(env, "records cursor must be a direct ByteBuffer of 64 bytes"); return -1; }
    *pcur = (tsgpu_parts_cursor*)direct(env, partsCursor, 0, &pcap, "parts cursor must be a direct ByteBuffer of 32 bytes");
    if (!*pcur) return -1;
    if (pcap < (jlong)sizeof(tsgpu_parts_cursor)) { throw_arg(env, "parts cursor must be a direct ByteBuffer of 32 bytes"); return -1; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return -1; }
    return 0;
}

/* Crc64.transformParts: PartsCursor.transformParts with CRC-64/NVME.  partCrc64 (direct, 8 bytes per part: its capacity / 8 is
 * part_cap) receives the CRCs of the parts the window completed, nPartsOut[0] their count, and objectCrc64Out (direct, 8 bytes)
 * on the segment's last window the object's CRC-64/NVME.  Nothing is written on failure. */
JNIEXPORT jint JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_Crc64_transformParts(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jint chunkSize, jbyteArray key, jbyteArray aad,
    jbyteArray ivs, jobject dst, jintArray transformedSizes, jobject recordsCursor, jboolean segmentEndsHere, jlong partSize,
    jobject partsCursor, jobject partCrc64, jintArray nPartsOut, jobject objectCrc64Out) {
    tsgpu_records_cursor* rcur; tsgpu_parts_cursor* pcur;
    if (parts_cursors(env, recordsCursor, partsCursor, partSize, &rcur, &pcur)) return -1;
    jlong ccap = 0;
    uint64_t* crcs = (uint64_t*)direct(env, partCrc64, 0, &ccap, "partCrc64 must be a direct ByteBuffer");
    if (!crcs) return -1;
    jlong ocap = 0;
    uint64_t* obj = (uint64_t*)direct(env, objectCrc64Out, 0, &ocap, "objectCrc64Out must be a direct ByteBuffer of 8 bytes");
    if (!obj) return -1;
    if (ocap < 8) { throw_arg(env, "objectCrc64Out must be a direct ByteBuffer of 8 bytes"); return -1; }
    if (!nPartsOut || (*env)->GetArrayLength(env, nPartsOut) < 1) { throw_arg(env, "nPartsOut must hold 1 int"); return -1; }
    parts_args pa = {(uint64_t)partSize, pcur, NULL, (uint32_t)(ccap / 8), 0, 0, crcs, 0};
    const jint n = transform_call(env, h, flags, src, srcLen, chunkSize, key, aad, ivs, dst, transformedSizes, rcur,
                                  segmentEndsHere ? 1 : 0, &pa);
    if (n < 0) return -1;
    jint* np = (*env)->GetIntArrayElements(env, nPartsOut, NULL);
    np[0] = (jint)pa.n;
    (*env)->ReleaseIntArrayElements(env, nPartsOut, np, 0);
    if (segmentEndsHere) *obj = pa.object_crc64;
    return n;
}

/* Crc64.checkObject: CheckCursor.checkObject with CRC-64/NVME.  crcsOut (direct, 16 bytes) receives, on the object's last window,
 * the CRC-64/NVME of the object and of the decoded segment. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_Crc64_checkObject(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray transformedSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray key, jbyteArray aad, jobject cursor, jboolean objectEndsHere, jobject crcsOut) {
    jlong ccap = 0;
    uint8_t* s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !s) return;
    tsgpu_check_cursor* cur = (tsgpu_check_cursor*)direct(env, cursor, 0, &ccap, "check cursor must be a direct ByteBuffer of 128 bytes");
    if (!cur) return;
    if (ccap < (jlong)sizeof(tsgpu_check_cursor)) { throw_arg(env, "check cursor must be a direct ByteBuffer of 128 bytes"); return; }
    jlong wcap = 0;
    uint64_t* out = (uint64_t*)direct(env, crcsOut, 0, &wcap, "crcsOut must be a direct ByteBuffer of 16 bytes");
    if (!out) return;
    if (wcap < 16) { throw_arg(env, "crcsOut must be a direct ByteBuffer of 16 bytes"); return; }
    if (!transformedSizes) { throw_arg(env, "chunks cannot be null"); return; }
    if (originalChunkSize < 1) { throw_arg(env, "Original chunk size must be positive"); return; }
    if (originalFileSize < 0) { throw_arg(env, "Original file size must be non-negative"); return; }
    if ((flags & TSGPU_FLAG_AES) && key && (*env)->GetArrayLength(env, key) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    jbyte* k = key ? (*env)->GetByteArrayElements(env, key, NULL) : NULL;
    jbyte* a = aad ? (*env)->GetByteArrayElements(env, aad, NULL) : NULL;
    jint alen = aad ? (*env)->GetArrayLength(env, aad) : 0;
    uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    jint* ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    uint64_t crcs[2] = {0, 0};
    int rc = tsgpu_check_object_crc64((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, s, (uint64_t)srcLen, (const uint32_t*)ts, n,
                                      (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)k, (const uint8_t*)a,
                                      (uint32_t)alen, cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1]);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, ts, JNI_ABORT);
    if (k) (*env)->ReleaseByteArrayElements(env, key, k, JNI_ABORT);
    if (a) (*env)->ReleaseByteArrayElements(env, aad, a, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    if (objectEndsHere) { out[0] = crcs[0]; out[1] = crcs[1]; }
}

/* Crc64.rewriteObject: RewriteCursor.rewriteObject with CRC-64/NVME.  partCrc64 (direct, 8 bytes per part: its capacity / 8 is
 * part_cap) receives the CRCs of the upload parts the window completes and nPartsOut[0] their count; crcsOut (direct, 24 bytes)
 * receives, on the object's last window, the CRC-64/NVME of the old object, of the new object and of the decoded segment. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_Crc64_rewriteObject(
    JNIEnv* env, jclass c, jlong h, jint fromFlags, jobject src, jlong srcLen, jintArray transformedSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray fromKey, jbyteArray fromAad, jint toFlags, jbyteArray toKey, jbyteArray toAad,
    jbyteArray toIvs, jobject dst, jlong dstCap, jintArray newTransformedSizes, jlong partSize, jobject partCrc64,
    jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jobject crcsOut) {
    jlong ccap = 0, pcap = 0;
    uint8_t* s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !s) return;
    uint8_t* d = dstCap ? direct(env, dst, dstCap, NULL, "dst must be a direct ByteBuffer") : NULL;
    if (dstCap && !d) return;
    tsgpu_rewrite_cursor* cur = (tsgpu_rewrite_cursor*)direct(env, cursor, 0, &ccap, "rewrite cursor must be a direct ByteBuffer of 192 bytes");
    if (!cur) return;
    if (ccap < (jlong)sizeof(tsgpu_rewrite_cursor)) { throw_arg(env, "rewrite cursor must be a direct ByteBuffer of 192 bytes"); return; }
    uint64_t* pc = (uint64_t*)direct(env, partCrc64, 0, &pcap, "partCrc64 must be a direct ByteBuffer");
    if (!pc) return;
    jlong wcap = 0;
    uint64_t* out = (uint64_t*)direct(env, crcsOut, 0, &wcap, "crcsOut must be a direct ByteBuffer of 24 bytes");
    if (!out) return;
    if (wcap < 24) { throw_arg(env, "crcsOut must be a direct ByteBuffer of 24 bytes"); return; }
    if (!transformedSizes) { throw_arg(env, "chunks cannot be null"); return; }
    const uint32_t n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    if (!newTransformedSizes || (uint32_t)(*env)->GetArrayLength(env, newTransformedSizes) < n) {
        throw_arg(env, "newTransformedSizes must hold one int per chunk"); return;
    }
    if (!nPartsOut || (*env)->GetArrayLength(env, nPartsOut) < 1) { throw_arg(env, "nPartsOut must hold 1 int"); return; }
    if (originalChunkSize < 1) { throw_arg(env, "Original chunk size must be positive"); return; }
    if (originalFileSize < 0) { throw_arg(env, "Original file size must be non-negative"); return; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return; }
    if ((fromFlags & TSGPU_FLAG_AES) && fromKey && (*env)->GetArrayLength(env, fromKey) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    if ((toFlags & TSGPU_FLAG_AES) && toKey && (*env)->GetArrayLength(env, toKey) != 32) { throw_arg(env, "data key must be 32 bytes"); return; }
    if ((toFlags & TSGPU_FLAG_AES) && n && (!toIvs || (uint32_t)(*env)->GetArrayLength(env, toIvs) < 12 * n)) {
        throw_arg(env, "toIvs must hold 12 bytes per chunk"); return;
    }
    jbyte* fk = fromKey ? (*env)->GetByteArrayElements(env, fromKey, NULL) : NULL;
    jbyte* fa = fromAad ? (*env)->GetByteArrayElements(env, fromAad, NULL) : NULL;
    jint falen = fromAad ? (*env)->GetArrayLength(env, fromAad) : 0;
    jbyte* tk = toKey ? (*env)->GetByteArrayElements(env, toKey, NULL) : NULL;
    jbyte* ta = toAad ? (*env)->GetByteArrayElements(env, toAad, NULL) : NULL;
    jint talen = toAad ? (*env)->GetArrayLength(env, toAad) : 0;
    jbyte* iv = toIvs ? (*env)->GetByteArrayElements(env, toIvs, NULL) : NULL;
    jint* ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    jint* nts = (*env)->GetIntArrayElements(env, newTransformedSizes, NULL);
    uint32_t nParts = 0;
    uint64_t crcs[3] = {0, 0, 0};
    int rc = tsgpu_rewrite_object_crc64((tsgpu_ctx*)(intptr_t)h, (uint32_t)fromFlags, s, (uint64_t)srcLen, (const uint32_t*)ts, n,
                                        (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)fk, (const uint8_t*)fa,
                                        (uint32_t)falen, (uint32_t)toFlags, (const uint8_t*)tk, (const uint8_t*)ta, (uint32_t)talen,
                                        (const uint8_t*)iv, d, (uint64_t)dstCap, (uint32_t*)nts, (uint64_t)partSize, pc,
                                        (uint32_t)(pcap / 8), &nParts, cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1], &crcs[2]);
    (*env)->ReleaseIntArrayElements(env, transformedSizes, ts, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, newTransformedSizes, nts, rc ? JNI_ABORT : 0);
    if (fk) (*env)->ReleaseByteArrayElements(env, fromKey, fk, JNI_ABORT);
    if (fa) (*env)->ReleaseByteArrayElements(env, fromAad, fa, JNI_ABORT);
    if (tk) (*env)->ReleaseByteArrayElements(env, toKey, tk, JNI_ABORT);
    if (ta) (*env)->ReleaseByteArrayElements(env, toAad, ta, JNI_ABORT);
    if (iv) (*env)->ReleaseByteArrayElements(env, toIvs, iv, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    jint* np = (*env)->GetIntArrayElements(env, nPartsOut, NULL);
    np[0] = (jint)nParts;
    (*env)->ReleaseIntArrayElements(env, nPartsOut, np, 0);
    if (objectEndsHere) { out[0] = crcs[0]; out[1] = crcs[1]; out[2] = crcs[2]; }
}

/* ---------------------------------------------------------------------------------------------------------------------------
 * Key rotation (RekeyCursor.java): one window of a stored object's AES-GCM chunks re-encrypted under a new key with nothing
 * decoded (tsgpu_rekey_object[_crc64]).  `cursor` a direct ByteBuffer of at least 64 bytes holding the tsgpu_rekey_cursor (zeros
 * at the start of the object), updated in place; dst a direct ByteBuffer receiving exactly the window's bytes (every chunk keeps
 * its size); toIvs 12 bytes per chunk of the window (an empty chunk takes none, its 12 bytes are not read). */

/* The arguments both widths check the same way; the key, AAD and IV arrays pinned.  Returns -1 with an exception pending. */
typedef struct {
    uint8_t* s; uint8_t* d; tsgpu_rekey_cursor* cur; uint32_t n;
    jint* ts; jbyte* fk; jbyte* fa; jint falen; jbyte* tk; jbyte* ta; jint talen; jbyte* iv;
} rekey_args;
static int rekey_begin(JNIEnv* env, jobject src, jlong srcLen, jintArray transformedSizes, jbyteArray fromKey, jbyteArray fromAad,
                       jbyteArray toKey, jbyteArray toAad, jbyteArray toIvs, jobject dst, jlong dstCap, jlong partSize,
                       jintArray nPartsOut, jobject cursor, rekey_args* r) {
    jlong ccap = 0;
    r->s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !r->s) return -1;
    r->d = dstCap ? direct(env, dst, dstCap, NULL, "dst must be a direct ByteBuffer") : NULL;
    if (dstCap && !r->d) return -1;
    r->cur = (tsgpu_rekey_cursor*)direct(env, cursor, 0, &ccap, "rekey cursor must be a direct ByteBuffer of 64 bytes");
    if (!r->cur) return -1;
    if (ccap < (jlong)sizeof(tsgpu_rekey_cursor)) { throw_arg(env, "rekey cursor must be a direct ByteBuffer of 64 bytes"); return -1; }
    if (!transformedSizes) { throw_arg(env, "chunks cannot be null"); return -1; }
    r->n = (uint32_t)(*env)->GetArrayLength(env, transformedSizes);
    if (!nPartsOut || (*env)->GetArrayLength(env, nPartsOut) < 1) { throw_arg(env, "nPartsOut must hold 1 int"); return -1; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return -1; }
    if ((fromKey && (*env)->GetArrayLength(env, fromKey) != 32) || (toKey && (*env)->GetArrayLength(env, toKey) != 32)) {
        throw_arg(env, "data key must be 32 bytes"); return -1;
    }
    if (toIvs && (uint32_t)(*env)->GetArrayLength(env, toIvs) < 12 * r->n) { throw_arg(env, "toIvs must hold 12 bytes per chunk"); return -1; }
    r->fk = fromKey ? (*env)->GetByteArrayElements(env, fromKey, NULL) : NULL;
    r->fa = fromAad ? (*env)->GetByteArrayElements(env, fromAad, NULL) : NULL;
    r->falen = fromAad ? (*env)->GetArrayLength(env, fromAad) : 0;
    r->tk = toKey ? (*env)->GetByteArrayElements(env, toKey, NULL) : NULL;
    r->ta = toAad ? (*env)->GetByteArrayElements(env, toAad, NULL) : NULL;
    r->talen = toAad ? (*env)->GetArrayLength(env, toAad) : 0;
    r->iv = toIvs ? (*env)->GetByteArrayElements(env, toIvs, NULL) : NULL;
    r->ts = (*env)->GetIntArrayElements(env, transformedSizes, NULL);
    return 0;
}
/* Releases what rekey_begin pinned; on success nPartsOut[0] receives the count of completed parts. */
static void rekey_end(JNIEnv* env, jintArray transformedSizes, jbyteArray fromKey, jbyteArray fromAad, jbyteArray toKey,
                      jbyteArray toAad, jbyteArray toIvs, jintArray nPartsOut, rekey_args* r, int rc, uint32_t nParts) {
    (*env)->ReleaseIntArrayElements(env, transformedSizes, r->ts, JNI_ABORT);
    if (r->fk) (*env)->ReleaseByteArrayElements(env, fromKey, r->fk, JNI_ABORT);
    if (r->fa) (*env)->ReleaseByteArrayElements(env, fromAad, r->fa, JNI_ABORT);
    if (r->tk) (*env)->ReleaseByteArrayElements(env, toKey, r->tk, JNI_ABORT);
    if (r->ta) (*env)->ReleaseByteArrayElements(env, toAad, r->ta, JNI_ABORT);
    if (r->iv) (*env)->ReleaseByteArrayElements(env, toIvs, r->iv, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    jint* np = (*env)->GetIntArrayElements(env, nPartsOut, NULL);
    np[0] = (jint)nParts;
    (*env)->ReleaseIntArrayElements(env, nPartsOut, np, 0);
}

/* RekeyCursor.rekeyObject: partCrcs (int[], its length is part_cap) receives the CRC-32C of the upload parts the window completes;
 * crcsOut (int[2]) receives, on the object's last window, the CRC-32C of the old object and of the new object. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_RekeyCursor_rekeyObject(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray transformedSizes, jbyteArray fromKey,
    jbyteArray fromAad, jbyteArray toKey, jbyteArray toAad, jbyteArray toIvs, jobject dst, jlong dstCap, jlong partSize,
    jintArray partCrcs, jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jintArray crcsOut) {
    if (!partCrcs) { throw_arg(env, "partCrcs cannot be null"); return; }
    if (!crcsOut || (*env)->GetArrayLength(env, crcsOut) < 2) { throw_arg(env, "crcsOut must hold 2 ints"); return; }
    rekey_args r;
    if (rekey_begin(env, src, srcLen, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, dst, dstCap, partSize, nPartsOut,
                    cursor, &r)) return;
    const uint32_t cap = (uint32_t)(*env)->GetArrayLength(env, partCrcs);
    jint* pc = (*env)->GetIntArrayElements(env, partCrcs, NULL);
    uint32_t nParts = 0, crcs[2] = {0, 0};
    int rc = tsgpu_rekey_object((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, r.s, (uint64_t)srcLen, (const uint32_t*)r.ts, r.n,
                                (const uint8_t*)r.fk, (const uint8_t*)r.fa, (uint32_t)r.falen, (const uint8_t*)r.tk, (const uint8_t*)r.ta,
                                (uint32_t)r.talen, (const uint8_t*)r.iv, r.d, (uint64_t)dstCap, (uint64_t)partSize, (uint32_t*)pc, cap,
                                &nParts, r.cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1]);
    (*env)->ReleaseIntArrayElements(env, partCrcs, pc, rc ? JNI_ABORT : 0);
    rekey_end(env, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, nPartsOut, &r, rc, nParts);
    if (!rc && objectEndsHere) {
        jint* out = (*env)->GetIntArrayElements(env, crcsOut, NULL);
        out[0] = (jint)crcs[0]; out[1] = (jint)crcs[1];
        (*env)->ReleaseIntArrayElements(env, crcsOut, out, 0);
    }
}

/* RekeyCursor.rekeyObjectCrc64: rekeyObject with CRC-64/NVME.  partCrc64 (direct, 8 bytes per part: its capacity / 8 is
 * part_cap) receives the CRCs of the upload parts the window completes; crcsOut (direct, 16 bytes) receives, on the object's last
 * window, the CRC-64/NVME of the old object and of the new object. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_RekeyCursor_rekeyObjectCrc64(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray transformedSizes, jbyteArray fromKey,
    jbyteArray fromAad, jbyteArray toKey, jbyteArray toAad, jbyteArray toIvs, jobject dst, jlong dstCap, jlong partSize,
    jobject partCrc64, jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jobject crcsOut) {
    jlong pcap = 0, wcap = 0;
    uint64_t* pc = (uint64_t*)direct(env, partCrc64, 0, &pcap, "partCrc64 must be a direct ByteBuffer");
    if (!pc) return;
    uint64_t* out = (uint64_t*)direct(env, crcsOut, 0, &wcap, "crcsOut must be a direct ByteBuffer of 16 bytes");
    if (!out) return;
    if (wcap < 16) { throw_arg(env, "crcsOut must be a direct ByteBuffer of 16 bytes"); return; }
    rekey_args r;
    if (rekey_begin(env, src, srcLen, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, dst, dstCap, partSize, nPartsOut,
                    cursor, &r)) return;
    uint32_t nParts = 0;
    uint64_t crcs[2] = {0, 0};
    int rc = tsgpu_rekey_object_crc64((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, r.s, (uint64_t)srcLen, (const uint32_t*)r.ts, r.n,
                                      (const uint8_t*)r.fk, (const uint8_t*)r.fa, (uint32_t)r.falen, (const uint8_t*)r.tk,
                                      (const uint8_t*)r.ta, (uint32_t)r.talen, (const uint8_t*)r.iv, r.d, (uint64_t)dstCap,
                                      (uint64_t)partSize, pc, (uint32_t)(pcap / 8), &nParts, r.cur, objectEndsHere ? 1 : 0, &crcs[0],
                                      &crcs[1]);
    rekey_end(env, transformedSizes, fromKey, fromAad, toKey, toAad, toIvs, nPartsOut, &r, rc, nParts);
    if (!rc && objectEndsHere) { out[0] = crcs[0]; out[1] = crcs[1]; }
}

/* ---------------------------------------------------------------------------------------------------------------------------
 * Encryption of a stored unencrypted object (EncryptCursor.java): one window of its chunks encrypted with nothing decoded
 * (tsgpu_encrypt_object[_crc64]).  `cursor` a direct ByteBuffer of at least 64 bytes holding the tsgpu_encrypt_cursor (zeros at
 * the start of the object), updated in place; dst a direct ByteBuffer receiving exactly the window's new bytes (every non-empty
 * chunk 28 bytes longer); newSizes (int[], one per chunk) the new chunk sizes; ivs 12 bytes per chunk of the window (an empty
 * chunk takes none, its 12 bytes are not read). */

/* The arguments both widths check the same way; the chunk sizes, key, AAD and IV arrays pinned.  Returns -1 with an exception
 * pending. */
typedef struct {
    uint8_t* s; uint8_t* d; tsgpu_encrypt_cursor* cur; uint32_t n;
    jint* cs; jint* ns; jbyte* k; jbyte* a; jint alen; jbyte* iv;
} encrypt_args;
static int encrypt_begin(JNIEnv* env, jobject src, jlong srcLen, jintArray chunkSizes, jbyteArray key, jbyteArray aad, jbyteArray ivs,
                         jobject dst, jlong dstCap, jintArray newSizes, jlong partSize, jintArray nPartsOut, jobject cursor,
                         encrypt_args* r) {
    jlong ccap = 0;
    r->s = srcLen ? direct(env, src, srcLen, NULL, "src must be a direct ByteBuffer") : NULL;
    if (srcLen && !r->s) return -1;
    r->d = dstCap ? direct(env, dst, dstCap, NULL, "dst must be a direct ByteBuffer") : NULL;
    if (dstCap && !r->d) return -1;
    r->cur = (tsgpu_encrypt_cursor*)direct(env, cursor, 0, &ccap, "encrypt cursor must be a direct ByteBuffer of 64 bytes");
    if (!r->cur) return -1;
    if (ccap < (jlong)sizeof(tsgpu_encrypt_cursor)) { throw_arg(env, "encrypt cursor must be a direct ByteBuffer of 64 bytes"); return -1; }
    if (!chunkSizes) { throw_arg(env, "chunks cannot be null"); return -1; }
    r->n = (uint32_t)(*env)->GetArrayLength(env, chunkSizes);
    if (!newSizes || (uint32_t)(*env)->GetArrayLength(env, newSizes) < r->n) { throw_arg(env, "newSizes must hold 1 int per chunk"); return -1; }
    if (!nPartsOut || (*env)->GetArrayLength(env, nPartsOut) < 1) { throw_arg(env, "nPartsOut must hold 1 int"); return -1; }
    if (partSize < 1) { throw_arg(env, "partSize must be positive"); return -1; }
    if (key && (*env)->GetArrayLength(env, key) != 32) { throw_arg(env, "data key must be 32 bytes"); return -1; }
    if (ivs && (uint32_t)(*env)->GetArrayLength(env, ivs) < 12 * r->n) { throw_arg(env, "ivs must hold 12 bytes per chunk"); return -1; }
    r->k = key ? (*env)->GetByteArrayElements(env, key, NULL) : NULL;
    r->a = aad ? (*env)->GetByteArrayElements(env, aad, NULL) : NULL;
    r->alen = aad ? (*env)->GetArrayLength(env, aad) : 0;
    r->iv = ivs ? (*env)->GetByteArrayElements(env, ivs, NULL) : NULL;
    r->cs = (*env)->GetIntArrayElements(env, chunkSizes, NULL);
    r->ns = (*env)->GetIntArrayElements(env, newSizes, NULL);
    return 0;
}
/* Releases what encrypt_begin pinned; on success newSizes keeps the new sizes and nPartsOut[0] receives the count of completed
 * parts. */
static void encrypt_end(JNIEnv* env, jintArray chunkSizes, jbyteArray key, jbyteArray aad, jbyteArray ivs, jintArray newSizes,
                        jintArray nPartsOut, encrypt_args* r, int rc, uint32_t nParts) {
    (*env)->ReleaseIntArrayElements(env, chunkSizes, r->cs, JNI_ABORT);
    (*env)->ReleaseIntArrayElements(env, newSizes, r->ns, rc ? JNI_ABORT : 0);
    if (r->k) (*env)->ReleaseByteArrayElements(env, key, r->k, JNI_ABORT);
    if (r->a) (*env)->ReleaseByteArrayElements(env, aad, r->a, JNI_ABORT);
    if (r->iv) (*env)->ReleaseByteArrayElements(env, ivs, r->iv, JNI_ABORT);
    if (rc) { throw_rt(env, rc); return; }
    jint* np = (*env)->GetIntArrayElements(env, nPartsOut, NULL);
    np[0] = (jint)nParts;
    (*env)->ReleaseIntArrayElements(env, nPartsOut, np, 0);
}

/* EncryptCursor.encryptObject: partCrcs (int[], its length is part_cap) receives the CRC-32C of the upload parts the window
 * completes; crcsOut (int[2]) receives, on the object's last window, the CRC-32C of the old object and of the new object. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_EncryptCursor_encryptObject(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray chunkSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray key, jbyteArray aad, jbyteArray ivs, jobject dst, jlong dstCap, jintArray newSizes,
    jlong partSize, jintArray partCrcs, jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jintArray crcsOut) {
    if (!partCrcs) { throw_arg(env, "partCrcs cannot be null"); return; }
    if (!crcsOut || (*env)->GetArrayLength(env, crcsOut) < 2) { throw_arg(env, "crcsOut must hold 2 ints"); return; }
    encrypt_args r;
    if (encrypt_begin(env, src, srcLen, chunkSizes, key, aad, ivs, dst, dstCap, newSizes, partSize, nPartsOut, cursor, &r)) return;
    const uint32_t cap = (uint32_t)(*env)->GetArrayLength(env, partCrcs);
    jint* pc = (*env)->GetIntArrayElements(env, partCrcs, NULL);
    uint32_t nParts = 0, crcs[2] = {0, 0};
    int rc = tsgpu_encrypt_object((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, r.s, (uint64_t)srcLen, (const uint32_t*)r.cs, r.n,
                                  (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)r.k, (const uint8_t*)r.a,
                                  (uint32_t)r.alen, (const uint8_t*)r.iv, r.d, (uint64_t)dstCap, (uint32_t*)r.ns, (uint64_t)partSize,
                                  (uint32_t*)pc, cap, &nParts, r.cur, objectEndsHere ? 1 : 0, &crcs[0], &crcs[1]);
    (*env)->ReleaseIntArrayElements(env, partCrcs, pc, rc ? JNI_ABORT : 0);
    encrypt_end(env, chunkSizes, key, aad, ivs, newSizes, nPartsOut, &r, rc, nParts);
    if (!rc && objectEndsHere) {
        jint* out = (*env)->GetIntArrayElements(env, crcsOut, NULL);
        out[0] = (jint)crcs[0]; out[1] = (jint)crcs[1];
        (*env)->ReleaseIntArrayElements(env, crcsOut, out, 0);
    }
}

/* EncryptCursor.encryptObjectCrc64: encryptObject with CRC-64/NVME.  partCrc64 (direct, 8 bytes per part: its capacity / 8 is
 * part_cap) receives the CRCs of the upload parts the window completes; crcsOut (direct, 16 bytes) receives, on the object's last
 * window, the CRC-64/NVME of the old object and of the new object. */
JNIEXPORT void JNICALL Java_io_aiven_kafka_tieredstorage_transform_gpu_EncryptCursor_encryptObjectCrc64(
    JNIEnv* env, jclass c, jlong h, jint flags, jobject src, jlong srcLen, jintArray chunkSizes, jint originalChunkSize,
    jlong originalFileSize, jbyteArray key, jbyteArray aad, jbyteArray ivs, jobject dst, jlong dstCap, jintArray newSizes,
    jlong partSize, jobject partCrc64, jintArray nPartsOut, jobject cursor, jboolean objectEndsHere, jobject crcsOut) {
    jlong pcap = 0, wcap = 0;
    uint64_t* pc = (uint64_t*)direct(env, partCrc64, 0, &pcap, "partCrc64 must be a direct ByteBuffer");
    if (!pc) return;
    uint64_t* out = (uint64_t*)direct(env, crcsOut, 0, &wcap, "crcsOut must be a direct ByteBuffer of 16 bytes");
    if (!out) return;
    if (wcap < 16) { throw_arg(env, "crcsOut must be a direct ByteBuffer of 16 bytes"); return; }
    encrypt_args r;
    if (encrypt_begin(env, src, srcLen, chunkSizes, key, aad, ivs, dst, dstCap, newSizes, partSize, nPartsOut, cursor, &r)) return;
    uint32_t nParts = 0;
    uint64_t crcs[2] = {0, 0};
    int rc = tsgpu_encrypt_object_crc64((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, r.s, (uint64_t)srcLen, (const uint32_t*)r.cs, r.n,
                                        (uint32_t)originalChunkSize, (uint64_t)originalFileSize, (const uint8_t*)r.k,
                                        (const uint8_t*)r.a, (uint32_t)r.alen, (const uint8_t*)r.iv, r.d, (uint64_t)dstCap,
                                        (uint32_t*)r.ns, (uint64_t)partSize, pc, (uint32_t)(pcap / 8), &nParts, r.cur,
                                        objectEndsHere ? 1 : 0, &crcs[0], &crcs[1]);
    encrypt_end(env, chunkSizes, key, aad, ivs, newSizes, nPartsOut, &r, rc, nParts);
    if (!rc && objectEndsHere) { out[0] = crcs[0]; out[1] = crcs[1]; }
}
