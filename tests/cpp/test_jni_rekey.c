/*
 * Drives the key-rotation path of jni/tsgpu_jni.c (RekeyCursor.rekeyObject and RekeyCursor.rekeyObjectCrc64) through a fake JNIEnv,
 * in the window flow of an operator tool: a Zstd+AES object the oracle wrote (libzstd level 3 + OpenSSL: what the Java plugin wrote)
 * is re-encrypted under a new key in windows of 1, 4 and 11 chunks.  Every new chunk is the oracle's encryption under the new key
 * and IV of the old chunk's frame, each keeps its size, and the part CRCs and the two object CRCs agree with a host CRC-32C and
 * CRC-64/NVME.  A flipped ciphertext byte throws RuntimeException naming the chunk; a flag other than FLAG_VERIFY throws
 * IllegalArgumentException.  Links the test-only SIMT build and the oracle.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jni.h>
#include "../../jni/tsgpu_jni.c"
#include "../../oracle/tsoracle.h"

struct _jobject { int kind; void* data; jlong len; };      /* kind: 1 int[], 2 byte[], 3 direct buffer, 4 class */
static int checks = 0, failures = 0;
#define CHECK(c) do { checks++; if (!(c)) { failures++; printf("FAIL %s:%d %s\n", __FILE__, __LINE__, #c); } } while (0)
static char thrown_class[128], thrown_msg[512];

static jclass f_FindClass(JNIEnv* e, const char* name) { struct _jobject* o = calloc(1, sizeof *o); o->kind = 4; o->data = strdup(name); return o; }
static jint f_ThrowNew(JNIEnv* e, jclass c, const char* msg) { snprintf(thrown_class, sizeof thrown_class, "%s", (char*)c->data); snprintf(thrown_msg, sizeof thrown_msg, "%s", msg); return 0; }
static jsize f_GetArrayLength(JNIEnv* e, jarray a) { return (jsize)a->len; }
static void* copy_out(jarray a, size_t elem) { void* p = malloc(a->len * elem + 1); memcpy(p, a->data, a->len * elem); return p; }
static void copy_back(jarray a, void* p, size_t elem, jint mode) { if (mode != JNI_ABORT) memcpy(a->data, p, a->len * elem); if (mode != JNI_COMMIT) free(p); }
static jbyte* f_GetByteArrayElements(JNIEnv* e, jbyteArray a, jboolean* c) { if (c) *c = 1; return copy_out(a, 1); }
static void f_ReleaseByteArrayElements(JNIEnv* e, jbyteArray a, jbyte* p, jint m) { copy_back(a, p, 1, m); }
static jint* f_GetIntArrayElements(JNIEnv* e, jintArray a, jboolean* c) { if (c) *c = 1; return copy_out(a, 4); }
static void f_ReleaseIntArrayElements(JNIEnv* e, jintArray a, jint* p, jint m) { copy_back(a, p, 4, m); }
static jobject f_NewDirectByteBuffer(JNIEnv* e, void* p, jlong cap) { struct _jobject* o = calloc(1, sizeof *o); o->kind = 3; o->data = p; o->len = cap; return o; }
static void* f_GetDirectBufferAddress(JNIEnv* e, jobject b) { return b->data; }
static jlong f_GetDirectBufferCapacity(JNIEnv* e, jobject b) { return b->len; }
static const struct JNINativeInterface_ table = { f_FindClass, f_ThrowNew, f_GetArrayLength, f_GetByteArrayElements, f_ReleaseByteArrayElements,
    f_GetIntArrayElements, f_ReleaseIntArrayElements, f_NewDirectByteBuffer, f_GetDirectBufferAddress, f_GetDirectBufferCapacity };

static jarray mk_array(int kind, const void* src, jlong n, size_t elem) {
    struct _jobject* o = calloc(1, sizeof *o); o->kind = kind; o->len = n; o->data = calloc((size_t)n + 1, elem);
    if (src) memcpy(o->data, src, (size_t)n * elem);
    return o;
}
static jobject mk_direct(void* p, jlong n) { struct _jobject* o = calloc(1, sizeof *o); o->kind = 3; o->data = p; o->len = n; return o; }
#define NS(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_TsGpu_##f

static uint32_t crc32c(const uint8_t* p, size_t n) {
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x82F63B78u & (0u - (c & 1u))); }
    return ~c;
}
static uint64_t crc64nvme(const uint8_t* p, size_t n) {
    uint64_t c = ~0ull;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x9A6C9329AC4BC9B5ull & (0ull - (c & 1ull))); }
    return ~c;
}
#define KC(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_RekeyCursor_##f

/* The object's windows of `win` chunks through RekeyCursor.rekeyObject (crc64: rekeyObjectCrc64) into neo; returns 0 with the
 * source and object CRCs in crcs (64-bit words either way) and the part CRCs in parts, or -1 with the exception pending. */
static int rekey_windows(JNIEnv* env, jlong h, jint flags, uint8_t* obj, const uint32_t* sizes, uint32_t n, uint32_t win, int crc64,
                         jarray fkey, jarray faad, jarray tkey, jarray taad, const uint8_t* ivs, uint8_t* neo, jlong part,
                         uint64_t* parts, uint32_t* nparts, uint64_t crcs[2]) {
    uint8_t cursor[64] = {0};
    uint64_t pc64[64], out64[2] = {0, 0};
    jobject cur = mk_direct(cursor, 64);
    jarray out = mk_array(1, NULL, 2, 4), np = mk_array(1, NULL, 1, 4), pc = mk_array(1, NULL, 64, 4);
    size_t pos = 0;
    *nparts = 0;
    for (uint32_t k = 0;; k += win) {
        const uint32_t m = k < n ? (n - k < win ? n - k : win) : 0;
        const int end = k + win > n;
        size_t bytes = 0;
        for (uint32_t i = 0; i < m; i++) bytes += sizes[k + i];
        jarray ts = mk_array(1, sizes + k, m, 4);
        jarray iv = mk_array(2, ivs + 12 * k, 12 * (jlong)m, 1);
        thrown_class[0] = 0;
        if (crc64)
            KC(rekeyObjectCrc64)(env, NULL, h, flags, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, ts, fkey, faad, tkey, taad, iv,
                                 mk_direct(neo + pos, (jlong)bytes), (jlong)bytes, part, mk_direct(pc64, sizeof pc64), np, cur, end ? 1 : 0,
                                 mk_direct(out64, sizeof out64));
        else
            KC(rekeyObject)(env, NULL, h, flags, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, ts, fkey, faad, tkey, taad, iv,
                            mk_direct(neo + pos, (jlong)bytes), (jlong)bytes, part, pc, np, cur, end ? 1 : 0, out);
        if (thrown_class[0]) return -1;
        const uint32_t got = ((uint32_t*)np->data)[0];
        for (uint32_t i = 0; i < got; i++) parts[*nparts + i] = crc64 ? pc64[i] : ((uint32_t*)pc->data)[i];
        *nparts += got;
        pos += bytes;
        if (end) {
            crcs[0] = crc64 ? out64[0] : ((uint32_t*)out->data)[0];
            crcs[1] = crc64 ? out64[1] : ((uint32_t*)out->data)[1];
            return 0;
        }
    }
}

int main(void) {
    JNIEnv env_ = &table, *env = &env_;
    const jint cs = 4096;
    jlong h = NS(create)(env, NULL, NULL, cs, 2);
    CHECK(h != 0);
    const size_t n = 9 * 4096 + 1234;
    uint8_t* seg = malloc(n);
    for (size_t i = 0; i < n; i++) seg[i] = (uint8_t)("kafka-record-batch "[i % 19] + (i / 977) % 3);
    uint8_t key[32], aad[32], key2[32], aad2[16];
    for (int i = 0; i < 32; i++) { key[i] = (uint8_t)i; aad[i] = 0xA5; key2[i] = (uint8_t)(200 - i); }
    for (int i = 0; i < 16; i++) aad2[i] = (uint8_t)(0x30 + i);
    uint8_t ivs[12 * 16] = {0}, ivs2[12 * 16];
    for (int i = 0; i < 16; i++) ivs[12 * i + 11] = (uint8_t)i;
    for (int i = 0; i < 12 * 16; i++) ivs2[i] = (uint8_t)(i * 37 + 5);
    jarray jkey = mk_array(2, key, 32, 1), jaad = mk_array(2, aad, 32, 1), jkey2 = mk_array(2, key2, 32, 1), jaad2 = mk_array(2, aad2, 16, 1);
    const jint ZA = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES;
    const uint64_t cap = ora_transform_bound((uint32_t)ZA, n, (uint32_t)cs) + 64;
    uint8_t* obj = malloc(cap);
    uint32_t sizes[16], got = 16;
    CHECK(ora_transform_segment((uint32_t)ZA, seg, n, (uint32_t)cs, key, aad, 32, ivs, obj, cap, sizes, &got) == 0);
    size_t total = 0;
    for (uint32_t i = 0; i < got; i++) total += sizes[i];
    /* what the new object must be: each old chunk decrypted under the old key and encrypted under the new key and IV */
    uint8_t* want = malloc(total), *neo = malloc(total), frame[8192];
    for (size_t i = 0, at = 0; i < got; at += sizes[i++]) {
        CHECK(ora_aesgcm_decrypt_chunk(key, aad, 32, obj + at, sizes[i], frame) == 0);
        CHECK(ora_aesgcm_encrypt_chunk(key2, ivs2 + 12 * i, aad2, 16, frame, sizes[i] - 28, want + at) == 0);
    }
    for (int crc64 = 0; crc64 < 2; crc64++) for (uint32_t win = 1; win <= 11; win += win == 1 ? 3 : 7) {
        const jint flags = win == 4 ? TSGPU_FLAG_VERIFY : 0;
        uint64_t crcs[2] = {0, 0}, parts[64];
        uint32_t np = 0;
        const jlong part = 3000;
        memset(neo, 0, total);
        CHECK(rekey_windows(env, h, flags, obj, sizes, got, win, crc64, jkey, jaad, jkey2, jaad2, ivs2, neo, part, parts, &np, crcs) == 0);
        CHECK(memcmp(neo, want, total) == 0);
        CHECK(crcs[0] == (crc64 ? crc64nvme(obj, total) : crc32c(obj, total)));
        CHECK(crcs[1] == (crc64 ? crc64nvme(want, total) : crc32c(want, total)));
        CHECK(np == (total + part - 1) / part);
        for (uint32_t p = 0; p < np; p++) {
            const size_t off = (size_t)p * part, len = total - off < (size_t)part ? total - off : (size_t)part;
            CHECK(parts[p] == (crc64 ? crc64nvme(neo + off, len) : crc32c(neo + off, len)));
        }
    }
    /* a flipped ciphertext byte in chunk 5: RuntimeException naming it, in the second window of 4 */
    {
        uint64_t crcs[2] = {7, 7}, parts[64];
        uint32_t np = 0;
        size_t at = 0;
        for (int i = 0; i < 5; i++) at += sizes[i];
        obj[at + 40] ^= 1;
        CHECK(rekey_windows(env, h, 0, obj, sizes, got, 4, 0, jkey, jaad, jkey2, jaad2, ivs2, neo, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strcmp(thrown_msg, "Tag mismatch in chunk 5") == 0);
        CHECK(crcs[0] == 7);
        obj[at + 40] ^= 1;
    }
    /* only FLAG_VERIFY applies */
    {
        uint64_t crcs[2], parts[64];
        uint32_t np = 0;
        CHECK(rekey_windows(env, h, TSGPU_FLAG_AES, obj, sizes, got, 4, 0, jkey, jaad, jkey2, jaad2, ivs2, neo, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "unknown flags") != NULL);
    }
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
