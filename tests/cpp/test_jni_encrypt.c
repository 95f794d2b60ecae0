/*
 * Drives the encryption path of jni/tsgpu_jni.c (EncryptCursor.encryptObject and EncryptCursor.encryptObjectCrc64) through a fake
 * JNIEnv, in the window flow of an operator tool: a Zstd-only object the oracle wrote (libzstd level 3: what the Java plugin wrote)
 * is encrypted in windows of 1, 4 and 11 chunks.  Every new chunk is the oracle's encryption of the old chunk under the key and its
 * IV, the new sizes are 28 bytes more, and the part CRCs and the two object CRCs agree with a host CRC-32C and CRC-64/NVME.  A
 * damaged frame throws RuntimeException naming the chunk; FLAG_AES and a reused IV throw IllegalArgumentException.  Links the
 * test-only SIMT build and the oracle.
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
#define EC(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_EncryptCursor_##f

/* The object's windows of `win` chunks through EncryptCursor.encryptObject (crc64: encryptObjectCrc64) into neo (new sizes in
 * nsz); returns 0 with the source and object CRCs in crcs (64-bit words either way) and the part CRCs in parts, or -1 with the
 * exception pending. */
static int encrypt_windows(JNIEnv* env, jlong h, jint flags, uint8_t* obj, const uint32_t* sizes, uint32_t n, uint32_t win, int crc64,
                           jint ocs, jlong ofs, jarray key, jarray aad, const uint8_t* ivs, uint8_t* neo, uint32_t* nsz, jlong part,
                           uint64_t* parts, uint32_t* nparts, uint64_t crcs[2]) {
    uint8_t cursor[64] = {0};
    uint64_t pc64[64], out64[2] = {0, 0};
    jobject cur = mk_direct(cursor, 64);
    jarray out = mk_array(1, NULL, 2, 4), np = mk_array(1, NULL, 1, 4), pc = mk_array(1, NULL, 64, 4);
    size_t pos = 0, npos = 0;
    *nparts = 0;
    for (uint32_t k = 0;; k += win) {
        const uint32_t m = k < n ? (n - k < win ? n - k : win) : 0;
        const int end = k + win > n;
        size_t bytes = 0, nbytes = 0;
        for (uint32_t i = 0; i < m; i++) { bytes += sizes[k + i]; nbytes += sizes[k + i] ? sizes[k + i] + 28 : 0; }
        jarray cs = mk_array(1, sizes + k, m, 4), ns = mk_array(1, NULL, m, 4);
        jarray iv = mk_array(2, ivs + 12 * k, 12 * (jlong)m, 1);
        thrown_class[0] = 0;
        if (crc64)
            EC(encryptObjectCrc64)(env, NULL, h, flags, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, cs, ocs, ofs, key, aad, iv,
                                   mk_direct(neo + npos, (jlong)nbytes), (jlong)nbytes, ns, part, mk_direct(pc64, sizeof pc64), np, cur,
                                   end ? 1 : 0, mk_direct(out64, sizeof out64));
        else
            EC(encryptObject)(env, NULL, h, flags, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, cs, ocs, ofs, key, aad, iv,
                              mk_direct(neo + npos, (jlong)nbytes), (jlong)nbytes, ns, part, pc, np, cur, end ? 1 : 0, out);
        if (thrown_class[0]) return -1;
        memcpy(nsz + k, ns->data, 4ull * m);
        const uint32_t got = ((uint32_t*)np->data)[0];
        for (uint32_t i = 0; i < got; i++) parts[*nparts + i] = crc64 ? pc64[i] : ((uint32_t*)pc->data)[i];
        *nparts += got;
        pos += bytes; npos += nbytes;
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
    uint8_t key[32], aad[16];
    for (int i = 0; i < 32; i++) key[i] = (uint8_t)(200 - i);
    for (int i = 0; i < 16; i++) aad[i] = (uint8_t)(0x30 + i);
    uint8_t ivs0[12 * 16] = {0}, ivs[12 * 16];
    for (int i = 0; i < 12 * 16; i++) ivs[i] = (uint8_t)(i * 37 + 5);
    jarray jkey = mk_array(2, key, 32, 1), jaad = mk_array(2, aad, 16, 1);
    const jint Z = TSGPU_FLAG_ZSTD;
    const uint64_t cap = ora_transform_bound((uint32_t)Z, n, (uint32_t)cs) + 64;
    uint8_t* obj = malloc(cap);
    uint32_t sizes[16], got = 16;
    CHECK(ora_transform_segment((uint32_t)Z, seg, n, (uint32_t)cs, key, aad, 16, ivs0, obj, cap, sizes, &got) == 0);
    size_t total = 0, ntotal = 0;
    for (uint32_t i = 0; i < got; i++) { total += sizes[i]; ntotal += sizes[i] + 28; }
    /* what the new object must be: each old chunk encrypted as it is under the key and its IV */
    uint8_t* want = malloc(ntotal), *neo = malloc(ntotal);
    for (size_t i = 0, at = 0, nat = 0; i < got; at += sizes[i], nat += sizes[i] + 28, i++)
        CHECK(ora_aesgcm_encrypt_chunk(key, ivs + 12 * i, aad, 16, obj + at, sizes[i], want + nat) == 0);
    for (int crc64 = 0; crc64 < 2; crc64++) for (uint32_t win = 1; win <= 11; win += win == 1 ? 3 : 7) {
        const jint flags = win == 4 ? (Z | TSGPU_FLAG_VERIFY) : Z;
        uint64_t crcs[2] = {0, 0}, parts[64];
        uint32_t np = 0, nsz[16];
        const jlong part = 3000;
        memset(neo, 0, ntotal);
        CHECK(encrypt_windows(env, h, flags, obj, sizes, got, win, crc64, cs, (jlong)n, jkey, jaad, ivs, neo, nsz, part, parts, &np, crcs) == 0);
        CHECK(memcmp(neo, want, ntotal) == 0);
        for (uint32_t i = 0; i < got; i++) CHECK(nsz[i] == sizes[i] + 28);
        CHECK(crcs[0] == (crc64 ? crc64nvme(obj, total) : crc32c(obj, total)));
        CHECK(crcs[1] == (crc64 ? crc64nvme(want, ntotal) : crc32c(want, ntotal)));
        CHECK(np == (ntotal + part - 1) / part);
        for (uint32_t p = 0; p < np; p++) {
            const size_t off = (size_t)p * part, len = ntotal - off < (size_t)part ? ntotal - off : (size_t)part;
            CHECK(parts[p] == (crc64 ? crc64nvme(neo + off, len) : crc32c(neo + off, len)));
        }
    }
    /* a damaged frame magic in chunk 5: RuntimeException naming it, in the second window of 4 */
    {
        uint64_t crcs[2] = {7, 7}, parts[64];
        uint32_t np = 0, nsz[16];
        size_t at = 0;
        for (int i = 0; i < 5; i++) at += sizes[i];
        obj[at] ^= 1;
        CHECK(encrypt_windows(env, h, Z, obj, sizes, got, 4, 0, cs, (jlong)n, jkey, jaad, ivs, neo, nsz, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strcmp(thrown_msg, "Invalid zstd frame in chunk 5 (code 2)") == 0);
        CHECK(crcs[0] == 7);
        obj[at] ^= 1;
    }
    /* the object is already encrypted: FLAG_AES is refused; a reused IV too */
    {
        uint64_t crcs[2], parts[64];
        uint32_t np = 0, nsz[16];
        CHECK(encrypt_windows(env, h, Z | TSGPU_FLAG_AES, obj, sizes, got, 4, 0, cs, (jlong)n, jkey, jaad, ivs, neo, nsz, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "tsgpu_rekey_object") != NULL);
        uint8_t dup[12 * 16];
        memcpy(dup, ivs, sizeof dup);
        memcpy(dup + 12, dup, 12);
        CHECK(encrypt_windows(env, h, Z, obj, sizes, got, 4, 0, cs, (jlong)n, jkey, jaad, dup, neo, nsz, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strcmp(thrown_msg, "to_ivs[0] repeats to_ivs[1]") == 0);
    }
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
