/*
 * Drives the object-check path of jni/tsgpu_jni.c (CheckCursor.checkObject) through a fake JNIEnv, in the window flow of an
 * operator tool: windows of `win` chunks of a stored object with one cursor, objectEndsHere on the last (possibly empty) window.
 * Checks that crcsOut receives the CRC-32C of the object and of the segment only at the end, for plain, compressed, encrypted and
 * compressed+encrypted objects; that a flipped byte of an encrypted object throws RuntimeException naming its chunk; and that the
 * export refuses a short cursor, a crcsOut of fewer than 2 ints and a zero chunk size (IllegalArgumentException).  Links the
 * test-only SIMT build.
 */
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <jni.h>
#include "../../jni/tsgpu_jni.c"

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
#define CC(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_CheckCursor_##f

/* The object's windows of `win` chunks through CheckCursor.checkObject; returns 0 with crcs[0..1] set, or -1 with the exception. */
static int check_windows(JNIEnv* env, jlong h, jint flags, uint8_t* obj, const uint32_t* sizes, uint32_t n, jint cs, jlong ofs,
                         uint32_t win, jarray jkey, jarray jaad, uint32_t crcs[2]) {
    uint8_t cursor[128] = {0};
    jobject cur = mk_direct(cursor, 128);
    jarray out = mk_array(1, NULL, 2, 4);
    size_t pos = 0;
    for (uint32_t k = 0;; k += win) {
        const uint32_t m = k < n ? (n - k < win ? n - k : win) : 0;
        const int end = k + win > n;
        size_t bytes = 0;
        for (uint32_t i = 0; i < m; i++) bytes += sizes[k + i];
        jarray ts = mk_array(1, sizes + k, m, 4);
        thrown_class[0] = 0;
        CC(checkObject)(env, NULL, h, flags, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, ts, cs, ofs, jkey, jaad, cur, end ? 1 : 0, out);
        if (thrown_class[0]) return -1;
        CHECK(end || ((uint32_t*)out->data)[0] == 0);                  /* nothing before the end */
        pos += bytes;
        if (end) { memcpy(crcs, out->data, 8); return 0; }
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
    uint8_t key[32], aad[32];
    for (int i = 0; i < 32; i++) { key[i] = (uint8_t)i; aad[i] = 0xA5; }
    uint8_t ivs[12 * 16] = {0};
    for (int i = 0; i < 16; i++) ivs[12 * i + 11] = (uint8_t)i;
    jarray jkey = mk_array(2, key, 32, 1), jaad = mk_array(2, aad, 32, 1);
    const uint32_t nch = (uint32_t)((n + cs - 1) / cs);
    for (jint flags = 0; flags <= 3; flags++) {
        uint64_t cap = tsgpu_transform_bound((uint32_t)flags, n, (uint32_t)cs) + 64;
        uint8_t* obj = malloc(cap);
        uint32_t sizes[16], got = 16;
        CHECK(tsgpu_transform((tsgpu_ctx*)(intptr_t)h, (uint32_t)flags, seg, n, (uint32_t)cs, key, aad, 32, ivs, obj, cap, sizes, &got) == 0);
        CHECK(got == nch);
        size_t total = 0;
        for (uint32_t i = 0; i < got; i++) total += sizes[i];
        for (uint32_t win = 1; win <= 11; win += 2) {
            uint32_t crcs[2] = {0, 0};
            CHECK(check_windows(env, h, flags, obj, sizes, got, cs, (jlong)n, win, jkey, jaad, crcs) == 0);
            CHECK(crcs[0] == crc32c(obj, total) && crcs[1] == crc32c(seg, n));
        }
        if (flags & TSGPU_FLAG_AES) {
            obj[sizes[0] + sizes[1] + 50] ^= 1;                       /* chunk 2's ciphertext */
            uint32_t crcs[2] = {7, 7};
            CHECK(check_windows(env, h, flags, obj, sizes, got, cs, (jlong)n, 3, jkey, jaad, crcs) == -1);
            CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strstr(thrown_msg, "chunk 2") != NULL);
            CHECK(crcs[0] == 7);
        }
        free(obj);
    }
    /* argument refusals */
    uint8_t small[64] = {0}, cursor[128] = {0};
    jarray ts0 = mk_array(1, NULL, 0, 4), out1 = mk_array(1, NULL, 1, 4), out2 = mk_array(1, NULL, 2, 4);
    thrown_class[0] = 0;
    CC(checkObject)(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, mk_direct(small, 64), 1, out2);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    thrown_class[0] = 0;
    CC(checkObject)(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, mk_direct(cursor, 128), 1, out1);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    thrown_class[0] = 0;
    CC(checkObject)(env, NULL, h, 0, NULL, 0, ts0, 0, 0, NULL, NULL, mk_direct(cursor, 128), 1, out2);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    thrown_class[0] = 0;
    CC(checkObject)(env, NULL, h, TSGPU_FLAG_ZSTD, NULL, 0, ts0, cs, 0, NULL, NULL, mk_direct(cursor, 128), 1, out2);   /* empty segment */
    CHECK(thrown_class[0] == 0);
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
