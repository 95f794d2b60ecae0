/*
 * Drives the object-rewrite path of jni/tsgpu_jni.c (RewriteCursor.rewriteObject) through a fake JNIEnv, in the window flow of an
 * operator tool: windows of `win` chunks of a stored object with one cursor, objectEndsHere on the last (possibly empty) window,
 * new IVs per window.  Checks that plain, compressed, encrypted and compressed+encrypted objects rewritten to Zstd+AES under a
 * new key decode back to the segment, that the part CRCs and, only at the end, crcsOut hold the CRC-32C of the old object, the
 * new object and the segment; that a flipped byte of an encrypted object and an old IV reused under the same key throw
 * (RuntimeException naming the chunk, IllegalArgumentException); and that the export refuses a short cursor, short output
 * arrays, missing IVs and a zero part size (IllegalArgumentException).  Links the test-only SIMT build.
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
#define RC(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_RewriteCursor_##f

/* The object's windows of `win` chunks through RewriteCursor.rewriteObject into neo (its new sizes in nsz); returns 0 with
 * crcs[0..2] set and the part CRCs in parts, or -1 with the exception pending. */
static int rewrite_windows(JNIEnv* env, jlong h, jint from, uint8_t* obj, const uint32_t* sizes, uint32_t n, jint cs, jlong ofs,
                           uint32_t win, jarray fkey, jarray faad, jint to, jarray tkey, jarray taad, const uint8_t* ivs,
                           uint8_t* neo, uint64_t neo_cap, uint32_t* nsz, jlong part, uint32_t* parts, uint32_t* nparts, uint32_t crcs[3]) {
    uint8_t cursor[192] = {0};
    jobject cur = mk_direct(cursor, 192);
    jarray out = mk_array(1, NULL, 3, 4), np = mk_array(1, NULL, 1, 4), pc = mk_array(1, NULL, 64, 4);
    size_t pos = 0, at = 0;
    *nparts = 0;
    for (uint32_t k = 0;; k += win) {
        const uint32_t m = k < n ? (n - k < win ? n - k : win) : 0;
        const int end = k + win > n;
        size_t bytes = 0;
        for (uint32_t i = 0; i < m; i++) bytes += sizes[k + i];
        jarray ts = mk_array(1, sizes + k, m, 4), nts = mk_array(1, NULL, m, 4);
        jarray iv = mk_array(2, ivs + 12 * k, 12 * (jlong)m, 1);
        thrown_class[0] = 0;
        RC(rewriteObject)(env, NULL, h, from, mk_direct(obj + pos, (jlong)bytes), (jlong)bytes, ts, cs, ofs, fkey, faad, to, tkey, taad, iv,
                          mk_direct(neo + at, (jlong)(neo_cap - at)), (jlong)(neo_cap - at), nts, part, pc, np, cur, end ? 1 : 0, out);
        if (thrown_class[0]) return -1;
        CHECK(end || ((uint32_t*)out->data)[0] == 0);                  /* nothing before the end */
        for (uint32_t i = 0; i < m; i++) { nsz[k + i] = ((uint32_t*)nts->data)[i]; at += nsz[k + i]; }
        const uint32_t got = ((uint32_t*)np->data)[0];
        memcpy(parts + *nparts, pc->data, 4 * got); *nparts += got;
        pos += bytes;
        if (end) { memcpy(crcs, out->data, 12); return 0; }
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
    const uint32_t nch = (uint32_t)((n + cs - 1) / cs);
    const jint ZA = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES;
    const uint64_t neo_cap = tsgpu_transform_bound((uint32_t)ZA, n, (uint32_t)cs) + 64;
    uint8_t* neo = malloc(neo_cap);
    uint8_t* back = malloc(n + 64);
    for (jint from = 0; from <= 3; from++) {
        uint64_t cap = tsgpu_transform_bound((uint32_t)from, n, (uint32_t)cs) + 64;
        uint8_t* obj = malloc(cap);
        uint32_t sizes[16], got = 16;
        CHECK(tsgpu_transform((tsgpu_ctx*)(intptr_t)h, (uint32_t)from, seg, n, (uint32_t)cs, key, aad, 32, ivs, obj, cap, sizes, &got) == 0);
        CHECK(got == nch);
        size_t total = 0;
        for (uint32_t i = 0; i < got; i++) total += sizes[i];
        for (uint32_t win = 1; win <= 11; win += 5) {
            uint32_t crcs[3] = {0, 0, 0}, nsz[16], parts[64], np = 0;
            const jlong part = 3000;
            CHECK(rewrite_windows(env, h, from, obj, sizes, got, cs, (jlong)n, win, jkey, jaad, ZA, jkey2, jaad2, ivs2, neo, neo_cap,
                                  nsz, part, parts, &np, crcs) == 0);
            size_t nt = 0;
            for (uint32_t i = 0; i < got; i++) nt += nsz[i];
            CHECK(crcs[0] == crc32c(obj, total) && crcs[1] == crc32c(neo, nt) && crcs[2] == crc32c(seg, n));
            CHECK(np == (nt + part - 1) / part);
            for (uint32_t p = 0; p < np; p++) {
                const size_t off = (size_t)p * part, len = nt - off < (size_t)part ? nt - off : (size_t)part;
                CHECK(parts[p] == crc32c(neo + off, len));
            }
            uint32_t osz[16];
            CHECK(tsgpu_detransform((tsgpu_ctx*)(intptr_t)h, (uint32_t)ZA, neo, nt, nsz, got, key2, aad2, 16, back, n + 64, osz) == 0);
            CHECK(memcmp(back, seg, n) == 0);
        }
        if (from & TSGPU_FLAG_AES) {
            uint32_t crcs[3] = {7, 7, 7}, nsz[16], parts[64], np = 0;
            /* the old object's own IVs under the same key */
            CHECK(rewrite_windows(env, h, from, obj, sizes, got, cs, (jlong)n, 3, jkey, jaad, ZA, jkey, jaad, ivs, neo, neo_cap,
                                  nsz, 3000, parts, &np, crcs) == -1);
            CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "repeats the IV") != NULL);
            obj[sizes[0] + sizes[1] + 50] ^= 1;                       /* chunk 2's ciphertext */
            CHECK(rewrite_windows(env, h, from, obj, sizes, got, cs, (jlong)n, 3, jkey, jaad, ZA, jkey2, jaad2, ivs2, neo, neo_cap,
                                  nsz, 3000, parts, &np, crcs) == -1);
            CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strstr(thrown_msg, "chunk 2") != NULL);
            CHECK(crcs[0] == 7);
        }
        free(obj);
    }
    /* argument refusals */
    uint8_t small[64] = {0}, cursor[192] = {0}, one[16];
    uint32_t s1 = 16;
    jarray ts0 = mk_array(1, NULL, 0, 4), ts1 = mk_array(1, &s1, 1, 4), nts0 = mk_array(1, NULL, 0, 4), nts1 = mk_array(1, NULL, 1, 4);
    jarray pc = mk_array(1, NULL, 4, 4), np0 = mk_array(1, NULL, 0, 4), np1 = mk_array(1, NULL, 1, 4);
    jarray out2 = mk_array(1, NULL, 2, 4), out3 = mk_array(1, NULL, 3, 4);
    jobject d = mk_direct(neo, 1024);
    #define TRY(...) do { thrown_class[0] = 0; RC(rewriteObject)(__VA_ARGS__); } while (0)
    TRY(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts0, 100, pc, np1, mk_direct(small, 64), 1, out3);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "192") != NULL);
    TRY(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts0, 100, pc, np1, mk_direct(cursor, 192), 1, out2);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    TRY(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts0, 100, pc, np0, mk_direct(cursor, 192), 1, out3);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    TRY(env, NULL, h, 0, NULL, 0, ts0, cs, 0, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts0, 0, pc, np1, mk_direct(cursor, 192), 1, out3);
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    memset(one, 'x', sizeof one);
    TRY(env, NULL, h, 0, mk_direct(one, 16), 16, ts1, cs, 16, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts1, 100, pc, np1,
        mk_direct(cursor, 192), 1, out3);                                                               /* AES without IVs */
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "toIvs") != NULL);
    TRY(env, NULL, h, 0, mk_direct(one, 16), 16, ts1, cs, 16, NULL, NULL, ZA, jkey2, jaad2, NULL, d, 1024, nts0, 100, pc, np1,
        mk_direct(cursor, 192), 1, out3);                                                               /* no room for the new sizes */
    CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0);
    TRY(env, NULL, h, TSGPU_FLAG_ZSTD, NULL, 0, ts0, cs, 0, NULL, NULL, TSGPU_FLAG_ZSTD, NULL, NULL, NULL, d, 1024, nts0, 100, pc, np1,
        mk_direct(cursor, 192), 1, out3);                                                               /* empty segment */
    CHECK(thrown_class[0] == 0 && ((uint32_t*)np1->data)[0] == 0);
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
