/*
 * Drives TsGpu.FLAG_REFRAME through the object-rewrite path of jni/tsgpu_jni.c (RewriteCursor.rewriteObject) and a fake JNIEnv, in
 * the window flow of an operator tool: a Zstd+AES object the oracle wrote (libzstd level 3, no Content_Checksum: what the Java
 * plugin wrote) is rewritten under a new key in windows of 1, 4 and 11 chunks, with toFlags passed through unchanged.  With
 * FLAG_REFRAME | ZSTD_CHECKSUM every new chunk is 4 bytes longer and its frame is libzstd's checksummed frame; with ZSTD_DENSE as
 * well no chunk grows by more than 4 bytes.  dst and partCrcs are sized for the 4 extra bytes per chunk; the part CRCs, the three
 * CRCs and a tsgpu_check_object of the new object agree with a host CRC-32C.  REFRAME without ZSTD in fromFlags throws
 * IllegalArgumentException naming the flag.  Links the test-only SIMT build and the oracle.
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
    const uint64_t cap = ora_transform_bound((uint32_t)ZA, n, (uint32_t)cs) + 64;
    uint8_t* obj = malloc(cap);
    uint32_t sizes[16], got = 16;
    CHECK(ora_transform_segment((uint32_t)ZA, seg, n, (uint32_t)cs, key, aad, 32, ivs, obj, cap, sizes, &got) == 0);
    CHECK(got == nch);
    size_t total = 0;
    for (uint32_t i = 0; i < got; i++) total += sizes[i];
    const uint64_t neo_cap = total + 32ull * nch + 64;                 /* the old chunks, 4 bytes more each, IV and tag: the dst bound */
    uint8_t* neo = malloc(neo_cap);
    uint8_t frame[8192], want[8192];
    const jint to[2] = {ZA | TSGPU_FLAG_ZSTD_CHECKSUM | (jint)TSGPU_FLAG_REFRAME,
                        ZA | TSGPU_FLAG_ZSTD_DENSE | TSGPU_FLAG_ZSTD_CHECKSUM | (jint)TSGPU_FLAG_REFRAME};
    CHECK(TSGPU_FLAG_REFRAME == 64);
    for (int t = 0; t < 2; t++) for (uint32_t win = 1; win <= 11; win += win == 1 ? 3 : 7) {
        uint32_t crcs[3] = {0, 0, 0}, nsz[16], parts[64], np = 0;
        const jlong part = 3000;
        CHECK(rewrite_windows(env, h, ZA, obj, sizes, got, cs, (jlong)n, win, jkey, jaad, to[t], jkey2,
                              jaad2, ivs2, neo, neo_cap, nsz, part, parts, &np, crcs) == 0);
        size_t nt = 0, at = 0;
        for (uint32_t i = 0; i < got; i++) {
            nt += nsz[i];
            CHECK(t ? nsz[i] <= sizes[i] + 4 : nsz[i] == sizes[i] + 4);
        }
        CHECK(crcs[0] == crc32c(obj, total) && crcs[1] == crc32c(neo, nt) && crcs[2] == crc32c(seg, n));
        CHECK(np == (nt + part - 1) / part);
        for (uint32_t p = 0; p < np; p++) {
            const size_t off = (size_t)p * part, len = nt - off < (size_t)part ? nt - off : (size_t)part;
            CHECK(parts[p] == crc32c(neo + off, len));
        }
        for (uint32_t i = 0; i < got; i++) {
            const size_t len = i + 1 < got ? (size_t)cs : n - (size_t)i * cs;
            CHECK(ora_aesgcm_decrypt_chunk(key2, aad2, 16, neo + at, nsz[i], frame) == 0);
            const size_t fl = nsz[i] - 28;
            CHECK(frame[4] & 0x04);                                     /* every frame carries its Content_Checksum */
            if (!t) {
                const int64_t m = ora_zstd_compress_checksum(seg + (size_t)i * cs, len, want, sizeof want, 3);
                CHECK(m == (int64_t)fl && memcmp(frame, want, fl) == 0);
            }
            CHECK(ora_zstd_decompress_chunk(frame, fl, want, sizeof want) == (int64_t)len && memcmp(want, seg + (size_t)i * cs, len) == 0);
            at += nsz[i];
        }
        /* the new object passes the check with the old object's segment CRC */
        uint8_t cur[128] = {0};
        uint32_t ocrc = 0, scrc = 0;
        CHECK(tsgpu_check_object((tsgpu_ctx*)(intptr_t)h, (uint32_t)ZA, neo, nt, nsz, got,
                                 (uint32_t)cs, n, key2, aad2, 16, (tsgpu_check_cursor*)cur, 1, &ocrc, &scrc) == 0);
        CHECK(ocrc == crcs[1] && scrc == crcs[2]);
    }
    /* REFRAME needs ZSTD on both sides */
    {
        uint32_t crcs[3] = {7, 7, 7}, nsz[16], parts[64], np = 0;
        uint32_t psz[16];
        for (uint32_t i = 0; i < nch; i++) psz[i] = i + 1 < nch ? (uint32_t)cs : (uint32_t)(n - (size_t)i * cs);
        CHECK(rewrite_windows(env, h, 0, seg, psz, nch, cs, (jlong)n, 4, NULL, NULL, to[0], jkey2, jaad2, ivs2, neo, neo_cap,
                              nsz, 3000, parts, &np, crcs) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "TSGPU_FLAG_REFRAME") != NULL);
        CHECK(crcs[0] == 7);
    }
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
