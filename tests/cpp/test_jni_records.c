/*
 * Drives the record-validation path of jni/tsgpu_jni.c (RecordsCursor.transformCursor) through a fake JNIEnv, in the window
 * flow of GpuTransformChunkEnumeration.fill: windows of batchChunks chunks, one cursor per segment, segmentEndsHere on the
 * short window, or on an empty call when the segment ends with a full window.  Checks that a valid segment whose record
 * batches cross the windows passes and transforms to the bytes of one whole-segment call; that a damaged batch across a
 * window boundary, and a segment ending inside a batch, throw RuntimeException (TSGPU_E_RECORDS) naming its position; and
 * that TSGPU_VALIDATE_RECORDS=1 reaches this call.  Links the test-only SIMT build.
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
#define RC(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_RecordsCursor_##f

/* ---- a Kafka log segment: v2 record batches (CRC-32C at +17 over [+21, end)) and v0 message sets (CRC-32 at +12 over [+16, end)) */
static uint32_t crc(uint32_t poly, const uint8_t* p, size_t n) {
    uint32_t c = 0xffffffffu;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (poly & (0u - (c & 1u))); }
    return ~c;
}
static void be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }
static size_t n_entries;
static size_t starts[256];
static size_t make_segment(uint8_t* seg, size_t cap) {
    static const uint32_t lens[] = {61, 700, 2999, 150, 5000, 90, 26, 1234, 4100, 61, 333, 40};   /* 26 and 40: v0 entries */
    size_t x = 0;
    n_entries = 0;
    for (int i = 0; x + 5000 < cap; i++) {
        const uint32_t len = lens[i % 12];
        const int v0 = len < 61;
        uint8_t* e = seg + x;
        for (uint32_t j = 0; j < len; j++) e[j] = (uint8_t)(j * 131 + i * 17 + (j >> 5));
        memset(e, 0, 8); be32(e + 4, (uint32_t)i);
        be32(e + 8, len - 12);
        e[16] = v0 ? 0 : 2;
        if (v0) be32(e + 12, crc(0xEDB88320u, e + 16, len - 16));
        else be32(e + 17, crc(0x82F63B78u, e + 21, len - 21));
        starts[n_entries++] = x;
        x += len;
    }
    return x;
}

static int pos_named(size_t at) {
    char want[64];
    snprintf(want, sizeof want, "segment position %zu", at);
    const char* p = strstr(thrown_msg, want);
    return p && (p[strlen(want)] < '0' || p[strlen(want)] > '9');
}

/* GpuTransformChunkEnumeration.fill over `seg`: windows of `win` chunks of `cs` bytes.  Returns 0, or -1 with the exception
 * of the window that failed; the transformed bytes go to out (when given) back to back. */
static int enumerate(JNIEnv* env, jlong h, jint flags, const uint8_t* seg, size_t n, jint cs, int win, uint8_t* out, size_t* out_len,
                     jarray jkey, jarray jaad) {
    uint8_t cursor[64] = {0};
    jobject cur = mk_direct(cursor, 64);
    const size_t wbytes = (size_t)win * cs;
    uint8_t* in = malloc(wbytes + 1); uint8_t* dst = malloc(wbytes * 2 + 4096);
    size_t pos = 0, o = 0;
    int rc = 0, eof = 0;
    while (!eof) {
        const size_t total = n - pos < wbytes ? n - pos : wbytes;
        memcpy(in, seg + pos, total);
        eof = total < wbytes;
        const int chunks = (int)((total + cs - 1) / cs);
        uint8_t ivs[12 * 64];
        for (int i = 0; i < 12 * chunks; i++) ivs[i] = (uint8_t)(pos / cs * 12 + i);
        jarray jivs = mk_array(2, ivs, chunks ? 12 * chunks : 12, 1), sizes = mk_array(1, NULL, chunks, 4);
        const jint got = RC(transformCursor)(env, NULL, h, flags, mk_direct(in, (jlong)wbytes), (jlong)total, cs, jkey, jaad, jivs,
                                             mk_direct(dst, (jlong)(wbytes * 2 + 4096)), sizes, cur, (jboolean)(eof || total == 0));
        if (got < 0) { rc = -1; break; }
        size_t t = 0;
        for (int i = 0; i < got; i++) t += (size_t)((jint*)sizes->data)[i];
        if (out) memcpy(out + o, dst, t);
        o += t;
        pos += total;
        if (total == 0) break;
    }
    if (out_len) *out_len = o;
    free(in); free(dst);
    return rc;
}

int main(void) {
    JNIEnv envp = &table; JNIEnv* env = &envp;
    const jint cs = 1000, win = 3, flags = TSGPU_FLAG_AES | TSGPU_FLAG_VALIDATE_RECORDS;
    jlong h = NS(create)(env, NULL, NULL, cs, 2);
    CHECK(h != 0);
    static uint8_t seg[60000], bad[60000], a[90000], b[90000];
    const size_t n = make_segment(seg, sizeof seg);
    uint8_t key[32], aad[16];
    for (int i = 0; i < 32; i++) key[i] = (uint8_t)(i * 5 + 3);
    for (int i = 0; i < 16; i++) aad[i] = (uint8_t)(100 + i);
    jarray jkey = mk_array(2, key, 32, 1), jaad = mk_array(2, aad, 16, 1);

    /* a valid segment whose batches cross windows: the windows give exactly the bytes of one whole-segment call */
    size_t alen = 0;
    CHECK(enumerate(env, h, flags, seg, n, cs, win, a, &alen, jkey, jaad) == 0 && thrown_msg[0] == 0);
    {
        const int chunks = (int)((n + cs - 1) / cs);
        uint8_t* ivs = malloc(12 * (size_t)chunks);
        for (int i = 0; i < 12 * chunks; i++) ivs[i] = (uint8_t)i;       /* window k's chunk j has IV bytes (3k + j) * 12 + ... */
        jarray jivs = mk_array(2, ivs, 12 * chunks, 1), sizes = mk_array(1, NULL, chunks, 4);
        const jint got = NS(transform)(env, NULL, h, flags, mk_direct(seg, (jlong)n), (jlong)n, cs, jkey, jaad, jivs,
                                       mk_direct(b, sizeof b), sizes);
        size_t blen = 0;
        for (int i = 0; i < got; i++) blen += (size_t)((jint*)sizes->data)[i];
        CHECK(got == chunks && blen == alen && memcmp(a, b, alen) == 0);
        free(ivs);
    }

    /* a damaged batch that crosses a window boundary: RuntimeException at its start, from the window where it ends */
    size_t e = 0;
    for (size_t i = 0; i + 1 < n_entries; i++)
        if (starts[i] / (win * cs) != (starts[i + 1] - 1) / (win * cs) && starts[i] > 0) { e = i; break; }
    CHECK(e > 0);
    memcpy(bad, seg, n);
    bad[(starts[e] + starts[e + 1]) / 2] ^= 0x20;
    thrown_msg[0] = 0;
    CHECK(enumerate(env, h, flags, bad, n, cs, win, NULL, NULL, jkey, jaad) == -1);
    CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strstr(thrown_msg, "Record is corrupt (stored crc = ") != NULL);
    CHECK(strstr(thrown_msg, "check: crc") != NULL && pos_named(starts[e]));

    /* a segment that ends inside a batch, with a full last window: the empty call that ends the segment fails with length */
    size_t cut = 0;
    for (size_t k = 1; k * win * cs < n; k++) {
        const size_t c = k * win * cs;
        for (size_t i = 0; i + 1 < n_entries; i++)
            if (starts[i] < c && c < starts[i + 1]) { if (starts[i] + 21 < c) cut = c; break; }
        if (cut) break;
    }
    CHECK(cut > 0);
    thrown_msg[0] = 0;
    CHECK(enumerate(env, h, flags, seg, cut, cs, win, NULL, NULL, jkey, jaad) == -1);
    CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strstr(thrown_msg, "check: length") != NULL);

    /* without the flag nothing is checked */
    thrown_msg[0] = 0;
    CHECK(enumerate(env, h, TSGPU_FLAG_AES, bad, n, cs, win, NULL, NULL, jkey, jaad) == 0 && thrown_msg[0] == 0);
    /* a cursor buffer shorter than 64 bytes is refused */
    {
        uint8_t small[32] = {0};
        jarray sizes = mk_array(1, NULL, 1, 4), jivs = mk_array(2, key, 12, 1);
        CHECK(RC(transformCursor)(env, NULL, h, flags, mk_direct(seg, 100), 100, cs, jkey, jaad, jivs, mk_direct(b, sizeof b), sizes,
                                  mk_direct(small, 32), 1) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "cursor") != NULL);
        thrown_msg[0] = 0;
    }
    NS(destroy)(env, NULL, h);

    /* TSGPU_VALIDATE_RECORDS=1 in the broker's environment reaches the enumeration's call without the flag */
    setenv("TSGPU_VALIDATE_RECORDS", "1", 1);
    jlong h2 = NS(create)(env, NULL, NULL, cs, 2);
    CHECK(h2 != 0);
    CHECK(enumerate(env, h2, TSGPU_FLAG_AES, seg, n, cs, win, NULL, NULL, jkey, jaad) == 0 && thrown_msg[0] == 0);
    CHECK(enumerate(env, h2, TSGPU_FLAG_AES, bad, n, cs, win, NULL, NULL, jkey, jaad) == -1);
    CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && pos_named(starts[e]));
    NS(destroy)(env, NULL, h2);
    unsetenv("TSGPU_VALIDATE_RECORDS");

    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
