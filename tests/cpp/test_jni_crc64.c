/*
 * Drives the CRC-64/NVME exports of jni/tsgpu_jni.c (Crc64.transformParts, Crc64.checkObject, Crc64.rewriteObject) through a
 * fake JNIEnv.  transformParts runs in the window flow of GpuTransformChunkEnumeration.fill with crc64Parts: windows of 1 and 3
 * chunks, one records cursor and one parts cursor per segment, segmentEndsHere on the short window or on an empty end call after
 * a full one; the part CRCs and the object CRC equal the CRC-64/NVME of the bytes the windows wrote.  checkObject and
 * rewriteObject give the 64-bit words of the object, the segment and the new object.  The exports refuse short checksum buffers
 * (IllegalArgumentException) and a partCrc64 buffer below the bound (RuntimeException, nothing written).  Links the test-only
 * SIMT build.
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
#define C64(f) Java_io_aiven_kafka_tieredstorage_transform_gpu_Crc64_##f

static uint64_t crc64nvme(const uint8_t* p, size_t n) {
    uint64_t c = ~0ull;
    for (size_t i = 0; i < n; i++) { c ^= p[i]; for (int k = 0; k < 8; k++) c = (c >> 1) ^ (0x9A6C9329AC4BC9B5ull & (0ull - (c & 1))); }
    return ~c;
}

/* The enumeration's windows with CRC-64 parts; returns 0, or -1 with the failing window's exception. */
static int enumerate(JNIEnv* env, jlong h, jint flags, const uint8_t* seg, size_t n, jint cs, int win, jlong part, uint8_t* out,
                     size_t* out_len, uint32_t* sizes_out, size_t* nsizes, uint64_t* crcs, size_t* nparts, uint64_t* ocrc,
                     jarray jkey, jarray jaad) {
    uint8_t rcursor[64] = {0}, pcursor[32] = {0};
    jobject rcur = mk_direct(rcursor, 64), pcur = mk_direct(pcursor, 32);
    const size_t wbytes = (size_t)win * cs;
    uint8_t* in = malloc(wbytes + 1); uint8_t* dst = malloc(wbytes * 2 + 4096);
    size_t pos = 0, o = 0, k = 0, ns = 0;
    int rc = 0, eof = 0;
    while (!eof) {
        const size_t total = n - pos < wbytes ? n - pos : wbytes;
        memcpy(in, seg + pos, total);
        eof = total < wbytes;
        const int chunks = (int)((total + cs - 1) / cs);
        uint8_t ivs[12 * 64];
        for (int i = 0; i < 12 * chunks; i++) ivs[i] = (uint8_t)(pos / cs * 12 + i);
        const jlong bound = total ? (jlong)tsgpu_transform_bound((uint32_t)flags, total, (uint32_t)cs) : 0;
        const jlong cap = (part - 1 + bound) / part + 1;                 /* what PartsCursor.transform passes */
        uint64_t* pc = calloc((size_t)cap + 1, 8);
        uint64_t obj = 0xdeadbeefdeadbeefull;
        jarray jivs = mk_array(2, ivs, chunks ? 12 * chunks : 12, 1), sizes = mk_array(1, NULL, chunks, 4), jn = mk_array(1, NULL, 1, 4);
        const jint got = C64(transformParts)(env, NULL, h, flags, mk_direct(in, (jlong)wbytes), (jlong)total, cs, jkey, jaad, jivs,
                                             mk_direct(dst, (jlong)(wbytes * 2 + 4096)), sizes, rcur, (jboolean)eof, part, pcur,
                                             mk_direct(pc, 8 * cap), jn, mk_direct(&obj, 8));
        if (got < 0) { rc = -1; free(pc); break; }
        size_t t = 0;
        for (int i = 0; i < got; i++) { sizes_out[ns++] = (uint32_t)((jint*)sizes->data)[i]; t += (size_t)((jint*)sizes->data)[i]; }
        memcpy(out + o, dst, t);
        o += t;
        for (jint i = 0; i < ((jint*)jn->data)[0]; i++) crcs[k++] = pc[i];
        if (eof) *ocrc = obj;
        else CHECK(obj == 0xdeadbeefdeadbeefull);
        free(pc);
        pos += total;
    }
    *out_len = o; *nparts = k; *nsizes = ns;
    free(in); free(dst);
    return rc;
}

int main(void) {
    JNIEnv envp = &table; JNIEnv* env = &envp;
    CHECK(crc64nvme((const uint8_t*)"123456789", 9) == 0xAE8B14860A799888ull);
    const jint cs = 1000;
    jlong h = NS(create)(env, NULL, NULL, cs, 2);
    CHECK(h != 0);
    static uint8_t seg[40000], obj[80000], neo[120000];
    static uint64_t crcs[80000];
    static uint32_t tsz[100];
    for (size_t i = 0; i < sizeof seg; i++) seg[i] = (uint8_t)("topic-partition-offset "[i % 23] + (i >> 9));
    uint8_t key[32], aad[16], key2[32];
    for (int i = 0; i < 32; i++) { key[i] = (uint8_t)(i * 5 + 3); key2[i] = (uint8_t)(i * 7 + 1); }
    for (int i = 0; i < 16; i++) aad[i] = (uint8_t)(100 + i);
    jarray jkey = mk_array(2, key, 32, 1), jaad = mk_array(2, aad, 16, 1), jkey2 = mk_array(2, key2, 32, 1);
    const jint flag_sets[3] = {TSGPU_FLAG_AES, TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES, TSGPU_FLAG_ZSTD};
    const size_t lens[2] = {30000, 30500};                                   /* a full last window (empty end call) and a short one */
    const jlong parts[3] = {7, 1028 * 2 + 1, 1 << 20};
    for (int f = 0; f < 3; f++) for (int l = 0; l < 2; l++) for (int p = 0; p < 3; p++) for (int win = 1; win <= 3; win += 2) {
        size_t olen = 0, np = 0, ns = 0; uint64_t ocrc = 0;
        thrown_msg[0] = 0;
        CHECK(enumerate(env, h, flag_sets[f], seg, lens[l], cs, win, parts[p], obj, &olen, tsz, &ns, crcs, &np, &ocrc, jkey, jaad) == 0);
        CHECK(thrown_msg[0] == 0);
        size_t k = 0; int ok = 1;
        for (size_t off = 0; off < olen; off += (size_t)parts[p], k++)
            ok = ok && k < np && crcs[k] == crc64nvme(obj + off, olen - off < (size_t)parts[p] ? olen - off : (size_t)parts[p]);
        CHECK(ok && k == np);
        CHECK(ocrc == crc64nvme(obj, olen));
        if (p || win != 3) continue;
        /* the check of the object just written, in one window, and its rewrite to Zstd+AES under another key */
        uint8_t ccur[128] = {0}, rcur[192] = {0};
        uint64_t words[3] = {0, 0, 0};
        jarray jts = mk_array(1, tsz, (jlong)ns, 4);
        C64(checkObject)(env, NULL, h, flag_sets[f], mk_direct(obj, (jlong)olen), (jlong)olen, jts, cs, (jlong)lens[l], jkey, jaad,
                         mk_direct(ccur, 128), 1, mk_direct(words, 16));
        CHECK(thrown_msg[0] == 0 && words[0] == crc64nvme(obj, olen) && words[1] == crc64nvme(seg, lens[l]));
        uint8_t nivs[12 * 64];
        for (size_t i = 0; i < sizeof nivs; i++) nivs[i] = (uint8_t)(i * 7 + 3);
        const jint to = (flag_sets[f] & TSGPU_FLAG_ZSTD) ? TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES : TSGPU_FLAG_ZSTD_DENSE | TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES;
        uint64_t pc[400], w3[3] = {0, 0, 0};
        jarray nts = mk_array(1, NULL, (jlong)ns, 4), jn = mk_array(1, NULL, 1, 4), jnivs = mk_array(2, nivs, sizeof nivs, 1);
        C64(rewriteObject)(env, NULL, h, flag_sets[f], mk_direct(obj, (jlong)olen), (jlong)olen, jts, cs, (jlong)lens[l], jkey, jaad,
                           to, jkey2, jaad, jnivs, mk_direct(neo, sizeof neo), sizeof neo, nts, 1000, mk_direct(pc, sizeof pc), jn,
                           mk_direct(rcur, 192), 1, mk_direct(w3, 24));
        CHECK(thrown_msg[0] == 0);
        size_t nlen = 0;
        for (size_t i = 0; i < ns; i++) nlen += (size_t)((jint*)nts->data)[i];
        CHECK(w3[0] == crc64nvme(obj, olen) && w3[1] == crc64nvme(neo, nlen) && w3[2] == crc64nvme(seg, lens[l]));
        int pok = ((jint*)jn->data)[0] == (jint)((nlen + 999) / 1000);
        for (size_t off = 0, i = 0; off < nlen; off += 1000, i++) pok = pok && pc[i] == crc64nvme(neo + off, nlen - off < 1000 ? nlen - off : 1000);
        CHECK(pok);
    }

    /* refusals: short checksum buffers, a partCrc64 buffer below the bound */
    {
        uint8_t r64[64] = {0}, p32[32] = {0}, c128[128] = {0};
        uint64_t small[2] = {77, 77}, o8 = 55;
        jarray sizes = mk_array(1, NULL, 4, 4), jivs = mk_array(2, key, 48, 1), jn = mk_array(1, NULL, 1, 4);
        const jint F = TSGPU_FLAG_AES;
        CHECK(C64(transformParts)(env, NULL, h, F, mk_direct(seg, 4000), 4000, cs, jkey, jaad, jivs, mk_direct(obj, sizeof obj), sizes,
                                  mk_direct(r64, 64), 1, 1000, mk_direct(p32, 32), mk_direct(small, 16), jn, mk_direct(&o8, 4)) == -1);
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "objectCrc64Out") != NULL);
        CHECK(C64(transformParts)(env, NULL, h, F, mk_direct(seg, 4000), 4000, cs, jkey, jaad, jivs, mk_direct(obj, sizeof obj), sizes,
                                  mk_direct(r64, 64), 1, 1000, mk_direct(p32, 32), mk_direct(small, 8), jn, mk_direct(&o8, 8)) == -1);
        CHECK(strcmp(thrown_class, "java/lang/RuntimeException") == 0 && strstr(thrown_msg, "part_crc64 too small") != NULL);
        CHECK(small[0] == 77 && small[1] == 77 && o8 == 55);
        jarray jts = mk_array(1, NULL, 1, 4);
        C64(checkObject)(env, NULL, h, F, mk_direct(seg, 4000), 4000, jts, cs, 1000, jkey, jaad, mk_direct(c128, 128), 1,
                         mk_direct(small, 8));
        CHECK(strcmp(thrown_class, "java/lang/IllegalArgumentException") == 0 && strstr(thrown_msg, "crcsOut") != NULL);
        thrown_msg[0] = 0;
    }
    NS(destroy)(env, NULL, h);
    printf("%s: %d checks, %d failures\n", failures ? "FAILED" : "OK", checks, failures);
    return failures ? 1 : 0;
}
