/*
 * tsoracle.c — CPU oracle (TEST INFRASTRUCTURE ONLY; see tsoracle.h for scope, citations and pinning).
 * Paths cited as core/M/... = <reference>/core/src/main/java/io/aiven/kafka/tieredstorage/...
 */
#define _GNU_SOURCE
#include "tsoracle.h"
#include <dlfcn.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <openssl/evp.h>

static __thread char g_err[256];
static int fail(int code, const char* fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
const char* ora_last_error(void) { return g_err; }

/* ------------------------------------------------------------------ zstd via dlopen (no zstd.h in the image) */
typedef struct ZSTD_CCtx_s ZSTD_CCtx;
static struct {
    void* h;
    ZSTD_CCtx* (*createCCtx)(void);
    size_t (*freeCCtx)(ZSTD_CCtx*);
    size_t (*setParameter)(ZSTD_CCtx*, int, int);
    size_t (*setPledgedSrcSize)(ZSTD_CCtx*, unsigned long long);
    size_t (*compress2)(ZSTD_CCtx*, void*, size_t, const void*, size_t);
    size_t (*compressBound)(size_t);
    unsigned long long (*getFrameContentSize)(const void*, size_t);
    size_t (*decompress)(void*, size_t, const void*, size_t);
    unsigned (*isError)(size_t);
    const char* (*getErrorName)(size_t);
    const char* (*versionString)(void);
} Z;
#define ZSTD_c_contentSizeFlag 200   /* zstd.h: ZSTD_cParameter */
#define ZSTD_CONTENTSIZE_UNKNOWN (0ULL - 1)
#define ZSTD_CONTENTSIZE_ERROR   (0ULL - 2)

static int zload(void) {
    if (Z.h) return 0;
    void* h = dlopen("libzstd.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!h) return fail(ORA_E_NOLIB, "dlopen libzstd.so.1: %s", dlerror());
#define L(f, n) *(void**)(&Z.f) = dlsym(h, n); if (!Z.f) return fail(ORA_E_NOLIB, "dlsym %s", n);
    L(createCCtx, "ZSTD_createCCtx") L(freeCCtx, "ZSTD_freeCCtx") L(setParameter, "ZSTD_CCtx_setParameter")
    L(setPledgedSrcSize, "ZSTD_CCtx_setPledgedSrcSize") L(compress2, "ZSTD_compress2")
    L(compressBound, "ZSTD_compressBound") L(getFrameContentSize, "ZSTD_getFrameContentSize")
    L(decompress, "ZSTD_decompress") L(isError, "ZSTD_isError") L(getErrorName, "ZSTD_getErrorName")
    L(versionString, "ZSTD_versionString")
#undef L
    Z.h = h;
    return 0;
}
const char* ora_zstd_version(void) { return zload() ? "" : Z.versionString(); }
size_t ora_zstd_bound(size_t n) { return zload() ? 0 : Z.compressBound(n); }

/* CompressionChunkEnumeration.nextElement (core/M/transform/CompressionChunkEnumeration.java:49-62):
 * new ZstdCompressCtx (default level 3), setPledgedSrcSize(len), setContentSize(true), compress(chunk). */
int64_t ora_zstd_compress_chunk(const uint8_t* src, size_t n, uint8_t* dst, size_t cap) {
    if (zload()) return ORA_E_NOLIB;
    ZSTD_CCtx* c = Z.createCCtx();
    if (!c) return fail(ORA_E_ARG, "ZSTD_createCCtx failed");
    Z.setPledgedSrcSize(c, n);
    Z.setParameter(c, ZSTD_c_contentSizeFlag, 1);
    size_t r = Z.compress2(c, dst, cap, src, n);
    Z.freeCCtx(c);
    if (Z.isError(r)) return fail(ORA_E_SHORT, "zstd compress: %s", Z.getErrorName(r));
    return (int64_t)r;
}
/* Same call sequence at another compression level: only used to widen the decoder's test coverage (the reference
 * itself always runs the default level). */
int64_t ora_zstd_compress_level(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int level) {
    if (zload()) return ORA_E_NOLIB;
    ZSTD_CCtx* c = Z.createCCtx();
    if (!c) return fail(ORA_E_ARG, "ZSTD_createCCtx failed");
    Z.setPledgedSrcSize(c, n);
    Z.setParameter(c, ZSTD_c_contentSizeFlag, 1);
    Z.setParameter(c, 100 /* ZSTD_c_compressionLevel */, level);
    size_t r = Z.compress2(c, dst, cap, src, n);
    Z.freeCCtx(c);
    if (Z.isError(r)) return fail(ORA_E_SHORT, "zstd compress: %s", Z.getErrorName(r));
    return (int64_t)r;
}
/* A frame WITH Content_Checksum (ZSTD_c_checksumFlag): the reference never writes one (no setChecksum call anywhere), but
 * zstd-jni's reader verifies it when present, so the decoder under test has to as well.  Test coverage only. */
int64_t ora_zstd_compress_checksum(const uint8_t* src, size_t n, uint8_t* dst, size_t cap, int level) {
    if (zload()) return ORA_E_NOLIB;
    ZSTD_CCtx* c = Z.createCCtx();
    if (!c) return fail(ORA_E_ARG, "ZSTD_createCCtx failed");
    Z.setPledgedSrcSize(c, n);
    Z.setParameter(c, ZSTD_c_contentSizeFlag, 1);
    Z.setParameter(c, 201 /* ZSTD_c_checksumFlag */, 1);
    Z.setParameter(c, 100 /* ZSTD_c_compressionLevel */, level);
    size_t r = Z.compress2(c, dst, cap, src, n);
    Z.freeCCtx(c);
    if (Z.isError(r)) return fail(ORA_E_SHORT, "zstd compress: %s", Z.getErrorName(r));
    return (int64_t)r;
}
/* Zstd.decompressedSize (DecompressionChunkEnumeration.java:41): <0 => "Invalid decompressed size" */
int64_t ora_zstd_content_size(const uint8_t* frame, size_t n) {
    if (zload()) return ORA_E_NOLIB;
    unsigned long long r = Z.getFrameContentSize(frame, n);
    if (r == ZSTD_CONTENTSIZE_UNKNOWN || r == ZSTD_CONTENTSIZE_ERROR)
        return fail(ORA_E_CORRUPT, "Invalid decompressed size: %lld", (long long)r);
    return (int64_t)r;
}
int64_t ora_zstd_decompress_chunk(const uint8_t* frame, size_t n, uint8_t* dst, size_t cap) {
    if (zload()) return ORA_E_NOLIB;
    size_t r = Z.decompress(dst, cap, frame, n);
    if (Z.isError(r)) return fail(ORA_E_CORRUPT, "zstd decompress: %s", Z.getErrorName(r));
    return (int64_t)r;
}

/* ------------------------------------------------------------------ AES-256-GCM through OpenSSL EVP
 * AesEncryptionProvider.encryptionCipher (core/M/security/AesEncryptionProvider.java:60-75):
 * fresh cipher per chunk, 12-byte IV, updateAAD(aad), 128-bit tag; layout IV||CT||TAG
 * (core/M/transform/EncryptionChunkEnumeration.java:65-84). */
int ora_aesgcm_encrypt_chunk(const uint8_t key[32], const uint8_t iv[12], const uint8_t* aad, size_t aad_len,
                             const uint8_t* pt, size_t n, uint8_t* out) {
    EVP_CIPHER_CTX* c = EVP_CIPHER_CTX_new();
    int len = 0, ok = 1;
    ok &= EVP_EncryptInit_ex(c, EVP_aes_256_gcm(), NULL, NULL, NULL);
    ok &= EVP_CIPHER_CTX_ctrl(c, EVP_CTRL_GCM_SET_IVLEN, ORA_IV_SIZE, NULL);
    ok &= EVP_EncryptInit_ex(c, NULL, NULL, key, iv);
    if (aad_len) ok &= EVP_EncryptUpdate(c, NULL, &len, aad, (int)aad_len);
    memcpy(out, iv, ORA_IV_SIZE);
    size_t done = 0;
    while (ok && done < n) {               /* EVP takes int lengths */
        size_t step = n - done > (1u << 30) ? (1u << 30) : n - done;
        ok &= EVP_EncryptUpdate(c, out + ORA_IV_SIZE + done, &len, pt + done, (int)step);
        done += step;
    }
    ok &= EVP_EncryptFinal_ex(c, out + ORA_IV_SIZE + n, &len);
    ok &= EVP_CIPHER_CTX_ctrl(c, EVP_CTRL_GCM_GET_TAG, ORA_TAG_SIZE, out + ORA_IV_SIZE + n);
    EVP_CIPHER_CTX_free(c);
    return ok ? ORA_OK : fail(ORA_E_ARG, "EVP encrypt failed");
}
/* DecryptionChunkEnumeration.nextElement (core/M/transform/DecryptionChunkEnumeration.java:53-62) with
 * AesEncryptionProvider.decryptionCipher (:77-98): IV = first 12 bytes of the chunk. */
int ora_aesgcm_decrypt_chunk(const uint8_t key[32], const uint8_t* aad, size_t aad_len,
                             const uint8_t* in, size_t m, uint8_t* out) {
    if (m < ORA_IV_SIZE + ORA_TAG_SIZE) return fail(ORA_E_AUTH, "Input too short - need tag");
    size_t n = m - ORA_IV_SIZE - ORA_TAG_SIZE;
    EVP_CIPHER_CTX* c = EVP_CIPHER_CTX_new();
    int len = 0, ok = 1;
    ok &= EVP_DecryptInit_ex(c, EVP_aes_256_gcm(), NULL, NULL, NULL);
    ok &= EVP_CIPHER_CTX_ctrl(c, EVP_CTRL_GCM_SET_IVLEN, ORA_IV_SIZE, NULL);
    ok &= EVP_DecryptInit_ex(c, NULL, NULL, key, in);
    if (aad_len) ok &= EVP_DecryptUpdate(c, NULL, &len, aad, (int)aad_len);
    size_t done = 0;
    while (ok && done < n) {
        size_t step = n - done > (1u << 30) ? (1u << 30) : n - done;
        ok &= EVP_DecryptUpdate(c, out + done, &len, in + ORA_IV_SIZE + done, (int)step);
        done += step;
    }
    ok &= EVP_CIPHER_CTX_ctrl(c, EVP_CTRL_GCM_SET_TAG, ORA_TAG_SIZE, (void*)(in + ORA_IV_SIZE + n));
    int fin = ok ? EVP_DecryptFinal_ex(c, out + n, &len) : 0;
    EVP_CIPHER_CTX_free(c);
    if (!ok) return fail(ORA_E_ARG, "EVP decrypt failed");
    if (fin <= 0) return fail(ORA_E_AUTH, "Tag mismatch");   /* javax.crypto.AEADBadTagException */
    return ORA_OK;
}

/* ------------------------------------------------------------------ plain-C AES-256 + GCM (FIPS-197, SP 800-38D) */
static uint8_t SBOX[256];
static int sbox_ready;
static uint8_t xt(uint8_t x) { return (uint8_t)((x << 1) ^ ((x >> 7) * 0x1b)); }
static void sbox_init(void) {
    if (sbox_ready) return;
    /* multiplicative inverse via log tables on generator 3, then the affine map */
    uint8_t p = 1, q = 1;
    do {
        p = p ^ (uint8_t)(p << 1) ^ ((p & 0x80) ? 0x1b : 0);
        q ^= q << 1; q ^= q << 2; q ^= q << 4; if (q & 0x80) q ^= 0x09;
        uint8_t x = q ^ (uint8_t)((q << 1) | (q >> 7)) ^ (uint8_t)((q << 2) | (q >> 6)) ^
                    (uint8_t)((q << 3) | (q >> 5)) ^ (uint8_t)((q << 4) | (q >> 4));
        SBOX[p] = x ^ 0x63;
    } while (p != 1);
    SBOX[0] = 0x63;
    sbox_ready = 1;
}
static void aes256_expand(const uint8_t key[32], uint8_t rk[240]) {
    sbox_init();
    memcpy(rk, key, 32);
    uint8_t rcon = 1;
    for (int i = 32; i < 240; i += 4) {
        uint8_t t[4] = { rk[i - 4], rk[i - 3], rk[i - 2], rk[i - 1] };
        if (i % 32 == 0) {
            uint8_t u = t[0];
            t[0] = SBOX[t[1]] ^ rcon; t[1] = SBOX[t[2]]; t[2] = SBOX[t[3]]; t[3] = SBOX[u];
            rcon = xt(rcon);
        } else if (i % 32 == 16) {
            for (int k = 0; k < 4; k++) t[k] = SBOX[t[k]];
        }
        for (int k = 0; k < 4; k++) rk[i + k] = rk[i - 32 + k] ^ t[k];
    }
}
static void aes256_block(const uint8_t rk[240], const uint8_t in[16], uint8_t out[16]) {
    uint8_t s[16], t[16];
    for (int i = 0; i < 16; i++) s[i] = in[i] ^ rk[i];
    for (int r = 1; r <= 14; r++) {
        for (int c = 0; c < 4; c++)            /* SubBytes + ShiftRows (column-major state) */
            for (int row = 0; row < 4; row++) t[4 * c + row] = SBOX[s[4 * ((c + row) & 3) + row]];
        if (r < 14) {
            for (int c = 0; c < 4; c++) {      /* MixColumns */
                uint8_t a0 = t[4 * c], a1 = t[4 * c + 1], a2 = t[4 * c + 2], a3 = t[4 * c + 3];
                s[4 * c]     = xt(a0) ^ (xt(a1) ^ a1) ^ a2 ^ a3;
                s[4 * c + 1] = a0 ^ xt(a1) ^ (xt(a2) ^ a2) ^ a3;
                s[4 * c + 2] = a0 ^ a1 ^ xt(a2) ^ (xt(a3) ^ a3);
                s[4 * c + 3] = (xt(a0) ^ a0) ^ a1 ^ a2 ^ xt(a3);
            }
        } else memcpy(s, t, 16);
        for (int i = 0; i < 16; i++) s[i] ^= rk[16 * r + i];
    }
    memcpy(out, s, 16);
}
void ora_aes256_encrypt_block(const uint8_t key[32], const uint8_t in[16], uint8_t out[16]) {
    uint8_t rk[240]; aes256_expand(key, rk); aes256_block(rk, in, out);
}
/* X <- X * Y in GF(2^128), SP 800-38D algorithm 1 (bit 0 = MSB of byte 0) */
static void gf_mul(uint8_t X[16], const uint8_t Y[16]) {
    uint8_t Zr[16] = {0}, V[16];
    memcpy(V, Y, 16);
    for (int i = 0; i < 128; i++) {
        if (X[i >> 3] & (0x80 >> (i & 7))) for (int k = 0; k < 16; k++) Zr[k] ^= V[k];
        int lsb = V[15] & 1;
        for (int k = 15; k > 0; k--) V[k] = (uint8_t)((V[k] >> 1) | (V[k - 1] << 7));
        V[0] >>= 1;
        if (lsb) V[0] ^= 0xe1;
    }
    memcpy(X, Zr, 16);
}
static void ghash_update(uint8_t Y[16], const uint8_t H[16], const uint8_t* d, size_t n) {
    while (n) {
        size_t k = n < 16 ? n : 16;
        for (size_t i = 0; i < k; i++) Y[i] ^= d[i];
        gf_mul(Y, H);
        d += k; n -= k;
    }
}
int ora_aesgcm_plain_encrypt(const uint8_t key[32], const uint8_t iv[12], const uint8_t* aad, size_t aad_len,
                             const uint8_t* pt, size_t n, uint8_t* ct, uint8_t tag[16]) {
    uint8_t rk[240], H[16] = {0}, J0[16], ctr[16], ks[16], Y[16] = {0}, L[16];
    aes256_expand(key, rk);
    aes256_block(rk, H, H);
    memcpy(J0, iv, 12); J0[12] = 0; J0[13] = 0; J0[14] = 0; J0[15] = 1;
    memcpy(ctr, J0, 16);
    for (size_t off = 0; off < n; off += 16) {
        for (int k = 15; k >= 12; k--) if (++ctr[k]) break;     /* inc32 */
        aes256_block(rk, ctr, ks);
        size_t m = n - off < 16 ? n - off : 16;
        for (size_t i = 0; i < m; i++) ct[off + i] = pt[off + i] ^ ks[i];
    }
    ghash_update(Y, H, aad, aad_len);
    ghash_update(Y, H, ct, n);
    uint64_t ab = (uint64_t)aad_len * 8, cb = (uint64_t)n * 8;
    for (int i = 0; i < 8; i++) { L[i] = (uint8_t)(ab >> (56 - 8 * i)); L[8 + i] = (uint8_t)(cb >> (56 - 8 * i)); }
    ghash_update(Y, H, L, 16);
    aes256_block(rk, J0, ks);
    for (int i = 0; i < 16; i++) tag[i] = Y[i] ^ ks[i];
    return ORA_OK;
}

/* ------------------------------------------------------------------ segment-level chains */
static uint32_t chunk_count_u64(uint64_t len, uint32_t cs) { return (uint32_t)((len + cs - 1) / cs); }

uint64_t ora_transform_bound(uint32_t flags, uint64_t src_len, uint32_t chunk_size) {
    if (chunk_size == 0) chunk_size = (uint32_t)src_len;
    if (src_len == 0) return 64;
    uint64_t n = chunk_count_u64(src_len, chunk_size);
    uint64_t per = chunk_size;
    if (flags & ORA_FLAG_ZSTD) per = ora_zstd_bound(chunk_size);
    if (flags & ORA_FLAG_AES) per += ORA_IV_SIZE + ORA_TAG_SIZE;
    return n * per;
}

/* BaseTransformChunkEnumeration (core/M/transform/BaseTransformChunkEnumeration.java:61-93) splits by
 * chunk_size (0 => whole stream, empty read => end); then compress, then encrypt
 * (core/M/RemoteStorageManager.java:434-453: compression first, encryption second). */
int ora_transform_segment(uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                          const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                          uint8_t* dst, uint64_t dst_cap, uint32_t* sizes, uint32_t* n_chunks) {
    if (chunk_size == 0) chunk_size = (uint32_t)src_len;
    uint32_t n = src_len ? chunk_count_u64(src_len, chunk_size) : 0;
    uint64_t pos = 0;
    uint8_t* tmp = NULL;
    if ((flags & ORA_FLAG_ZSTD) && (flags & ORA_FLAG_AES)) tmp = malloc(ora_zstd_bound(chunk_size) + 64);
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* p = src + (uint64_t)i * chunk_size;
        size_t len = (size_t)((uint64_t)(i + 1) * chunk_size <= src_len ? chunk_size : src_len - (uint64_t)i * chunk_size);
        size_t out_len;
        if (flags & ORA_FLAG_ZSTD) {
            uint8_t* z = (flags & ORA_FLAG_AES) ? tmp : dst + pos;
            size_t zcap = (flags & ORA_FLAG_AES) ? ora_zstd_bound(chunk_size) + 64 : (size_t)(dst_cap - pos);
            int64_t r = ora_zstd_compress_chunk(p, len, z, zcap);
            if (r < 0) { free(tmp); return (int)r; }
            p = z; len = (size_t)r;
        }
        if (flags & ORA_FLAG_AES) {
            if (pos + len + 28 > dst_cap) { free(tmp); return fail(ORA_E_SHORT, "dst too small"); }
            int rc = ora_aesgcm_encrypt_chunk(key, ivs + (size_t)i * ORA_IV_SIZE, aad, aad_len, p, len, dst + pos);
            if (rc) { free(tmp); return rc; }
            out_len = len + 28;
        } else {
            if (!(flags & ORA_FLAG_ZSTD)) {
                if (pos + len > dst_cap) { free(tmp); return fail(ORA_E_SHORT, "dst too small"); }
                memcpy(dst + pos, p, len);
            }
            out_len = len;
        }
        sizes[i] = (uint32_t)out_len;
        pos += out_len;
    }
    free(tmp);
    *n_chunks = n;
    return ORA_OK;
}

/* BaseDetransform -> Decryption -> Decompression (core/M/fetch/DefaultChunkManager.java:50-70). */
int ora_detransform_chunks(uint32_t flags, const uint8_t* src, const uint32_t* tsizes, uint32_t n,
                           const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                           uint8_t* dst, uint64_t dst_cap, uint32_t* osizes) {
    uint64_t ip = 0, op = 0;
    for (uint32_t i = 0; i < n; i++) {
        const uint8_t* p = src + ip;
        size_t len = tsizes[i];
        uint8_t* tmp = NULL;
        if (flags & ORA_FLAG_AES) {
            if (len < 28) return fail(ORA_E_AUTH, "Input too short - need tag");
            if (flags & ORA_FLAG_ZSTD) { tmp = malloc(len); }
            uint8_t* o = tmp ? tmp : dst + op;
            if (!tmp && op + len - 28 > dst_cap) return fail(ORA_E_SHORT, "dst too small");
            int rc = ora_aesgcm_decrypt_chunk(key, aad, aad_len, p, len, o);
            if (rc) { free(tmp); return rc; }
            p = o; len -= 28;
        }
        if (flags & ORA_FLAG_ZSTD) {
            int64_t sz = ora_zstd_content_size(p, len);
            if (sz < 0) { free(tmp); return (int)sz; }
            if (op + (uint64_t)sz > dst_cap) { free(tmp); return fail(ORA_E_SHORT, "dst too small"); }
            int64_t r = ora_zstd_decompress_chunk(p, len, dst + op, (size_t)sz);
            free(tmp);
            if (r < 0) return (int)r;
            len = (size_t)r;
        } else if (!(flags & ORA_FLAG_AES)) {
            if (op + len > dst_cap) return fail(ORA_E_SHORT, "dst too small");
            memcpy(dst + op, p, len);
        }
        if (osizes) osizes[i] = (uint32_t)len;
        ip += tsizes[i];
        op += len;
    }
    return ORA_OK;
}

/* ------------------------------------------------------------------ ChunkIndex builders
 * core/M/manifest/index/AbstractChunkIndexBuilder.java:39-96 */
struct ora_index_builder {
    int32_t ocs, ofs, tcs;      /* tcs < 0 => variable */
    int32_t added; int finished;
    int32_t* sizes; int32_t cap;
};
static int check_size(int32_t v, const char* name) {
    if (v < 0) return fail(ORA_E_ARG, "%s must be non-negative, %d given", name, v);
    return 0;
}
ora_index_builder* ora_builder_new(int32_t ocs, int32_t ofs, int32_t tcs) {
    if (check_size(ocs, "Original chunk size") || check_size(ofs, "Original file size")) return NULL;
    ora_index_builder* b = calloc(1, sizeof *b);
    b->ocs = ocs; b->ofs = ofs; b->tcs = tcs;
    return b;
}
static int32_t remain(const ora_index_builder* b) { return b->ofs - b->added * b->ocs; }
static void push(ora_index_builder* b, int32_t v) {
    if (b->added >= b->cap) { b->cap = b->cap ? b->cap * 2 : 16; b->sizes = realloc(b->sizes, sizeof(int32_t) * b->cap); }
    b->sizes[b->added] = v;
}
int ora_builder_add_chunk(ora_index_builder* b, int32_t t) {
    if (b->finished) return fail(ORA_E_STATE, "Cannot add chunk to already finished index");
    if (check_size(t, "Transformed chunk size")) return ORA_E_ARG;
    if (remain(b) <= b->ocs) return fail(ORA_E_STATE, "This must be final chunk. Call `finish` instead.");
    if (b->tcs >= 0) {
        if (t != b->tcs) return fail(ORA_E_ARG, "Non-final chunk must be of size %d, but %d given", b->tcs, t);
    } else push(b, t);
    b->added += 1;
    return ORA_OK;
}
int ora_builder_finish(ora_index_builder* b, int32_t ft, ora_chunk_index** out) {
    if (b->finished) return fail(ORA_E_STATE, "Cannot finish already finished index");
    if (check_size(ft, "Transformed chunk size")) return ORA_E_ARG;
    if (remain(b) > b->ocs)
        return fail(ORA_E_STATE, "This cannot be final chunk: not enough chunks to cover original file. "
                                 "Call `addChunk` instead.");
    int rc;
    if (b->tcs >= 0) rc = ora_index_new_fixed(b->ocs, b->ofs, b->tcs, ft, out);
    else { push(b, ft); rc = ora_index_new_variable(b->ocs, b->ofs, b->sizes, b->added + 1, out); }
    if (rc) return rc;
    b->added += 1; b->finished = 1;
    return ORA_OK;
}
void ora_builder_free(ora_index_builder* b) { if (b) { free(b->sizes); free(b); } }

/* core/M/manifest/index/FixedSizeChunkIndex.java:53-80, VariableSizeChunkIndex.java:55-69, AbstractChunkIndex.java:35-49 */
static int index_common(int32_t ocs, int32_t ofs, int32_t ftcs) {
    if (ocs <= 0) return fail(ORA_E_ARG, "Original chunk size must be positive, %d given", ocs);
    if (ofs < 0) return fail(ORA_E_ARG, "Original file size must be non-negative, %d given", ofs);
    if (ftcs < 0) return fail(ORA_E_ARG, "Final transformed chunk size must be non-negative, %d given", ftcs);
    return 0;
}
int ora_index_new_fixed(int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, ora_chunk_index** out) {
    if (index_common(ocs, ofs, ftcs)) return ORA_E_ARG;
    if (tcs < 0) return fail(ORA_E_ARG, "Transformed chunk size must be non-negative, %d given", tcs);
    ora_chunk_index* x = calloc(1, sizeof *x);
    x->original_chunk_size = ocs; x->original_file_size = ofs; x->transformed_chunk_size = tcs;
    x->final_transformed_chunk_size = ftcs;
    x->chunk_count = ofs % ocs == 0 ? ofs / ocs : ofs / ocs + 1;
    *out = x;
    return ORA_OK;
}
int ora_index_new_variable(int32_t ocs, int32_t ofs, const int32_t* sizes, int32_t n, ora_chunk_index** out) {
    if (n <= 0) return fail(ORA_E_ARG, "transformedChunks cannot be empty");
    if (index_common(ocs, ofs, sizes[n - 1])) return ORA_E_ARG;
    ora_chunk_index* x = calloc(1, sizeof *x);
    x->is_variable = 1; x->original_chunk_size = ocs; x->original_file_size = ofs;
    x->final_transformed_chunk_size = sizes[n - 1]; x->chunk_count = n;
    x->transformed_chunks = malloc(sizeof(int32_t) * n);
    memcpy(x->transformed_chunks, sizes, sizeof(int32_t) * n);
    *out = x;
    return ORA_OK;
}
void ora_index_free(ora_chunk_index* x) { if (x) { free(x->transformed_chunks); free(x); } }
static int32_t osz(const ora_chunk_index* x, int32_t i) {
    return i == x->chunk_count - 1 ? x->original_file_size - (x->chunk_count - 1) * x->original_chunk_size
                                   : x->original_chunk_size;
}
static int32_t tsz(const ora_chunk_index* x, int32_t i) {
    if (x->is_variable) return x->transformed_chunks[i];
    return i == x->chunk_count - 1 ? x->final_transformed_chunk_size : x->transformed_chunk_size;
}
int32_t ora_index_materialized_count(const ora_chunk_index* x) { return x->chunk_count == 0 ? 1 : x->chunk_count; }
/* AbstractChunkIndex.materializeChunks :52-72 */
int ora_index_chunks(const ora_chunk_index* x, ora_chunk* out) {
    if (x->chunk_count == 0) { memset(out, 0, sizeof *out); return 1; }
    int32_t op = 0, tp = 0;
    for (int32_t i = 0; i < x->chunk_count; i++) {
        out[i] = (ora_chunk){ i, op, osz(x, i), tp, tsz(x, i) };
        op += out[i].original_size; tp += out[i].transformed_size;
    }
    return x->chunk_count;
}
/* AbstractChunkIndex.findChunkForOriginalOffset :75-110 */
int ora_index_find(const ora_chunk_index* x, int32_t offset, ora_chunk* out) {
    if (offset < 0) return fail(ORA_E_ARG, "Offset must be non-negative, %d given", offset);
    if (offset >= x->original_file_size) return 0;
    int32_t i = 0, op = 0, tp = 0;
    for (; i < x->chunk_count; i++) {
        int64_t beyond = (int64_t)(i + 1) * x->original_chunk_size;
        if (offset < beyond) break;
        op += osz(x, i); tp += tsz(x, i);
    }
    *out = (ora_chunk){ i, op, osz(x, i), tp, tsz(x, i) };
    return 1;
}
/* AbstractChunkIndex.chunksForRange :113-123 (range inclusive, storage/core BytesRange) */
int ora_index_chunks_for_range(const ora_chunk_index* x, int32_t from, int32_t to, ora_chunk* out, int32_t cap) {
    int32_t n = 0;
    ora_chunk cur;
    for (int64_t i = from; i <= to && i < x->original_file_size; i += cur.original_size) {
        int rc = ora_index_find(x, (int32_t)i, &cur);
        if (rc <= 0) return rc < 0 ? rc : n;
        if (n >= cap) return fail(ORA_E_SHORT, "out too small");
        out[n++] = cur;
    }
    return n;
}

/* ------------------------------------------------------------------ base64 (java.util.Base64 basic, padded) */
static const char B64[] = "ABCDEFGHIJKLMNOPQRSTUVWXYZabcdefghijklmnopqrstuvwxyz0123456789+/";
int64_t ora_base64_encode(const uint8_t* in, size_t n, char* out, size_t cap) {
    size_t need = 4 * ((n + 2) / 3);
    if (cap < need + 1) return fail(ORA_E_SHORT, "base64 out too small");
    size_t o = 0;
    for (size_t i = 0; i < n; i += 3) {
        uint32_t v = in[i] << 16 | (i + 1 < n ? in[i + 1] << 8 : 0) | (i + 2 < n ? in[i + 2] : 0);
        out[o++] = B64[v >> 18]; out[o++] = B64[(v >> 12) & 63];
        out[o++] = i + 1 < n ? B64[(v >> 6) & 63] : '=';
        out[o++] = i + 2 < n ? B64[v & 63] : '=';
    }
    out[o] = 0;
    return (int64_t)o;
}
int64_t ora_base64_decode(const char* in, uint8_t* out, size_t cap) {
    size_t o = 0; uint32_t acc = 0; int bits = 0;
    for (; *in && *in != '='; in++) {
        const char* p = strchr(B64, *in);
        if (!p) return fail(ORA_E_CORRUPT, "Illegal base64 character %x", *in);
        acc = acc << 6 | (uint32_t)(p - B64); bits += 6;
        if (bits >= 8) { bits -= 8; if (o >= cap) return fail(ORA_E_SHORT, "base64 out too small"); out[o++] = (uint8_t)(acc >> bits); }
    }
    return (int64_t)o;
}

/* ------------------------------------------------------------------ ChunkSizesBinaryCodec
 * core/M/manifest/index/serde/ChunkSizesBinaryCodec.java:104-202 (all integers big-endian) */
static void be32(uint8_t* p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }
static uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] << 24 | p[1] << 16 | p[2] << 8 | p[3]; }
static int bytes_needed(int32_t v) { return v <= 0xFF ? 1 : v <= 0xFFFF ? 2 : v <= 0xFFFFFF ? 3 : 4; }
int64_t ora_codec_encode(const int32_t* v, int32_t n, uint8_t* out, size_t cap) {
    if (n == 0) { if (cap < 4) return ORA_E_SHORT; be32(out, 0); return 4; }
    int32_t last = v[n - 1];
    if (n == 1) {
        if (last < 0) return fail(ORA_E_ARG, "Values cannot be negative");
        if (cap < 8) return ORA_E_SHORT;
        be32(out, 1); be32(out + 4, (uint32_t)last); return 8;
    }
    int32_t min = v[0];
    for (int32_t i = 1; i < n - 1; i++) if (v[i] < min) min = v[i];
    if (min < 0 || last < 0) return fail(ORA_E_ARG, "Values cannot be negative");
    int bpv = 1;
    for (int32_t i = 0; i < n - 1; i++) { int b = bytes_needed(v[i] - min); if (b > bpv) bpv = b; }
    size_t need = 4 + 4 + 1 + (size_t)(n - 1) * bpv + 4;
    if (cap < need) return fail(ORA_E_SHORT, "codec out too small");
    be32(out, (uint32_t)n); be32(out + 4, (uint32_t)min); out[8] = (uint8_t)bpv;
    uint8_t* p = out + 9;
    for (int32_t i = 0; i < n - 1; i++) {
        uint8_t t[4]; be32(t, (uint32_t)(v[i] - min));
        memcpy(p, t + 4 - bpv, bpv); p += bpv;
    }
    be32(p, (uint32_t)last);
    return (int64_t)need;
}
int32_t ora_codec_decode(const uint8_t* in, size_t n, int32_t* out, int32_t cap) {
    if (n < 4) return fail(ORA_E_CORRUPT, "codec buffer underflow");
    int32_t count = (int32_t)rd32(in);
    if (count == 0) return 0;
    if (count < 0 || count > cap) return fail(ORA_E_SHORT, "codec count %d", count);
    if (count == 1) { if (n < 8) return fail(ORA_E_CORRUPT, "codec buffer underflow"); out[0] = (int32_t)rd32(in + 4); return 1; }
    if (n < 9) return fail(ORA_E_CORRUPT, "codec buffer underflow");
    int32_t base = (int32_t)rd32(in + 4);
    int bpv = in[8];
    if (bpv < 1 || bpv > 4 || n < 9 + (size_t)(count - 1) * bpv + 4) return fail(ORA_E_CORRUPT, "codec buffer underflow");
    const uint8_t* p = in + 9;
    for (int32_t i = 0; i < count - 1; i++) {
        uint32_t x = 0;
        for (int k = 0; k < bpv; k++) x = x << 8 | *p++;
        out[i] = (int32_t)x + base;
    }
    out[count - 1] = (int32_t)rd32(p);
    return count;
}
/* TransformedChunksSerializer.serialize :30-52 = Base64(zstd(contentSize=true)(codec)) */
int64_t ora_transformed_chunks_serialize(const int32_t* v, int32_t n, char* out, size_t cap) {
    size_t raw_cap = 16 + (size_t)(n > 0 ? n : 0) * 4;
    uint8_t* raw = malloc(raw_cap);
    int64_t rl = ora_codec_encode(v, n, raw, raw_cap);
    if (rl < 0) { free(raw); return rl; }
    if (zload()) { free(raw); return ORA_E_NOLIB; }
    size_t zb = Z.compressBound((size_t)rl);
    uint8_t* z = malloc(zb);
    ZSTD_CCtx* c = Z.createCCtx();
    Z.setParameter(c, ZSTD_c_contentSizeFlag, 1);      /* serializer does not pledge the size */
    size_t zl = Z.compress2(c, z, zb, raw, (size_t)rl);
    Z.freeCCtx(c);
    free(raw);
    if (Z.isError(zl)) { free(z); return fail(ORA_E_SHORT, "zstd: %s", Z.getErrorName(zl)); }
    int64_t r = ora_base64_encode(z, zl, out, cap);
    free(z);
    return r;
}
/* TransformedChunksDeserializer.deserialize :36-49 (10 MiB sanity cap :33,42) */
int32_t ora_transformed_chunks_deserialize(const char* b64, int32_t* out, int32_t cap) {
    size_t bl = strlen(b64);
    uint8_t* z = malloc(bl + 4);
    int64_t zl = ora_base64_decode(b64, z, bl + 4);
    if (zl < 0) { free(z); return (int32_t)zl; }
    int64_t sz = ora_zstd_content_size(z, (size_t)zl);
    if (sz < 0 || sz > 10 * 1024 * 1024) { free(z); return fail(ORA_E_CORRUPT, "Invalid decompressed size: %lld", (long long)sz); }
    uint8_t* raw = malloc((size_t)sz + 1);
    int64_t rl = ora_zstd_decompress_chunk(z, (size_t)zl, raw, (size_t)sz);
    free(z);
    if (rl < 0) { free(raw); return (int32_t)rl; }
    int32_t n = ora_codec_decode(raw, (size_t)rl, out, cap);
    free(raw);
    return n;
}
/* Jackson output: ChunkIndex.java:36-42 type tag first, then AbstractChunkIndex props, then subclass props */
int ora_index_to_json(const ora_chunk_index* x, char* out, size_t cap) {
    int n;
    if (!x->is_variable) {
        n = snprintf(out, cap, "{\"type\":\"fixed\",\"originalChunkSize\":%d,\"originalFileSize\":%d,"
                               "\"transformedChunkSize\":%d,\"finalTransformedChunkSize\":%d}",
                     x->original_chunk_size, x->original_file_size, x->transformed_chunk_size,
                     x->final_transformed_chunk_size);
    } else {
        size_t bcap = 64 + (size_t)x->chunk_count * 8;
        char* b = malloc(bcap);
        int64_t bl = ora_transformed_chunks_serialize(x->transformed_chunks, x->chunk_count, b, bcap);
        if (bl < 0) { free(b); return (int)bl; }
        n = snprintf(out, cap, "{\"type\":\"variable\",\"originalChunkSize\":%d,\"originalFileSize\":%d,"
                               "\"transformedChunks\":\"%s\"}",
                     x->original_chunk_size, x->original_file_size, b);
        free(b);
    }
    if (n < 0 || (size_t)n >= cap) return fail(ORA_E_SHORT, "json out too small");
    return n;
}

/* ------------------------------------------------------------------ FetchChunkEnumeration range plan
 * core/M/fetch/FetchChunkEnumeration.java:54-92 (first/last chunk), :100-138 (skip on first, bound on last) */
int ora_fetch_plan(const ora_chunk_index* x, int32_t from, int32_t to, ora_fetch_piece* out, int32_t cap) {
    if (to < from) return fail(ORA_E_ARG, "range cannot be empty");
    ora_chunk first, last;
    int rc = ora_index_find(x, from, &first);
    if (rc < 0) return rc;
    if (rc == 0) return fail(ORA_E_ARG, "Invalid start position %d in segment path", from);
    rc = ora_index_find(x, to, &last);
    if (rc < 0) return rc;
    if (rc == 0) {              /* beyond EOF: the final chunk */
        int32_t cnt = ora_index_materialized_count(x);
        ora_chunk* all = malloc(sizeof(ora_chunk) * cnt);
        ora_index_chunks(x, all);
        last = all[cnt - 1];
        free(all);
    }
    int32_t n = 0;
    int32_t cnt = ora_index_materialized_count(x);
    ora_chunk* all = malloc(sizeof(ora_chunk) * cnt);
    ora_index_chunks(x, all);
    for (int32_t id = first.id; id <= last.id; id++) {
        if (n >= cap) { free(all); return fail(ORA_E_SHORT, "out too small"); }
        int32_t start = all[id].original_position, size = all[id].original_size;
        int32_t skip = 0, take = size;
        int at_first = id == first.id, at_last = id == last.id;
        if (at_first && at_last) {           /* single chunk: skip then bound to range.size() */
            skip = from - start;
            int32_t want = to - from + 1;
            take = size - skip < want ? size - skip : want;
        } else {
            if (at_first) { skip = from - start; take = size - skip; }
            if (at_last) { int32_t bound = to - start + 1; take = size < bound ? size : bound; }
        }
        out[n++] = (ora_fetch_piece){ id, skip, take };
    }
    free(all);
    return n;
}
