// aesgcm.cuh — batched AES-256-GCM for sm_90a (kernels K3/K4 of SURVEY.md §2a).
//
// Replaces, per chunk, javax.crypto Cipher("AES/GCM/NoPadding").doFinal as called from
//   core/M/transform/EncryptionChunkEnumeration.java:65-80   (layout IV(12) || CT || TAG(16))
//   core/M/transform/DecryptionChunkEnumeration.java:53-62   (IV = first 12 bytes; tag verified)
// with the cipher parameters of core/M/security/AesEncryptionProvider.java:36-98 (AES-256 key, 12-byte IV,
// 128-bit tag, per-segment AAD).  Algorithm: NIST SP 800-38D.
//
// Decomposition (one launch handles a whole batch of chunks):
//   gcm_key_setup_kernel   once per key: H = E_K(0), H^1..H^512, H^(2^k), and the 64 KiB Shoup table of H^512
//   gcm_main_kernel        grid (ranges, chunks); each CTA takes a 256 KiB range of one chunk: 512 threads
//                          stride through its 16-byte blocks (coalesced 128-bit loads/stores), AES-CTR via a
//                          bank-conflict-free Te0/Te2 tables replicated per lane in shared memory, GHASH as a
//                          512-way interleaved Horner scheme whose fixed multiplier H^512 is the TMA-staged
//                          shared-memory table; emits one 16-byte partial per range
//   gcm_finalize_kernel    one warp per chunk: combines the range partials with H-powers, adds AAD and the
//                          length block, computes/verifies the tag, writes IV and TAG, sizes and status
//   gcm_rekey_kernel       the main kernel's grid over IV||CT||TAG chunks, re-encrypted in place under a second key: per block
//                          ct_new = ct_old ^ E_old(ctr) ^ E_new(ctr), ct_old folded into the old GHASH and ct_new into the new
//                          one (one H^256 table per key in shared memory); two partials per range
//   gcm_rekey_finalize_kernel  one warp per chunk: checks the old tag, writes the new IV and tag and the status
// Integer/byte arithmetic only; no tensor cores (nothing here is a dense contraction).
#pragma once
#include "ts_common.cuh"
#include "aes_tables.h"

namespace ts {

constexpr int GH_T = 512;                        // GHASH interleave = threads per CTA of gcm_main_kernel
constexpr uint32_t GH_RANGE_BLOCKS = 16384;      // 16-byte blocks per CTA range (256 KiB)
constexpr int GH_NSQ = 28;                       // H^(2^k), k < 28  (chunk.size < 2^30 => m+1 < 2^27)
constexpr uint32_t GCM_IV = 12, GCM_TAG = 16;
// Round tables: one 256-byte row per S-box input; words 0-31 = Te0[x] replicated per lane, words 32-63 = Te2[x]
// (= Te0 rotated by 16 bits) replicated per lane.  Lane l only ever touches banks l (conflict-free), and the row
// stride of 256 bytes lets ONE PRMT build the shared-memory offset (state byte -> bits 8-15, lane offset -> bits 0-7).
constexpr uint32_t GCM_SMEM_TE = 256 * 64 * 4;   // 64 KiB
constexpr uint32_t GCM_SMEM_HTAB = 16 * 256 * 16;  // 64 KiB
constexpr uint32_t GCM_SMEM_BYTES = GCM_SMEM_TE + GCM_SMEM_HTAB;
constexpr uint32_t GCM_REKEY_SMEM_BYTES = GCM_SMEM_TE + 2 * GCM_SMEM_HTAB;   // 192 KiB: one CTA per SM, as gcm_main_kernel

struct GcmKeyCtx {
    uint4 hsq[GH_NSQ];            // hsq[k] = H^(2^k)
    uint4 hpow[GH_T + 1];         // hpow[e] = H^e, hpow[0] = 1
    uint4 htab[16 * 256];         // htab[j*256+b] = (byte j = b, rest 0) * H^256
};

__constant__ AesTables g_aes_tables = make_aes_tables();

// ------------------------------------------------------------------------------------------ GF(2^128)
// Elements are kept as the 16 bytes of SP 800-38D in memory order (uint4 of little-endian words) so XOR and
// byte extraction need no conversion; the bitwise multiply works on the big-endian (hi, lo) view.
struct gf128 { uint64_t hi, lo; };
__device__ __forceinline__ gf128 gf_from_le(uint4 v) {
    gf128 r;
    r.hi = ((uint64_t)bswap32(v.x) << 32) | bswap32(v.y);
    r.lo = ((uint64_t)bswap32(v.z) << 32) | bswap32(v.w);
    return r;
}
__device__ __forceinline__ uint4 gf_to_le(gf128 g) {
    return make_uint4(bswap32((uint32_t)(g.hi >> 32)), bswap32((uint32_t)g.hi),
                      bswap32((uint32_t)(g.lo >> 32)), bswap32((uint32_t)g.lo));
}
__device__ __forceinline__ gf128 gf_mulx(gf128 v) {      // v * x  (SP 800-38D: V >> 1, conditional R)
    uint64_t lsb = v.lo & 1;
    v.lo = (v.lo >> 1) | (v.hi << 63);
    v.hi >>= 1;
    if (lsb) v.hi ^= 0xe100000000000000ull;
    return v;
}
__device__ TS_NOINLINE uint4 gf_mul(uint4 a, uint4 b) {   // generic product, used O(1) times per CTA/chunk
    gf128 x = gf_from_le(a), v = gf_from_le(b), z;
    z.hi = 0; z.lo = 0;
    for (int i = 0; i < 128; i++) {
        uint64_t bit = i < 64 ? (x.hi >> (63 - i)) & 1 : (x.lo >> (127 - i)) & 1;
        if (bit) { z.hi ^= v.hi; z.lo ^= v.lo; }
        v = gf_mulx(v);
    }
    return gf_to_le(z);
}
__device__ __forceinline__ uint4 gf_one() { return make_uint4(0x80u, 0, 0, 0); }
// H^e from the squares table
__device__ __forceinline__ uint4 gf_pow(const GcmKeyCtx* kc, uint32_t e) {
    uint4 r = gf_one();
    bool have = false;
    for (int k = 0; k < GH_NSQ && (e >> k); k++) {
        if ((e >> k) & 1) {
            r = have ? gf_mul(r, kc->hsq[k]) : kc->hsq[k];
            have = true;
        }
    }
    return r;
}

// y * G through the Shoup byte table of G (16 lookups of 16 bytes, XOR-accumulated)
__device__ __forceinline__ uint4 gf_mul_tab(const uint4* __restrict__ tab, uint4 y) {
    uint4 z = make_uint4(0, 0, 0, 0);
    const uint32_t w[4] = { y.x, y.y, y.z, y.w };
#pragma unroll
    for (int j = 0; j < 16; j++) {
        uint32_t b = (w[j >> 2] >> (8 * (j & 3))) & 0xff;
        uint4 e = tab[j * 256 + b];
        z.x ^= e.x; z.y ^= e.y; z.z ^= e.z; z.w ^= e.w;
    }
    return z;
}

// ------------------------------------------------------------------------------------------ AES-256
// One block through the lane-replicated tables.  off0 = 4*lane selects the Te0 half of a row, off2 = 128 + 4*lane
// the Te2 half; SEL(k) makes PRMT produce (byte k of x) << 8 | lane offset, i.e. the byte offset of the lookup.
// Per column and round: 4 PRMT (addresses) + 4 LDS + 1 PRMT (one shared 8-bit rotation) + 3 XOR-class ops:
//   t = Te0[a] ^ Te1[b] ^ Te2[c] ^ Te3[d] ^ rk = Te0[a] ^ Te2[c] ^ rk ^ rotl8(Te0[b] ^ Te2[d]).
#define TS_SEL(k) (0x5504u | ((k) << 4))
#define TS_T0(x, k) (*(const uint32_t*)(te + __byte_perm((x), off0, TS_SEL(k))))
#define TS_T2(x, k) (*(const uint32_t*)(te + __byte_perm((x), off2, TS_SEL(k))))
__device__ __forceinline__ void aes256_encrypt_te(const Aes256RoundKeys& rk, const uint8_t* __restrict__ te, uint32_t off0, uint32_t off2,
                                                  uint32_t& s0, uint32_t& s1, uint32_t& s2, uint32_t& s3) {
    s0 ^= rk.w[0]; s1 ^= rk.w[1]; s2 ^= rk.w[2]; s3 ^= rk.w[3];
#pragma unroll
    for (int r = 1; r < 14; r++) {
        const uint32_t t0 = TS_T0(s0, 0u) ^ TS_T2(s2, 2u) ^ rk.w[4 * r]     ^ __byte_perm(TS_T0(s1, 1u) ^ TS_T2(s3, 3u), 0, 0x2103);
        const uint32_t t1 = TS_T0(s1, 0u) ^ TS_T2(s3, 2u) ^ rk.w[4 * r + 1] ^ __byte_perm(TS_T0(s2, 1u) ^ TS_T2(s0, 3u), 0, 0x2103);
        const uint32_t t2 = TS_T0(s2, 0u) ^ TS_T2(s0, 2u) ^ rk.w[4 * r + 2] ^ __byte_perm(TS_T0(s3, 1u) ^ TS_T2(s1, 3u), 0, 0x2103);
        const uint32_t t3 = TS_T0(s3, 0u) ^ TS_T2(s1, 2u) ^ rk.w[4 * r + 3] ^ __byte_perm(TS_T0(s0, 1u) ^ TS_T2(s2, 3u), 0, 0x2103);
        s0 = t0; s1 = t1; s2 = t2; s3 = t3;
    }
    // final round: SubBytes + ShiftRows only; S[x] is byte 1 of Te0[x]
    const uint32_t a0 = TS_T0(s0, 0u), a1 = TS_T0(s1, 1u), a2 = TS_T0(s2, 2u), a3 = TS_T0(s3, 3u);
    const uint32_t b0 = TS_T0(s1, 0u), b1 = TS_T0(s2, 1u), b2 = TS_T0(s3, 2u), b3 = TS_T0(s0, 3u);
    const uint32_t c0 = TS_T0(s2, 0u), c1 = TS_T0(s3, 1u), c2 = TS_T0(s0, 2u), c3 = TS_T0(s1, 3u);
    const uint32_t d0 = TS_T0(s3, 0u), d1 = TS_T0(s0, 1u), d2 = TS_T0(s1, 2u), d3 = TS_T0(s2, 3u);
    // byte k of the result = byte 1 of the k-th lookup
    s0 = __byte_perm(__byte_perm(a0, a1, 0x0051), __byte_perm(a2, a3, 0x0051), 0x5410) ^ rk.w[56];
    s1 = __byte_perm(__byte_perm(b0, b1, 0x0051), __byte_perm(b2, b3, 0x0051), 0x5410) ^ rk.w[57];
    s2 = __byte_perm(__byte_perm(c0, c1, 0x0051), __byte_perm(c2, c3, 0x0051), 0x5410) ^ rk.w[58];
    s3 = __byte_perm(__byte_perm(d0, d1, 0x0051), __byte_perm(d2, d3, 0x0051), 0x5410) ^ rk.w[59];
}
#undef TS_T0
#undef TS_T2
#undef TS_SEL

// Byte-oriented AES for the O(1)-per-chunk blocks (H = E_K(0), E_K(J0)); constant-memory S-box.
__device__ TS_NOINLINE uint4 aes256_encrypt_slow(const Aes256RoundKeys& rk, uint4 in) {
    uint8_t s[16], t[16];
    uint32_t w[4] = { in.x ^ rk.w[0], in.y ^ rk.w[1], in.z ^ rk.w[2], in.w ^ rk.w[3] };
    for (int i = 0; i < 16; i++) s[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
    for (int r = 1; r <= 14; r++) {
        for (int c = 0; c < 4; c++)
            for (int row = 0; row < 4; row++) t[4 * c + row] = g_aes_tables.sbox[s[4 * ((c + row) & 3) + row]];
        if (r < 14) {
            for (int c = 0; c < 4; c++) {
                uint8_t a0 = t[4 * c], a1 = t[4 * c + 1], a2 = t[4 * c + 2], a3 = t[4 * c + 3];
                s[4 * c]     = (uint8_t)(aes_xtime(a0) ^ aes_xtime(a1) ^ a1 ^ a2 ^ a3);
                s[4 * c + 1] = (uint8_t)(a0 ^ aes_xtime(a1) ^ aes_xtime(a2) ^ a2 ^ a3);
                s[4 * c + 2] = (uint8_t)(a0 ^ a1 ^ aes_xtime(a2) ^ aes_xtime(a3) ^ a3);
                s[4 * c + 3] = (uint8_t)(aes_xtime(a0) ^ a0 ^ a1 ^ a2 ^ aes_xtime(a3));
            }
        } else {
            for (int i = 0; i < 16; i++) s[i] = t[i];
        }
        for (int i = 0; i < 16; i++) s[i] ^= (uint8_t)(rk.w[4 * r + (i >> 2)] >> (8 * (i & 3)));
    }
    uint32_t o[4] = {0, 0, 0, 0};
    for (int i = 0; i < 16; i++) o[i >> 2] |= (uint32_t)s[i] << (8 * (i & 3));
    return make_uint4(o[0], o[1], o[2], o[3]);
}

// ------------------------------------------------------------------------------------------ key set-up
__global__ void __launch_bounds__(GH_T) gcm_key_setup_kernel(const __grid_constant__ Aes256RoundKeys rk, GcmKeyCtx* kc) {
    __shared__ uint4 V[128];
    const int t = threadIdx.x;
    if (t == 0) {
        uint4 H = aes256_encrypt_slow(rk, make_uint4(0, 0, 0, 0));
        kc->hpow[0] = gf_one();
        kc->hpow[1] = H;
    }
    __syncthreads();
    for (int s = 1; s < GH_T; s <<= 1) {             // log-doubling: H^(s+t+1) = H^(t+1) * H^s
        if (t < s && s + t + 1 <= GH_T) kc->hpow[s + t + 1] = gf_mul(kc->hpow[t + 1], kc->hpow[s]);
        __threadfence_block();
        __syncthreads();
    }
    if (t == 0) {
        gf128 v = gf_from_le(kc->hpow[GH_T]);         // basis x^i * H^256
        for (int i = 0; i < 128; i++) { V[i] = gf_to_le(v); v = gf_mulx(v); }
    } else if (t == 32) {
        uint4 q = kc->hpow[1];
        kc->hsq[0] = q;
        for (int k = 1; k < GH_NSQ; k++) { q = gf_mul(q, q); kc->hsq[k] = q; }
    }
    __syncthreads();
    for (int idx = t; idx < 16 * 256; idx += blockDim.x) {
        int j = idx >> 8, b = idx & 255;
        uint4 e = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int k = 0; k < 8; k++)
            if (b & (0x80 >> k)) e = xor4(e, V[8 * j + k]);
        kc->htab[idx] = e;
    }
}

// ------------------------------------------------------------------------------------------ batch descriptors
struct GcmBatch {
    const uint8_t* in_base;  const uint64_t* in_off;  const uint32_t* in_len;   // ENC: plaintext; DEC: IV||CT||TAG
    uint8_t* out_base;       const uint64_t* out_off; uint32_t* out_len;        // ENC: IV||CT||TAG; DEC: plaintext
    const uint8_t* ivs;          // ENC only: 12 bytes per chunk
    const uint8_t* aad; uint32_t aad_len;
    uint4* partials; uint32_t max_ranges;
    uint32_t* status;            // DEC: 0 ok, 1 tag mismatch / malformed
    uint32_t n_chunks;
    uint32_t out_cap;            // DEC: plaintext bytes the destination holds per chunk; a longer chunk is rejected
                                 //      (status 1) BEFORE anything is written — sizes may come from a tampered manifest
};

__device__ __forceinline__ uint32_t ld_le32_bytes(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// ------------------------------------------------------------------------------------------ shared kernel pieces
// gcm_main_kernel / gcm_finalize_kernel and the rekey kernels share these pieces as macros, not functions: the compiler optimizes
// a function on its own before it inlines it, which reorders the instructions of its callers.  As text the pieces leave
// gcm_main_kernel and gcm_finalize_kernel compiling to the SASS they had before the rekey kernels shared them.

// The lane-replicated round tables into the first GCM_SMEM_TE bytes of shared memory.
#define GCM_FILL_TE(smem, tid)                                                                                                 \
    for (uint32_t i = tid; i < 256 * 64; i += GH_T) {                                                                          \
        const uint32_t t0 = g_aes_tables.te0[i >> 6];                                                                          \
        ((uint32_t*)smem)[i] = (i & 32) ? __byte_perm(t0, 0, 0x1032) : t0;       /* second half of a row: Te2 = rotl16(Te0) */ \
    }

// Block `off` (a multiple of 16) of an n-byte run: declares d = its bytes at src + off, the pad zeroed (one 128-bit load when the
// run is aligned and the block full), and o = d ^ (k0, k1, k2, k3), stored at dst + off (only the bytes inside the run) and left
// with its pad zeroed, as GHASH takes it.
#define GCM_XOR_BLOCK(src, dst, off, n, aligned, full, k0, k1, k2, k3, d, o)                                                   \
    uint4 d;                                                                                                                   \
    if (aligned && full) {                                                                                                     \
        d = ldg128_stream((const uint4*)(src + off));                                                                          \
    } else {                                                                                                                   \
        uint32_t w[4] = {0, 0, 0, 0};                                                                                          \
        uint32_t k = full ? 16 : n - (uint32_t)off;                                                                            \
        for (uint32_t q = 0; q < k; q++) w[q >> 2] |= (uint32_t)src[off + q] << (8 * (q & 3));                                 \
        d = make_uint4(w[0], w[1], w[2], w[3]);                                                                                \
    }                                                                                                                          \
    uint4 o = make_uint4(d.x ^ k0, d.y ^ k1, d.z ^ k2, d.w ^ k3);                                                              \
    if (aligned && full) {                                                                                                     \
        stg128_stream((uint4*)(dst + off), o);                                                                                 \
    } else {                                                                                                                   \
        uint32_t w[4] = { o.x, o.y, o.z, o.w };                                                                                \
        uint32_t k = full ? 16 : n - (uint32_t)off;                                                                            \
        for (uint32_t q = 0; q < k; q++) dst[off + q] = (uint8_t)(w[q >> 2] >> (8 * (q & 3)));                                 \
        if (!full) {                                  /* zero the pad bytes of the ciphertext block for GHASH */               \
            for (uint32_t q = k; q < 16; q++) w[q >> 2] &= ~(0xffu << (8 * (q & 3)));                                          \
            o = make_uint4(w[0], w[1], w[2], w[3]);                                                                            \
        }                                                                                                                      \
    }

// A lane's GHASH accumulator `acc` (last block `last`, 0xffffffff if none) aligned to the range end b1 and XOR-reduced over the
// CTA through `red` (GH_T / 32 entries, one __syncthreads); thread 0 stores the range's partial to `partial`.
#define GCM_RANGE_PARTIAL(kc, acc, last, b1, red, tid, partial)                                                                \
    if (last != 0xffffffffu) acc = gf_mul(acc, kc->hpow[b1 - last]);   /* align the lane to the range end */                   \
                                                                                                                               \
    /* XOR-reduce the 256 lanes */                                                                                             \
    for (int o = 16; o; o >>= 1) {                                                                                             \
        acc.x ^= __shfl_xor_sync(TS_FULL, acc.x, o); acc.y ^= __shfl_xor_sync(TS_FULL, acc.y, o);                              \
        acc.z ^= __shfl_xor_sync(TS_FULL, acc.z, o); acc.w ^= __shfl_xor_sync(TS_FULL, acc.w, o);                              \
    }                                                                                                                          \
    if ((tid & 31) == 0) red[tid >> 5] = acc;                                                                                  \
    __syncthreads();                                                                                                           \
    if (tid == 0) {                                                                                                            \
        uint4 p = red[0];                                                                                                      \
        for (int w = 1; w < GH_T / 32; w++) p = xor4(p, red[w]);                                                               \
        partial = p;                                                                                                           \
    }

// Declares `term`: the GHASH of an m-block chunk before its length block, summed over the warp -- its nr range partials
// P_r * H^(m - end_r) (at partials[chunk * max_ranges + r]) and the AAD's X_A * H^(m+1).
#define GCM_HASH_TERMS(kc, partials, max_ranges, chunk, m, nr, aad, aad_len, lane, term)                                       \
    uint4 term = make_uint4(0, 0, 0, 0);                                                                                       \
    for (uint32_t r = lane; r < nr; r += 32) {             /* P_r * H^(m - end_r) */                                           \
        uint32_t end_r = min((r + 1) * GH_RANGE_BLOCKS, m);                                                                    \
        uint4 p = partials[(size_t)chunk * max_ranges + r];                                                                    \
        uint32_t e = m - end_r;                                                                                                \
        term = xor4(term, e ? gf_mul(p, gf_pow(kc, e)) : p);                                                                   \
    }                                                                                                                          \
    if (lane == 31 && aad_len) {                           /* X_A * H^(m+1) */                                                 \
        uint4 x = make_uint4(0, 0, 0, 0);                                                                                      \
        const uint4 H = kc->hpow[1];                                                                                           \
        for (uint32_t off = 0; off < aad_len; off += 16) {                                                                     \
            uint32_t w[4] = {0, 0, 0, 0};                                                                                      \
            uint32_t k = min(16u, aad_len - off);                                                                              \
            for (uint32_t q = 0; q < k; q++) w[q >> 2] |= (uint32_t)aad[off + q] << (8 * (q & 3));                             \
            x = off ? gf_mul(x, H) : x;                                                                                        \
            x = xor4(x, make_uint4(w[0], w[1], w[2], w[3]));                                                                   \
        }                                                                                                                      \
        term = xor4(term, gf_mul(x, gf_pow(kc, m + 1)));                                                                       \
    }                                                                                                                          \
    for (int o = 16; o; o >>= 1) {                                                                                             \
        term.x ^= __shfl_xor_sync(TS_FULL, term.x, o); term.y ^= __shfl_xor_sync(TS_FULL, term.y, o);                          \
        term.z ^= __shfl_xor_sync(TS_FULL, term.z, o); term.w ^= __shfl_xor_sync(TS_FULL, term.w, o);                          \
    }

// Declares S = (term ^ length block) * H for an n-byte ciphertext: the tag is S ^ E_K(J0).
#define GCM_TAG_S(kc, term, aad_len, n, S)                                                                                     \
    const uint64_t abits = (uint64_t)aad_len * 8, cbits = (uint64_t)n * 8;                                                     \
    uint4 L = make_uint4(bswap32((uint32_t)(abits >> 32)), bswap32((uint32_t)abits),                                           \
                         bswap32((uint32_t)(cbits >> 32)), bswap32((uint32_t)cbits));                                          \
    uint4 S = gf_mul(xor4(term, L), kc->hpow[1]);

// ------------------------------------------------------------------------------------------ main kernel
template <bool ENC>
__global__ void __launch_bounds__(GH_T, 1)
gcm_main_kernel(const __grid_constant__ Aes256RoundKeys rk, const GcmKeyCtx* __restrict__ kc,
                const __grid_constant__ GcmBatch B) {
    TS_DYN_SMEM(smem);
    __shared__ uint4 red[GH_T / 32];
#if TS_DEVICE_ASM
    __shared__ __align__(8) uint64_t bar;
#else
    uint64_t bar_dummy = 0; uint64_t* barp = &bar_dummy;
#endif
    const uint8_t* te = smem;
    uint4* htab = (uint4*)(smem + GCM_SMEM_TE);

    const uint32_t chunk = blockIdx.y, range = blockIdx.x, tid = threadIdx.x;
    const uint32_t len = B.in_len[chunk];
    const uint32_t n = ENC ? len : (len >= GCM_IV + GCM_TAG ? len - (GCM_IV + GCM_TAG) : 0);
    const uint32_t m = (n + 15) >> 4;
    const uint32_t b0 = range * GH_RANGE_BLOCKS;
    if (b0 >= m) return;                                   // uniform for the CTA
    if (!ENC && n > B.out_cap) return;                     // oversize chunk: finalize reports it, nothing is written
    const uint32_t b1 = min(b0 + GH_RANGE_BLOCKS, m);

#if TS_DEVICE_ASM
    if (tid == 0) mbar_init(&bar, 1);
    uint64_t* barp = &bar;
#endif
    GCM_FILL_TE(smem, tid)
    __syncthreads();
    block_bulk_load(htab, kc->htab, GCM_SMEM_HTAB, barp, 0);   // TMA bulk copy of the H^256 table
    __syncthreads();

    const uint8_t* in = B.in_base + B.in_off[chunk];
    uint8_t* out = B.out_base + B.out_off[chunk];
    const uint8_t* ivp = ENC ? B.ivs + (size_t)chunk * GCM_IV : in;
    const uint8_t* src = ENC ? in : in + GCM_IV;
    uint8_t* dst = ENC ? out + GCM_IV : out;
    const uint32_t iv0 = ld_le32_bytes(ivp), iv1 = ld_le32_bytes(ivp + 4), iv2 = ld_le32_bytes(ivp + 8);
    const bool aligned = ((((uintptr_t)src) | ((uintptr_t)dst)) & 15) == 0;
    const uint32_t off0 = (tid & 31) * 4, off2 = 128 + off0;

    uint4 acc = make_uint4(0, 0, 0, 0);
    uint32_t last = 0xffffffffu;
    for (uint32_t i = b0 + tid; i < b1; i += GH_T) {
        uint32_t s0 = iv0, s1 = iv1, s2 = iv2, s3 = bswap32(i + 2);
        aes256_encrypt_te(rk, te, off0, off2, s0, s1, s2, s3);
        const size_t off = (size_t)i << 4;
        const bool full = off + 16 <= n;
        GCM_XOR_BLOCK(src, dst, off, n, aligned, full, s0, s1, s2, s3, d, o)
        const uint4 ct = ENC ? o : d;                     // (DEC: d was zero padded on load)
        acc = xor4(gf_mul_tab(htab, acc), ct);
        last = i;
    }
    GCM_RANGE_PARTIAL(kc, acc, last, b1, red, tid, B.partials[(size_t)chunk * B.max_ranges + range])
}

// ------------------------------------------------------------------------------------------ finalize
template <bool ENC>
__global__ void __launch_bounds__(128)
gcm_finalize_kernel(const __grid_constant__ Aes256RoundKeys rk, const GcmKeyCtx* __restrict__ kc,
                    const __grid_constant__ GcmBatch B) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t chunk = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (chunk >= B.n_chunks) return;                       // whole warp leaves together
    const uint32_t len = B.in_len[chunk];
    const bool malformed = !ENC && (len < GCM_IV + GCM_TAG || len - (GCM_IV + GCM_TAG) > B.out_cap);
    const uint32_t n = ENC ? len : (malformed ? 0 : len - (GCM_IV + GCM_TAG));
    const uint32_t m = (n + 15) >> 4;
    const uint32_t nr = (m + GH_RANGE_BLOCKS - 1) / GH_RANGE_BLOCKS;
    const uint8_t* in = B.in_base + B.in_off[chunk];
    uint8_t* out = B.out_base + B.out_off[chunk];

    GCM_HASH_TERMS(kc, B.partials, B.max_ranges, chunk, m, nr, B.aad, B.aad_len, lane, term)
    if (lane == 0) {
        GCM_TAG_S(kc, term, B.aad_len, n, S)
        const uint8_t* ivp = ENC ? B.ivs + (size_t)chunk * GCM_IV : in;
        uint4 j0 = make_uint4(0, 0, 0, 0x01000000u);
        if (!malformed) { j0.x = ld_le32_bytes(ivp); j0.y = ld_le32_bytes(ivp + 4); j0.z = ld_le32_bytes(ivp + 8); }
        uint4 tag = xor4(S, aes256_encrypt_slow(rk, j0));
        const uint32_t tw[4] = { tag.x, tag.y, tag.z, tag.w };
        if (ENC) {
            for (int q = 0; q < 12; q++) out[q] = ivp[q];
            for (int q = 0; q < 16; q++) out[GCM_IV + n + q] = (uint8_t)(tw[q >> 2] >> (8 * (q & 3)));
            B.out_len[chunk] = n + GCM_IV + GCM_TAG;
        } else {
            uint32_t diff = malformed ? 1u : 0u;
            if (!malformed)
                for (int q = 0; q < 16; q++) diff |= (uint32_t)(in[GCM_IV + n + q] ^ (uint8_t)(tw[q >> 2] >> (8 * (q & 3))));
            B.status[chunk] = diff ? 1u : 0u;
            B.out_len[chunk] = n;
        }
    }
}

// ------------------------------------------------------------------------------------------ re-encryption under a new key
// tsgpu_rekey_object: IV || CT || TAG chunks re-encrypted in place, the plaintext only in registers.  A chunk keeps its size.
struct GcmRekeyBatch {
    uint8_t* base; const uint64_t* off; const uint32_t* len;   // chunk i: len[i] bytes at base + off[i], 16 + off[i] 16-byte aligned
    const uint8_t* ivs;              // the new IVs, 12 bytes per chunk
    const uint8_t* aad_old; uint32_t aad_old_len;
    const uint8_t* aad_new; uint32_t aad_new_len;
    uint4* partials_old; uint4* partials_new; uint32_t max_ranges;   // [chunk * max_ranges + range]
    uint32_t* status;                // 0 ok or empty; 1 old tag mismatch, or a chunk of 1 to 27 bytes
    uint32_t n_chunks;
};

__global__ void __launch_bounds__(GH_T, 1)
gcm_rekey_kernel(const __grid_constant__ Aes256RoundKeys rk_old, const GcmKeyCtx* __restrict__ kc_old,
                 const __grid_constant__ Aes256RoundKeys rk_new, const GcmKeyCtx* __restrict__ kc_new,
                 const __grid_constant__ GcmRekeyBatch B) {
    TS_DYN_SMEM(smem);
    __shared__ uint4 red_old[GH_T / 32], red_new[GH_T / 32];
#if TS_DEVICE_ASM
    __shared__ __align__(8) uint64_t bar;
#else
    uint64_t bar_dummy = 0; uint64_t* barp = &bar_dummy;
#endif
    const uint8_t* te = smem;
    uint4* htab_old = (uint4*)(smem + GCM_SMEM_TE);
    uint4* htab_new = (uint4*)(smem + GCM_SMEM_TE + GCM_SMEM_HTAB);

    const uint32_t chunk = blockIdx.y, range = blockIdx.x, tid = threadIdx.x;
    const uint32_t len = B.len[chunk];
    const uint32_t n = len >= GCM_IV + GCM_TAG ? len - (GCM_IV + GCM_TAG) : 0;
    const uint32_t m = (n + 15) >> 4;
    const uint32_t b0 = range * GH_RANGE_BLOCKS;
    if (b0 >= m) return;                                   // uniform for the CTA
    const uint32_t b1 = min(b0 + GH_RANGE_BLOCKS, m);

#if TS_DEVICE_ASM
    if (tid == 0) mbar_init(&bar, 1);
    uint64_t* barp = &bar;
#endif
    GCM_FILL_TE(smem, tid)
    __syncthreads();
    block_bulk_load(htab_old, kc_old->htab, GCM_SMEM_HTAB, barp, 0);
    __syncthreads();             // every thread has seen phase 0 complete before phase 1 starts: parity 0 cannot come round again
    block_bulk_load(htab_new, kc_new->htab, GCM_SMEM_HTAB, barp, 1);
    __syncthreads();

    uint8_t* chunk_p = B.base + B.off[chunk];
    uint8_t* ct = chunk_p + GCM_IV;
    const uint8_t* ivn = B.ivs + (size_t)chunk * GCM_IV;
    const uint32_t iv0 = ld_le32_bytes(chunk_p), iv1 = ld_le32_bytes(chunk_p + 4), iv2 = ld_le32_bytes(chunk_p + 8);
    const uint32_t jv0 = ld_le32_bytes(ivn), jv1 = ld_le32_bytes(ivn + 4), jv2 = ld_le32_bytes(ivn + 8);
    const bool aligned = (((uintptr_t)ct) & 15) == 0;
    const uint32_t off0 = (tid & 31) * 4, off2 = 128 + off0;

    uint4 acc_old = make_uint4(0, 0, 0, 0), acc_new = make_uint4(0, 0, 0, 0);
    uint32_t last = 0xffffffffu;
    for (uint32_t i = b0 + tid; i < b1; i += GH_T) {
        uint32_t s0 = iv0, s1 = iv1, s2 = iv2, s3 = bswap32(i + 2);
        aes256_encrypt_te(rk_old, te, off0, off2, s0, s1, s2, s3);
        uint32_t t0 = jv0, t1 = jv1, t2 = jv2, t3 = bswap32(i + 2);
        aes256_encrypt_te(rk_new, te, off0, off2, t0, t1, t2, t3);
        const size_t off = (size_t)i << 4;
        const bool full = off + 16 <= n;
        GCM_XOR_BLOCK(ct, ct, off, n, aligned, full, (s0 ^ t0), (s1 ^ t1), (s2 ^ t2), (s3 ^ t3), d, o)   // d: ct_old, o: ct_new
        acc_old = xor4(gf_mul_tab(htab_old, acc_old), d);
        acc_new = xor4(gf_mul_tab(htab_new, acc_new), o);
        last = i;
    }
    { GCM_RANGE_PARTIAL(kc_old, acc_old, last, b1, red_old, tid, B.partials_old[(size_t)chunk * B.max_ranges + range]) }
    { GCM_RANGE_PARTIAL(kc_new, acc_new, last, b1, red_new, tid, B.partials_new[(size_t)chunk * B.max_ranges + range]) }
}

__global__ void __launch_bounds__(128)
gcm_rekey_finalize_kernel(const __grid_constant__ Aes256RoundKeys rk_old, const GcmKeyCtx* __restrict__ kc_old,
                          const __grid_constant__ Aes256RoundKeys rk_new, const GcmKeyCtx* __restrict__ kc_new,
                          const __grid_constant__ GcmRekeyBatch B) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t chunk = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (chunk >= B.n_chunks) return;                       // whole warp leaves together
    const uint32_t len = B.len[chunk];
    if (len < GCM_IV + GCM_TAG) {                          // an empty chunk passes through; a shorter one cannot hold IV and tag
        if (lane == 0) B.status[chunk] = len ? 1u : 0u;
        return;
    }
    const uint32_t n = len - (GCM_IV + GCM_TAG);
    const uint32_t m = (n + 15) >> 4;
    const uint32_t nr = (m + GH_RANGE_BLOCKS - 1) / GH_RANGE_BLOCKS;
    uint8_t* p = B.base + B.off[chunk];
    uint4 told = make_uint4(0, 0, 0, 0), tnew = told;      // lane 0: the old tag (recomputed) and the new one
    const uint8_t* ivn = B.ivs + (size_t)chunk * GCM_IV;
    {
        GCM_HASH_TERMS(kc_old, B.partials_old, B.max_ranges, chunk, m, nr, B.aad_old, B.aad_old_len, lane, term)
        if (lane == 0) {
            GCM_TAG_S(kc_old, term, B.aad_old_len, n, S)
            told = xor4(S, aes256_encrypt_slow(rk_old, make_uint4(ld_le32_bytes(p), ld_le32_bytes(p + 4), ld_le32_bytes(p + 8), 0x01000000u)));
        }
    }
    {
        GCM_HASH_TERMS(kc_new, B.partials_new, B.max_ranges, chunk, m, nr, B.aad_new, B.aad_new_len, lane, term)
        if (lane == 0) {
            GCM_TAG_S(kc_new, term, B.aad_new_len, n, S)
            tnew = xor4(S, aes256_encrypt_slow(rk_new, make_uint4(ld_le32_bytes(ivn), ld_le32_bytes(ivn + 4), ld_le32_bytes(ivn + 8), 0x01000000u)));
        }
    }
    if (lane == 0) {
        const uint32_t tw[4] = { told.x, told.y, told.z, told.w }, nw[4] = { tnew.x, tnew.y, tnew.z, tnew.w };
        uint32_t diff = 0;
        for (int q = 0; q < 16; q++) diff |= (uint32_t)(p[GCM_IV + n + q] ^ (uint8_t)(tw[q >> 2] >> (8 * (q & 3))));
        B.status[chunk] = diff ? 1u : 0u;
        for (int q = 0; q < 12; q++) p[q] = ivn[q];
        for (int q = 0; q < 16; q++) p[GCM_IV + n + q] = (uint8_t)(nw[q >> 2] >> (8 * (q & 3)));
    }
}

}  // namespace ts
