// crc32.cuh — GF(2) arithmetic of the reflected CRC-32 polynomials, shared by the record validation (records.cuh), the upload-part
// checksums (part_crc.cuh) and the host code that carries their state between batches and calls.
//
// A "raw" CRC is the register after the bytes with initial value 0 and no final xor.  It is linear:
//   raw(A || B) = raw(A) * x^(8|B|) mod P  ^  raw(B)          (crc_shift(raw(A), |B|) ^ raw(B))
//   crc(A)      = ~(raw(A) ^ crc_shift(0xFFFFFFFF, |A|))     (init and xorout 0xFFFFFFFF)
// so the CRC of a range is combined from the CRCs of its pieces, whichever thread or call hashed them.
#pragma once
#include "ts_common.cuh"

namespace ts {

constexpr uint32_t CRC32C_POLY = 0x82F63B78u;   // Castagnoli, reflected (index 0)
constexpr uint32_t CRC32_POLY = 0xEDB88320u;    // IEEE, reflected (index 1)
__host__ __device__ __forceinline__ uint32_t crc_poly(int pi) { return pi ? CRC32_POLY : CRC32C_POLY; }

// x^(2^k) mod P, k = 0..63, for the two reflected polynomials (shift of a CRC by n bytes: product over the bits of 8n)
#define TS_CRC_X2N_TABLE                                                                                                          \
    {{0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0x82f63b78u, 0x6ea2d55cu, 0x18b8ea18u, 0x510ac59au, 0xb82be955u, \
      0xb8fdb1e7u, 0x88e56f72u, 0x74c360a4u, 0xe4172b16u, 0x0d65762au, 0x35d73a62u, 0x28461564u, 0xbf455269u, 0xe2ea32dcu, 0xfe7740e6u, \
      0xf946610bu, 0x3c204f8fu, 0x538586e3u, 0x59726915u, 0x734d5309u, 0xbc1ac763u, 0x7d0722ccu, 0xd289cabeu, 0xe94ca9bcu, 0x05b74f3fu, \
      0xa51e1f42u, 0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0x82f63b78u, 0x6ea2d55cu, 0x18b8ea18u, 0x510ac59au, \
      0xb82be955u, 0xb8fdb1e7u, 0x88e56f72u, 0x74c360a4u, 0xe4172b16u, 0x0d65762au, 0x35d73a62u, 0x28461564u, 0xbf455269u, 0xe2ea32dcu, \
      0xfe7740e6u, 0xf946610bu, 0x3c204f8fu, 0x538586e3u, 0x59726915u, 0x734d5309u, 0xbc1ac763u, 0x7d0722ccu, 0xd289cabeu, 0xe94ca9bcu, \
      0x05b74f3fu, 0xa51e1f42u, 0x40000000u, 0x20000000u},                                                                            \
     {0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0xedb88320u, 0xb1e6b092u, 0xa06a2517u, 0xed627daeu, 0x88d14467u, \
      0xd7bbfe6au, 0xec447f11u, 0x8e7ea170u, 0x6427800eu, 0x4d47bae0u, 0x09fe548fu, 0x83852d0fu, 0x30362f1au, 0x7b5a9cc3u, 0x31fec169u, \
      0x9fec022au, 0x6c8dedc4u, 0x15d6874du, 0x5fde7a4eu, 0xbad90e37u, 0x2e4e5eefu, 0x4eaba214u, 0xa8a472c0u, 0x429a969eu, 0x148d302au, \
      0xc40ba6d0u, 0xc4e22c3cu, 0x40000000u, 0x20000000u, 0x08000000u, 0x00800000u, 0x00008000u, 0xedb88320u, 0xb1e6b092u, 0xa06a2517u, \
      0xed627daeu, 0x88d14467u, 0xd7bbfe6au, 0xec447f11u, 0x8e7ea170u, 0x6427800eu, 0x4d47bae0u, 0x09fe548fu, 0x83852d0fu, 0x30362f1au, \
      0x7b5a9cc3u, 0x31fec169u, 0x9fec022au, 0x6c8dedc4u, 0x15d6874du, 0x5fde7a4eu, 0xbad90e37u, 0x2e4e5eefu, 0x4eaba214u, 0xa8a472c0u, \
      0x429a969eu, 0x148d302au, 0xc40ba6d0u, 0xc4e22c3cu}}
__constant__ uint32_t g_crc_x2n[2][64] = TS_CRC_X2N_TABLE;
static const uint32_t h_crc_x2n[2][64] = TS_CRC_X2N_TABLE;      // the same table for host code (carries between batches)
#undef TS_CRC_X2N_TABLE
__host__ __device__ __forceinline__ uint32_t crc_x2n(int pi, int k) {
#ifdef __CUDA_ARCH__
    return g_crc_x2n[pi][k];
#else
    return h_crc_x2n[pi][k];
#endif
}

__host__ __device__ __forceinline__ uint32_t crc_mult(uint32_t a, uint32_t b, uint32_t poly) {      // a * b mod P (reflected)
    uint32_t p = 0;
#pragma unroll 4
    for (int i = 0; i < 32; i++) {
        p ^= (0u - ((a >> (31 - i)) & 1u)) & b;
        b = (b >> 1) ^ (poly & (0u - (b & 1u)));
    }
    return p;
}
__host__ __device__ __forceinline__ uint32_t crc_xn(uint64_t bytes, int pi) {   // x^(8 * bytes) mod P
    uint32_t p = 0x80000000u;
    for (int k = 3; bytes; bytes >>= 1, k++)
        if (bytes & 1) p = crc_mult(crc_x2n(pi, k), p, crc_poly(pi));
    return p;
}
// raw CRC of A followed by `bytes` more bytes whose raw CRC is 0 (the first operand of the combination above)
__host__ __device__ __forceinline__ uint32_t crc_shift(uint32_t crc, uint64_t bytes, int pi) {
    return crc ? crc_mult(crc_xn(bytes, pi), crc, crc_poly(pi)) : 0;
}
// the CRC (init and xorout 0xFFFFFFFF) of `bytes` bytes whose raw CRC is `raw`
__host__ __device__ __forceinline__ uint32_t crc_finish(uint32_t raw, uint64_t bytes, int pi) {
    return ~(raw ^ crc_shift(0xffffffffu, bytes, pi));
}

// Byte-table update: T is the 256-entry table of one polynomial.
__host__ __device__ __forceinline__ uint32_t crc_upd(const uint32_t* T, uint32_t c, uint32_t byte) { return T[(c ^ byte) & 0xffu] ^ (c >> 8); }
__host__ __device__ __forceinline__ uint32_t crc_bytes(const uint32_t* T, uint32_t c, const uint8_t* p, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) c = crc_upd(T, c, p[i]);
    return c;
}
__host__ __device__ __forceinline__ uint32_t crc_table_entry(uint32_t i, uint32_t poly) {
    uint32_t c = i;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (poly & (0u - (c & 1u)));
    return c;
}
// Byte tables of both polynomials (T[0]: CRC-32C, T[1]: CRC-32), block-cooperative.
__device__ __forceinline__ void crc_tables(uint32_t (*T)[256]) {
    for (uint32_t i = threadIdx.x; i < 512; i += blockDim.x) T[i >> 8][i & 255] = crc_table_entry(i & 255, crc_poly(i >> 8));
    __syncthreads();
}

}  // namespace ts
