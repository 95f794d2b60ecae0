// crc32.cuh — GF(2) arithmetic of the reflected CRC polynomials, shared by the record validation (records.cuh), the upload-part
// and object checksums (part_crc.cuh) and the host code that carries their state between batches and calls.  Generic over the
// CRC word W: uint32_t for CRC-32C (polynomial index 0) and CRC-32 (index 1), uint64_t for CRC-64/NVME (index 0).
//
// A "raw" CRC is the register after the bytes with initial value 0 and no final xor.  It is linear:
//   raw(A || B) = raw(A) * x^(8|B|) mod P  ^  raw(B)          (crc_shift(raw(A), |B|) ^ raw(B))
//   crc(A)      = ~(raw(A) ^ crc_shift(~0, |A|))              (init and xorout all ones)
// so the CRC of a range is combined from the CRCs of its pieces, whichever thread or call hashed them.
#pragma once
#include "ts_common.cuh"

namespace ts {

constexpr uint32_t CRC32C_POLY = 0x82F63B78u;   // Castagnoli, reflected (index 0)
constexpr uint32_t CRC32_POLY = 0xEDB88320u;    // IEEE, reflected (index 1)
constexpr uint64_t CRC64NVME_POLY = 0x9A6C9329AC4BC9B5ull;   // CRC-64/NVME, reflected (0xAD93D23594C93659 in normal form)
template <typename W = uint32_t> __host__ __device__ __forceinline__ W crc_poly(int pi) {
    if constexpr (sizeof(W) == 8) return CRC64NVME_POLY;
    else return pi ? CRC32_POLY : CRC32C_POLY;
}
template <typename W> struct crc_word { using type = W; };   // a W argument that takes no part in deduction (a literal 0 passes)

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
// x^(2^k) mod P, k = 0..63, for CRC-64/NVME (the squares of x, by crc_mult, from x = 0x4000000000000000)
#define TS_CRC64_X2N_TABLE                                                                                                       \
    {0x4000000000000000ull, 0x2000000000000000ull, 0x0800000000000000ull, 0x0080000000000000ull, 0x0000800000000000ull,     \
     0x0000000080000000ull, 0x9a6c9329ac4bc9b5ull, 0x10f4bb0f129310d6ull, 0x70f05dcea2ebd226ull, 0x311211205672822dull,     \
     0x2fc297db0f46c96eull, 0xca4d536fabf7da84ull, 0xfb4cdc3b379ee6edull, 0xea261148df25140aull, 0x59ccb2c07aa6c9b4ull,     \
     0x20b3674a839af27aull, 0x2d8e1986da94d583ull, 0x42cdf4c20337635dull, 0x1d78724bf0f26839ull, 0xb96c84e0afb34bd5ull,     \
     0x5d2e1fcd2df0a3eaull, 0xcd9506572332be42ull, 0x23bda2427f7d690full, 0x347a953232374f07ull, 0x1c2a807ac2a8ceeaull,     \
     0x9b92ad0e14fe1460ull, 0x2574114889f670b2ull, 0x4a84a6c45e3bf520ull, 0x915bbac21cd1c7ffull, 0xb0290ec579f291f5ull,     \
     0xcf2548505c624e6eull, 0xb154f27bf08a8207ull, 0xce4e92344baf7d35ull, 0x51da8d7e057c5eb3ull, 0x9fb10823f5be15dfull,     \
     0x73b825b3ff1f71cfull, 0x5db436c5406ebb74ull, 0xfa7ed8f3ec3f2bcaull, 0xc4d58efdc61b9ef6ull, 0xa7e39e61e855bd45ull,     \
     0x97ad46f9dd1bf2f1ull, 0x1a0abb01f853ee6bull, 0x3f0827c3348f8215ull, 0x4eb68c4506134607ull, 0x4a46f6de5df34e0aull,     \
     0x2d855d6a1c57a8ddull, 0x8688da58e1115812ull, 0x5232f417fc7c7300ull, 0xa4080fb2e767d8daull, 0xd515a7e17693e562ull,     \
     0x1181f7c862e94226ull, 0x9e23cd058204ca91ull, 0x9b8992c57a0aed82ull, 0xb2c0afb84609b6ffull, 0x2f7160553a5ea018ull,     \
     0x3cd378b5c99f2722ull, 0x814054ad61a3b058ull, 0xbf766189fce806d8ull, 0x85a5e898ac49f86full, 0x34830d11bc84f346ull,     \
     0x9644d95b173c8c1cull, 0x150401ac9ac759b1ull, 0xebe1f7f46fb00ebaull, 0x8ee4ce0c2e2bd662ull}
// in global memory rather than the constant bank, so that the constant offsets of every kernel built before it stay as they were
__device__ const uint64_t g_crc64_x2n[64] = TS_CRC64_X2N_TABLE;
static const uint64_t h_crc64_x2n[64] = TS_CRC64_X2N_TABLE;
#undef TS_CRC64_X2N_TABLE
template <typename W = uint32_t> __host__ __device__ __forceinline__ W crc_x2n(int pi, int k) {
#ifdef __CUDA_ARCH__
    if constexpr (sizeof(W) == 8) return g_crc64_x2n[k];
    else return g_crc_x2n[pi][k];
#else
    if constexpr (sizeof(W) == 8) return h_crc64_x2n[k];
    else return h_crc_x2n[pi][k];
#endif
}

template <typename W>
__host__ __device__ __forceinline__ W crc_mult(W a, W b, W poly) {      // a * b mod P (reflected)
    constexpr int N = 8 * sizeof(W);
    W p = 0;
#pragma unroll 4
    for (int i = 0; i < N; i++) {
        p ^= (W(0) - ((a >> (N - 1 - i)) & W(1))) & b;
        b = (b >> 1) ^ (poly & (W(0) - (b & W(1))));
    }
    return p;
}
template <typename W = uint32_t>
__host__ __device__ __forceinline__ W crc_xn(uint64_t bytes, int pi) {   // x^(8 * bytes) mod P
    W p = W(1) << (8 * sizeof(W) - 1);
    for (int k = 3; bytes; bytes >>= 1, k++)
        if (bytes & 1) p = crc_mult(crc_x2n<W>(pi, k), p, crc_poly<W>(pi));
    return p;
}
// raw CRC of A followed by `bytes` more bytes whose raw CRC is 0 (the first operand of the combination above)
template <typename W>
__host__ __device__ __forceinline__ W crc_shift(W crc, uint64_t bytes, int pi) {
    return crc ? crc_mult(crc_xn<W>(bytes, pi), crc, crc_poly<W>(pi)) : 0;
}
// the CRC (init and xorout all ones) of `bytes` bytes whose raw CRC is `raw`
template <typename W>
__host__ __device__ __forceinline__ W crc_finish(W raw, uint64_t bytes, int pi) {
    return ~(raw ^ crc_shift(W(~W(0)), bytes, pi));
}

// Byte-table update: T is the 256-entry table of one polynomial.
template <typename W>
__host__ __device__ __forceinline__ W crc_upd(const W* T, typename crc_word<W>::type c, uint32_t byte) { return T[(c ^ byte) & 0xffu] ^ (c >> 8); }
template <typename W>
__host__ __device__ __forceinline__ W crc_bytes(const W* T, typename crc_word<W>::type c, const uint8_t* p, uint32_t n) {
    for (uint32_t i = 0; i < n; i++) c = crc_upd(T, c, p[i]);
    return c;
}
template <typename W>
__host__ __device__ __forceinline__ W crc_table_entry(uint32_t i, W poly) {
    W c = i;
    for (int k = 0; k < 8; k++) c = (c >> 1) ^ (poly & (W(0) - (c & W(1))));
    return c;
}
// Byte tables of both polynomials (T[0]: CRC-32C, T[1]: CRC-32), block-cooperative.
__device__ __forceinline__ void crc_tables(uint32_t (*T)[256]) {
    for (uint32_t i = threadIdx.x; i < 512; i += blockDim.x) T[i >> 8][i & 255] = crc_table_entry(i & 255, crc_poly(i >> 8));
    __syncthreads();
}

}  // namespace ts
