/*
 * simt.h — TEST-ONLY SIMT emulator.  NOT part of the product; libtsgpu.so never includes this file.
 *
 * The build container has nvcc but no GPU, and GPU time (gpurun) is scarce.  To debug kernel *logic*
 * (bit-stream formats, table construction, index arithmetic) before going to an H100, the device
 * headers under tiered-storage-for-apache-kafka_b200/csrc/ are written in a restricted CUDA subset
 * that this header can also compile with plain g++: every CUDA thread of a block becomes a fiber
 * (hand-rolled x86-64 context switch), warp collectives and barriers are rendezvous points, blocks
 * run one after another.  Single OS thread => deterministic, no data races.  It models none of the
 * GPU's memory-ordering hazards, so the -m gpu parity tests and compute-sanitizer remain the real gate.
 */
#ifndef TSGPU_SIMT_H
#define TSGPU_SIMT_H
#ifndef TSGPU_SIMT
#error "simt.h is only for the test build (define TSGPU_SIMT)"
#endif
#include <algorithm>
#include <cassert>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>
#include <sys/mman.h>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __restrict__ __restrict
#define __shared__ static
#define __constant__ static
#define __align__(n) alignas(n)
#define __launch_bounds__(...)
#define __grid_constant__

struct uint3 { unsigned x, y, z; };
struct dim3 { unsigned x, y, z; dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {} };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(8) uint2 { uint32_t x, y; };
struct alignas(16) int4 { int32_t x, y, z, w; };
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }
static inline uint2 make_uint2(uint32_t a, uint32_t b) { return uint2{a, b}; }

namespace simt {

struct Warp {
    uint32_t buf[32];
    uint64_t buf64[32];
    int count = 0, gen = 0, alive = 0;
};
struct Fiber {
    void* sp = nullptr;
    uint3 tid{};
    int lane = 0, warp = 0;
    bool done = false;
    uint8_t* stack = nullptr;
};
struct Block {
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    int cur = 0;
    int alive = 0;
    int bar_count = 0, bar_gen = 0;
    int or_acc[3] = {0, 0, 0}, or_gen = 0;
    uint3 bid{};
    dim3 bdim, gdim;
    uint8_t* dyn_smem = nullptr;
    std::function<void()>* body = nullptr;
    void* sched_sp = nullptr;
};
extern Block* g_blk;
extern Fiber* g_cur;

extern "C" void simt_switch(void** save_sp, void* new_sp);
void yield();
void launch(dim3 grid, dim3 block, size_t dyn_smem_bytes, std::function<void()> body);
extern size_t g_collectives;

inline void warp_barrier() {
    Warp& w = g_blk->warps[g_cur->warp];
    g_collectives++;
    int my = w.gen;
    if (++w.count >= w.alive) { w.count = 0; w.gen++; }
    else while (w.gen == my) yield();
}
inline void block_barrier() {
    Block& b = *g_blk;
    int my = b.bar_gen;
    if (++b.bar_count >= b.alive) { b.bar_count = 0; b.bar_gen++; }
    else while (b.bar_gen == my) yield();
}
template <class T> inline T xchg(T v, int src) {
    static_assert(sizeof(T) <= 8, "");
    Warp& w = g_blk->warps[g_cur->warp];
    uint64_t raw = 0; memcpy(&raw, &v, sizeof(T));
    w.buf64[g_cur->lane] = raw;
    warp_barrier();
    uint64_t r = w.buf64[src & 31];
    warp_barrier();
    T out; memcpy(&out, &r, sizeof(T));
    return out;
}
}  // namespace simt

#define threadIdx (simt::g_cur->tid)
#define blockIdx (simt::g_blk->bid)
#define blockDim (simt::g_blk->bdim)
#define gridDim (simt::g_blk->gdim)
#define warpSize 32

static inline void __syncthreads() { simt::block_barrier(); }
static inline int __syncthreads_count(int pred) {
    simt::Block& b = *simt::g_blk;
    const int my = b.bar_gen, k = b.or_gen;          // or_gen moves only when a voting barrier completes
    if (pred) b.or_acc[k % 3] += 1;
    if (++b.bar_count >= b.alive) { b.bar_count = 0; b.or_acc[(k + 1) % 3] = 0; b.or_gen++; b.bar_gen++; }
    else while (b.bar_gen == my) simt::yield();
    return b.or_acc[k % 3];
}
static inline int __syncthreads_or(int pred) { return __syncthreads_count(pred) != 0; }
static inline void __syncwarp(unsigned = 0xffffffffu) { simt::warp_barrier(); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
template <class T> static inline T __shfl_sync(unsigned, T v, int src, int = 32) { return simt::xchg(v, src); }
template <class T> static inline T __shfl_up_sync(unsigned, T v, unsigned d, int = 32) {
    int l = simt::g_cur->lane; T r = simt::xchg(v, l - (int)d >= 0 ? l - (int)d : l); return l - (int)d >= 0 ? r : v;
}
template <class T> static inline T __shfl_down_sync(unsigned, T v, unsigned d, int = 32) {
    int l = simt::g_cur->lane; T r = simt::xchg(v, l + (int)d < 32 ? l + (int)d : l); return l + (int)d < 32 ? r : v;
}
template <class T> static inline T __shfl_xor_sync(unsigned, T v, int m, int = 32) {
    return simt::xchg(v, simt::g_cur->lane ^ m);
}
static inline unsigned __ballot_sync(unsigned, int pred) {
    simt::Warp& w = simt::g_blk->warps[simt::g_cur->warp];
    w.buf[simt::g_cur->lane] = pred ? 1u : 0u;
    simt::warp_barrier();
    unsigned r = 0;
    int base = simt::g_cur->warp * 32;
    for (int i = 0; i < 32; i++) {
        int t = base + i;
        if (t < (int)simt::g_blk->fibers.size() && !simt::g_blk->fibers[t].done && w.buf[i]) r |= 1u << i;
    }
    simt::warp_barrier();
    return r;
}
static inline int __any_sync(unsigned m, int p) { return __ballot_sync(m, p) != 0; }
static inline int __all_sync(unsigned m, int p) {
    unsigned alive = __ballot_sync(m, 1); return __ballot_sync(m, p) == alive;
}
static inline unsigned __reduce_add_sync(unsigned m, unsigned v) {
    unsigned s = v; for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(m, s, o); return s;
}
static inline unsigned __reduce_max_sync(unsigned m, unsigned v) {
    unsigned s = v; for (int o = 16; o; o >>= 1) { unsigned t = __shfl_xor_sync(m, s, o); s = t > s ? t : s; } return s;
}
static inline unsigned __reduce_min_sync(unsigned m, unsigned v) {
    unsigned s = v; for (int o = 16; o; o >>= 1) { unsigned t = __shfl_xor_sync(m, s, o); s = t < s ? t : s; } return s;
}
static inline unsigned __reduce_or_sync(unsigned m, unsigned v) {
    unsigned s = v; for (int o = 16; o; o >>= 1) s |= __shfl_xor_sync(m, s, o); return s;
}
static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __clzll(long long x) { return x ? __builtin_clzll((unsigned long long)x) : 64; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline int __ffsll(long long x) { return __builtin_ffsll(x); }
static inline unsigned __brev(unsigned x) {
    x = (x >> 16) | (x << 16); x = ((x & 0xff00ff00u) >> 8) | ((x & 0x00ff00ffu) << 8);
    x = ((x & 0xf0f0f0f0u) >> 4) | ((x & 0x0f0f0f0fu) << 4); x = ((x & 0xccccccccu) >> 2) | ((x & 0x33333333u) << 2);
    return ((x & 0xaaaaaaaau) >> 1) | ((x & 0x55555555u) << 1);
}
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned s) {
    uint64_t v = (uint64_t)b << 32 | a; unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        unsigned sel = (s >> (4 * i)) & 0xf; unsigned byte = (unsigned)(v >> (8 * (sel & 7))) & 0xff;
        if (sel & 8) byte = (byte & 0x80) ? 0xff : 0;
        r |= byte << (8 * i);
    }
    return r;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned s) {
    s &= 31; return s ? (lo >> s) | (hi << (32 - s)) : lo;
}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned s) {
    s &= 31; return s ? (hi << s) | (lo >> (32 - s)) : hi;
}
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
template <class T> static inline T __ldg(const T* p) { return *p; }
template <class T> static inline T atomicAdd(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicMax(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicMin(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicOr(T* p, T v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicXor(T* p, T v) { T o = *p; *p = o ^ v; return o; }
template <class T> static inline T atomicExch(T* p, T v) { T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T* p, T c, T v) { T o = *p; if (o == c) *p = v; return o; }
using std::max;
using std::min;

#endif
