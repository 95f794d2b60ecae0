// tsgpu.cu — libtsgpu.so: context, batch scheduling, C-ABI (include/tsgpu.h).
// Device code lives in the .cuh headers next to this file; this translation unit owns launches and copies.
//
// Host pipeline of tsgpu_transform (one segment):
//   split into batches of <= max_batch chunks -> dealt round-robin to (device, work-slot) pairs, each with its
//   own stream, device arenas and pinned descriptor block -> per batch: H2D original bytes, [zstd kernels],
//   [AES-GCM kernels], D2H of the chunk sizes, then per-chunk D2H of exactly transformed_size bytes to the
//   running offset in dst (the packed .log object layout, SURVEY.md appendix A.1).  Batches complete in order;
//   up to (devices x slots) batches are in flight so copies overlap kernels.  With TSGPU_FLAG_VERIFY each batch is
//   detransformed on the device and compared with its input before any of its bytes are copied out.
#include <condition_variable>
#include <mutex>
#include <new>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "../../include/tsgpu.h"
#include "ts_common.cuh"
#include "aesgcm.cuh"
#include "index_scan.cuh"
#include "pack.cuh"
#include "verify.cuh"
#include "rt.h"
#include "launch_prof.h"
#include "zstd_enc.cuh"
#include "zstd_enc_blk.cuh"
#include "zstd_dec.cuh"
#include "host_index.hpp"

using namespace ts;

static thread_local char g_err[512];
static int fail(int code, const char* fmt, ...) {
    va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap);
    return code;
}
#define RT(call) do { const char* e_ = (call); if (e_) return fail(TSGPU_E_CUDA, "%s: %s", #call, e_); } while (0)
#define CHECK_LAUNCH(what) do { const char* e_ = rt::last_error(); if (e_) return fail(TSGPU_E_CUDA, "launch %s: %s", what, e_); } while (0)

extern "C" const char* tsgpu_last_error(void) { return g_err; }
extern "C" const char* tsgpu_version(void) { return "tsgpu 0.1 (sm_90a)"; }

static inline uint64_t align_up(uint64_t v, uint64_t a) { return (v + a - 1) / a * a; }
static inline uint64_t frame_bound(uint64_t n) { return n + (n >> 8) + 64; }   // >= header + 3 bytes per 8 KiB block

// ------------------------------------------------------------------------------------------ context
namespace {

constexpr int NSLOT_MAX = 16;       // work slots per device; tsgpu_ctx::nslot of them are used
constexpr uint32_t MAX_AAD = 4096;
constexpr uint32_t KNOWN_FLAGS = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES | TSGPU_FLAG_ZSTD_DENSE;

struct Desc {            // device-side descriptor block of one work slot (all arrays sized for max_batch)
    uint64_t* a_off; uint64_t* b_off; uint64_t* c_off;
    uint32_t* a_len; uint32_t* b_len; uint32_t* c_len; uint32_t* status;
    uint32_t* v_len; uint32_t* v_diff;     // TSGPU_FLAG_VERIFY: read-back sizes, first differing byte per chunk
    uint8_t* ivs; uint8_t* aad;
};

struct Work {
    int device = 0;
    rt::stream_t stream{}, out_stream{};   // out_stream: copies of finished chunks back to the host
    rt::event_t ev_sizes{}, ev_done{};
    rt::event_t ev_dev_desc{}, ev_dev_done{};   // device API: descriptor upload of / end of the previous call on this slot
    bool dev_pending = false;
    bool out_pending = false;              // a copy-out on out_stream still reads this slot's final buffer
    bool ready = false;
    bool claimed = false;                  // owned by a call in progress (guarded by tsgpu_ctx::mu)
    Aes256RoundKeys key_rk{};      // the key this slot's GcmKeyCtx (H powers, Shoup table) was built for
    bool key_valid = false;        //   ... consecutive calls with one segment's data key skip the set-up kernel
    uint8_t* d_orig = nullptr;     // max_batch * chunk_cap
    uint8_t* d_frames = nullptr;   // max_batch * frame_stride        (zstd frames, 16-byte aligned slots)
    uint8_t* d_xf = nullptr;       // max_batch * slot_stride         (transformed slots)
    uint8_t* d_pack = nullptr;     // max_batch * slot_stride         (transformed chunks back to back: what one D2H takes home)
    uint8_t* d_desc = nullptr;  uint8_t* h_desc = nullptr;  size_t desc_bytes = 0;
    Desc dd{}, hd{};               // device / pinned-host views of the descriptor block
    uint4* d_partials = nullptr;  uint32_t max_ranges = 0;
    GcmKeyCtx* d_keyctx = nullptr;
    ZstdEncScratch zenc{};         // region kernel (TSGPU_FLAG_ZSTD_DENSE), allocated on first use
    ZstdBlkScratch zblk{};         // block kernel (default), allocated on first use
    ZstdDecScratch zdec{};
    uint32_t* h_sizes = nullptr;   // pinned: sizes/status (and the verify stage's first differing bytes) coming back
};

struct Lane { int device = 0; Work w[NSLOT_MAX]; };

}  // namespace

struct tsgpu_ctx {
    bool dense_default = false;    // TSGPU_ZSTD_MODE=dense: TSGPU_FLAG_ZSTD alone already means the region kernel
    bool verify_default = false;   // TSGPU_VERIFY=1: host-buffer transforms verify as if TSGPU_FLAG_VERIFY were set
    std::mutex mu;                 // guards slot ownership (Work::claimed, active_calls) and lazy slot allocation — NOT held while a call runs
    std::condition_variable cv;
    uint32_t active_calls = 0;
    std::vector<Lane> lanes;
    uint32_t chunk_cap = 0, max_batch = 0;
    uint64_t frame_stride = 0, slot_stride = 0;
    LaunchProf prof;
    uint32_t nslot = 16;           // work slots per device (TSGPU_SLOTS overrides); one call takes at most 8 of them
};

static void carve_desc(uint8_t* base, uint32_t nb, Desc& d, size_t* total) {
    size_t p = 0;
    auto take = [&](size_t bytes) { uint8_t* r = base ? base + p : nullptr; p += align_up(bytes, 256); return r; };
    d.a_off = (uint64_t*)take(8ull * nb); d.b_off = (uint64_t*)take(8ull * nb); d.c_off = (uint64_t*)take(8ull * (nb + 1));
    d.a_len = (uint32_t*)take(4ull * nb); d.b_len = (uint32_t*)take(4ull * nb); d.c_len = (uint32_t*)take(4ull * nb);
    d.status = (uint32_t*)take(4ull * nb);
    d.v_len = (uint32_t*)take(4ull * nb); d.v_diff = (uint32_t*)take(4ull * nb);
    d.ivs = take(12ull * nb); d.aad = take(MAX_AAD);
    if (total) *total = p;
}

static void work_free(Work& w);
static int work_init_impl(tsgpu_ctx* c, Work& w, int device);
// A slot that could not be fully allocated (out of memory on a busy GPU) is released again and stays "not ready", so a
// later call retries instead of running on half-initialised buffers.
static int work_init(tsgpu_ctx* c, Work& w, int device) {
    const int rc = work_init_impl(c, w, device);
    if (rc) { work_free(w); w = Work{}; w.device = device; }
    else w.ready = true;
    return rc;
}
static int work_init_impl(tsgpu_ctx* c, Work& w, int device) {
    w.device = device;
    RT(rt::set_device(device));
    RT(rt::stream_create(&w.stream));
    RT(rt::stream_create(&w.out_stream));
    RT(rt::event_create(&w.ev_sizes));
    RT(rt::event_create(&w.ev_done));
    RT(rt::event_create(&w.ev_dev_desc));
    RT(rt::event_create(&w.ev_dev_done));
    const uint64_t nb = c->max_batch;
    RT(rt::malloc_device((void**)&w.d_orig, nb * align_up(c->chunk_cap, 16) + 256));
    RT(rt::malloc_device((void**)&w.d_frames, nb * c->frame_stride + 256));
    RT(rt::malloc_device((void**)&w.d_xf, nb * c->slot_stride + 256));
    RT(rt::malloc_device((void**)&w.d_pack, nb * c->slot_stride + 256));
    carve_desc(nullptr, c->max_batch, w.dd, &w.desc_bytes);
    RT(rt::malloc_device((void**)&w.d_desc, w.desc_bytes));
    RT(rt::malloc_host((void**)&w.h_desc, w.desc_bytes));
    carve_desc(w.d_desc, c->max_batch, w.dd, nullptr);
    carve_desc(w.h_desc, c->max_batch, w.hd, nullptr);
    w.max_ranges = (uint32_t)((frame_bound(c->chunk_cap) / 16 + GH_RANGE_BLOCKS) / GH_RANGE_BLOCKS) + 1;
    RT(rt::malloc_device((void**)&w.d_partials, sizeof(uint4) * (size_t)w.max_ranges * nb));
    RT(rt::malloc_device((void**)&w.d_keyctx, sizeof(GcmKeyCtx)));
    RT(rt::malloc_host((void**)&w.h_sizes, 4ull * nb * 3 + 64));
    const char* e = zstd_dec_scratch_alloc(w.zdec, c->chunk_cap, c->max_batch);
    if (e) return fail(TSGPU_E_CUDA, "zstd dec scratch: %s", e);
    return TSGPU_OK;
}

static void work_free(Work& w) {
    if (!w.stream && !w.d_orig) return;                 // never initialised
    rt::set_device(w.device);
    if (w.stream) rt::stream_sync(w.stream);
    if (w.out_stream) rt::stream_sync(w.out_stream);
    rt::free_device(w.d_orig); rt::free_device(w.d_frames); rt::free_device(w.d_xf); rt::free_device(w.d_pack);
    rt::free_device(w.d_desc); rt::free_host(w.h_desc);
    rt::free_device(w.d_partials); rt::free_device(w.d_keyctx); rt::free_host(w.h_sizes);
    zstd_enc_scratch_free(w.zenc); zstd_blk_scratch_free(w.zblk); zstd_dec_scratch_free(w.zdec);
    memset(&w.key_rk, 0, sizeof w.key_rk); w.key_valid = false;
    rt::event_destroy(w.ev_sizes); rt::event_destroy(w.ev_done);
    rt::event_destroy(w.ev_dev_desc); rt::event_destroy(w.ev_dev_done);
    rt::stream_destroy(w.stream); rt::stream_destroy(w.out_stream);
}

extern "C" uint64_t tsgpu_slot_stride(uint32_t flags, uint32_t chunk_size) {
    uint64_t payload = (flags & TSGPU_FLAG_ZSTD) ? frame_bound(chunk_size) : chunk_size;
    return align_up(TSGPU_SLOT_HEAD + TSGPU_IV_SIZE + payload + TSGPU_TAG_SIZE, 16) + 16;
}

extern "C" uint64_t tsgpu_transform_bound(uint32_t flags, uint64_t src_len, uint32_t chunk_size) {
    if (src_len == 0) return 64;
    if (chunk_size == 0) chunk_size = (uint32_t)(src_len > 0x3fffffffu ? 0x3fffffffu : src_len);
    uint64_t n = (src_len + chunk_size - 1) / chunk_size;
    uint64_t per = (flags & TSGPU_FLAG_ZSTD) ? frame_bound(chunk_size) : chunk_size;
    if (flags & TSGPU_FLAG_AES) per += TSGPU_IV_SIZE + TSGPU_TAG_SIZE;
    return n * per;
}

extern "C" int tsgpu_create(const int* device_ids, int n_devices, uint32_t max_chunk_bytes, uint32_t max_batch,
                            tsgpu_ctx** out) {
    if (!out) return fail(TSGPU_E_ARG, "out cannot be null");
    *out = nullptr;
    if (max_chunk_bytes == 0 || max_chunk_bytes > 0x3fffffffu)
        return fail(TSGPU_E_ARG, "max_chunk_bytes must be in [1, 2^30-1], %u given", max_chunk_bytes);
    if (max_batch == 0) return fail(TSGPU_E_ARG, "max_batch must be positive");
    const int have = rt::device_count();
    if (have <= 0) return fail(TSGPU_E_NODEVICE, "no CUDA device visible: libtsgpu has no CPU fallback");
    std::vector<int> ids;
    if (!device_ids || n_devices <= 0) ids.push_back(0);
    else for (int i = 0; i < n_devices; i++) {
        if (device_ids[i] < 0 || device_ids[i] >= have) return fail(TSGPU_E_ARG, "device id %d out of range (have %d)", device_ids[i], have);
        ids.push_back(device_ids[i]);
    }
    tsgpu_ctx* c = new (std::nothrow) tsgpu_ctx();
    if (!c) return fail(TSGPU_E_NOMEM, "out of memory");
    c->chunk_cap = max_chunk_bytes; c->max_batch = max_batch;
    if (const char* e = getenv("TSGPU_SLOTS")) { int v = atoi(e); if (v >= 1 && v <= NSLOT_MAX) c->nslot = (uint32_t)v; }       // tuning knobs
    if (const char* e = getenv("TSGPU_ZSTD_MODE")) c->dense_default = strcmp(e, "dense") == 0;
    if (const char* e = getenv("TSGPU_VERIFY")) c->verify_default = strcmp(e, "1") == 0;
    c->frame_stride = align_up(frame_bound(max_chunk_bytes), 16) + 16;
    c->slot_stride = tsgpu_slot_stride(TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES, max_chunk_bytes);
    c->lanes.resize(ids.size());
    for (size_t l = 0; l < ids.size(); l++) {           // slot 0 now, the others on first use (claim_slots)
        c->lanes[l].device = ids[l];
        int rc = work_init(c, c->lanes[l].w[0], ids[l]);
        if (rc) { tsgpu_destroy(c); return rc; }
    }
    for (size_t l = 0; l < ids.size(); l++) {           // opt in to > 48 KiB dynamic shared memory, per device
        rt::set_device(ids[l]);
        const char* e = rt::allow_smem(gcm_main_kernel<true>, GCM_SMEM_BYTES);
        if (!e) e = rt::allow_smem(gcm_main_kernel<false>, GCM_SMEM_BYTES);
        if (e) { tsgpu_destroy(c); return fail(TSGPU_E_CUDA, "gcm kernel attributes: %s", e); }
        e = zstd_kernels_configure();
        if (e) { tsgpu_destroy(c); return fail(TSGPU_E_CUDA, "zstd kernel attributes: %s", e); }
    }
    *out = c;
    return TSGPU_OK;
}

extern "C" void tsgpu_destroy(tsgpu_ctx* c) {
    if (!c) return;
    for (auto& l : c->lanes) for (auto& w : l.w) work_free(w);
    delete c;
}

extern "C" void* tsgpu_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (rt::malloc_host(&p, bytes)) return nullptr;
    return p;
}
extern "C" void tsgpu_host_free(void* p) { rt::free_host(p); }
extern "C" uint64_t tsgpu_launch_count(const tsgpu_ctx* c) { return c ? c->prof.launches.load() : 0; }

// ------------------------------------------------------------------------------------------ stages
// A batch's chunks in one device buffer: chunk i is len[i] bytes at base + off[i] (off/len are device arrays).
namespace {
struct ChunksIn { const uint8_t* base; const uint64_t* off; const uint32_t* len; };
struct ChunksOut {
    uint8_t* base; uint64_t* off; uint32_t* len;
    operator ChunksIn() const { return {base, off, len}; }
};
// Per-chunk limits of the decrypt / decompress kernels.  Sizes of transformed chunks come from outside (a manifest): the
// kernels refuse a chunk that would overrun a buffer and report it in the status array.
struct DxBounds {
    uint32_t max_in;     // largest transformed chunk (sizes the GCM grid)
    uint32_t aes_room;   // plaintext bytes the GCM stage may write per chunk
    uint32_t zstd_in;    // frame bytes the zstd stage may read per chunk
    uint32_t zstd_out;   // original bytes per chunk
};
}

// zstd compress.  Two kernels, one contract (zstd_enc_blk.cuh: independent 8 KiB blocks, fastest; zstd_enc.cuh: 64 KiB
// regions with shared tables and history, densest).  Their scratch is allocated the first time a slot runs the mode.
static int zstd_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t flags, ChunksIn in, uint32_t nb, uint32_t cs, ChunksOut out) {
    const bool dense = (flags & TSGPU_FLAG_ZSTD_DENSE) || c->dense_default;
    int rc;
    if (dense) {
        if (!w.zenc.seqs) {
            const char* e = zstd_enc_scratch_alloc(w.zenc, c->chunk_cap, c->max_batch);
            if (e) { zstd_enc_scratch_free(w.zenc); return fail(TSGPU_E_CUDA, "zstd enc scratch: %s", e); }
        }
        rc = zstd_compress_batch(w.zenc, st, in.base, in.off, in.len, nb, cs, out.base, out.off, out.len, c->prof);
    } else {
        if (!w.zblk.seqs) {
            const char* e = zstd_blk_scratch_alloc(w.zblk, c->chunk_cap, c->max_batch);
            if (e) { zstd_blk_scratch_free(w.zblk); return fail(TSGPU_E_CUDA, "zstd enc scratch: %s", e); }
        }
        rc = zstd_compress_batch_blocks(w.zblk, st, in.base, in.off, in.len, nb, cs, out.base, out.off, out.len, c->prof);
    }
    if (rc) return fail(rc, "zstd compress: %s", zstd_last_error());
    return TSGPU_OK;
}

// AES-GCM: key set-up, the main kernel over (ranges x chunks) and the finalize kernel.  IVs (ENC) and AAD come from the
// slot's descriptor block.  The slot keeps the key tables of the last key it ran: consecutive calls with one segment's data
// key skip the set-up kernel.  Host and device calls share slot 0's tables; that is safe because device calls are ordered
// behind each other by events (dev_call_begin) and a host call takes the slot only once device work on it has completed.
template <bool ENC>
static int gcm_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, const Aes256RoundKeys& rk, ChunksIn in, ChunksOut out,
                     uint32_t aad_len, uint32_t* d_status, uint32_t n_chunks, uint32_t max_payload, uint32_t out_cap) {
    const bool key_ready = w.key_valid && memcmp(&w.key_rk, &rk, sizeof rk) == 0;
    w.key_rk = rk; w.key_valid = false;                      // valid again once the whole stage has been enqueued
    if (!key_ready) {
        TS_LAUNCH_P(c->prof, "gcm_key_setup", gcm_key_setup_kernel, dim3(1), dim3(GH_T), 0, st, rk, w.d_keyctx);
        CHECK_LAUNCH("gcm_key_setup_kernel");
    }
    GcmBatch B;
    B.in_base = in.base; B.in_off = in.off; B.in_len = in.len;
    B.out_base = out.base; B.out_off = out.off; B.out_len = out.len;
    B.ivs = ENC ? w.dd.ivs : nullptr; B.aad = w.dd.aad; B.aad_len = aad_len;
    B.partials = w.d_partials; B.max_ranges = w.max_ranges; B.status = d_status; B.n_chunks = n_chunks; B.out_cap = out_cap;
    uint32_t ranges = (uint32_t)(((uint64_t)max_payload + 15) / 16 + GH_RANGE_BLOCKS - 1) / GH_RANGE_BLOCKS;
    if (ranges > w.max_ranges) return fail(TSGPU_E_ARG, "chunk too large for this context");
    if (ranges) {
        TS_LAUNCH_P(c->prof, ENC ? "gcm_main_enc" : "gcm_main_dec", gcm_main_kernel<ENC>, dim3(ranges, n_chunks), dim3(GH_T),
                    GCM_SMEM_BYTES, st, rk, w.d_keyctx, B);
        CHECK_LAUNCH("gcm_main_kernel");
    }
    TS_LAUNCH_P(c->prof, ENC ? "gcm_finalize_enc" : "gcm_finalize_dec", gcm_finalize_kernel<ENC>, dim3((n_chunks + 3) / 4),
                dim3(128), 0, st, rk, w.d_keyctx, B);
    CHECK_LAUNCH("gcm_finalize_kernel");
    w.key_valid = true;
    return TSGPU_OK;
}

// A slot's next batch may start (copy-in, early kernels) while the previous batch's chunks are still going out on
// out_stream; the first kernel that overwrites the buffer they are read from waits for them here.
static int wait_copies_out(Work& w, rt::stream_t st) {
    if (w.out_pending) { RT(rt::stream_wait_event(st, w.ev_done)); w.out_pending = false; }
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ stage chains
// Used by the host-buffer and the device-resident calls alike; the caller has filled and uploaded the descriptor block.
// Between the two stages the chunks sit in the slot's frame buffer (16-byte aligned slots of frame_stride).

// [zstd ->] [AES-GCM encrypt]: nb chunks of at most cs bytes from `src` into `dst`.
static int transform_enqueue(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t flags, uint32_t nb, uint32_t cs,
                             const Aes256RoundKeys& rk, uint32_t aad_len, ChunksIn src, ChunksOut dst) {
    const bool aes = flags & TSGPU_FLAG_AES;
    uint32_t max_payload = cs;
    if (flags & TSGPU_FLAG_ZSTD) {
        const ChunksOut frames = aes ? ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len} : dst;
        int rc = zstd_stage(c, w, st, flags, src, nb, cs, frames);
        if (rc) return rc;
        src = frames; max_payload = (uint32_t)frame_bound(cs);
    }
    if (aes) return gcm_stage<true>(c, w, st, rk, src, dst, aad_len, w.dd.status, nb, max_payload, 0xffffffffu);
    return TSGPU_OK;
}

// [AES-GCM decrypt ->] [zstd]: nb chunks from `src` into `dst`.  packed: dst.off is written on the device as the running sum
// of the original sizes (chunks back to back) instead of being read as given.
static int detransform_enqueue(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t flags, uint32_t nb, const Aes256RoundKeys& rk,
                               uint32_t aad_len, ChunksIn src, ChunksOut dst, uint32_t* d_status, const DxBounds& lim, bool packed) {
    const bool zstd = flags & TSGPU_FLAG_ZSTD;
    if (flags & TSGPU_FLAG_AES) {
        const ChunksOut plain = zstd ? ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len} : dst;
        if (!zstd) { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }                        // dst is the final buffer
        int rc = gcm_stage<false>(c, w, st, rk, src, plain, aad_len, d_status, nb, lim.max_in, lim.aes_room);
        if (rc) return rc;
        src = plain;
    }
    if (zstd) {
        { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
        int rc = zstd_decompress_batch(w.zdec, st, src.base, src.off, src.len, nb, lim.zstd_out, dst.base, dst.off, dst.len,
                                       d_status, packed, c->prof, lim.zstd_in);
        if (rc) return fail(rc, "zstd decompress: %s", zstd_last_error());
    }
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ slot ownership
// Kafka drives this library from up to 10 copier threads plus the fetch pool (README.md:221 of the reference; SURVEY.md §8b
// "Threading").  A call does not hold a context-wide lock: it claims a set of work slots (streams + arenas + pinned
// descriptor block), runs on them, and gives them back.  The first caller gets up to 8 slots per device (what one segment
// needs to keep copies and kernels overlapped); later callers share what is free, so concurrent calls overlap on the GPU
// instead of queueing behind each other.
namespace {
struct SlotClaim {
    tsgpu_ctx* c = nullptr;
    std::vector<Work*> slots;
    ~SlotClaim() { release(); }
    void release() {
        if (!c || slots.empty()) { c = nullptr; return; }
        {
            std::lock_guard<std::mutex> lock(c->mu);
            for (Work* w : slots) w->claimed = false;
            c->active_calls--;
        }
        c->cv.notify_all();
        slots.clear(); c = nullptr;
    }
};
}
// Claims at least one slot (waiting if every slot is taken), at most `want` and at most the caller's fair share; slots are
// allocated on first use.  Returns TSGPU_OK with claim.slots interleaved across devices (round-robin dealing of batches).
static int claim_slots(tsgpu_ctx* c, uint32_t want, SlotClaim& claim, int only_device_index = -1, int only_slot = -1, bool wait_dev = true) {
    std::unique_lock<std::mutex> lock(c->mu);
    const uint32_t per_call_max = 8;
    while (true) {
        std::vector<Work*> got;
        const uint32_t share = std::max<uint32_t>(2, c->nslot / (c->active_calls + 1));
        const uint32_t per_dev = std::min(std::min(want, per_call_max), share);
        for (uint32_t k = 0; k < c->nslot && got.size() < (size_t)want; k++) {      // slot-major: interleaves the devices
            for (size_t l = 0; l < c->lanes.size(); l++) {
                if (only_device_index >= 0 && (int)l != only_device_index) continue;
                if (only_slot >= 0 && (int)k != only_slot) continue;
                Work& w = c->lanes[l].w[k];
                if (w.claimed) continue;
                uint32_t mine_on_dev = 0;
                for (Work* g : got) mine_on_dev += g->device == c->lanes[l].device ? 1u : 0u;
                if (only_slot < 0 && mine_on_dev >= per_dev) continue;
                got.push_back(&w);
            }
        }
        if (!got.empty()) {
            for (Work* w : got) w->claimed = true;
            c->active_calls++;
            claim.c = c; claim.slots = got;
            break;
        }
        c->cv.wait(lock);
    }
    // lazy allocation under the lock (rare: first use of a slot)
    for (Work* w : claim.slots) {
        if (!w->ready) {
            int rc = work_init(c, *w, w->device);
            if (rc) { lock.unlock(); claim.release(); return rc; }
        }
    }
    lock.unlock();
    if (wait_dev) for (Work* w : claim.slots) if (w->dev_pending) {        // device-API work enqueued on this slot's arenas: let it finish first
        const char* e = rt::set_device(w->device);
        if (!e) e = rt::event_sync(w->ev_dev_done);
        if (e) { claim.release(); return fail(TSGPU_E_CUDA, "event_sync: %s", e); }
        w->dev_pending = false;
    }
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ batches (host-buffer calls)
namespace {
struct Batch { Work* w; uint32_t c0, nb; };      // chunks [c0, c0 + nb) of a call, in flight on slot w
}

// Cuts n chunks into batches of max_batch and deals them round-robin over the slots it claims.  issue(batch) enqueues a
// batch on its slot's stream and ends with the D2H of its sizes (ev_sizes); drain(batch) runs once those sizes are on the
// host, in batch order, and sends the batch's bytes home (copy_out).  Returns with every claimed slot idle.
template <class Issue, class Drain>
static int run_batches(tsgpu_ctx* c, uint32_t n, Issue issue, Drain drain) {
    const uint32_t nbatches = (n + c->max_batch - 1) / c->max_batch;
    SlotClaim claim;
    { int rcc = claim_slots(c, nbatches, claim); if (rcc) return rcc; }
    const uint32_t nwork = (uint32_t)claim.slots.size();
    std::vector<Batch> inflight(nbatches);
    uint32_t drained = 0;
    auto drain_next = [&]() -> int {
        const Batch& bt = inflight[drained++];
        RT(rt::set_device(bt.w->device));
        RT(rt::event_sync(bt.w->ev_sizes));
        return drain(bt);
    };
    int rc = TSGPU_OK;
    for (uint32_t b = 0; b < nbatches && rc == TSGPU_OK; b++) {
        // From b = nwork on a slot is reused: its previous batch is drained first (sizes read on the host, copies-out
        // enqueued on the slot's out_stream); the new batch's copy-in and first kernels start right away and only the
        // kernel that overwrites the buffer being copied out waits for those copies (wait_copies_out) — the host never
        // waits here, which keeps all slots' queues full.
        if (b >= nwork) { rc = drain_next(); if (rc) break; }
        const uint32_t c0 = b * c->max_batch;
        inflight[b] = Batch{claim.slots[b % nwork], c0, std::min(c->max_batch, n - c0)};
        rc = issue(inflight[b]);
    }
    while (rc == TSGPU_OK && drained < nbatches) rc = drain_next();
    for (Work* w : claim.slots) {                    // always leave the claimed slots idle
        rt::set_device(w->device);
        const char* e = rt::stream_sync(w->stream);
        if (!e) e = rt::stream_sync(w->out_stream);
        if (e && rc == TSGPU_OK) rc = fail(TSGPU_E_CUDA, "stream_sync: %s", e);
        w->out_pending = false;
    }
    return rc;
}

// A drained batch's `total` bytes at `from` go to dst + dst_off on the slot's copy-out stream (the sizes event has
// completed: there is nothing to order them behind).
static int copy_out(Work& w, const uint8_t* from, uint64_t total, uint8_t* dst, uint64_t dst_cap, uint64_t& dst_off) {
    if (dst_off + total > dst_cap) return fail(TSGPU_E_SHORT, "dst too small");
    if (total) RT(rt::d2h(dst + dst_off, from, total, w.out_stream));
    dst_off += total;
    RT(rt::event_record(w.ev_done, w.out_stream));
    w.out_pending = true;
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ transform (host)
// TSGPU_FLAG_VERIFY: the batch's transformed chunks (`fin`, still in their slots once pack_chunks has run) go through the
// detransform stages and are compared with the input in d_orig.  No buffer beyond the slot's own: Z|A decrypts d_xf into
// d_frames and decodes that into d_xf; A decrypts d_xf into d_frames; Z decodes d_frames into d_xf.  The read-back chunk i
// lands at b_off[i] (a 16-byte aligned frame slot; d_xf's slots are larger) with its size in v_len, so a_len survives.
// Leaves per chunk: status 0 / 1 tag / 2 frame / VERIFY_ST_SIZE, and v_diff = first differing byte or VERIFY_NO_DIFF.
static int verify_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t flags, uint32_t nb, uint32_t cs,
                        const Aes256RoundKeys& rk, uint32_t aad_len, ChunksOut fin) {
    const bool zstd = flags & TSGPU_FLAG_ZSTD;
    RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
    RT(rt::memset_async(w.dd.v_diff, 0xff, 4ull * nb, st));
    DxBounds lim;
    lim.max_in = (uint32_t)((zstd ? frame_bound(cs) : cs) + TSGPU_IV_SIZE + TSGPU_TAG_SIZE);
    lim.aes_room = zstd ? (uint32_t)(c->frame_stride - 16) : c->chunk_cap;
    lim.zstd_in = (uint32_t)(c->frame_stride - 16);
    lim.zstd_out = cs;                                        // a frame claiming more than the batch's largest chunk is wrong
    const ChunksOut back{zstd ? w.d_xf : w.d_frames, w.dd.b_off, w.dd.v_len};
    { int rc = detransform_enqueue(c, w, st, flags & (TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES), nb, rk, aad_len, fin, back, w.dd.status,
                                   lim, /*packed=*/false); if (rc) return rc; }
    VerifyArgs V;
    V.orig = w.d_orig; V.orig_off = w.dd.a_off; V.orig_len = w.dd.a_len;
    V.back = back.base; V.back_off = back.off; V.back_len = back.len;
    V.status = w.dd.status; V.diff = w.dd.v_diff;
    TS_LAUNCH_P(c->prof, "verify_compare", verify_compare_kernel, dim3((cs + VERIFY_PIECE - 1) / VERIFY_PIECE, nb), dim3(VERIFY_T), 0, st, V);
    CHECK_LAUNCH("verify_compare_kernel");
    return TSGPU_OK;
}

#ifdef TSGPU_SIMT
// TEST-ONLY fault injection, compiled into the emulator build alone (device memory is host memory there and every kernel
// has finished when its launch returns).  TSGPU_SIMT_FLIP=<chunk>:<offset> flips the low bit of one byte of that chunk's
// transformed bytes -- frame, or IV || ciphertext || tag -- before they are packed and verified.  A negative offset counts
// from the chunk's end (-1: last tag byte).  tests/test_simt_verify.py drives it.
static void simt_inject_fault(ChunksOut fin, uint32_t c0, uint32_t nb) {
    const char* e = getenv("TSGPU_SIMT_FLIP");
    long k = 0, at = 0;
    if (!e || sscanf(e, "%ld:%ld", &k, &at) != 2 || k < (long)c0 || k >= (long)c0 + (long)nb) return;
    const uint32_t i = (uint32_t)(k - c0), n = fin.len[i];
    if (at < 0) at += n;
    if (at >= 0 && at < (long)n) fin.base[fin.off[i] + at] ^= 1;
}
#endif

// One batch: copy in, fill the descriptors, enqueue the stages, pack the transformed chunks, [verify them,] D2H of their
// sizes (and of the verify stage's verdicts).
// `off`/`len`: position and size of every chunk inside src (chunks are contiguous); `cs` = largest chunk of the call.
static int transform_issue(tsgpu_ctx* c, const Batch& bt, uint32_t flags, bool verify, const uint8_t* src, const uint64_t* off,
                           const uint32_t* len, uint32_t cs, const Aes256RoundKeys& rk, const uint8_t* aad, uint32_t aad_len,
                           const uint8_t* ivs) {
    Work& w = *bt.w;
    const uint32_t c0 = bt.c0, nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    const uint64_t byte0 = off[c0];
    const uint64_t byte1 = off[c0 + nb - 1] + len[c0 + nb - 1];
    RT(rt::h2d(w.d_orig, src + byte0, byte1 - byte0, st));
    // descriptor block: a = original chunks, b = frames, c = transformed slots
    for (uint32_t i = 0; i < nb; i++) {
        w.hd.a_off[i] = off[c0 + i] - byte0;
        w.hd.a_len[i] = len[c0 + i];
        w.hd.b_off[i] = (uint64_t)i * c->frame_stride;
        w.hd.c_off[i] = (uint64_t)i * c->slot_stride + TSGPU_SLOT_HEAD;
    }
    const bool aes = flags & TSGPU_FLAG_AES;
    if (aes) {
        memcpy(w.hd.ivs, ivs + (size_t)c0 * TSGPU_IV_SIZE, (size_t)nb * TSGPU_IV_SIZE);
        if (aad_len) memcpy(w.hd.aad, aad, aad_len);
    }
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    // encrypted chunks land in the transformed slots; zstd alone leaves its frames in the frame slots
    const ChunksOut fin = aes ? ChunksOut{w.d_xf, w.dd.c_off, w.dd.c_len} : ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len};
    { int rc = transform_enqueue(c, w, st, flags, nb, cs, rk, aad_len, ChunksIn{w.d_orig, w.dd.a_off, w.dd.a_len}, fin); if (rc) return rc; }
#ifdef TSGPU_SIMT
    simt_inject_fault(fin, c0, nb);
#endif
    // the transformed chunks, back to back, so the batch leaves in one copy (the previous batch's copy-out may still be
    // reading d_pack: this is the first kernel of the batch that has to wait for it)
    { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
    {
        PackArgs P;
        P.base = fin.base; P.stride = aes ? c->slot_stride : c->frame_stride; P.head = aes ? TSGPU_SLOT_HEAD : 0;
        P.len = fin.len; P.n = nb; P.out = w.d_pack;
        const uint64_t longest = (flags & TSGPU_FLAG_ZSTD) ? frame_bound(cs) + 28 : (uint64_t)cs + 28;
        TS_LAUNCH_P(c->prof, "pack_chunks", pack_chunks_kernel, dim3((uint32_t)((longest + PACK_PIECE - 1) / PACK_PIECE), nb), dim3(PACK_T), 0, st, P);
        CHECK_LAUNCH("pack_chunks_kernel");
    }
    if (verify) {
        int rc = verify_stage(c, w, st, flags, nb, cs, rk, aad_len, fin);
        if (rc) return rc;
        RT(rt::d2h(w.h_sizes + nb, w.dd.status, 4ull * nb, st));
        RT(rt::d2h(w.h_sizes + 2 * nb, w.dd.v_diff, 4ull * nb, st));
    }
    RT(rt::d2h(w.h_sizes, fin.len, 4ull * nb, st));
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

// The verify stage's verdict on a drained batch (h_sizes: sizes, status, first differing bytes); TSGPU_OK if every chunk
// read back.  `len`: the original chunk sizes of the call.
static int verify_verdict(const Batch& bt, const uint32_t* len) {
    const uint32_t* status = bt.w->h_sizes + bt.nb;
    const uint32_t* diff = bt.w->h_sizes + 2 * bt.nb;
    for (uint32_t i = 0; i < bt.nb; i++) {
        const uint32_t k = bt.c0 + i;
        if (status[i] == 1) return fail(TSGPU_E_VERIFY, "verify: chunk %u did not read back: tag check failed", k);
        if (status[i] == VERIFY_ST_SIZE)
            return fail(TSGPU_E_VERIFY, "verify: chunk %u did not read back: size check failed (original %u bytes)", k, len[k]);
        if (status[i] != 0) return fail(TSGPU_E_VERIFY, "verify: chunk %u did not read back: frame check failed (code %u)", k, status[i]);
        if (diff[i] != VERIFY_NO_DIFF)
            return fail(TSGPU_E_VERIFY, "verify: chunk %u did not read back: bytes differ from offset %u", k, diff[i]);
    }
    return TSGPU_OK;
}

static int transform_common(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const std::vector<uint64_t>& off,
                            const std::vector<uint32_t>& len, uint32_t cs, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                            const uint8_t* ivs, uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks);

static int transform_args_ok(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint8_t* key, const uint8_t* aad,
                             uint32_t aad_len, const uint8_t* ivs, uint32_t* transformed_sizes, uint32_t* n_chunks) {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!n_chunks || !transformed_sizes) return fail(TSGPU_E_ARG, "transformed_sizes/n_chunks cannot be null");
    if (src_len && !src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (flags & ~(KNOWN_FLAGS | TSGPU_FLAG_VERIFY)) return fail(TSGPU_E_ARG, "unknown flags %u", flags);
    if ((flags & TSGPU_FLAG_AES) && (!key || !ivs)) return fail(TSGPU_E_ARG, "key and ivs are required for encryption");
    if ((flags & TSGPU_FLAG_AES) && aad_len > MAX_AAD) return fail(TSGPU_E_ARG, "aad longer than %u bytes", MAX_AAD);
    if ((flags & TSGPU_FLAG_AES) && aad_len && !aad) return fail(TSGPU_E_ARG, "aad cannot be null");
    return TSGPU_OK;
}

extern "C" int tsgpu_transform(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                               const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                               uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks) try {
    int rc = transform_args_ok(c, flags, src, src_len, key, aad, aad_len, ivs, transformed_sizes, n_chunks);
    if (rc) return rc;
    // BaseTransformChunkEnumeration: originalChunkSize 0 disables chunking (one chunk = whole stream)
    uint64_t cs64 = chunk_size ? chunk_size : src_len;
    if (src_len == 0) { *n_chunks = 0; return TSGPU_OK; }
    if (cs64 > c->chunk_cap) return fail(TSGPU_E_ARG, "chunk size %llu exceeds the context's max_chunk_bytes %u", (unsigned long long)cs64, c->chunk_cap);
    const uint32_t cs = (uint32_t)cs64;
    const uint64_t n64 = (src_len + cs - 1) / cs;
    if (n64 > *n_chunks) return fail(TSGPU_E_SHORT, "transformed_sizes too small: %llu chunks", (unsigned long long)n64);
    std::vector<uint64_t> off(n64);
    std::vector<uint32_t> len(n64);
    for (uint64_t i = 0; i < n64; i++) { off[i] = i * cs; len[i] = (uint32_t)std::min<uint64_t>(cs, src_len - i * cs); }
    return transform_common(c, flags, src, src_len, off, len, cs, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, n_chunks);
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

// Ragged variant: chunk i is the next chunk_lens[i] bytes of src.  This is what RemoteStorageManager.transformIndex
// (RemoteStorageManager.java:455-490) needs: every Kafka index file is ONE chunk (chunking disabled), AES only, and the
// five of them ride in a single batch (SURVEY.md §8f.3).
extern "C" int tsgpu_transform_chunks(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, const uint32_t* chunk_lens, uint32_t n,
                                      const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                      uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes) try {
    uint32_t cap = n;
    if (n && !chunk_lens) return fail(TSGPU_E_ARG, "chunk_lens cannot be null");
    uint64_t total = 0; uint32_t mx = 0;
    std::vector<uint64_t> off(n);
    std::vector<uint32_t> len(n);
    for (uint32_t i = 0; i < n; i++) {
        if (chunk_lens[i] == 0) return fail(TSGPU_E_ARG, "chunk %u is empty", i);
        off[i] = total; len[i] = chunk_lens[i]; total += chunk_lens[i]; mx = std::max(mx, chunk_lens[i]);
    }
    int rc = transform_args_ok(c, flags, src, total, key, aad, aad_len, ivs, transformed_sizes, &cap);
    if (rc) return rc;
    if (n == 0) return TSGPU_OK;
    if (mx > c->chunk_cap) return fail(TSGPU_E_ARG, "chunk size %u exceeds the context's max_chunk_bytes %u", mx, c->chunk_cap);
    return transform_common(c, flags, src, total, off, len, mx, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, &cap);
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

static int transform_common(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const std::vector<uint64_t>& off,
                            const std::vector<uint32_t>& len, uint32_t cs, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                            const uint8_t* ivs, uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks) {
    const uint32_t n = (uint32_t)len.size();
    if (!dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (!(flags & TSGPU_FLAG_ZSTD)) flags &= ~TSGPU_FLAG_ZSTD_DENSE;   // a modifier of ZSTD: meaningless (and harmless) without it
    const bool verify = (flags & TSGPU_FLAG_VERIFY) || c->verify_default;
    flags &= ~TSGPU_FLAG_VERIFY;

    if (flags == 0) {       // TransformFinisher no-transform fast path (TransformFinisher.java:135-140): bytes unchanged, nothing to verify
        if (dst_cap < src_len) return fail(TSGPU_E_SHORT, "dst too small");
        memcpy(dst, src, src_len);
        for (uint32_t i = 0; i < n; i++) transformed_sizes[i] = len[i];
        *n_chunks = n;
        return TSGPU_OK;
    }
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);

    uint64_t dst_off = 0;
    const int rc = run_batches(c, n,
        [&](const Batch& bt) { return transform_issue(c, bt, flags, verify, src, off.data(), len.data(), cs, rk, aad, aad_len, ivs); },
        [&](const Batch& bt) {
            Work& w = *bt.w;
            if (verify) { int rcv = verify_verdict(bt, len.data()); if (rcv) return rcv; }   // none of the batch's bytes leave
            uint64_t total = 0;
            for (uint32_t i = 0; i < bt.nb; i++) { transformed_sizes[bt.c0 + i] = w.h_sizes[i]; total += w.h_sizes[i]; }
            return copy_out(w, w.d_pack, total, dst, dst_cap, dst_off);     // one copy per batch: packed on the device
        });
    if (rc) return rc;
    *n_chunks = n;
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ detransform (host)
// One batch: bound the sizes, copy the chunks in, fill the descriptors, enqueue the stages, D2H of sizes and status.
// `src`: the batch's first transformed chunk.
static int detransform_issue(tsgpu_ctx* c, const Batch& bt, uint32_t flags, const uint8_t* src, const uint32_t* tsizes,
                             const Aes256RoundKeys& rk, const uint8_t* aad, uint32_t aad_len) {
    Work& w = *bt.w;
    const uint32_t c0 = bt.c0, nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    // Sizes come from a manifest, i.e. from outside: bound them per mode BEFORE any kernel writes (the GCM kernel
    // releases plaintext into the next buffer before the tag is checked).  AES only: plaintext lands in d_orig
    // (chunk_cap per chunk); AES+zstd: in a d_frames slot; zstd only: the frame is read in place from d_xf.
    const uint32_t room = (flags & TSGPU_FLAG_ZSTD) ? (uint32_t)(c->frame_stride - 16) : c->chunk_cap;
    uint64_t ip = 0, op = 0;
    uint32_t max_t = 0;
    for (uint32_t i = 0; i < nb; i++) {
        const uint32_t t = tsizes[c0 + i];
        const uint64_t payload = (flags & TSGPU_FLAG_AES) ? (t >= 28 ? t - 28 : 0) : t;
        if (payload > room || t > c->slot_stride - TSGPU_SLOT_HEAD - 16)
            return fail(TSGPU_E_ARG, "transformed chunk of %u bytes exceeds the context's capacity", t);
        w.hd.c_off[i] = (uint64_t)i * c->slot_stride + TSGPU_SLOT_HEAD;
        w.hd.c_len[i] = t;
        w.hd.b_off[i] = (uint64_t)i * c->frame_stride;
        w.hd.a_off[i] = op;                              // used when there is no zstd stage (sizes are known)
        if (t) RT(rt::h2d(w.d_xf + w.hd.c_off[i], src + ip, t, st));
        ip += t;
        op += payload;
        max_t = std::max(max_t, t);
    }
    if ((flags & TSGPU_FLAG_AES) && aad_len) memcpy(w.hd.aad, aad, aad_len);
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
    const DxBounds lim{max_t, room, 0xffffffffu, c->chunk_cap};
    { int rc = detransform_enqueue(c, w, st, flags, nb, rk, aad_len, ChunksIn{w.d_xf, w.dd.c_off, w.dd.c_len},
                                   ChunksOut{w.d_orig, w.dd.a_off, w.dd.a_len}, w.dd.status, lim, /*packed=*/true); if (rc) return rc; }
    RT(rt::d2h(w.h_sizes, w.dd.a_len, 4ull * nb, st));
    RT(rt::d2h(w.h_sizes + nb, w.dd.status, 4ull * nb, st));
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

extern "C" int tsgpu_detransform(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len,
                                 const uint32_t* transformed_sizes, uint32_t n_chunks,
                                 const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                 uint8_t* dst, uint64_t dst_cap, uint32_t* original_sizes) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (n_chunks == 0) return TSGPU_OK;
    if (!src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (!transformed_sizes) return fail(TSGPU_E_ARG, "chunks cannot be null");
    if (!dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (flags & ~KNOWN_FLAGS) return fail(TSGPU_E_ARG, "unknown flags %u", flags);
    if ((flags & TSGPU_FLAG_AES) && !key) return fail(TSGPU_E_ARG, "key is required for decryption");
    if ((flags & TSGPU_FLAG_AES) && aad_len > MAX_AAD) return fail(TSGPU_E_ARG, "aad longer than %u bytes", MAX_AAD);
    flags &= ~TSGPU_FLAG_ZSTD_DENSE;                         // how a frame was compressed does not matter to the reader
    uint64_t need = 0;
    for (uint32_t i = 0; i < n_chunks; i++) need += transformed_sizes[i];
    if (need > src_len) return fail(TSGPU_E_SHORT, "Stream has fewer bytes than expected");

    if (flags == 0) {       // DetransformFinisher pass-through (DetransformFinisher.java:48-51)
        if (dst_cap < need) return fail(TSGPU_E_SHORT, "dst too small");
        memcpy(dst, src, need);
        if (original_sizes) for (uint32_t i = 0; i < n_chunks; i++) original_sizes[i] = transformed_sizes[i];
        return TSGPU_OK;
    }
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);

    uint64_t in_off = 0, dst_off = 0;                        // batches are issued in order: in_off walks src with them
    int soft = TSGPU_OK;
    const int rc = run_batches(c, n_chunks,
        [&](const Batch& bt) {
            const int r = detransform_issue(c, bt, flags, src + in_off, transformed_sizes, rk, aad, aad_len);
            for (uint32_t i = 0; i < bt.nb; i++) in_off += transformed_sizes[bt.c0 + i];
            return r;
        },
        [&](const Batch& bt) {
            Work& w = *bt.w;
            uint64_t total = 0;
            for (uint32_t i = 0; i < bt.nb; i++) {
                uint32_t stt = w.h_sizes[bt.nb + i];
                if (stt == 1 && soft == TSGPU_OK) soft = fail(TSGPU_E_AUTH, "Tag mismatch in chunk %u", bt.c0 + i);
                else if (stt > 1 && soft == TSGPU_OK) soft = fail(TSGPU_E_CORRUPT, "Invalid zstd frame in chunk %u (code %u)", bt.c0 + i, stt);
                if (original_sizes) original_sizes[bt.c0 + i] = w.h_sizes[i];
                total += w.h_sizes[i];
            }
            if (soft != TSGPU_OK) return soft;
            return copy_out(w, w.d_orig, total, dst, dst_cap, dst_off);
        });
    if (rc == TSGPU_E_AUTH || rc == TSGPU_E_CORRUPT) {
        // JCE releases no plaintext when the tag check fails: do not leave partial output behind
        memset(dst, 0, (size_t)dst_off);
    }
    return rc;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

// ------------------------------------------------------------------------------------------ device-resident API
// The device API reuses slot 0's pinned descriptor block and scratch arenas.  Two events make back-to-back calls safe on
// any streams: the host waits until the previous call's descriptor upload has left the pinned block before rewriting it,
// and the new call's stream waits for the previous call's kernels before touching the shared scratch.

// Argument checks of both device calls; n (the number of chunks) == 0 passes, and the call then has nothing to do.
static int dev_args_ok(tsgpu_ctx* c, int device_index, uint32_t flags, uint32_t chunk_size, uint64_t n, uint64_t slot_stride) {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (device_index < 0 || device_index >= (int)c->lanes.size()) return fail(TSGPU_E_ARG, "device_index %d out of range", device_index);
    if (flags & TSGPU_FLAG_VERIFY)
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_VERIFY (%u) applies to the host-buffer transform calls only", TSGPU_FLAG_VERIFY);
    if ((flags & (TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES)) == 0 || (flags & ~KNOWN_FLAGS)) return fail(TSGPU_E_ARG, "flags must name zstd and/or aes");
    if (chunk_size == 0 || chunk_size > c->chunk_cap) return fail(TSGPU_E_ARG, "chunk_size out of range for this context");
    if (n == 0) return TSGPU_OK;
    if (n > c->max_batch) return fail(TSGPU_E_ARG, "%llu chunks exceed the context's max_batch %u", (unsigned long long)n, c->max_batch);
    if (slot_stride < tsgpu_slot_stride(flags, chunk_size) || (slot_stride & 15)) return fail(TSGPU_E_ARG, "slot_stride too small or not a multiple of 16");
    return TSGPU_OK;
}

// Claims slot 0 of the device for the duration of the enqueue, orders this call behind the previous device call, lets
// fill(w) write the descriptor block and uploads it.  The slot is claim.slots[0].
template <class Fill>
static int dev_call_begin(tsgpu_ctx* c, int device_index, rt::stream_t st, SlotClaim& claim, Fill fill) {
    { int rcc = claim_slots(c, 1, claim, device_index, 0, /*wait_dev=*/false); if (rcc) return rcc; }
    Work& w = *claim.slots[0];
    RT(rt::set_device(w.device));
    if (w.dev_pending) { RT(rt::event_sync(w.ev_dev_desc)); RT(rt::stream_wait_event(st, w.ev_dev_done)); }
    fill(w);
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    RT(rt::event_record(w.ev_dev_desc, st));
    w.dev_pending = true;                                    // from here on the next call must order itself behind this one
    RT(rt::event_record(w.ev_dev_done, st));
    return TSGPU_OK;
}

extern "C" int tsgpu_transform_device(tsgpu_ctx* c, int device_index, uint32_t flags, const uint8_t* d_src, uint64_t src_len,
                                      uint32_t chunk_size, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                      const uint8_t* ivs, uint8_t* d_slots, uint64_t slot_stride,
                                      uint32_t* d_transformed_sizes, void* stream) {
    const uint64_t n64 = chunk_size ? (src_len + chunk_size - 1) / chunk_size : 0;
    int rc = dev_args_ok(c, device_index, flags, chunk_size, n64, slot_stride);
    if (rc || n64 == 0) return rc;
    if ((flags & TSGPU_FLAG_AES) && (!key || !ivs || aad_len > MAX_AAD)) return fail(TSGPU_E_ARG, "key/ivs/aad invalid");
    const uint32_t nb = (uint32_t)n64, cs = chunk_size;
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);
    rt::stream_t st = (rt::stream_t)stream;
    SlotClaim claim;
    rc = dev_call_begin(c, device_index, st, claim, [&](Work& w) {
        for (uint32_t i = 0; i < nb; i++) {
            w.hd.a_off[i] = (uint64_t)i * cs;
            w.hd.a_len[i] = (uint32_t)std::min<uint64_t>(cs, src_len - (uint64_t)i * cs);
            w.hd.b_off[i] = (uint64_t)i * c->frame_stride;
            w.hd.c_off[i] = (uint64_t)i * slot_stride + TSGPU_SLOT_HEAD;
        }
        if (flags & TSGPU_FLAG_AES) {
            memcpy(w.hd.ivs, ivs, (size_t)nb * TSGPU_IV_SIZE);
            if (aad_len) memcpy(w.hd.aad, aad, aad_len);
        }
    });
    if (rc) return rc;
    Work& w = *claim.slots[0];
    rc = transform_enqueue(c, w, st, flags, nb, cs, rk, aad_len, ChunksIn{d_src, w.dd.a_off, w.dd.a_len},
                           ChunksOut{d_slots, w.dd.c_off, d_transformed_sizes});
    if (rc) return rc;
    RT(rt::event_record(w.ev_dev_done, st));
    return TSGPU_OK;
}

extern "C" int tsgpu_detransform_device(tsgpu_ctx* c, int device_index, uint32_t flags, const uint8_t* d_slots,
                                        uint64_t slot_stride, const uint32_t* d_transformed_sizes, uint32_t n_chunks,
                                        uint32_t chunk_size, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                        uint8_t* d_dst, uint32_t* d_original_sizes, uint32_t* d_status, void* stream) {
    int rc = dev_args_ok(c, device_index, flags, chunk_size, n_chunks, slot_stride);
    if (rc || n_chunks == 0) return rc;
    if ((flags & TSGPU_FLAG_AES) && (!key || aad_len > MAX_AAD)) return fail(TSGPU_E_ARG, "key/aad invalid");
    if (!d_slots || !d_transformed_sizes || !d_dst || !d_original_sizes || !d_status) return fail(TSGPU_E_ARG, "null device pointer");
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);
    rt::stream_t st = (rt::stream_t)stream;
    SlotClaim claim;
    rc = dev_call_begin(c, device_index, st, claim, [&](Work& w) {
        for (uint32_t i = 0; i < n_chunks; i++) {
            w.hd.c_off[i] = (uint64_t)i * slot_stride + TSGPU_SLOT_HEAD;
            w.hd.b_off[i] = (uint64_t)i * c->frame_stride;
            w.hd.a_off[i] = (uint64_t)i * chunk_size;        // original side: chunk i at i * chunk_size
        }
        if ((flags & TSGPU_FLAG_AES) && aad_len) memcpy(w.hd.aad, aad, aad_len);
    });
    if (rc) return rc;
    Work& w = *claim.slots[0];
    RT(rt::memset_async(d_status, 0, 4ull * n_chunks, st));
    // sizes are device-resident (possibly from a manifest): the kernels bound them against these capacities
    const uint32_t in_room = (uint32_t)std::min<uint64_t>(slot_stride - TSGPU_SLOT_HEAD, 0xffffffffu);
    DxBounds lim;
    lim.max_in = (uint32_t)(slot_stride - TSGPU_SLOT_HEAD);
    lim.aes_room = (flags & TSGPU_FLAG_ZSTD) ? (uint32_t)std::min<uint64_t>(c->frame_stride - 16, in_room - 28) : chunk_size;
    lim.zstd_in = (flags & TSGPU_FLAG_AES) ? (uint32_t)(c->frame_stride - 16) : in_room;
    lim.zstd_out = chunk_size;
    rc = detransform_enqueue(c, w, st, flags, n_chunks, rk, aad_len, ChunksIn{d_slots, w.dd.c_off, d_transformed_sizes},
                             ChunksOut{d_dst, w.dd.a_off, d_original_sizes}, d_status, lim, /*packed=*/false);
    if (rc) return rc;
    RT(rt::event_record(w.ev_dev_done, st));
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ profiling
extern "C" int tsgpu_profile_enable(tsgpu_ctx* c, int on) {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    std::lock_guard<std::mutex> lock(c->mu);
    c->prof.reset();
    c->prof.on = on != 0;
    return TSGPU_OK;
}
extern "C" int tsgpu_profile_report(tsgpu_ctx* c, char* out, uint32_t* out_len) {
    if (!c || !out_len) return fail(TSGPU_E_ARG, "null argument");
    std::lock_guard<std::mutex> lock(c->mu);
    for (auto& l : c->lanes) { rt::set_device(l.device); RT(rt::device_sync()); }
    std::string s = c->prof.report_json();
    if (!out || *out_len < s.size() + 1) { *out_len = (uint32_t)s.size() + 1; return fail(TSGPU_E_SHORT, "out too small"); }
    memcpy(out, s.c_str(), s.size() + 1); *out_len = (uint32_t)s.size();
    return TSGPU_OK;
}

#if ZB_TUNE_PHASES && !defined(TSGPU_SIMT)
// Measurement builds only (-DZB_TUNE_PHASES=1): the speed-mode compressor's per-block phase records of the last launch
// (ts::ZbPhases, indexed chunk * blocks_per_chunk + block), `bytes` of them from the start, into host memory.
extern "C" int tsgpu_zb_phases(void* out, uint64_t bytes) {
    if (!out || bytes > sizeof(ts::g_zb_phases)) return fail(TSGPU_E_ARG, "bad phase-record request");
    RT(rt::device_sync());
    RT(rt::err(cudaMemcpyFromSymbol(out, ts::g_zb_phases, bytes)));
    return TSGPU_OK;
}
#endif

// Which decode path the zstd frames of this context's calls took so far (summed over devices and work slots):
// out[0] regions executed in shared memory, out[1] frames a region / block handed to the frame executor, out[2] frames executed
// whole (libzstd-shaped), out[3] frames on the serial kernel, out[4] independent blocks executed by a warp each, out[5..7] 0.
// Lets tests and bench.py assert that a workload ran on the path it is supposed to measure.
extern "C" int tsgpu_decode_path_stats(tsgpu_ctx* c, uint64_t out[8]) {
    if (!c || !out) return fail(TSGPU_E_ARG, "null argument");
    std::lock_guard<std::mutex> lock(c->mu);
    for (int k = 0; k < 8; k++) out[k] = 0;
    for (auto& l : c->lanes) for (auto& w : l.w) if (w.ready && w.zdec.stats) {
        RT(rt::set_device(w.device));
        RT(rt::device_sync());
        unsigned long long v[8];
        RT(rt::d2h(v, w.zdec.stats, sizeof v, nullptr));
        RT(rt::device_sync());
        for (int k = 0; k < 8; k++) out[k] += v[k];
    }
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ ChunkIndex plumbing
extern "C" int tsgpu_chunk_positions(tsgpu_ctx* c, const uint32_t* sizes, uint32_t n, uint64_t* positions) {
    if (!c || !positions || (n && !sizes)) return fail(TSGPU_E_ARG, "null argument");
    SlotClaim claim;
    { int rcc = claim_slots(c, 1, claim); if (rcc) return rcc; }
    Work& w = *claim.slots[0];
    RT(rt::set_device(w.device));
    uint32_t* d_sizes = nullptr; uint64_t* d_pos = nullptr;
    const char* e = rt::malloc_device((void**)&d_sizes, 4ull * (n + 1));
    if (!e) e = rt::malloc_device((void**)&d_pos, 8ull * (n + 1));
    if (!e && n) e = rt::h2d(d_sizes, sizes, 4ull * n, w.stream);
    if (!e) {
        TS_LAUNCH_P(c->prof, "chunk_index_scan", chunk_index_scan_kernel, dim3(1), dim3(32), 0, w.stream, d_sizes, n, d_pos);
        e = rt::last_error();
    }
    if (!e) e = rt::d2h(positions, d_pos, 8ull * (n + 1), w.stream);
    if (!e) e = rt::stream_sync(w.stream);
    rt::free_device(d_sizes); rt::free_device(d_pos);
    if (e) return fail(TSGPU_E_CUDA, "chunk_index_scan: %s", e);
    return TSGPU_OK;
}

extern "C" int tsgpu_chunk_sizes_encode(const int32_t* v, uint32_t n, uint8_t* out, uint32_t* out_len) {
    if (!out_len || (n && !v)) return fail(TSGPU_E_ARG, "null argument");
    std::vector<uint8_t> b; tshost::Error err;
    if (!tshost::ChunkSizesBinaryCodec::encode(v, n, b, err)) return fail(TSGPU_E_ARG, "%s", err.msg.c_str());
    if (!out || *out_len < b.size()) { *out_len = (uint32_t)b.size(); return fail(TSGPU_E_SHORT, "out too small, need %zu", b.size()); }
    memcpy(out, b.data(), b.size()); *out_len = (uint32_t)b.size();
    return TSGPU_OK;
}
extern "C" int tsgpu_chunk_sizes_decode(const uint8_t* in, uint32_t in_len, int32_t* out, uint32_t* n) {
    if (!in || !n) return fail(TSGPU_E_ARG, "null argument");
    std::vector<int32_t> v; tshost::Error err;
    if (!tshost::ChunkSizesBinaryCodec::decode(in, in_len, v, err)) return fail(TSGPU_E_CORRUPT, "%s", err.msg.c_str());
    if (!out || *n < v.size()) { *n = (uint32_t)v.size(); return fail(TSGPU_E_SHORT, "out too small, need %zu", v.size()); }
    if (!v.empty()) memcpy(out, v.data(), 4 * v.size());
    *n = (uint32_t)v.size();
    return TSGPU_OK;
}

// TransformedChunksSerializer: Base64(zstd-frame(codec bytes)).  The payload is <= ~1 KiB per segment; it is
// framed on the host as a single Raw block with Frame_Content_Size, which every zstd reader (including the
// reference's TransformedChunksDeserializer) accepts and which is byte-identical to libzstd's output for the
// reference's golden vector (ChunkIndexSerializationTest.java:39).
static bool serialize_transformed_chunks(const int32_t* v, uint32_t n, std::string& out, tshost::Error& err) {
    std::vector<uint8_t> raw;
    if (!tshost::ChunkSizesBinaryCodec::encode(v, n, raw, err)) return false;
    std::vector<uint8_t> f(raw.size() + 32 + 3 * (raw.size() / 131072 + 1));
    size_t p = tshost::zstdFrameHeader(f.data(), raw.size());
    size_t off = 0;
    do {
        size_t k = std::min<size_t>(131072, raw.size() - off);
        bool last = off + k == raw.size();
        uint32_t h = (uint32_t)(last ? 1 : 0) | (0u << 1) | ((uint32_t)k << 3);
        f[p++] = (uint8_t)h; f[p++] = (uint8_t)(h >> 8); f[p++] = (uint8_t)(h >> 16);
        memcpy(f.data() + p, raw.data() + off, k); p += k; off += k;
    } while (off < raw.size());
    out = tshost::base64Encode(f.data(), p);
    return true;
}
extern "C" int tsgpu_transformed_chunks_serialize(const int32_t* v, uint32_t n, char* out, uint32_t* out_len) {
    if (!out_len || (n && !v)) return fail(TSGPU_E_ARG, "null argument");
    std::string s; tshost::Error err;
    if (!serialize_transformed_chunks(v, n, s, err)) return fail(TSGPU_E_ARG, "%s", err.msg.c_str());
    if (!out || *out_len < s.size() + 1) { *out_len = (uint32_t)s.size() + 1; return fail(TSGPU_E_SHORT, "out too small"); }
    memcpy(out, s.c_str(), s.size() + 1); *out_len = (uint32_t)s.size();
    return TSGPU_OK;
}
// TransformedChunksSerializer.java:40-48 compresses the codec bytes with libzstd before Base64; the ctx-taking form does the
// same with this library's dense compressor (one frame with Frame_Content_Size, the codec bytes as ONE chunk) and keeps
// whichever of {compressed frame, Raw-block frame} is shorter — so manifests of segments whose chunk sizes repeat or cluster
// are as small as the reference's instead of carrying the bit-packed list verbatim.
static int serialize_transformed_chunks_ctx(tsgpu_ctx* c, const int32_t* v, uint32_t n, std::string& out) {
    tshost::Error err;
    if (!serialize_transformed_chunks(v, n, out, err)) return fail(TSGPU_E_ARG, "%s", err.msg.c_str());
    std::vector<uint8_t> raw;
    if (!tshost::ChunkSizesBinaryCodec::encode(v, n, raw, err)) return fail(TSGPU_E_ARG, "%s", err.msg.c_str());
    if (raw.size() < 64 || raw.size() > c->chunk_cap) return TSGPU_OK;          // nothing to gain / larger than the context's chunks
    const uint32_t fl = TSGPU_FLAG_ZSTD | TSGPU_FLAG_ZSTD_DENSE;
    std::vector<uint8_t> z((size_t)tsgpu_transform_bound(fl, raw.size(), 0) + 64);
    uint32_t tsz = 0, nch = 1;
    const int rc = tsgpu_transform(c, fl, raw.data(), raw.size(), 0, nullptr, nullptr, 0, nullptr, z.data(), z.size(), &tsz, &nch);
    if (rc) return rc;
    if (nch == 1 && tsz) {
        std::string b = tshost::base64Encode(z.data(), tsz);
        if (b.size() < out.size()) out.swap(b);
    }
    return TSGPU_OK;
}
extern "C" int tsgpu_transformed_chunks_serialize_ctx(tsgpu_ctx* c, const int32_t* v, uint32_t n, char* out, uint32_t* out_len) try {
    if (!c || !out_len || (n && !v)) return fail(TSGPU_E_ARG, "null argument");
    std::string s;
    if (int rc = serialize_transformed_chunks_ctx(c, v, n, s)) return rc;
    if (!out || *out_len < s.size() + 1) { *out_len = (uint32_t)s.size() + 1; return fail(TSGPU_E_SHORT, "out too small"); }
    memcpy(out, s.c_str(), s.size() + 1); *out_len = (uint32_t)s.size();
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }
extern "C" int tsgpu_transformed_chunks_deserialize(tsgpu_ctx* c, const char* b64, int32_t* out, uint32_t* n) {
    if (!c || !b64 || !n) return fail(TSGPU_E_ARG, "null argument");
    std::vector<uint8_t> z; tshost::Error err;
    if (!tshost::base64Decode(b64, z, err)) return fail(TSGPU_E_CORRUPT, "%s", err.msg.c_str());
    // the frame may come from the reference (libzstd-compressed): decode it with the GPU zstd decoder
    const uint32_t cap = 10u * 1024 * 1024;                  // TransformedChunksDeserializer.java:33 sanity cap
    std::vector<uint8_t> raw(std::min<uint64_t>(cap, c->chunk_cap));
    uint32_t tsz = (uint32_t)z.size(), osz = 0;
    int rc = tsgpu_detransform(c, TSGPU_FLAG_ZSTD, z.data(), z.size(), &tsz, 1, nullptr, nullptr, 0, raw.data(), raw.size(), &osz);
    if (rc) return rc;
    std::vector<int32_t> v;
    if (!tshost::ChunkSizesBinaryCodec::decode(raw.data(), osz, v, err)) return fail(TSGPU_E_CORRUPT, "%s", err.msg.c_str());
    if (!out || *n < v.size()) { *n = (uint32_t)v.size(); return fail(TSGPU_E_SHORT, "out too small, need %zu", v.size()); }
    if (!v.empty()) memcpy(out, v.data(), 4 * v.size());
    *n = (uint32_t)v.size();
    return TSGPU_OK;
}

static int chunk_index_json_impl(tsgpu_ctx* c, int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, const int32_t* sizes, uint32_t n,
                                 char* out, uint32_t* out_len);
extern "C" int tsgpu_chunk_index_json(int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, const int32_t* sizes, uint32_t n,
                                      char* out, uint32_t* out_len) {
    return chunk_index_json_impl(nullptr, ocs, ofs, tcs, ftcs, sizes, n, out, out_len);
}
extern "C" int tsgpu_chunk_index_json_ctx(tsgpu_ctx* c, int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, const int32_t* sizes, uint32_t n,
                                          char* out, uint32_t* out_len) try {
    if (!c) return fail(TSGPU_E_ARG, "null argument");
    return chunk_index_json_impl(c, ocs, ofs, tcs, ftcs, sizes, n, out, out_len);
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }
static int chunk_index_json_impl(tsgpu_ctx* c, int32_t ocs, int32_t ofs, int32_t tcs, int32_t ftcs, const int32_t* sizes, uint32_t n,
                                 char* out, uint32_t* out_len) {
    if (!out_len) return fail(TSGPU_E_ARG, "null argument");
    if (ocs <= 0) return fail(TSGPU_E_ARG, "Original chunk size must be positive, %d given", ocs);
    if (ofs < 0) return fail(TSGPU_E_ARG, "Original file size must be non-negative, %d given", ofs);
    std::string s;
    char buf[256];
    if (tcs >= 0) {
        if (ftcs < 0) return fail(TSGPU_E_ARG, "Final transformed chunk size must be non-negative, %d given", ftcs);
        snprintf(buf, sizeof buf, "{\"type\":\"fixed\",\"originalChunkSize\":%d,\"originalFileSize\":%d,"
                                  "\"transformedChunkSize\":%d,\"finalTransformedChunkSize\":%d}", ocs, ofs, tcs, ftcs);
        s = buf;
    } else {
        if (!sizes || n == 0) return fail(TSGPU_E_ARG, "transformedChunks cannot be null");
        std::string b64; tshost::Error err;
        if (c) { if (int rc = serialize_transformed_chunks_ctx(c, sizes, n, b64)) return rc; }
        else if (!serialize_transformed_chunks(sizes, n, b64, err)) return fail(TSGPU_E_ARG, "%s", err.msg.c_str());
        snprintf(buf, sizeof buf, "{\"type\":\"variable\",\"originalChunkSize\":%d,\"originalFileSize\":%d,\"transformedChunks\":\"", ocs, ofs);
        s = std::string(buf) + b64 + "\"}";
    }
    if (!out || *out_len < s.size() + 1) { *out_len = (uint32_t)s.size() + 1; return fail(TSGPU_E_SHORT, "out too small"); }
    memcpy(out, s.c_str(), s.size() + 1); *out_len = (uint32_t)s.size();
    return TSGPU_OK;
}
