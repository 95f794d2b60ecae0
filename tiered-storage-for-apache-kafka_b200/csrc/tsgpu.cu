// tsgpu.cu — libtsgpu.so: context, batch scheduling, C-ABI (include/tsgpu.h).
// Device code lives in the .cuh headers next to this file; this translation unit owns launches and copies.
//
// Host pipeline of tsgpu_transform (one segment):
//   split into batches of <= max_batch chunks -> dealt round-robin to (device, work-slot) pairs, each with its
//   own stream, device arenas and pinned descriptor block -> per batch: H2D original bytes, [zstd kernels],
//   [AES-GCM kernels], D2H of the chunk sizes, then per-chunk D2H of exactly transformed_size bytes to the
//   running offset in dst (the packed .log object layout, SURVEY.md appendix A.1).  Batches complete in order;
//   up to (devices x slots) batches are in flight so copies overlap kernels.  With TSGPU_FLAG_VERIFY each batch is
//   detransformed on the device and compared with its input before any of its bytes are copied out.  With
//   TSGPU_FLAG_VALIDATE_RECORDS the Kafka log entries of each batch are checked on the device (records.cuh) and the batch's
//   verdict is resolved, in batch order, before its bytes are copied out.  tsgpu_transform_parts also hashes each packed batch
//   (part_crc.cuh) and combines the CRC-32C of the object's upload parts on the host once the call's streams are idle;
//   tsgpu_transform_parts_crc64 does the same with CRC-64/NVME (one source, instantiated for each CRC word).
#include <algorithm>
#include <array>
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
#include "records.cuh"
#include "part_crc.cuh"
#include "rt.h"
#include "launch_prof.h"
#include "zstd_enc.cuh"
#include "zstd_enc_blk.cuh"
#include "zstd_dec.cuh"
#include "reframe.cuh"
#include "frame_walk.cuh"
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
// Largest frame of an n-byte chunk, in either mode: a header of at most 10 bytes, at most ceil(n / 8 KiB) blocks of 3 header bytes
// + at most 8 KiB each (a block that would not shrink goes out Raw), and the 4-byte Content_Checksum with
// TSGPU_FLAG_ZSTD_CHECKSUM: n + 3 ceil(n / 8192) + 14 <= n + 3 n / 8192 + 17.  As n >> 8 >= n / 256 - 1 = 32 n / 8192 - 1, the
// bound below exceeds that by at least 29 n / 8192 + 46 > 0 bytes for every n, with or without the checksum.
static inline uint64_t frame_bound(uint64_t n) { return n + (n >> 8) + 64; }

// ------------------------------------------------------------------------------------------ context
namespace {

constexpr int NSLOT_MAX = 16;       // work slots per device; tsgpu_ctx::nslot of them are used
constexpr uint32_t MAX_AAD = 4096;
constexpr uint32_t KNOWN_FLAGS = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES | TSGPU_FLAG_ZSTD_DENSE | TSGPU_FLAG_ZSTD_CHECKSUM;
constexpr uint32_t ZSTD_MODIFIERS = TSGPU_FLAG_ZSTD_DENSE | TSGPU_FLAG_ZSTD_CHECKSUM;   // how to compress: the reader ignores them

struct Desc {            // device-side descriptor block of one work slot (all arrays sized for max_batch)
    uint64_t* a_off; uint64_t* b_off; uint64_t* c_off;
    uint32_t* a_len; uint32_t* b_len; uint32_t* c_len; uint32_t* status;
    uint32_t* v_len; uint32_t* v_diff;     // TSGPU_FLAG_VERIFY: read-back sizes, first differing byte per chunk
    uint8_t* ivs; uint8_t* aad;
};

// Pinned read-back block of one work slot (arrays sized for max_batch): what a drained batch reads on the host.
struct Back {
    uint32_t* sizes;         // sizes of what the batch copies out
    uint32_t* status;        // per chunk: the verify stage's status, or the detransform's tag / frame status
    uint32_t* diff;          // TSGPU_FLAG_VERIFY: first differing byte per chunk
    uint32_t* src_sizes;     // the source half (source_stage): decoded sizes
    uint32_t* src_status;    //   ... their tag / frame statuses
    uint64_t* words;         //   ... the object and segment CRC words, as W[2] for either CRC word W
};

// Device arrays of the record validation of one slot (records.cuh), sized for batches of up to `cap` bytes.
struct RecScratch {
    uint8_t* d = nullptr;
    uint64_t cap = 0;
    RecArgs a{};                   // the batch last enqueued on the slot: rec_resolve reads the same arrays at its drain
    RecOut* d_out = nullptr;
    RecOut* h_out = nullptr;       // pinned
};

// Device arrays of the upload-part checksums of one slot (part_crc.cuh), sized for batches of up to `cap` packed bytes, for one
// CRC word W (uint32_t: CRC-32C, uint64_t: CRC-64/NVME).
template <typename W> struct PcrcScratch {
    uint8_t* d = nullptr;
    uint64_t cap = 0;
    PcrcArgs<W> a{};               // the batch last enqueued on the slot: pcrc_cuts reads the same arrays at its drain
    W* d_cuts = nullptr;           // pcrc_cuts output and its pinned copy, cuts_cap words
    W* h_cuts = nullptr;
    uint32_t cuts_cap = 0;
    int32_t pending = -1;          // the call's batch whose prefixes h_cuts receives (collected at the slot's next drain or at the end)
};

// One AES-GCM key of a slot: the key tables (H powers, Shoup table) of the last key it ran, so consecutive calls with one
// segment's data key skip the set-up kernel, and the AAD the GCM kernels read.
struct GcmKeys {
    Aes256RoundKeys rk{};          // the key `ctx` was built for
    bool valid = false;
    GcmKeyCtx* ctx = nullptr;
    uint8_t* d_aad = nullptr;      // [0]: the descriptor block's; [1]: its own MAX_AAD bytes, uploaded from h_aad (pinned)
    uint8_t* h_aad = nullptr;
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
    GcmKeys keys[2];               // [0] every call's; [1] the new key of tsgpu_rewrite_object / tsgpu_rekey_object (allocated on first use)
    uint8_t* d_orig = nullptr;     // max_batch * chunk_cap
    uint8_t* d_frames = nullptr;   // max_batch * frame_stride        (zstd frames, 16-byte aligned slots)
    uint8_t* d_xf = nullptr;       // max_batch * slot_stride         (transformed slots)
    uint8_t* d_pack = nullptr;     // max_batch * slot_stride         (transformed chunks back to back: what one D2H takes home)
    uint8_t* d_desc = nullptr;  uint8_t* h_desc = nullptr;  size_t desc_bytes = 0;
    Desc dd{}, hd{};               // device / pinned-host views of the descriptor block
    uint4* d_partials = nullptr;  uint32_t max_ranges = 0;   // 2 * max_ranges * max_batch: [0] every GCM stage's, [1] the rekey's new key
    ZstdEncScratch zenc{};         // region kernel (TSGPU_FLAG_ZSTD_DENSE), allocated on first use
    ZstdBlkScratch zblk{};         // block kernel (default), allocated on first use
    ZstdDecScratch zdec{};
    uint8_t* h_back = nullptr;  size_t back_bytes = 0;
    Back back{};                   // views of h_back
    RecScratch rec{};              // TSGPU_FLAG_VALIDATE_RECORDS, allocated on first use
    PcrcScratch<uint32_t> pcrc{};  // CRC-32C part and object checksums, allocated on first use
    PcrcScratch<uint64_t> pcrc64{};   // CRC-64/NVME (the _crc64 calls), allocated on first use
};
template <typename W> PcrcScratch<W>& pcrc_of(Work& w) {
    if constexpr (sizeof(W) == 8) return w.pcrc64;
    else return w.pcrc;
}

struct Lane { int device = 0; Work w[NSLOT_MAX]; };

}  // namespace

struct tsgpu_ctx {
    bool dense_default = false;    // TSGPU_ZSTD_MODE=dense: TSGPU_FLAG_ZSTD alone already means the region kernel
    bool verify_default = false;   // TSGPU_VERIFY=1: host-buffer transforms verify as if TSGPU_FLAG_VERIFY were set
    bool checksum_default = false; // TSGPU_ZSTD_CHECKSUM=1: every frame carries its Content_Checksum, as with TSGPU_FLAG_ZSTD_CHECKSUM
    bool records_default = false;  // TSGPU_VALIDATE_RECORDS=1: tsgpu_transform_cursor calls with ZSTD or AES validate their record batches
    std::mutex mu;                 // guards slot ownership (Work::claimed, active_calls) and lazy slot allocation — NOT held while a call runs
    std::condition_variable cv;
    uint32_t active_calls = 0;
    std::vector<Lane> lanes;
    uint32_t chunk_cap = 0, max_batch = 0;
    uint64_t frame_stride = 0, slot_stride = 0;
    LaunchProf prof;
    uint32_t nslot = 16;           // work slots per device (TSGPU_SLOTS overrides); one call takes at most 8 of them
};

struct Carver {                 // consecutive 256-byte aligned pieces of a block at `base` (nullptr: only adds up its size, p)
    uint8_t* base; size_t p = 0;
    template <typename T> T* take(size_t n) { T* r = base ? (T*)(base + p) : nullptr; p += align_up(sizeof(T) * n, 256); return r; }
};

static size_t carve_desc(uint8_t* base, uint32_t nb, Desc& d) {
    Carver k{base};
    d.a_off = k.take<uint64_t>(nb); d.b_off = k.take<uint64_t>(nb); d.c_off = k.take<uint64_t>(nb + 1);
    d.a_len = k.take<uint32_t>(nb); d.b_len = k.take<uint32_t>(nb); d.c_len = k.take<uint32_t>(nb);
    d.status = k.take<uint32_t>(nb); d.v_len = k.take<uint32_t>(nb); d.v_diff = k.take<uint32_t>(nb);
    d.ivs = k.take<uint8_t>(12ull * nb); d.aad = k.take<uint8_t>(MAX_AAD);
    return k.p;
}

static size_t carve_back(uint8_t* base, uint32_t nb, Back& b) {
    Carver k{base};
    b.sizes = k.take<uint32_t>(nb); b.status = k.take<uint32_t>(nb); b.diff = k.take<uint32_t>(nb);
    b.src_sizes = k.take<uint32_t>(nb); b.src_status = k.take<uint32_t>(nb); b.words = k.take<uint64_t>(2);
    return k.p;
}

// The frame and transformed slots of nb chunks in a descriptor block (the device calls pass their caller's slot_stride).
static void slot_layout(const tsgpu_ctx* c, Desc& d, uint32_t nb, uint64_t slot_stride) {
    for (uint32_t i = 0; i < nb; i++) { d.b_off[i] = (uint64_t)i * c->frame_stride; d.c_off[i] = (uint64_t)i * slot_stride + TSGPU_SLOT_HEAD; }
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
    w.desc_bytes = carve_desc(nullptr, c->max_batch, w.dd);
    RT(rt::malloc_device((void**)&w.d_desc, w.desc_bytes));
    RT(rt::malloc_host((void**)&w.h_desc, w.desc_bytes));
    carve_desc(w.d_desc, c->max_batch, w.dd);
    carve_desc(w.h_desc, c->max_batch, w.hd);
    w.back_bytes = carve_back(nullptr, c->max_batch, w.back);
    RT(rt::malloc_host((void**)&w.h_back, w.back_bytes));
    carve_back(w.h_back, c->max_batch, w.back);
    w.max_ranges = (uint32_t)((frame_bound(c->chunk_cap) / 16 + GH_RANGE_BLOCKS) / GH_RANGE_BLOCKS) + 1;
    RT(rt::malloc_device((void**)&w.d_partials, 2 * sizeof(uint4) * (size_t)w.max_ranges * nb));   // the rekey takes two sets
    RT(rt::malloc_device((void**)&w.keys[0].ctx, sizeof(GcmKeyCtx)));
    w.keys[0].d_aad = w.dd.aad;
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
    rt::free_device(w.d_partials); rt::free_device(w.keys[0].ctx); rt::free_host(w.h_back);
    rt::free_device(w.keys[1].ctx); rt::free_device(w.keys[1].d_aad); rt::free_host(w.keys[1].h_aad);
    zstd_enc_scratch_free(w.zenc); zstd_blk_scratch_free(w.zblk); zstd_dec_scratch_free(w.zdec);
    rt::free_device(w.rec.d); rt::free_device(w.rec.d_out); rt::free_host(w.rec.h_out); w.rec = RecScratch{};
    rt::free_device(w.pcrc.d); rt::free_device(w.pcrc.d_cuts); rt::free_host(w.pcrc.h_cuts); w.pcrc = PcrcScratch<uint32_t>{};
    rt::free_device(w.pcrc64.d); rt::free_device(w.pcrc64.d_cuts); rt::free_host(w.pcrc64.h_cuts); w.pcrc64 = PcrcScratch<uint64_t>{};
    for (GcmKeys& k : w.keys) k = GcmKeys{};                // forgets the keys too
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
    if (const char* e = getenv("TSGPU_ZSTD_CHECKSUM")) c->checksum_default = strcmp(e, "1") == 0;
    if (const char* e = getenv("TSGPU_VALIDATE_RECORDS")) c->records_default = strcmp(e, "1") == 0;
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
        if (!e) e = rt::allow_smem(gcm_rekey_kernel, GCM_REKEY_SMEM_BYTES);
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
// With the checksum either kernel also hashes every chunk, in extra CTAs of the same launch, and ends its frame with it.
static int zstd_stage_modes(tsgpu_ctx* c, Work& w, rt::stream_t st, bool dense, bool checksum, ChunksIn in, uint32_t nb, uint32_t cs,
                            ChunksOut out) {
    int rc;
    if (dense) {
        if (!w.zenc.seqs) {
            const char* e = zstd_enc_scratch_alloc(w.zenc, c->chunk_cap, c->max_batch);
            if (e) { zstd_enc_scratch_free(w.zenc); return fail(TSGPU_E_CUDA, "zstd enc scratch: %s", e); }
        }
        rc = zstd_compress_batch(w.zenc, st, in.base, in.off, in.len, nb, cs, checksum, out.base, out.off, out.len, c->prof);
    } else {
        if (!w.zblk.seqs) {
            const char* e = zstd_blk_scratch_alloc(w.zblk, c->chunk_cap, c->max_batch);
            if (e) { zstd_blk_scratch_free(w.zblk); return fail(TSGPU_E_CUDA, "zstd enc scratch: %s", e); }
        }
        rc = zstd_compress_batch_blocks(w.zblk, st, in.base, in.off, in.len, nb, cs, checksum, out.base, out.off, out.len, c->prof);
    }
    if (rc) return fail(rc, "zstd compress: %s", zstd_last_error());
    return TSGPU_OK;
}
// The modifiers of `flags`, or the context's defaults.
static int zstd_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t flags, ChunksIn in, uint32_t nb, uint32_t cs, ChunksOut out) {
    return zstd_stage_modes(c, w, st, (flags & TSGPU_FLAG_ZSTD_DENSE) || c->dense_default,
                            (flags & TSGPU_FLAG_ZSTD_CHECKSUM) || c->checksum_default, in, nb, cs, out);
}

// AES-GCM: key set-up, the main kernel over (ranges x chunks) and the finalize kernel.  IVs (ENC) come from the slot's
// descriptor block, the AAD from `k`.  The slot keeps the key tables of the last key each of its GcmKeys ran: consecutive calls
// with one segment's data key skip the set-up kernel.  Host and device calls share slot 0's tables; that is safe because device
// calls are ordered behind each other by events (dev_call_begin) and a host call takes the slot only once device work on it has
// completed.
// The key tables of `rk` in k.ctx: the set-up kernel unless they are there already.  k.valid stays false until the caller has
// enqueued the kernels that read them.
static int gcm_key_tables(tsgpu_ctx* c, GcmKeys& k, rt::stream_t st, const Aes256RoundKeys& rk) {
    const bool key_ready = k.valid && memcmp(&k.rk, &rk, sizeof rk) == 0;
    k.rk = rk; k.valid = false;                              // valid again once the whole stage has been enqueued
    if (!key_ready) {
        TS_LAUNCH_P(c->prof, "gcm_key_setup", gcm_key_setup_kernel, dim3(1), dim3(GH_T), 0, st, rk, k.ctx);
        CHECK_LAUNCH("gcm_key_setup_kernel");
    }
    return TSGPU_OK;
}

template <bool ENC>
static int gcm_stage(tsgpu_ctx* c, Work& w, GcmKeys& k, rt::stream_t st, const Aes256RoundKeys& rk, ChunksIn in, ChunksOut out,
                     uint32_t aad_len, uint32_t* d_status, uint32_t n_chunks, uint32_t max_payload, uint32_t out_cap) {
    { int rc = gcm_key_tables(c, k, st, rk); if (rc) return rc; }
    GcmBatch B;
    B.in_base = in.base; B.in_off = in.off; B.in_len = in.len;
    B.out_base = out.base; B.out_off = out.off; B.out_len = out.len;
    B.ivs = ENC ? w.dd.ivs : nullptr; B.aad = k.d_aad; B.aad_len = aad_len;
    B.partials = w.d_partials; B.max_ranges = w.max_ranges; B.status = d_status; B.n_chunks = n_chunks; B.out_cap = out_cap;
    uint32_t ranges = (uint32_t)(((uint64_t)max_payload + 15) / 16 + GH_RANGE_BLOCKS - 1) / GH_RANGE_BLOCKS;
    if (ranges > w.max_ranges) return fail(TSGPU_E_ARG, "chunk too large for this context");
    if (ranges) {
        TS_LAUNCH_P(c->prof, ENC ? "gcm_main_enc" : "gcm_main_dec", gcm_main_kernel<ENC>, dim3(ranges, n_chunks), dim3(GH_T),
                    GCM_SMEM_BYTES, st, rk, k.ctx, B);
        CHECK_LAUNCH("gcm_main_kernel");
    }
    TS_LAUNCH_P(c->prof, ENC ? "gcm_finalize_enc" : "gcm_finalize_dec", gcm_finalize_kernel<ENC>, dim3((n_chunks + 3) / 4),
                dim3(128), 0, st, rk, k.ctx, B);
    CHECK_LAUNCH("gcm_finalize_kernel");
    k.valid = true;
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
static int transform_enqueue(tsgpu_ctx* c, Work& w, GcmKeys& k, rt::stream_t st, uint32_t flags, uint32_t nb, uint32_t cs,
                             const Aes256RoundKeys& rk, uint32_t aad_len, ChunksIn src, ChunksOut dst) {
    const bool aes = flags & TSGPU_FLAG_AES;
    uint32_t max_payload = cs;
    if (flags & TSGPU_FLAG_ZSTD) {
        const ChunksOut frames = aes ? ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len} : dst;
        int rc = zstd_stage(c, w, st, flags, src, nb, cs, frames);
        if (rc) return rc;
        src = frames; max_payload = (uint32_t)frame_bound(cs);
    }
    if (aes) return gcm_stage<true>(c, w, k, st, rk, src, dst, aad_len, w.dd.status, nb, max_payload, 0xffffffffu);
    return TSGPU_OK;
}

// [AES-GCM decrypt ->] [zstd]: nb chunks from `src` into `dst`.  packed: dst.off is written on the device as the running sum
// of the original sizes (chunks back to back) instead of being read as given.
static int detransform_enqueue(tsgpu_ctx* c, Work& w, GcmKeys& k, rt::stream_t st, uint32_t flags, uint32_t nb, const Aes256RoundKeys& rk,
                               uint32_t aad_len, ChunksIn src, ChunksOut dst, uint32_t* d_status, const DxBounds& lim, bool packed) {
    const bool zstd = flags & TSGPU_FLAG_ZSTD;
    if (flags & TSGPU_FLAG_AES) {
        const ChunksOut plain = zstd ? ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len} : dst;
        if (!zstd) { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }                        // dst is the final buffer
        int rc = gcm_stage<false>(c, w, k, st, rk, src, plain, aad_len, d_status, nb, lim.max_in, lim.aes_room);
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
// Chunks [c0, c0 + nb) of a call, in flight on slot w; in_off: chunk c0's byte offset in the call's transformed input.
struct Batch { Work* w; uint32_t c0, nb; uint64_t in_off; };
}

// Cuts n chunks into batches of max_batch and deals them round-robin over the slots it claims.  issue(batch) enqueues a
// batch on its slot's stream and ends with the D2H of its sizes (ev_sizes); drain(batch) runs once those sizes are on the
// host, in batch order, and sends the batch's bytes home (copy_out).  idle(slots, rc) runs once every claimed slot is idle,
// before the slots are given back.  Returns with every claimed slot idle.  `tsizes`: the transformed sizes of the n chunks of
// a call that reads transformed chunks (Batch::in_off), else nullptr.
namespace { struct NoIdle { int operator()(const std::vector<Work*>&, int rc) const { return rc; } }; }
template <class Issue, class Drain, class Idle = NoIdle>
static int run_batches(tsgpu_ctx* c, uint32_t n, const uint32_t* tsizes, Issue issue, Drain drain, Idle idle = Idle()) {
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
    uint64_t in_off = 0;
    for (uint32_t b = 0; b < nbatches && rc == TSGPU_OK; b++) {
        // From b = nwork on a slot is reused: its previous batch is drained first (sizes read on the host, copies-out
        // enqueued on the slot's out_stream); the new batch's copy-in and first kernels start right away and only the
        // kernel that overwrites the buffer being copied out waits for those copies (wait_copies_out) — the host never
        // waits here, which keeps all slots' queues full.
        if (b >= nwork) { rc = drain_next(); if (rc) break; }
        const uint32_t c0 = b * c->max_batch;
        inflight[b] = Batch{claim.slots[b % nwork], c0, std::min(c->max_batch, n - c0), in_off};
        if (tsizes) for (uint32_t i = 0; i < inflight[b].nb; i++) in_off += tsizes[c0 + i];
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
    return idle(claim.slots, rc);
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
// `payload`: the largest transformed chunk without IV and tag.
static int verify_stage(tsgpu_ctx* c, Work& w, GcmKeys& k, rt::stream_t st, uint32_t flags, uint32_t nb, uint32_t cs, uint64_t payload,
                        const Aes256RoundKeys& rk, uint32_t aad_len, ChunksOut fin) {
    const bool zstd = flags & TSGPU_FLAG_ZSTD;
    RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
    RT(rt::memset_async(w.dd.v_diff, 0xff, 4ull * nb, st));
    DxBounds lim;
    lim.max_in = (uint32_t)(payload + TSGPU_IV_SIZE + TSGPU_TAG_SIZE);
    lim.aes_room = zstd ? (uint32_t)(c->frame_stride - 16) : c->chunk_cap;
    lim.zstd_in = (uint32_t)(c->frame_stride - 16);
    lim.zstd_out = cs;                                        // a frame claiming more than the batch's largest chunk is wrong
    const ChunksOut back{zstd ? w.d_xf : w.d_frames, w.dd.b_off, w.dd.v_len};
    { int rc = detransform_enqueue(c, w, k, st, flags & (TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES), nb, rk, aad_len, fin, back, w.dd.status,
                                   lim, /*packed=*/false); if (rc) return rc; }
    VerifyArgs V;
    V.orig = w.d_orig; V.orig_off = w.dd.a_off; V.orig_len = w.dd.a_len;
    V.back = back.base; V.back_off = back.off; V.back_len = back.len;
    V.status = w.dd.status; V.diff = w.dd.v_diff;
    TS_LAUNCH_P(c->prof, "verify_compare", verify_compare_kernel, dim3((cs + VERIFY_PIECE - 1) / VERIFY_PIECE, nb), dim3(VERIFY_T), 0, st, V);
    CHECK_LAUNCH("verify_compare_kernel");
    return TSGPU_OK;
}

// ------------------------------------------------------------------------------------------ record validation
// Largest batch the validation indexes: positions are 31-bit (node indices carry a terminal bit).
constexpr uint64_t REC_MAX_BATCH = 0x7fffff00ull;

static int records_alloc(RecScratch& r, uint64_t L) {
    if (r.cap >= L) return TSGPU_OK;
    rt::free_device(r.d); r.d = nullptr; r.cap = 0;
    const uint64_t np = (L + REC_PIECE - 1) / REC_PIECE, nt = (L + REC_TILE - 1) / REC_TILE;
    const uint64_t sz[7] = {8 * np, 8 * nt, 8 * nt, 4 * nt, 4 * (nt + 1), 4 * L, 8 * L};
    uint64_t total = 0;
    for (uint64_t b : sz) total += align_up(b, 256);
    RT(rt::malloc_device((void**)&r.d, total));
    if (!r.d_out) RT(rt::malloc_device((void**)&r.d_out, sizeof(RecOut)));
    if (!r.h_out) RT(rt::malloc_host((void**)&r.h_out, sizeof(RecOut)));
    uint8_t* p = r.d;
    auto take = [&](uint64_t b) { uint8_t* q = p; p += align_up(b, 256); return q; };
    r.a.pin = (uint32_t*)take(sz[0]); r.a.ttot = (uint32_t*)take(sz[1]); r.a.tex = (uint32_t*)take(sz[2]);
    r.a.cnt = (uint32_t*)take(sz[3]); r.a.tbase = (uint32_t*)take(sz[4]); r.a.cpos = (uint32_t*)take(sz[5]);
    r.a.node = (unsigned long long*)take(sz[6]);
    r.cap = L;
    return TSGPU_OK;
}

// Enqueues the validation of the batch's L original bytes in d_orig: every kernel but the resolve, which waits for the drain.
static int records_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, uint64_t L) {
    RecArgs& a = w.rec.a;
    a.b = w.d_orig; a.L = (uint32_t)L;
    a.npieces = (uint32_t)((L + REC_PIECE - 1) / REC_PIECE); a.ntiles = (uint32_t)((L + REC_TILE - 1) / REC_TILE);
    TS_LAUNCH_P(c->prof, "rec_scan", rec_scan_kernel, dim3(a.ntiles), dim3(REC_T), 0, st, a);
    CHECK_LAUNCH("rec_scan_kernel");
    TS_LAUNCH_P(c->prof, "rec_tiles", rec_tiles_kernel, dim3(1), dim3(REC_TILES_T), 0, st, a);
    CHECK_LAUNCH("rec_tiles_kernel");
    TS_LAUNCH_P(c->prof, "rec_place", rec_place_kernel, dim3(a.ntiles), dim3(REC_T), 0, st, a);
    CHECK_LAUNCH("rec_place_kernel");
    const uint32_t grid = (uint32_t)std::min<uint64_t>(264, (L + 16383) / 16384);
    TS_LAUNCH_P(c->prof, "rec_link", rec_link_kernel, dim3(grid), dim3(REC_LINK_T), 0, st, a);
    CHECK_LAUNCH("rec_link_kernel");
    for (uint64_t reach = 1; reach < L; reach *= REC_JUMPS + 1) {       // at most L candidates; every launch multiplies the reach
        TS_LAUNCH_P(c->prof, "rec_jump", rec_jump_kernel, dim3(grid), dim3(REC_LINK_T), 0, st, a);
        CHECK_LAUNCH("rec_jump_kernel");
    }
    return TSGPU_OK;
}

static int records_failure(const RecOut& o) {
    const unsigned long long at = (unsigned long long)o.fail;
    switch (o.kind) {
    case REC_MAGIC:
        return fail(TSGPU_E_RECORDS, "Record batch is corrupt (check: magic): the entry at segment position %llu has magic %u, not 0, 1 or 2", at, o.magic);
    case REC_LENGTH:
        return fail(TSGPU_E_RECORDS, "Record batch is corrupt (check: length): the entry at segment position %llu does not fit: size %d, "
                    "below the minimum for its magic or past the end of the segment", at, o.size);
    case REC_CRC:
        return fail(TSGPU_E_RECORDS, "Record is corrupt (stored crc = %u, computed crc = %u) (check: crc): the entry at segment position %llu",
                    o.stored, o.computed, at);
    default:
        return fail(TSGPU_E_CUDA, "record validation did not resolve the entry at segment position %llu", at);
    }
}

// The drained batch's verdict, in batch order: the carry of the batches before it goes in, its own comes out.
static int records_resolve(tsgpu_ctx* c, Work& w, RecCarry& carry) {
    TS_LAUNCH_P(c->prof, "rec_resolve", rec_resolve_kernel, dim3(1), dim3(32), 0, w.stream, w.rec.a, carry, w.rec.d_out);
    CHECK_LAUNCH("rec_resolve_kernel");
    RT(rt::d2h(w.rec.h_out, w.rec.d_out, sizeof(RecOut), w.stream));
    RT(rt::stream_sync(w.stream));
    if (w.rec.h_out->kind != REC_OK) return records_failure(*w.rec.h_out);
    carry = w.rec.h_out->carry;
    return TSGPU_OK;
}

// A segment that ends inside an entry: the entry is too long for it (or, with its magic byte there, has a bad one).
static int records_segment_end(const RecCarry& carry) {
    if (!carry.open) return TSGPU_OK;
    RecOut o{};
    o.fail = carry.start; o.kind = REC_LENGTH;
    o.size = carry.hlen >= 12 ? (int32_t)((uint32_t)carry.hdr[8] << 24 | (uint32_t)carry.hdr[9] << 16 | (uint32_t)carry.hdr[10] << 8 | carry.hdr[11]) : 0;
    if (carry.hlen > 16) { o.magic = carry.hdr[16]; if (o.magic > 2) o.kind = REC_MAGIC; }
    return records_failure(o);
}

// ------------------------------------------------------------------------------------------ upload-part checksums
// The state of an object between calls: the public tsgpu_parts_cursor (32 bytes, zero = start of the object).  The two raw CRCs
// take 8 of the last 16 bytes with CRC-32C (the other 8 are reserved) and all 16 with CRC-64/NVME.
template <typename W> struct PartsCarry {
    uint64_t obj_len;      // object bytes so far
    uint64_t part_size;    // the segment's part size (checked against every later call)
    W raw[16 / sizeof(W)]; // [0]: raw CRC of the open part's bytes (obj_len % part_size of them); [1]: of the object so far
};
static_assert(sizeof(PartsCarry<uint32_t>) == sizeof(tsgpu_parts_cursor) && sizeof(PartsCarry<uint64_t>) == sizeof(tsgpu_parts_cursor),
              "the cursor holds the carry");

// Names of the checksum arguments in messages.
template <typename W> constexpr const char* crc_arg() { return sizeof(W) == 8 ? "crc64" : "crc32c"; }

// One batch of a tsgpu_transform_parts call, L packed bytes: words[k] is the raw CRC of [0, x_k) of the batch,
// x_k = first + k * part_size for k < m (the part boundaries strictly inside it), x_m = L.
template <typename W> struct PcrcBatch { uint32_t L = 0, first = 0, m = 0; std::vector<W> words; };
// The part-checksum arguments of tsgpu_transform_parts, tsgpu_rewrite_object and their _crc64 twins.
template <typename W> struct PartsReq {
    uint64_t part_size; tsgpu_parts_cursor* cursor;
    W* crcs; uint32_t cap; uint32_t* n; W* object_crc;
};
// The part checksums of one call.  Its entry point takes it through parts_begin, then parts_drain at each batch's drain
// (target_drain), parts_idle once the call's slots are idle, and parts_finish after a successful call.
template <typename W> struct PartsRun {
    PartsReq<W> q{};
    PartsCarry<W> cur{};                  // the cursor as the call found it
    std::vector<PcrcBatch<W>> batches;    // by batch index, as they drain
};

// The part-checksum arguments, checked before any GPU work, and the cursor.  `bound`: the most bytes the call can add to the object.
template <typename W>
static int parts_begin(PartsRun<W>& run, const PartsReq<W>& q, uint32_t flags, uint64_t bound, int segment_ends_here) {
    if (!(flags & (TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES)))
        return fail(TSGPU_E_ARG, "%s needs TSGPU_FLAG_ZSTD or TSGPU_FLAG_AES: without them no byte reaches the GPU",
                    sizeof(W) == 8 ? "tsgpu_transform_parts_crc64" : "tsgpu_transform_parts");
    if (q.part_size == 0) return fail(TSGPU_E_ARG, "part_size must be at least 1");
    if (!q.cursor || !q.n || !q.object_crc) return fail(TSGPU_E_ARG, "parts cursor, n_parts and object_%s cannot be null", crc_arg<W>());
    PartsCarry<W>& cur = run.cur;
    memcpy(&cur, q.cursor, sizeof cur);
    if (cur.obj_len && cur.part_size != q.part_size)
        return fail(TSGPU_E_ARG, "part_size %llu differs from the %llu the object started with", (unsigned long long)q.part_size,
                    (unsigned long long)cur.part_size);
    const uint64_t most = (cur.obj_len % q.part_size + bound) / q.part_size + (segment_ends_here ? 1 : 0);
    if (most > q.cap) return fail(TSGPU_E_SHORT, "part_%s too small: the call may complete %llu parts, part_cap is %u",
                                  crc_arg<W>(), (unsigned long long)most, q.cap);
    if (q.cap && !q.crcs) return fail(TSGPU_E_ARG, "part_%s cannot be null", crc_arg<W>());
    run.q = q;
    return TSGPU_OK;
}

template <typename W>
static int parts_alloc(PcrcScratch<W>& r, uint64_t cap, rt::stream_t st) {
    if (r.cap >= cap) return TSGPU_OK;
    rt::free_device(r.d); r.d = nullptr; r.cap = 0;
    const uint64_t np = (cap + PCRC_PIECE - 1) / PCRC_PIECE, nt = (cap + PCRC_TILE - 1) / PCRC_TILE;
    const uint64_t sz[3] = {sizeof(W) * np, sizeof(W) * nt, 4};
    uint64_t total = 0;
    for (uint64_t b : sz) total += align_up(b, 256);
    RT(rt::malloc_device((void**)&r.d, total));
    uint8_t* p = r.d;
    auto take = [&](uint64_t b) { uint8_t* q = p; p += align_up(b, 256); return q; };
    r.a.pin = (W*)take(sz[0]); r.a.ttot = (W*)take(sz[1]); r.a.done = (uint32_t*)take(sz[2]);
    RT(rt::memset_async(r.a.done, 0, 4, st));
    r.cap = cap;
    return TSGPU_OK;
}

// Enqueues pcrc_tiles over the batch's packed chunks (d_pack, sizes `len` on the device, at most `bound` bytes in all).
template <typename W>
static int parts_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, const uint32_t* len, uint32_t nb, uint64_t bound) {
    { int rc = parts_alloc(pcrc_of<W>(w), (uint64_t)c->max_batch * c->slot_stride, st); if (rc) return rc; }
    PcrcArgs<W>& a = pcrc_of<W>(w).a;
    a.b = w.d_pack; a.len = len; a.nb = nb;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(PCRC_GRID, (bound + PCRC_TILE - 1) / PCRC_TILE);
    TS_LAUNCH_P(c->prof, sizeof(W) == 8 ? "pcrc64_tiles" : "pcrc_tiles", (pcrc_tiles_kernel<W, false>), dim3(std::max(grid, 1u)),
                dim3(PCRC_T), 0, st, a);
    CHECK_LAUNCH("pcrc_tiles_kernel");
    return TSGPU_OK;
}

// The prefixes of the slot's previous batch are on the host once this slot's sizes event has completed: the batch's first
// kernel that rewrites d_pack waited for the previous copy-out (wait_copies_out), and pcrc_cuts and its D2H precede that copy.
template <typename W>
static void parts_collect(Work& w, PartsRun<W>& pr) {
    PcrcScratch<W>& p = pcrc_of<W>(w);
    if (p.pending < 0) return;
    PcrcBatch<W>& b = pr.batches[(size_t)p.pending];
    b.words.assign(p.h_cuts, p.h_cuts + b.m + 1);
    p.pending = -1;
}

// At the drain of batch `bi` (L packed bytes at `dst_off` in the call's output): pcrc_cuts and the D2H of its m + 1 words on
// out_stream, ahead of the batch's copy-out.
template <typename W>
static int parts_drain(tsgpu_ctx* c, Work& w, PartsRun<W>& pr, uint32_t bi, uint64_t dst_off, uint64_t L) {
    parts_collect(w, pr);
    PcrcScratch<W>& p = pcrc_of<W>(w);
    const uint64_t P = pr.q.part_size;
    const uint64_t at = pr.cur.obj_len + dst_off;                        // the batch's offset in the object
    const uint64_t first = P - at % P;                                   // the first part boundary after the batch's start
    const uint32_t m = first < L ? (uint32_t)((L - 1 - first) / P + 1) : 0;
    if (m + 1 > p.cuts_cap) {                                            // nothing on the slot reads the old arrays any more
        rt::free_device(p.d_cuts); rt::free_host(p.h_cuts); p.d_cuts = nullptr; p.h_cuts = nullptr; p.cuts_cap = 0;
        const uint32_t cap = std::max<uint32_t>(64, m + 1);
        RT(rt::malloc_device((void**)&p.d_cuts, sizeof(W) * cap));
        RT(rt::malloc_host((void**)&p.h_cuts, sizeof(W) * cap));
        p.cuts_cap = cap;
    }
    TS_LAUNCH_P(c->prof, sizeof(W) == 8 ? "pcrc64_cuts" : "pcrc_cuts", (pcrc_cuts_kernel<W, false>), dim3((m + PCRC_CUTS_T) / PCRC_CUTS_T),
                dim3(PCRC_CUTS_T), 0, w.out_stream, p.a, (uint32_t)L, m ? (uint32_t)first : 0u, P, m, p.d_cuts);
    CHECK_LAUNCH("pcrc_cuts_kernel");
    RT(rt::d2h(p.h_cuts, p.d_cuts, sizeof(W) * (m + 1), w.out_stream));
    if (pr.batches.size() <= bi) pr.batches.resize(bi + 1);
    PcrcBatch<W>& b = pr.batches[bi];
    b.L = (uint32_t)L; b.first = m ? (uint32_t)first : 0u; b.m = m; b.words.clear();
    p.pending = (int32_t)bi;
    return TSGPU_OK;
}

// The call's batches in order: their pieces extend the open part and the object; a part whose last byte arrives is emitted.
template <typename W>
static void parts_combine(const PartsRun<W>& pr, PartsCarry<W>& cur, std::vector<W>& emitted) {
    const uint64_t P = pr.q.part_size;
    for (const PcrcBatch<W>& b : pr.batches) {
        W prev = 0;
        uint32_t prev_x = 0;
        for (uint32_t k = 0; k <= b.m; k++) {
            const uint32_t x = k < b.m ? (uint32_t)(b.first + k * P) : b.L;
            const uint32_t n = x - prev_x;
            const W raw = b.words[k] ^ crc_shift(prev, n, 0);             // raw CRC of [prev_x, x)
            cur.raw[0] = crc_shift(cur.raw[0], n, 0) ^ raw;
            cur.obj_len += n;
            if (n && cur.obj_len % P == 0) { emitted.push_back(crc_finish(cur.raw[0], P, 0)); cur.raw[0] = 0; }
            prev = b.words[k]; prev_x = x;
        }
        cur.raw[1] = crc_shift(cur.raw[1], b.L, 0) ^ b.words[b.m];
    }
}

// The idle step of a call with a target half (pr: nullptr without part checksums): the last batches' part prefixes, once every
// slot of the call is idle.
template <typename W>
static int parts_idle(PartsRun<W>* pr, const std::vector<Work*>& slots, int rc) {
    if (pr) for (Work* w : slots) { if (rc == TSGPU_OK) parts_collect(*w, *pr); pcrc_of<W>(*w).pending = -1; }
    return rc;
}

// After a successful call: the completed parts (and at the segment's end the open part and the object CRC) go out, and the
// cursor moves on.  Nothing is written before: a failed call leaves the part and object checksums as they were.
template <typename W>
static void parts_finish(const PartsRun<W>& pr, int segment_ends_here) {
    const PartsReq<W>& q = pr.q;
    PartsCarry<W> cur = pr.cur;
    std::vector<W> emitted;
    parts_combine(pr, cur, emitted);
    cur.part_size = q.part_size;
    if (segment_ends_here) {
        const uint64_t open = cur.obj_len % q.part_size;
        if (open) { emitted.push_back(crc_finish(cur.raw[0], open, 0)); cur.raw[0] = 0; }
        *q.object_crc = crc_finish(cur.raw[1], cur.obj_len, 0);
    }
    if (!emitted.empty()) memcpy(q.crcs, emitted.data(), sizeof(W) * emitted.size());
    *q.n = (uint32_t)emitted.size();
    memcpy(q.cursor, &cur, sizeof cur);
}

#ifdef TSGPU_SIMT
// TEST-ONLY fault injection, compiled into the emulator build alone (device memory is host memory there and every kernel
// has finished when its launch returns).  The variable `var` = <chunk>:<offset> flips the low bit of one byte of that chunk of
// the batch's chunks [c0, c0 + nb) in `chunks`.  A negative offset counts from the chunk's end.
//   TSGPU_SIMT_FLIP: the chunk's transformed bytes -- frame, or IV || ciphertext || tag -- before they are packed and verified
//     (-1: last tag byte).  tests/test_simt_verify.py drives it, and tests/test_simt_encrypt.py for tsgpu_encrypt_object.
//   TSGPU_SIMT_FLIP_DECODED: the chunk's decoded bytes in d_orig right after the source decode of tsgpu_check_object /
//     tsgpu_rewrite_object -- a decoder that misread the chunk.  tests/test_simt_reframe.py drives it: TSGPU_FLAG_REFRAME must
//     not stamp the checksum of such a chunk.
//   TSGPU_SIMT_FLIP_REKEYED: the chunk's re-encrypted bytes in its d_xf slot right after the rekey kernels of tsgpu_rekey_object
//     -- a rekey that wrote a wrong byte.  tests/test_simt_rekey.py drives it: TSGPU_FLAG_VERIFY must catch it.
static void simt_flip(const char* var, ChunksOut chunks, uint32_t c0, uint32_t nb) {
    const char* e = getenv(var);
    long k = 0, at = 0;
    if (!e || sscanf(e, "%ld:%ld", &k, &at) != 2 || k < (long)c0 || k >= (long)c0 + (long)nb) return;
    const uint32_t i = (uint32_t)(k - c0), n = chunks.len[i];
    if (at < 0) at += n;
    if (at >= 0 && at < (long)n) chunks.base[chunks.off[i] + at] ^= 1;
}
#endif

// TSGPU_FLAG_REFRAME (`reframe`: its ZSTD_DENSE and ZSTD_CHECKSUM bits) on the batch's kept frames in the d_frames slots (b_off,
// b_len): with CHECKSUM each frame is sealed with the checksum of its decoded chunk in `orig`; with DENSE the dense compressor
// writes every chunk anew into d_xf at the same slot offsets, and the smaller of the two frames stays in the slot.  d_xf is free
// here: the source half read its encrypted chunks before, and the target half encrypts into it after.  b_len ends with each
// slot's frame size.  XXH64 is a serial chain per chunk: the seal kernel takes one warp per chunk, and the other slots' batches
// run beside it on their own streams.
static int reframe_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, uint32_t reframe, uint32_t nb, uint32_t cs, ChunksIn orig) {
    ReframeArgs R;
    R.frames = w.d_frames; R.f_off = w.dd.b_off; R.f_len = w.dd.b_len;
    R.orig = orig.base; R.o_off = orig.off; R.o_len = orig.len;
    R.cand = w.d_xf; R.cand_len = w.dd.c_len;
    R.n = nb; R.room = (uint32_t)(c->frame_stride - 16);
    const bool checksum = reframe & TSGPU_FLAG_ZSTD_CHECKSUM;
    if (checksum) {
        TS_LAUNCH_P(c->prof, "reframe_seal", reframe_seal_kernel, dim3((nb + RF_WPB - 1) / RF_WPB), dim3(RF_WPB * 32), 0, st, R);
        CHECK_LAUNCH("reframe_seal_kernel");
    }
    if (reframe & TSGPU_FLAG_ZSTD_DENSE) {
        int rc = zstd_stage_modes(c, w, st, /*dense=*/true, checksum, orig, nb, cs, ChunksOut{w.d_xf, w.dd.b_off, w.dd.c_len});
        if (rc) return rc;
        TS_LAUNCH_P(c->prof, "reframe_pick", reframe_pick_kernel, dim3(nb), dim3(RF_PICK_T), 0, st, R);
        CHECK_LAUNCH("reframe_pick_kernel");
    }
    return TSGPU_OK;
}

// The new object's side of a transform or a rewrite.
struct TargetReq {
    uint32_t flags;                  // ZSTD, modifiers and AES of the new object
    bool verify, kept;               // kept (rewrite): the source frames go into the new object as they are
    uint32_t reframe;                // TSGPU_FLAG_REFRAME: the ZSTD_DENSE and ZSTD_CHECKSUM bits that act on the kept frames, else 0
    Aes256RoundKeys rk;
    const uint8_t* aad; uint32_t aad_len;
    const uint8_t* ivs;
};

// The target half of a batch whose original chunks are `orig` in d_orig (each at most cs bytes): [zstd ->] [AES-GCM encrypt]
// with the keys `k`, or with t.kept the batch's frames in the d_frames slots (b_off, b_len; frames_max bytes at most) as they are
// [-> AES-GCM encrypt]; the transformed chunks packed into d_pack, [pcrc_tiles over them for part checksums of CRC word W,] [the
// verify stage and the D2H of its verdicts to the read-back block.]  `fin` receives the transformed chunks in their slots.
// t.reframe: with t.kept, the bits TSGPU_FLAG_REFRAME applies to the kept frames first (reframe_stage); a sealed frame is 4
// bytes longer than frames_max.
template <typename W>
static int target_stage(tsgpu_ctx* c, Work& w, GcmKeys& k, rt::stream_t st, const TargetReq& t, bool parts, uint32_t c0, uint32_t nb,
                        uint32_t cs, ChunksIn orig, uint64_t frames_max, ChunksOut& fin) {
    const bool aes = t.flags & TSGPU_FLAG_AES;
    // encrypted chunks land in the transformed slots; zstd alone leaves its frames in the frame slots
    fin = aes ? ChunksOut{w.d_xf, w.dd.c_off, w.dd.c_len} : ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len};
    uint64_t payload;                        // the largest transformed chunk without IV and tag
    if (t.kept) {
        payload = frames_max + ((t.reframe & TSGPU_FLAG_ZSTD_CHECKSUM) ? 4 : 0);
        if (t.reframe) { int rc = reframe_stage(c, w, st, t.reframe, nb, cs, orig); if (rc) return rc; }
        if (aes) {
            int rc = gcm_stage<true>(c, w, k, st, t.rk, ChunksIn{w.d_frames, w.dd.b_off, w.dd.b_len}, fin, t.aad_len, w.dd.status, nb,
                                     (uint32_t)payload, 0xffffffffu);
            if (rc) return rc;
        }
    } else {
        payload = (t.flags & TSGPU_FLAG_ZSTD) ? frame_bound(cs) : cs;
        int rc = transform_enqueue(c, w, k, st, t.flags, nb, cs, t.rk, t.aad_len, orig, fin);
        if (rc) return rc;
    }
#ifdef TSGPU_SIMT
    simt_flip("TSGPU_SIMT_FLIP", fin, c0, nb);
#endif
    // the transformed chunks, back to back, so the batch leaves in one copy (the previous batch's copy-out may still be
    // reading d_pack: this is the first kernel of the batch that has to wait for it)
    { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
    {
        PackArgs P;
        P.base = fin.base; P.stride = aes ? c->slot_stride : c->frame_stride; P.head = aes ? TSGPU_SLOT_HEAD : 0;
        P.len = fin.len; P.n = nb; P.out = w.d_pack;
        const uint64_t longest = payload + 28;
        TS_LAUNCH_P(c->prof, "pack_chunks", pack_chunks_kernel, dim3((uint32_t)((longest + PACK_PIECE - 1) / PACK_PIECE), nb), dim3(PACK_T), 0, st, P);
        CHECK_LAUNCH("pack_chunks_kernel");
        if (parts) { int rc = parts_stage<W>(c, w, st, fin.len, nb, longest * nb); if (rc) return rc; }
    }
    if (t.verify) {
        int rc = verify_stage(c, w, k, st, t.flags, nb, cs, payload, t.rk, t.aad_len, fin);
        if (rc) return rc;
        RT(rt::d2h(w.back.status, w.dd.status, 4ull * nb, st));
        RT(rt::d2h(w.back.diff, w.dd.v_diff, 4ull * nb, st));
    }
    return TSGPU_OK;
}

// One batch: copy in, fill the descriptors, the target half, [the record kernels,] D2H of the transformed sizes.
// `off`/`len`: position and size of every chunk inside src (chunks are contiguous); `cs` = largest chunk of the call.
template <typename W>
static int transform_issue(tsgpu_ctx* c, const Batch& bt, const TargetReq& t, bool records, bool parts, const uint8_t* src,
                           const uint64_t* off, const uint32_t* len, uint32_t cs) {
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
    }
    slot_layout(c, w.hd, nb, c->slot_stride);
    if (t.flags & TSGPU_FLAG_AES) {
        memcpy(w.hd.ivs, t.ivs + (size_t)c0 * TSGPU_IV_SIZE, (size_t)nb * TSGPU_IV_SIZE);
        if (t.aad_len) memcpy(w.hd.aad, t.aad, t.aad_len);
    }
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    ChunksOut fin;
    { int rc = target_stage<W>(c, w, w.keys[0], st, t, parts, c0, nb, cs, ChunksIn{w.d_orig, w.dd.a_off, w.dd.a_len}, 0, fin); if (rc) return rc; }
    if (records) {
        int rc = records_alloc(w.rec, (uint64_t)c->max_batch * cs);
        if (!rc) rc = records_stage(c, w, st, byte1 - byte0);
        if (rc) return rc;
    }
    RT(rt::d2h(w.back.sizes, fin.len, 4ull * nb, st));
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

// The verify stage's verdict on a drained batch; TSGPU_OK if every chunk read back.  `len`: the original chunk sizes of the
// call; `first`: the number the call's first chunk has in the messages.
static int verify_verdict(const Batch& bt, const uint32_t* len, uint64_t first = 0) {
    const uint32_t* status = bt.w->back.status;
    const uint32_t* diff = bt.w->back.diff;
    for (uint32_t i = 0; i < bt.nb; i++) {
        const uint32_t k = bt.c0 + i;
        const unsigned long long g = first + k;
        if (status[i] == 1) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: tag check failed", g);
        if (status[i] == VERIFY_ST_SIZE)
            return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: size check failed (original %u bytes)", g, len[k]);
        if (status[i] != 0) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: frame check failed (code %u)", g, status[i]);
        if (diff[i] != VERIFY_NO_DIFF)
            return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: bytes differ from offset %u", g, diff[i]);
    }
    return TSGPU_OK;
}

// The drain of a batch whose target half ran (transform, rewrite, rekey), once its verdicts have passed: its new sizes go to the
// caller's `sizes` (nullptr: the caller knows them), [its part prefixes are cut,] and its bytes leave.
template <typename W>
static int target_drain(tsgpu_ctx* c, const Batch& bt, uint32_t* sizes, PartsRun<W>* parts, uint8_t* dst, uint64_t dst_cap,
                        uint64_t& dst_off) {
    Work& w = *bt.w;
    uint64_t total = 0;
    for (uint32_t i = 0; i < bt.nb; i++) { if (sizes) sizes[bt.c0 + i] = w.back.sizes[i]; total += w.back.sizes[i]; }
    if (parts && dst_off + total <= dst_cap) {
        int rc = parts_drain(c, w, *parts, bt.c0 / c->max_batch, dst_off, total);
        if (rc) return rc;
    }
    return copy_out(w, w.d_pack, total, dst, dst_cap, dst_off);     // one copy per batch: packed on the device
}

template <typename W = uint32_t>
static int transform_common(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const std::vector<uint64_t>& off,
                            const std::vector<uint32_t>& len, uint32_t cs, const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                            const uint8_t* ivs, uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                            RecCarry* records, PartsRun<W>* parts = nullptr) {
    const uint32_t n = (uint32_t)len.size();
    if (!dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (!(flags & TSGPU_FLAG_ZSTD)) flags &= ~ZSTD_MODIFIERS;         // modifiers of ZSTD: meaningless (and harmless) without it
    const bool verify = (flags & TSGPU_FLAG_VERIFY) || c->verify_default;
    flags &= ~TSGPU_FLAG_VERIFY;

    if (flags == 0) {       // TransformFinisher no-transform fast path (TransformFinisher.java:135-140): bytes unchanged, nothing to verify
        if (dst_cap < src_len) return fail(TSGPU_E_SHORT, "dst too small");
        memcpy(dst, src, src_len);
        for (uint32_t i = 0; i < n; i++) transformed_sizes[i] = len[i];
        *n_chunks = n;
        return TSGPU_OK;
    }
    TargetReq t{};
    t.flags = flags; t.verify = verify; t.kept = false; t.reframe = 0;
    if (flags & TSGPU_FLAG_AES) t.rk = aes256_expand_key(key);
    t.aad = aad; t.aad_len = aad_len; t.ivs = ivs;

    uint64_t dst_off = 0;
    const int rc = run_batches(c, n, nullptr,
        [&](const Batch& bt) { return transform_issue<W>(c, bt, t, records != nullptr, parts != nullptr, src, off.data(), len.data(), cs); },
        [&](const Batch& bt) {
            if (records) { int rcr = records_resolve(c, *bt.w, *records); if (rcr) return rcr; }   // the input first: none of the batch's bytes leave
            if (verify) { int rcv = verify_verdict(bt, len.data()); if (rcv) return rcv; }   // none of the batch's bytes leave
            return target_drain(c, bt, transformed_sizes, parts, dst, dst_cap, dst_off);
        },
        [&](const std::vector<Work*>& slots, int rcb) { return parts_idle(parts, slots, rcb); });
    if (rc) return rc;
    *n_chunks = n;
    return TSGPU_OK;
}

// The key, IV and AAD arguments of a call with TSGPU_FLAG_AES in `flags`.  `side`: what the call does with the key, which names
// the arguments in the messages (AES_TO: the new key of tsgpu_rewrite_object, its arguments named to_*).  `ivs`: the IVs the
// call needs are there (each call has its own rule; decryption reads them from the chunks).
enum AesSide { AES_ENC, AES_DEC, AES_TO };
static int aes_args_ok(uint32_t flags, AesSide side, const uint8_t* key, bool ivs, const uint8_t* aad, uint32_t aad_len) {
    if (!(flags & TSGPU_FLAG_AES)) return TSGPU_OK;
    if (!key || !ivs)
        return fail(TSGPU_E_ARG, side == AES_ENC ? "key and ivs are required for encryption"
                                 : side == AES_TO ? "to_key and to_ivs are required for encryption" : "key is required for decryption");
    if (aad_len > MAX_AAD) return fail(TSGPU_E_ARG, side == AES_TO ? "to_aad longer than %u bytes" : "aad longer than %u bytes", MAX_AAD);
    if (aad_len && !aad) return fail(TSGPU_E_ARG, side == AES_TO ? "to_aad cannot be null" : "aad cannot be null");
    return TSGPU_OK;
}

static int transform_args_ok(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint8_t* key, const uint8_t* aad,
                             uint32_t aad_len, const uint8_t* ivs, uint32_t* transformed_sizes, uint32_t* n_chunks) {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!n_chunks || !transformed_sizes) return fail(TSGPU_E_ARG, "transformed_sizes/n_chunks cannot be null");
    if (src_len && !src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (flags & ~(KNOWN_FLAGS | TSGPU_FLAG_VERIFY | TSGPU_FLAG_VALIDATE_RECORDS)) return fail(TSGPU_E_ARG, "unknown flags %u", flags);
    return aes_args_ok(flags, AES_ENC, key, ivs != nullptr, aad, aad_len);
}

static_assert(sizeof(tsgpu_records_cursor) == sizeof(RecCarry), "the cursor holds the carry");
template <typename W = uint32_t>
static int transform_segment(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size, const uint8_t key[32],
                             const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs, uint8_t* dst, uint64_t dst_cap,
                             uint32_t* transformed_sizes, uint32_t* n_chunks, tsgpu_records_cursor* cursor, int segment_ends_here,
                             bool env_default, const PartsReq<W>* parts = nullptr) try {
    int rc = transform_args_ok(c, flags, src, src_len, key, aad, aad_len, ivs, transformed_sizes, n_chunks);
    if (rc) return rc;
    const uint32_t xf = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES;
    if ((flags & TSGPU_FLAG_VALIDATE_RECORDS) && !(flags & xf))
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_VALIDATE_RECORDS (%u) needs TSGPU_FLAG_ZSTD or TSGPU_FLAG_AES: without them no byte reaches the GPU",
                    TSGPU_FLAG_VALIDATE_RECORDS);
    const bool records = (flags & TSGPU_FLAG_VALIDATE_RECORDS) || (env_default && c->records_default && (flags & xf));
    if (records && !cursor) return fail(TSGPU_E_ARG, "cursor cannot be null when record batches are validated");
    RecCarry carry{};
    if (records) memcpy(&carry, cursor, sizeof carry);
    PartsRun<W> run;
    if (parts) {
        rc = parts_begin(run, *parts, flags, src_len ? tsgpu_transform_bound(flags, src_len, chunk_size) : 0, segment_ends_here);
        if (rc) return rc;
    }
    // BaseTransformChunkEnumeration: originalChunkSize 0 disables chunking (one chunk = whole stream)
    uint64_t cs64 = chunk_size ? chunk_size : src_len;
    if (src_len == 0) {
        if (records && segment_ends_here) { rc = records_segment_end(carry); if (rc) return rc; }
        *n_chunks = 0;
        if (parts) parts_finish(run, segment_ends_here);
        return TSGPU_OK;
    }
    if (cs64 > c->chunk_cap) return fail(TSGPU_E_ARG, "chunk size %llu exceeds the context's max_chunk_bytes %u", (unsigned long long)cs64, c->chunk_cap);
    const uint32_t cs = (uint32_t)cs64;
    if (records && (uint64_t)c->max_batch * cs > REC_MAX_BATCH)
        return fail(TSGPU_E_ARG, "record validation needs batches below 2 GiB: max_batch %u x chunk size %u is more", c->max_batch, cs);
    if (parts && (uint64_t)c->max_batch * c->slot_stride > 0xffffff00ull)
        return fail(TSGPU_E_ARG, "part checksums need batches below 4 GiB: max_batch %u x slot stride %llu is more", c->max_batch,
                    (unsigned long long)c->slot_stride);
    const uint64_t n64 = (src_len + cs - 1) / cs;
    if (n64 > *n_chunks) return fail(TSGPU_E_SHORT, "transformed_sizes too small: %llu chunks", (unsigned long long)n64);
    std::vector<uint64_t> off(n64);
    std::vector<uint32_t> len(n64);
    for (uint64_t i = 0; i < n64; i++) { off[i] = i * cs; len[i] = (uint32_t)std::min<uint64_t>(cs, src_len - i * cs); }
    rc = transform_common(c, flags & ~TSGPU_FLAG_VALIDATE_RECORDS, src, src_len, off, len, cs, key, aad, aad_len, ivs, dst, dst_cap,
                          transformed_sizes, n_chunks, records ? &carry : nullptr, parts ? &run : nullptr);
    if (rc) return rc;
    if (records) {
        if (segment_ends_here) { rc = records_segment_end(carry); if (rc) return rc; }
        memcpy(cursor, &carry, sizeof carry);
    }
    if (parts) parts_finish(run, segment_ends_here);
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

extern "C" int tsgpu_transform(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                               const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                               uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks) {
    // One call is the whole segment.  The environment default does not reach this call: streaming callers (the JNI
    // enumeration) pass one window of a segment per call, and a window validated as a segment would fail where an entry
    // crosses its end.
    tsgpu_records_cursor whole{};
    return transform_segment(c, flags, src, src_len, chunk_size, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, n_chunks,
                             &whole, 1, /*env_default=*/false);
}

extern "C" int tsgpu_transform_cursor(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                                      const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                      uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                                      tsgpu_records_cursor* cursor, int segment_ends_here) {
    return transform_segment(c, flags, src, src_len, chunk_size, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, n_chunks,
                             cursor, segment_ends_here, /*env_default=*/true);
}

extern "C" int tsgpu_transform_parts(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                                     const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                     uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                                     tsgpu_records_cursor* records, int segment_ends_here,
                                     uint64_t part_size, tsgpu_parts_cursor* parts,
                                     uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts, uint32_t* object_crc32c) {
    const PartsReq<uint32_t> req{part_size, parts, part_crc32c, part_cap, n_parts, object_crc32c};
    return transform_segment(c, flags, src, src_len, chunk_size, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, n_chunks,
                             records, segment_ends_here, /*env_default=*/true, &req);
}

extern "C" int tsgpu_transform_parts_crc64(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, uint32_t chunk_size,
                                           const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                           uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes, uint32_t* n_chunks,
                                           tsgpu_records_cursor* records, int segment_ends_here,
                                           uint64_t part_size, tsgpu_parts_cursor* parts,
                                           uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts, uint64_t* object_crc64) {
    const PartsReq<uint64_t> req{part_size, parts, part_crc64, part_cap, n_parts, object_crc64};
    return transform_segment(c, flags, src, src_len, chunk_size, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, n_chunks,
                             records, segment_ends_here, /*env_default=*/true, &req);
}

// Ragged variant: chunk i is the next chunk_lens[i] bytes of src.  This is what RemoteStorageManager.transformIndex
// (RemoteStorageManager.java:455-490) needs: every Kafka index file is ONE chunk (chunking disabled), AES only, and the
// five of them ride in a single batch (SURVEY.md §8f.3).
extern "C" int tsgpu_transform_chunks(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, const uint32_t* chunk_lens, uint32_t n,
                                      const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                      uint8_t* dst, uint64_t dst_cap, uint32_t* transformed_sizes) try {
    uint32_t cap = n;
    if (flags & TSGPU_FLAG_VALIDATE_RECORDS)
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_VALIDATE_RECORDS (%u) applies to segments, not to ragged chunks such as index files",
                    TSGPU_FLAG_VALIDATE_RECORDS);
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
    return transform_common(c, flags, src, total, off, len, mx, key, aad, aad_len, ivs, dst, dst_cap, transformed_sizes, &cap, nullptr);
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

// ------------------------------------------------------------------------------------------ detransform (host)
// A batch's transformed chunks into the slot's d_xf, one per slot at i * slot_stride + TSGPU_SLOT_HEAD (16-byte aligned ciphertext
// for the GCM kernel), and the descriptor block filled for detransform_enqueue (not yet uploaded).  Returns the bounds of the stages.
// `src`: the call's transformed chunks.  to_frames (zstd only): the frames go to the d_frames slots (b_off, b_len) instead.
static int dx_load(tsgpu_ctx* c, Work& w, rt::stream_t st, const Batch& bt, uint32_t flags, const uint8_t* src, const uint32_t* tsizes,
                   const uint8_t* aad, uint32_t aad_len, DxBounds& lim, bool to_frames = false) {
    const uint32_t c0 = bt.c0, nb = bt.nb;
    // Sizes come from a manifest, i.e. from outside: bound them per mode BEFORE any kernel writes (the GCM kernel
    // releases plaintext into the next buffer before the tag is checked).  AES only: plaintext lands in d_orig
    // (chunk_cap per chunk); AES+zstd: in a d_frames slot; zstd only: the frame is read in place from d_xf.
    const uint32_t room = (flags & TSGPU_FLAG_ZSTD) ? (uint32_t)(c->frame_stride - 16) : c->chunk_cap;
    uint64_t ip = bt.in_off, op = 0;
    uint32_t max_t = 0;
    slot_layout(c, w.hd, nb, c->slot_stride);
    for (uint32_t i = 0; i < nb; i++) {
        const uint32_t t = tsizes[c0 + i];
        const uint64_t payload = (flags & TSGPU_FLAG_AES) ? (t >= 28 ? t - 28 : 0) : t;
        if (payload > room || t > c->slot_stride - TSGPU_SLOT_HEAD - 16)
            return fail(TSGPU_E_ARG, "transformed chunk of %u bytes exceeds the context's capacity", t);
        w.hd.c_len[i] = t;
        w.hd.b_len[i] = (uint32_t)payload;               // what the GCM stage writes there (AES), or the frame (to_frames)
        w.hd.a_off[i] = op;                              // used when there is no zstd stage (sizes are known)
        if (t) RT(rt::h2d((to_frames ? w.d_frames + w.hd.b_off[i] : w.d_xf + w.hd.c_off[i]), src + ip, t, st));
        ip += t;
        op += payload;
        max_t = std::max(max_t, t);
    }
    if ((flags & TSGPU_FLAG_AES) && aad_len) memcpy(w.hd.aad, aad, aad_len);
    lim = DxBounds{max_t, room, 0xffffffffu, c->chunk_cap};
    return TSGPU_OK;
}

// One batch: bound the sizes, copy the chunks in, fill the descriptors, enqueue the stages, D2H of sizes and status.
static int detransform_issue(tsgpu_ctx* c, const Batch& bt, uint32_t flags, const uint8_t* src, const uint32_t* tsizes,
                             const Aes256RoundKeys& rk, const uint8_t* aad, uint32_t aad_len) {
    Work& w = *bt.w;
    const uint32_t nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    DxBounds lim;
    { int rc = dx_load(c, w, st, bt, flags, src, tsizes, aad, aad_len, lim); if (rc) return rc; }
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
    { int rc = detransform_enqueue(c, w, w.keys[0], st, flags, nb, rk, aad_len, ChunksIn{w.d_xf, w.dd.c_off, w.dd.c_len},
                                   ChunksOut{w.d_orig, w.dd.a_off, w.dd.a_len}, w.dd.status, lim, /*packed=*/true); if (rc) return rc; }
    RT(rt::d2h(w.back.sizes, w.dd.a_len, 4ull * nb, st));
    RT(rt::d2h(w.back.status, w.dd.status, 4ull * nb, st));
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

extern "C" int tsgpu_detransform(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len,
                                 const uint32_t* transformed_sizes, uint32_t n_chunks,
                                 const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                 uint8_t* dst, uint64_t dst_cap, uint32_t* original_sizes) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    flags &= ~TSGPU_FLAG_VALIDATE_RECORDS;                   // a property of the upload: nothing to do on the way back
    if (n_chunks == 0) return TSGPU_OK;
    if (!src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (!transformed_sizes) return fail(TSGPU_E_ARG, "chunks cannot be null");
    if (!dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (flags & ~KNOWN_FLAGS) return fail(TSGPU_E_ARG, "unknown flags %u", flags);
    if (int rc = aes_args_ok(flags, AES_DEC, key, true, aad, aad_len)) return rc;
    flags &= ~ZSTD_MODIFIERS;                                // how a frame was compressed does not matter to the reader
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

    uint64_t dst_off = 0;
    int soft = TSGPU_OK;
    const int rc = run_batches(c, n_chunks, transformed_sizes,
        [&](const Batch& bt) { return detransform_issue(c, bt, flags, src, transformed_sizes, rk, aad, aad_len); },
        [&](const Batch& bt) {
            Work& w = *bt.w;
            uint64_t total = 0;
            for (uint32_t i = 0; i < bt.nb; i++) {
                uint32_t stt = w.back.status[i];
                if (stt == 1 && soft == TSGPU_OK) soft = fail(TSGPU_E_AUTH, "Tag mismatch in chunk %u", bt.c0 + i);
                else if (stt > 1 && soft == TSGPU_OK) soft = fail(TSGPU_E_CORRUPT, "Invalid zstd frame in chunk %u (code %u)", bt.c0 + i, stt);
                if (original_sizes) original_sizes[bt.c0 + i] = w.back.sizes[i];
                total += w.back.sizes[i];
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

// ------------------------------------------------------------------------------------------ object check (host)
// tsgpu_check_object: the detransform of a stored object with nothing copied out.  Per batch, on the compute stream, the source
// half (source_stage): the transformed chunks into d_xf (flags 0: the plain chunks straight into d_orig), pcrc over them where
// they sit (the object word), the detransform stages into d_orig at the chunk index's offsets, pcrc over d_orig by the index's
// sizes (the segment word), [the record kernels,] and one D2H each of the decoded sizes, the statuses and the two words.  At the
// drain (source_drain), in object order: tag and frame statuses, decoded sizes against the chunk index, the record verdict, then
// the words extend the cursor's CRCs.

// The state of an object between calls: the public tsgpu_check_cursor (128 bytes, zero = start of the object).  CRC-64/NVME's
// wider words take 8 of the 32 bytes CRC-32C leaves reserved.
template <typename W> struct CheckCarry {
    uint64_t chunks;       // chunks checked so far
    uint64_t obj_len;      // object bytes so far
    uint64_t seg_len;      // decoded segment bytes so far
    W obj_raw;             // raw CRC of the object so far
    W seg_raw;             //   ... and of the decoded segment so far
    RecCarry rec;          // TSGPU_FLAG_VALIDATE_RECORDS
    uint64_t reserved[sizeof(W) == 8 ? 3 : 4];
};
static_assert(sizeof(CheckCarry<uint32_t>) == sizeof(tsgpu_check_cursor) && sizeof(CheckCarry<uint64_t>) == sizeof(tsgpu_check_cursor),
              "the cursor holds the carry");

// The chunk index of the manifest (AbstractChunkIndex.materializeChunks): ceil(ofs / ocs) chunks of ocs original bytes, the
// last one holding the remainder; an empty segment has none.
struct ChunkLayout {
    uint32_t ocs; uint64_t ofs, count;
    uint32_t size(uint64_t g) const { return g + 1 < count ? ocs : g + 1 == count ? (uint32_t)(ofs - g * ocs) : 0u; }
};

// Chunk g of the object reads to `got` bytes (decoded, or a frame's Frame_Content_Size): TSGPU_OK when the chunk index gives it
// that many.
static int index_size_ok(const ChunkLayout& index, unsigned long long g, uint32_t got) {
    if (g >= index.count)
        return fail(TSGPU_E_CORRUPT, "chunk %llu decoded to %u bytes, but the chunk index (original chunk size %u, original file "
                    "size %llu) has %llu chunks", g, got, index.ocs, (unsigned long long)index.ofs, (unsigned long long)index.count);
    if (got != index.size(g))
        return fail(TSGPU_E_CORRUPT, "chunk %llu decoded to %u bytes, the chunk index gives %u", g, got, index.size(g));
    return TSGPU_OK;
}

// At the object's end: TSGPU_OK when it had as many chunks as the chunk index.
static int index_count_ok(const ChunkLayout& index, uint64_t chunks) {
    if (chunks != index.count)
        return fail(TSGPU_E_CORRUPT, "the object has %llu chunks, the chunk index (original chunk size %u, original file size %llu) "
                    "has %llu", (unsigned long long)chunks, index.ocs, (unsigned long long)index.ofs, (unsigned long long)index.count);
    return TSGPU_OK;
}

// One window of a stored object, its arguments checked (source_args).
struct SourceReq {
    uint32_t flags;                  // ZSTD and AES of the object (0: plain)
    bool records;                    // TSGPU_FLAG_VALIDATE_RECORDS
    const uint8_t* src; const uint32_t* tsizes;
    uint32_t n;                      // chunks of the window (the empty segment's one empty chunk is not one)
    uint64_t need;                   // bytes of the window
    ChunkLayout index;
    Aes256RoundKeys rk;
    const uint8_t* aad; uint32_t aad_len;
};

static int source_args(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                       uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size, const uint8_t* key,
                       const uint8_t* aad, uint32_t aad_len, uint64_t chunks_before, SourceReq& q) {
    if (flags & ~(KNOWN_FLAGS | TSGPU_FLAG_VALIDATE_RECORDS)) return fail(TSGPU_E_ARG, "unknown flags %u", flags);
    if (n_chunks && !transformed_sizes) return fail(TSGPU_E_ARG, "chunks cannot be null");
    if (original_chunk_size == 0) return fail(TSGPU_E_ARG, "Original chunk size must be positive, 0 given");
    if (original_chunk_size > c->chunk_cap)
        return fail(TSGPU_E_ARG, "original chunk size %u exceeds the context's max_chunk_bytes %u", original_chunk_size, c->chunk_cap);
    if (int rc = aes_args_ok(flags, AES_DEC, key, true, aad, aad_len)) return rc;
    q.records = flags & TSGPU_FLAG_VALIDATE_RECORDS;
    if (q.records && (uint64_t)c->max_batch * original_chunk_size > REC_MAX_BATCH)
        return fail(TSGPU_E_ARG, "record validation needs batches below 2 GiB: max_batch %u x chunk size %u is more", c->max_batch,
                    original_chunk_size);
    if ((uint64_t)c->max_batch * c->slot_stride > 0xffffff00ull)
        return fail(TSGPU_E_ARG, "object checksums need batches below 4 GiB: max_batch %u x slot stride %llu is more", c->max_batch,
                    (unsigned long long)c->slot_stride);
    q.flags = flags & ~(ZSTD_MODIFIERS | TSGPU_FLAG_VALIDATE_RECORDS);   // how a frame was compressed does not matter to the reader
    q.need = 0;
    for (uint32_t i = 0; i < n_chunks; i++) q.need += transformed_sizes[i];
    if (q.need && !src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (q.need > src_len) return fail(TSGPU_E_SHORT, "Stream has fewer bytes than expected");
    q.src = src; q.tsizes = transformed_sizes;
    q.index = ChunkLayout{original_chunk_size, original_file_size, (original_file_size + original_chunk_size - 1) / original_chunk_size};
    // The index of an empty segment materialises one chunk of 0 transformed bytes: a caller that walks it passes that chunk.
    q.n = n_chunks;
    if (q.index.count == 0 && chunks_before == 0 && q.n == 1 && transformed_sizes[0] == 0) q.n = 0;
    q.rk = Aes256RoundKeys{};
    if (q.flags & TSGPU_FLAG_AES) q.rk = aes256_expand_key(key);
    q.aad = aad; q.aad_len = aad_len;
    return TSGPU_OK;
}

// The raw CRC of a batch's L bytes into pcrc.d_cuts[k]: pcrc_tiles, then pcrc_cuts without part boundaries.
template <typename W, bool SLOTS>
static int check_crc_word(tsgpu_ctx* c, Work& w, rt::stream_t st, const uint8_t* b, const uint64_t* off, const uint32_t* len,
                          uint32_t nb, uint64_t L, uint32_t k) {
    PcrcScratch<W>& p = pcrc_of<W>(w);
    { int rc = parts_alloc(p, (uint64_t)c->max_batch * c->slot_stride, st); if (rc) return rc; }
    if (!p.d_cuts) {
        RT(rt::malloc_device((void**)&p.d_cuts, sizeof(W) * 64));
        RT(rt::malloc_host((void**)&p.h_cuts, sizeof(W) * 64));
        p.cuts_cap = 64;
    }
    p.a.b = b; p.a.len = len; p.a.nb = nb;
    PcrcIn<W, SLOTS> a{};
    static_cast<PcrcArgs<W>&>(a) = p.a;
    if constexpr (SLOTS) a.off = off;
    const uint32_t grid = (uint32_t)std::min<uint64_t>(PCRC_GRID, (L + PCRC_TILE - 1) / PCRC_TILE);
    const bool w64 = sizeof(W) == 8;
    TS_LAUNCH_P(c->prof, SLOTS ? (w64 ? "pcrc64_tiles_slots" : "pcrc_tiles_slots") : (w64 ? "pcrc64_tiles" : "pcrc_tiles"),
                (pcrc_tiles_kernel<W, SLOTS>), dim3(std::max(grid, 1u)), dim3(PCRC_T), 0, st, a);
    CHECK_LAUNCH("pcrc_tiles_kernel");
    TS_LAUNCH_P(c->prof, SLOTS ? (w64 ? "pcrc64_cuts_slots" : "pcrc_cuts_slots") : (w64 ? "pcrc64_cuts" : "pcrc_cuts"),
                (pcrc_cuts_kernel<W, SLOTS>), dim3(1), dim3(PCRC_CUTS_T), 0, st, a, (uint32_t)L, 0u, (uint64_t)1, 0u, p.d_cuts + k);
    CHECK_LAUNCH("pcrc_cuts_kernel");
    return TSGPU_OK;
}

// The source half of one batch.  `g0`: the object's chunk number of the call's first chunk.  A zstd-only object's frames go to
// the d_frames slots with to_frames, else in place in d_xf.  Chunk i decodes to d_orig + a_off[i], the offset the chunk index
// gives it, and v_len[i] holds its size by the index: what later stages read, so a damaged chunk cannot steer them (its batch
// fails at the drain).  The descriptor block is uploaded here: a caller fills its other fields first.  The read-back block
// receives the decoded sizes, the statuses and the object and segment words.
template <typename W>
static int source_stage(tsgpu_ctx* c, Work& w, rt::stream_t st, const Batch& bt, const SourceReq& q, uint64_t g0, bool to_frames) {
    const uint32_t nb = bt.nb, flags = q.flags;
    uint64_t L = 0, obj = 0;                 // the batch's length by the chunk index (what it decodes to when it is sound)
    for (uint32_t i = 0; i < nb; i++) {
        w.hd.v_len[i] = q.index.size(g0 + bt.c0 + i);
        L += w.hd.v_len[i];
        obj += q.tsizes[bt.c0 + i];
    }
    DxBounds lim{};
    if (flags) {
        int rc = dx_load(c, w, st, bt, flags, q.src, q.tsizes, q.aad, q.aad_len, lim, to_frames);
        if (rc) return rc;
        // Chunk i decodes to a_off[i] = i * ocs: a frame may not write past ocs bytes, or it would overwrite the next chunk's
        // region while that one decodes (and reads its own output back).  A larger frame is refused as an invalid frame.
        lim.zstd_out = q.index.ocs;
    } else {                                 // a plain object is the segment: its chunks go to d_orig back to back
        for (uint32_t i = 0; i < nb; i++) {
            if (q.tsizes[bt.c0 + i] > c->chunk_cap)
                return fail(TSGPU_E_ARG, "transformed chunk of %u bytes exceeds the context's capacity", q.tsizes[bt.c0 + i]);
            w.back.src_sizes[i] = w.hd.a_len[i] = q.tsizes[bt.c0 + i];     // a_len: the decoded sizes, as the stages write them
            w.back.src_status[i] = 0;
        }
        slot_layout(c, w.hd, nb, c->slot_stride);              // the slots a target half writes
        if (obj) RT(rt::h2d(w.d_orig, q.src + bt.in_off, obj, st));
    }
    for (uint64_t i = 0, a = 0; i < nb; a += w.hd.v_len[i++]) w.hd.a_off[i] = a;
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    // the slot's previous batch may still be copying out, its part prefixes read from the pcrc scratch this batch rewrites
    { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
    if (flags) {
        const ChunksIn in = to_frames ? ChunksIn{w.d_frames, w.dd.b_off, w.dd.b_len} : ChunksIn{w.d_xf, w.dd.c_off, w.dd.c_len};
        { int rc = check_crc_word<W, true>(c, w, st, in.base, in.off, in.len, nb, obj, 0); if (rc) return rc; }
        RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
        int rc = detransform_enqueue(c, w, w.keys[0], st, flags, nb, q.rk, q.aad_len, in, ChunksOut{w.d_orig, w.dd.a_off, w.dd.a_len},
                                     w.dd.status, lim, /*packed=*/false);
        if (rc) return rc;
#ifdef TSGPU_SIMT
        simt_flip("TSGPU_SIMT_FLIP_DECODED", ChunksOut{w.d_orig, w.dd.a_off, w.dd.v_len}, bt.c0, nb);
#endif
    }
    // The segment word and the records over the L bytes the index gives: a batch that decodes to another length fails first.
    { int rc = check_crc_word<W, false>(c, w, st, w.d_orig, nullptr, w.dd.v_len, nb, L, 1); if (rc) return rc; }
    if (q.records && L) {
        int rc = records_alloc(w.rec, (uint64_t)c->max_batch * q.index.ocs);
        if (!rc) rc = records_stage(c, w, st, L);
        if (rc) return rc;
    }
    if (flags) {
        RT(rt::d2h(w.back.src_sizes, w.dd.a_len, 4ull * nb, st));
        RT(rt::d2h(w.back.src_status, w.dd.status, 4ull * nb, st));
    }
    RT(rt::d2h(w.back.words, pcrc_of<W>(w).d_cuts, 2 * sizeof(W), st));
    return TSGPU_OK;
}

// A drained batch in object order (as source_stage left it): every chunk's tag, frame and decoded size, then the record verdict,
// then the CRC words extend the carry.
template <typename W>
static int source_drain(tsgpu_ctx* c, const Batch& bt, const SourceReq& q, CheckCarry<W>& cur) {
    Work& w = *bt.w;
    const uint32_t nb = bt.nb;
    const uint32_t* got = w.back.src_sizes;
    const uint32_t* status = w.back.src_status;
    const ChunkLayout& index = q.index;
    uint64_t L = 0, obj = 0;
    for (uint32_t i = 0; i < nb; i++) {
        const unsigned long long g = cur.chunks + bt.c0 + i;
        if (status[i] == 1) return fail(TSGPU_E_AUTH, "Tag mismatch in chunk %llu", g);
        if (status[i] > 1) return fail(TSGPU_E_CORRUPT, "Invalid zstd frame in chunk %llu (code %u)", g, status[i]);
        if (int rc = index_size_ok(index, g, got[i])) return rc;
        L += got[i];
        obj += q.tsizes[bt.c0 + i];
    }
    if (q.records) { int rc = records_resolve(c, w, cur.rec); if (rc) return rc; }
    const W* words = reinterpret_cast<const W*>(w.back.words);
    const W seg_word = words[1], obj_word = q.flags ? words[0] : seg_word;
    cur.obj_raw = crc_shift(cur.obj_raw, obj, 0) ^ obj_word;
    cur.seg_raw = crc_shift(cur.seg_raw, L, 0) ^ seg_word;
    return TSGPU_OK;
}

// After a window's batches: the carry moves past its chunks, and at the object's end the chunk count and the last record entry
// are checked.
template <typename W>
static int source_finish(const SourceReq& q, CheckCarry<W>& cur, int object_ends_here) {
    cur.chunks += q.n;
    cur.obj_len += q.need;
    for (uint32_t i = 0; i < q.n; i++) cur.seg_len += q.index.size(cur.chunks - q.n + i);
    if (!object_ends_here) return TSGPU_OK;
    if (int rc = index_count_ok(q.index, cur.chunks)) return rc;
    if (q.records) { int rc = records_segment_end(cur.rec); if (rc) return rc; }
    return TSGPU_OK;
}

template <typename W>
static int check_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                        uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size, const uint8_t key[32],
                        const uint8_t* aad, uint32_t aad_len, tsgpu_check_cursor* cursor, int object_ends_here, W* object_crc,
                        W* segment_crc) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!cursor) return fail(TSGPU_E_ARG, "cursor cannot be null");
    if (object_ends_here && (!object_crc || !segment_crc))
        return fail(TSGPU_E_ARG, "object_%s/segment_%s cannot be null", crc_arg<W>(), crc_arg<W>());
    CheckCarry<W> cur;
    memcpy(&cur, cursor, sizeof cur);
    SourceReq q;
    int rc = source_args(c, flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, key, aad, aad_len,
                         cur.chunks, q);
    if (rc) return rc;
    if (q.n) {
        rc = run_batches(c, q.n, transformed_sizes,
            [&](const Batch& bt) {
                Work& w = *bt.w;
                RT(rt::set_device(w.device));
                { int r = source_stage<W>(c, w, w.stream, bt, q, cur.chunks, /*to_frames=*/false); if (r) return r; }
                RT(rt::event_record(w.ev_sizes, w.stream));
                return TSGPU_OK;
            },
            [&](const Batch& bt) { return source_drain(c, bt, q, cur); });
        if (rc) return rc;
    }
    if ((rc = source_finish(q, cur, object_ends_here))) return rc;
    if (object_ends_here) {
        *object_crc = crc_finish(cur.obj_raw, cur.obj_len, 0);
        *segment_crc = crc_finish(cur.seg_raw, cur.seg_len, 0);
    }
    memcpy(cursor, &cur, sizeof cur);
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

extern "C" int tsgpu_check_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                                  uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size,
                                  const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                  tsgpu_check_cursor* cursor, int object_ends_here, uint32_t* object_crc32c, uint32_t* segment_crc32c) {
    return check_object(c, flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, key, aad, aad_len,
                        cursor, object_ends_here, object_crc32c, segment_crc32c);
}

extern "C" int tsgpu_check_object_crc64(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                                        uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size,
                                        const uint8_t key[32], const uint8_t* aad, uint32_t aad_len,
                                        tsgpu_check_cursor* cursor, int object_ends_here, uint64_t* object_crc64, uint64_t* segment_crc64) {
    return check_object(c, flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, key, aad, aad_len,
                        cursor, object_ends_here, object_crc64, segment_crc64);
}

// ------------------------------------------------------------------------------------------ object rewrite (host)
// tsgpu_rewrite_object: the source half of the check, then the target half of the transform (target_stage) from the decoded
// chunks in d_orig, so the plaintext never leaves the GPU.  When both sides compress, the source frames are kept: they are in
// d_frames (a zstd-only object is loaded there rather than into d_xf, where each encrypted chunk would overlap its own frame
// 12 bytes further on; an encrypted one is decrypted there), and the target half only encrypts or packs them.  At the drain, in
// object order: the source's statuses, sizes and records (source_drain), the verify verdict on the new chunks, then the new
// chunks' sizes, part prefixes and copy-out.

// The state of a rewrite between calls: the public tsgpu_rewrite_cursor (192 bytes, zero = start of the object).
template <typename W> struct RewriteCarry {
    CheckCarry<W> src;         // the old object and the decoded segment
    tsgpu_parts_cursor out;    // the new object's parts (a PartsCarry<W>)
    uint64_t reserved[4];
};
static_assert(sizeof(RewriteCarry<uint32_t>) == sizeof(tsgpu_rewrite_cursor) && sizeof(RewriteCarry<uint64_t>) == sizeof(tsgpu_rewrite_cursor),
              "the cursor holds the carry");

// GCM breaks when one key encrypts two plaintexts under one IV: no two chunks of a window of n chunks may share a new IV, nor,
// with same_key (the new key is the old one), a new IV an old chunk of the window has (an old chunk's IV is its first 12 bytes of
// `src`).  `first`: the object's number of the window's first chunk.  skip_empty: a chunk of 0 bytes takes no new IV.
static int new_ivs_ok(const uint8_t* to_ivs, uint32_t n, const uint8_t* src, const uint32_t* tsizes, bool same_key, uint64_t first,
                      bool skip_empty) {
    struct Iv { std::array<uint8_t, TSGPU_IV_SIZE> b; uint32_t i; bool old; };
    std::vector<Iv> ivs;
    for (uint32_t i = 0; i < n; i++) {
        if (skip_empty && tsizes[i] == 0) continue;
        Iv v{{}, i, false};
        memcpy(v.b.data(), to_ivs + (size_t)i * TSGPU_IV_SIZE, TSGPU_IV_SIZE);
        ivs.push_back(v);
    }
    if (same_key) {
        uint64_t at = 0;
        for (uint32_t i = 0; i < n; at += tsizes[i++]) {
            if (tsizes[i] < TSGPU_IV_SIZE) continue;
            Iv v{{}, i, true};
            memcpy(v.b.data(), src + at, TSGPU_IV_SIZE);
            ivs.push_back(v);
        }
    }
    std::sort(ivs.begin(), ivs.end(), [](const Iv& x, const Iv& y) { return x.b != y.b ? x.b < y.b : x.old < y.old; });
    for (size_t j = 1; j < ivs.size(); j++) {
        const Iv &x = ivs[j - 1], &y = ivs[j];
        if (x.b != y.b || (x.old && y.old)) continue;           // two old chunks sharing an IV is the old object's business
        if (y.old) return fail(TSGPU_E_ARG, "to_ivs[%u] repeats the IV of chunk %llu under the same key", x.i,
                               (unsigned long long)(first + y.i));
        return fail(TSGPU_E_ARG, "to_ivs[%u] repeats to_ivs[%u]", std::min(x.i, y.i), std::max(x.i, y.i));
    }
    return TSGPU_OK;
}

// One batch of a rewrite: the target's IVs and AAD, the source half, the target half, the D2H of the new sizes.
template <typename W>
static int rewrite_issue(tsgpu_ctx* c, const Batch& bt, const SourceReq& q, const TargetReq& t, uint64_t g0) {
    Work& w = *bt.w;
    const uint32_t nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    GcmKeys& k = w.keys[1];
    if (t.flags & TSGPU_FLAG_AES) {
        memcpy(w.hd.ivs, t.ivs + (size_t)bt.c0 * TSGPU_IV_SIZE, (size_t)nb * TSGPU_IV_SIZE);
        if (!k.ctx) {
            RT(rt::malloc_device((void**)&k.ctx, sizeof(GcmKeyCtx)));
            RT(rt::malloc_device((void**)&k.d_aad, MAX_AAD));
            RT(rt::malloc_host((void**)&k.h_aad, MAX_AAD));
        }
        if (t.aad_len) {                     // the slot's previous batch has drained: its upload of h_aad is done
            memcpy(k.h_aad, t.aad, t.aad_len);
            RT(rt::h2d(k.d_aad, k.h_aad, t.aad_len, st));
        }
    }
    { int rc = source_stage<W>(c, w, st, bt, q, g0, /*to_frames=*/q.flags == TSGPU_FLAG_ZSTD); if (rc) return rc; }
    uint64_t frames_max = 0;                 // the largest kept frame, by the object's sizes
    for (uint32_t i = 0; i < nb; i++) {
        const uint32_t ts = q.tsizes[bt.c0 + i];
        frames_max = std::max<uint64_t>(frames_max, (q.flags & TSGPU_FLAG_AES) ? (ts >= 28 ? ts - 28 : 0) : ts);
    }
    ChunksOut fin;
    { int rc = target_stage<W>(c, w, k, st, t, /*parts=*/true, bt.c0, nb, q.index.ocs, ChunksIn{w.d_orig, w.dd.a_off, w.dd.v_len},
                               frames_max, fin); if (rc) return rc; }
    RT(rt::d2h(w.back.sizes, fin.len, 4ull * nb, st));
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

template <typename W>
static int rewrite_object(tsgpu_ctx* c, uint32_t from_flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                          uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size, const uint8_t from_key[32],
                          const uint8_t* from_aad, uint32_t from_aad_len, uint32_t to_flags, const uint8_t to_key[32],
                          const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs, uint8_t* dst, uint64_t dst_cap,
                          uint32_t* new_transformed_sizes, uint64_t part_size, W* part_crc, uint32_t part_cap, uint32_t* n_parts,
                          tsgpu_rewrite_cursor* cursor, int object_ends_here, W* source_crc, W* object_crc, W* segment_crc) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!cursor) return fail(TSGPU_E_ARG, "cursor cannot be null");
    if (object_ends_here && (!source_crc || !segment_crc))
        return fail(TSGPU_E_ARG, "source_%s/object_%s/segment_%s cannot be null", crc_arg<W>(), crc_arg<W>(), crc_arg<W>());
    const uint32_t xf = TSGPU_FLAG_ZSTD | TSGPU_FLAG_AES;
    if (to_flags & ~(KNOWN_FLAGS | TSGPU_FLAG_VERIFY | TSGPU_FLAG_REFRAME)) return fail(TSGPU_E_ARG, "unknown to_flags %u", to_flags);
    const bool kept = (from_flags & TSGPU_FLAG_ZSTD) && (to_flags & TSGPU_FLAG_ZSTD);
    const bool reframe = to_flags & TSGPU_FLAG_REFRAME;
    if (reframe && !kept)
        return fail(TSGPU_E_ARG, "to_flags %u: TSGPU_FLAG_REFRAME acts on kept frames and needs TSGPU_FLAG_ZSTD in from_flags and "
                    "to_flags", to_flags);
    if (reframe && !(to_flags & ZSTD_MODIFIERS))
        return fail(TSGPU_E_ARG, "to_flags %u: TSGPU_FLAG_REFRAME needs TSGPU_FLAG_ZSTD_DENSE or TSGPU_FLAG_ZSTD_CHECKSUM", to_flags);
    if (!(to_flags & xf))
        return fail(TSGPU_E_ARG, "to_flags needs TSGPU_FLAG_ZSTD or TSGPU_FLAG_AES: the plain object is what tsgpu_detransform gives");
    if (!(to_flags & TSGPU_FLAG_ZSTD) && (to_flags & ZSTD_MODIFIERS))
        return fail(TSGPU_E_ARG, "to_flags %u: TSGPU_FLAG_ZSTD_DENSE and TSGPU_FLAG_ZSTD_CHECKSUM need TSGPU_FLAG_ZSTD", to_flags);
    if (kept && !reframe && (to_flags & ZSTD_MODIFIERS))
        return fail(TSGPU_E_ARG, "to_flags %u: the source frames are kept as they are, so TSGPU_FLAG_ZSTD_DENSE and "
                    "TSGPU_FLAG_ZSTD_CHECKSUM have nothing to act on", to_flags);
    if (int rc = aes_args_ok(to_flags, AES_TO, to_key, !n_chunks || to_ivs, to_aad, to_aad_len)) return rc;
    if (n_chunks && !new_transformed_sizes) return fail(TSGPU_E_ARG, "new_transformed_sizes cannot be null");
    RewriteCarry<W> cur;
    memcpy(&cur, cursor, sizeof cur);
    SourceReq q;
    int rc = source_args(c, from_flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size,
                         from_key, from_aad, from_aad_len, cur.src.chunks, q);
    if (rc) return rc;
    if (q.n && !dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if ((to_flags & TSGPU_FLAG_AES) && q.n) {
        const bool same_key = (q.flags & TSGPU_FLAG_AES) && memcmp(from_key, to_key, 32) == 0;
        if ((rc = new_ivs_ok(to_ivs, q.n, src, transformed_sizes, same_key, cur.src.chunks, /*skip_empty=*/false))) return rc;
    }
    // part_cap: the transform bound of the window's length by the chunk index, or of its kept frames (4 bytes more each when
    // TSGPU_FLAG_REFRAME seals them: a dense frame replaces one only when it is smaller)
    const uint32_t seal = (reframe && (to_flags & TSGPU_FLAG_ZSTD_CHECKSUM)) ? 4 : 0;
    uint64_t L = 0, frames = 0;
    for (uint32_t i = 0; i < q.n; i++) {
        L += q.index.size(cur.src.chunks + i);
        const uint32_t ts = transformed_sizes[i];
        const uint64_t frame = (q.flags & TSGPU_FLAG_AES) ? (ts >= 28 ? ts - 28 : 0) : ts;
        if (seal && frame + seal > c->frame_stride - 16)
            return fail(TSGPU_E_ARG, "chunk %llu: its sealed frame of %llu bytes would not fit the context's frame slot of %llu bytes",
                        (unsigned long long)(cur.src.chunks + i), (unsigned long long)(frame + seal),
                        (unsigned long long)(c->frame_stride - 16));
        frames += frame + seal + ((to_flags & TSGPU_FLAG_AES) ? 28 : 0);
    }
    const uint64_t bound = !q.n ? 0 : kept ? frames : tsgpu_transform_bound(to_flags, L, original_chunk_size);
    PartsRun<W> run;
    if ((rc = parts_begin(run, PartsReq<W>{part_size, &cur.out, part_crc, part_cap, n_parts, object_crc}, to_flags, bound,
                          object_ends_here))) return rc;

    TargetReq t{};
    t.flags = to_flags & ~(TSGPU_FLAG_VERIFY | TSGPU_FLAG_REFRAME);
    // a reframed chunk is read back, and its new checksum checked, before its batch leaves: no checksum of a misread chunk leaves
    t.verify = (to_flags & TSGPU_FLAG_VERIFY) || c->verify_default || reframe;
    t.kept = kept;
    t.reframe = reframe ? to_flags & ZSTD_MODIFIERS : 0;
    if (to_flags & TSGPU_FLAG_AES) t.rk = aes256_expand_key(to_key);
    t.aad = to_aad; t.aad_len = to_aad_len; t.ivs = to_ivs;
    if (q.n) {
        std::vector<uint32_t> len(q.n);                          // the window's original sizes (verify_verdict's messages)
        for (uint32_t i = 0; i < q.n; i++) len[i] = q.index.size(cur.src.chunks + i);
        uint64_t dst_off = 0;
        rc = run_batches(c, q.n, transformed_sizes,
            [&](const Batch& bt) { return rewrite_issue<W>(c, bt, q, t, cur.src.chunks); },
            [&](const Batch& bt) {
                { int r = source_drain(c, bt, q, cur.src); if (r) return r; }
                if (t.verify) { int r = verify_verdict(bt, len.data(), cur.src.chunks); if (r) return r; }
                return target_drain(c, bt, new_transformed_sizes, &run, dst, dst_cap, dst_off);
            },
            [&](const std::vector<Work*>& slots, int rcb) { return parts_idle(&run, slots, rcb); });
        if (rc) return rc;
    }
    if ((rc = source_finish(q, cur.src, object_ends_here))) return rc;
    if (n_chunks && !q.n) new_transformed_sizes[0] = 0;                    // the empty segment's one empty chunk stays one
    parts_finish(run, object_ends_here);                                   // writes cur.out and the part CRCs
    if (object_ends_here) {
        *source_crc = crc_finish(cur.src.obj_raw, cur.src.obj_len, 0);
        *segment_crc = crc_finish(cur.src.seg_raw, cur.src.seg_len, 0);
    }
    memcpy(cursor, &cur, sizeof cur);
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

extern "C" int tsgpu_rewrite_object(tsgpu_ctx* c, uint32_t from_flags, const uint8_t* src, uint64_t src_len,
                                    const uint32_t* transformed_sizes, uint32_t n_chunks, uint32_t original_chunk_size,
                                    uint64_t original_file_size, const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                                    uint32_t to_flags, const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len,
                                    const uint8_t* to_ivs, uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                                    uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts,
                                    tsgpu_rewrite_cursor* cursor, int object_ends_here,
                                    uint32_t* source_crc32c, uint32_t* object_crc32c, uint32_t* segment_crc32c) {
    return rewrite_object(c, from_flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, from_key,
                          from_aad, from_aad_len, to_flags, to_key, to_aad, to_aad_len, to_ivs, dst, dst_cap, new_transformed_sizes,
                          part_size, part_crc32c, part_cap, n_parts, cursor, object_ends_here, source_crc32c, object_crc32c, segment_crc32c);
}

extern "C" int tsgpu_rewrite_object_crc64(tsgpu_ctx* c, uint32_t from_flags, const uint8_t* src, uint64_t src_len,
                                          const uint32_t* transformed_sizes, uint32_t n_chunks, uint32_t original_chunk_size,
                                          uint64_t original_file_size, const uint8_t from_key[32], const uint8_t* from_aad,
                                          uint32_t from_aad_len, uint32_t to_flags, const uint8_t to_key[32], const uint8_t* to_aad,
                                          uint32_t to_aad_len, const uint8_t* to_ivs, uint8_t* dst, uint64_t dst_cap,
                                          uint32_t* new_transformed_sizes, uint64_t part_size, uint64_t* part_crc64, uint32_t part_cap,
                                          uint32_t* n_parts, tsgpu_rewrite_cursor* cursor, int object_ends_here,
                                          uint64_t* source_crc64, uint64_t* object_crc64, uint64_t* segment_crc64) {
    return rewrite_object(c, from_flags, src, src_len, transformed_sizes, n_chunks, original_chunk_size, original_file_size, from_key,
                          from_aad, from_aad_len, to_flags, to_key, to_aad, to_aad_len, to_ivs, dst, dst_cap, new_transformed_sizes,
                          part_size, part_crc64, part_cap, n_parts, cursor, object_ends_here, source_crc64, object_crc64, segment_crc64);
}

// ------------------------------------------------------------------------------------------ object rekey (host)
// tsgpu_rekey_object: a stored object's IV || CT || TAG chunks re-encrypted under a new key with nothing decoded.  Per batch, on the
// compute stream: the chunks into the d_xf slots, pcrc over them where they sit (the source word), [VERIFY: the DEC kernels
// decrypt them under the old key into the d_frames slots,] the rekey kernels in place, [VERIFY: the DEC kernels decrypt the new
// chunks under the new key into d_pack at the frame slots' offsets and verify_compare compares the two plaintexts,] pack_chunks
// into d_pack and pcrc_tiles over it.  No original chunk, frame or decoder is involved, and without VERIFY neither the d_frames
// slots nor d_orig are touched.  At the drain, in object order: the old tags, the verify verdict, then the source word extends the
// carry and target_drain cuts the part prefixes and copies the batch out.

// The state of a rekey between calls: the public tsgpu_rekey_cursor (64 bytes, zero = start of the object).
template <typename W> struct RekeyCarry {
    tsgpu_parts_cursor out;    // the new object's parts (a PartsCarry<W>)
    uint64_t chunks;           // chunks rekeyed so far
    uint64_t src_len;          // source object bytes so far
    W src_raw;                 // raw CRC of the source object so far
    uint64_t reserved;
};
static_assert(sizeof(RekeyCarry<uint32_t>) == sizeof(tsgpu_rekey_cursor) && sizeof(RekeyCarry<uint64_t>) == sizeof(tsgpu_rekey_cursor),
              "the cursor holds the carry");

struct RekeyReq {
    bool verify;
    const uint8_t* src; const uint32_t* tsizes;
    Aes256RoundKeys rk_old, rk_new;
    const uint8_t* aad_old; uint32_t aad_old_len;
    const uint8_t* aad_new; uint32_t aad_new_len;
    const uint8_t* ivs;
};

template <typename W>
static int rekey_issue(tsgpu_ctx* c, const Batch& bt, const RekeyReq& q) {
    Work& w = *bt.w;
    const uint32_t c0 = bt.c0, nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    GcmKeys &ko = w.keys[0], &kn = w.keys[1];
    if (!kn.ctx) {
        RT(rt::malloc_device((void**)&kn.ctx, sizeof(GcmKeyCtx)));
        RT(rt::malloc_device((void**)&kn.d_aad, MAX_AAD));
        RT(rt::malloc_host((void**)&kn.h_aad, MAX_AAD));
    }
    if (q.aad_new_len) {                 // the slot's previous batch has drained: its upload of h_aad is done
        memcpy(kn.h_aad, q.aad_new, q.aad_new_len);
        RT(rt::h2d(kn.d_aad, kn.h_aad, q.aad_new_len, st));
    }
    memcpy(w.hd.ivs, q.ivs + (size_t)c0 * TSGPU_IV_SIZE, (size_t)nb * TSGPU_IV_SIZE);
    if (q.aad_old_len) memcpy(w.hd.aad, q.aad_old, q.aad_old_len);
    slot_layout(c, w.hd, nb, c->slot_stride);
    uint64_t at = bt.in_off, obj = 0;
    uint32_t max_t = 0;
    for (uint32_t i = 0; i < nb; i++) {  // the sizes were bounded by the slot before any GPU work
        const uint32_t t = q.tsizes[c0 + i];
        w.hd.c_len[i] = t;
        w.back.sizes[i] = t;             // a chunk keeps its size
        if (t) RT(rt::h2d(w.d_xf + w.hd.c_off[i], q.src + at, t, st));
        at += t; obj += t;
        max_t = std::max(max_t, t);
    }
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    // the slot's previous batch may still be copying d_pack out, its part prefixes read from the pcrc scratch this batch rewrites
    { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
    const ChunksIn in{w.d_xf, w.dd.c_off, w.dd.c_len};
    { int rc = check_crc_word<W, true>(c, w, st, in.base, in.off, in.len, nb, obj, 0); if (rc) return rc; }
    RT(rt::d2h(w.back.words, pcrc_of<W>(w).d_cuts, sizeof(W), st));
    const uint32_t payload = max_t >= 28 ? max_t - 28 : 0, room = (uint32_t)(c->frame_stride - 16);
    if (q.verify) {                      // the old plaintext, for the comparison below
        RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
        int rc = gcm_stage<false>(c, w, ko, st, q.rk_old, in, ChunksOut{w.d_frames, w.dd.b_off, w.dd.b_len}, q.aad_old_len, w.dd.status,
                                  nb, max_t, room);
        if (rc) return rc;
    }
    { int rc = gcm_key_tables(c, ko, st, q.rk_old); if (!rc) rc = gcm_key_tables(c, kn, st, q.rk_new); if (rc) return rc; }
    GcmRekeyBatch R;
    R.base = w.d_xf; R.off = w.dd.c_off; R.len = w.dd.c_len; R.ivs = w.dd.ivs;
    R.aad_old = ko.d_aad; R.aad_old_len = q.aad_old_len; R.aad_new = kn.d_aad; R.aad_new_len = q.aad_new_len;
    R.partials_old = w.d_partials; R.partials_new = w.d_partials + (size_t)w.max_ranges * c->max_batch; R.max_ranges = w.max_ranges;
    R.status = w.dd.status; R.n_chunks = nb;
    const uint32_t ranges = (uint32_t)(((uint64_t)payload + 15) / 16 + GH_RANGE_BLOCKS - 1) / GH_RANGE_BLOCKS;
    if (ranges) {
        TS_LAUNCH_P(c->prof, "gcm_rekey", gcm_rekey_kernel, dim3(ranges, nb), dim3(GH_T), GCM_REKEY_SMEM_BYTES, st, q.rk_old, ko.ctx,
                    q.rk_new, kn.ctx, R);
        CHECK_LAUNCH("gcm_rekey_kernel");
    }
    TS_LAUNCH_P(c->prof, "gcm_rekey_finalize", gcm_rekey_finalize_kernel, dim3((nb + 3) / 4), dim3(128), 0, st, q.rk_old, ko.ctx,
                q.rk_new, kn.ctx, R);
    CHECK_LAUNCH("gcm_rekey_finalize_kernel");
    ko.valid = kn.valid = true;
    RT(rt::d2h(w.back.src_status, w.dd.status, 4ull * nb, st));
#ifdef TSGPU_SIMT
    simt_flip("TSGPU_SIMT_FLIP_REKEYED", ChunksOut{w.d_xf, w.dd.c_off, w.dd.c_len}, c0, nb);
#endif
    if (q.verify) {                      // the new chunks read back under the new key
        RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
        RT(rt::memset_async(w.dd.v_diff, 0xff, 4ull * nb, st));
        int rc = gcm_stage<false>(c, w, kn, st, q.rk_new, in, ChunksOut{w.d_pack, w.dd.b_off, w.dd.v_len}, q.aad_new_len, w.dd.status,
                                  nb, max_t, room);
        if (rc) return rc;
        VerifyArgs V;
        V.orig = w.d_frames; V.orig_off = w.dd.b_off; V.orig_len = w.dd.b_len;
        V.back = w.d_pack; V.back_off = w.dd.b_off; V.back_len = w.dd.v_len;
        V.status = w.dd.status; V.diff = w.dd.v_diff;
        TS_LAUNCH_P(c->prof, "verify_compare", verify_compare_kernel, dim3(std::max(1u, (payload + VERIFY_PIECE - 1) / VERIFY_PIECE), nb),
                    dim3(VERIFY_T), 0, st, V);
        CHECK_LAUNCH("verify_compare_kernel");
        RT(rt::d2h(w.back.status, w.dd.status, 4ull * nb, st));
        RT(rt::d2h(w.back.diff, w.dd.v_diff, 4ull * nb, st));
    }
    PackArgs P;
    P.base = w.d_xf; P.stride = c->slot_stride; P.head = TSGPU_SLOT_HEAD; P.len = w.dd.c_len; P.n = nb; P.out = w.d_pack;
    TS_LAUNCH_P(c->prof, "pack_chunks", pack_chunks_kernel, dim3(std::max(1u, (max_t + PACK_PIECE - 1) / PACK_PIECE), nb), dim3(PACK_T),
                0, st, P);
    CHECK_LAUNCH("pack_chunks_kernel");
    { int rc = parts_stage<W>(c, w, st, w.dd.c_len, nb, obj); if (rc) return rc; }
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

// A drained batch's verdicts in object order: every old tag, then (VERIFY) every read-back.  `first`: the object's number of the
// call's first chunk.
static int rekey_verdict(const Batch& bt, const RekeyReq& q, uint64_t first) {
    const Back& b = bt.w->back;
    for (uint32_t i = 0; i < bt.nb; i++)
        if (b.src_status[i]) return fail(TSGPU_E_AUTH, "Tag mismatch in chunk %llu", (unsigned long long)(first + bt.c0 + i));
    if (!q.verify) return TSGPU_OK;
    for (uint32_t i = 0; i < bt.nb; i++) {
        const unsigned long long g = first + bt.c0 + i;
        if (q.tsizes[bt.c0 + i] == 0) continue;          // nothing to read back (the DEC kernels call an empty chunk malformed)
        if (b.status[i] == 1) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back under the new key: tag check failed", g);
        if (b.status[i] != 0) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back under the new key: size check failed", g);
        if (b.diff[i] != VERIFY_NO_DIFF)
            return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back under the new key: plaintext differs from byte %u", g, b.diff[i]);
    }
    return TSGPU_OK;
}

template <typename W>
static int rekey_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                        uint32_t n_chunks, const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                        const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs,
                        uint8_t* dst, uint64_t dst_cap, uint64_t part_size, W* part_crc, uint32_t part_cap, uint32_t* n_parts,
                        tsgpu_rekey_cursor* cursor, int object_ends_here, W* source_crc, W* object_crc) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!cursor) return fail(TSGPU_E_ARG, "cursor cannot be null");
    if (object_ends_here && (!source_crc || !object_crc))
        return fail(TSGPU_E_ARG, "source_%s/object_%s cannot be null", crc_arg<W>(), crc_arg<W>());
    if (flags & ~TSGPU_FLAG_VERIFY) return fail(TSGPU_E_ARG, "unknown flags %u: only TSGPU_FLAG_VERIFY applies to a rekey", flags);
    if (n_chunks && !transformed_sizes) return fail(TSGPU_E_ARG, "chunks cannot be null");
    if (int rc = aes_args_ok(TSGPU_FLAG_AES, AES_DEC, from_key, true, from_aad, from_aad_len)) return rc;
    if ((uint64_t)c->max_batch * c->slot_stride > 0xffffff00ull)
        return fail(TSGPU_E_ARG, "part checksums need batches below 4 GiB: max_batch %u x slot stride %llu is more", c->max_batch,
                    (unsigned long long)c->slot_stride);
    RekeyCarry<W> cur;
    memcpy(&cur, cursor, sizeof cur);
    uint64_t need = 0;
    for (uint32_t i = 0; i < n_chunks; i++) {
        // a chunk goes into one transformed slot (what tsgpu_detransform reads one into)
        if (transformed_sizes[i] > c->slot_stride - TSGPU_SLOT_HEAD - 16)
            return fail(TSGPU_E_ARG, "chunk %llu: transformed chunk of %u bytes exceeds the context's capacity",
                        (unsigned long long)(cur.chunks + i), transformed_sizes[i]);
        need += transformed_sizes[i];
    }
    if (int rc = aes_args_ok(TSGPU_FLAG_AES, AES_TO, to_key, !need || to_ivs, to_aad, to_aad_len)) return rc;   // empty chunks take no IV
    if (need && !src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (need > src_len) return fail(TSGPU_E_SHORT, "Stream has fewer bytes than expected");
    if (need && !dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (need > dst_cap) return fail(TSGPU_E_SHORT, "dst too small: the window's chunks are %llu bytes, dst_cap is %llu",
                                    (unsigned long long)need, (unsigned long long)dst_cap);
    if (need) {
        if (int rc = new_ivs_ok(to_ivs, n_chunks, src, transformed_sizes, memcmp(from_key, to_key, 32) == 0, cur.chunks,
                                /*skip_empty=*/true)) return rc;
    }
    PartsRun<W> run;
    if (int rc = parts_begin(run, PartsReq<W>{part_size, &cur.out, part_crc, part_cap, n_parts, object_crc}, TSGPU_FLAG_AES, need,
                             object_ends_here)) return rc;
    RekeyReq q;
    q.verify = (flags & TSGPU_FLAG_VERIFY) || c->verify_default;
    q.src = src; q.tsizes = transformed_sizes;
    q.rk_old = aes256_expand_key(from_key); q.rk_new = aes256_expand_key(to_key);
    q.aad_old = from_aad; q.aad_old_len = from_aad_len; q.aad_new = to_aad; q.aad_new_len = to_aad_len;
    q.ivs = to_ivs;
    if (need) {                                                            // a window of empty chunks writes nothing
        uint64_t dst_off = 0;
        const int rc = run_batches(c, n_chunks, transformed_sizes,
            [&](const Batch& bt) { return rekey_issue<W>(c, bt, q); },
            [&](const Batch& bt) {
                { int r = rekey_verdict(bt, q, cur.chunks); if (r) return r; }
                uint64_t obj = 0;
                for (uint32_t i = 0; i < bt.nb; i++) obj += transformed_sizes[bt.c0 + i];
                cur.src_raw = crc_shift(cur.src_raw, obj, 0) ^ reinterpret_cast<const W*>(bt.w->back.words)[0];
                return target_drain<W>(c, bt, nullptr, &run, dst, dst_cap, dst_off);
            },
            [&](const std::vector<Work*>& slots, int rcb) { return parts_idle(&run, slots, rcb); });
        if (rc) return rc;
    }
    cur.chunks += n_chunks;
    cur.src_len += need;
    parts_finish(run, object_ends_here);                                   // writes cur.out and the part CRCs
    if (object_ends_here) *source_crc = crc_finish(cur.src_raw, cur.src_len, 0);
    memcpy(cursor, &cur, sizeof cur);
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

extern "C" int tsgpu_rekey_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* transformed_sizes,
                                  uint32_t n_chunks, const uint8_t from_key[32], const uint8_t* from_aad, uint32_t from_aad_len,
                                  const uint8_t to_key[32], const uint8_t* to_aad, uint32_t to_aad_len, const uint8_t* to_ivs,
                                  uint8_t* dst, uint64_t dst_cap, uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap,
                                  uint32_t* n_parts, tsgpu_rekey_cursor* cursor, int object_ends_here, uint32_t* source_crc32c,
                                  uint32_t* object_crc32c) {
    return rekey_object(c, flags, src, src_len, transformed_sizes, n_chunks, from_key, from_aad, from_aad_len, to_key, to_aad,
                        to_aad_len, to_ivs, dst, dst_cap, part_size, part_crc32c, part_cap, n_parts, cursor, object_ends_here,
                        source_crc32c, object_crc32c);
}

extern "C" int tsgpu_rekey_object_crc64(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len,
                                        const uint32_t* transformed_sizes, uint32_t n_chunks, const uint8_t from_key[32],
                                        const uint8_t* from_aad, uint32_t from_aad_len, const uint8_t to_key[32], const uint8_t* to_aad,
                                        uint32_t to_aad_len, const uint8_t* to_ivs, uint8_t* dst, uint64_t dst_cap, uint64_t part_size,
                                        uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts, tsgpu_rekey_cursor* cursor,
                                        int object_ends_here, uint64_t* source_crc64, uint64_t* object_crc64) {
    return rekey_object(c, flags, src, src_len, transformed_sizes, n_chunks, from_key, from_aad, from_aad_len, to_key, to_aad,
                        to_aad_len, to_ivs, dst, dst_cap, part_size, part_crc64, part_cap, n_parts, cursor, object_ends_here,
                        source_crc64, object_crc64);
}

// ------------------------------------------------------------------------------------------ object encryption (host)
// tsgpu_encrypt_object: a stored unencrypted object's chunks (frames or plain chunks) encrypted with nothing decoded.  Per batch,
// on the compute stream: each chunk into its d_xf slot where its ciphertext goes (c_off + 12, a_off / a_len), [VERIFY: again
// into its d_frames slot,] pcrc over them where they sit (the source word), [ZSTD: frame_walk over them,] the GCM encrypt stage
// in place (each 16-byte block is read once, by the thread that then writes its ciphertext over it), IV and tag around it, [VERIFY:
// the DEC kernels decrypt the new chunks into d_pack at the frame slots' offsets and verify_compare compares them with the copy,]
// pack_chunks into d_pack and pcrc_tiles over it.  d_orig, the decoder and the compressor are never involved.  At the drain, in
// object order: the frame statuses and the sizes against the chunk index, the verify verdict, then the source word extends the
// carry and target_drain cuts the part prefixes and copies the batch out.

// The encrypt cursor holds what the rekey cursor holds: the new object's parts, the chunk count and the source's CRC and length.
static_assert(sizeof(RekeyCarry<uint32_t>) == sizeof(tsgpu_encrypt_cursor) && sizeof(RekeyCarry<uint64_t>) == sizeof(tsgpu_encrypt_cursor),
              "the cursor holds the carry");

struct EncryptReq {
    bool zstd, verify;
    bool indexed;                    // a .log object: its chunks are checked against the chunk index
    ChunkLayout index;
    const uint8_t* src; const uint32_t* tsizes;
    Aes256RoundKeys rk;
    const uint8_t* aad; uint32_t aad_len;
    const uint8_t* ivs;
};

template <typename W>
static int encrypt_issue(tsgpu_ctx* c, const Batch& bt, const EncryptReq& q) {
    Work& w = *bt.w;
    const uint32_t c0 = bt.c0, nb = bt.nb;
    RT(rt::set_device(w.device));
    rt::stream_t st = w.stream;
    memcpy(w.hd.ivs, q.ivs + (size_t)c0 * TSGPU_IV_SIZE, (size_t)nb * TSGPU_IV_SIZE);
    if (q.aad_len) memcpy(w.hd.aad, q.aad, q.aad_len);
    slot_layout(c, w.hd, nb, c->slot_stride);
    uint64_t at = bt.in_off, obj = 0, out = 0;
    uint32_t max_t = 0;
    for (uint32_t i = 0; i < nb; i++) {  // the sizes were bounded by the slot before any GPU work
        const uint32_t t = q.tsizes[c0 + i];
        w.hd.a_off[i] = w.hd.c_off[i] + TSGPU_IV_SIZE;
        w.hd.a_len[i] = t;
        w.hd.c_len[i] = w.back.sizes[i] = t ? t + TSGPU_IV_SIZE + TSGPU_TAG_SIZE : 0;   // an empty chunk stays empty
        if (t) {
            RT(rt::h2d(w.d_xf + w.hd.a_off[i], q.src + at, t, st));
            if (q.verify) RT(rt::h2d(w.d_frames + w.hd.b_off[i], q.src + at, t, st));
        }
        at += t; obj += t; out += w.hd.c_len[i];
        max_t = std::max(max_t, t);
    }
    RT(rt::h2d(w.d_desc, w.h_desc, w.desc_bytes, st));
    // the slot's previous batch may still be copying d_pack out, its part prefixes read from the pcrc scratch this batch rewrites
    { int rcw = wait_copies_out(w, st); if (rcw) return rcw; }
    const ChunksIn in{w.d_xf, w.dd.a_off, w.dd.a_len};
    { int rc = check_crc_word<W, true>(c, w, st, in.base, in.off, in.len, nb, obj, 0); if (rc) return rc; }
    RT(rt::d2h(w.back.words, pcrc_of<W>(w).d_cuts, sizeof(W), st));
    if (q.zstd) {
        FrameWalkArgs F;
        F.base = in.base; F.off = in.off; F.len = in.len; F.status = w.dd.status; F.fcs = w.dd.v_len; F.n = nb;
        TS_LAUNCH_P(c->prof, "frame_walk", frame_walk_kernel, dim3((nb + FW_T - 1) / FW_T), dim3(FW_T), 0, st, F);
        CHECK_LAUNCH("frame_walk_kernel");
        RT(rt::d2h(w.back.src_status, w.dd.status, 4ull * nb, st));
        RT(rt::d2h(w.back.src_sizes, w.dd.v_len, 4ull * nb, st));
    }
    // the GCM stage writes every chunk's IV || CT || TAG, an empty chunk's 28 bytes included; c_len (what pack, the part checksums
    // and VERIFY read) keeps the sizes the chunks leave with, and the stage's own sizes go to b_len, which nothing reads after it
    { int rc = gcm_stage<true>(c, w, w.keys[0], st, q.rk, in, ChunksOut{w.d_xf, w.dd.c_off, w.dd.b_len}, q.aad_len, w.dd.status, nb,
                               max_t, 0xffffffffu); if (rc) return rc; }
    const ChunksOut fin{w.d_xf, w.dd.c_off, w.dd.c_len};
#ifdef TSGPU_SIMT
    simt_flip("TSGPU_SIMT_FLIP", fin, c0, nb);
#endif
    if (q.verify) {                      // the new chunks read back, against the copy of their source in the frame slots
        RT(rt::memset_async(w.dd.status, 0, 4ull * nb, st));
        RT(rt::memset_async(w.dd.v_diff, 0xff, 4ull * nb, st));
        int rc = gcm_stage<false>(c, w, w.keys[0], st, q.rk, fin, ChunksOut{w.d_pack, w.dd.b_off, w.dd.v_len}, q.aad_len, w.dd.status,
                                  nb, max_t + TSGPU_IV_SIZE + TSGPU_TAG_SIZE, (uint32_t)(c->frame_stride - 16));
        if (rc) return rc;
        VerifyArgs V;
        V.orig = w.d_frames; V.orig_off = w.dd.b_off; V.orig_len = w.dd.a_len;
        V.back = w.d_pack; V.back_off = w.dd.b_off; V.back_len = w.dd.v_len;
        V.status = w.dd.status; V.diff = w.dd.v_diff;
        TS_LAUNCH_P(c->prof, "verify_compare", verify_compare_kernel, dim3(std::max(1u, (max_t + VERIFY_PIECE - 1) / VERIFY_PIECE), nb),
                    dim3(VERIFY_T), 0, st, V);
        CHECK_LAUNCH("verify_compare_kernel");
        RT(rt::d2h(w.back.status, w.dd.status, 4ull * nb, st));
        RT(rt::d2h(w.back.diff, w.dd.v_diff, 4ull * nb, st));
    }
    PackArgs P;
    P.base = w.d_xf; P.stride = c->slot_stride; P.head = TSGPU_SLOT_HEAD; P.len = w.dd.c_len; P.n = nb; P.out = w.d_pack;
    const uint32_t longest = max_t + TSGPU_IV_SIZE + TSGPU_TAG_SIZE;
    TS_LAUNCH_P(c->prof, "pack_chunks", pack_chunks_kernel, dim3((longest + PACK_PIECE - 1) / PACK_PIECE, nb), dim3(PACK_T), 0, st, P);
    CHECK_LAUNCH("pack_chunks_kernel");
    { int rc = parts_stage<W>(c, w, st, w.dd.c_len, nb, out); if (rc) return rc; }
    RT(rt::event_record(w.ev_sizes, st));
    return TSGPU_OK;
}

// A drained batch's verdicts in object order: every chunk's frame and size against the chunk index, then (VERIFY) every
// read-back.  `first`: the object's number of the call's first chunk.
static int encrypt_verdict(const Batch& bt, const EncryptReq& q, uint64_t first) {
    const Back& b = bt.w->back;
    if (q.indexed) {
        for (uint32_t i = 0; i < bt.nb; i++) {
            const unsigned long long g = first + bt.c0 + i;
            const uint32_t t = q.tsizes[bt.c0 + i];
            if (q.zstd && t && b.src_status[i]) return fail(TSGPU_E_CORRUPT, "Invalid zstd frame in chunk %llu (code %u)", g, b.src_status[i]);
            if (int rc = index_size_ok(q.index, g, q.zstd && t ? b.src_sizes[i] : t)) return rc;
        }
    }
    if (!q.verify) return TSGPU_OK;
    for (uint32_t i = 0; i < bt.nb; i++) {
        const unsigned long long g = first + bt.c0 + i;
        if (q.tsizes[bt.c0 + i] == 0) continue;          // nothing to read back (the DEC kernels call an empty chunk malformed)
        if (b.status[i] == 1) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: tag check failed", g);
        if (b.status[i] != 0) return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: size check failed", g);
        if (b.diff[i] != VERIFY_NO_DIFF)
            return fail(TSGPU_E_VERIFY, "verify: chunk %llu did not read back: bytes differ from offset %u", g, b.diff[i]);
    }
    return TSGPU_OK;
}

template <typename W>
static int encrypt_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* chunk_sizes,
                          uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size, const uint8_t key[32],
                          const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs, uint8_t* dst, uint64_t dst_cap,
                          uint32_t* new_transformed_sizes, uint64_t part_size, W* part_crc, uint32_t part_cap, uint32_t* n_parts,
                          tsgpu_encrypt_cursor* cursor, int object_ends_here, W* source_crc, W* object_crc) try {
    if (!c) return fail(TSGPU_E_ARG, "ctx cannot be null");
    if (!cursor) return fail(TSGPU_E_ARG, "cursor cannot be null");
    if (object_ends_here && (!source_crc || !object_crc))
        return fail(TSGPU_E_ARG, "source_%s/object_%s cannot be null", crc_arg<W>(), crc_arg<W>());
    if (flags & TSGPU_FLAG_AES)
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_AES: the object is already encrypted; tsgpu_rekey_object re-encrypts it under a new key");
    if (flags & ~(TSGPU_FLAG_ZSTD | TSGPU_FLAG_VERIFY))
        return fail(TSGPU_E_ARG, "unknown flags %u: only TSGPU_FLAG_ZSTD and TSGPU_FLAG_VERIFY apply to an encryption", flags);
    if ((flags & TSGPU_FLAG_ZSTD) && original_chunk_size == 0)
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_ZSTD needs the chunk index (original_chunk_size > 0): an .indexes object is not compressed");
    if (n_chunks && !chunk_sizes) return fail(TSGPU_E_ARG, "chunks cannot be null");
    if (n_chunks && !new_transformed_sizes) return fail(TSGPU_E_ARG, "new_transformed_sizes cannot be null");
    if ((uint64_t)c->max_batch * c->slot_stride > 0xffffff00ull)
        return fail(TSGPU_E_ARG, "part checksums need batches below 4 GiB: max_batch %u x slot stride %llu is more", c->max_batch,
                    (unsigned long long)c->slot_stride);
    RekeyCarry<W> cur;
    memcpy(&cur, cursor, sizeof cur);
    uint64_t need = 0, out = 0;
    for (uint32_t i = 0; i < n_chunks; i++) {
        const uint32_t t = chunk_sizes[i];
        // the new chunk goes into one transformed slot (what tsgpu_detransform reads one into)
        if ((uint64_t)t + TSGPU_IV_SIZE + TSGPU_TAG_SIZE > c->slot_stride - TSGPU_SLOT_HEAD - 16)
            return fail(TSGPU_E_ARG, "chunk %llu: a chunk of %u bytes encrypted exceeds the context's capacity",
                        (unsigned long long)(cur.chunks + i), t);
        need += t;
        out += t ? (uint64_t)t + TSGPU_IV_SIZE + TSGPU_TAG_SIZE : 0;
    }
    if (int rc = aes_args_ok(TSGPU_FLAG_AES, AES_ENC, key, !need || ivs, aad, aad_len)) return rc;   // empty chunks take no IV
    if (need && !src) return fail(TSGPU_E_ARG, "inputStream cannot be null");
    if (need > src_len) return fail(TSGPU_E_SHORT, "Stream has fewer bytes than expected");
    if (need && !dst) return fail(TSGPU_E_ARG, "dst cannot be null");
    if (out > dst_cap) return fail(TSGPU_E_SHORT, "dst too small: the window's new chunks are %llu bytes, dst_cap is %llu",
                                   (unsigned long long)out, (unsigned long long)dst_cap);
    if (need) {
        if (int rc = new_ivs_ok(ivs, n_chunks, src, chunk_sizes, /*same_key=*/false, cur.chunks, /*skip_empty=*/true)) return rc;
    }
    PartsRun<W> run;
    if (int rc = parts_begin(run, PartsReq<W>{part_size, &cur.out, part_crc, part_cap, n_parts, object_crc}, TSGPU_FLAG_AES, out,
                             object_ends_here)) return rc;
    EncryptReq q;
    q.zstd = flags & TSGPU_FLAG_ZSTD;
    q.verify = (flags & TSGPU_FLAG_VERIFY) || c->verify_default;
    q.indexed = original_chunk_size > 0;
    q.index = ChunkLayout{original_chunk_size, original_file_size,
                          original_chunk_size ? (original_file_size + original_chunk_size - 1) / original_chunk_size : 0};
    q.src = src; q.tsizes = chunk_sizes;
    q.rk = aes256_expand_key(key);
    q.aad = aad; q.aad_len = aad_len; q.ivs = ivs;
    // The index of an empty segment materialises one chunk of 0 bytes: a caller that walks it passes that chunk.
    uint32_t n = n_chunks;
    if (q.indexed && q.index.count == 0 && cur.chunks == 0 && n == 1 && chunk_sizes[0] == 0) n = 0;
    if (q.indexed && !need) {                                              // no GPU work: the sizes are checked here
        for (uint32_t i = 0; i < n; i++) if (int rc = index_size_ok(q.index, cur.chunks + i, 0)) return rc;
    }
    if (need) {                                                            // a window of empty chunks writes nothing
        uint64_t dst_off = 0;
        const int rc = run_batches(c, n, chunk_sizes,
            [&](const Batch& bt) { return encrypt_issue<W>(c, bt, q); },
            [&](const Batch& bt) {
                { int r = encrypt_verdict(bt, q, cur.chunks); if (r) return r; }
                uint64_t obj = 0;
                for (uint32_t i = 0; i < bt.nb; i++) obj += chunk_sizes[bt.c0 + i];
                cur.src_raw = crc_shift(cur.src_raw, obj, 0) ^ reinterpret_cast<const W*>(bt.w->back.words)[0];
                return target_drain<W>(c, bt, nullptr, &run, dst, dst_cap, dst_off);
            },
            [&](const std::vector<Work*>& slots, int rcb) { return parts_idle(&run, slots, rcb); });
        if (rc) return rc;
    }
    cur.chunks += n;
    cur.src_len += need;
    if (object_ends_here && q.indexed) { if (int rc = index_count_ok(q.index, cur.chunks)) return rc; }
    for (uint32_t i = 0; i < n_chunks; i++)
        new_transformed_sizes[i] = chunk_sizes[i] ? chunk_sizes[i] + TSGPU_IV_SIZE + TSGPU_TAG_SIZE : 0;
    parts_finish(run, object_ends_here);                                   // writes cur.out and the part CRCs
    if (object_ends_here) *source_crc = crc_finish(cur.src_raw, cur.src_len, 0);
    memcpy(cursor, &cur, sizeof cur);
    return TSGPU_OK;
} catch (const std::bad_alloc&) { return fail(TSGPU_E_NOMEM, "out of memory"); }

extern "C" int tsgpu_encrypt_object(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* chunk_sizes,
                                    uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size,
                                    const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                    uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                                    uint64_t part_size, uint32_t* part_crc32c, uint32_t part_cap, uint32_t* n_parts,
                                    tsgpu_encrypt_cursor* cursor, int object_ends_here, uint32_t* source_crc32c, uint32_t* object_crc32c) {
    return encrypt_object(c, flags, src, src_len, chunk_sizes, n_chunks, original_chunk_size, original_file_size, key, aad, aad_len,
                          ivs, dst, dst_cap, new_transformed_sizes, part_size, part_crc32c, part_cap, n_parts, cursor, object_ends_here,
                          source_crc32c, object_crc32c);
}

extern "C" int tsgpu_encrypt_object_crc64(tsgpu_ctx* c, uint32_t flags, const uint8_t* src, uint64_t src_len, const uint32_t* chunk_sizes,
                                          uint32_t n_chunks, uint32_t original_chunk_size, uint64_t original_file_size,
                                          const uint8_t key[32], const uint8_t* aad, uint32_t aad_len, const uint8_t* ivs,
                                          uint8_t* dst, uint64_t dst_cap, uint32_t* new_transformed_sizes,
                                          uint64_t part_size, uint64_t* part_crc64, uint32_t part_cap, uint32_t* n_parts,
                                          tsgpu_encrypt_cursor* cursor, int object_ends_here, uint64_t* source_crc64, uint64_t* object_crc64) {
    return encrypt_object(c, flags, src, src_len, chunk_sizes, n_chunks, original_chunk_size, original_file_size, key, aad, aad_len,
                          ivs, dst, dst_cap, new_transformed_sizes, part_size, part_crc64, part_cap, n_parts, cursor, object_ends_here,
                          source_crc64, object_crc64);
}

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
    if (flags & TSGPU_FLAG_VALIDATE_RECORDS)
        return fail(TSGPU_E_ARG, "TSGPU_FLAG_VALIDATE_RECORDS (%u) applies to the host-buffer segment transform only", TSGPU_FLAG_VALIDATE_RECORDS);
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
    if ((rc = aes_args_ok(flags, AES_ENC, key, ivs != nullptr, aad, aad_len))) return rc;
    const uint32_t nb = (uint32_t)n64, cs = chunk_size;
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);
    rt::stream_t st = (rt::stream_t)stream;
    SlotClaim claim;
    rc = dev_call_begin(c, device_index, st, claim, [&](Work& w) {
        for (uint32_t i = 0; i < nb; i++) {
            w.hd.a_off[i] = (uint64_t)i * cs;
            w.hd.a_len[i] = (uint32_t)std::min<uint64_t>(cs, src_len - (uint64_t)i * cs);
        }
        slot_layout(c, w.hd, nb, slot_stride);
        if (flags & TSGPU_FLAG_AES) {
            memcpy(w.hd.ivs, ivs, (size_t)nb * TSGPU_IV_SIZE);
            if (aad_len) memcpy(w.hd.aad, aad, aad_len);
        }
    });
    if (rc) return rc;
    Work& w = *claim.slots[0];
    rc = transform_enqueue(c, w, w.keys[0], st, flags, nb, cs, rk, aad_len, ChunksIn{d_src, w.dd.a_off, w.dd.a_len},
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
    flags &= ~ZSTD_MODIFIERS;                                // how a frame was compressed does not matter to the reader
    if ((rc = aes_args_ok(flags, AES_DEC, key, true, aad, aad_len))) return rc;
    if (!d_slots || !d_transformed_sizes || !d_dst || !d_original_sizes || !d_status) return fail(TSGPU_E_ARG, "null device pointer");
    Aes256RoundKeys rk{};
    if (flags & TSGPU_FLAG_AES) rk = aes256_expand_key(key);
    rt::stream_t st = (rt::stream_t)stream;
    SlotClaim claim;
    rc = dev_call_begin(c, device_index, st, claim, [&](Work& w) {
        slot_layout(c, w.hd, n_chunks, slot_stride);
        for (uint32_t i = 0; i < n_chunks; i++) w.hd.a_off[i] = (uint64_t)i * chunk_size;     // original side: chunk i at i * chunk_size
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
    rc = detransform_enqueue(c, w, w.keys[0], st, flags, n_chunks, rk, aad_len, ChunksIn{d_slots, w.dd.c_off, d_transformed_sizes},
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
