"""Runs the REAL zstd compressor/decompressor kernel sources under the test-only SIMT emulator (tests/simt/)
through the C-ABI and checks them against the oracle (system libzstd): our frames decode with libzstd, libzstd's
level-3 frames decode with ours, Frame_Content_Size is present, corrupt input is an error and never a crash.
Logic check for the GPU-less build box; the -m gpu tests repeat this on an H100 at full sizes."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import oracle as ora
import tsgpu
from tsgpu import binding, corpus
from executor_shapes import executor_shapes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    c = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=SIMT_LIB)
    yield c
    c.close()


def _mixed(n, seed):
    rng = np.random.default_rng(seed)
    src = rng.integers(0, 256, n, dtype=np.uint8)
    src[: n // 2] = corpus.gen_chunk("K", seed, 0, n // 2)
    if n > 4000:
        src[n // 2: n // 2 + 1500] = 7            # a run inside the random half
    return src


CASES = [("K", 1, 0), ("K", 4, 0), ("K", 5, 0), ("K", 255, 0), ("K", 256, 0), ("K", 300, 0), ("K", 16383, 0),
         ("K", 16384, 0), ("K", 16385, 0), ("K", 65791, 0), ("K", 65792, 0), ("R", 40000, 0), ("Z", 70000, 32768),
         ("K", 200000, 65536), ("M", 150000, 50000), ("K", 1 << 20, 1 << 20), ("R", 300000, 1 << 17)]


@pytest.mark.parametrize("kind,n,cs", CASES)
def test_simt_zstd_both_directions(ctx, kind, n, cs):
    src = _mixed(n, 11) if kind == "M" else corpus.gen_segment(kind, 0, n, cs if cs else n)
    out, sizes = ctx.transform(Z, src, cs)
    c = cs if cs else n
    pos = 0
    for i, s in enumerate(sizes):
        frame = out[pos:pos + s]
        pos += s
        want = src[i * c:min(n, (i + 1) * c)]
        assert ora.zstd_content_size(frame) == want.size
        assert ora.zstd_decompress_chunk(frame) == want.tobytes()
    back, osz = ctx.detransform(Z, out, sizes, n)
    assert np.array_equal(back, src)
    ref, rs = ora.transform_segment(Z, src, cs)
    back, osz = ctx.detransform(Z, ref, rs, n)
    assert np.array_equal(back, src)


def test_simt_frame_headers_match_libzstd_choice(ctx):
    # same Frame_Header_Descriptor / FCS field width libzstd picks for a pledged size (golden vector form 28B52FFD 20 0F)
    for n in (15, 255, 256, 65791, 65792, 300000):
        src = corpus.gen_chunk("K", 1, 0, n)
        mine, _ = ctx.transform(Z, src, 0)
        ref = ora.zstd_compress_chunk(src)
        hl = 6 if n < 256 else 7 if n < 65792 else 9
        assert bytes(mine[:hl]) == ref[:hl]


@pytest.mark.parametrize("flags", [Z | A])
@pytest.mark.parametrize("cs", [0, 1, 13, 1024, 5123, 60000])
def test_simt_full_chain_round_trip(ctx, flags, cs):
    n = 60001 if cs == 0 or cs >= 1024 else 300
    src = _mixed(n, cs + 3)
    rng = np.random.default_rng(cs)
    nch = (n + cs - 1) // cs if cs else 1
    key, aad, ivs = rng.bytes(32), rng.bytes(32), rng.bytes(12 * nch)
    got, gs = ctx.transform(flags, src, cs, key, aad, ivs)
    back_ref, _ = ora.detransform_chunks(flags, got, gs, n, key, aad)
    assert np.array_equal(back_ref, src)
    ref, rs = ora.transform_segment(flags, src, cs, key, aad, ivs)
    back, _ = ctx.detransform(flags, ref, rs, n, key, aad)
    assert np.array_equal(back, src)
    back2, _ = ctx.detransform(flags, got, gs, n, key, aad)
    assert np.array_equal(back2, src)


def test_simt_corrupt_frames_never_crash(ctx):
    src = corpus.gen_chunk("K", 5, 0, 120000)
    for frame in (np.frombuffer(ora.zstd_compress_chunk(src), dtype=np.uint8), ctx.transform(Z, src, 0)[0]):
        rng = np.random.default_rng(1)
        for trial in range(40):
            bad = frame.copy()
            where = int(rng.integers(0, len(bad)))
            bad[where] ^= 1 << int(rng.integers(0, 8))
            try:
                back, osz = ctx.detransform(Z, bad, [len(bad)], len(src))
            except tsgpu.TsgpuError as e:
                assert e.code == binding.E_CORRUPT
            else:
                assert len(back) == len(src)
        for cut in (3, 5, 9, len(frame) // 2, len(frame) - 1):
            with pytest.raises(tsgpu.TsgpuError) as e:
                ctx.detransform(Z, frame[:cut], [cut], len(src))
            assert e.value.code == binding.E_CORRUPT


def test_simt_frame_without_content_size_is_invalid(ctx):
    # DecompressionChunkEnumeration.java:41-44: "Invalid decompressed size"
    frame = bytes.fromhex("28b52ffd") + bytes([0x00, 0x58]) + bytes([0x01 | (0 << 1) | (3 << 3), 0, 0]) + b"abc"
    with pytest.raises(tsgpu.TsgpuError) as e:
        ctx.detransform(Z, np.frombuffer(frame, dtype=np.uint8), [len(frame)], 100)
    assert e.value.code == binding.E_CORRUPT


def test_simt_reference_written_index_deserializes(ctx):
    sizes = [1000000 + (i * 7919) % 5000 for i in range(600)]
    assert ctx.transformed_chunks_deserialize(ora.transformed_chunks_serialize(sizes)) == sizes
    assert ctx.transformed_chunks_deserialize("KLUv/SAPeQAAAAAAAwAAAAoBAAoAAAAe") == [10, 20, 30]
    pos = ctx.chunk_positions(sizes)
    assert [int(p) for p in pos[:-1]] == [c[3] for c in ora.ChunkIndex.variable(1 << 20, 599 * (1 << 20) + 1, sizes).chunks()]


def test_simt_transformed_chunks_compressed_like_the_reference(ctx):
    # TransformedChunksSerializer.java:40-48 compresses the codec bytes; the ctx-taking serializer does so with the dense
    # compressor.  Both readers must accept the result, the golden vector must not change, and lists that repeat / cluster
    # must come out about as small as libzstd makes them (the Raw-block framing of the ctx-less call does not shrink them).
    rng = np.random.default_rng(5)
    lists = {"equal": [4194332] * 256, "clustered": (1350000 + rng.integers(-70000, 70000, 256)).tolist(),
             "tight": (1350000 + rng.integers(-700, 700, 1024)).tolist(), "golden": [10, 20, 30], "one": [123456]}
    for name, sizes in lists.items():
        mine, ref, raw = ctx.transformed_chunks_serialize(sizes), ora.transformed_chunks_serialize(sizes), binding.transformed_chunks_serialize(sizes, lib_path=SIMT_LIB)
        assert ora.transformed_chunks_deserialize(mine) == sizes, name           # the reference-side reader (libzstd)
        assert ctx.transformed_chunks_deserialize(mine) == sizes, name
        assert len(mine) <= len(raw), name
        if name == "golden":
            assert mine == ref == "KLUv/SAPeQAAAAAAAwAAAAoBAAoAAAAe"
        if name in ("equal", "clustered", "tight"):
            print(name, len(mine), len(ref), len(raw))
            assert len(mine) <= len(ref) + max(40, len(ref) // 10), (name, len(mine), len(ref), len(raw))
    js = json.loads(ctx.chunk_index_json(1 << 22, 255 * (1 << 22) + 5, None, sizes=lists["clustered"]))
    want = json.loads(ora.ChunkIndex.variable(1 << 22, 255 * (1 << 22) + 5, lists["clustered"]).to_json())
    assert list(js) == list(want) and all(js[k] == want[k] for k in js if k != "transformedChunks")
    assert ora.transformed_chunks_deserialize(js["transformedChunks"]) == lists["clustered"]


def test_simt_index_files_ride_one_ragged_batch(ctx):
    # RemoteStorageManager.transformIndex (RemoteStorageManager.java:455-490): each Kafka index is ONE chunk, encryption
    # only; the object is their concatenation and SegmentIndexesV1 records (position, size) of each transformed blob
    rng = np.random.default_rng(77)
    blobs = [rng.integers(0, 256, n, dtype=np.uint8) for n in (10485, 9000, 37, 126, 2048)]   # offset, time, snapshot, epoch, txn
    src = np.concatenate(blobs)
    key, aad, ivs = rng.bytes(32), rng.bytes(32), rng.bytes(12 * 5)
    out, sizes = ctx.transform_chunks(A, src, [b.size for b in blobs], key, aad, ivs)
    assert sizes == [b.size + 28 for b in blobs]
    pos = 0
    for i, b in enumerate(blobs):
        want = ora.aesgcm_encrypt_chunk(key, ivs[12 * i:12 * i + 12], aad, b)
        assert bytes(out[pos:pos + sizes[i]]) == want            # bit-exact with the reference-side cipher
        pos += sizes[i]
    back, osz = ctx.detransform(A, out, sizes, src.size, key, aad)      # fetchIndexBytes direction
    assert np.array_equal(back, src) and osz == [b.size for b in blobs]
    with pytest.raises(tsgpu.TsgpuError):
        ctx.transform_chunks(A, src, [10, 0, 5], key, aad, ivs)


def test_simt_frame_header_fields_refused_like_libzstd(ctx):
    # header fields a reader without a dictionary has to refuse, exactly where libzstd does: a Dictionary_ID other than 0
    # ("Dictionary mismatch"), a Window_Descriptor above windowLog 31; a zero Dictionary_ID field and windowLog 31 are fine
    src = corpus.gen_segment("K", 1, 600000, 600000)
    f = np.frombuffer(ora.zstd_compress_level(src, 1), dtype=np.uint8).copy()
    assert f[4] & 0x20 == 0                                          # not Single_Segment: byte 5 is the Window_Descriptor
    small = corpus.gen_segment("K", 1, 9000, 9000)
    f2 = np.frombuffer(ora.zstd_compress_level(small, 3), dtype=np.uint8).copy()
    assert f2[4] & 0x20
    u8 = lambda *v: np.array(v, np.uint8)
    cases = [("plain", f, src), ("windowLog 32", np.concatenate([f[:5], u8(22 << 3), f[6:]]), src),
             ("windowLog 31", np.concatenate([f[:5], u8(21 << 3), f[6:]]), src),
             ("dictionary id 7", np.concatenate([f[:4], u8(f[4] | 1), f[5:6], u8(7), f[6:]]), src),
             ("dictionary id field 0", np.concatenate([f[:4], u8(f[4] | 1), f[5:6], u8(0), f[6:]]), src),
             ("single segment, dictionary id 257", np.concatenate([f2[:4], u8(f2[4] | 2), u8(1, 1), f2[5:]]), small),
             ("reserved bit", np.concatenate([f2[:4], u8(f2[4] | 8), f2[5:]]), small)]
    for name, frame, want in cases:
        frame = np.ascontiguousarray(frame)
        try:
            ref_ok = ora.zstd_decompress_chunk(frame) == want.tobytes()
        except Exception:
            ref_ok = False
        try:
            back, _ = ctx.detransform(Z, frame, [frame.size], want.size)
            mine_ok = bool(np.array_equal(back, want))
        except tsgpu.TsgpuError as e:
            assert e.code == binding.E_CORRUPT
            mine_ok = False
        assert mine_ok == ref_ok, (name, ref_ok, mine_ok)
        assert ref_ok == (name in ("plain", "windowLog 31", "dictionary id field 0")), name


def test_simt_content_checksum_is_verified_like_libzstd(ctx):
    # zstd-jni's Zstd.decompress verifies the Content_Checksum (low 32 bits of XXH64 of the content) when a frame announces one; the
    # reference's writer never does, a foreign writer (zstd CLI default) may: accepted when right, refused when wrong — as libzstd does
    for n in (1, 31, 32, 33, 100, 8192, 70001, 300000):
        src = corpus.gen_segment("K", n % 97, n, n)
        for level in (1, 3):
            f = np.frombuffer(ora.zstd_compress_checksum(src, level), dtype=np.uint8)
            assert f[4] & 4
            back, _ = ctx.detransform(Z, f, [f.size], n)
            assert np.array_equal(back, src), (n, level)
            bad = f.copy()
            bad[-1 - (n % 4)] ^= 0x21
            with pytest.raises(Exception):
                ora.zstd_decompress_chunk(bad)
            with pytest.raises(tsgpu.TsgpuError) as e:
                ctx.detransform(Z, bad, [bad.size], n)
            assert e.value.code == binding.E_CORRUPT


def test_simt_bytes_after_the_frame_are_refused_like_libzstd(ctx):
    # DecompressionChunkEnumeration.java:41-45 hands the whole chunk to Zstd.decompress(chunk, size): libzstd refuses bytes after the
    # frame ("Src size is incorrect") and a second frame ("Destination buffer is too small"), and steps over skippable frames
    src = corpus.gen_segment("K", 3, 9000, 9000)
    skippable = np.frombuffer(bytes([0x53, 0x2A, 0x4D, 0x18, 3, 0, 0, 0, 9, 9, 9]), dtype=np.uint8)
    frames = {"libzstd": np.frombuffer(ora.zstd_compress_level(src, 3), dtype=np.uint8)}
    for name, flags in (("speed", Z), ("dense", Z | tsgpu.FLAG_ZSTD_DENSE)):
        out, sizes = ctx.transform(flags, src, 0)
        frames[name] = np.array(out[:sizes[0]], copy=True)
    for name, f in frames.items():
        for what, tail, accepted in (("exact", np.zeros(0, np.uint8), True), ("garbage", np.array([1, 2, 3, 4, 5], np.uint8), False),
                                     ("one byte", np.zeros(1, np.uint8), False), ("second frame", f, False),
                                     ("skippable frame", skippable, True), ("truncated skippable frame", skippable[:9], False)):
            chunk = np.concatenate([f, tail])
            try:
                ref_ok = ora.zstd_decompress_chunk(chunk) == src.tobytes()
            except Exception:
                ref_ok = False
            assert ref_ok == accepted, (name, what)                       # the expectation IS libzstd's behaviour
            try:
                back, _ = ctx.detransform(Z, chunk, [chunk.size], 9000)
                mine_ok = np.array_equal(back, src)
            except tsgpu.TsgpuError as e:
                assert e.code == binding.E_CORRUPT
                mine_ok = False
            assert mine_ok == accepted, (name, what)


@pytest.mark.parametrize("mode", [0, tsgpu.FLAG_ZSTD_DENSE])
def test_simt_matches_that_end_at_the_block_end(ctx, mode):
    # the per-lane extension measures 16 bytes past a position and the warp-wide one 128 per probe, both clamped to the block:
    # matches that run exactly to the last byte of a block / slice / chunk, for every alignment of that end
    rng = np.random.default_rng(21)
    head = rng.integers(0, 256, 3000, dtype=np.uint8)
    for n in [3000 + k for k in (5, 6, 7, 8, 15, 16, 17, 19, 20, 21, 130, 131)] + [8189, 8190, 8191, 8192, 8193, 8197, 16383, 16384 + 5, 65536, 65536 + 11]:
        src = np.concatenate([head, np.resize(head[:1000], n - 3000)]) if n > 3000 else head[:n]
        out, sizes = ctx.transform(Z | mode, src, 0)
        assert ora.zstd_decompress_chunk(out[:sizes[0]]) == src.tobytes(), n
        assert sizes[0] < n // 2 or n < 3200, (n, sizes)
        back, _ = ctx.detransform(Z, out, sizes, n)
        assert np.array_equal(back, src), n


def test_simt_straight_line_extension_is_the_same_parse(tmp_path):
    # The per-lane match extension of the speed-mode compressor exists as a loop (ZB_TUNE_STRAIGHT=0, the code until round 2)
    # and as straight-line branch-free code (=1, the product: faster on the GPU, see the ZB_TUNE_STRAIGHT note).  It is a restructuring, not a different
    # parse: with the emulator's fixed lane order both builds must emit identical frames.
    libs = {}
    for v in (0, 1):
        so = str(tmp_path / ("libtsgpu_simt_straight%d.so" % v))
        subprocess.check_call(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-DTSGPU_SIMT=1", "-DZB_TUNE_STRAIGHT=%d" % v,
                               "-I" + os.path.join(ROOT, "tests", "simt"), "-I" + os.path.join(ROOT, "tiered-storage-for-apache-kafka_b200", "csrc"),
                               "-x", "c++", os.path.join(ROOT, "tiered-storage-for-apache-kafka_b200", "csrc", "tsgpu.cu"),
                               os.path.join(ROOT, "tests", "simt", "simt.cpp"), "-o", so, "-Wno-unknown-pragmas"])
        libs[v] = so
    code = ("import sys, hashlib; sys.path.insert(0, %r); import numpy as np, tsgpu; from tsgpu import corpus\n"
            "c = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=sys.argv[1])\n"
            "h = hashlib.sha256()\n"
            "for kind, n, cs in (('K', 300000, 131072), ('K', 70001, 0), ('R', 40000, 0), ('Z', 70000, 32768), ('M', 150000, 50000)):\n"
            "    src = corpus.gen_segment(kind, 0, n, cs if cs else n) if kind != 'M' else np.concatenate([corpus.gen_chunk('K', 3, 0, n // 2), np.random.default_rng(3).integers(0, 256, n - n // 2, dtype=np.uint8)])\n"
            "    out, sizes = c.transform(1, src, cs)\n"
            "    h.update(out.tobytes()); h.update(repr(sizes).encode())\n"
            "print(h.hexdigest(), len(out))\n") % ROOT
    digests = {v: subprocess.check_output([sys.executable, "-c", code, libs[v]], text=True).strip() for v in (0, 1)}
    assert digests[0] == digests[1], digests


def test_simt_frames_do_not_depend_on_lane_order():
    # Retried uploads must produce identical objects (VERDICT r1 #9): in the dense mode (TSGPU_FLAG_ZSTD_DENSE) hash-slot
    # winners are the highest position of a step, so the frame bytes may not depend on which lane the hardware (here: the
    # emulator's scheduler) serves first.  (The speed mode keeps whichever lane wins: INTEGRATION.md says so.)
    code = ("import sys, hashlib; sys.path.insert(0, %r); import numpy as np, tsgpu; from tsgpu import corpus\n"
            "c = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=%r)\n"
            "h = hashlib.sha256()\n"
            "for kind, n, cs in (('K', 300000, 131072), ('K', 70001, 0), ('R', 40000, 0), ('Z', 70000, 32768)):\n"
            "    out, sizes = c.transform(1 | 4, corpus.gen_segment(kind, 0, n, cs if cs else n), cs)\n"
            "    h.update(out.tobytes()); h.update(repr(sizes).encode())\n"
            "print(h.hexdigest())\n") % (ROOT, SIMT_LIB)
    digests = set()
    for order in ("", "reverse", "random:7", "random:1234"):
        env = dict(os.environ)
        env.pop("TSGPU_SIMT_ORDER", None)
        if order:
            env["TSGPU_SIMT_ORDER"] = order
        out = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert out.returncode == 0, out.stderr[-2000:]
        digests.add(out.stdout.strip())
    assert len(digests) == 1, digests


def test_simt_decode_paths_libzstd_frames_and_own_regions():
    # entropy stage per block in parallel; libzstd-written frames are executed whole by one CTA, this library's frames region
    # by region in shared memory (DESIGN.md §4.3) — the path counters say which one ran
    c2 = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=SIMT_LIB)
    try:
        c2.profile_enable(True)
        for kind, n, level in (("K", 1 << 20, 3), ("K", 700000, 1), ("K", 700000, 19), ("M", 300000, 3), ("R", 200000, 3),
                               ("Z", 500000, 3), ("K", 131072, 3), ("K", 131073, 3), ("K", 5, 3)):
            src = _mixed(n, 5) if kind == "M" else corpus.gen_chunk(kind, 3, 0, n)
            frame = np.frombuffer(ora.zstd_compress_level(src, level), dtype=np.uint8)
            back, osz = c2.detransform(Z, frame, [frame.size], n)
            assert osz == [n] and np.array_equal(back, src), (kind, n, level)
        st0 = c2.decode_path_stats()
        # (the 5-byte frame is a single small block: that shape qualifies for the independent-block path)
        assert st0["whole_frames"] == 8 and st0["blocks"] == 1 and st0["regions"] == 0 and st0["serial_frames"] == 0
        # several frames in one batch, mixed with this library's own frames: speed mode (a warp per self-contained block) and
        # dense mode (a CTA per 64 KiB region)
        srcs = [corpus.gen_chunk("K", 9 + i, 0, 300000) for i in range(2)]
        frames = [np.frombuffer(ora.zstd_compress_chunk(s), dtype=np.uint8) for s in srcs]
        mine, msz = c2.transform(Z, srcs[0], 0)
        frames.append(mine[:msz[0]])
        dense, dsz = c2.transform(Z | 4, srcs[1], 0)
        frames.append(dense[:dsz[0]])
        blob = np.concatenate(frames)
        back, osz = c2.detransform(Z, blob, [f.size for f in frames], 4 * 300000)
        assert np.array_equal(back, np.concatenate(srcs + srcs))
        names = set(c2.profile_report())
        assert {"zstd_dec_entropy", "zstd_dec_frame_exec", "zstd_dec_regions", "zstd_dec_blk_literals", "zstd_dec_blk_sequences", "zstd_dec_blk_exec"} <= names
        st1 = c2.decode_path_stats()
        assert st1["whole_frames"] == st0["whole_frames"] + 2 and st1["regions"] == 5 and st1["blocks"] == 1 + 37
        assert st1["region_fallback_frames"] == 0 and st1["serial_frames"] == 0
        rng = np.random.default_rng(4)
        base = frames[1]
        for trial in range(60):
            bad = base.copy()
            bad[int(rng.integers(0, bad.size))] ^= 1 << int(rng.integers(0, 8))
            try:
                out, _ = c2.detransform(Z, bad, [bad.size], 300000)
            except tsgpu.TsgpuError as e:
                assert e.code == binding.E_CORRUPT
            else:
                assert len(out) == 300000
    finally:
        c2.close()


def test_simt_frame_executor_pointer_jumping_shapes():
    c2 = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=2, lib_path=SIMT_LIB)
    try:
        for name, src in executor_shapes().items():
            for level in (1, 3, 19):
                frame = np.frombuffer(ora.zstd_compress_level(src, level), dtype=np.uint8)
                back, osz = c2.detransform(Z, frame, [frame.size], src.size)
                assert osz == [src.size] and np.array_equal(back, src), (name, level)
        st = c2.decode_path_stats()
        assert st["whole_frames"] == 15 and st["serial_frames"] == 0
    finally:
        c2.close()
