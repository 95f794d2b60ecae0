"""TSGPU_FLAG_REFRAME of tsgpu_rewrite_object on the SIMT emulator.  Sources: oracle ZSTD and ZSTD|AES objects (what the Java
plugin wrote: libzstd level 3, no checksum), this library's speed and dense objects with and without checksum, frames followed by
a skippable frame, and the empty segment; each is rewritten in one call and in windows of 1 and 3 chunks through one cursor (an
object of 10 chunks ends on a full window of 1, so that walk ends with an empty window).  Sealed frames are libzstd's checksummed
frames byte for byte, re-encoded chunks are the smaller of the sealed (or kept) frame and tsgpu_transform's dense frame, and the
new object passes tsgpu_check_object with the source's segment CRC.  A decoded byte flipped before sealing fails the call, and
every refusal names its cause."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import check_util as K  # noqa: E402
import crc64_util as U64  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import reframe_util as F  # noqa: E402
import rewrite_util as W  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, CK, V, VR, RF = F.Z, F.A, F.D, F.CK, F.V, F.VR, F.RF
assert RF == tsgpu.FLAG_REFRAME == binding.FLAG_REFRAME
CS = 8192
PART = 5000
# (id, from_flags, writer, flags of the writer)
SOURCES = [("oracleZ", Z, "oracle", Z), ("oracleZA", Z | A, "oracle", Z | A), ("speedZ", Z, "lib", Z), ("denseZA", Z | A, "lib", Z | D | A),
           ("speedZck", Z, "lib", Z | CK), ("denseZAck", Z | A, "lib", Z | D | CK | A), ("skippableZ", Z, "skippable", Z)]
TARGETS = [("seal", Z | CK | RF), ("sealA", Z | CK | A | RF), ("dense", Z | D | RF), ("denseckA", Z | D | CK | A | RF)]


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=2, lib_path=SIMT_LIB)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(2, 80000, big=20000)          # 10 chunks of 8 KiB: 5 slot batches, entries across chunks and batches


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


def _source(c, writer, wflags, s):
    key, aad, ivs = _keys(s.size)
    if writer == "lib":
        obj, sizes = c.transform(wflags, s, CS, key, aad, ivs)
        return obj.copy(), sizes, key, aad
    obj, sizes = ora.transform_segment(wflags, s, CS, key, aad, ivs)
    if writer == "skippable":
        obj, sizes = F.with_skippable(obj, sizes)
    return obj, sizes, key, aad


def _fails(code, call):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    return str(ei.value)


@pytest.fixture(scope="module")
def dense_frames(ctx, seg):
    """tsgpu_transform's dense frames of every chunk, without and with checksum"""
    out = {}
    for ck in (0, CK):
        obj, sizes = ctx.transform(Z | D | ck, seg, CS)
        out[ck] = W.frames(Z, obj, sizes)
    return out


# ---------------------------------------------------------------------------------------------------- the matrix
@pytest.mark.parametrize("tid,tf", TARGETS, ids=[t[0] for t in TARGETS])
@pytest.mark.parametrize("sid,ff,writer,wflags", SOURCES, ids=[s[0] for s in SOURCES])
def test_reframed_object(ctx, seg, dense_frames, sid, ff, writer, wflags, tid, tf):
    obj, sizes, key, aad = _source(ctx, writer, wflags, seg)
    old = W.frames(ff, obj, sizes, key, aad)
    chunks = F.chunks_of(seg, CS)
    want = F.expected(tf, old, chunks, dense_frames[tf & CK])
    nk, na, ivs = W.new_key_material(len(sizes))
    readf = tf & (Z | A)
    for win in (None, 1, 3):
        new, nsz, parts, crc3 = W.rewrite_windows(ctx, ff | VR, obj, sizes, CS, seg.size, tf, PART, win, key, aad, nk, na, ivs)
        got = W.frames(tf, new, nsz, nk, na)
        assert got == want, (win, [i for i in range(len(got)) if got[i] != want[i]])
        for f, o, ch in zip(got, old, chunks):
            assert len(f) <= len(o) + 4
            assert ora.zstd_decompress_chunk(f) == ch                 # libzstd verifies every checksum
            if tf & CK:
                assert f[4] & 4
            if o[4] & 4 and not tf & D:
                assert f == o                                        # it had a checksum: kept as it is
        if writer == "oracle" and not tf & D:
            assert got == [ora.zstd_compress_checksum(ch, 3) for ch in chunks], win
        assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(seg)), win
        assert parts == U.part_crcs(new, PART), win
        assert K.check_windows(ctx, readf | VR, new, nsz, CS, seg.size, 3, nk, na) == (crc3[1], crc3[2])
        assert K.check_windows(ctx, ff, obj, sizes, CS, seg.size, None, key, aad)[0] == crc3[0]


@pytest.mark.parametrize("tf", [Z | CK | A | RF, Z | D | RF], ids=["sealA", "dense"])
def test_crc64_twin(ctx, seg, tf):
    obj, sizes, key, aad = _source(ctx, "oracle", Z | A, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    new, nsz, _, crc3 = W.rewrite_windows(ctx, Z | A, obj, sizes, CS, seg.size, tf, PART, None, key, aad, nk, na, ivs)
    cur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
    new64, nsz64, parts64, crc64 = ctx.rewrite_object_crc64(Z | A, obj, sizes, CS, seg.size, tf, PART, cur, True, key, aad, nk, na, ivs)
    assert np.array_equal(new64, new) and nsz64 == nsz
    assert crc64 == (U64.crc64nvme(obj), U64.crc64nvme(new), U64.crc64nvme(seg))
    assert parts64 == U64.part_crcs(new, PART)


def test_sealing_is_reversible(ctx, seg):
    obj, sizes, key, aad = _source(ctx, "skippable", Z, seg)
    new, nsz, _, _ = W.rewrite_windows(ctx, Z, obj, sizes, CS, seg.size, Z | CK | RF, PART)
    for f, o in zip(W.frames(Z, new, nsz), W.frames(Z, obj, sizes)):
        body, tail = F.split_tail(f)
        assert body[:4] + bytes([body[4] & ~4]) + body[5:-4] + tail == o


def test_empty_segment(ctx):
    key, aad, _ = _keys(0)
    nk, na, ivs = W.new_key_material(1)
    for ff in (Z, Z | A):
        for tf in (Z | CK | RF, Z | D | CK | A | RF):
            for sizes in ([], [0]):
                new, nsz, parts, crc3 = ctx.rewrite_object(ff | VR, b"", sizes, CS, 0, tf, PART, from_key=key, from_aad=aad,
                                                           to_key=nk, to_aad=na, to_ivs=ivs)
                assert new.size == 0 and nsz == [0] * len(sizes) and parts == [] and crc3 == (0, 0, 0)


def test_context_defaults_do_not_add_to_the_bits(ctx, seg, dense_frames, monkeypatch):
    """on a context whose defaults are dense mode and checksums, only the bits given act: from speed-mode frames, which dense
    frames beat, a seal must not re-encode and a re-encode must not add checksums"""
    obj, sizes, key, aad = _source(ctx, "lib", Z | A, seg)           # speed frames, written by a context without defaults
    old, chunks = W.frames(Z | A, obj, sizes, key, aad), F.chunks_of(seg, CS)
    monkeypatch.setenv("TSGPU_ZSTD_MODE", "dense")
    monkeypatch.setenv("TSGPU_ZSTD_CHECKSUM", "1")
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=2, lib_path=SIMT_LIB)
    nk, na, ivs = W.new_key_material(len(sizes))
    new, nsz, _, _ = W.rewrite_windows(c, Z | A, obj, sizes, CS, seg.size, Z | CK | RF, PART, None, key, aad, nk, na, ivs)
    assert W.frames(Z, new, nsz) == F.expected(Z | CK, old, chunks)
    new, nsz, _, _ = W.rewrite_windows(c, Z | A, obj, sizes, CS, seg.size, Z | D | RF, PART, None, key, aad, nk, na, ivs)
    got = W.frames(Z, new, nsz)
    assert got == F.expected(Z | D, old, chunks, dense_frames[0])
    assert sum(f != o for f, o in zip(got, old)) > len(old) // 2       # dense frames won: the test can see a leaked bit
    assert not any(f[4] & 4 for f in got)
    c.close()


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals(ctx, seg):
    obj, sizes, key, aad = _source(ctx, "oracle", Z | A, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    plain = [CS] * (seg.size // CS) + [seg.size % CS]
    probe = ctx.launch_count()
    for ff, o, s, tf in ((Z | A, obj, sizes, A | CK | RF), (0, seg, plain, Z | CK | RF), (Z | A, obj, sizes, A | RF)):
        msg = _fails(binding.E_ARG, lambda: W.rewrite_windows(ctx, ff, o, s, CS, seg.size, tf, PART, None, key, aad, nk, na, ivs))
        assert "TSGPU_FLAG_REFRAME acts on kept frames and needs TSGPU_FLAG_ZSTD in from_flags and to_flags" in msg, msg
    for tf in (Z | RF, Z | A | RF, Z | A | V | RF):
        msg = _fails(binding.E_ARG, lambda: W.rewrite_windows(ctx, Z | A, obj, sizes, CS, seg.size, tf, PART, None, key, aad, nk, na, ivs))
        assert "TSGPU_FLAG_REFRAME needs TSGPU_FLAG_ZSTD_DENSE or TSGPU_FLAG_ZSTD_CHECKSUM" in msg, msg
    for tf in (Z | CK, Z | D | A):                                    # without REFRAME: refused as before
        msg = _fails(binding.E_ARG, lambda: W.rewrite_windows(ctx, Z | A, obj, sizes, CS, seg.size, tf, PART, None, key, aad, nk, na, ivs))
        assert "have nothing to act on" in msg, msg
    assert ctx.launch_count() == probe
    # every other call refuses the bit
    key1, aad1, ivs1 = _keys(seg.size)
    _fails(binding.E_ARG, lambda: ctx.transform(Z | RF, seg, CS))
    _fails(binding.E_ARG, lambda: ctx.detransform(Z | A | RF, obj, sizes, seg.size, key, aad))
    _fails(binding.E_ARG, lambda: ctx.check_object(Z | A | RF, obj, sizes, CS, seg.size, key=key, aad=aad))
    _fails(binding.E_ARG, lambda: W.rewrite_windows(ctx, Z | A | RF, obj, sizes, CS, seg.size, Z | CK | RF, PART, None, key, aad, nk, na, ivs))


def test_sealed_frame_that_would_not_fit_its_slot_is_refused_before_any_gpu_work(seg):
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=2, lib_path=SIMT_LIB)
    obj, sizes = ora.transform_segment(Z, seg, CS)
    room = (int(c.lib.tsgpu_transform_bound(Z, CS, CS)) + 15) // 16 * 16   # a frame slot of this context: the frame bound, aligned
    frames = W.frames(Z, obj, sizes)
    k = 6
    frames[k] = frames[k] + F.skippable(bytes(room - 2 - len(frames[k]) - 8))     # room - 2 bytes: sealed, 2 bytes too many
    big = np.frombuffer(b"".join(frames), np.uint8).copy()
    bsz = [len(f) for f in frames]
    probe = c.launch_count()
    msg = _fails(binding.E_ARG, lambda: W.rewrite_windows(c, Z, big, bsz, CS, seg.size, Z | CK | RF, PART, 3))
    assert msg.endswith("chunk %d: its sealed frame of %d bytes would not fit the context's frame slot of %d bytes" % (k, room + 2, room)), msg
    probe = c.launch_count()
    _fails(binding.E_ARG, lambda: c.rewrite_object(Z, big, bsz, CS, seg.size, Z | D | CK | RF, PART))
    assert c.launch_count() == probe
    new, nsz, _, _ = W.rewrite_windows(c, Z, big, bsz, CS, seg.size, Z | D | RF, PART)       # not sealed: it fits
    assert W.frames(Z, new, nsz)[k] != frames[k] and nsz[k] < bsz[k]
    nk, na, ivs = W.new_key_material(len(bsz))
    new, nsz, _, _ = W.rewrite_windows(c, Z, big, bsz, CS, seg.size, Z | A, PART, None, None, b"", nk, na, ivs)   # kept as it is
    assert W.frames(Z | A, new, nsz, nk, na) == frames
    c.close()


# ---------------------------------------------------------------------------------------------------- the guard
def _raw(c, ff, obj, sizes, n, tf, nk, na, ivs, dst, key=None, aad=b""):
    ts = np.ascontiguousarray(sizes, dtype=np.uint32)
    o = np.ascontiguousarray(obj, dtype=np.uint8)
    nsz = np.zeros(len(sizes), np.uint32)
    crcs = np.zeros(4096, np.uint32)
    cur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
    np_, a, b, d = (np.zeros(1, np.uint32) for _ in range(4))
    f = lambda x: np.frombuffer(x, np.uint8) if x is not None else None     # noqa: E731
    rc = c.lib.tsgpu_rewrite_object(c.handle, ff, o.ctypes.data, o.size, ts.ctypes.data, ts.size, CS, n,
                                    f(key).ctypes.data if key else None, f(aad).ctypes.data if aad else None, len(aad or b""),
                                    tf, f(nk).ctypes.data, f(na).ctypes.data, len(na), f(ivs).ctypes.data, dst.ctypes.data, dst.size,
                                    nsz.ctypes.data, PART, crcs.ctypes.data, crcs.size, np_.ctypes.data, cur.ctypes.data, 1,
                                    a.ctypes.data, b.ctypes.data, d.ctypes.data)
    return rc, c.lib.tsgpu_last_error().decode() if rc else "", (int(np_[0]), int(a[0]), int(b[0]), int(d[0]), crcs.any())


def _inside_a_v2_body(seg, k):
    """an offset in chunk k that lies in the CRC-covered body of a v2 record batch"""
    st = R.starts(seg)
    ends = np.append(st[1:], seg.size)
    for e in range(len(st)):
        lo, hi = max(int(st[e]) + 21, k * CS), min(int(ends[e]), (k + 1) * CS)
        if seg[int(st[e]) + 16] == 2 and hi - lo > 8:
            return lo + 4 - k * CS
    raise AssertionError("no v2 body in chunk %d" % k)


@pytest.mark.parametrize("tf", [Z | CK | RF, Z | CK | A | RF, Z | D | CK | A | RF], ids=["seal", "sealA", "densecheckA"])
def test_misread_chunk_is_not_sealed(ctx, seg, tf, monkeypatch):
    obj, sizes, key, aad = _source(ctx, "oracle", Z, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    k = 5
    sound, ssz, _, _ = W.rewrite_windows(ctx, Z, obj, sizes, CS, seg.size, tf, PART, None, None, b"", nk, na, ivs)
    before = int(sum(ssz[:2 * (k // 2)]))                          # the chunks of the batches before chunk k's (2 per batch)
    monkeypatch.setenv("TSGPU_SIMT_FLIP_DECODED", "%d:%d" % (k, _inside_a_v2_body(seg, k)))
    for ff, code, pattern in ((Z, binding.E_VERIFY, r"verify: chunk %d did not read back" % k),
                              (Z | VR, binding.E_RECORDS, r"Record is corrupt .*\(check: crc\)")):
        msg = _fails(code, lambda: W.rewrite_windows(ctx, ff, obj, sizes, CS, seg.size, tf, PART, None, None, b"", nk, na, ivs))
        assert re.search(pattern, msg), msg
        dst = np.zeros(len(sizes) * (CS + 200), np.uint8)
        rc, msg, outs = _raw(ctx, ff, obj, sizes, seg.size, tf, nk, na, ivs, dst)
        assert rc == code and re.search(pattern, msg), msg
        assert np.array_equal(dst[:before], sound[:before]) and not dst[before:].any(), "bytes of the failing batch reached dst"
        assert outs == (0, 0, 0, 0, False), "a failed call wrote a CRC"
    monkeypatch.delenv("TSGPU_SIMT_FLIP_DECODED")
    again, _, _, _ = W.rewrite_windows(ctx, Z, obj, sizes, CS, seg.size, tf, PART, None, None, b"", nk, na, ivs)
    assert np.array_equal(again, sound)


# ---------------------------------------------------------------------------------------------------- sanitizers and lane orders
def _sweep(lib, env_extra, preload=None):
    env = dict(os.environ, **env_extra)
    if preload:
        env["LD_PRELOAD"] = preload
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_reframe.py"), lib], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "reframe sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]


def test_reframe_is_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so", "oracle"])
    U._oracle(); R._oracle()                                          # built before libasan is preloaded
    _sweep("libtsgpu_simt_asan.so", {"ASAN_OPTIONS": "detect_leaks=0"}, runtime)


@pytest.mark.parametrize("env", [{"TSGPU_SIMT_POISON": "1"}, {"TSGPU_SIMT_ORDER": "reverse"}, {"TSGPU_SIMT_ORDER": "random:7"}],
                         ids=["poison", "reverse", "random"])
def test_reframe_with_poison_and_lane_orders(env):
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    _sweep("libtsgpu_simt.so", env)
