"""tsgpu_rewrite_object on the SIMT emulator.  Kafka segments stored plain, AES, ZSTD or ZSTD|AES by tsgpu_transform, and ZSTD or
ZSTD|AES by the oracle (libzstd + OpenSSL, what the Java plugin wrote), are rewritten to AES, ZSTD, ZSTD|AES, ZSTD|DENSE|AES and
ZSTD|CHECKSUM|AES under a new key, in one call and in windows of 1 and 3 chunks.  The new object decodes to the segment through
the library and through the oracle; the source, object, segment and part CRCs equal the CPU CRC-32C (tests/part_crc_util.py);
when both sides compress, the new frames are the old ones byte for byte.  Refusals and failures name their cause, and no byte of
a failing batch reaches dst.  tests/test_gpu_rewrite.py runs 1 GiB objects on an H100."""
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
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import rewrite_util as W  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, CK, VR, V = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_VALIDATE_RECORDS,
                      tsgpu.FLAG_VERIFY)
CS = 8192
PART = 5000
SOURCES = [("plain", 0, False), ("A", A, False), ("Z", Z, False), ("ZA", Z | A, False), ("oracleZ", Z, True), ("oracleZA", Z | A, True)]
TARGETS = [("A", A), ("Z", Z), ("ZA", Z | A), ("ZDA", Z | D | A), ("ZCKA", Z | CK | A)]
PAIRS = [(s, t) for s in SOURCES for t in TARGETS if not (s[1] & Z and t[1] & (D | CK))]


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=2, lib_path=SIMT_LIB)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(2, 80000, big=20000)          # ~10 chunks of 8 KiB: 5 slot batches, entries across chunks and batches


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


def _source(c, flags, s, oracle=False):
    key, aad, ivs = _keys(s.size)
    if oracle:
        obj, sizes = ora.transform_segment(flags, s, CS, key, aad, ivs)
    else:
        obj, sizes = c.transform(flags, s, CS, key, aad, ivs)
    return obj.copy(), sizes, key, aad


def _fails(code, call):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    return str(ei.value)


def _rewrite(c, ff, obj, sizes, n, tf, win=None, key=None, aad=b"", nk=None, na=W.NEW_AAD, ivs=None, part=PART):
    if nk is None:
        nk, na, ivs = W.new_key_material(len(sizes))
    return W.rewrite_windows(c, ff, obj, sizes, CS, n, tf, part, win, key, aad, nk, na, ivs)


# ---------------------------------------------------------------------------------------------------- the matrix
@pytest.mark.parametrize("src,dst", PAIRS, ids=["%s-%s" % (s[0], t[0]) for s, t in PAIRS])
def test_rewritten_object_decodes_with_the_new_key(ctx, seg, src, dst):
    _, ff, oracle = src
    tf = dst[1]
    obj, sizes, key, aad = _source(ctx, ff, seg, oracle)
    nk, na, ivs = W.new_key_material(len(sizes))
    readf = tf & (Z | A)
    for win in (None, 1, 3):
        new, nsz, parts, crc3 = _rewrite(ctx, ff | VR, obj, sizes, seg.size, tf, win, key, aad, nk, na, ivs)
        assert len(nsz) == len(sizes) and sum(nsz) == new.size, win
        assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(seg)), win
        assert parts == U.part_crcs(new, PART), win
        back, _ = ctx.detransform(readf, new, nsz, seg.size, nk, na)
        assert np.array_equal(back, seg), win
        back, _ = ora.detransform_chunks(readf, new, nsz, seg.size, nk, na)
        assert np.array_equal(back, seg), win
        if ff & Z and tf & Z:                                           # the frames are kept
            assert W.frames(tf, new, nsz, nk, na) == W.frames(ff, obj, sizes, key, aad), win
        # the new object passes the check, with the segment CRC of the old one
        assert K.check_windows(ctx, readf | VR, new, nsz, CS, seg.size, 3, nk, na) == (crc3[1], crc3[2])


def test_verify_and_records_on_every_kind_of_target(ctx, seg):
    obj, sizes, key, aad = _source(ctx, Z | A, seg)
    for ff, o in ((Z | A, obj), (0, seg)):
        for tf in (A, Z | A, Z):
            sz = sizes if ff else [CS] * (seg.size // CS) + [seg.size % CS]
            new, nsz, _, crc3 = _rewrite(ctx, ff | VR, o, sz, seg.size, tf | V, 3, key, aad)
            assert crc3[1] == U.crc32c(new) and crc3[2] == U.crc32c(seg)


def test_same_key_with_fresh_ivs(ctx, seg):
    obj, sizes, key, aad = _source(ctx, A, seg)
    _, _, ivs = W.new_key_material(len(sizes))
    new, nsz, _, _ = _rewrite(ctx, A, obj, sizes, seg.size, Z | A, None, key, aad, key, aad, ivs)
    back, _ = ora.detransform_chunks(Z | A, new, nsz, seg.size, key, aad)
    assert np.array_equal(back, seg)


def test_empty_segment(ctx):
    key, aad, _ = _keys(0)
    nk, na, ivs = W.new_key_material(1)
    for ff in (0, Z, Z | A):
        for sizes in ([], [0]):
            new, nsz, parts, crc3 = ctx.rewrite_object(ff | VR, b"", sizes, CS, 0, Z | A, PART, from_key=key, from_aad=aad,
                                                       to_key=nk, to_aad=na, to_ivs=ivs)
            assert new.size == 0 and nsz == [0] * len(sizes) and parts == [] and crc3 == (0, 0, 0)


def test_cursor_carries_and_outputs_wait_for_the_end(ctx, seg):
    obj, sizes, key, aad = _source(ctx, Z | A, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    cur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
    n = sum(sizes[:2])
    b0, _, _, crc3 = ctx.rewrite_object(Z | A, obj[:n], sizes[:2], CS, seg.size, A, 1 << 30, cur, False, key, aad, nk, na, ivs[:24])
    assert crc3 is None and cur.any()
    b1, _, parts, crc3 = ctx.rewrite_object(Z | A, obj[n:], sizes[2:], CS, seg.size, A, 1 << 30, cur, True, key, aad, nk, na, ivs[24:])
    new = np.concatenate([b0, b1])
    assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(seg)) and parts == [U.crc32c(new)]


# ---------------------------------------------------------------------------------------------------- refusals
def test_refusals(ctx, seg):
    obj, sizes, key, aad = _source(ctx, Z | A, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    for tf in (Z | D | A, Z | CK | A, Z | D, Z | CK):                    # frames are kept: nothing for the modifiers to act on
        msg = _fails(binding.E_ARG, lambda: _rewrite(ctx, Z | A, obj, sizes, seg.size, tf, None, key, aad))
        assert "kept" in msg
    for tf in (0, V, D, VR, Z | VR, A | 64):                             # no ZSTD or AES, or a bit the target does not take
        _fails(binding.E_ARG, lambda: _rewrite(ctx, Z | A, obj, sizes, seg.size, tf, None, key, aad))
    _fails(binding.E_ARG, lambda: _rewrite(ctx, Z | A, obj, sizes, seg.size, A, None, key, aad, nk, na, None))   # no IVs
    # an IV reused under the same key: chunk 4's own IV
    bad_ivs = bytearray(ivs)
    bad_ivs[48:60] = bytes(obj[sum(sizes[:4]):sum(sizes[:4]) + 12])
    msg = _fails(binding.E_ARG, lambda: _rewrite(ctx, Z | A, obj, sizes, seg.size, Z | A, None, key, aad, key, na, bytes(bad_ivs)))
    assert "chunk 4" in msg
    _rewrite(ctx, Z | A, obj, sizes, seg.size, Z | A, None, key, aad, nk, na, bytes(bad_ivs))   # under a new key it may repeat
    # another old chunk's IV under the same key, and two equal new IVs under any key
    bad_ivs = bytearray(ivs)
    bad_ivs[12:24] = bytes(obj[sum(sizes[:6]):sum(sizes[:6]) + 12])
    msg = _fails(binding.E_ARG, lambda: _rewrite(ctx, Z | A, obj, sizes, seg.size, Z | A, None, key, aad, key, na, bytes(bad_ivs)))
    assert "to_ivs[1] repeats the IV of chunk 6" in msg, msg
    bad_ivs = bytearray(ivs)
    bad_ivs[84:96] = bad_ivs[24:36]
    for ff in (0, Z | A):
        msg = _fails(binding.E_ARG, lambda: _rewrite(ctx, ff, obj if ff else seg, sizes if ff else [CS] * (seg.size // CS) + [seg.size % CS],
                                                     seg.size, A, None, key, aad, nk, na, bytes(bad_ivs)))
        assert "to_ivs[2] repeats to_ivs[7]" in msg, msg


def test_frame_larger_than_the_index_chunk_size_is_an_invalid_frame(ctx, seg):
    """chunks decode to the offsets of the chunk index: a frame that decodes to more than its original chunk size is refused in
    place, for the check as for the rewrite, and named as chunk 0's invalid frame whatever the timing of the other chunks"""
    obj, sizes, key, aad = _source(ctx, Z | A, seg)
    for win in (None, 3):
        msg = _fails(binding.E_CORRUPT, lambda: K.check_windows(ctx, Z | A, obj, sizes, CS // 2, seg.size, win, key, aad))
        assert msg.startswith("Invalid zstd frame in chunk 0 "), msg
        msg = _fails(binding.E_CORRUPT, lambda: W.rewrite_windows(ctx, Z | A, obj, sizes, CS // 2, seg.size, Z | A, PART, win, key, aad,
                                                                  *W.new_key_material(2 * len(sizes))))
        assert msg.startswith("Invalid zstd frame in chunk 0 "), msg


def test_small_part_cap_fails_before_any_gpu_work(ctx, seg):
    obj, sizes, key, aad = _source(ctx, A, seg)
    nk, na, ivs = W.new_key_material(len(sizes))
    dst_probe = ctx.launch_count()
    L = seg.size
    bound = ctx.lib.tsgpu_transform_bound(Z | A, L, CS)
    need = bound // PART + 1
    msg = _fails(binding.E_SHORT, lambda: ctx.rewrite_object(A, obj, sizes, CS, L, Z | A, PART, from_key=key, from_aad=aad,
                                                             to_key=nk, to_aad=na, to_ivs=ivs, part_cap=need - 1))
    assert "part_cap" in msg and ctx.launch_count() == dst_probe
    ctx.rewrite_object(A, obj, sizes, CS, L, Z | A, PART, from_key=key, from_aad=aad, to_key=nk, to_aad=na, to_ivs=ivs, part_cap=need)


# ---------------------------------------------------------------------------------------------------- failures
def _chunk_start(sizes, k):
    return int(sum(sizes[:k]))


def _raw(c, ff, obj, sizes, n, tf, key, aad, nk, na, ivs, dst):
    """tsgpu_rewrite_object straight into `dst` (to see what a failing call left there)"""
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
    return rc, c.lib.tsgpu_last_error().decode() if rc else ""


@pytest.fixture(scope="module")
def objects(ctx, seg):
    return {ff: _source(ctx, ff, seg) for ff in (0, A, Z, Z | CK, Z | A)}


def _sound_prefix(ctx, seg, objects, ff, tf, k):
    """the new sizes of the sound object's chunks before slot batch k // 2"""
    obj, sizes, key, aad = objects[ff]
    nk, na, ivs = W.new_key_material(len(sizes))
    _, nsz, _, _ = _rewrite(ctx, ff, obj, sizes, seg.size, tf & ~V, None, key, aad, nk, na, ivs)
    return nsz[:2 * (k // 2)]


def _failing_call_leaves_its_batch_out(ctx, seg, objects, ff, tf, bad, sizes, n, key, aad, code, k, pattern, wins=(None, 1, 3)):
    nk, na, ivs = W.new_key_material(len(sizes))
    for win in wins:
        msg = _fails(code, lambda: _rewrite(ctx, ff, bad, sizes, n, tf, win, key, aad, nk, na, ivs))
        assert re.search(pattern, msg), (win, msg)
    dst = np.zeros(len(sizes) * (CS + 200), np.uint8)
    rc, msg = _raw(ctx, ff, bad, sizes, n, tf, key, aad, nk, na, ivs, dst)
    assert rc == code and re.search(pattern, msg), msg
    before = int(sum(_sound_prefix(ctx, seg, objects, ff, tf, k)))
    assert not dst[before:].any(), "bytes of the failing batch reached dst"


@pytest.mark.parametrize("ff", [A, Z | A], ids=["A", "ZA"])
def test_flipped_source_ciphertext_byte_fails_the_tag(ctx, seg, objects, ff):
    obj, sizes, key, aad = objects[ff]
    k = 5
    bad = obj.copy()
    bad[_chunk_start(sizes, k) + 12 + 100] ^= 0x04
    _failing_call_leaves_its_batch_out(ctx, seg, objects, ff, Z | A, bad, sizes, seg.size, key, aad, binding.E_AUTH, k,
                                       r"Tag mismatch in chunk %d\b" % k)


@pytest.mark.parametrize("ff,where", [(Z, "magic"), (Z | CK, "checksum")], ids=["frame", "checksum"])
def test_damaged_frame_fails(ctx, seg, objects, ff, where):
    obj, sizes, key, aad = objects[ff]
    k = 4 if where == "magic" else 7
    bad = obj.copy()
    if where == "magic":
        bad[_chunk_start(sizes, k)] ^= 0xFF
    else:
        bad[_chunk_start(sizes, k + 1) - 1] ^= 0x10                    # the last byte of the frame: its Content_Checksum
    _failing_call_leaves_its_batch_out(ctx, seg, objects, ff, Z | A, bad, sizes, seg.size, key, aad, binding.E_CORRUPT, k,
                                       r"chunk %d\b" % k)


@pytest.mark.parametrize("ff", [0, A, Z], ids=["plain", "A", "Z"])
def test_index_that_disagrees_fails(ctx, seg, objects, ff):
    obj, sizes, key, aad = objects[ff]
    n, last = seg.size, len(sizes) - 1
    tail = n - last * CS
    nk, na, ivs = W.new_key_material(len(sizes))
    msg = _fails(binding.E_CORRUPT, lambda: _rewrite(ctx, ff, obj, sizes, n - 1, Z | A, None, key, aad, nk, na, ivs))
    assert "chunk %d decoded to %d bytes, the chunk index gives %d" % (last, tail, tail - 1) in msg
    msg = _fails(binding.E_CORRUPT, lambda: _rewrite(ctx, ff, obj[:_chunk_start(sizes, last)], sizes[:-1], n, A, 3, key, aad,
                                                     nk, na, ivs))
    assert "the object has %d chunks" % last in msg


def _bad_batch(s, e):
    st = R.starts(s)
    b = s.copy()
    b[int(st[e]) + 17 + 2] ^= 0x01                                       # the stored CRC of a v2 batch
    return b


def _v2_entry_across(s, unit):
    st = R.starts(s)
    ends = np.append(st[1:], s.size)
    for e in range(len(st)):
        if s[int(st[e]) + 16] == 2 and int(st[e]) // unit != (int(ends[e]) - 1) // unit:
            return e
    raise AssertionError("no v2 entry crosses a %d-byte boundary" % unit)


@pytest.mark.parametrize("ff", [0, Z | A], ids=["plain", "ZA"])
def test_bad_record_batch_across_a_window_end(ctx, seg, ff):
    e = _v2_entry_across(seg, 3 * CS)                                    # crosses a 3-chunk window end
    bad = _bad_batch(seg, e)
    key, aad, ivs = _keys(bad.size)
    upload = _fails(binding.E_RECORDS, lambda: ctx.transform(Z | VR, bad, CS, key, aad, ivs))
    obj, sizes, key, aad = _source(ctx, ff, bad)
    at = int(R.starts(seg)[e])
    new, nsz, _, crc3 = _rewrite(ctx, ff, obj, sizes, bad.size, Z | A, 3, key, aad)     # without the flag it passes
    assert crc3[2] == U.crc32c(bad)
    for win in (None, 1, 3):
        msg = _fails(binding.E_RECORDS, lambda: _rewrite(ctx, ff | VR, obj, sizes, bad.size, Z | A, win, key, aad))
        assert msg == upload and re.search(r"segment position %d\b" % at, msg), msg
    nk, na, ivs = W.new_key_material(len(sizes))
    dst = np.zeros(len(sizes) * (CS + 200), np.uint8)
    rc, msg = _raw(ctx, ff | VR, obj, sizes, bad.size, Z | A, key, aad, nk, na, ivs, dst)
    assert rc == binding.E_RECORDS
    k = (int(R.starts(seg)[e + 1]) - 1) // CS                            # the entry's last chunk: its slot batch (2 chunks) fails
    before = int(sum(nsz[:2 * (k // 2)]))
    assert not dst[before:].any()


def test_flipped_byte_in_a_new_chunk_fails_verify(ctx, seg, objects, monkeypatch):
    obj, sizes, key, aad = objects[Z | A]
    k = 3
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "%d:40" % k)                 # chunk k of a call
    for tf in (Z | A, A):
        _failing_call_leaves_its_batch_out(ctx, seg, objects, Z | A, tf | V, obj, sizes, seg.size, key, aad, binding.E_VERIFY, k,
                                           r"verify: chunk %d did not read back" % k, wins=(None,))
    monkeypatch.delenv("TSGPU_SIMT_FLIP")
    _rewrite(ctx, Z | A, obj, sizes, seg.size, Z | A | V, None, key, aad)


def test_source_failure_comes_before_verify(ctx, seg, objects, monkeypatch):
    obj, sizes, key, aad = objects[A]
    bad = obj.copy()
    bad[_chunk_start(sizes, 1) + 40] ^= 1
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "0:40")
    msg = _fails(binding.E_AUTH, lambda: _rewrite(ctx, A, bad, sizes, seg.size, Z | A | V, None, key, aad))
    assert "chunk 1" in msg


def test_rewrite_is_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so", "oracle"])
    U._oracle(); R._oracle()                                            # built before libasan is preloaded
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", LD_PRELOAD=runtime)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_rewrite.py"), "libtsgpu_simt_asan.so"], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "rewrite sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]


def test_rewrite_is_clean_under_ubsan():
    runtime = subprocess.run(["gcc", "-print-file-name=libubsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libubsan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_ubsan.so", "oracle"])
    U._oracle(); R._oracle()
    env = dict(os.environ, LD_PRELOAD=runtime, UBSAN_OPTIONS="print_stacktrace=1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_rewrite.py"), "libtsgpu_simt_ubsan.so"], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "rewrite sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
