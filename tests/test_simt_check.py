"""tsgpu_check_object on the SIMT emulator: Kafka segments written by tsgpu_transform with every flag set {0, AES, ZSTD,
ZSTD|DENSE, ZSTD|CHECKSUM, ZSTD|AES, ZSTD|DENSE|AES}, with and without VALIDATE_RECORDS, pass and give the CPU CRC-32C
(tests/part_crc_util.py) of the object and of the segment, in one call or in windows of 1 and 3 chunks; so do objects written by
the oracle (libzstd + OpenSSL, what the Java plugin wrote).  Every kind of damage fails with its code and names the chunk or the
segment position: a flipped ciphertext byte, a damaged frame or Content_Checksum, a chunk index that disagrees with the decoded
sizes, a short src, a bad record batch (also across two windows) and a segment that ends inside an entry.
tests/test_gpu_check.py runs 1 GiB objects on an H100."""
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, CK, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_VALIDATE_RECORDS
CS = 8192
FLAG_SETS = [0, A, Z, Z | D, Z | CK, Z | A, Z | D | A]
FLAG_IDS = ["plain", "A", "Z", "ZD", "ZC", "ZA", "ZDA"]


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


def _write(c, flags, s):
    key, aad, ivs = _keys(s.size)
    out, sizes = c.transform(flags, s, CS, key, aad, ivs)
    return out.copy(), sizes, key, aad


def _fails(code, call):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    return str(ei.value)


# ---------------------------------------------------------------------------------------------------- sound objects
@pytest.mark.parametrize("records", [False, True], ids=["", "VR"])
@pytest.mark.parametrize("flags", FLAG_SETS, ids=FLAG_IDS)
def test_written_object_passes_with_the_oracle_crcs(ctx, seg, flags, records):
    obj, sizes, key, aad = _write(ctx, flags, seg)
    want = (U.crc32c(obj), U.crc32c(seg))
    cf = flags | (VR if records else 0)
    for win in (None, 1, 3):
        assert K.check_windows(ctx, cf, obj, sizes, CS, seg.size, win, key, aad) == want, win


@pytest.mark.parametrize("flags", [Z, A, Z | A], ids=["Z", "A", "ZA"])
def test_oracle_written_object_passes(ctx, seg, flags):
    key, aad, ivs = _keys(seg.size)
    obj, sizes = ora.transform_segment(flags, seg, CS, key, aad, ivs)
    want = (U.crc32c(obj), U.crc32c(seg))
    for win in (None, 3):
        assert K.check_windows(ctx, flags | VR, obj, sizes, CS, seg.size, win, key, aad) == want


def test_empty_segment(ctx):
    key, aad, _ = _keys(0)
    for flags in (0, Z, Z | A):
        assert ctx.check_object(flags | VR, b"", [], CS, 0, key=key, aad=aad) == (0, 0)
        assert ctx.check_object(flags | VR, b"", [0], CS, 0, key=key, aad=aad) == (0, 0)   # the index's one empty chunk


def test_cursor_carries_and_outputs_wait_for_the_end(ctx, seg):
    obj, sizes, key, aad = _write(ctx, Z | A, seg)
    cur = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8)
    n = sum(sizes[:2])
    assert ctx.check_object(Z | A | VR, obj[:n], sizes[:2], CS, seg.size, cur, False, key, aad) is None
    assert cur.any()
    got = ctx.check_object(Z | A | VR, obj[n:], sizes[2:], CS, seg.size, cur, True, key, aad)
    assert got == (U.crc32c(obj), U.crc32c(seg))


# ---------------------------------------------------------------------------------------------------- failures
def _chunk_start(sizes, k):
    return int(sum(sizes[:k]))


@pytest.mark.parametrize("flags", [A, Z | A], ids=["A", "ZA"])
def test_flipped_ciphertext_byte_fails_the_tag(ctx, seg, flags):
    obj, sizes, key, aad = _write(ctx, flags, seg)
    k = 5
    bad = obj.copy()
    bad[_chunk_start(sizes, k) + 12 + 100] ^= 0x04
    for win in (None, 1):
        msg = _fails(binding.E_AUTH, lambda: K.check_windows(ctx, flags | VR, bad, sizes, CS, seg.size, win, key, aad))
        assert "chunk %d" % k in msg


def test_damaged_frame_fails(ctx, seg):
    obj, sizes, _, _ = _write(ctx, Z, seg)
    k = 4
    bad = obj.copy()
    bad[_chunk_start(sizes, k)] ^= 0xFF                              # the frame's magic number
    msg = _fails(binding.E_CORRUPT, lambda: K.check_windows(ctx, Z, bad, sizes, CS, seg.size, 3))
    assert re.search(r"chunk %d\b" % k, msg), msg


def test_damaged_content_checksum_fails(ctx, seg):
    obj, sizes, _, _ = _write(ctx, Z | CK, seg)
    k = 7
    bad = obj.copy()
    bad[_chunk_start(sizes, k + 1) - 1] ^= 0x10                      # the last byte of the frame: its Content_Checksum
    msg = _fails(binding.E_CORRUPT, lambda: K.check_windows(ctx, Z, bad, sizes, CS, seg.size))
    assert re.search(r"chunk %d\b" % k, msg), msg


@pytest.mark.parametrize("flags", [0, A, Z], ids=["plain", "A", "Z"])
def test_chunk_index_that_disagrees_fails(ctx, seg, flags):
    obj, sizes, key, aad = _write(ctx, flags, seg)
    n, last = seg.size, len(sizes) - 1
    tail = n - last * CS
    msg = _fails(binding.E_CORRUPT, lambda: ctx.check_object(flags, obj, sizes, CS, n - 1, key=key, aad=aad))
    assert "chunk %d decoded to %d bytes, the chunk index gives %d" % (last, tail, tail - 1) in msg
    msg = _fails(binding.E_CORRUPT, lambda: ctx.check_object(flags, obj, sizes, 2 * CS, n, key=key, aad=aad))
    assert "chunk 0 decoded to %d bytes, the chunk index gives %d" % (CS, 2 * CS) in msg
    head = obj[:_chunk_start(sizes, last)]                           # the object without its last chunk
    msg = _fails(binding.E_CORRUPT, lambda: K.check_windows(ctx, flags, head, sizes[:-1], CS, n, 3, key, aad))
    assert "the object has %d chunks" % last in msg and "has %d" % (last + 1) in msg
    msg = _fails(binding.E_CORRUPT, lambda: ctx.check_object(flags, obj, sizes, CS, n - tail, key=key, aad=aad))
    assert "chunk %d decoded to %d bytes" % (last, tail) in msg and "has %d chunks" % last in msg


def test_short_src_fails(ctx, seg):
    obj, sizes, key, aad = _write(ctx, Z | A, seg)
    _fails(binding.E_SHORT, lambda: ctx.check_object(Z | A, obj[:-1], sizes, CS, seg.size, key=key, aad=aad))


def _bad_batch(s, e):
    st = R.starts(s)
    b = s.copy()
    b[int(st[e]) + 17 + 2] ^= 0x01                                   # the stored CRC of a v2 batch
    return b


def _v2_entry_across(s, unit):
    st = R.starts(s)
    ends = np.append(st[1:], s.size)
    for e in range(len(st)):
        if s[int(st[e]) + 16] == 2 and int(st[e]) // unit != (int(ends[e]) - 1) // unit:
            return e
    raise AssertionError("no v2 entry crosses a %d-byte boundary" % unit)


@pytest.mark.parametrize("flags", [0, Z, Z | A], ids=["plain", "Z", "ZA"])
def test_bad_record_batch_fails_with_the_upload_message(ctx, seg, flags):
    bad = _bad_batch(seg, len(R.starts(seg)) // 2)
    key, aad, ivs = _keys(bad.size)
    upload = _fails(binding.E_RECORDS, lambda: ctx.transform(Z | VR, bad, CS, key, aad, ivs))
    obj, sizes, key, aad = _write(ctx, flags, bad)                   # written without the flag
    assert K.check_windows(ctx, flags, obj, sizes, CS, bad.size, None, key, aad) == (U.crc32c(obj), U.crc32c(bad))
    for win in (None, 1, 3):
        assert _fails(binding.E_RECORDS, lambda: K.check_windows(ctx, flags | VR, obj, sizes, CS, bad.size, win, key, aad)) == upload


def test_bad_batch_across_two_windows(ctx, seg):
    e = _v2_entry_across(seg, 2 * CS)                                # crosses a 2-chunk window (and slot batch) end
    bad = _bad_batch(seg, e)
    at, kind, _, _ = R.walk(bad)
    assert at == int(R.starts(seg)[e]) and kind == "crc"
    obj, sizes, key, aad = _write(ctx, Z | A, bad)
    for win in (1, 2):
        msg = _fails(binding.E_RECORDS, lambda: K.check_windows(ctx, Z | A | VR, obj, sizes, CS, bad.size, win, key, aad))
        assert re.search(r"segment position %d\b" % at, msg) and "check: crc" in msg, msg


def test_segment_ending_inside_an_entry(ctx, seg):
    cut = int(R.starts(seg)[-1]) + 30
    short = seg[:cut].copy()
    obj, sizes, key, aad = _write(ctx, Z, short)
    assert K.check_windows(ctx, Z, obj, sizes, CS, cut) == (U.crc32c(obj), U.crc32c(short))
    for win in (None, 1, len(sizes)):                                # len(sizes): a full last window, then an empty one
        msg = _fails(binding.E_RECORDS, lambda: K.check_windows(ctx, Z | VR, obj, sizes, CS, cut, win))
        assert "check: length" in msg and "segment position %d" % int(R.starts(seg)[-1]) in msg


def test_chunk_failure_comes_before_the_batch_record_verdict(ctx, seg):
    """a tag failure and a bad record batch in the same slot batch: the tag is reported"""
    bad = _bad_batch(seg, 0)
    obj, sizes, key, aad = _write(ctx, A, bad)
    obj[_chunk_start(sizes, 1) + 40] ^= 1
    msg = _fails(binding.E_AUTH, lambda: ctx.check_object(A | VR, obj, sizes, CS, bad.size, key=key, aad=aad))
    assert "chunk 1" in msg


def test_arguments(ctx, seg):
    obj, sizes, key, aad = _write(ctx, Z, seg)
    _fails(binding.E_ARG, lambda: ctx.check_object(Z | tsgpu.FLAG_VERIFY, obj, sizes, CS, seg.size))
    _fails(binding.E_ARG, lambda: ctx.check_object(Z, obj, sizes, 0, seg.size))
    _fails(binding.E_ARG, lambda: ctx.check_object(Z, obj, sizes, (1 << 16) + 1, seg.size))
    _fails(binding.E_ARG, lambda: ctx.check_object(A, obj, sizes, CS, seg.size))           # no key


def test_check_object_is_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so", "oracle"])
    U._oracle(); R._oracle()                                        # built before libasan is preloaded
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0", LD_PRELOAD=runtime)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_check.py"), "libtsgpu_simt_asan.so"], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "check sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
