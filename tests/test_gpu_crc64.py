"""The CRC-64/NVME calls on an H100: tsgpu_transform_parts_crc64 over 256 MiB segments in 4 MiB chunks with the reference's S3
part size (5 MiB) for Zstd, Zstd+dense, Zstd+checksum, AES, Zstd+AES, and with VERIFY and VALIDATE_RECORDS, in one call and in
the JNI enumeration's windows of 32 chunks; every part CRC and the object CRC equal the CPU CRC-64/NVME of the returned bytes, and
the deterministic writers return the bytes and sizes of tsgpu_transform_parts.  tsgpu_check_object_crc64 on objects this library
wrote and on objects the oracle's libzstd + OpenSSL wrote, and tsgpu_rewrite_object_crc64 with kept frames and with a plain
source compressed, give the oracle's words.  An empty segment, an empty last window and a part_cap one below the bound."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crc64_util as U  # noqa: E402
import records_util as R  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D, V, CK, VR = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM,
                      tsgpu.FLAG_VALIDATE_RECORDS)
CS = 4 << 20
MIB = 1 << 20
PART = 5 * MIB
FLAGS = [Z, Z | D, Z | CK, A, Z | A, Z | A | V]
FLAG_IDS = ["Z", "ZD", "ZC", "A", "ZA", "ZAV"]


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return corpus.gen_segment("K", 31, 256 * MIB + 12345, CS)


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


def _check(obj, crcs, ocrc, part=PART):
    assert crcs == U.part_crcs(obj, part), "part CRCs differ from the CPU CRC-64/NVME of the returned bytes"
    assert ocrc == U.crc64nvme(obj)


def _windows(c, flags, s, keys, fn, records=False):
    """the JNI enumeration's windows of 32 chunks, with the empty end call when the last window is full"""
    key, aad, ivs = keys
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    rc = np.zeros(binding.CURSOR_SIZE, np.uint8) if records else None
    outs, sizes, crcs, w, lo = [], [], [], 32 * CS, 0
    while True:
        win = s[lo:lo + w]
        end = win.size < w
        iv = ivs[12 * (lo // CS):] if win.size else np.zeros(12, np.uint8)
        o, z, p, oc = fn(flags, win, CS, PART, pc, end, rc, key, aad, iv)
        outs.append(o.copy()); sizes += z; crcs += p
        if end:
            return np.concatenate(outs), sizes, crcs, oc
        lo += w


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_parts_one_call_and_windows(ctx, seg, flags):
    keys = _keys(seg.size)
    out, sizes, crcs, ocrc = ctx.transform_parts_crc64(flags, seg, CS, PART, np.zeros(32, np.uint8), True, None, *keys)
    out = out.copy()
    assert len(crcs) == (out.size + PART - 1) // PART
    _check(out, crcs, ocrc)
    if flags & D or not flags & Z:                                   # deterministic writers: the bytes of the CRC-32C twin
        out32, sizes32, crcs32, _ = ctx.transform_parts(flags, seg, CS, PART, np.zeros(32, np.uint8), True, None, *keys)
        assert sizes == sizes32 and np.array_equal(out, out32) and len(crcs32) == len(crcs)
    obj, wsizes, wcrcs, wocrc = _windows(ctx, flags, seg, keys, ctx.transform_parts_crc64)
    _check(obj, wcrcs, wocrc)
    if flags & D or not flags & Z:
        assert wsizes == sizes and np.array_equal(obj, out)


def test_parts_with_record_validation_in_windows(ctx):
    s = R.gen_segment(12, 40 * MIB, big=300000)
    obj, _, crcs, ocrc = _windows(ctx, Z | D | A | VR, s, _keys(s.size), ctx.transform_parts_crc64, records=True)
    _check(obj, crcs, ocrc)


def test_empty_segment_and_empty_last_window(ctx, seg):
    keys = _keys(0)
    out, sizes, crcs, ocrc = ctx.transform_parts_crc64(Z | A, seg[:0], CS, PART, np.zeros(32, np.uint8), True, None, *keys)
    assert out.size == 0 and crcs == [] and ocrc == 0
    s = seg[:256 * MIB]                                              # two full windows of 32 chunks, then the empty end call
    assert s.size % (32 * CS) == 0
    for flags in (A, Z | A):                                         # the open part is finished by the empty call alone
        obj, _, crcs, ocrc = _windows(ctx, flags, s, _keys(s.size), ctx.transform_parts_crc64)
        assert obj.size % PART != 0
        _check(obj, crcs, ocrc)


def test_part_cap_one_below_the_bound(ctx, seg):
    s = seg[:32 * MIB]
    key, aad, ivs = (np.frombuffer(bytes(x), np.uint8) for x in _keys(s.size))
    bound = int(ctx.lib.tsgpu_transform_bound(Z | A, s.size, CS))
    need = bound // PART + 1
    dst = np.empty(bound + 64, np.uint8)
    sizes = np.zeros(16, np.uint32)
    n = C.c_uint32(sizes.size)
    crcs = np.full(need, 0xDEADBEEFDEADBEEF, np.uint64)
    n_parts, obj = C.c_uint32(12345), C.c_uint64(0xDEADBEEFDEADBEEF)
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    rc = ctx.lib.tsgpu_transform_parts_crc64(ctx.handle, Z | A, s.ctypes.data, s.size, CS, key.ctypes.data, aad.ctypes.data,
                                             aad.size, ivs.ctypes.data, dst.ctypes.data, dst.size, sizes.ctypes.data,
                                             C.addressof(n), None, 1, PART, pc.ctypes.data, crcs.ctypes.data,
                                             need - 1, C.addressof(n_parts), C.addressof(obj))
    assert rc == binding.E_SHORT
    assert (crcs == 0xDEADBEEFDEADBEEF).all() and n_parts.value == 12345 and obj.value == 0xDEADBEEFDEADBEEF


@pytest.mark.parametrize("flags", [0, A, Z | A, Z | D | A], ids=["plain", "A", "ZA", "ZDA"])
def test_check_object_on_our_objects(ctx, seg, flags):
    key, aad, ivs = _keys(seg.size)
    out, sizes = ctx.transform(flags, seg, CS, key, aad, ivs)
    out = out.copy()
    want = (U.crc64nvme(out), U.crc64nvme(seg))
    assert ctx.check_object_crc64(flags, out, sizes, CS, seg.size, key=key, aad=aad) == want
    cur, lo = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8), 0       # windows of 32 chunks through one cursor
    for i in range(0, len(sizes), 32):
        n = sum(sizes[i:i + 32])
        r = ctx.check_object_crc64(flags, out[lo:lo + n], sizes[i:i + 32], CS, seg.size, cur, i + 32 >= len(sizes), key, aad)
        lo += n
    assert r == want


def test_check_object_on_oracle_objects(ctx):
    # a Kafka segment with corpus-K payloads, the shape tests/test_gpu_check.py checks libzstd objects with
    s = R.gen_segment(13, 64 * MIB, payload=corpus.gen_segment("K", 13, 16 * MIB, MIB), big=(4 << 20) + (1 << 19))
    key, aad, ivs = _keys(s.size)
    for flags in (ora.FLAG_ZSTD, ora.FLAG_ZSTD | ora.FLAG_AES):
        ref, rsizes = ora.transform_segment(flags, s, CS, key, aad, ivs)
        ref = np.asarray(ref, np.uint8)
        assert ctx.check_object_crc64(flags, ref, rsizes, CS, s.size, key=key, aad=aad) == (U.crc64nvme(ref), U.crc64nvme(s))


@pytest.mark.parametrize("from_flags,to_flags", [(Z, Z | A), (0, Z | D)], ids=["kept-frames", "plain-compressed"])
def test_rewrite_object_words(ctx, seg, from_flags, to_flags):
    s = seg[:96 * MIB + 5]
    key, aad, ivs = _keys(s.size)
    old, osizes = ctx.transform(from_flags, s, CS, key, aad, ivs)
    old = old.copy()
    nivs = np.frombuffer(bytes(ivs), np.uint8)[::-1].copy()          # distinct from the old IVs
    kw = dict(from_key=key, from_aad=aad, to_key=bytes(range(32)), to_aad=aad, to_ivs=nivs)
    out, sizes, crcs, words = ctx.rewrite_object_crc64(from_flags, old, osizes, CS, s.size, to_flags, PART, **kw)
    out = out.copy()
    assert words == (U.crc64nvme(old), U.crc64nvme(out), U.crc64nvme(s)) and crcs == U.part_crcs(out, PART)
    out32, sizes32, _, _ = ctx.rewrite_object(from_flags, old, osizes, CS, s.size, to_flags, PART, **kw)
    assert sizes == sizes32 and np.array_equal(out, out32)
