"""tsgpu_rekey_object on the SIMT emulator.  Objects of AES chunks -- written by the oracle (OpenSSL, and libzstd + OpenSSL, what the
Java plugin wrote), by tsgpu_transform_parts in speed and dense mode, and shaped like an .indexes object with an empty blob -- are
re-encrypted under a new key in one call and in windows.  Every new chunk equals the oracle's decrypt-then-encrypt of the old one;
the part, source and object CRCs equal the CPU CRC-32C and CRC-64/NVME.  Refusals name their cause, a failing batch leaves no
byte in dst and no CRC is written.  tests/test_gpu_rekey.py runs 256 MiB objects on an H100."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crc64_util as U64  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import rekey_util as K  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
CAP = 1 << 16                     # the context's max_chunk_bytes
CS = 8192
PART = 5000
NEW_KEY, NEW_AAD = bytes(range(100, 132)), b"rotated-segment-key"


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=CAP, max_batch=2, lib_path=SIMT_LIB)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(4, 60000, big=15000)


def _ivs(n, seed=11):
    return np.random.default_rng(seed).bytes(12 * max(n, 1))


def _fails(code, call):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    return str(ei.value)


def _check(ctx, obj, sizes, key, aad, nk=NEW_KEY, na=NEW_AAD, wins=(None, 1, 2), flags=0):
    """the new object is the oracle's for every window size, with the same CRCs; returns it"""
    ivs = _ivs(len(sizes))
    want = K.expected(obj, sizes, key, aad, nk, na, ivs)
    for win in wins:
        new, parts, crc2 = K.rekey_windows(ctx, obj, sizes, key, nk, ivs, PART, win, aad, na, flags)
        assert np.array_equal(new, want), win
        assert parts == U.part_crcs(want, PART), win
        assert crc2 == (U.crc32c(obj), U.crc32c(want)), win
    return want


# ---------------------------------------------------------------------------------------------------- what the new object is
@pytest.mark.parametrize("aad_len", [0, 1, 16, 17, 64])
def test_chunk_sizes_and_aad_lengths(ctx, aad_len):
    # plaintexts of 0 (an empty chunk, no IV and tag), 0 (28 bytes), 1, 16 and 16 k +- 1 bytes, and a full chunk of the context
    rng = np.random.default_rng(aad_len)
    aad = rng.bytes(aad_len)
    plain = [None] + [rng.bytes(n) for n in (0, 1, 16, 16 * 5 - 1, 16 * 5 + 1, 16 * 33 - 1, 16 * 33 + 1, CAP)]
    obj, sizes = K.encrypt_chunks(b"k" * 32, aad, plain)
    assert sizes[:5] == [0, 28, 29, 44, 28 + 79]
    _check(ctx, obj, sizes, b"k" * 32, aad, na=rng.bytes((aad_len * 7) % 65))


@pytest.mark.parametrize("flags,oracle", [(A, True), (Z | A, True), (Z | A, False), (Z | D | A, False)],
                         ids=["oracleA", "oracleZA-libzstd", "ZA-speed", "ZA-dense"])
def test_stored_log_objects(ctx, seg, flags, oracle):
    nch = (seg.size + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    if oracle:
        obj, sizes = ora.transform_segment(flags, seg, CS, key, aad, ivs)
    else:
        cur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
        obj, sizes, _, _ = ctx.transform_parts(flags, seg, CS, PART, cur, True, np.zeros(binding.CURSOR_SIZE, np.uint8), key, aad, ivs)
    obj = np.asarray(obj).copy()
    want = _check(ctx, obj, sizes, key, aad, wins=(None, 1, 2, 3))
    back, _ = ora.detransform_chunks(flags & (Z | A), want, sizes, seg.size, NEW_KEY, NEW_AAD)   # the segment, under the new key
    assert np.array_equal(back, seg)
    with pytest.raises(Exception):                                                            # and no more under the old one
        ora.detransform_chunks(flags & (Z | A), want, sizes, seg.size, key, aad)


def test_indexes_shaped_object(ctx):
    # five index blobs of SegmentIndexesV1, the transaction index empty: one chunk each, sizes from the manifest
    rng = np.random.default_rng(5)
    plain = [rng.bytes(800), rng.bytes(1200), rng.bytes(33), None, rng.bytes(4000)]
    key, aad = rng.bytes(32), b"segment-aad"
    obj, sizes = K.encrypt_chunks(key, aad, plain)
    assert sizes[3] == 0
    _check(ctx, obj, sizes, key, aad, wins=(None, 1, 2, 4))
    # the empty blob takes no IV: an entry equal to another's passes
    ivs = bytearray(_ivs(5))
    ivs[36:48] = ivs[0:12]
    new, _, _ = ctx.rekey_object(obj, sizes, key, NEW_KEY, bytes(ivs), PART, aad, NEW_AAD)
    assert np.array_equal(new, K.expected(obj, sizes, key, aad, NEW_KEY, NEW_AAD, bytes(ivs)))


def test_same_key_fresh_ivs_and_empty_windows(ctx):
    rng = np.random.default_rng(6)
    key, aad = rng.bytes(32), b""
    obj, sizes = K.encrypt_chunks(key, aad, [rng.bytes(3000) for _ in range(3)])
    _check(ctx, obj, sizes, key, aad, nk=key, na=aad, wins=(None, 3))      # the last window is empty
    new, parts, crc2 = ctx.rekey_object(b"", [], key, NEW_KEY, None, PART)
    assert new.size == 0 and parts == [] and crc2 == (0, 0)
    new, parts, crc2 = ctx.rekey_object(b"", [0], key, NEW_KEY, None, PART)   # the empty segment's one chunk
    assert new.size == 0 and parts == [] and crc2 == (0, 0)


def test_crc64_twin_writes_the_same_bytes(ctx, seg):
    key, aad, ivs = corpus.fixed_key_material((seg.size + CS - 1) // CS)
    obj, sizes = ora.transform_segment(Z | A, seg, CS, key, aad, ivs)
    nivs = _ivs(len(sizes))
    for win in (None, 2):
        new32, _, _ = K.rekey_windows(ctx, obj, sizes, key, NEW_KEY, nivs, PART, win, aad, NEW_AAD)
        new64, parts, crc2 = K.rekey_windows(ctx, obj, sizes, key, NEW_KEY, nivs, PART, win, aad, NEW_AAD, crc64=True)
        assert np.array_equal(new32, new64), win
        assert parts == U64.part_crcs(new64, PART), win
        assert crc2 == (U64.crc64nvme(obj), U64.crc64nvme(new64)), win


def test_verify_passes_clean_objects(ctx, seg):
    key, aad, ivs = corpus.fixed_key_material((seg.size + CS - 1) // CS)
    obj, sizes = ora.transform_segment(A, seg, CS, key, aad, ivs)
    _check(ctx, obj, sizes, key, aad, wins=(None, 3), flags=V)
    rng = np.random.default_rng(8)
    obj, sizes = K.encrypt_chunks(key, aad, [rng.bytes(40), None, b"", rng.bytes(1)])
    _check(ctx, obj, sizes, key, aad, wins=(None,), flags=V)


# ---------------------------------------------------------------------------------------------------- refusals and failures
def _raw(ctx, obj, sizes, key, ivs, dst_cap=None, part_cap=64, flags=0, cursor=None, end=1, nk=NEW_KEY, fill=0xEE, src_len=None):
    """tsgpu_rekey_object called directly: (rc, message, dst after the call, (source, object) CRC words after the call)"""
    s = np.ascontiguousarray(obj, np.uint8)
    ts = np.ascontiguousarray(sizes, np.uint32)
    total = int(ts.sum())
    dst = np.full(total if dst_cap is None else dst_cap, fill, np.uint8)
    crcs = np.zeros(max(part_cap, 1), np.uint32)
    n_parts, src_crc, obj_crc = C.c_uint32(0), C.c_uint32(0xABCD), C.c_uint32(0xABCD)
    cur = np.zeros(binding.REKEY_CURSOR_SIZE, np.uint8) if cursor is None else cursor
    k, tk, iv = np.frombuffer(key, np.uint8), np.frombuffer(nk, np.uint8), np.frombuffer(ivs, np.uint8)
    rc = ctx.lib.tsgpu_rekey_object(ctx._h, flags, s.ctypes.data, s.size if src_len is None else src_len, ts.ctypes.data, ts.size,
                                    k.ctypes.data, None, 0, tk.ctypes.data, None, 0, iv.ctypes.data, dst.ctypes.data, dst.size,
                                    PART, crcs.ctypes.data, part_cap, C.addressof(n_parts), cur.ctypes.data, end,
                                    C.addressof(src_crc), C.addressof(obj_crc))
    return rc, ctx.lib.tsgpu_last_error().decode(), dst, (src_crc.value, obj_crc.value)


@pytest.fixture(scope="module")
def aes_obj():
    rng = np.random.default_rng(9)
    key = rng.bytes(32)
    obj, sizes = K.encrypt_chunks(key, b"", [rng.bytes(2000 + 100 * i) for i in range(7)])
    return obj, sizes, key


@pytest.mark.parametrize("k", [0, 4, 6])
def test_flipped_byte_fails_its_batch_in_a_later_window(ctx, aes_obj, k):
    obj, sizes, key = aes_obj
    bad = obj.copy()
    starts = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    bad[starts[k] + 20] ^= 1
    ivs = _ivs(len(sizes))
    cur = np.zeros(binding.REKEY_CURSOR_SIZE, np.uint8)
    w0 = 3 if k >= 3 else 0                                  # windows of 3 chunks: chunk k sits in a later window when k >= 3
    if w0:
        rc, msg, _, _ = _raw(ctx, bad[:starts[3]], sizes[:3], key, ivs[:36], cursor=cur, end=0)
        assert rc == 0, msg
    rc, msg, dst, words = _raw(ctx, bad[starts[w0]:], sizes[w0:], key, ivs[12 * w0:], cursor=cur)
    assert rc == binding.E_AUTH and msg == "Tag mismatch in chunk %d" % k, msg
    # batches of max_batch = 2 chunks: nothing of chunk k's batch, nor of any later one, reached dst
    b0 = starts[w0 + (k - w0) // 2 * 2] - starts[w0]
    assert (dst[b0:] == 0xEE).all() and words == (0xABCD, 0xABCD)
    want = K.expected(obj[starts[w0]:], sizes[w0:], key, b"", NEW_KEY, b"", ivs[12 * w0:])
    assert np.array_equal(dst[:b0], want[:b0])              # the batches before it did


def test_short_chunks_fail_their_tag(ctx, aes_obj):
    obj, sizes, key = aes_obj
    for n in (1, 12, 27):
        rc, msg, _, _ = _raw(ctx, obj[:n], [n], key, _ivs(1))
        assert rc == binding.E_AUTH and msg == "Tag mismatch in chunk 0", (n, msg)


def test_iv_rules_give_the_rewrites_messages(ctx, aes_obj):
    obj, sizes, key = aes_obj
    ivs = bytearray(_ivs(len(sizes)))
    ivs[5 * 12:6 * 12] = ivs[2 * 12:3 * 12]
    assert _fails(binding.E_ARG, lambda: ctx.rekey_object(obj, sizes, key, NEW_KEY, bytes(ivs), PART)) == "to_ivs[2] repeats to_ivs[5]"
    ivs = bytearray(_ivs(len(sizes)))
    ivs[0:12] = obj[sizes[0] + sizes[1]:sizes[0] + sizes[1] + 12].tobytes()      # chunk 2's IV
    cur = np.zeros(binding.REKEY_CURSOR_SIZE, np.uint8)
    cur[32:40] = np.frombuffer(np.uint64(10).tobytes(), np.uint8)                  # the window starts at chunk 10 of the object
    msg = _fails(binding.E_ARG, lambda: ctx.rekey_object(obj, sizes, key, key, bytes(ivs), PART, cursor=cur, object_ends_here=False))
    assert msg == "to_ivs[0] repeats the IV of chunk 12 under the same key"
    new, _, _ = ctx.rekey_object(obj, sizes, key, NEW_KEY, bytes(ivs), PART)      # under another key it is allowed
    assert new.size == obj.size


def test_short_buffers_and_part_cap(ctx, aes_obj):
    obj, sizes, key = aes_obj
    ivs = _ivs(len(sizes))
    total = int(sum(sizes))
    rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs, src_len=total - 1)
    assert rc == binding.E_SHORT and "fewer bytes" in msg, msg
    rc, msg, dst, words = _raw(ctx, obj, sizes, key, ivs, dst_cap=total - 1)
    assert rc == binding.E_SHORT and "dst too small" in msg and (dst == 0xEE).all() and words == (0xABCD, 0xABCD), msg
    # the bound is exact: floor(total / PART) + 1 parts at the object's end
    rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs, part_cap=total // PART)
    assert rc == binding.E_SHORT and "part_crc32c too small" in msg, msg
    rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs, part_cap=total // PART + 1)
    assert rc == 0, msg
    rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs, part_cap=total // PART, end=0)
    assert rc == 0, msg


def test_oversize_chunk_and_unknown_flags(ctx, aes_obj):
    obj, sizes, key = aes_obj
    stride = ctx.slot_stride(Z | A, CAP)
    big = stride - binding.SLOT_HEAD - 16 + 1                 # one byte more than the context's transformed slot holds
    rc, msg, _, _ = _raw(ctx, np.zeros(big, np.uint8), [big], key, _ivs(1))
    assert rc == binding.E_ARG and "exceeds the context's capacity" in msg, msg
    for f in (tsgpu.FLAG_ZSTD, A, tsgpu.FLAG_REFRAME, 1 << 20):
        msg = _fails(binding.E_ARG, lambda: ctx.rekey_object(obj, sizes, key, NEW_KEY, _ivs(len(sizes)), PART, flags=f | V))
        assert msg.startswith("unknown flags"), msg


def test_null_arguments(ctx, aes_obj):
    obj, sizes, key = aes_obj
    L, h = ctx.lib, ctx._h
    s = np.ascontiguousarray(obj)
    ts = np.ascontiguousarray(sizes, np.uint32)
    dst = np.empty(s.size, np.uint8)
    crcs = np.zeros(64, np.uint32)
    k, nk, iv = (np.frombuffer(b, np.uint8) for b in (key, NEW_KEY, _ivs(len(sizes))))
    n_parts, w = C.c_uint32(0), C.c_uint32(0)
    cur = np.zeros(binding.REKEY_CURSOR_SIZE, np.uint8)
    args = dict(h=h, src=s.ctypes.data, ts=ts.ctypes.data, k=k.ctypes.data, nk=nk.ctypes.data, iv=iv.ctypes.data, dst=dst.ctypes.data,
                crcs=crcs.ctypes.data, n=C.addressof(n_parts), cur=cur.ctypes.data, sw=C.addressof(w), ow=C.addressof(w), aad=None)

    def call(**kw):
        a = dict(args, **kw)
        rc = L.tsgpu_rekey_object(a["h"], 0, a["src"], s.size, a["ts"], ts.size, a["k"], None, 0 if a["aad"] is None else 4,
                                  a["nk"], None, 0, a["iv"], a["dst"], dst.size, PART, a["crcs"], 64, a["n"], a["cur"], 1, a["sw"], a["ow"])
        return rc, L.tsgpu_last_error().decode()

    assert call()[0] == 0
    for kw, want in ((dict(h=None), "ctx cannot be null"), (dict(cur=None), "cursor cannot be null"),
                     (dict(sw=None), "source_crc32c/object_crc32c cannot be null"), (dict(ow=None), "source_crc32c/object_crc32c cannot be null"),
                     (dict(ts=None), "chunks cannot be null"), (dict(k=None), "key is required for decryption"),
                     (dict(aad=True), "aad cannot be null"), (dict(nk=None), "to_key and to_ivs are required for encryption"),
                     (dict(iv=None), "to_key and to_ivs are required for encryption"), (dict(src=None), "inputStream cannot be null"),
                     (dict(dst=None), "dst cannot be null"), (dict(n=None), "n_parts and object_crc32c cannot be null"),
                     (dict(crcs=None), "part_crc32c cannot be null")):
        rc, msg = call(**kw)
        assert rc == binding.E_ARG and want in msg, (kw, msg)


def test_verify_catches_a_wrong_byte_of_the_rekey(ctx, aes_obj):
    obj, sizes, key = aes_obj
    ivs = _ivs(len(sizes))
    os.environ["TSGPU_SIMT_FLIP_REKEYED"] = "5:100"           # one byte of chunk 5's new ciphertext, as a faulty rekey would write it
    try:
        rc, msg, dst, words = _raw(ctx, obj, sizes, key, ivs, flags=V)
        assert rc == binding.E_VERIFY and msg.startswith("verify: chunk 5 did not read back under the new key"), msg
        starts = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
        assert (dst[starts[4]:] == 0xEE).all() and words == (0xABCD, 0xABCD)
        os.environ["TSGPU_SIMT_FLIP_REKEYED"] = "5:-1"        # the last byte of its new tag
        rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs, flags=V)
        assert rc == binding.E_VERIFY and msg == "verify: chunk 5 did not read back under the new key: tag check failed", msg
        rc, msg, _, _ = _raw(ctx, obj, sizes, key, ivs)       # without VERIFY the damaged chunk would have left
        assert rc == 0, msg
    finally:
        del os.environ["TSGPU_SIMT_FLIP_REKEYED"]
