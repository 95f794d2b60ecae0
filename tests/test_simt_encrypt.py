"""tsgpu_encrypt_object on the SIMT emulator.  Unencrypted objects -- written by the oracle (libzstd level 3, what the Java plugin
wrote, and plain), by this library in speed and dense mode with and without the Content_Checksum, and shaped like an .indexes
object with an empty blob -- are encrypted in one call and in windows.  Every new chunk equals OpenSSL's IV || AES-256-GCM(chunk)
|| TAG, the new object detransforms through libzstd and OpenSSL to the segment, and the part, source and object CRCs equal the CPU
CRC-32C and CRC-64/NVME.  The output equals tsgpu_rewrite_object's (frames kept) and tsgpu_transform_parts' with the same IVs.
Refusals name their cause, a failing batch leaves no byte in dst and no CRC is written.  tests/test_gpu_encrypt.py runs 256 MiB
objects on an H100."""
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
import encrypt_util as E  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V, K = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM
CAP = 1 << 16                     # the context's max_chunk_bytes
CS = 8192
PART = 5000
KEY, AAD = bytes(range(7, 39)), b"segment-aad"


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


def _plain_chunks(seg, cs=CS):
    return seg.copy(), [min(cs, seg.size - i) for i in range(0, seg.size, cs)]


def _stored(ctx, seg, kind):
    """(object, sizes, flags) of the segment stored unencrypted"""
    nch = (seg.size + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    if kind == "libzstd":
        obj, sizes = ora.transform_segment(Z, seg, CS, key, aad, ivs)
        return np.asarray(obj).copy(), list(sizes), Z
    if kind == "plain":
        return (*_plain_chunks(seg), 0)
    mode = {"speed": Z, "speed-sum": Z | K, "dense": Z | D, "dense-sum": Z | D | K}[kind]
    cur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    obj, sizes, _, _ = ctx.transform_parts(mode, seg, CS, PART, cur, True, np.zeros(binding.CURSOR_SIZE, np.uint8), key, aad, ivs)
    return np.asarray(obj).copy(), list(sizes), Z


def _check(ctx, obj, sizes, ocs=0, ofs=0, flags=0, aad=AAD, wins=(None, 1, 2), key=KEY):
    """the new object is the oracle's for every window size, with the same sizes and CRCs, in both widths; returns it"""
    ivs = _ivs(len(sizes))
    want, wsz = E.expected(obj, sizes, key, aad, ivs)
    for win in wins:
        new, nsz, parts, crc2 = E.encrypt_windows(ctx, obj, sizes, key, ivs, PART, win, ocs, ofs, aad, flags)
        assert np.array_equal(new, want), win
        assert nsz == wsz and parts == U.part_crcs(want, PART), win
        assert crc2 == (U.crc32c(obj), U.crc32c(want)), win
    new, _, parts, crc2 = E.encrypt_windows(ctx, obj, sizes, key, ivs, PART, wins[-1], ocs, ofs, aad, flags, crc64=True)
    assert np.array_equal(new, want)
    assert parts == U64.part_crcs(want, PART) and crc2 == (U64.crc64nvme(obj), U64.crc64nvme(want))
    return want, wsz


# ---------------------------------------------------------------------------------------------------- what the new object is
@pytest.mark.parametrize("kind", ["libzstd", "speed", "speed-sum", "dense", "dense-sum", "plain"])
def test_stored_log_objects(ctx, seg, kind):
    obj, sizes, flags = _stored(ctx, seg, kind)
    want, wsz = _check(ctx, obj, sizes, CS, seg.size, flags, wins=(None, 1, 2, 3))
    back, _ = ora.detransform_chunks(flags | A, want, wsz, seg.size, KEY, AAD)       # the segment, through libzstd and OpenSSL
    assert np.array_equal(back, seg)


@pytest.mark.parametrize("aad_len", [0, 1, 16, 17, 64])
def test_chunk_sizes_and_aad_lengths(ctx, aad_len):
    # an .indexes-shaped object of blobs of 0 (an empty blob), 1, 15, 16, 17 bytes and a chunk as large as the slot takes
    rng = np.random.default_rng(aad_len)
    aad = rng.bytes(aad_len)
    big = ctx.slot_stride(Z | A, CAP) - binding.SLOT_HEAD - 16 - 28
    blobs = [rng.bytes(n) for n in (0, 1, 15, 16, 17, 16 * 33 + 1, CAP, big)]
    obj = np.frombuffer(b"".join(blobs), np.uint8).copy()
    _check(ctx, obj, [len(b) for b in blobs], aad=aad)


def test_plain_chunk_sizes_against_the_index(ctx):
    # a plain .log object of chunks of 1, 15, 16 and 17 bytes: the chunk index of a 49-byte segment in chunks of 17 is 17, 17, 15
    rng = np.random.default_rng(3)
    for ocs, sizes in ((17, [17, 17, 15]), (1, [1] * 5), (16, [16, 16, 16, 1])):
        obj = np.frombuffer(rng.bytes(sum(sizes)), np.uint8).copy()
        _check(ctx, obj, sizes, ocs, sum(sizes), 0, wins=(None, 1, 2))


def test_indexes_shaped_object(ctx):
    rng = np.random.default_rng(5)
    blobs = [rng.bytes(800), rng.bytes(1200), rng.bytes(33), b"", rng.bytes(4000)]
    obj = np.frombuffer(b"".join(blobs), np.uint8).copy()
    want, wsz = _check(ctx, obj, [len(b) for b in blobs], wins=(None, 1, 2, 4))
    assert wsz[3] == 0 and wsz[0] == 828
    # the empty blob takes no IV: an entry equal to another's passes
    ivs = bytearray(_ivs(5))
    ivs[36:48] = ivs[0:12]
    new, _, _, _ = ctx.encrypt_object(obj, [len(b) for b in blobs], KEY, bytes(ivs), PART, aad=AAD)
    assert np.array_equal(new, E.expected(obj, [len(b) for b in blobs], KEY, AAD, bytes(ivs))[0])


def test_empty_segment_and_empty_windows(ctx):
    new, nsz, parts, crc2 = ctx.encrypt_object(b"", [0], KEY, None, PART, CS, 0)     # the empty segment's one chunk
    assert new.size == 0 and nsz == [0] and parts == [] and crc2 == (0, 0)
    new, nsz, parts, crc2 = ctx.encrypt_object(b"", [], KEY, None, PART, CS, 0)
    assert new.size == 0 and nsz == [] and crc2 == (0, 0)
    rng = np.random.default_rng(6)
    obj = np.frombuffer(rng.bytes(3 * CS), np.uint8).copy()
    _check(ctx, obj, [CS] * 3, CS, 3 * CS, wins=(None, 3))                          # the last window is empty


def test_same_bytes_as_the_rewrite_and_the_transform(ctx, seg):
    nch = (seg.size + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    # an own-writer Zstd-only object rewritten to Zstd+AES with its frames kept
    obj, sizes, _ = _stored(ctx, seg, "speed")
    new, nsz, _, _ = ctx.encrypt_object(obj, sizes, key, ivs, PART, CS, seg.size, aad, Z)
    rw, rsz, _, _ = ctx.rewrite_object(Z, obj, sizes, CS, seg.size, Z | A, PART, to_key=key, to_aad=aad, to_ivs=ivs)
    assert np.array_equal(new, rw) and nsz == rsz
    # a plain object against tsgpu_transform_parts AES-only of the segment
    obj, sizes = _plain_chunks(seg)
    new, nsz, _, _ = ctx.encrypt_object(obj, sizes, key, ivs, PART, CS, seg.size, aad)
    cur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    tp, tsz, _, _ = ctx.transform_parts(A, seg, CS, PART, cur, True, np.zeros(binding.CURSOR_SIZE, np.uint8), key, aad, ivs)
    assert np.array_equal(new, np.asarray(tp)) and nsz == list(tsz)


def test_verify_passes_clean_objects(ctx, seg):
    obj, sizes, flags = _stored(ctx, seg, "libzstd")
    _check(ctx, obj, sizes, CS, seg.size, flags | V, wins=(None, 3))
    blobs = [b"\x01" * 40, b"", b"x", b"\x02" * 5000]
    _check(ctx, np.frombuffer(b"".join(blobs), np.uint8).copy(), [len(b) for b in blobs], flags=V, wins=(None,))


# ---------------------------------------------------------------------------------------------------- refusals and failures
def _raw(ctx, obj, sizes, ocs=0, ofs=0, flags=0, ivs=None, dst_cap=None, part_cap=64, cursor=None, end=1, fill=0xEE, src_len=None):
    """tsgpu_encrypt_object called directly: (rc, message, dst after the call, (source, object) CRC words after the call)"""
    s = np.ascontiguousarray(obj, np.uint8)
    cs = np.ascontiguousarray(sizes, np.uint32)
    total = int(sum(int(x) + 28 for x in cs if x))
    dst = np.full(total if dst_cap is None else dst_cap, fill, np.uint8)
    nsz = np.zeros(max(cs.size, 1), np.uint32)
    crcs = np.zeros(max(part_cap, 1), np.uint32)
    n_parts, src_crc, obj_crc = C.c_uint32(0), C.c_uint32(0xABCD), C.c_uint32(0xABCD)
    cur = np.zeros(binding.ENCRYPT_CURSOR_SIZE, np.uint8) if cursor is None else cursor
    k = np.frombuffer(KEY, np.uint8)
    iv = np.frombuffer(_ivs(cs.size) if ivs is None else ivs, np.uint8)
    rc = ctx.lib.tsgpu_encrypt_object(ctx._h, flags, s.ctypes.data, s.size if src_len is None else src_len, cs.ctypes.data, cs.size,
                                      ocs, ofs, k.ctypes.data, None, 0, iv.ctypes.data, dst.ctypes.data, dst.size, nsz.ctypes.data,
                                      PART, crcs.ctypes.data, part_cap, C.addressof(n_parts), cur.ctypes.data, end,
                                      C.addressof(src_crc), C.addressof(obj_crc))
    return rc, ctx.lib.tsgpu_last_error().decode(), dst, (src_crc.value, obj_crc.value)


@pytest.fixture(scope="module")
def zobj(ctx):
    """a libzstd-written Zstd-only object of 7 chunks of CS bytes: (object, sizes, chunk starts, segment)"""
    rng = np.random.default_rng(9)
    seg = np.frombuffer(b"".join(rng.bytes(300) * 28 for _ in range(7))[:7 * CS - 100], np.uint8).copy()
    nch = (seg.size + CS - 1) // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    obj, sizes = ora.transform_segment(Z, seg, CS, key, aad, ivs)
    obj = np.asarray(obj).copy()
    return obj, list(sizes), np.concatenate([[0], np.cumsum(sizes)]).astype(int), seg


def _frame(obj, starts, k):
    return bytearray(obj[starts[k]:starts[k + 1]].tobytes())


def _with_chunk(zobj, k, chunk):
    """the object with chunk k replaced by `chunk`: (object, sizes)"""
    obj, sizes, starts, _ = zobj
    new = np.concatenate([obj[:starts[k]], np.frombuffer(bytes(chunk), np.uint8), obj[starts[k + 1]:]])
    return new, sizes[:k] + [len(chunk)] + sizes[k + 1:]


def _first_block(f):
    """offset of the first block header of a frame"""
    fhd = f[4]
    single, dict_, fcs = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    return 5 + (0 if single else 1) + [0, 1, 2, 4][dict_] + ([1 if single else 0, 2, 4, 8][fcs])


def _bad_frames(zobj, k):
    """(name, damaged chunk k) for every frame refusal"""
    obj, sizes, starts, seg = zobj
    f = _frame(obj, starts, k)
    out = []
    g = bytearray(f); g[0] ^= 1
    out.append(("magic", g))
    # no Frame_Content_Size: a single-segment frame cannot drop it, so the frame gets a window descriptor instead
    fb = _first_block(f)
    fhd = f[4]
    hdr_fcs = [1 if (fhd >> 5) & 1 else 0, 2, 4, 8][fhd >> 6]
    g = bytearray(f[:4]) + bytes([(fhd & 0x07) | 0x00]) + bytes([0x58]) + f[fb:]
    out.append(("no FCS", g))
    g = bytearray(f); fcs_at = fb - hdr_fcs
    g[fcs_at] ^= 1
    out.append(("wrong FCS", g))
    g = bytearray(f[:4]) + bytes([fhd | 0x01]) + f[5:fb - hdr_fcs] + b"\x07" + f[fb - hdr_fcs:]
    out.append(("dictionary", g))
    g = bytearray(f); g[fb] |= 0x06                                              # Block_Type 3 (reserved)
    out.append(("reserved block", g))
    out.append(("past the chunk", bytearray(f[:-3])))
    out.append(("trailing bytes", bytearray(f) + b"\x00\x01"))
    out.append(("second frame", bytearray(f) + bytearray(f)))
    return out


@pytest.mark.parametrize("k", [0, 4, 6])
def test_frame_refusals_name_their_chunk(ctx, zobj, k):
    obj, sizes, starts, seg = zobj
    for name, chunk in _bad_frames(zobj, k):
        bad, bsz = _with_chunk(zobj, k, chunk)
        ivs = _ivs(len(bsz))
        # windows of 3 chunks: chunk k sits in a later window when k >= 3
        cur = np.zeros(binding.ENCRYPT_CURSOR_SIZE, np.uint8)
        w0 = 3 if k >= 3 else 0
        bstarts = np.concatenate([[0], np.cumsum(bsz)]).astype(int)
        if w0:
            rc, msg, _, _ = _raw(ctx, bad[:bstarts[3]], bsz[:3], CS, seg.size, Z, ivs=ivs[:36], cursor=cur, end=0)
            assert rc == 0, (name, msg)
        rc, msg, dst, words = _raw(ctx, bad[bstarts[w0]:], bsz[w0:], CS, seg.size, Z, ivs=ivs[12 * w0:], cursor=cur)
        if name == "wrong FCS":
            assert rc == binding.E_CORRUPT and msg.startswith("chunk %d decoded to " % k), (name, msg)
            assert msg.endswith("the chunk index gives %d" % min(CS, seg.size - k * CS)), (name, msg)
        else:
            assert rc == binding.E_CORRUPT and msg == "Invalid zstd frame in chunk %d (code 2)" % k, (name, msg)
        # batches of max_batch = 2 chunks: nothing of chunk k's batch, nor of any later one, reached dst; no CRC was written
        want, wsz = E.expected(bad[bstarts[w0]:], bsz[w0:], KEY, b"", ivs[12 * w0:])
        b0 = sum(wsz[:(k - w0) // 2 * 2])
        assert (dst[b0:] == 0xEE).all() and words == (0xABCD, 0xABCD), name
        assert np.array_equal(dst[:b0], want[:b0]), name                    # the batches before it did


def test_a_good_frame_with_a_checksum_and_skippable_frames_passes(ctx, zobj):
    obj, sizes, starts, seg = zobj
    skip = b"\x5a\x2a\x4d\x18" + (5).to_bytes(4, "little") + b"12345"
    bad, bsz = _with_chunk(zobj, 2, _frame(obj, starts, 2) + skip)
    rc, msg, _, _ = _raw(ctx, bad, bsz, CS, seg.size, Z)
    assert rc == 0, msg
    rc, msg, _, _ = _raw(ctx, bad, bsz, CS, seg.size, Z | V)
    assert rc == 0, msg


def test_sizes_and_chunk_count_against_the_index(ctx, zobj):
    obj, sizes, starts, seg = zobj
    # a plain object: a chunk one byte short, then the index's chunk count at the end
    plain, psz = _plain_chunks(seg)
    rc, msg, _, _ = _raw(ctx, plain[:-1], psz[:-1] + [psz[-1] - 1], CS, seg.size)
    assert rc == binding.E_CORRUPT and msg == "chunk 6 decoded to %d bytes, the chunk index gives %d" % (psz[-1] - 1, psz[-1]), msg
    rc, msg, _, _ = _raw(ctx, plain[:-psz[-1]], psz[:-1], CS, seg.size)
    assert rc == binding.E_CORRUPT and msg.startswith("the object has 6 chunks, the chunk index"), msg
    rc, msg, _, _ = _raw(ctx, plain[:-psz[-1]], psz[:-1], CS, seg.size, end=0)       # not at the end: no count yet
    assert rc == 0, msg
    rc, msg, _, _ = _raw(ctx, np.concatenate([plain, plain[:5]]), psz + [5], CS, seg.size)
    assert rc == binding.E_CORRUPT and msg.startswith("chunk 7 decoded to 5 bytes, but the chunk index"), msg
    # a zstd object with one frame too many
    rc, msg, _, _ = _raw(ctx, np.concatenate([obj, obj[:starts[1]]]), sizes + [sizes[0]], CS, seg.size, Z)
    assert rc == binding.E_CORRUPT and "but the chunk index" in msg, msg
    # a zstd object with an empty chunk where the index has one
    rc, msg, _, _ = _raw(ctx, obj[:starts[1]], [sizes[0], 0], CS, seg.size, Z, end=0)
    assert rc == binding.E_CORRUPT and msg == "chunk 1 decoded to 0 bytes, the chunk index gives %d" % CS, msg


def test_flag_refusals(ctx, zobj):
    obj, sizes, starts, seg = zobj
    msg = _fails(binding.E_ARG, lambda: ctx.encrypt_object(obj, sizes, KEY, _ivs(7), PART, CS, seg.size, flags=Z | A))
    assert "tsgpu_rekey_object" in msg, msg
    for f in (D, K, tsgpu.FLAG_VALIDATE_RECORDS, tsgpu.FLAG_REFRAME, 1 << 20):
        msg = _fails(binding.E_ARG, lambda: ctx.encrypt_object(obj, sizes, KEY, _ivs(7), PART, CS, seg.size, flags=Z | f))
        assert msg.startswith("unknown flags"), msg
    msg = _fails(binding.E_ARG, lambda: ctx.encrypt_object(obj, sizes, KEY, _ivs(7), PART, 0, 0, flags=Z))
    assert "chunk index" in msg, msg


def test_duplicate_iv(ctx, zobj):
    obj, sizes, starts, seg = zobj
    ivs = bytearray(_ivs(len(sizes)))
    ivs[5 * 12:6 * 12] = ivs[2 * 12:3 * 12]
    msg = _fails(binding.E_ARG, lambda: ctx.encrypt_object(obj, sizes, KEY, bytes(ivs), PART, CS, seg.size, flags=Z))
    assert msg == "to_ivs[2] repeats to_ivs[5]", msg


def test_short_buffers_part_cap_and_oversize(ctx, zobj):
    obj, sizes, starts, seg = zobj
    total = int(sum(sizes)) + 28 * len(sizes)
    rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z, src_len=obj.size - 1)
    assert rc == binding.E_SHORT and "fewer bytes" in msg, msg
    rc, msg, dst, words = _raw(ctx, obj, sizes, CS, seg.size, Z, dst_cap=total - 1)
    assert rc == binding.E_SHORT and "dst too small" in msg and (dst == 0xEE).all() and words == (0xABCD, 0xABCD), msg
    # the bound is exact: floor(total / PART) + 1 parts at the object's end
    rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z, part_cap=total // PART)
    assert rc == binding.E_SHORT and "part_crc32c too small" in msg, msg
    rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z, part_cap=total // PART + 1)
    assert rc == 0, msg
    rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z, part_cap=total // PART, end=0)
    assert rc == 0, msg
    big = ctx.slot_stride(Z | A, CAP) - binding.SLOT_HEAD - 16 - 28 + 1      # one byte more than the transformed slot takes
    rc, msg, _, _ = _raw(ctx, np.zeros(big, np.uint8), [big])
    assert rc == binding.E_ARG and "exceeds the context's capacity" in msg, msg
    rc, msg, _, _ = _raw(ctx, np.zeros(big - 1, np.uint8), [big - 1])
    assert rc == 0, msg


def test_verify_catches_a_flipped_byte(ctx, zobj):
    obj, sizes, starts, seg = zobj
    os.environ["TSGPU_SIMT_FLIP"] = "5:100"                   # one byte of chunk 5's ciphertext, as a faulty encryption would write it
    try:
        rc, msg, dst, words = _raw(ctx, obj, sizes, CS, seg.size, Z | V)
        assert rc == binding.E_VERIFY and msg.startswith("verify: chunk 5 did not read back"), msg
        want, wsz = E.expected(obj, sizes, KEY, b"", _ivs(len(sizes)))
        assert (dst[sum(wsz[:4]):] == 0xEE).all() and words == (0xABCD, 0xABCD)
        os.environ["TSGPU_SIMT_FLIP"] = "5:-1"                # the last byte of its tag
        rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z | V)
        assert rc == binding.E_VERIFY and msg == "verify: chunk 5 did not read back: tag check failed", msg
        rc, msg, _, _ = _raw(ctx, obj, sizes, CS, seg.size, Z)   # without VERIFY the damaged chunk would have left
        assert rc == 0, msg
    finally:
        del os.environ["TSGPU_SIMT_FLIP"]
