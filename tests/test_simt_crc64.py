"""The CRC-64/NVME calls on the SIMT emulator (tsgpu_transform_parts_crc64, tsgpu_check_object_crc64,
tsgpu_rewrite_object_crc64): every part CRC and the object CRC equal the CPU CRC-64/NVME (tests/crc64_util.py) of the returned
object, for objects of 0, 29 (one AES chunk of 1 byte), 255, 256 and 257 bytes, 32 KiB - 1, 32 KiB and 32 KiB + 1 (one 256-byte piece and one 32 KiB tile
either side of their ends) and several tiles per batch; part sizes of 1, 7 and 256 bytes and 5 MiB; a part boundary exactly at a
chunk end; and a segment in windows through one cursor.  The check and the rewrite give the oracle's object, source and segment
words, in one call and in windows.  Each call writes the bytes and sizes of its CRC-32C twin, and an error writes no checksum.
The kernels also run under AddressSanitizer, with poisoned scratch and with reversed and random lane orders.
tests/test_gpu_crc64.py runs them on an H100."""
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
import crc64_util as U  # noqa: E402
import records_util as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V, CK, VR = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM,
                      tsgpu.FLAG_VALIDATE_RECORDS)
CS = 4096
TILE = 32768
MIB = 1 << 20


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=16, lib_path=SIMT_LIB)     # up to 16 chunks: several tiles per batch
    yield c
    c.close()


def _keys(n, cs=CS):
    return corpus.fixed_key_material(max((n + cs - 1) // cs, 1))


def _check(obj, crcs, ocrc, part):
    assert crcs == U.part_crcs(obj, part), part
    assert ocrc == U.crc64nvme(obj)


def _both(c, flags, s, cs, part, keys):
    """the CRC-64 call and its CRC-32C twin on one segment: the 64-bit results, after checking that the bytes agree"""
    pc64, pc32 = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8), np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    out, sizes, crcs, ocrc = c.transform_parts_crc64(flags, s, cs, part, pc64, True, None, *keys)
    out = out.copy()
    out32, sizes32, crcs32, _ = c.transform_parts(flags, s, cs, part, pc32, True, None, *keys)
    assert len(crcs32) == len(crcs)
    if flags & D or not flags & Z:                                   # deterministic writers: the same bytes
        assert sizes == sizes32 and np.array_equal(out, out32)
    return out, sizes, crcs, ocrc


def test_oracle_is_crc64_nvme():
    assert U.crc64nvme(b"123456789") == U.CHECK == 0xAE8B14860A799888
    assert U.crc64nvme(b"") == 0 and U.part_crcs(b"", 5) == []
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 8, 9, 63, 64, 65, 300, 1000):
        b = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        assert U.crc64nvme(b) == U.crc64nvme_bitwise(b), n
    b = rng.integers(0, 256, 1000, dtype=np.uint8).tobytes()
    assert U.part_crcs(b, 7) == [U.crc64nvme_bitwise(b[i:i + 7]) for i in range(0, 1000, 7)]


# ---------------------------------------------------------------------------------------------------- object lengths
# AES alone writes n + 28 bytes per chunk: one chunk of n bytes is an object of exactly n + 28
@pytest.mark.parametrize("obj_len", [29, 255, 256, 257, TILE - 1, TILE, TILE + 1])
def test_object_lengths_around_pieces_and_tiles(ctx, obj_len):
    s, cs, flags = corpus.gen_segment("K", 1, obj_len - 28, obj_len - 28), obj_len - 28, A
    keys = _keys(s.size, cs)
    for part in (1, 7, 256, 5 * MIB):
        out, sizes, crcs, ocrc = _both(ctx, flags, s, cs, part, keys)
        assert out.size == obj_len
        _check(out, crcs, ocrc, part)


def test_empty_segment(ctx):
    s = np.zeros(0, np.uint8)
    out, sizes, crcs, ocrc = ctx.transform_parts_crc64(Z | A, s, CS, 256, np.zeros(32, np.uint8), True, None, *_keys(0))
    assert out.size == 0 and sizes == [] and crcs == [] and ocrc == 0


@pytest.mark.parametrize("flags", [Z, Z | D, A, Z | A, Z | D | A, Z | CK | A, Z | A | V],
                         ids=["Z", "ZD", "A", "ZA", "ZDA", "ZCA", "ZAV"])
def test_several_tiles_per_batch(ctx, flags):
    s = corpus.gen_segment("R", 3, 20 * CS + 123, CS)                 # 21 chunks: a 16-chunk batch of 2+ tiles and a short one
    keys = _keys(s.size)
    for part in (7, 256, 5000, 5 * MIB):
        out, _, crcs, ocrc = _both(ctx, flags, s, CS, part, keys)
        _check(out, crcs, ocrc, part)


def test_part_boundary_at_a_chunk_end(ctx):
    s = corpus.gen_segment("K", 4, 7 * CS + 99, CS)
    keys = _keys(s.size)
    for part in (CS + 28, 2 * (CS + 28), CS + 27, CS + 29):           # AES alone: every chunk is CS + 28 bytes
        out, sizes, crcs, ocrc = _both(ctx, A, s, CS, part, keys)
        assert sizes[0] == CS + 28
        _check(out, crcs, ocrc, part)


# ---------------------------------------------------------------------------------------------------- windows
def _windows(c, flags, s, part, win_chunks, keys, records=False):
    key, aad, ivs = keys
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    rc = np.zeros(binding.CURSOR_SIZE, np.uint8) if records else None
    outs, sizes, crcs, lo, w = [], [], [], 0, win_chunks * CS
    while True:
        win = s[lo:lo + w]
        end = win.size < w                                            # after a full last window, an empty end call
        iv = ivs[12 * (lo // CS):] if win.size else b"\0" * 12
        o, z, p, oc = c.transform_parts_crc64(flags, win, CS, part, pc, end, rc, key, aad, iv)
        outs.append(o.copy()); sizes += z; crcs += p
        if end:
            return np.concatenate(outs), sizes, crcs, oc
        lo += w


@pytest.mark.parametrize("n", [6 * CS, 6 * CS + 777], ids=["whole-windows", "short-last-window"])
@pytest.mark.parametrize("flags", [Z | D, A, Z | A], ids=["ZD", "A", "ZA"])
def test_windows_through_one_cursor(ctx, flags, n):
    """6 CS in windows of 1 and 3 chunks ends with a full window: an empty end call finishes the open part and the object"""
    s = corpus.gen_segment("K", 6, n, CS)
    keys = _keys(s.size)
    whole, wsizes, _, _ = _both(ctx, flags, s, CS, 256, keys)
    for part in (7, 256, CS + 28, 5 * MIB):
        for win_chunks in (1, 3):
            obj, sizes, crcs, ocrc = _windows(ctx, flags, s, part, win_chunks, keys)
            _check(obj, crcs, ocrc, part)
            if flags & D or not flags & Z:
                assert sizes == wsizes and np.array_equal(obj, whole)


def test_windows_with_record_validation(ctx):
    s = R.gen_segment(8, 60000, big=9000)
    obj, _, crcs, ocrc = _windows(ctx, Z | D | A | VR, s, 5000, 3, _keys(s.size), records=True)
    _check(obj, crcs, ocrc, 5000)


# ---------------------------------------------------------------------------------------------------- check and rewrite
@pytest.mark.parametrize("flags", [0, A, Z, Z | A, Z | D | A], ids=["plain", "A", "Z", "ZA", "ZDA"])
def test_check_object_words(ctx, flags):
    s = R.gen_segment(2, 50000, big=9000)
    key, aad, ivs = _keys(s.size)
    out, sizes = ctx.transform(flags, s, CS, key, aad, ivs)
    out = out.copy()
    want = (U.crc64nvme(out), U.crc64nvme(s))
    assert ctx.check_object_crc64(flags, out, sizes, CS, s.size, key=key, aad=aad) == want
    # in windows of 3 chunks through one cursor, with the records checked too
    cur, lo = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8), 0
    for i in range(0, len(sizes), 3):
        n = sum(sizes[i:i + 3])
        r = ctx.check_object_crc64(flags | VR, out[lo:lo + n], sizes[i:i + 3], CS, s.size, cur, i + 3 >= len(sizes), key, aad)
        lo += n
    assert r == want


def test_check_object_written_by_the_oracle(ctx):
    s = R.gen_segment(3, 40000, big=7000)
    key, aad, ivs = _keys(s.size)
    for flags in (ora.FLAG_AES, ora.FLAG_ZSTD, ora.FLAG_ZSTD | ora.FLAG_AES):
        ref, rsizes = ora.transform_segment(flags, s, CS, key, aad, ivs)
        ref = np.asarray(ref, np.uint8)
        assert ctx.check_object_crc64(flags, ref, rsizes, CS, s.size, key=key, aad=aad) == (U.crc64nvme(ref), U.crc64nvme(s))


def test_check_empty_segment(ctx):
    assert ctx.check_object_crc64(Z | A, np.zeros(0, np.uint8), [0], CS, 0, key=_keys(0)[0]) == (0, 0)


@pytest.mark.parametrize("from_flags,to_flags", [(Z, Z | A), (0, Z), (A, Z | D | A)], ids=["kept-frames", "plain-compressed", "A-ZDA"])
def test_rewrite_words(ctx, from_flags, to_flags):
    s = R.gen_segment(4, 45000, big=8000)
    key, aad, ivs = _keys(s.size)
    old, osizes = ctx.transform(from_flags, s, CS, key, aad, ivs)
    old = old.copy()
    new_key = bytes(range(32))
    nivs = bytes((i * 7 + 3) & 255 for i in range(12 * len(osizes)))
    kw = dict(from_key=key, from_aad=aad, to_key=new_key, to_aad=aad, to_ivs=nivs)
    out, sizes, crcs, words = ctx.rewrite_object_crc64(from_flags, old, osizes, CS, s.size, to_flags, 5000, **kw)
    out = out.copy()
    assert words == (U.crc64nvme(old), U.crc64nvme(out), U.crc64nvme(s))
    assert crcs == U.part_crcs(out, 5000)
    out32, sizes32, crcs32, _ = ctx.rewrite_object(from_flags, old, osizes, CS, s.size, to_flags, 5000, **kw)
    if to_flags & D or not (to_flags & Z) or (from_flags & Z):       # deterministic writers (kept frames included)
        assert sizes == sizes32 and np.array_equal(out, out32)
    # in windows of 2 chunks through one cursor
    cur, lo, objs, pcs = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8), 0, [], []
    for i in range(0, len(osizes), 2):
        n = sum(osizes[i:i + 2])
        kw["to_ivs"] = nivs[12 * i:]
        o, _, p, w = ctx.rewrite_object_crc64(from_flags, old[lo:lo + n], osizes[i:i + 2], CS, s.size, to_flags, 5000, cur,
                                              i + 2 >= len(osizes), **kw)
        objs.append(o.copy()); pcs += p; lo += n
    obj = np.concatenate(objs)
    assert w == (U.crc64nvme(old), U.crc64nvme(obj), U.crc64nvme(s)) and pcs == U.part_crcs(obj, 5000)


# ---------------------------------------------------------------------------------------------------- errors write nothing
def test_part_cap_one_below_the_bound_writes_nothing(ctx):
    s = corpus.gen_segment("K", 1, 3 * CS, CS)
    key, aad, ivs = (np.frombuffer(bytes(x), np.uint8) for x in _keys(s.size))
    bound = int(ctx.lib.tsgpu_transform_bound(Z | A, s.size, CS))
    need = bound // 4096 + 1

    def raw(cap):
        dst = np.empty(bound + 64, np.uint8)
        sizes = np.zeros(8, np.uint32)
        n = C.c_uint32(sizes.size)
        crcs = np.full(need + 1, 0xDEADBEEFDEADBEEF, np.uint64)
        n_parts, obj = C.c_uint32(12345), C.c_uint64(0xDEADBEEFDEADBEEF)
        pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
        rc = ctx.lib.tsgpu_transform_parts_crc64(ctx.handle, Z | A, s.ctypes.data, s.size, CS, key.ctypes.data, aad.ctypes.data,
                                                 aad.size, ivs.ctypes.data, dst.ctypes.data, dst.size, sizes.ctypes.data,
                                                 C.addressof(n), None, 1, 4096, pc.ctypes.data,
                                                 crcs.ctypes.data, cap, C.addressof(n_parts), C.addressof(obj))
        return rc, crcs, n_parts.value, obj.value
    rc, crcs, k, obj = raw(need - 1)
    assert rc == binding.E_SHORT and (crcs == 0xDEADBEEFDEADBEEF).all() and k == 12345 and obj == 0xDEADBEEFDEADBEEF
    assert "part_crc64 too small" in ctx.lib.tsgpu_last_error().decode()
    rc, crcs, k, obj = raw(need)
    assert rc == binding.OK and obj != 0xDEADBEEFDEADBEEF and k > 0


def test_damaged_object_writes_no_word(ctx):
    s = corpus.gen_segment("K", 2, 5 * CS, CS)
    key, aad, ivs = _keys(s.size)
    out, sizes = ctx.transform(A, s, CS, key, aad, ivs)
    bad = out.copy()
    bad[100] ^= 1
    obj, seg = C.c_uint64(7), C.c_uint64(7)
    ts = np.asarray(sizes, np.uint32)
    k = np.frombuffer(bytes(key), np.uint8)
    a = np.frombuffer(bytes(aad), np.uint8)
    cur = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8)
    rc = ctx.lib.tsgpu_check_object_crc64(ctx.handle, A, bad.ctypes.data, bad.size, ts.ctypes.data, ts.size, CS, s.size,
                                          k.ctypes.data, a.ctypes.data, a.size, cur.ctypes.data, 1,
                                          C.addressof(obj), C.addressof(seg))
    assert rc == binding.E_AUTH and obj.value == 7 and seg.value == 7


# ---------------------------------------------------------------------------------------------------- sanitizers and lane orders
def _sweep(lib, env_extra, preload=None):
    env = dict(os.environ, **env_extra)
    if preload:
        env["LD_PRELOAD"] = preload
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_crc64.py"), lib], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "crc64 sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]


def test_crc64_shapes_are_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    U._oracle()                                                       # built before libasan is preloaded
    _sweep("libtsgpu_simt_asan.so", {"ASAN_OPTIONS": "detect_leaks=0"}, runtime)


@pytest.mark.parametrize("env", [{"TSGPU_SIMT_POISON": "1"}, {"TSGPU_SIMT_ORDER": "reverse"}, {"TSGPU_SIMT_ORDER": "random:7"}],
                         ids=["poison", "reverse", "random"])
def test_crc64_shapes_with_poison_and_lane_orders(env):
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    _sweep("libtsgpu_simt.so", env)
