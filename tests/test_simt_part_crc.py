"""tsgpu_transform_parts on the SIMT emulator: every part CRC equals the CPU CRC-32C (tests/part_crc_util.py) of bytes
[k*P, (k+1)*P) of the returned object and the object CRC equals that of the whole object, for every flag mix, corpora K, R and
Z, segment lengths around a chunk, part sizes from 1 byte to more than the object, a context whose 2-chunk batches put part
boundaries inside batches, at batch ends and at chunk ends, and segments cut into windows at every alignment to the parts.
The bytes are those of tsgpu_transform_cursor; argument errors and a VERIFY or RECORDS failure write no part CRC.
tests/test_gpu_part_crc.py runs 1 GiB segments on an H100."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V, CK, VR = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM,
                      tsgpu.FLAG_VALIDATE_RECORDS)
CS = 4096
FLAG_MIXES = [Z, Z | D, A, Z | A, Z | D | A, Z | CK | A, Z | A | V, Z | D | V]
FLAG_IDS = ["Z", "ZD", "A", "ZA", "ZDA", "ZCA", "ZAV", "ZDV"]
LENGTHS = [0, 1, CS - 1, CS, CS + 1, 3 * CS + 1234, 9 * CS + 100]
KINDS = ["K", "R", "Z"]


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=2, lib_path=SIMT_LIB)
    yield c
    c.close()


def _seg(kind, n, seed=1):
    return corpus.gen_segment(kind, seed, n, CS) if n else np.zeros(0, np.uint8)


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


def _parts(c, flags, s, part, **kw):
    return c.transform_parts(flags, s, CS, part, np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8), True, **kw)


def _check(obj, crcs, ocrc, part):
    assert crcs == U.part_crcs(obj, part), part
    assert ocrc == U.crc32c(obj)


def test_oracle_check_value():
    assert U.crc32c(b"123456789") == 0xE3069283 and U.crc32c(b"") == 0


# ---------------------------------------------------------------------------------------------------- one call
@pytest.mark.parametrize("n", LENGTHS)
@pytest.mark.parametrize("flags", FLAG_MIXES, ids=FLAG_IDS)
def test_every_part_of_one_call(ctx, flags, n):
    s = _seg(KINDS[LENGTHS.index(n) % 3], n)
    key, aad, ivs = _keys(n)
    ref, rsizes = ctx.transform_cursor(flags, s, CS, np.zeros(binding.CURSOR_SIZE, np.uint8), True, key, aad, ivs)
    ref = ref.copy()
    one_chunk = rsizes[0] if rsizes else 1                       # exactly one chunk's output
    for part in (1, 7, 4095, 4096, 65536, one_chunk, ref.size + 1):
        if part in (1, 7) and n > 2 * CS:                         # byte-sized parts on the short segments only (emulator time)
            continue
        out, sizes, crcs, ocrc = _parts(ctx, flags, s, part, key=key, aad=aad, ivs=ivs)
        _check(out, crcs, ocrc, part)
        assert len(crcs) == (out.size + part - 1) // part
        if flags & D or not flags & Z:                            # deterministic writers: tsgpu_transform_cursor's bytes
            assert sizes == rsizes and np.array_equal(out, ref)
    if n == 0:
        assert crcs == [] and ocrc == 0


@pytest.mark.parametrize("kind", KINDS)
def test_part_boundaries_at_batch_and_chunk_ends(ctx, kind):
    """AES alone: every chunk is CS + 28 bytes, so parts of one chunk, one batch (2 chunks) and their neighbours end exactly at
    chunk and batch ends, one byte before and one after"""
    s = _seg(kind, 7 * CS + 99)
    key, aad, ivs = _keys(s.size)
    for part in (CS + 28, 2 * (CS + 28), CS + 27, CS + 29, 2 * (CS + 28) - 1, 2 * (CS + 28) + 1):
        out, sizes, crcs, ocrc = _parts(ctx, A, s, part, key=key, aad=aad, ivs=ivs)
        assert sizes[0] == CS + 28
        _check(out, crcs, ocrc, part)


# ---------------------------------------------------------------------------------------------------- windows
def _windows(c, flags, s, part, win_chunks, keys, records=None):
    """the segment in windows of win_chunks chunks, as GpuTransformChunkEnumeration cuts it (an empty end call after a full last
    window), with one parts cursor"""
    key, aad, ivs = keys
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    rc = np.zeros(binding.CURSOR_SIZE, np.uint8) if records is None else records
    outs, sizes, crcs, lo, w = [], [], [], 0, win_chunks * CS
    while True:
        win = s[lo:lo + w]
        end = win.size < w
        iv = ivs[12 * (lo // CS):] if win.size else b"\0" * 12
        o, z, p, oc = c.transform_parts(flags, win, CS, part, pc, end, rc, key, aad, iv)
        outs.append(o.copy()); sizes += z; crcs += p
        if end:
            return np.concatenate(outs), sizes, crcs, oc
        lo += w


@pytest.mark.parametrize("flags", [Z, Z | D, A, Z | A, Z | D | A], ids=["Z", "ZD", "A", "ZA", "ZDA"])
@pytest.mark.parametrize("n", [6 * CS, 6 * CS + 777])
def test_windows_give_the_parts_of_one_call(ctx, flags, n):
    s = _seg("K", n, seed=4)
    keys = _keys(n)
    whole, wsizes = ctx.transform_cursor(flags, s, CS, np.zeros(binding.CURSOR_SIZE, np.uint8), True, *keys)
    whole = whole.copy()
    for part in (1, 7, 3000, CS + 28, whole.size // 3):
        if part == 1 and n % CS:
            continue
        for win_chunks in (1, 2, 3):
            obj, sizes, crcs, ocrc = _windows(ctx, flags, s, part, win_chunks, keys)
            _check(obj, crcs, ocrc, part)                        # speed mode: against the bytes of the run that produced them
            if flags & D or not flags & Z:
                assert sizes == wsizes and np.array_equal(obj, whole)


def test_part_carried_across_many_windows(ctx):
    s = _seg("R", 11 * CS + 5, seed=6)
    keys = _keys(s.size)
    obj, sizes, crcs, ocrc = _windows(ctx, A, s, 5 * CS + 1, 1, keys)       # each part spans five or six windows
    _check(obj, crcs, ocrc, 5 * CS + 1)


def test_empty_end_call_finishes_the_object(ctx):
    s = _seg("K", 4 * CS, seed=7)
    key, aad, ivs = _keys(s.size)
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    out, _, crcs, oc = ctx.transform_parts(A, s, CS, 3000, pc, False, None, key, aad, ivs)
    assert oc is None and len(crcs) == out.size // 3000
    _, _, last, oc = ctx.transform_parts(A, s[:0], CS, 3000, pc, True, None, key, aad, ivs[:12])
    obj = out.copy()
    _check(obj, crcs + last, oc, 3000)
    assert len(last) == 1                                            # the open part


# ---------------------------------------------------------------------------------------------------- with record validation
def test_with_record_validation_in_windows(ctx):
    s = R.gen_segment(8, 60000, big=9000)
    keys = _keys(s.size)
    whole, _ = ctx.transform_cursor(Z | D | A | VR, s, CS, np.zeros(binding.CURSOR_SIZE, np.uint8), True, *keys)
    for part in (7, 5000):
        obj, _, crcs, ocrc = _windows(ctx, Z | D | A | VR, s, part, 3, keys)
        _check(obj, crcs, ocrc, part)
        assert np.array_equal(obj, whole)


# ---------------------------------------------------------------------------------------------------- errors write nothing
def _raw(c, flags, s, part, part_cap, pcur, rcur=None, ends=1):
    """tsgpu_transform_parts with sentinel-filled outputs: (rc, crcs, n_parts, object crc)"""
    key, aad, ivs = (np.frombuffer(bytes(x), np.uint8) for x in _keys(s.size))
    dst = np.empty(int(c.lib.tsgpu_transform_bound(flags, s.size, CS)) + 64, np.uint8)
    sizes = np.zeros(s.size // CS + 2, np.uint32)
    n = C.c_uint32(sizes.size)
    crcs = np.full(max(part_cap, 1), 0xDEADBEEF, np.uint32)
    n_parts, obj = C.c_uint32(12345), C.c_uint32(0xDEADBEEF)
    rc = c.lib.tsgpu_transform_parts(c.handle, flags, s.ctypes.data, s.size, CS, key.ctypes.data, aad.ctypes.data, aad.size,
                                     ivs.ctypes.data, dst.ctypes.data, dst.size, sizes.ctypes.data, C.addressof(n),
                                     None if rcur is None else rcur.ctypes.data, ends, part, None if pcur is None else pcur.ctypes.data,
                                     crcs.ctypes.data, part_cap, C.addressof(n_parts), C.addressof(obj))
    return rc, crcs, n_parts.value, obj.value


def _untouched(res):
    rc, crcs, n_parts, obj = res
    assert (crcs == 0xDEADBEEF).all() and n_parts == 12345 and obj == 0xDEADBEEF
    return rc


def test_argument_errors(ctx):
    s = _seg("K", 3 * CS)
    pc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    assert _untouched(_raw(ctx, Z | A, s, 0, 100, pc)) == binding.E_ARG                 # part_size 0
    assert _untouched(_raw(ctx, 0, s, 4096, 100, pc)) == binding.E_ARG                  # flags 0: no byte reaches the GPU
    assert _untouched(_raw(ctx, Z | A, s, 4096, 100, None)) == binding.E_ARG            # NULL parts cursor
    assert _untouched(_raw(ctx, Z | A | VR, s, 4096, 100, pc, None)) == binding.E_ARG   # NULL records cursor with the flag
    bound = int(ctx.lib.tsgpu_transform_bound(Z | A, s.size, CS))
    need = bound // 4096 + 1
    assert _untouched(_raw(ctx, Z | A, s, 4096, need - 1, pc)) == binding.E_SHORT       # part_cap below the bound
    assert _raw(ctx, Z | A, s, 4096, need, pc)[0] == binding.OK
    # a carried open part counts: 4000 bytes of a 4096-byte part are open after this call
    pc2 = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
    rc, _, k, _ = _raw(ctx, A, _seg("K", 4096 * 3), 4096, 10, pc2, ends=0)
    assert rc == 0 and k == 3                                                            # 3 * 4124 bytes: 3 parts and 84 open
    need2 = (84 + int(ctx.lib.tsgpu_transform_bound(A, CS, CS))) // 4096 + 1
    assert _untouched(_raw(ctx, A, _seg("K", CS), 4096, need2 - 1, pc2.copy())) == binding.E_SHORT
    assert _raw(ctx, A, _seg("K", CS), 4096, need2, pc2.copy())[0] == binding.OK
    assert _untouched(_raw(ctx, A, _seg("K", CS), 4097, 10, pc2.copy())) == binding.E_ARG   # another part size mid-object


def test_verify_failure_writes_no_part_crc(ctx, monkeypatch):
    s = _seg("K", 9 * CS)
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "6:100")                 # a fault in the 4th batch's output: 3 batches drained first
    rc = _untouched(_raw(ctx, Z | A | V, s, 1000, 1000, np.zeros(32, np.uint8)))
    assert rc == binding.E_VERIFY
    monkeypatch.delenv("TSGPU_SIMT_FLIP")
    rc, crcs, k, obj = _raw(ctx, Z | A | V, s, 1000, 1000, np.zeros(32, np.uint8))
    assert rc == 0 and k > 0


def test_records_failure_writes_no_part_crc(ctx):
    s = R.gen_segment(9, 40000, big=3000)
    bad = s.copy()
    bad[int(R.starts(s)[-2]) + 30] ^= 1                             # an entry near the end: earlier batches drain first
    rc = _untouched(_raw(ctx, Z | VR, bad, 500, 1000, np.zeros(32, np.uint8), np.zeros(64, np.uint8)))
    assert rc == binding.E_RECORDS
    assert _raw(ctx, Z | VR, s, 500, 1000, np.zeros(32, np.uint8), np.zeros(64, np.uint8))[0] == 0


# ---------------------------------------------------------------------------------------------------- sanitizers and lane orders
def _sweep(lib, env_extra, preload=None):
    env = dict(os.environ, **env_extra)
    if preload:
        env["LD_PRELOAD"] = preload
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_part_crc.py"), lib], env=env,
                         capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "part crc sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]


def test_part_crc_shapes_are_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    U._oracle(); R._oracle()                                        # built before libasan is preloaded
    _sweep("libtsgpu_simt_asan.so", {"ASAN_OPTIONS": "detect_leaks=0"}, runtime)


def test_part_crc_shapes_are_clean_under_ubsan():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_ubsan.so"])
    runtime = subprocess.run(["gcc", "-print-file-name=libubsan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libubsan not available")
    _sweep("libtsgpu_simt_ubsan.so", {}, runtime)


@pytest.mark.parametrize("env", [{"TSGPU_SIMT_POISON": "1"}, {"TSGPU_SIMT_ORDER": "reverse"}, {"TSGPU_SIMT_ORDER": "random:7"}],
                         ids=["poison", "reverse", "random"])
def test_part_crc_shapes_with_poison_and_lane_orders(env):
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    _sweep("libtsgpu_simt.so", env)
