"""TSGPU_FLAG_VALIDATE_RECORDS on the SIMT emulator: generated Kafka segments (v2 batches from 61 bytes to larger than a chunk
and a slot batch, legacy v0/v1 entries, K or R payloads) pass with every flag mix and transform to exactly the flag-off bytes;
every class of damage fails with TSGPU_E_RECORDS at the CPU oracle's first position and check, wherever the damaged entry lies
(first, last, across a chunk, a slot batch or a call).  tests/test_gpu_records.py runs 1 GiB segments on an H100."""
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
import records_util as R  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V, C, VR = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM,
                     tsgpu.FLAG_VALIDATE_RECORDS)
CAP = 1 << 16


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=CAP, max_batch=2, lib_path=SIMT_LIB)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    # ~400 KB: small v2 batches, legacy entries, and batches larger than a 64 KiB chunk and a 128 KiB slot batch
    return R.gen_segment(1, 400000, big=200000)


def expect_failure(c, flags, bad, cs, call=None):
    """the call fails with TSGPU_E_RECORDS at the oracle's first invalid entry, naming its check (and CRCs)"""
    want = R.walk(bad)
    assert want is not None
    at, kind, stored, computed = want
    with pytest.raises(tsgpu.TsgpuError) as ei:
        (call or (lambda: c.transform(flags, bad, cs, *corpus.fixed_key_material((bad.size + cs - 1) // cs))))()
    msg = str(ei.value)
    assert ei.value.code == binding.E_RECORDS, msg
    assert re.search(r"segment position %d\b" % at, msg) and "check: %s" % kind in msg, (want, msg)
    if kind == "crc":
        assert "stored crc = %d, computed crc = %d" % (stored, computed) in msg, (want, msg)
    return at, kind


# ---------------------------------------------------------------------------------------------------- valid segments
FLAG_MIXES = [Z, Z | D, A, Z | A, Z | D | A, Z | C, Z | D | C | A, Z | V, Z | D | A | V]
FLAG_IDS = ["Z", "ZD", "A", "ZA", "ZDA", "ZC", "ZDCA", "ZV", "ZDAV"]


@pytest.mark.parametrize("flags", FLAG_MIXES, ids=FLAG_IDS)
@pytest.mark.parametrize("cs", [4096, CAP])
def test_valid_segment_transforms_to_the_flag_off_bytes(ctx, seg, flags, cs):
    key, aad, ivs = corpus.fixed_key_material((seg.size + cs - 1) // cs)
    plain, psizes = ctx.transform(flags, seg, cs, key, aad, ivs)
    plain = plain.copy()
    out, sizes = ctx.transform(flags | VR, seg, cs, key, aad, ivs)
    assert sizes == psizes and np.array_equal(out, plain)
    back, _ = ora.detransform_chunks(flags & (Z | A), out, sizes, seg.size, key, aad)
    assert np.array_equal(back, seg)


@pytest.mark.parametrize("kind", ["K", "R"])
@pytest.mark.parametrize("shape", ["small", "legacy", "large"])
def test_generated_shapes_pass(ctx, kind, shape):
    opts = {"small": dict(big=256), "legacy": dict(legacy=0.9, big=4096), "large": dict(small=60000, big=300000)}[shape]
    s = R.gen_segment(2, 300000, kind=kind, **opts)
    out, sizes = ctx.transform(Z | VR, s, 8192)
    plain, psizes = ctx.transform(Z, s, 8192)
    assert sizes == psizes and np.array_equal(out, plain)


def test_empty_segment_is_valid(ctx):
    out, sizes = ctx.transform(Z | VR, np.zeros(0, np.uint8), 4096)
    assert sizes == []


def test_one_byte_chunks(ctx):
    s = R.gen_segment(3, 300, big=100)
    out, sizes = ctx.transform(Z | VR, s, 1)
    assert len(sizes) == s.size
    bad = s.copy()
    bad[R.starts(s)[1] + 30] ^= 1
    expect_failure(ctx, Z | VR, bad, 1)


# ---------------------------------------------------------------------------------------------------- damage
def _damage(s, how, e):
    """`s` with entry `e` (index into its entries) damaged in one way"""
    st = R.starts(s)
    x = int(st[e])
    end = int(st[e + 1]) if e + 1 < len(st) else s.size
    m = int(s[x + 16])
    b = s.copy()
    size_at = slice(x + 8, x + 12)
    if how == "payload":
        b[(x + end) // 2 + 20] ^= 0x08
    elif how == "crc":
        b[x + (17 if m == 2 else 12) + 2] ^= 0x01
    elif how == "magic":
        b[x + 16] ^= 0x80
    elif how in ("shorter", "longer", "past_end"):
        size = int.from_bytes(bytes(b[size_at]), "big")
        size = {"shorter": size - 7, "longer": size + 5, "past_end": size + s.size}[how]
        b[size_at] = np.frombuffer(size.to_bytes(4, "big"), np.uint8)
    elif how == "too_small":
        b[size_at] = np.frombuffer((10).to_bytes(4, "big"), np.uint8)
    return b


HOWS = ["payload", "crc", "magic", "shorter", "longer", "past_end", "too_small"]


@pytest.mark.parametrize("how", HOWS)
@pytest.mark.parametrize("where", ["first", "last", "chunk", "slot_batch"])
def test_damage_is_found_at_the_oracles_position(ctx, seg, how, where):
    cs = 4096
    st = R.starts(seg)
    ends = np.append(st[1:], seg.size)
    if where == "first":
        e = 0
    elif where == "last":
        e = len(st) - 1
    else:                   # an entry that straddles a chunk boundary / a slot-batch boundary (2 chunks per batch)
        unit = cs if where == "chunk" else 2 * cs
        e = next(i for i in range(1, len(st)) if st[i] // unit != (ends[i] - 1) // unit and st[i] // (2 * cs) > 3)
    expect_failure(ctx, Z | VR, _damage(seg, how, e), cs)


@pytest.mark.parametrize("max_batch", [1, 2])
def test_entry_larger_than_a_slot_batch(max_batch):
    c = tsgpu.Context(max_chunk_bytes=8192, max_batch=max_batch, lib_path=SIMT_LIB)
    try:
        s = R.gen_segment(4, 120000, big=60000, small=30000)
        assert np.diff(np.append(R.starts(s), s.size)).max() > 2 * 8192
        c.transform(Z | VR, s, 8192)
        e = int(np.argmax(np.diff(np.append(R.starts(s), s.size))))
        for how in ("payload", "crc", "past_end"):
            expect_failure(c, Z | VR, _damage(s, how, e), 8192)
    finally:
        c.close()


def test_truncated_last_entry_and_trailing_garbage(ctx, seg):
    expect_failure(ctx, Z | VR, seg[:-10].copy(), 4096)                 # ends inside the last entry: length
    expect_failure(ctx, Z | VR, seg[:-(seg.size - int(R.starts(seg)[-1]) - 19)].copy(), 4096)   # ... inside its header
    garbage = np.concatenate([seg, np.frombuffer(b"not a record batch", np.uint8)])
    at, kind = expect_failure(ctx, Z | VR, garbage, 4096)
    assert at == seg.size
    tail = np.concatenate([seg, np.zeros(5, np.uint8)])                 # fewer than 17 bytes left
    assert expect_failure(ctx, Z | VR, tail, 4096) == (seg.size, "length")


def test_corpus_k_is_not_a_segment(ctx):
    k = corpus.gen_segment("K", 1, 200000, 4096)
    assert expect_failure(ctx, Z | VR, k, 4096)[0] == 0


# ---------------------------------------------------------------------------------------------------- calls in windows
def _windows(c, flags, s, cs, cuts):
    """s transformed in windows [cuts[i], cuts[i+1]) (multiples of cs but the last) with one cursor"""
    cur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    outs, sizes = [], []
    bounds = [0] + list(cuts) + [s.size]
    for i in range(len(bounds) - 1):
        o, z = c.transform_cursor(flags, s[bounds[i]:bounds[i + 1]], cs, cur, i == len(bounds) - 2)
        outs.append(o.copy()); sizes += z
    return np.concatenate(outs), sizes


def _cut_inside_a_header(s, cs):
    """a window end (multiple of cs) that falls inside some entry's first 21 bytes, and that entry"""
    st = R.starts(s)
    for i, x in enumerate(st):
        for k in range(1, 21):
            if (int(x) + k) % cs == 0:
                return int(x) + k, i
    raise AssertionError("no header crosses a chunk boundary")


def test_cursor_windows_equal_one_call(ctx):
    cs = 512
    s = R.gen_segment(5, 200000, big=20000)
    whole, wsizes = ctx.transform(Z | VR, s, cs)
    cut, e = _cut_inside_a_header(s, cs)
    cuts = sorted({cs * 32, cut, cut + cs * 3, cs * 300})
    out, sizes = _windows(ctx, Z | VR, s, cs, cuts)
    assert sizes == wsizes and np.array_equal(out, whole)
    # damage in the entry whose header the window end cuts, and in an entry that spans several windows
    for how in ("magic", "crc", "payload", "too_small"):
        bad = _damage(s, how, e)
        expect_failure(ctx, Z | VR, bad, cs, call=lambda: _windows(ctx, Z | VR, bad, cs, cuts))
    big = int(np.argmax(np.diff(np.append(R.starts(s), s.size))))
    x = int(R.starts(s)[big])
    cuts2 = [(x // cs + 1) * cs, (x // cs + 3) * cs]
    bad = _damage(s, "payload", big)
    expect_failure(ctx, Z | VR, bad, cs, call=lambda: _windows(ctx, Z | VR, bad, cs, cuts2))


def test_segment_ending_inside_an_entry_needs_the_last_window(ctx):
    s = R.gen_segment(6, 20000)
    cur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    cut = int(R.starts(s)[3]) + 40
    cut -= cut % 8
    ctx.transform_cursor(Z | VR, s[:cut], 8, cur, False)                # not the end: the open entry is carried
    assert cur.any()
    with pytest.raises(tsgpu.TsgpuError) as ei:                          # an empty last window: the segment ends there
        ctx.transform_cursor(Z | VR, s[:0], 8, cur.copy(), True)
    assert ei.value.code == binding.E_RECORDS and "check: length" in str(ei.value)
    ctx.transform_cursor(Z | VR, s[cut:], 8, cur, True)                  # the rest of the segment completes it


def test_transform_is_cursor_with_a_zero_cursor(ctx, seg):
    a, asz = ctx.transform(Z | A | VR, seg, 4096, *corpus.fixed_key_material(seg.size // 4096 + 1))
    a = a.copy()
    cur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    b, bsz = ctx.transform_cursor(Z | A | VR, seg, 4096, cur, True, *corpus.fixed_key_material(seg.size // 4096 + 1))
    assert asz == bsz and np.array_equal(a, b)
    bad = _damage(seg, "crc", 7)
    m1 = expect_failure(ctx, Z | VR, bad, 4096)
    m2 = expect_failure(ctx, Z | VR, bad, 4096, call=lambda: ctx.transform_cursor(Z | VR, bad, 4096, np.zeros(64, np.uint8), True))
    assert m1 == m2


# ---------------------------------------------------------------------------------------------------- interactions
def test_verify_and_validate_together(ctx, seg, monkeypatch):
    ctx.transform(Z | V | VR, seg, 4096)
    st = R.starts(seg)
    ends = np.append(st[1:], seg.size)
    e = next(i for i in range(len(st)) if st[i] // 8192 == (ends[i] - 1) // 8192 and st[i] >= 8192)   # inside one slot batch
    chunk = 2 * int(st[e] // 8192) + 1
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "%d:100" % chunk)             # a fault in that batch's output
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform(Z | V | VR, seg, 4096)                             # the input is sound
    assert ei.value.code == binding.E_VERIFY and "chunk %d " % chunk in str(ei.value)
    expect_failure(ctx, Z | V | VR, _damage(seg, "crc", e), 4096)        # both in one batch: the input's fault is named


def test_flag_is_refused_where_it_does_not_apply(ctx, seg):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform(VR, seg, 4096)
    assert ei.value.code == binding.E_ARG
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform_chunks(A | VR, seg[:1000], [400, 600], *corpus.fixed_key_material(2))
    assert ei.value.code == binding.E_ARG
    stride = ctx.slot_stride(Z, 4096)
    slots = np.zeros(2 * stride, np.uint8)
    sizes = np.zeros(2, np.uint32)
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform_device(Z | VR, seg.ctypes.data, 8192, 4096, None, b"", None, slots.ctypes.data, stride, sizes.ctypes.data)
    assert ei.value.code == binding.E_ARG
    out, tsz = ctx.transform(Z, seg[:8192], 4096)
    dst, osz, status = np.zeros(8192, np.uint8), np.zeros(2, np.uint32), np.zeros(2, np.uint32)
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.detransform_device(Z | VR, slots.ctypes.data, stride, sizes.ctypes.data, 2, 4096, None, b"", dst.ctypes.data,
                               osz.ctypes.data, status.ctypes.data)
    assert ei.value.code == binding.E_ARG
    back, _ = ctx.detransform(Z | VR, out, tsz, 8192)                    # detransform ignores the bit
    assert np.array_equal(back, seg[:8192])


def test_environment_makes_validation_the_default_of_cursor_calls():
    code = """
import sys, numpy as np, tsgpu
sys.path.insert(0, "tests")
import records_util as R
s = R.gen_segment(7, 50000)
c = tsgpu.Context(max_chunk_bytes=65536, max_batch=2, lib_path=%r)
bad = s.copy(); bad[R.starts(s)[2] + 30] ^= 1
c.transform(tsgpu.FLAG_ZSTD, bad, 4096)       # tsgpu_transform also carries windows of a segment: not validated
c.transform_cursor(0, bad[:100], 4096, np.zeros(64, np.uint8), True)   # no ZSTD / AES: a memcpy, nothing is validated
c.transform_cursor(tsgpu.FLAG_ZSTD, s, 4096, np.zeros(64, np.uint8), True)
try:
    c.transform_cursor(tsgpu.FLAG_ZSTD, bad, 4096, np.zeros(64, np.uint8), True)
except tsgpu.TsgpuError as e:
    assert e.code == -10, e
    print("env default ok")
""" % SIMT_LIB
    env = dict(os.environ, TSGPU_VALIDATE_RECORDS="1")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "env default ok" in r.stdout, r.stdout + r.stderr


def test_record_shapes_are_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    R._oracle()                                                          # built before libasan is preloaded
    env = dict(os.environ, LD_PRELOAD=runtime, ASAN_OPTIONS="detect_leaks=0")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_records.py"), "libtsgpu_simt_asan.so"],
                         env=env, capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "records sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
