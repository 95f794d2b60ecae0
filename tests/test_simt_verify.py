"""TSGPU_FLAG_VERIFY on the SIMT emulator: every host-buffer transform reads each batch back on the device before releasing
it.  Clean runs must pass and change no output byte; a byte flipped in a chunk's frame or ciphertext (the emulator build's
TSGPU_SIMT_FLIP hook, absent from libtsgpu.so) must fail the call with TSGPU_E_VERIFY, name the chunk and the check, and keep
every byte of the failing batch out of dst.  tests/test_gpu_verify.py runs the clean shapes on an H100."""
import os
import subprocess
import sys
import threading

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
CS = 1 << 16
BATCH = 2
N = 3 * CS - 777                 # three chunks, the last one ragged: two batches of at most BATCH chunks
SENTINEL = 0xEE


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=BATCH, lib_path=SIMT_LIB)
    yield c
    c.close()


def _segment(kind, n=N):
    src = corpus.gen_segment(kind, 7, n, CS)
    key, aad, ivs = corpus.fixed_key_material((n + CS - 1) // CS)
    return src, key, aad, ivs


def _oracle_reads(flags, out, sizes, src, key, aad):
    try:
        back, _ = ora.detransform_chunks(flags & (Z | A), out, sizes, src.size, key, aad)
    except ora.OracleError:
        return False
    return np.array_equal(back, src)


@pytest.mark.parametrize("kind", ["K", "R", "Z"])
@pytest.mark.parametrize("flags", [Z, Z | D, A, Z | A, Z | D | A], ids=["Z", "ZD", "A", "ZA", "ZDA"])
def test_verify_passes_and_changes_no_output(ctx, flags, kind):
    src, key, aad, ivs = _segment(kind)
    plain, psizes = ctx.transform(flags, src, CS, key, aad, ivs)
    out, sizes = ctx.transform(flags | V, src, CS, key, aad, ivs)
    assert len(sizes) == 3
    assert _oracle_reads(flags, out, sizes, src, key, aad)
    if flags & D or flags == A:          # dense frames and AES with fixed IVs are deterministic
        assert sizes == psizes and np.array_equal(out, plain)


@pytest.mark.parametrize("flags", [A, Z | A, Z | D | A], ids=["A", "ZA", "ZDA"])
def test_verify_ragged_index_blobs(ctx, flags):
    # the five index files of a segment, one chunk each, at unaligned offsets of src: three batches
    rng = np.random.default_rng(11)
    blobs = [rng.integers(0, 256, 10485, dtype=np.uint8), corpus.gen_chunk("K", 1, 0, 37),
             corpus.gen_chunk("K", 1, 1, 40001), np.zeros(126, np.uint8), corpus.gen_chunk("K", 1, 2, 1)]
    src = np.concatenate(blobs)
    lens = [b.size for b in blobs]
    key, aad, ivs = corpus.fixed_key_material(len(blobs))
    plain, psizes = ctx.transform_chunks(flags, src, lens, key, aad, ivs)
    out, sizes = ctx.transform_chunks(flags | V, src, lens, key, aad, ivs)
    pos = 0
    for blob, t in zip(blobs, sizes):
        back, _ = ora.detransform_chunks(flags & (Z | A), out[pos:pos + t], [t], blob.size, key, aad)
        assert np.array_equal(back, blob)
        pos += t
    if flags & D or flags == A:
        assert sizes == psizes and np.array_equal(out, plain)


def test_verify_two_concurrent_callers(ctx):
    errors = []

    def caller(kind, flags):
        try:
            src, key, aad, ivs = _segment(kind, 5 * CS - 4000)
            for _ in range(2):
                out, sizes = ctx.transform(flags | V, src, CS, key, aad, ivs)
                assert _oracle_reads(flags, out, sizes, src, key, aad), (kind, flags)
        except Exception as e:          # noqa: BLE001 — reported below
            errors.append(e)

    threads = [threading.Thread(target=caller, args=("K", Z | A)), threading.Thread(target=caller, args=("R", Z | D | A))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


# ---------------------------------------------------------------------------------------------------- injected faults
def _first_wrong_decode(frame, want):
    """(offset, first differing byte) of a one-bit flip of `frame` that libzstd still decodes, to the right length but
    wrong bytes"""
    for at in range(frame.size // 2, frame.size):
        bad = frame.copy()
        bad[at] ^= 1
        try:
            got = np.frombuffer(ora.zstd_decompress_chunk(bad), np.uint8)
        except ora.OracleError:
            continue
        if got.size == want.size and not np.array_equal(got, want):
            return at, int(np.flatnonzero(got != want)[0])
    raise AssertionError("no flip of the frame decodes to wrong bytes")


def _run_with_flip(ctx, monkeypatch, flags, src, key, aad, ivs, k, at, dst):
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "%d:%d" % (k, at))
    try:
        return ctx.transform(flags, src, CS, key, aad, ivs, dst=dst)
    finally:
        monkeypatch.delenv("TSGPU_SIMT_FLIP")


def _fault_case(ctx, case):
    """(flags, kind, chunk, offset, expected message part) of one injected fault"""
    if case == "frame_misread":
        src, *_ = _segment("R")
        out, sizes = ctx.transform(Z | D, src, CS)
        k = 2                                                       # the second batch: the first one has left already
        start = sum(sizes[:k])
        at, first = _first_wrong_decode(out[start:start + sizes[k]].copy(), src[k * CS:(k + 1) * CS])
        return Z | D, "R", k, at, "bytes differ from offset %d" % first
    if case == "frame_broken":
        return Z | D, "K", 1, 0, "frame check failed"               # the magic number
    if case == "ciphertext":
        return Z | D | A, "K", 0, binding.IV_SIZE + 100, "tag check failed"
    if case == "tag":
        return A, "R", 2, -1, "tag check failed"
    raise ValueError(case)


@pytest.mark.parametrize("case", ["frame_misread", "frame_broken", "ciphertext", "tag"])
def test_injected_fault_fails_verify_and_keeps_batch_out_of_dst(ctx, monkeypatch, case):
    flags, kind, k, at, what = _fault_case(ctx, case)
    src, key, aad, ivs = _segment(kind)
    good, sizes = ctx.transform(flags, src, CS, key, aad, ivs)      # deterministic flags: same sizes as the faulty runs
    cap = int(binding.load(SIMT_LIB).tsgpu_transform_bound(flags, src.size, CS)) + 64
    dst = np.full(cap, SENTINEL, np.uint8)
    with pytest.raises(tsgpu.TsgpuError) as ei:
        _run_with_flip(ctx, monkeypatch, flags | V, src, key, aad, ivs, k, at, dst)
    assert ei.value.code == binding.E_VERIFY
    msg = str(ei.value)
    assert ("chunk %d " % k) in msg and what in msg, msg
    batch_start = sum(sizes[:k // BATCH * BATCH])
    assert np.all(dst[batch_start:] == SENTINEL)                   # nothing of the failing batch (or after it)
    assert np.array_equal(dst[:batch_start], good[:batch_start])   # earlier batches did go out, unharmed
    # the same fault without the check: the call succeeds and the object does not read back
    out, bsizes = _run_with_flip(ctx, monkeypatch, flags, src, key, aad, ivs, k, at, None)
    assert bsizes == sizes
    assert not _oracle_reads(flags, out, bsizes, src, key, aad)


def test_environment_turns_verify_on(monkeypatch):
    monkeypatch.setenv("TSGPU_VERIFY", "1")
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=BATCH, lib_path=SIMT_LIB)
    monkeypatch.delenv("TSGPU_VERIFY")                               # read once, by tsgpu_create
    try:
        src, key, aad, ivs = _segment("K")
        out, sizes = c.transform(Z | A, src, CS, key, aad, ivs)
        assert _oracle_reads(Z | A, out, sizes, src, key, aad)
        with pytest.raises(tsgpu.TsgpuError) as ei:
            _run_with_flip(c, monkeypatch, A, src, key, aad, ivs, 1, -3, None)
        assert ei.value.code == binding.E_VERIFY and "chunk 1 " in str(ei.value)
    finally:
        c.close()


def test_device_transform_refuses_the_verify_bit(ctx):
    src, key, aad, ivs = _segment("K", CS)
    stride = ctx.slot_stride(Z | A, CS)
    slots = np.zeros(stride, np.uint8)
    sizes = np.zeros(1, np.int32)
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform_device(Z | A | V, src.ctypes.data, src.size, CS, key, aad, ivs, slots.ctypes.data, stride,
                             sizes.ctypes.data, 0)
    assert ei.value.code == binding.E_ARG and "TSGPU_FLAG_VERIFY" in str(ei.value)


def test_fault_hook_is_absent_from_the_product_library():
    lib = binding.DEFAULT_LIB
    if not os.path.exists(lib):
        pytest.skip("libtsgpu.so not built")
    with open(lib, "rb") as f:
        assert b"TSGPU_SIMT_FLIP" not in f.read()


def test_verify_shapes_are_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    env = dict(os.environ, LD_PRELOAD=runtime, ASAN_OPTIONS="detect_leaks=0")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_verify.py"), "libtsgpu_simt_asan.so"],
                         env=env, capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and "verify sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
