"""TSGPU_FLAG_ZSTD_CHECKSUM on the SIMT emulator: every frame written with the flag is the frame written without it, with
Frame_Header_Descriptor bit 2 set and the low 32 bits of XXH64(chunk) appended; libzstd (an independent XXH64) agrees on the
4 bytes and verifies them, and so does tsgpu_detransform.  A damaged byte inside a Raw block decodes to wrong bytes without
an error when the frame has no checksum, and fails every reader when it has one.  tests/test_gpu_checksum.py runs 1 GiB
segments on an H100."""
import os
import subprocess
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D, V, C = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY, tsgpu.FLAG_ZSTD_CHECKSUM
MIB = 1 << 20
CAP = MIB
FLAGS = [Z, Z | D, Z | A, Z | D | A]
FLAG_IDS = ["Z", "ZD", "ZA", "ZDA"]
CHUNK_SIZES = [1, 31, 32, 33, 8191, 8192, 65537, MIB]


@pytest.fixture(scope="module")
def ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so", "oracle"])
    c = tsgpu.Context(max_chunk_bytes=CAP, max_batch=4, lib_path=SIMT_LIB)
    yield c
    c.close()


def _seg_len(cs):
    return 5 * cs if cs < 64 else cs + cs // 2 + 3           # several chunks, the last one ragged (but for tiny chunks)


def _frames(flags, out, sizes, key, aad):
    """the zstd frames of a transformed object, decrypted when AES is on"""
    frames, pos = [], 0
    for t in sizes:
        ch = out[pos:pos + t]
        frames.append(np.frombuffer(ora.aesgcm_decrypt_chunk(key, aad, ch), np.uint8).copy() if flags & A else ch.copy())
        pos += t
    return frames


def check_checksummed(c, flags, src, cs):
    """transform `src` with and without the flag and hold every frame to the contract; returns the checksummed output"""
    n = src.size
    nch = (n + cs - 1) // cs
    key, aad, ivs = corpus.fixed_key_material(nch)
    plain, psizes = c.transform(flags, src, cs, key, aad, ivs)
    out, sizes = c.transform(flags | C, src, cs, key, aad, ivs)
    out = out.copy()
    assert len(sizes) == nch and [t - 4 for t in sizes] == psizes
    assert sum(sizes) <= int(binding.load(SIMT_LIB).tsgpu_transform_bound(flags | C, n, cs))
    for i, (f0, f1) in enumerate(zip(_frames(flags, plain, psizes, key, aad), _frames(flags, out, sizes, key, aad))):
        chunk = src[i * cs:(i + 1) * cs]
        assert f0[4] & 0x04 == 0 and f1[4] == f0[4] | 0x04
        f0[4] |= 0x04
        assert np.array_equal(f1[:-4], f0), (i, "the frame is the flag-off frame plus the checksum")
        assert bytes(f1[-4:]) == bytes(ora.zstd_compress_checksum(chunk)[-4:]), i       # libzstd's XXH64
        assert np.array_equal(np.frombuffer(ora.zstd_decompress_chunk(f1), np.uint8), chunk), i
    back, _ = c.detransform(flags & (Z | A), out, sizes, n, key, aad)
    assert np.array_equal(back, src)
    return out, sizes


@pytest.mark.parametrize("cs", CHUNK_SIZES)
@pytest.mark.parametrize("kind", ["K", "R", "Z"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_checksummed_frames_are_the_plain_frames_plus_the_checksum(ctx, flags, kind, cs):
    check_checksummed(ctx, flags, corpus.gen_segment(kind, 5, _seg_len(cs), cs), cs)


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_checksummed_ragged_chunks(ctx, flags):
    rng = np.random.default_rng(3)
    blobs = [rng.integers(0, 256, 10485, dtype=np.uint8), corpus.gen_chunk("K", 1, 0, 37), corpus.gen_chunk("K", 1, 1, 40001),
             np.zeros(126, np.uint8), corpus.gen_chunk("K", 1, 2, 1), corpus.gen_chunk("K", 1, 3, 65537)]
    src = np.concatenate(blobs)
    lens = [b.size for b in blobs]
    key, aad, ivs = corpus.fixed_key_material(len(blobs))
    plain, psizes = ctx.transform_chunks(flags, src, lens, key, aad, ivs)
    out, sizes = ctx.transform_chunks(flags | C, src, lens, key, aad, ivs)
    assert [t - 4 for t in sizes] == psizes
    for blob, f0, f1 in zip(blobs, _frames(flags, plain, psizes, key, aad), _frames(flags, out, sizes, key, aad)):
        f0[4] |= 0x04
        assert np.array_equal(f1[:-4], f0)
        assert bytes(f1[-4:]) == bytes(ora.zstd_compress_checksum(blob)[-4:])
        assert np.array_equal(np.frombuffer(ora.zstd_decompress_chunk(f1), np.uint8), blob)
    back, _ = ctx.detransform(flags & (Z | A), out, sizes, src.size, key, aad)
    assert np.array_equal(back, src)


# ---------------------------------------------------------------------------------------------------- the gap it closes
def _raw_block_flip(frame):
    """offset of a byte inside the first block of `frame`, which must be a Raw block"""
    fhd = frame[4]
    hs = 4 + 1 + (0 if fhd & 0x20 else 1) + {0: 1 if fhd & 0x20 else 0, 1: 2, 2: 4, 3: 8}[fhd >> 6]
    bh = int(frame[hs]) | int(frame[hs + 1]) << 8 | int(frame[hs + 2]) << 16
    assert (bh >> 1) & 3 == 0 and (bh >> 3) > 200, "corpus R compresses to Raw blocks"
    return hs + 3 + 100


@pytest.mark.parametrize("checksum", [False, True], ids=["plain", "checksum"])
def test_damaged_raw_block_byte(ctx, checksum):
    cs = 65536
    src = corpus.gen_segment("R", 9, 2 * cs, cs)
    out, sizes = ctx.transform(Z | (C if checksum else 0), src, cs)
    bad = out.copy()
    at = _raw_block_flip(bad[:sizes[0]])
    bad[at] ^= 0x10
    if not checksum:        # a different byte and no error, in libzstd and here alike
        got = np.frombuffer(ora.zstd_decompress_chunk(bad[:sizes[0]]), np.uint8)
        assert got.size == cs and not np.array_equal(got, src[:cs])
        back, _ = ctx.detransform(Z, bad, sizes, src.size)
        assert back.size == src.size and not np.array_equal(back, src)
    else:                   # every reader refuses the frame
        with pytest.raises(ora.OracleError):
            ora.zstd_decompress_chunk(bad[:sizes[0]])
        with pytest.raises(tsgpu.TsgpuError) as ei:
            ctx.detransform(Z, bad, sizes, src.size)
        assert ei.value.code == binding.E_CORRUPT and "chunk 0" in str(ei.value)


# ---------------------------------------------------------------------------------------------------- interactions
def test_environment_makes_checksum_the_default():
    # read once by tsgpu_create: run in a fresh process so that no other context of this one sees the variable
    code = """
import numpy as np, tsgpu
from tsgpu import corpus
from oracle import oracle as ora
src = corpus.gen_segment("K", 2, 100000, 65536)
c = tsgpu.Context(max_chunk_bytes=65536, max_batch=2, lib_path=%r)
for flags in (tsgpu.FLAG_ZSTD, tsgpu.FLAG_ZSTD | tsgpu.FLAG_ZSTD_DENSE):
    out, sizes = c.transform(flags, src, 65536)
    f = out[:sizes[0]]
    assert f[4] & 4 and bytes(f[-4:]) == bytes(ora.zstd_compress_checksum(src[:65536])[-4:])
c.close()
print("env default ok")
""" % SIMT_LIB
    env = dict(os.environ, TSGPU_ZSTD_CHECKSUM="1")
    r = subprocess.run([sys.executable, "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "env default ok" in r.stdout, r.stdout + r.stderr


@pytest.mark.parametrize("flags", [Z, Z | D | A], ids=["Z", "ZDA"])
def test_detransform_ignores_the_bit(ctx, flags):
    src = corpus.gen_segment("K", 4, 150000, 65536)
    key, aad, ivs = corpus.fixed_key_material(3)
    for wf in (flags, flags | C):
        out, sizes = ctx.transform(wf, src, 65536, key, aad, ivs)
        for rf in (flags & (Z | A), flags | C):
            back, _ = ctx.detransform(rf, out, sizes, src.size, key, aad)
            assert np.array_equal(back, src)


@pytest.mark.parametrize("flags", [Z, Z | D, Z | A], ids=["Z", "ZD", "ZA"])
def test_device_transform_with_the_bit(ctx, flags):
    cs = 65536
    src = corpus.gen_segment("K", 6, 3 * cs - 5, cs)
    nch = 3
    key, aad, ivs = corpus.fixed_key_material(nch)
    host, hsizes = ctx.transform(flags | C, src, cs, key, aad, ivs)
    stride = ctx.slot_stride(flags | C, cs)
    assert stride == ctx.slot_stride(flags, cs)
    slots = np.zeros(nch * stride, np.uint8)
    sizes = np.zeros(nch, np.uint32)
    ctx.transform_device(flags | C, src.ctypes.data, src.size, cs, key, aad, ivs, slots.ctypes.data, stride, sizes.ctypes.data, 0)
    assert [int(x) for x in sizes] == hsizes
    dev = np.concatenate([slots[i * stride + binding.SLOT_HEAD:i * stride + binding.SLOT_HEAD + int(sizes[i])] for i in range(nch)])
    if flags & D or not flags & A:       # (speed mode is deterministic on the emulator, AES with fixed IVs too)
        assert np.array_equal(dev, host)
    dst = np.zeros(src.size, np.uint8)
    osz = np.zeros(nch, np.uint32)
    status = np.zeros(nch, np.uint32)
    ctx.detransform_device(flags | C, slots.ctypes.data, stride, sizes.ctypes.data, nch, cs, key, aad, dst.ctypes.data,
                           osz.ctypes.data, status.ctypes.data, 0)
    assert not status.any() and np.array_equal(dst, src)


def test_checksum_with_verify_and_an_injected_fault(ctx, monkeypatch):
    cs = 65536
    src = corpus.gen_segment("R", 7, 3 * cs - 777, cs)
    for flags in (Z, Z | D, Z | D | A):
        key, aad, ivs = corpus.fixed_key_material(3)
        out, sizes = ctx.transform(flags | C | V, src, cs, key, aad, ivs)
        back, _ = ora.detransform_chunks(flags & (Z | A), out, sizes, src.size, key, aad)
        assert np.array_equal(back, src)
    # a flipped byte inside chunk 1's first Raw block: without the checksum libzstd would decode it to wrong bytes
    out, sizes = ctx.transform(Z | C, src, cs)
    at = _raw_block_flip(out[sizes[0]:sizes[0] + sizes[1]])
    monkeypatch.setenv("TSGPU_SIMT_FLIP", "1:%d" % at)
    with pytest.raises(tsgpu.TsgpuError) as ei:
        ctx.transform(Z | C | V, src, cs)
    assert ei.value.code == binding.E_VERIFY and "chunk 1 " in str(ei.value)


@pytest.mark.parametrize("cs", [1, 33, 8192, 65537, MIB])
def test_transform_bound_holds_with_the_bit(ctx, cs):
    n = _seg_len(cs)
    src = corpus.gen_segment("R", 8, n, cs)
    lib = binding.load(SIMT_LIB)
    for flags in (Z, Z | D, Z | A):
        _, sizes = ctx.transform(flags | C, src, cs, *corpus.fixed_key_material((n + cs - 1) // cs))
        assert sum(sizes) <= int(lib.tsgpu_transform_bound(flags | C, n, cs)) == int(lib.tsgpu_transform_bound(flags, n, cs))
        assert max(sizes) + binding.SLOT_HEAD <= ctx.slot_stride(flags | C, cs)


def test_checksum_shapes_are_clean_under_asan():
    runtime = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("libasan not available")
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt_asan.so"])
    env = dict(os.environ, LD_PRELOAD=runtime, ASAN_OPTIONS="detect_leaks=0")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_checksum.py"), "libtsgpu_simt_asan.so"],
                         env=env, capture_output=True, text=True, timeout=3000)
    assert out.returncode == 0 and "checksum sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
