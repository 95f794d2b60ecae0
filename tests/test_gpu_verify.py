"""-m gpu tests of TSGPU_FLAG_VERIFY on an H100: 1 GiB segments in 4 MiB chunks read back without a false positive, the
outputs of the deterministic modes do not change, the read-back runs on the fast decode paths, and TSGPU_VERIFY=1 turns the
check on.  tests/test_simt_verify.py covers the failure side (injected faults) on the emulator."""
import numpy as np
import pytest

from oracle import oracle as ora
import tsgpu
from tsgpu import corpus

Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
DECODES = ("regions", "region_fallback_frames", "whole_frames", "serial_frames", "blocks")


def _segment(kind):
    # 16 distinct 4 MiB chunks repeated to 1 GiB (chunks are transformed independently; K text is slow to generate)
    return np.resize(corpus.gen_segment(kind, 21, 16 * CS, CS), SEG)


def _delta(ctx, before):
    after = ctx.decode_path_stats()
    return {k: after[k] - before[k] for k in DECODES}


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["K", "R", "Z"])
def test_gpu_verify_1gib_segments(ctx, kind):
    src = _segment(kind)
    nch = SEG // CS
    key, aad, ivs = corpus.fixed_key_material(nch)
    for flags in (Z | A, Z | D | A, A):
        s0 = ctx.decode_path_stats()
        out, sizes = ctx.transform(flags | V, src, CS, key, aad, ivs)            # no false positive on 256 chunks
        out = out.copy()
        dv = _delta(ctx, s0)
        # the read-back took the same decode paths as a fetch of the object does
        s1 = ctx.decode_path_stats()
        back, _ = ctx.detransform(flags & (Z | A), out, sizes, SEG, key, aad)
        assert np.array_equal(back, src), (kind, flags)
        assert dv == _delta(ctx, s1), (kind, flags, dv)
        if flags == A:
            assert all(v == 0 for v in dv.values())
        elif kind == "K":                                                         # this library's frames, fast paths only
            want = {"blocks": nch * (CS // 8192)} if not flags & D else {"regions": nch * (CS // 65536)}
            assert dv == dict({k: 0 for k in DECODES}, **want), (flags, dv)
        if flags & D or flags == A:                                              # deterministic: unchanged by the check
            plain, psizes = ctx.transform(flags, src, CS, key, aad, ivs)
            assert psizes == sizes and np.array_equal(plain, out), (kind, flags)
        if kind == "K" and flags == Z | A:                                       # the reference's reader agrees
            head = sum(sizes[:8])
            got, _ = ora.detransform_chunks(Z | A, out[:head], sizes[:8], 8 * CS, key, aad)
            assert np.array_equal(got, src[:8 * CS])


@pytest.mark.gpu
def test_gpu_verify_index_blobs_and_profile():
    # ragged index files up to 10 MiB, 8 per call, at unaligned offsets of src
    c = tsgpu.Context(max_chunk_bytes=10 * MIB, max_batch=8)
    try:
        c.profile_enable(True)
        rng = np.random.default_rng(5)
        lens = [10 * MIB, 10 * MIB - 1, 3 * MIB + 7, 65536 + 3, 4099, 37, 1, 1234567]
        blobs = [rng.integers(0, 256, n, dtype=np.uint8) if i % 2 else np.resize(corpus.gen_chunk("K", 4, i, 65536), n)
                 for i, n in enumerate(lens)]
        src = np.concatenate(blobs)
        key, aad, ivs = corpus.fixed_key_material(len(lens))
        for flags in (A, Z | A, Z | D | A):
            out, sizes = c.transform_chunks(flags | V, src, lens, key, aad, ivs)
            out = out.copy()
            pos = 0
            for blob, t in zip(blobs, sizes):
                back, _ = ora.detransform_chunks(flags & (Z | A), out[pos:pos + t], [t], blob.size, key, aad)
                assert np.array_equal(back, blob), flags
                pos += t
            if flags != Z | A:
                plain, psizes = c.transform_chunks(flags, src, lens, key, aad, ivs)
                assert psizes == sizes and np.array_equal(plain, out), flags
        assert "verify_compare" in c.profile_report()
    finally:
        c.close()


@pytest.mark.gpu
def test_gpu_environment_turns_verify_on(monkeypatch):
    src = corpus.gen_segment("K", 2, 3 * MIB, MIB)
    key, aad, ivs = corpus.fixed_key_material(3)
    monkeypatch.setenv("TSGPU_VERIFY", "1")
    c = tsgpu.Context(max_chunk_bytes=MIB, max_batch=4)
    monkeypatch.delenv("TSGPU_VERIFY")
    try:
        c.profile_enable(True)
        out, sizes = c.transform(Z | A, src, MIB, key, aad, ivs)
        back, _ = ora.detransform_chunks(Z | A, out, sizes, src.size, key, aad)
        assert np.array_equal(back, src)
        assert c.decode_path_stats()["blocks"] == 3 * (MIB // 8192)             # read back without a detransform call
        assert c.profile_report()["verify_compare"]["launches"] == 1
    finally:
        c.close()
