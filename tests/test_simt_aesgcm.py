"""Runs the REAL AES-GCM kernel sources under the test-only SIMT emulator (tests/simt/) through the C-ABI and
checks them bit-exact against the oracle.  This is a logic check on the GPU-less build box; the -m gpu tests
are the parity gate on an H100."""
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as ora
import tsgpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")


@pytest.fixture(scope="module")
def simt_ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    ctx = tsgpu.Context(max_chunk_bytes=1 << 20, max_batch=4, lib_path=SIMT_LIB)
    yield ctx
    ctx.close()


@pytest.mark.parametrize("n,chunk", [(1, 0), (15, 0), (16, 0), (17, 0), (100, 16), (4096, 1024), (5000, 1024),
                                     (70001, 16384), (300000, 0), (3 * 262144 + 5, 2 * 262144)])
def test_simt_encrypt_bit_exact_and_decrypt(simt_ctx, n, chunk):
    rng = np.random.default_rng(n)
    src = rng.integers(0, 256, n, dtype=np.uint8)
    key, aad = rng.bytes(32), rng.bytes(32)
    nch = (n + chunk - 1) // chunk if chunk else 1
    ivs = rng.bytes(12 * nch)
    want, wsizes = ora.transform_segment(ora.FLAG_AES, src, chunk, key, aad, ivs)
    got, gsizes = simt_ctx.transform(tsgpu.FLAG_AES, src, chunk, key, aad, ivs)
    assert gsizes == wsizes
    assert np.array_equal(got, want)
    back, osz = simt_ctx.detransform(tsgpu.FLAG_AES, got, gsizes, n, key, aad)
    assert np.array_equal(back, src)
    bad = got.copy()
    bad[len(bad) // 2] ^= 0x40
    with pytest.raises(tsgpu.TsgpuError) as e:
        simt_ctx.detransform(tsgpu.FLAG_AES, bad, gsizes, n, key, aad)
    assert e.value.code == tsgpu.binding.E_AUTH


def test_simt_aad_lengths(simt_ctx):
    rng = np.random.default_rng(5)
    src = rng.integers(0, 256, 1000, dtype=np.uint8)
    for alen in (0, 1, 16, 20, 33):
        key, aad, ivs = rng.bytes(32), rng.bytes(alen), rng.bytes(12)
        want, _ = ora.transform_segment(ora.FLAG_AES, src, 0, key, aad, ivs)
        got, _ = simt_ctx.transform(tsgpu.FLAG_AES, src, 0, key, aad, ivs)
        assert np.array_equal(got, want)


def test_simt_key_tables_follow_the_key_across_calls(simt_ctx):
    # a slot keeps its GHASH tables while calls use the same key (one data key per segment) and rebuilds them when it changes
    rng = np.random.default_rng(99)
    src = rng.integers(0, 256, 50000, dtype=np.uint8)
    k1, k2, aad = rng.bytes(32), rng.bytes(32), rng.bytes(32)
    ivs = rng.bytes(12 * 4)
    for key in (k1, k1, k2, k1, k2, k2):
        want, wsizes = ora.transform_segment(ora.FLAG_AES, src, 16384, key, aad, ivs)
        got, gsizes = simt_ctx.transform(tsgpu.FLAG_AES, src, 16384, key, aad, ivs)
        assert gsizes == wsizes and np.array_equal(got, want)
        back, _ = simt_ctx.detransform(tsgpu.FLAG_AES, want, wsizes, src.size, key, aad)
        assert np.array_equal(back, src)
    simt_ctx.profile_enable(True)
    simt_ctx.transform(tsgpu.FLAG_AES, src, 16384, k2, aad, ivs)      # same key as the previous call: no set-up launch
    assert "gcm_key_setup" not in simt_ctx.profile_report()
    simt_ctx.transform(tsgpu.FLAG_AES, src, 16384, k1, aad, ivs)
    assert "gcm_key_setup" in simt_ctx.profile_report()
    simt_ctx.profile_enable(False)
