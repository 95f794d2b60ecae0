"""The device-resident calls (tsgpu_transform_device / tsgpu_detransform_device) on the SIMT emulator.  There "device"
memory is host memory and the stream is ignored, so numpy buffers stand in for HBM and stream 0 for a CUDA stream.  The
-m gpu tests in test_gpu_bench_shape.py run the same calls on an H100."""
import os
import subprocess

import numpy as np
import pytest

import tsgpu
from tsgpu import corpus
from oracle import oracle as ora

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIMT_LIB = os.path.join(ROOT, "tests", "simt", "libtsgpu_simt.so")
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE
CS = 1 << 16


@pytest.fixture(scope="module")
def simt_ctx():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4, lib_path=SIMT_LIB)
    yield ctx
    ctx.close()


def _transform_device(ctx, flags, src, key, aad, ivs):
    """Returns (slots, stride, transformed sizes) of one device call over src."""
    nch = (src.size + CS - 1) // CS
    stride = ctx.slot_stride(flags, CS)
    slots = np.zeros(nch * stride, np.uint8)
    sizes = np.zeros(nch, np.int32)
    ctx.transform_device(flags, src.ctypes.data, src.size, CS, key, aad, ivs, slots.ctypes.data, stride, sizes.ctypes.data, 0)
    return slots, stride, sizes


def _chunk(slots, stride, sizes, i):
    head = i * stride + tsgpu.binding.SLOT_HEAD
    return slots[head:head + int(sizes[i])]


@pytest.mark.parametrize("flags", [A, Z, Z | A, Z | A | D, Z | D], ids=["A", "Z", "ZA", "ZAD", "ZD"])
def test_simt_device_round_trip(simt_ctx, flags):
    nch = 3
    key, aad, ivs = corpus.fixed_key_material(nch)
    src = corpus.gen_segment("K", 3, CS * nch - 1000, CS)                 # ragged last chunk
    want_osz = [CS, CS, CS - 1000]
    slots, stride, sizes = _transform_device(simt_ctx, flags, src, key, aad, ivs)
    for i in range(nch):
        back, osz = ora.detransform_chunks(flags & (Z | A), _chunk(slots, stride, sizes, i), [int(sizes[i])], CS, key, aad)
        assert osz == [want_osz[i]] and np.array_equal(back, src[i * CS:i * CS + want_osz[i]]), i
    dst = np.zeros(nch * CS, np.uint8)
    osz = np.zeros(nch, np.int32)
    status = np.full(nch, 7, np.int32)
    simt_ctx.detransform_device(flags, slots.ctypes.data, stride, sizes.ctypes.data, nch, CS, key, aad, dst.ctypes.data,
                                osz.ctypes.data, status.ctypes.data, 0)
    assert status.tolist() == [0] * nch
    assert osz.tolist() == want_osz
    assert np.array_equal(dst[:src.size], src)


def test_simt_device_detransform_rejects_oversize_sizes(simt_ctx):
    # sizes in device memory are untrusted: the tampered chunk gets status 1 and nothing is written for it
    nch = 4
    key, aad, ivs = corpus.fixed_key_material(nch)
    src = corpus.gen_segment("R", 1, CS * nch, CS)
    slots, stride, sizes = _transform_device(simt_ctx, A, src, key, aad, ivs)
    sizes[2] = CS + 28 + 4096
    guard = 1 << 16
    dst = np.full(CS * nch + guard, 0x5A, np.uint8)
    osz = np.zeros(nch, np.int32)
    status = np.zeros(nch, np.int32)
    simt_ctx.detransform_device(A, slots.ctypes.data, stride, sizes.ctypes.data, nch, CS, key, aad, dst.ctypes.data,
                                osz.ctypes.data, status.ctypes.data, 0)
    assert status.tolist() == [0, 0, 1, 0]
    assert np.all(dst[2 * CS:3 * CS] == 0x5A) and np.all(dst[CS * nch:] == 0x5A)
    assert np.array_equal(dst[:2 * CS], src[:2 * CS]) and np.array_equal(dst[3 * CS:CS * nch], src[3 * CS:])


def test_simt_key_tables_follow_the_key_across_device_and_host_calls(simt_ctx):
    # device calls and host calls share slot 0's GCM key tables: a key change in either must rebuild them
    nch = 2
    _, aad, ivs = corpus.fixed_key_material(nch)
    rng = np.random.default_rng(17)
    k1, k2 = rng.bytes(32), rng.bytes(32)
    src = corpus.gen_segment("K", 5, CS * nch - 333, CS)
    for key, device in ((k1, True), (k2, False), (k1, True)):
        want, wsizes = ora.transform_segment(A, src, CS, key, aad, ivs)
        if device:
            slots, stride, sizes = _transform_device(simt_ctx, A, src, key, aad, ivs)
            assert sizes.tolist() == wsizes
            got = np.concatenate([_chunk(slots, stride, sizes, i) for i in range(nch)])
        else:
            got, gsizes = simt_ctx.transform(A, src, CS, key, aad, ivs)
            assert gsizes == wsizes
        assert np.array_equal(got, want)
