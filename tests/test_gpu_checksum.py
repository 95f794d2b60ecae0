"""-m gpu tests of TSGPU_FLAG_ZSTD_CHECKSUM on an H100: 1 GiB K, R and Z segments in 4 MiB chunks, Z and Z|A, speed and dense
mode, through the device-resident transform.  The hashing CTAs run inside the compressor's launch (no extra launch); every
sampled frame carries libzstd's checksum and reads back through libzstd; the whole segment round-trips on the device; dense
frames are the flag-off frames plus the 4 bytes; a 16 MiB window of checksummed frames fetches on the usual decode paths; a
damaged byte is refused.  tests/test_simt_checksum.py covers the small shapes on the emulator."""
import numpy as np
import pytest
import torch

from oracle import oracle as ora
import tsgpu
from tsgpu import binding, corpus

Z, A, D, C = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM
MIB = 1 << 20
CS = 4 * MIB
SEG = 1024 * MIB
NCH = SEG // CS
WIN = 4                                                      # chunks of a 16 MiB fetch window
SAMPLE = (0, 1, 77, NCH - 1)
DECODES = ("regions", "region_fallback_frames", "whole_frames", "serial_frames", "blocks")


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=NCH)
    yield c
    c.close()


@pytest.fixture(scope="module", params=["K", "R", "Z"])
def segment(request):
    # 16 distinct 4 MiB chunks repeated to 1 GiB (chunks are transformed independently; K text is slow to generate)
    src = np.resize(corpus.gen_segment(request.param, 31, 16 * CS, CS), SEG)
    return request.param, src, torch.from_numpy(src).cuda()


def _device_transform(ctx, flags, d_src, key, aad, ivs):
    stride = ctx.slot_stride(flags, CS)
    slots = torch.zeros(NCH * stride, dtype=torch.uint8, device="cuda")
    sizes = torch.zeros(NCH, dtype=torch.int32, device="cuda")
    before = ctx.launch_count()
    ctx.transform_device(flags, d_src.data_ptr(), SEG, CS, key, aad, ivs, slots.data_ptr(), stride, sizes.data_ptr())
    torch.cuda.synchronize()
    return slots, stride, [int(x) for x in sizes.cpu()], ctx.launch_count() - before


def _chunk(slots, stride, sizes, i):
    at = i * stride + binding.SLOT_HEAD
    return slots[at:at + sizes[i]].cpu().numpy()


def _frame(flags, chunk, key, aad):
    return np.frombuffer(ora.aesgcm_decrypt_chunk(key, aad, chunk), np.uint8).copy() if flags & A else chunk.copy()


def _delta(ctx, before):
    after = ctx.decode_path_stats()
    return {k: after[k] - before[k] for k in DECODES}


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["speed", "dense"])
@pytest.mark.parametrize("aes", [False, True], ids=["Z", "ZA"])
def test_gpu_checksum_1gib(ctx, segment, mode, aes):
    kind, src, d_src = segment
    flags = Z | (D if mode == "dense" else 0) | (A if aes else 0)
    key, aad, ivs = corpus.fixed_key_material(NCH)
    _device_transform(ctx, flags, d_src, key, aad, ivs)                         # (a new key adds its set-up launch once)
    slots0, stride, sizes0, launches0 = _device_transform(ctx, flags, d_src, key, aad, ivs)
    slots, stride1, sizes, launches = _device_transform(ctx, flags | C, d_src, key, aad, ivs)
    assert stride1 == stride and launches == launches0                       # the hash rides in the compressor's launch
    assert all(t <= stride - binding.SLOT_HEAD for t in sizes)
    if mode == "dense":
        assert sizes == [t + 4 for t in sizes0]
    # sampled chunks: the flag-off frame plus libzstd's checksum (dense), libzstd reads them and verifies the checksum
    for i in SAMPLE:
        want = src[i * CS:(i + 1) * CS]
        f = _frame(flags, _chunk(slots, stride, sizes, i), key, aad)
        assert f[4] & 0x04 and bytes(f[-4:]) == bytes(ora.zstd_compress_checksum(want)[-4:]), (kind, i)
        assert np.array_equal(np.frombuffer(ora.zstd_decompress_chunk(f), np.uint8), want), (kind, i)
        if mode == "dense":
            f0 = _frame(flags, _chunk(slots0, stride, sizes0, i), key, aad)
            f0[4] |= 0x04
            assert np.array_equal(f[:-4], f0), (kind, i)
    if mode == "dense" and not aes:                                          # every frame, on the device
        for i in range(NCH):
            a = slots[i * stride + binding.SLOT_HEAD:i * stride + binding.SLOT_HEAD + sizes[i] - 4]
            b = slots0[i * stride + binding.SLOT_HEAD:i * stride + binding.SLOT_HEAD + sizes0[i]].clone()
            b[4] |= 0x04
            assert torch.equal(a, b), (kind, i)
    del slots0
    # the whole segment round-trips on the device (every checksum verified by the decoder)
    d_sizes = torch.tensor(sizes, dtype=torch.int32, device="cuda")
    dst = torch.zeros(SEG, dtype=torch.uint8, device="cuda")
    osz = torch.zeros(NCH, dtype=torch.int32, device="cuda")
    status = torch.zeros(NCH, dtype=torch.int32, device="cuda")
    ctx.detransform_device(flags | C, slots.data_ptr(), stride, d_sizes.data_ptr(), NCH, CS, key, aad, dst.data_ptr(),
                           osz.data_ptr(), status.data_ptr())
    torch.cuda.synchronize()
    assert int(status.abs().sum()) == 0 and torch.equal(dst, d_src), kind
    del dst
    # a 16 MiB fetch window of checksummed frames (host-buffer call): right bytes, the decode paths of flag-off frames
    k0 = 100
    win = np.concatenate([_chunk(slots, stride, sizes, i) for i in range(k0, k0 + WIN)])
    s0 = ctx.decode_path_stats()
    back, _ = ctx.detransform(flags & (Z | A), win, sizes[k0:k0 + WIN], WIN * CS, key, aad)
    dv = _delta(ctx, s0)
    assert np.array_equal(back, src[k0 * CS:(k0 + WIN) * CS])
    if kind == "K":
        want = {"blocks": WIN * (CS // 8192)} if mode == "speed" else {"regions": WIN * (CS // 65536)}
        assert dv == dict({k: 0 for k in DECODES}, **want), dv
    # a damaged byte in the middle of the window's first frame (with AES the tag would refuse it first)
    if not aes:
        bad = win.copy()
        bad[sizes[k0] // 2] ^= 0x04
        with pytest.raises(tsgpu.TsgpuError) as ei:
            ctx.detransform(Z, bad, sizes[k0:k0 + WIN], WIN * CS)
        assert ei.value.code == binding.E_CORRUPT, kind
