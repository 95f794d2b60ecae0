"""-m gpu test of the zstd decoder's serial kernel (`zstd_dec_frames_kernel`): frames with more blocks than the index walks."""
import numpy as np
import pytest

import tsgpu
from serial_frames import serial_kernel_frames

Z = tsgpu.FLAG_ZSTD


@pytest.mark.gpu
def test_gpu_serial_kernel_frames():
    # libzstd, own and checksummed frames, one warp per frame; only the serial counter moves
    ctx = tsgpu.Context(max_chunk_bytes=4 << 20, max_batch=2)
    try:
        for name, src, f in serial_kernel_frames(ctx):
            st0 = ctx.decode_path_stats()
            back, osz = ctx.detransform(Z, f, [f.size], src.size)
            assert osz == [src.size] and np.array_equal(back, src), name
            assert ctx.decode_path_stats() == dict(st0, serial_frames=st0["serial_frames"] + 1), name
    finally:
        ctx.close()
