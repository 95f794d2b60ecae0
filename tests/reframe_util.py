"""What TSGPU_FLAG_REFRAME must make of each source frame, computed on the CPU from the frames, libzstd and the library's own dense
frames.  Shared by tests/test_simt_reframe.py, tests/simt/asan_reframe.py and tests/test_gpu_reframe.py."""
import struct

import numpy as np

from oracle import oracle as ora

Z, A, D, CK, V, VR, RF = 1, 2, 4, 16, 8, 32, 64
SKIP_MAGIC = 0x184D2A53


def skippable(payload):
    return struct.pack("<II", SKIP_MAGIC, len(payload)) + payload


def split_tail(frame):
    """(the zstd frame with its checksum if any, the skippable frames after it), found by walking the block headers"""
    fhd = frame[4]
    single, dict_flag, fcs_flag = (fhd >> 5) & 1, fhd & 3, fhd >> 6
    pos = 5 + (0 if single else 1) + (0, 1, 2, 4)[dict_flag] + ((1 if single else 0), 2, 4, 8)[fcs_flag]
    while True:
        bh = frame[pos] | frame[pos + 1] << 8 | frame[pos + 2] << 16
        pos += 3 + (1 if (bh >> 1) & 3 == 1 else bh >> 3)
        if bh & 1:
            break
    if fhd & 4:
        pos += 4
    return frame[:pos], frame[pos:]


def sealed(frame, chunk):
    """`frame` with its Content_Checksum: FHD bit 2 and libzstd's checksum of `chunk` after the last block, skippable frames after"""
    body, tail = split_tail(frame)
    if frame[4] & 4:
        return frame
    ck = ora.zstd_compress_checksum(bytes(chunk), 1)[-4:]
    return body[:4] + bytes([body[4] | 4]) + body[5:] + ck + tail


def expected(tf, old_frames, chunks, dense_frames=None):
    """the frames a REFRAME rewrite with to_flags `tf` writes for `old_frames` (decrypted source frames) of `chunks`;
    dense_frames: the frames tsgpu_transform writes for the chunks with ZSTD|DENSE (|CHECKSUM as tf has it)"""
    out = []
    for i, (f, ch) in enumerate(zip(old_frames, chunks)):
        keep = sealed(f, ch) if tf & CK else f
        if tf & D and len(dense_frames[i]) < len(keep):
            keep = dense_frames[i]
        out.append(keep)
    return out


def with_skippable(obj, sizes, every=2):
    """a zstd-only object whose every `every`-th chunk carries a skippable frame after its frame"""
    out, new, pos = [], [], 0
    for i, t in enumerate(sizes):
        ch = bytes(obj[pos:pos + t])
        pos += t
        if i % every == 0:
            ch += skippable(bytes(range(i % 7, i % 7 + 37)))
        out.append(ch)
        new.append(len(ch))
    return np.frombuffer(b"".join(out), np.uint8).copy(), new


def chunks_of(seg, cs):
    return [bytes(seg[i:i + cs]) for i in range(0, seg.size, cs)]
