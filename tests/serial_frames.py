"""Frames that the zstd decoder hands to its serial kernel (`zstd_dec_frames_kernel`, one warp walking a frame's blocks in order),
shared by the emulator, sanitizer and GPU tests of that kernel."""
import numpy as np


def serial_routed(frame, blocks=200):
    """The same zstd frame with `blocks` empty Raw blocks (header bytes 00 00 00) right after its frame header: libzstd decodes it
    to the same bytes, and the decoder's index walk gives up once a frame has more than ceil(FCS / 8 KiB) + 1 blocks, which sends
    the frame to the serial kernel.  200 blocks are enough for frames up to ~1.6 MB."""
    f = np.frombuffer(bytes(frame), dtype=np.uint8)
    fhd = int(f[4])
    single, fcs_flag = (fhd >> 5) & 1, fhd >> 6
    hs = 5 + (1 - single) + (0, 1, 2, 4)[fhd & 3] + ((1 if single else 0), 2, 4, 8)[fcs_flag]
    return np.concatenate([f[:hs], np.zeros(3 * blocks, dtype=np.uint8), f[hs:]])


def serial_kernel_frames(ctx):
    """(name, source, frame) for every frame shape the serial kernel must decode, each already passed through serial_routed:
    libzstd levels 1 / 3 / 19 of four sources, this library's speed- and dense-mode frames, a frame with a Content_Checksum."""
    import tsgpu
    from tsgpu import corpus
    from oracle import oracle as ora
    srcs = {kind: corpus.gen_chunk(kind, 3, 0, n) for kind, n in (("K", 300000), ("R", 200000), ("Z", 500000))}
    rng = np.random.default_rng(5)
    mixed = rng.integers(0, 256, 300000, dtype=np.uint8)
    mixed[:150000] = corpus.gen_chunk("K", 5, 0, 150000)
    mixed[200000:201500] = 7
    srcs["M"] = mixed
    out = []
    for kind, src in srcs.items():
        for level in (1, 3, 19):
            out.append(("%s level %d" % (kind, level), src, ora.zstd_compress_level(src, level)))
    for name, flags in (("speed", tsgpu.FLAG_ZSTD), ("dense", tsgpu.FLAG_ZSTD | tsgpu.FLAG_ZSTD_DENSE)):
        f, sizes = ctx.transform(flags, srcs["K"], 0)
        out.append((name, srcs["K"], np.array(f[:sizes[0]], copy=True)))
    out.append(("checksum", srcs["K"], ora.zstd_compress_checksum(srcs["K"], 3)))
    return [(name, src, serial_routed(f)) for name, src, f in out]
