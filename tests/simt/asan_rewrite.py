"""Run by tests/test_simt_rewrite.py in a subprocess (argv[1] = the library to load, the ASan or the UBSan build):
tsgpu_rewrite_object over the source x target matrix, on objects from 1 byte to several batches in chunks from 1 byte to 4 KiB,
one and two chunks per slot batch, in one call and in windows, so the source half (frames loaded into the frame slots, the
in-slot object checksum, the decode to the chunk index's offsets) and the target half (kept frames encrypted or packed,
chunks compressed) are checked for overruns; damaged sources must fail, never overrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import rewrite_util as W  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, D, CK, V, VR = (tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_VERIFY,
                      tsgpu.FLAG_VALIDATE_RECORDS)

for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 40), (257, 3000), (4096, 4096 * 3 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        nch = (n + cs - 1) // cs
        key, aad, ivs = corpus.fixed_key_material(nch)
        nk, na, nivs = W.new_key_material(nch)
        for ff in (0, A, Z, Z | A):
            obj, sizes = c.transform(ff, src, cs, key, aad, ivs)
            obj = obj.copy()
            for tf in (A, Z | V, Z | A | V, Z | D | A):
                if ff & Z and tf & D:
                    continue
                for win in ((None, 3) if tf & A else (None,)):
                    new, nsz, parts, crc3 = W.rewrite_windows(c, ff, obj, sizes, cs, n, tf, 1000, win, key, aad, nk, na, nivs)
                    assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(src)), (cs, ff, tf, win)
            if ff:
                bad = obj.copy()
                bad[obj.size // 2] ^= 0x40
                try:
                    W.rewrite_windows(c, ff, bad, sizes, cs, n, Z | A, 1000, 2, key, aad, nk, na, nivs)
                    assert not (ff & A), "a flipped ciphertext byte passed"
                except tsgpu.TsgpuError:
                    pass
    seg = R.gen_segment(3, 30000, big=9000)
    key, aad, ivs = corpus.fixed_key_material(64)
    nk, na, nivs = W.new_key_material(64)
    for ff in (0, Z | A):
        obj, sizes = c.transform(ff, seg, 1024, key, aad, ivs)
        obj = obj.copy()
        for win in (None, 5):
            new, _, _, crc3 = W.rewrite_windows(c, ff | VR, obj, sizes, 1024, seg.size, Z | A, 4096, win, key, aad, nk, na, nivs)
            assert crc3 == (U.crc32c(obj), U.crc32c(new), U.crc32c(seg))
    c.close()
print("rewrite sweep ok")
