"""Run by tests/test_simt_check.py in a subprocess (argv[1] = the library to load, the ASan build): tsgpu_check_object over
objects from 1 byte to several batches in chunks from 1 byte to 4 KiB, one and two chunks per slot batch, every flag set, with
record validation, in one call and in windows, so the in-slot reads of the object checksum (pieces at every alignment, across
chunk ends, the word after a piece) and the record and segment-checksum kernels over the decoded bytes are checked for overruns;
a damaged chunk must fail, never overrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import check_util as K  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, D, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VALIDATE_RECORDS

for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 40), (21, 700), (257, 3000), (4096, 4096 * 5 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        key, aad, ivs = corpus.fixed_key_material((n + cs - 1) // cs)
        for flags in (0, A, Z, Z | D | A):
            obj, sizes = c.transform(flags, src, cs, key, aad, ivs)
            obj = obj.copy()
            want = (U.crc32c(obj), U.crc32c(src))
            for win in (None, 1, 3):
                assert K.check_windows(c, flags, obj, sizes, cs, n, win, key, aad) == want, (cs, flags, win)
            if flags:
                bad = obj.copy()
                bad[obj.size // 2] ^= 0x40
                try:
                    K.check_windows(c, flags, bad, sizes, cs, n, 2, key, aad)
                    assert not (flags & A), "a flipped ciphertext byte passed"
                except tsgpu.TsgpuError:
                    pass
    seg = R.gen_segment(3, 30000, big=9000)
    key, aad, ivs = corpus.fixed_key_material(64)
    for flags in (0, Z, Z | A):
        obj, sizes = c.transform(flags, seg, 1024, key, aad, ivs)
        obj = obj.copy()
        for win in (None, 1, 5):
            assert K.check_windows(c, flags | VR, obj, sizes, 1024, seg.size, win, key, aad) == (U.crc32c(obj), U.crc32c(seg))
    c.close()
print("check sweep ok")
