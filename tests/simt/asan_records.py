"""Run by tests/test_simt_records.py in a subprocess with libasan preloaded (argv[1] = the library to load): valid segments and
damaged ones in chunks from 1 byte to 64 KiB, one and two chunks per slot batch, and windows of a cursor, so the record kernels'
tail reads (headers at the batch end, partial pieces and tiles) and the carry's header bytes are checked for overruns."""
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
import records_util as R  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_VALIDATE_RECORDS
s = R.gen_segment(8, 90000, big=40000)
st = R.starts(s)
tiny = R.gen_segment(9, 1500, big=300)
mid = R.gen_segment(10, 12000, big=3000)
for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs in (1, 21, 257, 4096, 1 << 16):
        src = s if cs >= 4096 else tiny if cs == 1 else mid
        c.transform(Z | VR, src, cs)
        at = int(R.starts(src)[2])
        bad = src.copy()
        bad[at + 40] ^= 1
        try:
            c.transform(Z | VR, bad, cs)
            raise AssertionError("damage not found")
        except tsgpu.TsgpuError as e:
            assert e.code == -10 and re.search(r"segment position %d\b" % at, str(e)), e
    cur = np.zeros(64, np.uint8)
    cuts = [0, 4096, int(st[5]) + 7 - (int(st[5]) + 7) % 256, 40960, s.size]
    for i in range(len(cuts) - 1):
        c.transform_cursor(Z | VR, s[cuts[i]:cuts[i + 1]], 256, cur, i == len(cuts) - 2)
    c.close()
print("records sweep ok")
