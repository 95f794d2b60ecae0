"""Run by tests/test_simt_part_crc.py in a subprocess (argv[1] = the library to load: the ASan or UBSan build, or the plain one
with TSGPU_SIMT_POISON=1 or a TSGPU_SIMT_ORDER): objects from 1 byte to several batches in chunks from 1 byte to 4 KiB, one and
two chunks per slot batch, part sizes from 1 byte to more than the object, and windows with a parts cursor, so the part-checksum
kernels' tail reads (partial pieces and tiles, boundaries at the batch end) are checked for overruns and every CRC is compared
with the CPU oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import part_crc_util as U  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE


def check(obj, crcs, ocrc, part):
    assert crcs == U.part_crcs(obj, part), part
    assert ocrc == U.crc32c(obj), part


for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 40), (21, 700), (257, 3000), (4096, 4096 * 5 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        key, aad, ivs = corpus.fixed_key_material((n + cs - 1) // cs)
        for flags in (Z, A, Z | D | A):
            for part in (1, 7, 4095, 1 << 20):
                out, _, crcs, ocrc = c.transform_parts(flags, src, cs, part, np.zeros(32, np.uint8), True, None, key, aad, ivs)
                check(out.copy(), crcs, ocrc, part)
    src = corpus.gen_segment("R", 5, 4096 * 7 + 5, 4096)
    key, aad, ivs = corpus.fixed_key_material(8)
    for part in (7, 5000):
        pc, outs, crcs, lo = np.zeros(32, np.uint8), [], [], 0
        while True:
            win = src[lo:lo + 2 * 4096]
            end = win.size < 2 * 4096
            o, _, p, oc = c.transform_parts(A, win, 4096, part, pc, end, None, key, aad, ivs[12 * (lo // 4096):])
            outs.append(o.copy()); crcs += p
            if end:
                break
            lo += 2 * 4096
        check(np.concatenate(outs), crcs, oc, part)
    c.close()
print("part crc sweep ok")
