"""Run by tests/test_simt_crc64.py in a subprocess (argv[1] = the library to load: the ASan build, or the plain one with
TSGPU_SIMT_POISON=1 or a TSGPU_SIMT_ORDER): CRC-64/NVME part checksums of objects from 1 byte to several tiles, one and several
chunks per slot batch, part sizes from 1 byte to more than the object, windows through one parts cursor, and the check's and the
rewrite's words (the slots variant of the kernels), each compared with the CPU oracle."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import crc64_util as U  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE


def check(obj, crcs, ocrc, part):
    assert crcs == U.part_crcs(obj, part), part
    assert ocrc == U.crc64nvme(obj), part


for max_batch in (1, 12):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 40), (257, 3000), (4096, 4096 * 13 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        key, aad, ivs = corpus.fixed_key_material((n + cs - 1) // cs)
        for flags in (Z, A, Z | D | A):
            for part in (1, 7, 4095, 1 << 20):
                if part == 1 and n > 5000:
                    continue
                out, _, crcs, ocrc = c.transform_parts_crc64(flags, src, cs, part, np.zeros(32, np.uint8), True, None, key, aad, ivs)
                check(out.copy(), crcs, ocrc, part)
    src = corpus.gen_segment("R", 5, 4096 * 7 + 5, 4096)
    key, aad, ivs = corpus.fixed_key_material(8)
    pc, outs, crcs, lo = np.zeros(32, np.uint8), [], [], 0
    while True:
        win = src[lo:lo + 2 * 4096]
        end = win.size < 2 * 4096
        o, _, p, oc = c.transform_parts_crc64(A, win, 4096, 5000, pc, end, None, key, aad, ivs[12 * (lo // 4096):])
        outs.append(o.copy()); crcs += p
        if end:
            break
        lo += 2 * 4096
    check(np.concatenate(outs), crcs, oc, 5000)
    for flags in (A, Z | A):
        obj, sizes = c.transform(flags, src, 4096, key, aad, ivs)
        obj = obj.copy()
        assert c.check_object_crc64(flags, obj, sizes, 4096, src.size, key=key, aad=aad) == (U.crc64nvme(obj), U.crc64nvme(src))
        to = Z | A if flags & Z else Z | D | A                     # a zstd source keeps its frames
        new, _, p, w = c.rewrite_object_crc64(flags, obj, sizes, 4096, src.size, to, 3000, from_key=key, from_aad=aad,
                                              to_key=bytes(32), to_aad=aad, to_ivs=bytes((i * 7 + 3) & 255 for i in range(12 * 8)))
        new = new.copy()
        assert w == (U.crc64nvme(obj), U.crc64nvme(new), U.crc64nvme(src)) and p == U.part_crcs(new, 3000)
    c.close()
print("crc64 sweep ok")
