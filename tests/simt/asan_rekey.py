"""Run by tests/test_simt_rekey_sanitizers.py in a subprocess (argv[1] = the library to load, the ASan or the UBSan build):
tsgpu_rekey_object on AES and Zstd+AES objects from 12 bytes to several batches in chunks from 1 byte to 4 KiB, with empty chunks
and chunks of 1 to 27 bytes among them, one and two chunks per slot batch, in one call and in windows with VERIFY, so the
in-place rekey kernels, the two read-back decrypts, the pack and the part checksums are checked for overruns; damaged sources must
fail, never overrun."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import part_crc_util as U  # noqa: E402
import rekey_util as K  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, A, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_VERIFY
nk, na = bytes(range(1, 33)), b"new-aad"

for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 12), (257, 1300), (4096, 4096 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        nch = (n + cs - 1) // cs
        key, aad, ivs = corpus.fixed_key_material(nch)
        nivs = np.random.default_rng(cs).bytes(12 * nch)
        for ff in ((A, Z | A) if max_batch == 2 else (A,)):
            obj, sizes = c.transform(ff, src, cs, key, aad, ivs)
            obj = obj.copy()
            want = K.expected(obj, sizes, key, aad, nk, na, nivs)
            for win, flags in ((None, 0), (3, V)):
                new, parts, crc2 = K.rekey_windows(c, obj, sizes, key, nk, nivs, 1000, win, aad, na, flags)
                assert np.array_equal(new, want) and crc2 == (U.crc32c(obj), U.crc32c(want)), (cs, ff, win, flags)
            if max_batch == 1:
                continue
            bad = obj.copy()
            bad[obj.size // 2] ^= 0x40
            try:
                K.rekey_windows(c, bad, sizes, key, nk, nivs, 1000, 2, aad, na, V)
                raise AssertionError("a flipped byte passed")
            except tsgpu.TsgpuError:
                pass
    # empty chunks and chunks too short for IV and tag between ordinary ones
    rng = np.random.default_rng(9)
    plain = [rng.bytes(k) for k in (100, 0, 17, 4000)]
    obj, sizes = K.encrypt_chunks(b"k" * 32, b"", [plain[0], None, plain[1], plain[2], None, plain[3]])
    nivs = rng.bytes(12 * len(sizes))
    for flags in (0, V):
        new, _, _ = c.rekey_object(obj, sizes, b"k" * 32, nk, nivs, 1000, flags=flags)
        assert np.array_equal(new, K.expected(obj, sizes, b"k" * 32, b"", nk, b"", nivs))
    for short in (1, 27):
        try:
            c.rekey_object(np.concatenate([obj, np.zeros(short, np.uint8)]), sizes + [short], b"k" * 32, nk, nivs + bytes(12), 1000)
            raise AssertionError("a %d-byte chunk passed" % short)
        except tsgpu.TsgpuError:
            pass
    c.close()
print("rekey sweep ok")
