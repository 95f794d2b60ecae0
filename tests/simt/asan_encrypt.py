"""Run by tests/test_simt_encrypt_sanitizers.py in a subprocess (argv[1] = the library to load, the ASan or the UBSan build):
tsgpu_encrypt_object on plain and Zstd-only objects from 12 bytes to several batches in chunks from 1 byte to 4 KiB, with empty
chunks among them, one and two chunks per slot batch, in one call and in windows with VERIFY, so the frame walk, the in-place
encryption, the read-back decrypt, the pack and the part checksums are checked for overruns.  Single frames with mutated headers
and block headers, cut short or grown, must fail or pass, and the walk over them must stay inside the slot buffers."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402
import encrypt_util as E  # noqa: E402
import part_crc_util as U  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
Z, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_VERIFY
key, aad = bytes(range(1, 33)), b"aad"

for max_batch in (1, 2):
    c = tsgpu.Context(max_chunk_bytes=1 << 16, max_batch=max_batch, lib_path=lib)
    for cs, n in ((1, 12), (257, 1300), (4096, 4096 + 17)):
        src = corpus.gen_segment("K", cs, n, cs)
        nch = (n + cs - 1) // cs
        k0, a0, ivs = corpus.fixed_key_material(nch)
        nivs = np.random.default_rng(cs).bytes(12 * nch)
        plain = (src.copy(), [min(cs, n - i) for i in range(0, n, cs)], 0)
        zo, zs = ora.transform_segment(Z, src, cs, k0, a0, ivs)
        for obj, sizes, ff in (plain, (np.asarray(zo).copy(), list(zs), Z)):
            want, _ = E.expected(obj, sizes, key, aad, nivs)
            for win, flags in ((None, 0), (3, V)):
                new, _, parts, crc2 = E.encrypt_windows(c, obj, sizes, key, nivs, 1000, win, cs, n, aad, ff | flags)
                assert np.array_equal(new, want) and crc2 == (U.crc32c(obj), U.crc32c(want)), (cs, ff, win, flags)
    # an .indexes-shaped object with empty blobs between ordinary ones
    rng = np.random.default_rng(9)
    blobs = [rng.bytes(k) for k in (100, 0, 17, 4000, 0, 1)]
    obj = np.frombuffer(b"".join(blobs), np.uint8).copy()
    sizes = [len(b) for b in blobs]
    nivs = rng.bytes(12 * len(sizes))
    for flags in (0, V):
        new, _, _, _ = c.encrypt_object(obj, sizes, key, nivs, 1000, flags=flags)
        assert np.array_equal(new, E.expected(obj, sizes, key, b"", nivs)[0])
    # mutated frames: the header bytes and the first block headers flipped, bytes set at random, the frame cut and grown
    seg = corpus.gen_segment("K", 3, 3000, 3000)
    zo, zs = ora.transform_segment(Z, seg, 3000, key, aad, np.zeros(12, np.uint8).tobytes())
    f = bytes(np.asarray(zo)[:zs[0]])
    rng = np.random.default_rng(max_batch)
    cases = [f[:k] for k in range(0, len(f), 7)] + [f + bytes(k) for k in (1, 7, 8, 9)]
    for i in range(min(len(f), 24)):
        for v in (0x00, 0xff, 0x01 << (i % 8)):
            g = bytearray(f); g[i] ^= v or 0xff; cases.append(bytes(g))
    for _ in range(40):
        g = bytearray(f); g[int(rng.integers(0, len(f)))] = int(rng.integers(0, 256)); cases.append(bytes(g))
    for g in cases:
        chunk = np.frombuffer(g, np.uint8).copy()
        try:
            c.encrypt_object(chunk, [chunk.size], key, nivs[:12], 1000, 3000, 3000, aad, Z | V)
        except tsgpu.TsgpuError:
            pass
    c.close()
print("encrypt sweep ok")
