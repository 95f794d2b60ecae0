"""Run by tests/test_simt_checksum.py in a subprocess with libasan preloaded (argv[1] = the library to load): the shapes of that
test with TSGPU_FLAG_ZSTD_CHECKSUM -- every flag mix over corpora K, R and Z, chunk sizes from 1 byte to 64 KiB + 1 with a
ragged last chunk, ragged blobs -- so the hashing warps' staging and the checksum hand-over are checked for overruns."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import corpus  # noqa: E402
import test_simt_checksum as T  # noqa: E402

lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
T.SIMT_LIB = lib
c = tsgpu.Context(max_chunk_bytes=1 << 17, max_batch=2, lib_path=lib)
for kind in "KRZ":
    for cs in (1, 31, 32, 33, 8191, 8192, 65537):
        for flags in T.FLAGS:
            T.check_checksummed(c, flags, corpus.gen_segment(kind, 5, T._seg_len(cs), cs), cs)
rng = np.random.default_rng(3)
blobs = [rng.integers(0, 256, 10485, dtype=np.uint8), corpus.gen_chunk("K", 1, 0, 37), corpus.gen_chunk("K", 1, 1, 40001)]
key, aad, ivs = corpus.fixed_key_material(len(blobs))
for flags in T.FLAGS:
    out, sizes = c.transform_chunks(flags | T.C | T.V, np.concatenate(blobs), [b.size for b in blobs], key, aad, ivs)
    back, _ = c.detransform(flags & (T.Z | T.A), out, sizes, sum(b.size for b in blobs), key, aad)
    assert np.array_equal(back, np.concatenate(blobs))
c.close()
print("checksum sweep ok")
