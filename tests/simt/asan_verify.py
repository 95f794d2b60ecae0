"""Run by tests/test_simt_verify.py in a subprocess with libasan preloaded (argv[1] = the library to load): the shapes of that
test with TSGPU_FLAG_VERIFY -- every flag mix over corpora K, R and Z in two batches, ragged index blobs -- and one fault of each
kind through the emulator's TSGPU_SIMT_FLIP hook, so the read-back stage's buffer reuse is checked for overruns."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import tsgpu  # noqa: E402
from tsgpu import binding, corpus  # noqa: E402
from oracle import oracle as ora  # noqa: E402

Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
CS = 1 << 16
lib = os.path.join(ROOT, "tests", "simt", sys.argv[1] if len(sys.argv) > 1 else "libtsgpu_simt_asan.so")
c = tsgpu.Context(max_chunk_bytes=CS, max_batch=2, lib_path=lib)
n = 3 * CS - 777
key, aad, ivs = corpus.fixed_key_material(3)
for kind in "KRZ":
    src = corpus.gen_segment(kind, 7, n, CS)
    for flags in (Z, Z | D, A, Z | A, Z | D | A):
        out, sizes = c.transform(flags | V, src, CS, key, aad, ivs)
        back, _ = ora.detransform_chunks(flags & (Z | A), out, sizes, n, key, aad)
        assert np.array_equal(back, src), (kind, flags)
rng = np.random.default_rng(11)
blobs = [rng.integers(0, 256, 10485, dtype=np.uint8), corpus.gen_chunk("K", 1, 0, 37), corpus.gen_chunk("K", 1, 1, 40001),
         np.zeros(126, np.uint8), corpus.gen_chunk("K", 1, 2, 1)]
bkey, baad, bivs = corpus.fixed_key_material(len(blobs))
for flags in (A, Z | A, Z | D | A):
    out, sizes = c.transform_chunks(flags | V, np.concatenate(blobs), [b.size for b in blobs], bkey, baad, bivs)
    pos = 0
    for blob, t in zip(blobs, sizes):
        back, _ = ora.detransform_chunks(flags & (Z | A), out[pos:pos + t], [t], blob.size, bkey, baad)
        assert np.array_equal(back, blob)
        pos += t
src = corpus.gen_segment("K", 7, n, CS)
for flags, flip, what in ((Z | D, "1:0", "frame"), (Z | D, "2:-40", None), (Z | D | A, "0:112", "tag"), (A, "2:-1", "tag")):
    os.environ["TSGPU_SIMT_FLIP"] = flip
    try:
        c.transform(flags | V, src, CS, key, aad, ivs)
        raise SystemExit("fault %s not detected (flags %d)" % (flip, flags))
    except tsgpu.TsgpuError as e:
        assert e.code == binding.E_VERIFY and (what is None or what in str(e)), e
    finally:
        del os.environ["TSGPU_SIMT_FLIP"]
c.close()
print("verify sweep ok")
