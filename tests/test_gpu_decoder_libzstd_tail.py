"""Tracking test of a decoder defect on the H100: a 48 MiB + 77 B corpus-K segment (seed 32) in 4 MiB chunks, written by libzstd
(the oracle, what the Java plugin writes), has been detransformed to wrong bytes in some runs and not in others: silently, with
every frame accepted and every size right (first wrong byte seen at offset 30 801 934, in chunk 7).  The same decoder serves
tsgpu_detransform, tsgpu_check_object and tsgpu_rewrite_object, so their segment words then disagree with the segment too.  The
test is expected to fail until the decoder is fixed; it is not strict, since the defect does not show in every run."""
import numpy as np
import pytest

import tsgpu
from tsgpu import corpus
from oracle import oracle as ora

CS = 4 << 20


@pytest.mark.gpu
@pytest.mark.xfail(strict=False, reason="the zstd decoder intermittently returns wrong bytes for this libzstd object")
def test_libzstd_object_with_a_77_byte_last_chunk_decodes_to_the_segment():
    n = 48 * (1 << 20) + 77
    s = corpus.gen_segment("K", 32, n, CS)
    key, aad, ivs = corpus.fixed_key_material((n + CS - 1) // CS)
    ref, sizes = ora.transform_segment(ora.FLAG_ZSTD, s, CS, key, aad, ivs)
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    try:
        back, _ = ctx.detransform(tsgpu.FLAG_ZSTD, np.asarray(ref, np.uint8), sizes, n + 64)
        assert back.size == n
        bad = np.flatnonzero(back != s)
        assert bad.size == 0, "first wrong byte at %d (chunk %d)" % (bad[0], bad[0] // CS)
    finally:
        ctx.close()
