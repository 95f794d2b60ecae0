"""TSGPU_FLAG_REFRAME on an H100: a 256 MiB generated Kafka segment in 4 MiB chunks (the records of tests/test_gpu_check.py),
stored ZSTD|AES by the oracle (libzstd level 3, what the Java plugin wrote) and ZSTD or ZSTD|AES by tsgpu_transform, is sealed or
re-encoded under a new key in one call and in windows of 32 chunks (the last window is empty).  Every new frame is the one the CPU
derives from the old frame, libzstd and tsgpu_transform's dense frame; the source, object, segment and part CRCs equal the CPU's;
the new object passes tsgpu_check_object with the source's segment CRC.  The profile shows the seal kernel with CHECKSUM and the
dense compressor and the pick kernel with DENSE only."""
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import check_util as K  # noqa: E402
import crc64_util as U64  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import reframe_util as F  # noqa: E402
import rewrite_util as W  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D, CK, VR, RF = F.Z, F.A, F.D, F.CK, F.VR, F.RF
CS = 4 << 20
PART = 64 << 20


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(13, 256 << 20, payload=corpus.gen_segment("K", 13, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))


@pytest.fixture(scope="module")
def chunks(seg):
    return F.chunks_of(seg, CS)


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


# The zstd decoder misreads chunk 13 of this segment's libzstd object in some decodes, with or without REFRAME: a bare
# tsgpu_detransform returned wrong bytes from offset 56 098 828, and libzstd's own checksummed frames of the chunks failed there as
# an invalid frame (DESIGN.md §9, tests/test_gpu_decoder_libzstd_records.py).  Sealing turns that misread into TSGPU_E_RECORDS or
# TSGPU_E_VERIFY, as it should, so these rows cannot pass until the decoder is fixed.
_DECODER = pytest.mark.xfail(strict=False, reason="the zstd decoder misreads chunk 13 of this libzstd object (DESIGN.md §9)")
ROWS = [pytest.param(Z | A, True, Z | CK | A | RF, id="oracleZA-seal", marks=_DECODER),
        pytest.param(Z | A, True, Z | D | CK | A | RF, id="oracleZA-denseck", marks=_DECODER),
        pytest.param(Z, False, Z | CK | RF, id="speedZ-seal"), pytest.param(Z | A, False, Z | D | A | RF, id="speedZA-dense")]


@pytest.mark.parametrize("ff,oracle,tf", ROWS)
def test_reframe_rows(ctx, seg, chunks, ff, oracle, tf):
    key, aad, ivs = _keys(seg.size)
    if oracle:
        obj, sizes = ora.transform_segment(ff, seg, CS, key, aad, ivs)
    else:
        obj, sizes = ctx.transform(ff, seg, CS, key, aad, ivs)
        obj = obj.copy()
    old = W.frames(ff, obj, sizes, key, aad)
    dense = None
    if tf & D:
        dobj, dsz = ctx.transform(Z | D | (tf & CK), seg, CS)
        dense = W.frames(Z, dobj, dsz)
    want = F.expected(tf, old, chunks, dense)
    if oracle and not tf & D:
        assert want == [ora.zstd_compress_checksum(ch, 3) for ch in chunks]
    nk, na, nivs = W.new_key_material(len(sizes))
    src_crc, seg_crc = U.crc32c(obj), U.crc32c(seg)
    for win in (None, 32):
        new, nsz, parts, crc3 = W.rewrite_windows(ctx, ff | VR, obj, sizes, CS, seg.size, tf, PART, win, key, aad, nk, na, nivs)
        got = W.frames(tf, new, nsz, nk, na)
        assert got == want, (win, [i for i in range(len(got)) if got[i] != want[i]][:8])
        assert crc3 == (src_crc, U.crc32c(new), seg_crc), win
        assert parts == U.part_crcs(new, PART), win
        assert all(len(f) <= len(o) + 4 for f, o in zip(got, old))
    for k in sorted({0, len(got) // 2, len(got) - 1}):
        assert ora.zstd_decompress_chunk(got[k]) == chunks[k], k               # libzstd verifies the checksum
    assert K.check_windows(ctx, (tf & (Z | A)) | VR, new, nsz, CS, seg.size, None, nk, na) == (crc3[1], seg_crc)


def test_crc64_twin(ctx, seg):
    key, aad, ivs = _keys(seg.size)
    obj, sizes = ctx.transform(Z | A, seg, CS, key, aad, ivs)             # this library's frames: the §9 defect is libzstd's
    obj = obj.copy()
    nk, na, nivs = W.new_key_material(len(sizes))
    new, nsz, _, _ = W.rewrite_windows(ctx, Z | A, obj, sizes, CS, seg.size, Z | CK | A | RF, PART, None, key, aad, nk, na, nivs)
    new64, nsz64, parts64, crc64 = ctx.rewrite_object_crc64(Z | A, obj, sizes, CS, seg.size, Z | CK | A | RF, PART, None, True, key,
                                                            aad, nk, na, nivs)
    assert np.array_equal(new64, new) and nsz64 == nsz
    assert crc64 == (U64.crc64nvme(obj), U64.crc64nvme(new), U64.crc64nvme(seg))
    assert parts64 == U64.part_crcs(new, PART)


def test_profile(seg):
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    obj, sizes = ctx.transform(Z, seg, CS)
    obj = obj.copy()
    for tf, seal, dense in ((Z | CK | RF, True, False), (Z | D | RF, False, True), (Z | D | CK | RF, True, True)):
        ctx.profile_enable(True)
        W.rewrite_windows(ctx, Z, obj, sizes, CS, seg.size, tf, PART)
        rep = ctx.profile_report()
        assert ("reframe_seal" in rep) == seal and ("reframe_pick" in rep) == dense, sorted(rep)
        assert any(n.startswith("zstd_enc_") for n in rep) == dense, sorted(rep)
        assert "verify_compare" in rep, sorted(rep)                                  # VERIFY is always on
        if seal:
            assert rep["reframe_seal"]["launches"] == (len(sizes) + 3) // 4
    ctx.profile_enable(False)
    ctx.close()
