"""tsgpu_rewrite_object on an H100: a 1 GiB generated Kafka segment in 4 MiB chunks, stored ZSTD|AES by tsgpu_transform and by the
oracle (libzstd + OpenSSL, what the Java plugin wrote), and plain, is rewritten under a new key in one call and in windows of 32
chunks.  The source, object, segment and part CRCs equal the CPU CRC-32C, sampled chunks of the new object decode with the oracle,
and the new object passes tsgpu_check_object.  The profile shows no compressor when frames are kept and the compressor when a
plain object is compressed, no record kernel without VALIDATE_RECORDS, and at most two GCM key set-ups per claimed slot."""
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import check_util as K  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import rewrite_util as W  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, VR, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_VALIDATE_RECORDS, tsgpu.FLAG_VERIFY
CS = 4 << 20
GIB = 1 << 30
PART = 64 << 20


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(13, GIB, payload=corpus.gen_segment("K", 13, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))


@pytest.fixture(scope="module")
def seg_crc(seg):
    return U.crc32c(seg)


def _keys(n):
    return corpus.fixed_key_material(max((n + CS - 1) // CS, 1))


def _plain_sizes(n):
    return [min(CS, n - i * CS) for i in range((n + CS - 1) // CS)]


def _sample_decodes(tf, new, nsz, seg, nk, na):
    starts = np.concatenate([[0], np.cumsum(nsz, dtype=np.uint64)]).astype(np.int64)
    for k in sorted({0, 1, len(nsz) // 2, len(nsz) - 1}):
        ch = new[starts[k]:starts[k + 1]]
        b = ora.aesgcm_decrypt_chunk(nk, na, ch) if tf & A else bytes(ch)
        if tf & Z:
            b = ora.zstd_decompress_chunk(b)
        assert b == bytes(seg[k * CS:min((k + 1) * CS, seg.size)]), k


ROWS = [("ZA-ZA", Z | A, False, Z | A), ("oracleZA-ZA", Z | A, True, Z | A), ("plain-ZA", 0, False, Z | A), ("ZA-A", Z | A, False, A)]


@pytest.mark.parametrize("ff,oracle,tf", [r[1:] for r in ROWS], ids=[r[0] for r in ROWS])
def test_rewrite_matrix_rows(ctx, seg, seg_crc, ff, oracle, tf):
    key, aad, ivs = _keys(seg.size)
    if ff == 0:
        obj, sizes = seg, _plain_sizes(seg.size)
    elif oracle:
        obj, sizes = ora.transform_segment(ff, seg, CS, key, aad, ivs)
    else:
        obj, sizes = ctx.transform(ff, seg, CS, key, aad, ivs)
        obj = obj.copy()
    nk, na, nivs = W.new_key_material(len(sizes))
    src_crc = U.crc32c(obj)
    for win in (None, 32):
        new, nsz, parts, crc3 = W.rewrite_windows(ctx, ff | VR, obj, sizes, CS, seg.size, tf | V, PART, win, key, aad, nk, na, nivs)
        assert crc3 == (src_crc, U.crc32c(new), seg_crc), win
        assert parts == U.part_crcs(new, PART), win
        _sample_decodes(tf, new, nsz, seg, nk, na)
        if ff & Z and tf & Z:
            starts = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
            k = len(sizes) // 3
            old = W.frames(ff, obj[starts[k]:starts[k + 1]], [sizes[k]], key, aad)
            nst = np.concatenate([[0], np.cumsum(nsz)]).astype(np.int64)
            assert W.frames(tf, new[nst[k]:nst[k + 1]], [nsz[k]], nk, na) == old   # kept byte for byte
    assert K.check_windows(ctx, tf | VR, new, nsz, CS, seg.size, None, nk, na) == (crc3[1], seg_crc)


def test_profile(seg):
    ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)             # no key tables built yet
    key, aad, ivs = _keys(seg.size)
    obj, sizes = ora.transform_segment(Z | A, seg, CS, key, aad, ivs)
    nk, na, nivs = W.new_key_material(len(sizes))
    ctx.profile_enable(True)
    W.rewrite_windows(ctx, Z | A, obj, sizes, CS, seg.size, Z | A, PART, None, key, aad, nk, na, nivs)
    rep = ctx.profile_report()
    assert not any(n.startswith("zstd_enc_") for n in rep), sorted(rep)             # frames kept
    assert not any(n.startswith("rec_") for n in rep), sorted(rep)                  # no VALIDATE_RECORDS
    slots = min(8, (len(sizes) + 3) // 4)
    assert 2 <= rep["gcm_key_setup"]["launches"] <= 2 * slots, rep["gcm_key_setup"]
    ctx.profile_enable(True)
    W.rewrite_windows(ctx, 0, seg, _plain_sizes(seg.size), CS, seg.size, Z, PART, None)
    rep = ctx.profile_report()
    assert "zstd_enc_blocks" in rep and "gcm_key_setup" not in rep, sorted(rep)
    ctx.profile_enable(False)
    ctx.close()
