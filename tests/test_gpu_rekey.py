"""tsgpu_rekey_object on an H100: 256 MiB Kafka segments in 4 MiB chunks, stored Zstd+AES by this library (speed mode) and by the
oracle (libzstd + OpenSSL, what the Java plugin wrote), and AES only, are re-encrypted under a new key in one call and in windows of
16 chunks.  Every new chunk equals OpenSSL's decrypt-then-encrypt of the old one, the CRCs equal the CPU CRC-32C and CRC-64/NVME,
the libzstd object's segment comes back through the oracle alone, and no zstd kernel runs: the decoder's path counters do not move
and the profile lists no zstd_* kernel."""
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crc64_util as U64  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402
import rekey_util as K  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_VERIFY
CS = 4 << 20
SEG = 256 << 20
PART = 64 << 20
NEW_KEY, NEW_AAD = bytes(range(64, 96)), b"rotated-segment-key"


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(17, SEG, payload=corpus.gen_segment("K", 17, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))


def _stored(ctx, seg, kind):
    key, aad, ivs = corpus.fixed_key_material((seg.size + CS - 1) // CS)
    if kind == "libzstd-ZA":
        obj, sizes = ora.transform_segment(Z | A, seg, CS, key, aad, ivs)
    elif kind == "speed-ZA":
        obj, sizes = ctx.transform(Z | A, seg, CS, key, aad, ivs)
    else:
        obj, sizes = ctx.transform(A, seg, CS, key, aad, ivs)
    return np.asarray(obj).copy(), sizes, key, aad


@pytest.mark.parametrize("kind", ["speed-ZA", "libzstd-ZA", "A"])
def test_rekeyed_object_is_the_oracles(ctx, seg, kind):
    obj, sizes, key, aad = _stored(ctx, seg, kind)
    ivs = np.random.default_rng(3).bytes(12 * len(sizes))
    want = K.expected(obj, sizes, key, aad, NEW_KEY, NEW_AAD, ivs)
    src_crc, want_crc = U.crc32c(obj), U.crc32c(want)
    before = ctx.decode_path_stats()
    ctx.profile_enable(True)
    for win, flags in ((None, 0), (16, 0), (None, V)):
        new, parts, crc2 = K.rekey_windows(ctx, obj, sizes, key, NEW_KEY, ivs, PART, win, aad, NEW_AAD, flags)
        assert np.array_equal(new, want), (win, flags)
        assert crc2 == (src_crc, want_crc) and parts == U.part_crcs(want, PART), (win, flags)
    rep = ctx.profile_report()
    ctx.profile_enable(False)
    assert ctx.decode_path_stats() == before                                       # nothing was decoded
    assert not any(n.startswith("zstd_") for n in rep), sorted(rep)
    assert "gcm_rekey" in rep and "gcm_rekey_finalize" in rep, sorted(rep)
    if kind == "libzstd-ZA":                                                       # the segment, through libzstd + OpenSSL alone
        back, _ = ora.detransform_chunks(Z | A, new, sizes, seg.size, NEW_KEY, NEW_AAD)
        assert np.array_equal(back, seg)


def test_crc64_twin_writes_the_same_bytes(ctx, seg):
    obj, sizes, key, aad = _stored(ctx, seg, "speed-ZA")
    ivs = np.random.default_rng(4).bytes(12 * len(sizes))
    new32, _, _ = K.rekey_windows(ctx, obj, sizes, key, NEW_KEY, ivs, PART, 16, aad, NEW_AAD)
    new64, parts, crc2 = K.rekey_windows(ctx, obj, sizes, key, NEW_KEY, ivs, PART, 16, aad, NEW_AAD, crc64=True)
    assert np.array_equal(new32, new64)
    assert crc2 == (U64.crc64nvme(obj), U64.crc64nvme(new64)) and parts == U64.part_crcs(new64, PART)


def test_bad_tag_names_its_chunk(ctx, seg):
    obj, sizes, key, aad = _stored(ctx, seg, "A")
    ivs = np.random.default_rng(5).bytes(12 * len(sizes))
    k = len(sizes) // 2
    bad = obj.copy()
    bad[int(np.sum(sizes[:k])) + 12345] ^= 0x10
    with pytest.raises(tsgpu.TsgpuError) as ei:
        K.rekey_windows(ctx, bad, sizes, key, NEW_KEY, ivs, PART, 16, aad, NEW_AAD)
    assert str(ei.value) == "Tag mismatch in chunk %d" % k
