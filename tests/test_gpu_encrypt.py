"""tsgpu_encrypt_object on an H100: 256 MiB Kafka segments in 4 MiB chunks, stored Zstd-only by the oracle (libzstd level 3, what
the Java plugin wrote), by this library in speed and in dense mode, and stored plain, are encrypted in one call and in windows of
16 chunks.  Every new chunk equals OpenSSL's IV || AES-256-GCM(chunk) || TAG, the CRCs equal the CPU CRC-32C and CRC-64/NVME, and
no decoder runs: the decoder's path counters do not move and the profile lists no zstd_dec_* kernel.  The seed-13 segment whose
libzstd frames the decoder misreads (DESIGN.md §9) encrypts to OpenSSL's bytes, chunk for chunk: the call does not depend on the
decoder."""
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import crc64_util as U64  # noqa: E402
import encrypt_util as E  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D, V = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_VERIFY
CS = 4 << 20
SEG = 256 << 20
PART = 64 << 20
KEY, AAD = bytes(range(64, 96)), b"encrypted-after-the-fact"


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(17, SEG, payload=corpus.gen_segment("K", 17, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))


def _stored(ctx, seg, kind):
    """(object, chunk sizes, flags) of the segment stored unencrypted"""
    key, aad, ivs = corpus.fixed_key_material((seg.size + CS - 1) // CS)
    if kind == "plain":
        return seg.copy(), [min(CS, seg.size - i) for i in range(0, seg.size, CS)], 0
    if kind == "libzstd":
        obj, sizes = ora.transform_segment(Z, seg, CS, key, aad, ivs)
    else:
        cur = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8)
        obj, sizes, _, _ = ctx.transform_parts(Z | (D if kind == "dense" else 0), seg, CS, PART, cur, True,
                                               np.zeros(binding.CURSOR_SIZE, np.uint8), key, aad, ivs)
    return np.asarray(obj).copy(), list(sizes), Z


@pytest.mark.parametrize("kind", ["libzstd", "speed", "dense", "plain"])
def test_encrypted_object_is_openssls(ctx, seg, kind):
    obj, sizes, flags = _stored(ctx, seg, kind)
    ivs = np.random.default_rng(3).bytes(12 * len(sizes))
    want, wsz = E.expected(obj, sizes, KEY, AAD, ivs)
    src_crc, want_crc = U.crc32c(obj), U.crc32c(want)
    before = ctx.decode_path_stats()
    ctx.profile_enable(True)
    for win, f in ((None, 0), (16, 0), (None, V)):
        new, nsz, parts, crc2 = E.encrypt_windows(ctx, obj, sizes, KEY, ivs, PART, win, CS, seg.size, AAD, flags | f)
        assert np.array_equal(new, want), (win, f)
        assert nsz == wsz and crc2 == (src_crc, want_crc) and parts == U.part_crcs(want, PART), (win, f)
    rep = ctx.profile_report()
    ctx.profile_enable(False)
    assert ctx.decode_path_stats() == before                                       # nothing was decoded
    assert not any(n.startswith("zstd_") for n in rep), sorted(rep)
    assert "gcm_main_enc" in rep and ("frame_walk" in rep) == (flags == Z), sorted(rep)
    if kind == "libzstd":                                                          # the segment, through libzstd + OpenSSL alone
        back, _ = ora.detransform_chunks(Z | A, new, nsz, seg.size, KEY, AAD)
        assert np.array_equal(back, seg)


def test_crc64_twin_writes_the_same_bytes(ctx, seg):
    obj, sizes, flags = _stored(ctx, seg, "speed")
    ivs = np.random.default_rng(4).bytes(12 * len(sizes))
    new32, _, _, _ = E.encrypt_windows(ctx, obj, sizes, KEY, ivs, PART, 16, CS, seg.size, AAD, flags)
    new64, _, parts, crc2 = E.encrypt_windows(ctx, obj, sizes, KEY, ivs, PART, 16, CS, seg.size, AAD, flags, crc64=True)
    assert np.array_equal(new32, new64)
    assert crc2 == (U64.crc64nvme(obj), U64.crc64nvme(new64)) and parts == U64.part_crcs(new64, PART)


def test_seed13_libzstd_object_the_decoder_misreads(ctx):
    s = R.gen_segment(13, 256 << 20, payload=corpus.gen_segment("K", 13, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))
    key, aad, ivs = corpus.fixed_key_material((s.size + CS - 1) // CS)
    obj, sizes = ora.transform_segment(Z, s, CS, key, aad, ivs)
    obj = np.asarray(obj).copy()
    nivs = np.random.default_rng(13).bytes(12 * len(sizes))
    want, wsz = E.expected(obj, sizes, KEY, AAD, nivs)
    new, nsz, _, crc2 = E.encrypt_windows(ctx, obj, sizes, KEY, nivs, PART, 16, CS, s.size, AAD, Z)
    starts = np.concatenate([[0], np.cumsum(wsz)]).astype(int)
    bad = [i for i in range(len(wsz)) if not np.array_equal(new[starts[i]:starts[i + 1]], want[starts[i]:starts[i + 1]])]
    assert bad == [] and nsz == wsz and crc2 == (U.crc32c(obj), U.crc32c(want))
