"""tsgpu_check_object on an H100: 1 GiB generated Kafka segments in 4 MiB chunks, written by tsgpu_transform with every flag set
{0, AES, ZSTD, ZSTD|DENSE, ZSTD|CHECKSUM, ZSTD|AES, ZSTD|DENSE|AES} and by the oracle (libzstd + OpenSSL), pass with and without
VALIDATE_RECORDS and give the CPU CRC-32C of the object and of the segment, in one call and in windows of 1, 3 and 32 chunks.
Every kind of damage fails with its code, naming the chunk or the segment position; without the flag no record kernel runs."""
import os
import re
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import check_util as K  # noqa: E402
import part_crc_util as U  # noqa: E402
import records_util as R  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D, CK, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_VALIDATE_RECORDS
CS = 4 << 20
GIB = 1 << 30
FLAG_SETS = [0, A, Z, Z | D, Z | CK, Z | A, Z | D | A]
FLAG_IDS = ["plain", "A", "Z", "ZD", "ZC", "ZA", "ZDA"]


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


def _write(c, flags, s):
    key, aad, ivs = _keys(s.size)
    out, sizes = c.transform(flags, s, CS, key, aad, ivs)
    return out.copy(), sizes, key, aad


def _fails(code, call):
    with pytest.raises(tsgpu.TsgpuError) as ei:
        call()
    assert ei.value.code == code, str(ei.value)
    return str(ei.value)


@pytest.mark.parametrize("flags", FLAG_SETS, ids=FLAG_IDS)
def test_written_object_passes_with_the_oracle_crcs(ctx, seg, seg_crc, flags):
    obj, sizes, key, aad = _write(ctx, flags, seg)
    want = (U.crc32c(obj), seg_crc)
    for records in (0, VR):
        for win in (None, 1, 3, 32):
            if win in (1, 3) and records == 0 and flags not in (Z | A, 0):
                continue                                         # small windows: the record cursor and two flag sets suffice
            assert K.check_windows(ctx, flags | records, obj, sizes, CS, seg.size, win, key, aad) == want, (records, win)


@pytest.mark.parametrize("flags", [Z, Z | A], ids=["Z", "ZA"])
def test_oracle_written_object_passes(ctx, seg, seg_crc, flags):
    key, aad, ivs = _keys(seg.size)
    obj, sizes = ora.transform_segment(flags, seg, CS, key, aad, ivs)
    for win in (None, 32):
        assert K.check_windows(ctx, flags | VR, obj, sizes, CS, seg.size, win, key, aad) == (U.crc32c(obj), seg_crc)


# ---------------------------------------------------------------------------------------------------- 64 MiB
@pytest.fixture(scope="module")
def small(seg):
    cut = int(R.starts(seg)[np.searchsorted(R.starts(seg), 64 << 20)])
    return seg[:cut].copy()


def test_without_the_flag_no_record_kernel_runs(ctx, small):
    obj, sizes, key, aad = _write(ctx, Z | A, small)
    ctx.profile_enable(True)
    ctx.check_object(Z | A, obj, sizes, CS, small.size, key=key, aad=aad)
    names = set(ctx.profile_report())
    assert not any(n.startswith("rec_") for n in names), names
    assert {"pcrc_tiles_slots", "pcrc_tiles"} <= names, names
    ctx.profile_enable(True)
    ctx.check_object(Z | A | VR, obj, sizes, CS, small.size, key=key, aad=aad)
    assert "rec_resolve" in ctx.profile_report()
    ctx.profile_enable(False)


def _chunk_start(sizes, k):
    return int(sum(sizes[:k]))


def test_damage_names_the_chunk(ctx, small):
    n = small.size
    obj, sizes, key, aad = _write(ctx, Z | A, small)
    bad = obj.copy()
    bad[_chunk_start(sizes, 9) + 5000] ^= 1
    assert "chunk 9" in _fails(binding.E_AUTH, lambda: K.check_windows(ctx, Z | A | VR, bad, sizes, CS, n, 3, key, aad))
    obj, sizes, _, _ = _write(ctx, Z | CK, small)
    bad = obj.copy()
    bad[_chunk_start(sizes, 6) - 1] ^= 0x20                        # chunk 5's Content_Checksum
    assert re.search(r"chunk 5\b", _fails(binding.E_CORRUPT, lambda: K.check_windows(ctx, Z, bad, sizes, CS, n, 4)))
    bad = obj.copy()
    bad[_chunk_start(sizes, 11)] ^= 0xFF                           # chunk 11's frame magic
    assert re.search(r"chunk 11\b", _fails(binding.E_CORRUPT, lambda: ctx.check_object(Z, bad, sizes, CS, n)))
    last = len(sizes) - 1
    tail = n - last * CS
    msg = _fails(binding.E_CORRUPT, lambda: ctx.check_object(Z, obj, sizes, CS, n + 1))
    assert "chunk %d decoded to %d bytes, the chunk index gives %d" % (last, tail, tail + 1) in msg
    _fails(binding.E_SHORT, lambda: ctx.check_object(Z, obj[:-1], sizes, CS, n))


def test_bad_record_batch_fails_with_the_upload_message(ctx, small):
    st = R.starts(small)
    ends = np.append(st[1:], small.size)
    e = next(i for i in range(len(st)) if small[int(st[i]) + 16] == 2 and int(st[i]) // (3 * CS) != (int(ends[i]) - 1) // (3 * CS))
    bad = small.copy()
    bad[int(st[e]) + 19] ^= 1                                      # its stored CRC; the entry crosses a 3-chunk window end
    key, aad, ivs = _keys(bad.size)
    upload = _fails(binding.E_RECORDS, lambda: ctx.transform(Z | A | VR, bad, CS, key, aad, ivs))
    obj, sizes, key, aad = _write(ctx, Z | A, bad)
    for win in (None, 3):
        assert _fails(binding.E_RECORDS, lambda: K.check_windows(ctx, Z | A | VR, obj, sizes, CS, bad.size, win, key, aad)) == upload
    cut = int(st[-1]) + 20                                         # inside the last entry's header
    obj, sizes, _, _ = _write(ctx, Z, small[:cut])
    msg = _fails(binding.E_RECORDS, lambda: K.check_windows(ctx, Z | VR, obj, sizes, CS, cut, 3))
    assert "check: length" in msg and "segment position %d" % int(st[-1]) in msg
