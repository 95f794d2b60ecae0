"""tsgpu_transform_parts on an H100: 1 GiB segments of corpora K and R in 4 MiB chunks, with the reference's S3 part size (5 MiB),
8 MiB + 1 and 25 MiB, for Zstd+AES in speed and dense mode and AES alone, in one call and in the 32-chunk windows of the JNI
enumeration.  Every part CRC and the object CRC equal the CPU CRC-32C of the returned bytes; dense mode and AES alone return the
bytes of tsgpu_transform_cursor; a call without the new entry point launches what it did before and no part-checksum kernel."""
import os
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import part_crc_util as U  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE
CS = 4 << 20
GIB = 1 << 30
MIB = 1 << 20
FLAGS = [Z | A, Z | D | A, A]
FLAG_IDS = ["ZA", "ZDA", "A"]


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


_segs = {}


def _seg(kind):
    if kind not in _segs:
        _segs.clear()
        _segs[kind] = corpus.gen_segment(kind, 21, GIB, CS)
    return _segs[kind]


def _keys(s):
    return corpus.fixed_key_material((s.size + CS - 1) // CS)


def _check(obj, crcs, ocrc, part):
    assert crcs == U.part_crcs(obj, part), "part CRCs differ from the CPU CRC-32C of the returned bytes"
    assert ocrc == U.crc32c(obj)


def _windows(c, flags, s, part, keys):
    """the JNI enumeration's windows of 32 chunks, with the empty end-of-segment call when the last window is full"""
    key, aad, ivs = keys
    pc, rc = np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8), np.zeros(binding.CURSOR_SIZE, np.uint8)
    outs, crcs, ocrc, w, lo = [], [], None, 32 * CS, 0
    while True:
        win = s[lo:lo + w]
        end = win.size < w                              # a short window ends the segment; after a full one, an empty call does
        iv = ivs[12 * (lo // CS):] if win.size else np.zeros(12, np.uint8)     # the empty call still carries an IV, as in Java
        o, _, p, oc = c.transform_parts(flags, win, CS, part, pc, end, rc, key, aad, iv)
        outs.append(o.copy()); crcs += p
        if end:
            ocrc = oc
            break
        lo += w
    return np.concatenate(outs), crcs, ocrc


@pytest.mark.parametrize("kind", ["K", "R"])
@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_one_call_every_part(ctx, kind, flags):
    s = _seg(kind)
    key, aad, ivs = _keys(s)
    ref = None
    if flags & D or not flags & Z:                   # deterministic writers: the bytes of tsgpu_transform_cursor
        ref, _ = ctx.transform_cursor(flags, s, CS, np.zeros(binding.CURSOR_SIZE, np.uint8), True, key, aad, ivs)
        ref = ref.copy()
    for part in (5 * MIB, 8 * MIB + 1, 25 * MIB):
        out, sizes, crcs, ocrc = ctx.transform_parts(flags, s, CS, part, np.zeros(binding.PARTS_CURSOR_SIZE, np.uint8), True,
                                                     None, key, aad, ivs)
        assert len(crcs) == (out.size + part - 1) // part
        _check(out, crcs, ocrc, part)
        if ref is not None:
            assert np.array_equal(out, ref)


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
def test_windows_of_32_chunks(ctx, flags):
    s = _seg("K")
    keys = _keys(s)
    for part in (5 * MIB, 8 * MIB + 1):
        obj, crcs, ocrc = _windows(ctx, flags, s, part, keys)
        _check(obj, crcs, ocrc, part)


def test_launches_without_the_new_call_are_unchanged(ctx):
    s = _seg("K")[:64 * MIB]
    keys = _keys(s)

    def launches(call):
        before = ctx.launch_count()
        call()
        return ctx.launch_count() - before
    plain = lambda: ctx.transform(Z | A, s, CS, *keys)                                          # noqa: E731
    parts = lambda: ctx.transform_parts(Z | A, s, CS, 5 * MIB, np.zeros(32, np.uint8), True, None, *keys)   # noqa: E731
    launches(plain)                                                      # the slots have this key's tables
    off0 = launches(plain)
    on = launches(parts)
    off1 = launches(plain)
    assert off0 == off1 and on > off0, (off0, on, off1)
    ctx.profile_enable(True)
    plain()
    names = ctx.profile_report()
    ctx.profile_enable(False)
    assert names and not any(k.startswith("pcrc_") for k in names), names
