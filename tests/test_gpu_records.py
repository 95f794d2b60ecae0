"""TSGPU_FLAG_VALIDATE_RECORDS on an H100: 1 GiB generated Kafka segments (v2 batches from 61 bytes to more than 4 MiB, legacy
entries) in 4 MiB chunks pass in both zstd modes with and without AES and the checksum, and transform to the flag-off objects
(dense mode and AES alone byte for byte; speed mode read back by libzstd + OpenSSL); sampled damages fail at the CPU oracle's
position; without the flag no record kernel runs."""
import os
import re
import sys

import numpy as np
import pytest

import tsgpu
from tsgpu import binding, corpus
from oracle import oracle as ora

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import records_util as R  # noqa: E402

pytestmark = pytest.mark.gpu
Z, A, D, C, VR = tsgpu.FLAG_ZSTD, tsgpu.FLAG_AES, tsgpu.FLAG_ZSTD_DENSE, tsgpu.FLAG_ZSTD_CHECKSUM, tsgpu.FLAG_VALIDATE_RECORDS
CS = 4 << 20
GIB = 1 << 30


@pytest.fixture(scope="module")
def ctx():
    c = tsgpu.Context(max_chunk_bytes=CS, max_batch=4)
    yield c
    c.close()


@pytest.fixture(scope="module")
def seg():
    return R.gen_segment(11, GIB, payload=corpus.gen_segment("K", 11, 64 << 20, 1 << 20), big=(4 << 20) + (1 << 19))


def _keys(s):
    return corpus.fixed_key_material((s.size + CS - 1) // CS)


@pytest.mark.parametrize("flags", [Z, Z | D, A, Z | A, Z | D | A, Z | C, Z | D | A | C], ids=["Z", "ZD", "A", "ZA", "ZDA", "ZC", "ZDAC"])
def test_valid_gib_segment(ctx, seg, flags):
    assert np.diff(np.append(R.starts(seg), seg.size)).max() > CS
    key, aad, ivs = _keys(seg)
    out, sizes = ctx.transform(flags | VR, seg, CS, key, aad, ivs)
    out = out.copy()
    if flags & D or not flags & Z:                       # deterministic writers: the flag-off object byte for byte
        plain, psizes = ctx.transform(flags, seg, CS, key, aad, ivs)
        assert sizes == psizes and np.array_equal(out, plain)
    else:                                                # speed mode: libzstd + OpenSSL read sampled chunks back
        pos = np.concatenate([[0], np.cumsum(sizes)])
        for i in (0, 1, len(sizes) // 2, len(sizes) - 1):
            ch = out[pos[i]:pos[i + 1]]
            fr = ora.aesgcm_decrypt_chunk(key, aad, ch) if flags & A else ch
            assert np.array_equal(np.frombuffer(ora.zstd_decompress_chunk(fr), np.uint8), seg[i * CS:(i + 1) * CS]), i


def test_sampled_damage(ctx, seg):
    rng = np.random.default_rng(5)
    st = R.starts(seg)
    for how in ("payload", "crc", "magic", "size", "payload", "crc"):
        e = int(rng.integers(0, len(st)))
        x = int(st[e])
        end = int(st[e + 1]) if e + 1 < len(st) else seg.size
        covered = x + (21 if seg[x + 16] == 2 else 16)                    # the CRC covers [covered, end)
        at = {"payload": covered + (end - covered) // 2, "crc": x + (17 if seg[x + 16] == 2 else 12), "magic": x + 16,
              "size": x + 11}[how]
        seg[at] ^= 0x10
        try:
            want = R.walk(seg)
            with pytest.raises(tsgpu.TsgpuError) as ei:
                ctx.transform(Z | A | VR, seg, CS, *_keys(seg))
            assert ei.value.code == binding.E_RECORDS
            assert re.search(r"segment position %d\b" % want[0], str(ei.value)) and "check: %s" % want[1] in str(ei.value), (want, str(ei.value))
        finally:
            seg[at] ^= 0x10


def test_cursor_windows_of_32_chunks(ctx, seg):
    whole, wsizes = ctx.transform(Z | D | VR, seg, CS)
    whole = whole.copy()
    cur = np.zeros(binding.CURSOR_SIZE, np.uint8)
    outs, sizes, w = [], [], 32 * CS
    for lo in range(0, seg.size, w):
        o, z = ctx.transform_cursor(Z | D | VR, seg[lo:lo + w], CS, cur, lo + w >= seg.size)
        outs.append(o.copy()); sizes += z
    assert sizes == wsizes and np.array_equal(np.concatenate(outs), whole)


def test_launches_without_the_flag_are_unchanged(ctx, seg):
    """a flag-off call launches what it did before any validated call, and no record kernel"""
    st = R.starts(seg)
    part = seg[:int(st[np.searchsorted(st, 64 << 20, "right") - 1])]     # whole entries: a valid segment of ~64 MiB
    keys = _keys(part)

    def launches(flags):
        before = ctx.launch_count()
        ctx.transform(flags, part, CS, *keys)
        return ctx.launch_count() - before
    launches(Z | A)                                                      # the slots have this key's tables
    off0 = launches(Z | A)
    on = launches(Z | A | VR)
    off1 = launches(Z | A)
    assert off0 == off1 and on > off0, (off0, on, off1)
    ctx.profile_enable(True)
    ctx.transform(Z | A, part, CS, *keys)
    names = ctx.profile_report()
    ctx.profile_enable(False)
    assert names and not any(k.startswith("rec_") for k in names), names
