"""Drives tsgpu_rewrite_object over a stored object the way an operator tool does: windows of chunks in object order with one
cursor, an empty last window when the object ends with a full one, new IVs per window.  Shared by tests/test_simt_rewrite.py,
tests/simt/asan_rewrite.py and tests/test_gpu_rewrite.py."""
import numpy as np

from tsgpu import binding
from oracle import oracle as ora

NEW_AAD = b"segment-key-2"


def new_key_material(n_chunks, seed=7):
    """(key, aad, ivs) of the new object: a key unlike corpus.fixed_key_material's and seeded random IVs"""
    rng = np.random.default_rng(seed)
    return rng.bytes(32), NEW_AAD, rng.bytes(12 * max(n_chunks, 1))


def rewrite_windows(c, from_flags, obj, sizes, ocs, ofs, to_flags, part_size, win=None, from_key=None, from_aad=b"",
                    to_key=None, to_aad=b"", to_ivs=None):
    """(new object, [new sizes], [part CRC-32C], (source, object, segment) CRC-32C) of `obj` (transformed chunks `sizes` back to
    back) rewritten in windows of `win` chunks (None: one call)"""
    sizes = [int(x) for x in sizes]
    if win is None:
        return c.rewrite_object(from_flags, obj, sizes, ocs, ofs, to_flags, part_size, from_key=from_key, from_aad=from_aad,
                                to_key=to_key, to_aad=to_aad, to_ivs=to_ivs)
    cur = np.zeros(binding.REWRITE_CURSOR_SIZE, np.uint8)
    out, new_sizes, parts = [], [], []
    pos, k = 0, 0
    while True:
        part = sizes[k:k + win]
        n = sum(part)
        end = len(part) < win
        ivs = to_ivs[12 * k:12 * (k + len(part))] if to_ivs is not None else None
        b, s, p, crc3 = c.rewrite_object(from_flags, obj[pos:pos + n], part, ocs, ofs, to_flags, part_size, cur, end, from_key,
                                         from_aad, to_key, to_aad, ivs)
        out.append(b.copy())
        new_sizes += s
        parts += p
        if end:
            return np.concatenate(out) if out else np.zeros(0, np.uint8), new_sizes, parts, crc3
        pos += n
        k += win


def frames(flags, obj, sizes, key=None, aad=b""):
    """the zstd frames of an object with ZSTD, decrypted when it has AES"""
    out, pos = [], 0
    for t in sizes:
        ch = obj[pos:pos + t]
        out.append(ora.aesgcm_decrypt_chunk(key, aad, ch) if flags & 2 else bytes(ch))
        pos += t
    return out
