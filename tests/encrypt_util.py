"""Drives tsgpu_encrypt_object over a stored object the way an operator tool does (windows of chunks in object order with one
cursor, an empty last window when the object ends with a full one), and states what the new object must be with the oracle
(OpenSSL): every non-empty chunk encrypted as it is, an empty chunk staying empty.  Shared by tests/test_simt_encrypt.py,
tests/simt/asan_encrypt.py and tests/test_gpu_encrypt.py."""
import numpy as np

from tsgpu import binding
from oracle import oracle as ora


def encrypt_windows(c, obj, sizes, key, ivs, part_size, win=None, ocs=0, ofs=0, aad=b"", flags=0, crc64=False):
    """(new object, [new sizes], [part CRCs], (source, object) CRC) of `obj` (chunks `sizes` back to back) encrypted in windows
    of `win` chunks (None: one call)"""
    fn = c.encrypt_object_crc64 if crc64 else c.encrypt_object
    sizes = [int(x) for x in sizes]
    if win is None:
        out, nsz, parts, crc2 = fn(obj, sizes, key, ivs, part_size, ocs, ofs, aad, flags)
        return out.copy(), nsz, parts, crc2
    cur = np.zeros(binding.ENCRYPT_CURSOR_SIZE, np.uint8)
    out, nsz, parts = [], [], []
    pos, k = 0, 0
    while True:
        part = sizes[k:k + win]
        n = sum(part)
        end = len(part) < win
        b, s, p, crc2 = fn(obj[pos:pos + n], part, key, ivs[12 * k:12 * (k + len(part))], part_size, ocs, ofs, aad, flags, cur, end)
        out.append(b.copy())
        nsz += s
        parts += p
        if end:
            return np.concatenate(out), nsz, parts, crc2
        pos += n
        k += win


def expected(obj, sizes, key, aad, ivs):
    """the oracle's encrypted object: aesgcm_encrypt_chunk(key, iv_i, aad, chunk_i) for every non-empty chunk, and its sizes"""
    out, nsz, pos = [], [], 0
    for i, t in enumerate(int(x) for x in sizes):
        ch = bytes(obj[pos:pos + t])
        pos += t
        if t:
            out.append(ora.aesgcm_encrypt_chunk(key, bytes(ivs[12 * i:12 * i + 12]), aad, ch))
        nsz.append(t + 28 if t else 0)
    return np.frombuffer(b"".join(out), np.uint8), nsz
