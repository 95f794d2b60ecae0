"""Drives tsgpu_rekey_object over a stored object the way an operator tool does (windows of chunks in object order with one cursor,
an empty last window when the object ends with a full one), and states what the new object must be with the oracle (OpenSSL):
every chunk decrypted under the old key and encrypted under the new one.  Shared by tests/test_simt_rekey.py,
tests/simt/asan_rekey.py and tests/test_gpu_rekey.py."""
import numpy as np

from tsgpu import binding
from oracle import oracle as ora


def rekey_windows(c, obj, sizes, from_key, to_key, to_ivs, part_size, win=None, from_aad=b"", to_aad=b"", flags=0, crc64=False):
    """(new object, [part CRCs], (source, object) CRC) of `obj` (chunks `sizes` back to back) rekeyed in windows of `win` chunks
    (None: one call)"""
    fn = c.rekey_object_crc64 if crc64 else c.rekey_object
    sizes = [int(x) for x in sizes]
    if win is None:
        out, parts, crc2 = fn(obj, sizes, from_key, to_key, to_ivs, part_size, from_aad, to_aad, flags)
        return out.copy(), parts, crc2
    cur = np.zeros(binding.REKEY_CURSOR_SIZE, np.uint8)
    out, parts = [], []
    pos, k = 0, 0
    while True:
        part = sizes[k:k + win]
        n = sum(part)
        end = len(part) < win
        b, p, crc2 = fn(obj[pos:pos + n], part, from_key, to_key, to_ivs[12 * k:12 * (k + len(part))], part_size, from_aad, to_aad,
                        flags, cur, end)
        out.append(b.copy())
        parts += p
        if end:
            return np.concatenate(out), parts, crc2
        pos += n
        k += win


def expected(obj, sizes, from_key, from_aad, to_key, to_aad, to_ivs):
    """the oracle's rekeyed object: aesgcm_encrypt_chunk(to_key, iv_i, to_aad, aesgcm_decrypt_chunk(from_key, from_aad, chunk_i)),
    an empty chunk staying empty"""
    out, pos = [], 0
    for i, t in enumerate(int(x) for x in sizes):
        ch = bytes(obj[pos:pos + t])
        pos += t
        if t:
            out.append(ora.aesgcm_encrypt_chunk(to_key, to_ivs[12 * i:12 * i + 12], to_aad, ora.aesgcm_decrypt_chunk(from_key, from_aad, ch)))
    return np.frombuffer(b"".join(out), np.uint8)


def encrypt_chunks(key, aad, plain_chunks, seed=3):
    """an object of AES chunks (IV || CT || TAG) of the given plaintexts under random IVs; None gives an empty chunk (an empty
    index blob), b"" a chunk of IV and tag only"""
    rng = np.random.default_rng(seed)
    chunks = [b"" if p is None else ora.aesgcm_encrypt_chunk(key, rng.bytes(12), aad, p) for p in plain_chunks]
    return np.frombuffer(b"".join(chunks), np.uint8).copy(), [len(c) for c in chunks]
