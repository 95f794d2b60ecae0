"""Drives tsgpu_check_object over a stored object the way an operator tool does: windows of chunks in object order with one
cursor, an empty last window when the object ends with a full one.  Shared by tests/test_simt_check.py and
tests/test_gpu_check.py."""
import numpy as np

from tsgpu import binding


def check_windows(c, flags, obj, sizes, ocs, ofs, win=None, key=None, aad=b""):
    """(object CRC-32C, segment CRC-32C) of `obj` (transformed chunks `sizes` back to back) checked in windows of `win` chunks
    (None: one call)"""
    sizes = [int(x) for x in sizes]
    if win is None:
        return c.check_object(flags, obj, sizes, ocs, ofs, key=key, aad=aad)
    cur = np.zeros(binding.CHECK_CURSOR_SIZE, np.uint8)
    pos, k = 0, 0
    while True:
        part = sizes[k:k + win]
        n = sum(part)
        end = len(part) < win
        got = c.check_object(flags, obj[pos:pos + n], part, ocs, ofs, cur, end, key, aad)
        if end:
            return got
        pos += n
        k += win
