"""CPU oracle of the CRC-64/NVME calls: the catalogue CRC (tests/cpp/crc64_oracle.cpp, built on first use) of every part of the
returned object and of the whole object, and a bitwise Python restatement that the oracle itself is tested against."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpp", "crc64_oracle.cpp")
_LIB = os.path.join(ROOT, "tests", "cpp", "libcrc64_oracle.so")
_lib = None
POLY = 0x9A6C9329AC4BC9B5                      # reflected; 0xAD93D23594C93659 in normal form
CHECK = 0xAE8B14860A799888                     # crc64nvme(b"123456789")


def _oracle():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < os.path.getmtime(_SRC):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", _LIB, _SRC])
        L = C.CDLL(_LIB)
        L.pc_crc64nvme.restype = C.c_uint64
        L.pc_crc64nvme.argtypes = [C.c_void_p, C.c_uint64]
        L.pc_parts64.restype = C.c_uint64
        L.pc_parts64.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def _arr(b):
    return np.ascontiguousarray(np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray)) else b, dtype=np.uint8).reshape(-1)


def crc64nvme(b):
    a = _arr(b)
    return int(_oracle().pc_crc64nvme(a.ctypes.data if a.size else None, a.size))


def part_crcs(b, part_size):
    """[crc64nvme(b[k*P:(k+1)*P]) for every part k]"""
    a = _arr(b)
    out = np.zeros(max((a.size + part_size - 1) // part_size, 1), np.uint64)
    k = _oracle().pc_parts64(a.ctypes.data if a.size else None, a.size, part_size, out.ctypes.data)
    return [int(x) for x in out[:k]]


def crc64nvme_bitwise(b):
    """The definition, one bit at a time (slow: short inputs only)."""
    c = (1 << 64) - 1
    for x in bytes(_arr(b)):
        c ^= x
        for _ in range(8):
            c = (c >> 1) ^ (POLY if c & 1 else 0)
    return c ^ ((1 << 64) - 1)
