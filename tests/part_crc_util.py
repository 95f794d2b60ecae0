"""CPU oracle of tsgpu_transform_parts: the CRC-32C restatement of host/segment_upload.hpp applied to every part of the
returned object and to the whole object (tests/cpp/crc32c_oracle.cpp, built on first use)."""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpp", "crc32c_oracle.cpp")
_LIB = os.path.join(ROOT, "tests", "cpp", "libcrc32c_oracle.so")
_HDR = os.path.join(ROOT, "tiered-storage-for-apache-kafka_b200", "host", "segment_upload.hpp")
_lib = None


def _oracle():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(_SRC), os.path.getmtime(_HDR)):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", _LIB, _SRC])
        L = C.CDLL(_LIB)
        L.pc_crc32c.restype = C.c_uint32
        L.pc_crc32c.argtypes = [C.c_void_p, C.c_uint64]
        L.pc_parts.restype = C.c_uint64
        L.pc_parts.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
        _lib = L
    return _lib


def _arr(b):
    return np.ascontiguousarray(np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray)) else b, dtype=np.uint8).reshape(-1)


def crc32c(b):
    a = _arr(b)
    return int(_oracle().pc_crc32c(a.ctypes.data if a.size else None, a.size))


def part_crcs(b, part_size):
    """[crc32c(b[k*P:(k+1)*P]) for every part k]"""
    a = _arr(b)
    out = np.zeros(max((a.size + part_size - 1) // part_size, 1), np.uint32)
    k = _oracle().pc_parts(a.ctypes.data if a.size else None, a.size, part_size, out.ctypes.data)
    return [int(x) for x in out[:k]]
