"""Kafka log segments for the TSGPU_FLAG_VALIDATE_RECORDS tests: a seeded generator of real record-formatted segments and the
CPU oracle that walks every entry (tests/cpp/records_oracle.cpp, the restatement of host/segment_upload.hpp, built on first use).

A generated segment mixes v2 record batches (61 bytes up to `big` bytes, the compression attribute bits set at random) with
legacy v0/v1 message sets; the payload bytes are drawn from corpus K (Kafka-like text) or R (random)."""
import ctypes as C
import os
import subprocess

import numpy as np

from tsgpu import corpus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(ROOT, "tests", "cpp", "records_oracle.cpp")
_LIB = os.path.join(ROOT, "tests", "cpp", "librecords_oracle.so")
_HDR = os.path.join(ROOT, "tiered-storage-for-apache-kafka_b200", "host", "segment_upload.hpp")
KINDS = {1: "length", 2: "magic", 3: "crc"}
_lib = None


def _oracle():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(_SRC), os.path.getmtime(_HDR)):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", _LIB, _SRC])
        L = C.CDLL(_LIB)
        L.rec_walk.restype = C.c_int64
        L.rec_walk.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(C.c_int), C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
        L.rec_seal.argtypes = [C.c_void_p, C.c_uint64]
        L.rec_starts.restype = C.c_uint64
        L.rec_starts.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
        _lib = L
    return _lib


def walk(seg):
    """None for a valid segment, else (position of the first invalid entry, 'length' | 'magic' | 'crc', stored, computed)"""
    s = np.ascontiguousarray(seg, dtype=np.uint8)
    k, st, co = C.c_int(0), C.c_uint32(0), C.c_uint32(0)
    at = _oracle().rec_walk(s.ctypes.data, s.size, C.byref(k), C.byref(st), C.byref(co))
    return None if at < 0 else (int(at), KINDS[k.value], int(st.value), int(co.value))


def seal(seg):
    """writes the right CRC into every entry of `seg` (in place)"""
    _oracle().rec_seal(seg.ctypes.data, seg.size)


def starts(seg):
    """start position of every entry (np.uint64)"""
    n = int(_oracle().rec_starts(seg.ctypes.data, seg.size, None, 0))
    out = np.zeros(max(n, 1), np.uint64)
    _oracle().rec_starts(seg.ctypes.data, seg.size, out.ctypes.data, n)
    return out[:n]


def entry_lengths(rng, size, small=61, big=1 << 16, legacy=0.1):
    """entry lengths (12 + size) summing to `size` bytes or a little more, and the magic of each entry"""
    mean = (big - small) / max(np.log(big / small), 1e-9) if big > small else small
    lens, mags, total = [], [], 0
    while total < size:
        n = int((size - total) / (legacy * 1000 + (1 - legacy) * mean)) + 16
        leg = rng.random(n) < legacy
        L = np.where(leg, rng.integers(26, 2048, n), np.maximum(61, np.exp(rng.uniform(np.log(small), np.log(big), n)).astype(np.int64)))
        M = np.where(leg, rng.integers(0, 2, n), 2).astype(np.uint8)
        lens.append(L); mags.append(M); total += int(L.sum())
    L, M = np.concatenate(lens), np.concatenate(mags)
    k = int(np.searchsorted(np.cumsum(L), size)) + 1
    return L[:k].astype(np.int64), M[:k]


def gen_segment(seed, size, kind="K", small=61, big=1 << 16, legacy=0.1, payload=None):
    """a valid Kafka log segment of at least `size` bytes (it ends at an entry boundary); `payload`: bytes to draw the
    payloads from instead of corpus `kind` (tiled as needed)"""
    rng = np.random.default_rng(0x7EC0 + seed)
    L, M = entry_lengths(rng, size, small, big, legacy)
    n = int(L.sum())
    if payload is None:
        seg = corpus.gen_segment(kind, 40 + seed, n, 1 << 20).copy()
    else:
        seg = np.resize(np.asarray(payload, np.uint8), n)
    pos = np.concatenate([[0], np.cumsum(L)[:-1]]).astype(np.int64)
    be = lambda v, w: ((np.asarray(v, np.uint64)[:, None] >> (8 * np.arange(w - 1, -1, -1, dtype=np.uint64))) & 0xFF).astype(np.uint8)
    idx = lambda off, w: pos[:, None] + off + np.arange(w)
    seg[idx(0, 8)] = be(np.arange(len(L)) * 7 + 1000, 8)                       # offset
    seg[idx(8, 4)] = be(L - 12, 4)                                            # size
    seg[pos + 16] = M                                                          # magic
    v2, v0 = M == 2, M != 2
    seg[idx(12, 4)[v2]] = be(np.full(v2.sum(), 5), 4)                          # v2: partitionLeaderEpoch
    attr = rng.integers(0, 256, len(L)).astype(np.uint8)                       # compression codec bits at random
    seg[(pos + 22)[v2]] = attr[v2]
    seg[(pos + 21)[v2]] = 0
    seg[(pos + 17)[v0]] = attr[v0]                                             # v0/v1: attributes i8
    seal(seg)
    assert walk(seg) is None
    return seg
