"""ctypes binding of the C-ABI in include/tsgpu.h (libtsgpu.so, built in-tree by `make` / __graft_entry__.build()).

This is the same surface a JNI shim binds (INTEGRATION.md).  There is no CPU fallback: if the CUDA library
is missing or no device is visible, construction fails loudly.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libtsgpu.so")

FLAG_ZSTD = 1
FLAG_AES = 2
FLAG_ZSTD_DENSE = 4
FLAG_VERIFY = 8          # host-buffer transforms: read each batch back on the device before releasing it
FLAG_ZSTD_CHECKSUM = 16  # with FLAG_ZSTD: every frame ends with its Content_Checksum (XXH64 of the chunk, checked by every reader)
FLAG_VALIDATE_RECORDS = 32  # segment transforms with ZSTD or AES: check every Kafka record batch's length, magic and CRC first
FLAG_REFRAME = 64        # rewrite_object to_flags: seal (ZSTD_CHECKSUM) or re-encode (ZSTD_DENSE) the kept source frames
IV_SIZE = 12
TAG_SIZE = 16
SLOT_HEAD = 4
OK, E_ARG, E_STATE, E_AUTH, E_CORRUPT, E_SHORT, E_NODEVICE, E_CUDA, E_NOMEM = 0, -1, -2, -3, -4, -5, -6, -7, -8
E_VERIFY = -9
E_RECORDS = -10
CURSOR_SIZE = 64         # tsgpu_records_cursor
PARTS_CURSOR_SIZE = 32   # tsgpu_parts_cursor
CHECK_CURSOR_SIZE = 128  # tsgpu_check_cursor
REWRITE_CURSOR_SIZE = 192  # tsgpu_rewrite_cursor
REKEY_CURSOR_SIZE = 64   # tsgpu_rekey_cursor
ENCRYPT_CURSOR_SIZE = 64  # tsgpu_encrypt_cursor

SYMBOLS = [
    "tsgpu_last_error", "tsgpu_version", "tsgpu_create", "tsgpu_destroy", "tsgpu_host_alloc", "tsgpu_host_free",
    "tsgpu_transform_bound", "tsgpu_transform", "tsgpu_transform_chunks", "tsgpu_detransform", "tsgpu_slot_stride",
    "tsgpu_transform_device", "tsgpu_detransform_device", "tsgpu_launch_count", "tsgpu_chunk_positions",
    "tsgpu_chunk_sizes_encode", "tsgpu_chunk_sizes_decode", "tsgpu_transformed_chunks_serialize",
    "tsgpu_transformed_chunks_deserialize", "tsgpu_chunk_index_json", "tsgpu_profile_enable", "tsgpu_profile_report",
    "tsgpu_decode_path_stats", "tsgpu_transformed_chunks_serialize_ctx", "tsgpu_chunk_index_json_ctx",
    "tsgpu_transform_cursor", "tsgpu_transform_parts", "tsgpu_check_object", "tsgpu_rewrite_object",
    "tsgpu_transform_parts_crc64", "tsgpu_check_object_crc64", "tsgpu_rewrite_object_crc64",
    "tsgpu_rekey_object", "tsgpu_rekey_object_crc64", "tsgpu_encrypt_object", "tsgpu_encrypt_object_crc64",
]


class TsgpuError(RuntimeError):
    """Maps to the unchecked RuntimeException the reference's operators throw (SURVEY.md §8b)."""

    def __init__(self, code, msg):
        super().__init__(msg)
        self.code = code


_libs = {}


def load(path=None):
    path = path or os.environ.get("TSGPU_LIB") or DEFAULT_LIB
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise TsgpuError(E_NODEVICE, "libtsgpu.so not built at %s (run `make` or __graft_entry__.build()); "
                                     "there is no CPU fallback" % path)
    L = C.CDLL(path)
    vp, u32, u64, i32 = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32
    L.tsgpu_last_error.restype = C.c_char_p
    L.tsgpu_version.restype = C.c_char_p
    L.tsgpu_create.argtypes = [vp, C.c_int, u32, u32, C.POINTER(vp)]
    L.tsgpu_destroy.argtypes = [vp]
    L.tsgpu_host_alloc.restype = vp
    L.tsgpu_host_alloc.argtypes = [C.c_size_t]
    L.tsgpu_host_free.argtypes = [vp]
    L.tsgpu_transform_bound.restype = u64
    L.tsgpu_transform_bound.argtypes = [u32, u64, u32]
    L.tsgpu_slot_stride.restype = u64
    L.tsgpu_slot_stride.argtypes = [u32, u32]
    L.tsgpu_transform.argtypes = [vp, u32, vp, u64, u32, vp, vp, u32, vp, vp, u64, vp, vp]
    L.tsgpu_transform_cursor.argtypes = [vp, u32, vp, u64, u32, vp, vp, u32, vp, vp, u64, vp, vp, vp, C.c_int]
    L.tsgpu_transform_parts.argtypes = [vp, u32, vp, u64, u32, vp, vp, u32, vp, vp, u64, vp, vp, vp, C.c_int,
                                        u64, vp, vp, u32, vp, vp]
    L.tsgpu_transform_chunks.argtypes = [vp, u32, vp, vp, u32, vp, vp, u32, vp, vp, u64, vp]
    L.tsgpu_detransform.argtypes = [vp, u32, vp, u64, vp, u32, vp, vp, u32, vp, u64, vp]
    L.tsgpu_check_object.argtypes = [vp, u32, vp, u64, vp, u32, u32, u64, vp, vp, u32, vp, C.c_int, vp, vp]
    L.tsgpu_rewrite_object.argtypes = [vp, u32, vp, u64, vp, u32, u32, u64, vp, vp, u32, u32, vp, vp, u32, vp, vp, u64, vp,
                                       u64, vp, u32, vp, vp, C.c_int, vp, vp, vp]
    L.tsgpu_transform_parts_crc64.argtypes = L.tsgpu_transform_parts.argtypes
    L.tsgpu_check_object_crc64.argtypes = L.tsgpu_check_object.argtypes
    L.tsgpu_rewrite_object_crc64.argtypes = L.tsgpu_rewrite_object.argtypes
    L.tsgpu_rekey_object.argtypes = [vp, u32, vp, u64, vp, u32, vp, vp, u32, vp, vp, u32, vp, vp, u64, u64, vp, u32, vp, vp,
                                     C.c_int, vp, vp]
    L.tsgpu_rekey_object_crc64.argtypes = L.tsgpu_rekey_object.argtypes
    L.tsgpu_encrypt_object.argtypes = [vp, u32, vp, u64, vp, u32, u32, u64, vp, vp, u32, vp, vp, u64, vp, u64, vp, u32, vp, vp,
                                       C.c_int, vp, vp]
    L.tsgpu_encrypt_object_crc64.argtypes = L.tsgpu_encrypt_object.argtypes
    L.tsgpu_transform_device.argtypes = [vp, C.c_int, u32, vp, u64, u32, vp, vp, u32, vp, vp, u64, vp, vp]
    L.tsgpu_detransform_device.argtypes = [vp, C.c_int, u32, vp, u64, vp, u32, u32, vp, vp, u32, vp, vp, vp, vp]
    L.tsgpu_launch_count.restype = u64
    L.tsgpu_launch_count.argtypes = [vp]
    L.tsgpu_decode_path_stats.argtypes = [vp, vp]
    L.tsgpu_profile_enable.argtypes = [vp, C.c_int]
    L.tsgpu_profile_report.argtypes = [vp, C.c_char_p, C.POINTER(u32)]
    L.tsgpu_chunk_positions.argtypes = [vp, vp, u32, vp]
    L.tsgpu_chunk_sizes_encode.argtypes = [vp, u32, vp, C.POINTER(u32)]
    L.tsgpu_chunk_sizes_decode.argtypes = [vp, u32, vp, C.POINTER(u32)]
    L.tsgpu_transformed_chunks_serialize.argtypes = [vp, u32, C.c_char_p, C.POINTER(u32)]
    L.tsgpu_transformed_chunks_deserialize.argtypes = [vp, C.c_char_p, vp, C.POINTER(u32)]
    L.tsgpu_chunk_index_json.argtypes = [i32, i32, i32, i32, vp, u32, C.c_char_p, C.POINTER(u32)]
    L.tsgpu_transformed_chunks_serialize_ctx.argtypes = [vp, vp, u32, C.c_char_p, C.POINTER(u32)]
    L.tsgpu_chunk_index_json_ctx.argtypes = [vp, i32, i32, i32, i32, vp, u32, C.c_char_p, C.POINTER(u32)]
    _libs[path] = L
    return L


def _u8(b):
    if b is None:
        return np.zeros(0, np.uint8)
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b).view(np.uint8).reshape(-1)
    return np.frombuffer(bytes(b), dtype=np.uint8)


def _p(a):
    return a.ctypes.data if a is not None and a.size else None


def _np_word(word):
    return np.uint64 if word is C.c_uint64 else np.uint32


class Context:
    """tsgpu_ctx: one per process (JVM); thread-safe."""

    def __init__(self, max_chunk_bytes, max_batch=32, devices=None, lib_path=None):
        self.lib = load(lib_path)
        self._h = C.c_void_p()
        ids = (C.c_int * len(devices))(*devices) if devices else None
        rc = self.lib.tsgpu_create(ids, len(devices) if devices else 0, max_chunk_bytes, max_batch, C.byref(self._h))
        if rc:
            raise TsgpuError(rc, self.lib.tsgpu_last_error().decode())
        self.max_chunk_bytes = max_chunk_bytes
        self.max_batch = max_batch

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self.lib.tsgpu_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc:
            raise TsgpuError(rc, self.lib.tsgpu_last_error().decode())

    @property
    def handle(self):
        return self._h

    def launch_count(self):
        return int(self.lib.tsgpu_launch_count(self._h))

    def decode_path_stats(self):
        """{'regions': n, 'region_fallback_frames': n, 'whole_frames': n, 'serial_frames': n, 'blocks': n} since the context was created"""
        v = (C.c_uint64 * 8)()
        self._check(self.lib.tsgpu_decode_path_stats(self._h, v))
        return dict(zip(("regions", "region_fallback_frames", "whole_frames", "serial_frames", "blocks"), [int(x) for x in v]))

    def profile_enable(self, on=True):
        self._check(self.lib.tsgpu_profile_enable(self._h, 1 if on else 0))

    def profile_report(self):
        import json
        buf = C.create_string_buffer(1 << 16)
        n = C.c_uint32(len(buf))
        self._check(self.lib.tsgpu_profile_report(self._h, buf, C.byref(n)))
        return json.loads(buf.value.decode())

    # ---- host-buffer API (what the JNI shim calls) ----
    def transform(self, flags, src, chunk_size, key=None, aad=b"", ivs=None, dst=None):
        """Returns (np.uint8 view of the transformed bytes, [transformed sizes])."""
        s = _u8(src)
        cs = chunk_size if chunk_size else max(s.size, 1)
        n_max = (s.size + cs - 1) // cs + 1
        cap = int(self.lib.tsgpu_transform_bound(flags, s.size, chunk_size)) + 64
        if dst is None:
            dst = np.empty(cap, dtype=np.uint8)
        sizes = np.zeros(n_max, dtype=np.uint32)
        n = C.c_uint32(n_max)
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(self.lib.tsgpu_transform(self._h, flags, _p(s), s.size, chunk_size, _p(k), _p(a), a.size, _p(iv),
                                             dst.ctypes.data, dst.size, sizes.ctypes.data, C.addressof(n)))
        sizes = sizes[:n.value]
        return dst[:int(sizes.sum(dtype=np.uint64))], [int(x) for x in sizes]

    def transform_cursor(self, flags, src, chunk_size, cursor, segment_ends_here, key=None, aad=b"", ivs=None):
        """One window of a segment with FLAG_VALIDATE_RECORDS: `cursor` is a 64-byte np.uint8 array (zeros at the start of the
        segment), updated in place on success.  Returns (transformed bytes, [transformed sizes])."""
        s = _u8(src)
        if not (isinstance(cursor, np.ndarray) and cursor.dtype == np.uint8 and cursor.size == CURSOR_SIZE and cursor.flags.c_contiguous):
            raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % CURSOR_SIZE)
        cs = chunk_size if chunk_size else max(s.size, 1)
        n_max = (s.size + cs - 1) // cs + 1
        dst = np.empty(int(self.lib.tsgpu_transform_bound(flags, s.size, chunk_size)) + 64, dtype=np.uint8)
        sizes = np.zeros(n_max, dtype=np.uint32)
        n = C.c_uint32(n_max)
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(self.lib.tsgpu_transform_cursor(self._h, flags, _p(s), s.size, chunk_size, _p(k), _p(a), a.size, _p(iv),
                                                    dst.ctypes.data, dst.size, sizes.ctypes.data, C.addressof(n),
                                                    cursor.ctypes.data, 1 if segment_ends_here else 0))
        sizes = sizes[:n.value]
        return dst[:int(sizes.sum(dtype=np.uint64))], [int(x) for x in sizes]

    def transform_parts(self, flags, src, chunk_size, part_size, parts_cursor, segment_ends_here, records_cursor=None,
                        key=None, aad=b"", ivs=None, part_cap=None):
        """One window of a segment with the CRC-32C of its upload parts: `parts_cursor` is a 32-byte np.uint8 array (zeros at the
        start of the object), updated in place on success; `records_cursor` a 64-byte one as transform_cursor takes (needed with
        FLAG_VALIDATE_RECORDS).  Returns (transformed bytes, [transformed sizes], [CRC-32C of the parts this call completed],
        CRC-32C of the whole object or None when the segment does not end here)."""
        return self._transform_parts(self.lib.tsgpu_transform_parts, C.c_uint32, flags, src, chunk_size, part_size, parts_cursor,
                                     segment_ends_here, records_cursor, key, aad, ivs, part_cap)

    def transform_parts_crc64(self, flags, src, chunk_size, part_size, parts_cursor, segment_ends_here, records_cursor=None,
                              key=None, aad=b"", ivs=None, part_cap=None):
        """transform_parts with CRC-64/NVME part and object checksums (tsgpu_transform_parts_crc64): the same bytes and sizes,
        the checksums as ints below 2**64.  A parts cursor carries one width: start and continue it with the same method."""
        return self._transform_parts(self.lib.tsgpu_transform_parts_crc64, C.c_uint64, flags, src, chunk_size, part_size,
                                     parts_cursor, segment_ends_here, records_cursor, key, aad, ivs, part_cap)

    def _transform_parts(self, fn, word, flags, src, chunk_size, part_size, parts_cursor, segment_ends_here, records_cursor,
                         key, aad, ivs, part_cap):
        s = _u8(src)
        for cur, size in ((parts_cursor, PARTS_CURSOR_SIZE), (records_cursor, CURSOR_SIZE)):
            if cur is not None and not (isinstance(cur, np.ndarray) and cur.dtype == np.uint8 and cur.size == size
                                        and cur.flags.c_contiguous):
                raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % size)
        cs = chunk_size if chunk_size else max(s.size, 1)
        n_max = (s.size + cs - 1) // cs + 1
        bound = int(self.lib.tsgpu_transform_bound(flags, s.size, chunk_size)) if s.size else 0
        dst = np.empty(bound + 64, dtype=np.uint8)
        sizes = np.zeros(n_max, dtype=np.uint32)
        n = C.c_uint32(n_max)
        if part_cap is None:
            part_cap = (bound + part_size) // max(part_size, 1) + 1
        crcs = np.zeros(max(part_cap, 1), dtype=_np_word(word))
        n_parts, obj = C.c_uint32(0), word(0)
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(fn(
            self._h, flags, _p(s), s.size, chunk_size, _p(k), _p(a), a.size, _p(iv), dst.ctypes.data, dst.size,
            sizes.ctypes.data, C.addressof(n), None if records_cursor is None else records_cursor.ctypes.data,
            1 if segment_ends_here else 0, part_size, None if parts_cursor is None else parts_cursor.ctypes.data,
            crcs.ctypes.data, part_cap, C.addressof(n_parts), C.addressof(obj)))
        sizes = sizes[:n.value]
        return (dst[:int(sizes.sum(dtype=np.uint64))], [int(x) for x in sizes], [int(x) for x in crcs[:n_parts.value]],
                int(obj.value) if segment_ends_here else None)

    def transform_chunks(self, flags, src, chunk_lens, key=None, aad=b"", ivs=None):
        """Ragged chunks (e.g. the index files of a segment): returns (transformed bytes, [transformed sizes])."""
        s = _u8(src)
        lens = np.ascontiguousarray(chunk_lens, dtype=np.uint32)
        cap = int(sum(int(self.lib.tsgpu_transform_bound(flags, int(x), int(x))) for x in lens)) + 64
        dst = np.empty(cap, dtype=np.uint8)
        sizes = np.zeros(max(lens.size, 1), dtype=np.uint32)
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(self.lib.tsgpu_transform_chunks(self._h, flags, _p(s), _p(lens), lens.size, _p(k), _p(a), a.size, _p(iv),
                                                    dst.ctypes.data, dst.size, sizes.ctypes.data))
        sizes = sizes[:lens.size]
        return dst[:int(sizes.sum(dtype=np.uint64))], [int(x) for x in sizes]

    def detransform(self, flags, src, transformed_sizes, dst_cap, key=None, aad=b"", dst=None):
        """Returns (np.uint8 view of the original bytes, [original sizes])."""
        s = _u8(src)
        ts = np.ascontiguousarray(transformed_sizes, dtype=np.uint32)
        if dst is None:
            dst = np.empty(max(int(dst_cap), 1), dtype=np.uint8)
        osz = np.zeros(max(ts.size, 1), dtype=np.uint32)
        k, a = _u8(key), _u8(aad)
        self._check(self.lib.tsgpu_detransform(self._h, flags, _p(s), s.size, _p(ts), ts.size, _p(k), _p(a), a.size,
                                               dst.ctypes.data, int(dst_cap), osz.ctypes.data))
        osz = osz[:ts.size]
        return dst[:int(osz.sum(dtype=np.uint64))], [int(x) for x in osz]

    def check_object(self, flags, src, transformed_sizes, original_chunk_size, original_file_size, cursor=None,
                     object_ends_here=True, key=None, aad=b""):
        """Checks one window of a stored object against its chunk index on the GPU (tsgpu_check_object) without copying its
        plaintext back.  `cursor`: a 128-byte np.uint8 array (zeros at the start of the object), updated in place on success; None
        checks a whole object.  Returns (object CRC-32C, segment CRC-32C) when the object ends here, else None."""
        return self._check_object(self.lib.tsgpu_check_object, C.c_uint32, flags, src, transformed_sizes, original_chunk_size,
                                  original_file_size, cursor, object_ends_here, key, aad)

    def check_object_crc64(self, flags, src, transformed_sizes, original_chunk_size, original_file_size, cursor=None,
                           object_ends_here=True, key=None, aad=b""):
        """check_object with CRC-64/NVME words (tsgpu_check_object_crc64): (object CRC-64/NVME, segment CRC-64/NVME) when the
        object ends here, else None.  A cursor carries one width: start and continue it with the same method."""
        return self._check_object(self.lib.tsgpu_check_object_crc64, C.c_uint64, flags, src, transformed_sizes, original_chunk_size,
                                  original_file_size, cursor, object_ends_here, key, aad)

    def _check_object(self, fn, word, flags, src, transformed_sizes, original_chunk_size, original_file_size, cursor,
                      object_ends_here, key, aad):
        s = _u8(src)
        if cursor is None:
            cursor = np.zeros(CHECK_CURSOR_SIZE, np.uint8)
        if not (isinstance(cursor, np.ndarray) and cursor.dtype == np.uint8 and cursor.size == CHECK_CURSOR_SIZE
                and cursor.flags.c_contiguous):
            raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % CHECK_CURSOR_SIZE)
        ts = np.ascontiguousarray(transformed_sizes, dtype=np.uint32)
        obj, seg = word(0), word(0)
        k, a = _u8(key), _u8(aad)
        self._check(fn(self._h, flags, _p(s), s.size, _p(ts), ts.size, original_chunk_size,
                                                original_file_size, _p(k), _p(a), a.size, cursor.ctypes.data,
                                                1 if object_ends_here else 0, C.addressof(obj), C.addressof(seg)))
        return (int(obj.value), int(seg.value)) if object_ends_here else None

    def rewrite_object(self, from_flags, src, transformed_sizes, original_chunk_size, original_file_size, to_flags, part_size,
                       cursor=None, object_ends_here=True, from_key=None, from_aad=b"", to_key=None, to_aad=b"", to_ivs=None,
                       part_cap=None):
        """Rewrites one window of a stored object on the GPU (tsgpu_rewrite_object): checked as check_object checks it, then
        transformed with `to_flags` under `to_key` / `to_ivs` (one 12-byte IV per chunk of the window).  `cursor`: a 192-byte
        np.uint8 array (zeros at the start of the object), updated in place on success; None rewrites a whole object.  Returns
        (new bytes, [new transformed sizes], [CRC-32C of the parts this call completed], (source, object, segment) CRC-32C or None
        when the object does not end here)."""
        return self._rewrite_object(self.lib.tsgpu_rewrite_object, C.c_uint32, from_flags, src, transformed_sizes,
                                    original_chunk_size, original_file_size, to_flags, part_size, cursor, object_ends_here,
                                    from_key, from_aad, to_key, to_aad, to_ivs, part_cap)

    def rewrite_object_crc64(self, from_flags, src, transformed_sizes, original_chunk_size, original_file_size, to_flags,
                             part_size, cursor=None, object_ends_here=True, from_key=None, from_aad=b"", to_key=None, to_aad=b"",
                             to_ivs=None, part_cap=None):
        """rewrite_object with CRC-64/NVME part, source, object and segment checksums (tsgpu_rewrite_object_crc64): the same new
        bytes and sizes.  A cursor carries one width: start and continue it with the same method."""
        return self._rewrite_object(self.lib.tsgpu_rewrite_object_crc64, C.c_uint64, from_flags, src, transformed_sizes,
                                    original_chunk_size, original_file_size, to_flags, part_size, cursor, object_ends_here,
                                    from_key, from_aad, to_key, to_aad, to_ivs, part_cap)

    def _rewrite_object(self, fn, word, from_flags, src, transformed_sizes, original_chunk_size, original_file_size, to_flags,
                        part_size, cursor, object_ends_here, from_key, from_aad, to_key, to_aad, to_ivs, part_cap):
        s = _u8(src)
        if cursor is None:
            cursor = np.zeros(REWRITE_CURSOR_SIZE, np.uint8)
        if not (isinstance(cursor, np.ndarray) and cursor.dtype == np.uint8 and cursor.size == REWRITE_CURSOR_SIZE
                and cursor.flags.c_contiguous):
            raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % REWRITE_CURSOR_SIZE)
        ts = np.ascontiguousarray(transformed_sizes, dtype=np.uint32)
        n = ts.size
        # every chunk of the window at most a frame bound (or its source frame, when frames are kept) plus IV and tag
        per = int(self.lib.tsgpu_transform_bound(to_flags | FLAG_ZSTD, original_chunk_size, original_chunk_size)) + 28
        # (a frame TSGPU_FLAG_REFRAME seals is 4 bytes longer than its source frame)
        cap = max(n * per, int(ts.sum(dtype=np.uint64)) + 32 * n) + 64
        dst = np.empty(cap, dtype=np.uint8)
        sizes = np.zeros(max(n, 1), dtype=np.uint32)
        if part_cap is None:
            part_cap = (cap + part_size) // max(part_size, 1) + 1
        crcs = np.zeros(max(part_cap, 1), dtype=_np_word(word))
        n_parts, src_crc, obj_crc, seg_crc = C.c_uint32(0), word(0), word(0), word(0)
        fk, fa, tk, ta, iv = _u8(from_key), _u8(from_aad), _u8(to_key), _u8(to_aad), _u8(to_ivs)
        self._check(fn(
            self._h, from_flags, _p(s), s.size, _p(ts), n, original_chunk_size, original_file_size, _p(fk), _p(fa), fa.size,
            to_flags, _p(tk), _p(ta), ta.size, _p(iv), dst.ctypes.data, dst.size, sizes.ctypes.data, part_size,
            crcs.ctypes.data, part_cap, C.addressof(n_parts), cursor.ctypes.data, 1 if object_ends_here else 0,
            C.addressof(src_crc), C.addressof(obj_crc), C.addressof(seg_crc)))
        sizes = sizes[:n]
        crc3 = (int(src_crc.value), int(obj_crc.value), int(seg_crc.value)) if object_ends_here else None
        return dst[:int(sizes.sum(dtype=np.uint64))], [int(x) for x in sizes], [int(x) for x in crcs[:n_parts.value]], crc3

    def rekey_object(self, src, transformed_sizes, from_key, to_key, to_ivs, part_size, from_aad=b"", to_aad=b"", flags=0,
                     cursor=None, object_ends_here=True, part_cap=None, dst_cap=None):
        """Re-encrypts one window of a stored object's AES-GCM chunks under a new key with nothing decoded (tsgpu_rekey_object):
        chunk i keeps its size and gets to_ivs[i].  `flags`: 0 or FLAG_VERIFY.  `cursor`: a 64-byte np.uint8 array (zeros at
        the start of the object), updated in place on success; None rekeys a whole object.  Returns (new bytes, [CRC-32C of the
        parts this call completed], (source, object) CRC-32C or None when the object does not end here)."""
        return self._rekey_object(self.lib.tsgpu_rekey_object, C.c_uint32, src, transformed_sizes, from_key, to_key, to_ivs,
                                  part_size, from_aad, to_aad, flags, cursor, object_ends_here, part_cap, dst_cap)

    def rekey_object_crc64(self, src, transformed_sizes, from_key, to_key, to_ivs, part_size, from_aad=b"", to_aad=b"", flags=0,
                           cursor=None, object_ends_here=True, part_cap=None, dst_cap=None):
        """rekey_object with CRC-64/NVME part, source and object checksums (tsgpu_rekey_object_crc64): the same new bytes.  A
        cursor carries one width: start and continue it with the same method."""
        return self._rekey_object(self.lib.tsgpu_rekey_object_crc64, C.c_uint64, src, transformed_sizes, from_key, to_key,
                                  to_ivs, part_size, from_aad, to_aad, flags, cursor, object_ends_here, part_cap, dst_cap)

    def _rekey_object(self, fn, word, src, transformed_sizes, from_key, to_key, to_ivs, part_size, from_aad, to_aad, flags,
                      cursor, object_ends_here, part_cap, dst_cap):
        s = _u8(src)
        if cursor is None:
            cursor = np.zeros(REKEY_CURSOR_SIZE, np.uint8)
        if not (isinstance(cursor, np.ndarray) and cursor.dtype == np.uint8 and cursor.size == REKEY_CURSOR_SIZE
                and cursor.flags.c_contiguous):
            raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % REKEY_CURSOR_SIZE)
        ts = np.ascontiguousarray(transformed_sizes, dtype=np.uint32)
        total = int(ts.sum(dtype=np.uint64))
        dst = np.empty(total if dst_cap is None else dst_cap, dtype=np.uint8)
        if part_cap is None:                                 # the exact bound: (carried + window) // part_size, + 1 at the end
            part_cap = (int(np.frombuffer(cursor[:8].tobytes(), np.uint64)[0]) % max(part_size, 1) + total) // max(part_size, 1) + 1
        crcs = np.zeros(max(part_cap, 1), dtype=_np_word(word))
        n_parts, src_crc, obj_crc = C.c_uint32(0), word(0), word(0)
        fk, fa, tk, ta, iv = _u8(from_key), _u8(from_aad), _u8(to_key), _u8(to_aad), _u8(to_ivs)
        self._check(fn(
            self._h, flags, _p(s), s.size, _p(ts), ts.size, _p(fk), _p(fa), fa.size, _p(tk), _p(ta), ta.size, _p(iv),
            _p(dst), dst.size, part_size, _p(crcs), part_cap, C.addressof(n_parts), cursor.ctypes.data,
            1 if object_ends_here else 0, C.addressof(src_crc), C.addressof(obj_crc)))
        crc2 = (int(src_crc.value), int(obj_crc.value)) if object_ends_here else None
        return dst[:total], [int(x) for x in crcs[:n_parts.value]], crc2

    def encrypt_object(self, src, chunk_sizes, key, ivs, part_size, original_chunk_size=0, original_file_size=0, aad=b"",
                       flags=0, cursor=None, object_ends_here=True, part_cap=None, dst_cap=None):
        """Encrypts one window of a stored unencrypted object's chunks with nothing decoded (tsgpu_encrypt_object): chunk i
        becomes ivs[i] || AES-GCM(key, aad, chunk i) || tag, an empty chunk stays empty.  `flags`: FLAG_ZSTD for a compressed
        object, FLAG_VERIFY.  original_chunk_size / original_file_size: the chunk index of a .log object, 0 for an .indexes object.
        `cursor`: a 64-byte np.uint8 array (zeros at the start of the object), updated in place on success; None encrypts a whole
        object.  Returns (new bytes, [new sizes], [CRC-32C of the parts this call completed], (source, object) CRC-32C or None
        when the object does not end here)."""
        return self._encrypt_object(self.lib.tsgpu_encrypt_object, C.c_uint32, src, chunk_sizes, key, ivs, part_size,
                                    original_chunk_size, original_file_size, aad, flags, cursor, object_ends_here, part_cap, dst_cap)

    def encrypt_object_crc64(self, src, chunk_sizes, key, ivs, part_size, original_chunk_size=0, original_file_size=0, aad=b"",
                             flags=0, cursor=None, object_ends_here=True, part_cap=None, dst_cap=None):
        """encrypt_object with CRC-64/NVME part, source and object checksums (tsgpu_encrypt_object_crc64): the same new bytes.  A
        cursor carries one width: start and continue it with the same method."""
        return self._encrypt_object(self.lib.tsgpu_encrypt_object_crc64, C.c_uint64, src, chunk_sizes, key, ivs, part_size,
                                    original_chunk_size, original_file_size, aad, flags, cursor, object_ends_here, part_cap, dst_cap)

    def _encrypt_object(self, fn, word, src, chunk_sizes, key, ivs, part_size, original_chunk_size, original_file_size, aad, flags,
                        cursor, object_ends_here, part_cap, dst_cap):
        s = _u8(src)
        if cursor is None:
            cursor = np.zeros(ENCRYPT_CURSOR_SIZE, np.uint8)
        if not (isinstance(cursor, np.ndarray) and cursor.dtype == np.uint8 and cursor.size == ENCRYPT_CURSOR_SIZE
                and cursor.flags.c_contiguous):
            raise TypeError("cursor must be a contiguous np.uint8 array of %d bytes" % ENCRYPT_CURSOR_SIZE)
        cs = np.ascontiguousarray(chunk_sizes, dtype=np.uint32)
        total = int(sum(int(x) + 28 for x in cs if x))
        dst = np.empty(total if dst_cap is None else dst_cap, dtype=np.uint8)
        sizes = np.zeros(max(cs.size, 1), dtype=np.uint32)
        if part_cap is None:                                 # the exact bound: (carried + window) // part_size, + 1 at the end
            part_cap = (int(np.frombuffer(cursor[:8].tobytes(), np.uint64)[0]) % max(part_size, 1) + total) // max(part_size, 1) + 1
        crcs = np.zeros(max(part_cap, 1), dtype=_np_word(word))
        n_parts, src_crc, obj_crc = C.c_uint32(0), word(0), word(0)
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(fn(
            self._h, flags, _p(s), s.size, _p(cs), cs.size, original_chunk_size, original_file_size, _p(k), _p(a), a.size, _p(iv),
            _p(dst), dst.size, _p(sizes), part_size, _p(crcs), part_cap, C.addressof(n_parts), cursor.ctypes.data,
            1 if object_ends_here else 0, C.addressof(src_crc), C.addressof(obj_crc)))
        crc2 = (int(src_crc.value), int(obj_crc.value)) if object_ends_here else None
        return dst[:total], [int(x) for x in sizes[:cs.size]], [int(x) for x in crcs[:n_parts.value]], crc2

    # ---- device-resident API (raw device pointers as ints; bench.py passes torch data_ptr()) ----
    def slot_stride(self, flags, chunk_size):
        return int(self.lib.tsgpu_slot_stride(flags, chunk_size))

    def transform_device(self, flags, d_src, src_len, chunk_size, key, aad, ivs, d_slots, slot_stride, d_sizes,
                         stream=0, device_index=0):
        k, a, iv = _u8(key), _u8(aad), _u8(ivs)
        self._check(self.lib.tsgpu_transform_device(self._h, device_index, flags, d_src, src_len, chunk_size, _p(k), _p(a),
                                                    a.size, _p(iv), d_slots, slot_stride, d_sizes, stream))

    def detransform_device(self, flags, d_slots, slot_stride, d_sizes, n_chunks, chunk_size, key, aad, d_dst,
                           d_original_sizes, d_status, stream=0, device_index=0):
        k, a = _u8(key), _u8(aad)
        self._check(self.lib.tsgpu_detransform_device(self._h, device_index, flags, d_slots, slot_stride, d_sizes, n_chunks,
                                                      chunk_size, _p(k), _p(a), a.size, d_dst, d_original_sizes, d_status,
                                                      stream))

    # ---- ChunkIndex plumbing ----
    def chunk_positions(self, sizes):
        s = np.ascontiguousarray(sizes, dtype=np.uint32)
        pos = np.zeros(s.size + 1, dtype=np.uint64)
        self._check(self.lib.tsgpu_chunk_positions(self._h, _p(s), s.size, pos.ctypes.data))
        return pos

    def transformed_chunks_deserialize(self, b64, cap=1 << 22):
        out = np.zeros(cap, dtype=np.int32)
        n = C.c_uint32(cap)
        self._check(self.lib.tsgpu_transformed_chunks_deserialize(self._h, b64.encode(), out.ctypes.data, C.byref(n)))
        return [int(x) for x in out[:n.value]]

    def transformed_chunks_serialize(self, values):
        """TransformedChunksSerializer with the codec bytes compressed (dense compressor), like the reference's manifests"""
        v = np.ascontiguousarray(values, dtype=np.int32)
        buf = C.create_string_buffer(256 + 8 * v.size)
        n = C.c_uint32(len(buf))
        self._check(self.lib.tsgpu_transformed_chunks_serialize_ctx(self._h, _p(v), v.size, buf, C.byref(n)))
        return buf.value.decode()

    def chunk_index_json(self, original_chunk_size, original_file_size, transformed_chunk_size=None,
                         final_transformed_chunk_size=0, sizes=None):
        v = np.ascontiguousarray(sizes if sizes is not None else [], dtype=np.int32)
        buf = C.create_string_buffer(1024 + 8 * v.size)
        n = C.c_uint32(len(buf))
        tcs = -1 if transformed_chunk_size is None else transformed_chunk_size
        self._check(self.lib.tsgpu_chunk_index_json_ctx(self._h, original_chunk_size, original_file_size, tcs,
                                                        final_transformed_chunk_size, _p(v), v.size, buf, C.byref(n)))
        return buf.value.decode()


def _raise(L, rc):
    raise TsgpuError(rc, L.tsgpu_last_error().decode())


def chunk_sizes_encode(values, lib_path=None):
    L = load(lib_path)
    v = np.ascontiguousarray(values, dtype=np.int32)
    out = np.zeros(32 + 4 * v.size, dtype=np.uint8)
    n = C.c_uint32(out.size)
    rc = L.tsgpu_chunk_sizes_encode(_p(v), v.size, out.ctypes.data, C.byref(n))
    if rc:
        _raise(L, rc)
    return out[:n.value].tobytes()


def chunk_sizes_decode(data, cap=1 << 22, lib_path=None):
    L = load(lib_path)
    d = _u8(data)
    out = np.zeros(cap, dtype=np.int32)
    n = C.c_uint32(cap)
    rc = L.tsgpu_chunk_sizes_decode(_p(d), d.size, out.ctypes.data, C.byref(n))
    if rc:
        _raise(L, rc)
    return [int(x) for x in out[:n.value]]


def transformed_chunks_serialize(values, lib_path=None):
    L = load(lib_path)
    v = np.ascontiguousarray(values, dtype=np.int32)
    buf = C.create_string_buffer(256 + 8 * v.size)
    n = C.c_uint32(len(buf))
    rc = L.tsgpu_transformed_chunks_serialize(_p(v), v.size, buf, C.byref(n))
    if rc:
        _raise(L, rc)
    return buf.value.decode()


def chunk_index_json(original_chunk_size, original_file_size, transformed_chunk_size=None,
                     final_transformed_chunk_size=0, sizes=None, lib_path=None):
    L = load(lib_path)
    v = np.ascontiguousarray(sizes if sizes is not None else [], dtype=np.int32)
    buf = C.create_string_buffer(1024 + 8 * v.size)
    n = C.c_uint32(len(buf))
    tcs = -1 if transformed_chunk_size is None else transformed_chunk_size
    rc = L.tsgpu_chunk_index_json(original_chunk_size, original_file_size, tcs, final_transformed_chunk_size,
                                  _p(v), v.size, buf, C.byref(n))
    if rc:
        _raise(L, rc)
    return buf.value.decode()
