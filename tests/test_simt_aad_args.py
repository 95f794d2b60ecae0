"""A NULL aad with a positive aad_len is refused with TSGPU_E_ARG by the calls that used to copy from it on the host:
tsgpu_detransform, tsgpu_transform_device and tsgpu_detransform_device, on the SIMT emulator build.  Each call runs in its own
process, so a build that dereferences the NULL pointer fails this test instead of taking pytest down."""
import json
import os
import subprocess
import sys

import pytest

from tsgpu import binding

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_DRIVER = r"""
import ctypes as C, json, os, sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import tsgpu
from tsgpu import binding, corpus

CS = 4096
call = sys.argv[2]
ctx = tsgpu.Context(max_chunk_bytes=CS, max_batch=2, lib_path=os.path.join(sys.argv[1], "tests", "simt", "libtsgpu_simt.so"))
L, h = ctx.lib, ctx._h
key, _, ivs = corpus.fixed_key_material(1)
k, iv = binding._u8(key), binding._u8(ivs)
src = np.zeros(CS, np.uint8)
stride = ctx.slot_stride(tsgpu.FLAG_AES, CS)
slots = np.zeros(stride, np.uint8)
sizes = np.array([CS + 28], np.uint32)
dst = np.zeros(CS, np.uint8)
osz = np.zeros(1, np.uint32)
status = np.zeros(1, np.uint32)
A, NULL, AAD_LEN = tsgpu.FLAG_AES, None, 16
if call == "detransform":
    rc = L.tsgpu_detransform(h, A, slots.ctypes.data, slots.size, sizes.ctypes.data, 1, binding._p(k), NULL, AAD_LEN,
                             dst.ctypes.data, dst.size, osz.ctypes.data)
elif call == "transform_device":
    rc = L.tsgpu_transform_device(h, 0, A, src.ctypes.data, src.size, CS, binding._p(k), NULL, AAD_LEN, binding._p(iv),
                                  slots.ctypes.data, stride, sizes.ctypes.data, None)
else:
    rc = L.tsgpu_detransform_device(h, 0, A, slots.ctypes.data, stride, sizes.ctypes.data, 1, CS, binding._p(k), NULL, AAD_LEN,
                                    dst.ctypes.data, osz.ctypes.data, status.ctypes.data, None)
print(json.dumps({"rc": int(rc), "err": L.tsgpu_last_error().decode()}))
ctx.close()
"""


@pytest.fixture(scope="module")
def simt_lib():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/libtsgpu_simt.so"])


@pytest.mark.parametrize("call", ["detransform", "transform_device", "detransform_device"])
def test_null_aad_with_length_is_refused(simt_lib, call):
    out = subprocess.run([sys.executable, "-c", _DRIVER, ROOT, call], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, "the call did not return (exit %d): %s" % (out.returncode, (out.stdout + out.stderr)[-2000:])
    got = json.loads(out.stdout.strip().splitlines()[-1])
    assert got["rc"] == binding.E_ARG, got
    assert "aad cannot be null" in got["err"], got
