"""tsgpu_encrypt_object's kernels and host pipeline under AddressSanitizer and UndefinedBehaviorSanitizer on the SIMT emulator
(tests/simt/asan_encrypt.py): the frame walk reads mutated frame headers, the GCM stage encrypts in place in the transformed slots
and VERIFY decrypts into the packing buffer, so a read outside a chunk, an overrun of any buffer, or a misaligned vector access
aborts here."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("san,lib", [("asan", "libtsgpu_simt_asan.so"), ("ubsan", "libtsgpu_simt_ubsan.so")])
def test_encrypt_is_clean_under_sanitizers(san, lib):
    runtime = subprocess.run(["gcc", "-print-file-name=lib%s.so" % san], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(runtime) or not os.path.exists(runtime):
        pytest.skip("lib%s not available" % san)
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/simt/" + lib, "oracle"])
    env = dict(os.environ, LD_PRELOAD=runtime, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "simt", "asan_encrypt.py"), lib], env=env,
                         capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0 and "encrypt sweep ok" in out.stdout, (out.stdout + out.stderr)[-4000:]
