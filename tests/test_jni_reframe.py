"""TsGpu.FLAG_REFRAME through the JNI glue: RewriteCursor.rewriteObject driven through the fake JNIEnv on an oracle-written
Zstd+AES object (tests/cpp/test_jni_reframe.c), and the Java constant checked by source against the C header, as there is no JDK
here."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def test_reframe_through_a_fake_jnienv():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/cpp/test_jni_reframe_simt"], stderr=subprocess.DEVNULL)
    out = subprocess.run([os.path.join(ROOT, "tests/cpp/test_jni_reframe_simt")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_java_constant_matches_the_header():
    java = open(os.path.join(ROOT, "jni", PKG, "TsGpu.java")).read()
    header = open(os.path.join(ROOT, "include", "tsgpu.h")).read()
    j = re.search(r"public static final int FLAG_REFRAME = (\d+);", java)
    c = re.search(r"#define TSGPU_FLAG_REFRAME (\d+)u", header)
    assert j and c and j.group(1) == c.group(1) == "64"
    assert "FLAG_REFRAME" in open(os.path.join(ROOT, "jni", PKG, "RewriteCursor.java")).read()
