"""The encryption path of the JNI glue: EncryptCursor.encryptObject and encryptObjectCrc64 driven through the fake JNIEnv in the
window flow of an operator tool (tests/cpp/test_jni_encrypt.c), and the Java side checked by source, as there is no JDK here: the
native declarations match their exports with the right arity and the cursor is a 64-byte direct buffer."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def test_encrypt_cursor_through_a_fake_jnienv():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/cpp/test_jni_encrypt_simt"], stderr=subprocess.DEVNULL)
    out = subprocess.run([os.path.join(ROOT, "tests/cpp/test_jni_encrypt_simt")], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_java_side_of_the_encrypt_cursor():
    java = open(os.path.join(ROOT, "jni", PKG, "EncryptCursor.java")).read()
    c = open(os.path.join(ROOT, "jni", "tsgpu_jni.c")).read()
    natives = re.findall(r"public static native\s+\S+\s+(\w+)\(([^)]*)\)", java, flags=re.S)
    assert [n for n, _ in natives] == ["encryptObject", "encryptObjectCrc64"]
    for name, params in natives:
        m = re.search(r"Java_" + PKG.replace("/", "_") + r"_EncryptCursor_" + name + r"\(([^)]*)\)", c, flags=re.S)
        assert m, name
        assert len([p for p in m.group(1).split(",") if p.strip()]) == len([p for p in params.split(",") if p.strip()]) + 2, name
    assert "allocateDirect(SIZE)" in java and "SIZE = 64" in java
