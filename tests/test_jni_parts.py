"""The part-checksum path of the JNI glue: PartsCursor.transformParts driven through the fake JNIEnv in the window flow of
GpuTransformChunkEnumeration (tests/cpp/test_jni_parts.c), and the Java side checked by source, as there is no JDK here: the
native declaration matches its export, and the enumeration sends every window through the parts cursor when it has a part size."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def test_parts_cursor_through_a_fake_jnienv():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/cpp/test_jni_parts_simt"], stderr=subprocess.DEVNULL)
    env = {k: v for k, v in os.environ.items() if k != "TSGPU_VALIDATE_RECORDS"}
    out = subprocess.run([os.path.join(ROOT, "tests/cpp/test_jni_parts_simt")], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_java_side_of_the_parts_cursor():
    java = open(os.path.join(ROOT, "jni", PKG, "PartsCursor.java")).read()
    c = open(os.path.join(ROOT, "jni", "tsgpu_jni.c")).read()
    natives = re.findall(r"public static native\s+\S+\s+(\w+)\(([^)]*)\)", java, flags=re.S)
    assert [n for n, _ in natives] == ["transformParts"]
    m = re.search(r"Java_" + PKG.replace("/", "_") + r"_PartsCursor_transformParts\(([^)]*)\)", c, flags=re.S)
    assert m
    assert len([p for p in m.group(1).split(",") if p.strip()]) == len([p for p in natives[0][1].split(",") if p.strip()]) + 2
    assert "allocateDirect(SIZE)" in java and "SIZE = 32" in java
    enum = open(os.path.join(ROOT, "jni", PKG, "GpuTransformChunkEnumeration.java")).read()
    assert re.search(r"final boolean validateRecords,\s*final long partSize\)", enum)           # the new constructor argument
    assert re.search(r"new PartsCursor\(partSize\)", enum)                                         # one per enumeration = object
    assert len(re.findall(r"parts\.transform\(", enum)) == 4                                      # every window, and the empty end
    assert "public int partCrc32c(final int partNumber)" in enum and "public int objectCrc32c()" in enum
