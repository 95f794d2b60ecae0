"""The record-validation path of the JNI glue: RecordsCursor.transformCursor driven through the fake JNIEnv in the window
flow of GpuTransformChunkEnumeration (tests/cpp/test_jni_records.c), and the Java side checked by source, as there is no
JDK here: the native declaration matches its export, and the enumeration keeps one cursor per segment across fill() and
marks the segment's last window."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def test_records_cursor_through_a_fake_jnienv():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/cpp/test_jni_records_simt"], stderr=subprocess.DEVNULL)
    env = {k: v for k, v in os.environ.items() if k != "TSGPU_VALIDATE_RECORDS"}
    out = subprocess.run([os.path.join(ROOT, "tests/cpp/test_jni_records_simt")], capture_output=True, text=True, timeout=600, env=env)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_java_side_of_the_cursor():
    java = open(os.path.join(ROOT, "jni", PKG, "RecordsCursor.java")).read()
    c = open(os.path.join(ROOT, "jni", "tsgpu_jni.c")).read()
    natives = re.findall(r"public static native\s+\S+\s+(\w+)\(([^)]*)\)", java, flags=re.S)
    assert [n for n, _ in natives] == ["transformCursor"]
    m = re.search(r"Java_" + PKG.replace("/", "_") + r"_RecordsCursor_transformCursor\(([^)]*)\)", c, flags=re.S)
    assert m
    assert len([p for p in m.group(1).split(",") if p.strip()]) == len([p for p in natives[0][1].split(",") if p.strip()]) + 2
    assert "allocateDirect(SIZE)" in java and "SIZE = 64" in java
    tsgpu = open(os.path.join(ROOT, "jni", PKG, "TsGpu.java")).read()
    assert "FLAG_VALIDATE_RECORDS = 32" in tsgpu
    enum = open(os.path.join(ROOT, "jni", PKG, "GpuTransformChunkEnumeration.java")).read()
    assert re.search(r"private final RecordsCursor records = new RecordsCursor\(\);", enum)    # one per enumeration = segment
    assert "TsGpu.transform(" not in enum                                                    # every window goes through it
    assert re.search(r"records\.transform\([^;]*ivs, out, sizes, eof\);", enum, flags=re.S)  # the short window ends the segment
    assert re.search(r"total == 0\) \{[^}]*records\.transform\([^;]*, true\);", enum, flags=re.S)   # ... or an empty one
