"""The CRC-64/NVME calls through the JNI glue and the C++ host mirror, on the SIMT emulator: Crc64.transformParts,
Crc64.checkObject and Crc64.rewriteObject driven through the fake JNIEnv (tests/cpp/test_jni_crc64.c), SegmentLogUploader with
crc64Parts, RemoteSegmentChecker::check64 and RemoteSegmentRewriter::crc64 (tests/cpp/test_crc64_mirror.cpp); and the Java side
checked by source, as there is no JDK here: the new natives match their exports in arity, the existing classes keep their
natives, and the enumeration has a CRC-64 constructor beside its unchanged ones."""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def _run(target):
    subprocess.check_call(["make", "-s", "-C", ROOT, target], stderr=subprocess.DEVNULL)
    env = {k: v for k, v in os.environ.items() if k != "TSGPU_VALIDATE_RECORDS"}
    out = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=900, env=env)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_jni_crc64_through_a_fake_jnienv():
    _run("tests/cpp/test_jni_crc64_simt")


def test_host_mirror_crc64():
    _run("tests/cpp/test_crc64_mirror_simt")


def _natives(cls):
    java = open(os.path.join(ROOT, "jni", PKG, cls + ".java")).read()
    return java, re.findall(r"public static native\s+\S+\s+(\w+)\(([^)]*)\)", java, flags=re.S)


def test_java_natives_match_their_exports():
    c = open(os.path.join(ROOT, "jni", "tsgpu_jni.c")).read()
    java, natives = _natives("Crc64")
    assert [n for n, _ in natives] == ["transformParts", "checkObject", "rewriteObject"]
    for name, params in natives:
        m = re.search(r"Java_" + PKG.replace("/", "_") + r"_Crc64_" + name + r"\(([^)]*)\)", c, flags=re.S)
        assert m, name
        assert len([p for p in m.group(1).split(",") if p.strip()]) == len([p for p in params.split(",") if p.strip()]) + 2, name
    for cls, native in (("PartsCursor", "transformParts"), ("CheckCursor", "checkObject"), ("RewriteCursor", "rewriteObject")):
        src, nat = _natives(cls)
        assert [n for n, _ in nat] == [native], cls                 # the CRC-32C native stays the class's only one
        assert re.search(r"public " + cls + r"\([^)]*final boolean crc64\)", src), cls
        assert "Crc64." in src, cls
    parts, _ = _natives("PartsCursor")
    assert "public long partCrc64(final int partNumber)" in parts and "public long objectCrc64()" in parts
    check, _ = _natives("CheckCursor")
    assert "public long objectCrc64()" in check and "public long segmentCrc64()" in check
    rewrite, _ = _natives("RewriteCursor")
    for m in ("sourceCrc64", "objectCrc64", "segmentCrc64"):
        assert "public long " + m + "()" in rewrite, m
    enum = open(os.path.join(ROOT, "jni", PKG, "GpuTransformChunkEnumeration.java")).read()
    assert re.search(r"final long partSize,\s*final boolean crc64Parts\)", enum)
    assert "new PartsCursor(partSize, true)" in enum
    assert "public long partCrc64(final int partNumber)" in enum and "public long objectCrc64()" in enum
