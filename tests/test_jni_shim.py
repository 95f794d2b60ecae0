"""JNI glue (jni/tsgpu_jni.c): compiled as it stands against a test-only stand-in for <jni.h> and driven through a fake
JNIEnv by tests/cpp/test_jni_shim.c (copy-in/copy-out array semantics, exception mapping, round trip checked by the
oracle); plus a check that every `native` method TsGpu.java declares has its Java_* export with the right arity."""
import json
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "io/aiven/kafka/tieredstorage/transform/gpu"


def test_jni_glue_through_a_fake_jnienv():
    subprocess.check_call(["make", "-s", "-C", ROOT, "tests/cpp/test_jni_shim_simt"], stderr=subprocess.DEVNULL)
    out = subprocess.run([os.path.join(ROOT, "tests/cpp/test_jni_shim_simt")], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().splitlines()[-1].startswith("OK:"), out.stdout + out.stderr


def test_java_native_declarations_match_the_exports():
    java = open(os.path.join(ROOT, "jni", PKG, "TsGpu.java")).read()
    c = open(os.path.join(ROOT, "jni", "tsgpu_jni.c")).read()
    natives = re.findall(r"public static native\s+\S+\s+(\w+)\(([^)]*)\)", java, flags=re.S)
    assert len(natives) == 7
    for name, params in natives:
        m = re.search(r"Java_" + PKG.replace("/", "_") + "_TsGpu_" + name + r"\(([^)]*)\)", c, flags=re.S)
        assert m, name
        n_java = len([p for p in params.split(",") if p.strip()])
        n_c = len([p for p in m.group(1).split(",") if p.strip()])
        assert n_c == n_java + 2, (name, n_java, n_c)         # JNIEnv*, jclass + the Java parameters
    # the enumerations the plugin would instantiate implement the reference's interfaces by name
    enum = open(os.path.join(ROOT, "jni", PKG, "GpuTransformChunkEnumeration.java")).read()
    assert "implements TransformChunkEnumeration, AutoCloseable" in enum
    for method in ("originalChunkSize", "transformedChunkSize", "hasMoreElements", "nextElement", "close"):
        assert re.search(r"\b" + method + r"\s*\(", enum), method
    assert "readNBytes" not in enum and "channel.read(in)" in enum            # the stream lands in pinned memory, no byte[] bounce
    de = open(os.path.join(ROOT, "jni", PKG, "GpuDetransformChunkEnumeration.java")).read()
    assert "implements DetransformChunkEnumeration, AutoCloseable" in de and "Stream has fewer bytes than expected" in de
    for method in ("hasMoreElements", "nextElement", "close"):
        assert re.search(r"\b" + method + r"\s*\(", de), method
    cm = open(os.path.join(ROOT, "jni", "io/aiven/kafka/tieredstorage/fetch/gpu/GpuChunkManager.java")).read()
    assert "implements ChunkManager" in cm and "getChunks" in cm and "BytesRange.of(" in cm
    pool = open(os.path.join(ROOT, "jni", PKG, "PinnedPool.java")).read()
    assert "TsGpu.freePinned" in pool and "Cleaner" in pool                   # pinned memory is returned, also for leaked leases


def test_java_sources_reference_only_existing_reference_members():
    """No JDK in the test environment, so the Java cannot be compiled: at least every reference type / member the sources
    name must exist in the reference, whose declarations tests/golden/reference_java_api.json records."""
    files = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_java_api.json")))["files"]

    def decl(path):
        return "\n".join(files[path])
    ref = "core/src/main/java/io/aiven/kafka/tieredstorage"
    chunk = decl(ref + "/Chunk.java")
    for field in ("transformedPosition", "transformedSize", "originalSize"):
        assert re.search(r"public final int " + field, chunk)
    assert "SecretKey dataKey();" in decl(ref + "/manifest/SegmentEncryptionMetadata.java")
    assert "InputStream getChunk(" in decl(ref + "/fetch/ChunkManager.java")
    assert "interface DetransformChunkEnumeration extends Enumeration<byte[]>" in decl(ref + "/transform/DetransformChunkEnumeration.java")
    br = decl("storage/core/src/main/java/io/aiven/kafka/tieredstorage/storage/BytesRange.java")
    assert "public static BytesRange of(final int from, final int to)" in br

    # ... and what the Java glue under jni/ actually uses of those types is declared there
    java = {}
    for d, _, names in os.walk(os.path.join(ROOT, "jni")):
        for n in names:
            if n.endswith(".java"):
                java[n] = open(os.path.join(d, n)).read()
    by_type = {os.path.basename(p)[:-len(".java")]: "\n".join(v) for p, v in files.items()}
    used = 0
    for name, src in java.items():
        # fields read from a Chunk (variables of type Chunk, elements of a List<Chunk>)
        chunk_vars = re.findall(r"\bChunk\s+(\w+)\s*=", src)
        lists = re.findall(r"\bList<Chunk>\s+(\w+)\b", src)
        exprs = [re.escape(v) for v in chunk_vars] + [re.escape(v) + r"\.get\([^()]*\)" for v in lists]
        for e in exprs:
            for field in re.findall(r"\b" + e + r"\.(\w+)\b(?!\s*\()", src):
                assert re.search(r"public final int " + field + ";", by_type["Chunk"]), (name, "Chunk." + field)
                used += 1
        for method in re.findall(r"\bBytesRange\.(\w+)\(", src):
            assert re.search(r"public static BytesRange " + method + r"\(", by_type["BytesRange"]), (name, "BytesRange." + method)
            used += 1
        if "Optional<SegmentEncryptionMetadata>" in src or "SegmentEncryptionMetadata::" in src:
            refs = re.findall(r"SegmentEncryptionMetadata::(\w+)", src) + re.findall(r"\bmap\((\w+)\s*->\s*\1\.(\w+)\(", src)
            for m in refs:
                m = m[1] if isinstance(m, tuple) else m
                assert re.search(r"\b" + m + r"\(\);", by_type["SegmentEncryptionMetadata"]), (name, "SegmentEncryptionMetadata." + m)
                used += 1
        # a class implementing a reference interface overrides only what the interface (or Enumeration / AutoCloseable) declares
        for iface in re.findall(r"\bimplements\s+([\w\s,]+?)\s*\{", src):
            for t in (x.strip() for x in iface.split(",")):
                if t not in by_type:
                    assert t == "AutoCloseable", (name, t)
                    continue
                assert "interface " + t in by_type[t]
                for m in re.findall(r"@Override\s+public\s+[\w<>\[\]]+\s+(\w+)\(", src):
                    assert m in ("hasMoreElements", "nextElement", "close") or re.search(r"\b" + m + r"\(", by_type[t]), \
                        (name, t + "." + m)
                    used += 1
    assert used >= 10, used
