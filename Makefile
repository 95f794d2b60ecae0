# Builds libtsgpu.so (product, sm_90a only), the CPU oracle and the test-only SIMT build.
PKG := tiered-storage-for-apache-kafka_b200
CSRC := $(PKG)/csrc
NVCC ?= nvcc
NVCCFLAGS := -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v \
             --expt-relaxed-constexpr
HDRS := $(wildcard $(CSRC)/*.cuh $(CSRC)/*.h $(CSRC)/*.hpp) include/tsgpu.h

all: $(PKG)/libtsgpu.so oracle tests/simt/libtsgpu_simt.so
libtsgpu.so: $(PKG)/libtsgpu.so

$(PKG)/libtsgpu.so: $(CSRC)/tsgpu.cu $(HDRS)
	$(NVCC) $(NVCCFLAGS) -shared -o $@ $(CSRC)/tsgpu.cu -lcudart 2> build_ptxas.log || (cat build_ptxas.log; false)
	@grep -E "error|warning: .*spill|bytes spill" build_ptxas.log | grep -v " 0 bytes spill" | head -20 || true

oracle:
	$(MAKE) -s -C oracle

# TEST-ONLY: the same sources compiled for the fiber emulator (never loaded by the package)
tests/simt/libtsgpu_simt.so: $(CSRC)/tsgpu.cu $(HDRS) tests/simt/simt.h tests/simt/simt.cpp
	g++ -O2 -g -std=c++17 -fPIC -shared -DTSGPU_SIMT=1 -Itests/simt -I$(CSRC) -x c++ $(CSRC)/tsgpu.cu tests/simt/simt.cpp \
	    -o $@ -Wall -Wno-unknown-pragmas -Wno-unused-function -Wno-unused-variable

# TEST-ONLY: the emulator build under AddressSanitizer (shared memory and scratch are heap blocks there, so overruns show)
tests/simt/libtsgpu_simt_asan.so: $(CSRC)/tsgpu.cu $(HDRS) tests/simt/simt.h tests/simt/simt.cpp
	g++ -O1 -g -std=c++17 -fPIC -shared -fsanitize=address -DTSGPU_SIMT=1 -Itests/simt -I$(CSRC) -x c++ $(CSRC)/tsgpu.cu tests/simt/simt.cpp \
	    -o $@ -Wno-unknown-pragmas
# TEST-ONLY: the emulator build under UndefinedBehaviorSanitizer: shift counts >= width (x86 masks them, a GPU clamps) and
# misaligned vector accesses (x86 tolerates them, a GPU faults) are the two that matter
tests/simt/libtsgpu_simt_ubsan.so: $(CSRC)/tsgpu.cu $(HDRS) tests/simt/simt.h tests/simt/simt.cpp
	g++ -O1 -g -std=c++17 -fPIC -shared -fsanitize=undefined -fno-sanitize=vptr -fno-sanitize-recover=undefined -DTSGPU_SIMT=1 -Itests/simt -I$(CSRC) -x c++ $(CSRC)/tsgpu.cu tests/simt/simt.cpp \
	    -o $@ -Wno-unknown-pragmas

clean:
	rm -f $(PKG)/libtsgpu.so tests/simt/libtsgpu_simt.so tests/simt/libtsgpu_simt_asan.so tests/simt/libtsgpu_simt_ubsan.so build_ptxas.log
	$(MAKE) -C oracle clean
.PHONY: all oracle clean libtsgpu.so

# C++ host-mirror tests: `_simt` links the test-only emulator build (CPU box), `_gpu` links the product library.
tests/cpp/test_host_mirror_simt: tests/cpp/test_host_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp tests/simt/libtsgpu_simt.so oracle
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_host_mirror.cpp -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
tests/cpp/test_host_mirror_gpu: tests/cpp/test_host_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/libtsgpu.so oracle
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_host_mirror.cpp -L$(PKG) -ltsgpu -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../../$(PKG)' -Wl,-rpath,'$$ORIGIN/../../oracle' -Wl,-rpath,/usr/local/cuda/lib64

# JNI glue compiled as it stands against a test-only stand-in for <jni.h> and driven through a fake JNIEnv (no JDK here)
tests/cpp/test_jni_shim_simt: tests/cpp/test_jni_shim.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_shim.c -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# JNI glue's record-validation path (RecordsCursor.transformCursor) in the window flow of GpuTransformChunkEnumeration, same fake JNIEnv
tests/cpp/test_jni_records_simt: tests/cpp/test_jni_records.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_records.c -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# Host mirror with upload-part checksums (SegmentLogUploader::partChecksums), on the emulator build
tests/cpp/test_part_crc_mirror_simt: tests/cpp/test_part_crc_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_part_crc_mirror.cpp -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# JNI glue's part-checksum path (PartsCursor.transformParts) in the window flow of GpuTransformChunkEnumeration, same fake JNIEnv
tests/cpp/test_jni_parts_simt: tests/cpp/test_jni_parts.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_parts.c -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# Host mirror of the object check (RemoteSegmentChecker, tsgpu_check_object), on the emulator build
tests/cpp/test_check_mirror_simt: tests/cpp/test_check_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_check.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_check_mirror.cpp -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# JNI glue's object-check path (CheckCursor.checkObject) in the window flow of an operator tool, same fake JNIEnv
tests/cpp/test_jni_check_simt: tests/cpp/test_jni_check.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_check.c -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# Host mirror of the object rewrite (RemoteSegmentRewriter, tsgpu_rewrite_object), on the emulator build
tests/cpp/test_rewrite_mirror_simt: tests/cpp/test_rewrite_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_rewrite.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_rewrite_mirror.cpp -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# JNI glue's object-rewrite path (RewriteCursor.rewriteObject) in the window flow of an operator tool, same fake JNIEnv
tests/cpp/test_jni_rewrite_simt: tests/cpp/test_jni_rewrite.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_rewrite.c -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# Host mirror with CRC-64/NVME (crc64Parts, check64, RemoteSegmentRewriter::crc64), on the emulator build
tests/cpp/test_crc64_mirror_simt: tests/cpp/test_crc64_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_check.hpp $(PKG)/host/segment_rewrite.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_crc64_mirror.cpp -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# JNI glue's CRC-64/NVME exports (Crc64.transformParts, checkObject, rewriteObject), same fake JNIEnv
tests/cpp/test_jni_crc64_simt: tests/cpp/test_jni_crc64.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_crc64.c -Ltests/simt -ltsgpu_simt -Wl,-rpath,'$$ORIGIN/../simt'
# Host mirror of TSGPU_FLAG_REFRAME (RemoteSegmentRewriter::addChecksums, ::denseFrames) on an oracle-written object, on the emulator build
tests/cpp/test_reframe_mirror_simt: tests/cpp/test_reframe_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_check.hpp $(PKG)/host/segment_rewrite.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_reframe_mirror.cpp -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# JNI glue's REFRAME path (RewriteCursor.rewriteObject with TsGpu.FLAG_REFRAME) on an oracle-written object, same fake JNIEnv
tests/cpp/test_jni_reframe_simt: tests/cpp/test_jni_reframe.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_reframe.c -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# JNI glue's key-rotation path (RekeyCursor.rekeyObject, rekeyObjectCrc64) on an oracle-written object, same fake JNIEnv
tests/cpp/test_jni_rekey_simt: tests/cpp/test_jni_rekey.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_rekey.c -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# Host mirror of key rotation (RemoteSegmentRekeyer, tsgpu_rekey_object) on an oracle-written segment, on the emulator build
tests/cpp/test_rekey_mirror_simt: tests/cpp/test_rekey_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_rekey.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_rekey_mirror.cpp -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# JNI glue's encryption path (EncryptCursor.encryptObject, encryptObjectCrc64) on an oracle-written object, same fake JNIEnv
tests/cpp/test_jni_encrypt_simt: tests/cpp/test_jni_encrypt.c jni/tsgpu_jni.c tests/jni_stub/jni.h include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	gcc -O1 -g -std=gnu11 -Wall -Wno-unused-parameter -Wno-unused-function -Itests/jni_stub -Iinclude -o $@ tests/cpp/test_jni_encrypt.c -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
# Host mirror of encryption (RemoteSegmentEncryptor, tsgpu_encrypt_object) on an oracle-written segment, on the emulator build
tests/cpp/test_encrypt_mirror_simt: tests/cpp/test_encrypt_mirror.cpp $(PKG)/host/chunk_transform.hpp $(PKG)/host/segment_upload.hpp $(PKG)/host/segment_encrypt.hpp include/tsgpu.h tests/simt/libtsgpu_simt.so oracle
	g++ -O1 -g -std=c++17 -o $@ tests/cpp/test_encrypt_mirror.cpp -Ltests/simt -ltsgpu_simt -Loracle -ltsoracle -Wl,-rpath,'$$ORIGIN/../simt' -Wl,-rpath,'$$ORIGIN/../../oracle'
