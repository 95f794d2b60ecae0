# Builds libtsgpu.so (product, sm_90a only), the CPU oracle and the test-only SIMT build.
PKG := tiered-storage-for-apache-kafka_b200
CSRC := $(PKG)/csrc
NVCC ?= nvcc
NVCCFLAGS := -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v \
             --expt-relaxed-constexpr
HDRS := $(wildcard $(CSRC)/*.cuh $(CSRC)/*.h $(CSRC)/*.hpp $(CSRC)/*.inc) include/tsgpu.h

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
