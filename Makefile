# Build recipe for the product library, the CPU-only device-code emulation used by
# the `-m "not gpu"` tests, and the oracle.  __graft_entry__.build() drives this.
PKG    = fluent-bit_b200
CSRC   = $(PKG)/csrc
NVCC  ?= nvcc
ARCH   = -gencode arch=compute_90a,code=sm_90a
NVFLAGS = $(ARCH) -lineinfo -O3 -std=c++17 -Xcompiler -fPIC
CFLAGS = -O2 -g -fPIC -Wall -Wno-unused-function

all: product hostsim oracle

product: $(PKG)/libflbgpu.so
HDRS = $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/flbgpu.h
# one object per translation unit, so that `make -j` compiles the .cu files side by side (kernels.cu alone takes minutes)
$(CSRC)/kernels.o: $(CSRC)/kernels.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -c $(CSRC)/kernels.cu -o $@
$(CSRC)/kernels_ml.o: $(CSRC)/kernels_ml.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -c $(CSRC)/kernels_ml.cu -o $@
$(CSRC)/kernels_tojson.o: $(CSRC)/kernels_tojson.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -c $(CSRC)/kernels_tojson.cu -o $@
$(CSRC)/kernels_lines.o: $(CSRC)/kernels_lines.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -c $(CSRC)/kernels_lines.cu -o $@
$(CSRC)/runtime.o: $(CSRC)/runtime.c $(HDRS)
	gcc $(CFLAGS) -c $(CSRC)/runtime.c -o $@
$(CSRC)/rx_compile.o: $(CSRC)/rx_compile.c $(HDRS)
	gcc $(CFLAGS) -c $(CSRC)/rx_compile.c -o $@
$(PKG)/libflbgpu.so: $(CSRC)/kernels.o $(CSRC)/kernels_ml.o $(CSRC)/kernels_tojson.o $(CSRC)/kernels_lines.o $(CSRC)/runtime.o $(CSRC)/rx_compile.o
	$(NVCC) $(ARCH) -shared -o $@ $(CSRC)/kernels.o $(CSRC)/kernels_ml.o $(CSRC)/kernels_tojson.o $(CSRC)/kernels_lines.o $(CSRC)/runtime.o $(CSRC)/rx_compile.o -lcudart -lpthread -ldl

hostsim: tests/hostsim/libhostsim.so
tests/hostsim/libhostsim.so: tests/hostsim/hostsim.cpp tests/hostsim/hostsim_tail.cpp tests/hostsim/hostsim_gelf.cpp $(CSRC)/runtime.c $(CSRC)/rx_compile.c $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h)
	gcc $(CFLAGS) -c $(CSRC)/runtime.c -o tests/hostsim/runtime.o
	gcc $(CFLAGS) -c $(CSRC)/rx_compile.c -o tests/hostsim/rx_compile.o
	g++ $(CFLAGS) -shared -o $@ tests/hostsim/hostsim.cpp tests/hostsim/hostsim_tail.cpp tests/hostsim/hostsim_gelf.cpp tests/hostsim/runtime.o tests/hostsim/rx_compile.o -lrt -lpthread

# the same emulation under AddressSanitizer + UBSan (host runtime and the device code as the CPU compiles it):
#   make hostsim-asan && FLBGPU_HOSTSIM_SO=/tmp/flbgpu-asan/libhostsim.so LD_PRELOAD=$$(gcc -print-file-name=libasan.so) \
#       ASAN_OPTIONS=detect_leaks=0 python -m pytest tests -q -s -m "not gpu"
SAN = -O1 -g -fPIC -fsanitize=address,undefined -fno-omit-frame-pointer -Wno-unused-function
hostsim-asan:
	mkdir -p /tmp/flbgpu-asan
	gcc $(SAN) -c $(CSRC)/runtime.c -o /tmp/flbgpu-asan/runtime.o
	gcc $(SAN) -c $(CSRC)/rx_compile.c -o /tmp/flbgpu-asan/rx_compile.o
	g++ $(SAN) -shared -o /tmp/flbgpu-asan/libhostsim.so tests/hostsim/hostsim.cpp tests/hostsim/hostsim_tail.cpp tests/hostsim/hostsim_gelf.cpp /tmp/flbgpu-asan/runtime.o /tmp/flbgpu-asan/rx_compile.o

# the emulation with "device" allocations filled with a byte pattern (cudaMalloc does not hand out zeroes; a fresh malloc often does):
#   make hostsim-poison && FLBGPU_HOSTSIM_SO=/tmp/flbgpu-poison/libhostsim.so python -m pytest tests -q -m "not gpu"
hostsim-poison:
	mkdir -p /tmp/flbgpu-poison
	gcc $(CFLAGS) -c $(CSRC)/runtime.c -o /tmp/flbgpu-poison/runtime.o
	gcc $(CFLAGS) -c $(CSRC)/rx_compile.c -o /tmp/flbgpu-poison/rx_compile.o
	g++ $(CFLAGS) -DHS_POISON=0xA5 -shared -o /tmp/flbgpu-poison/libhostsim.so tests/hostsim/hostsim.cpp tests/hostsim/hostsim_tail.cpp tests/hostsim/hostsim_gelf.cpp /tmp/flbgpu-poison/runtime.o /tmp/flbgpu-poison/rx_compile.o -lrt -lpthread

ORC_SRC = oracle/flb_oracle.c oracle/orc_parsers.c oracle/orc_regex.c oracle/orc_time.c oracle/orc_msgpack.c
oracle: oracle/liboracle.so
	@if [ -d /root/reference ]; then $(MAKE) -s -C oracle/refshim && $(MAKE) -s -C oracle/refshim -f tail.mk tail && $(MAKE) -s -C oracle/refshim -f gelf.mk gelf; else echo "oracle/_ref: reference tree absent, using prebuilt"; fi
oracle/liboracle.so: $(ORC_SRC) oracle/orc.h oracle/orc_flb.h
	gcc $(CFLAGS) -shared -o $@ $(ORC_SRC) -lm

clean:
	rm -f $(PKG)/libflbgpu.so $(CSRC)/*.o tests/hostsim/*.so tests/hostsim/*.o oracle/liboracle.so
.PHONY: all product hostsim hostsim-asan hostsim-poison oracle clean
