# starway_b200 build (sm_90a only: H100).  `make` builds everything __graft_entry__.build() needs.
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := $(ARCH) -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -cudart static
CXXFLAGS  := -O2 -g -std=c++17 -fPIC -Wall -Wextra -Wno-unused-parameter -pthread
CFLAGS    := -O2 -g -std=c11 -fPIC -Wall -Wextra

CSRC      := starway_b200/csrc
LIB       := starway_b200/libstarway_b200.so
ORACLE    := oracle/liboracle_tagmatch.so
CPUENG    := oracle/libstarway_cpu.so
HOSTSIM   := tests/hostsim/libstarway_hostsim.so
FASTPATH  := starway_b200/_fastpath.so
PYINC     := $(shell python -c "import sysconfig; print(sysconfig.get_paths()['include'])")
PROBE     := tests/gpu_probe/sw_probe
ABIBENCH  := tests/gpu_probe/abi_bench
KTEST     := tests/gpu_kernels/libsw_kernels_test.so

ENGINE_SRCS := $(CSRC)/engine.cpp
ENGINE_HDRS := $(CSRC)/gpu.h $(CSRC)/sw_device.h include/starway_b200.h

all: lib oracle hostsim probe

lib: $(LIB) $(FASTPATH)
oracle: $(ORACLE) $(CPUENG)
oracle-core: $(ORACLE)
hostsim: $(HOSTSIM)
probe: $(PROBE) $(ABIBENCH) $(KTEST)

build/gpu_cuda.o: $(CSRC)/gpu_cuda.cu $(CSRC)/kernels.cuh $(CSRC)/progress.cuh $(CSRC)/gpu.h $(CSRC)/sw_device.h $(CSRC)/bulk_jobs.h
	@mkdir -p build
	$(NVCC) $(NVFLAGS) -c $< -o $@

build/engine.o: $(ENGINE_SRCS) $(ENGINE_HDRS)
	@mkdir -p build
	$(CXX) $(CXXFLAGS) -Iinclude -c $< -o $@

# The product library: host progress engine + CUDA kernels.  No CPU fallback is linked in.
$(LIB): build/engine.o build/gpu_cuda.o
	$(NVCC) $(ARCH) -shared -cudart static -Xlinker -Bsymbolic -Xlinker --version-script=$(CSRC)/exports.map -o $@ $^ -lpthread -lrt -ldl

# CPython fast path of the binding layer (post / poll / future resolution); optional at run time
$(FASTPATH): $(CSRC)/fastpath.c
	$(CC) -O2 -g -fPIC -shared -Wall -I$(PYINC) -o $@ $<

# Test infrastructure -------------------------------------------------------------
build/tagmatch.o: oracle/tagmatch.c oracle/tagmatch.h
	@mkdir -p build
	$(CC) $(CFLAGS) -c $< -o $@

$(ORACLE): build/tagmatch.o
	$(CC) -shared -o $@ $^

$(CPUENG): oracle/cpu_engine.cpp build/tagmatch.o oracle/tagmatch.h
	$(CXX) $(CXXFLAGS) -shared -o $@ oracle/cpu_engine.cpp build/tagmatch.o -lpthread -lrt

build/engine_sim.o: $(ENGINE_SRCS) $(ENGINE_HDRS)
	@mkdir -p build
	$(CXX) $(CXXFLAGS) -Iinclude -c $< -o $@

build/gpu_sim.o: tests/hostsim/gpu_sim.cpp $(CSRC)/gpu.h $(CSRC)/sw_device.h $(CSRC)/bulk_jobs.h oracle/tagmatch.h
	@mkdir -p build
	$(CXX) $(CXXFLAGS) -c $< -o $@

build/reduce_sim.o: tests/hostsim/reduce_sim.cpp $(CSRC)/gpu.h $(CSRC)/sw_device.h
	@mkdir -p build
	$(CXX) $(CXXFLAGS) -c $< -o $@

# Host-logic simulator: the SAME engine.cpp linked against a CPU stand-in for the device
# backend, used only by `pytest -m "not gpu"` to exercise connection/protocol/flush/close
# logic (world_size 2 on CPU).  Never loaded by the starway_b200 package.
$(HOSTSIM): build/engine_sim.o build/gpu_sim.o build/reduce_sim.o build/tagmatch.o
	$(CXX) -shared -Wl,-Bsymbolic -Wl,--version-script=tests/hostsim/exports_sim.map -o $@ $^ -lpthread -lrt -ldl

$(PROBE): tests/gpu_probe/probe.cu build/gpu_cuda.o
	$(NVCC) $(NVFLAGS) -o $@ tests/gpu_probe/probe.cu build/gpu_cuda.o

# Flat C entry points over the CUDA backend for tests/test_gpu_kernels.py (one kernel per launch, shapes chosen by
# the test); test-only, never linked into $(LIB)
$(KTEST): tests/gpu_kernels/kernels_test.cu tests/gpu_kernels/exports.map build/gpu_cuda.o $(CSRC)/gpu.h $(CSRC)/sw_device.h
	$(NVCC) $(NVFLAGS) -shared -Xlinker -Bsymbolic -Xlinker --version-script=tests/gpu_kernels/exports.map -o $@ tests/gpu_kernels/kernels_test.cu build/gpu_cuda.o -lpthread -lrt

$(ABIBENCH): tests/gpu_probe/abi_bench.cpp $(LIB) include/starway_b200.h
	$(CXX) -O2 -std=c++17 -I/usr/local/cuda/include -o $@ tests/gpu_probe/abi_bench.cpp -Lstarway_b200 -lstarway_b200 -L/usr/local/cuda/lib64 -lcudart -Wl,-rpath,'$$ORIGIN/../../starway_b200' -Wl,-rpath,/usr/local/cuda/lib64

clean:
	rm -rf build $(LIB) $(FASTPATH) $(ORACLE) $(CPUENG) $(HOSTSIM) $(PROBE) $(ABIBENCH) $(KTEST)

# Instrumented builds of the host-logic simulator (same sources) for sanitizer runs of the CPU suite:
#   make hostsim-asan && SW_HOSTSIM_LIB=$PWD/build/asan/libstarway_hostsim.so ASAN_OPTIONS=detect_leaks=0 \
#     LD_PRELOAD=$(gcc -print-file-name=libasan.so) python -m pytest tests/test_hostlogic_sim.py tests/test_chaos_sim.py
#   make hostsim-tsan && SW_HOSTSIM_LIB=$PWD/build/tsan/libstarway_hostsim.so \
#     LD_PRELOAD=$(gcc -print-file-name=libtsan.so) python -m pytest -s tests/test_binding_paths.py tests/test_hostlogic_sim.py
SAN_CXX ?= /usr/bin/g++
hostsim-asan hostsim-tsan: hostsim-%:
	@mkdir -p build/$*
	$(SAN_CXX) -O1 -g -fsanitize=$(if $(filter asan,$*),address,thread) -fno-omit-frame-pointer -std=c++17 -fPIC -pthread -Iinclude \
	  -shared -Wl,-Bsymbolic -Wl,--version-script=tests/hostsim/exports_sim.map -o build/$*/libstarway_hostsim.so \
	  $(CSRC)/engine.cpp tests/hostsim/gpu_sim.cpp tests/hostsim/reduce_sim.cpp -x c oracle/tagmatch.c -lpthread -lrt -ldl

.PHONY: all lib oracle oracle-core hostsim probe clean hostsim-asan hostsim-tsan
