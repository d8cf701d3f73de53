# Builds dgraph_b200/libdgx.so (sm_90a only: H100) and the CPU oracle.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS ?= -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-maybe-uninitialized -Xptxas -v
CSRC := dgraph_b200/csrc
HDRS := $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.hpp) include/dgx.h

.PHONY: all prof clean
all: dgraph_b200/libdgx.so oracle/liboracle.so

dgraph_b200/libdgx.so: $(CSRC)/dgx_api.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -shared -o $@ $(CSRC)/dgx_api.cu -lcudart

# instrumented build for tools/prof_pipe_waits.py (per-role wait / phase cycle counters; slower, never benchmarked)
prof: dgraph_b200/libdgx_prof.so
dgraph_b200/libdgx_prof.so: $(CSRC)/dgx_api.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -DDGX_PIPE_PROF -shared -o $@ $(CSRC)/dgx_api.cu -lcudart

oracle/liboracle.so: oracle/oracle.c oracle/oracle.h
	$(MAKE) -C oracle liboracle.so

clean:
	rm -f dgraph_b200/libdgx.so dgraph_b200/libdgx_prof.so oracle/liboracle.so
