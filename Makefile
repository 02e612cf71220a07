# Build of the H100-native (sm_90a) Pire scan path.
#   make            product library (pire_b200/libpire_b200.so) + oracle restatement
#   make ref        the real reference compiled from /root/reference into oracle/_ref
#   make microbench load-path / step-scheme microbenchmarks (tools/)
NVCC      ?= nvcc
CC        ?= gcc
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -Wall -Xptxas -v

CSRC      := pire_b200/csrc
LIB       := pire_b200/libpire_b200.so
LIB_SRC   := $(CSRC)/pire_image.cpp $(CSRC)/dfa_tables.cpp $(CSRC)/scan_kernels.cu $(CSRC)/capi.cu $(CSRC)/capi_host.cu $(CSRC)/capi_dist.cu \
            $(CSRC)/slow_image.cpp $(CSRC)/capi_slow.cu
LIB_HDR   := $(CSRC)/capi_internal.hpp $(CSRC)/pire_image.hpp $(CSRC)/dfa_tables.hpp $(CSRC)/scan_kernels.cuh $(CSRC)/synth.h $(CSRC)/stage_copy.hpp $(CSRC)/slow_image.hpp include/pire_b200.h

ORACLE    := oracle/libpire_oracle.so

all: $(LIB) $(ORACLE)

$(LIB): $(LIB_SRC) $(LIB_HDR) Makefile
	$(NVCC) $(NVCCFLAGS) -shared $(LIB_SRC) -o $@ -ldl 2> build/ptxas_$(notdir $@).log || (cat build/ptxas_$(notdir $@).log; false)
	@grep -E "registers|spill" build/ptxas_$(notdir $@).log | sort | uniq -c | sort -rn | head -20 || true

$(ORACLE): oracle/pire_oracle.c oracle/pire_oracle.h
	$(CC) -O2 -std=c99 -Wall -fPIC -shared oracle/pire_oracle.c -o $@

ref:
	./oracle/build_ref.sh

microbench: build/microbench

build/microbench: tools/microbench.cu
	$(NVCC) $(ARCH) -O3 -std=c++17 -lineinfo tools/microbench.cu -o $@ -lcuda

clean:
	rm -f $(LIB) $(ORACLE) build/microbench build/*.log

$(shell mkdir -p build)

.PHONY: all ref microbench clean
