# libgemm_f16_harness.so — test-only entry points into the fp16 sweep (gemm_f16_harness.cu), built with the library's
# flags (as libgemm_harness.so in Makefile).  Not installed, not part of the library's ABI.
#   make -C tests/kernels -f f16.mk
NVCC ?= /usr/local/cuda/bin/nvcc
CSRC := ../../oramacore_b200/csrc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xcompiler -Wall --expt-relaxed-constexpr --extended-lambda -I../../include -I$(CSRC)
OUT := libgemm_f16_harness.so
HDRS := $(CSRC)/oc_common.cuh $(CSRC)/emb_gemm.cuh $(CSRC)/emb_scan.cuh $(CSRC)/tmap.cuh
all: $(OUT)
$(OUT): gemm_f16_harness.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -shared -o $@ gemm_f16_harness.cu
clean:
	rm -f $(OUT)
.PHONY: all clean
