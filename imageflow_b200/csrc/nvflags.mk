# nvcc flags of the product library, shared with tests/gpu_units/Makefile so that the unit probes compile the product's device
# functions exactly as libifb200.so does.
NVCC    ?= /usr/local/cuda/bin/nvcc
ARCH    := -gencode arch=compute_90a,code=sm_90a
# -fmad=false: the only fused multiply-adds are the explicit __fmaf_rn in the kernels (bit parity with the oracle)
EXTRA   ?=
NVFLAGS := $(EXTRA) $(ARCH) -O3 -lineinfo -std=c++17 -fmad=false -ccbin g++ -Xcompiler -fPIC,-O2,-ffp-contract=off,-Wall -Xptxas -v
