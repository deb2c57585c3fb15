# tests/native/device_ready.mk -- TEST INFRASTRUCTURE: the device ready-set test driver (device_ready.cu), user kernels
# built for sm_90a against the public headers include/b200_device.cuh and include/b200_device_block.cuh.
# make -C tests/native -f device_ready.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_device_block.cuh $(ROOT)/include/b200_pair.h \
        $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh $(ROOT)/grpc-rdma_b200/csrc/b200_block.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_ready.so ready_arith.so
libdevice_ready.so: device_ready.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_ready.cu
# the queue arithmetic of b200_dev.cuh compiled for the host (tests/test_device_ready_cpu.py)
ready_arith.so: ready_arith.cc $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
	g++ -O2 -std=c++17 -fPIC -shared -Wall -x c++ -o $@ ready_arith.cc
.PHONY: all
