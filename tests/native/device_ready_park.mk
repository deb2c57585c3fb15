# tests/native/device_ready_park.mk -- TEST INFRASTRUCTURE: the parking ready-set test driver (device_ready_park.cu),
# user kernels built for sm_90a against the public header include/b200_device.cuh.
# make -C tests/native -f device_ready_park.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_pair.h $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_ready_park.so
libdevice_ready_park.so: device_ready_park.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_ready_park.cu
# the control words of b200_dev.cuh compiled for the host (tests/test_device_ready_park_cpu.py)
park_arith.so: park_arith.cc $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
	g++ -O2 -std=c++17 -fPIC -shared -Wall -x c++ -o $@ park_arith.cc
.PHONY: all
