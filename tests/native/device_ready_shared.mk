# tests/native/device_ready_shared.mk -- TEST INFRASTRUCTURE: the shared ready-set test driver (device_ready_shared.cu),
# user kernels built for sm_90a against the public header include/b200_device.cuh.
# make -C tests/native -f device_ready_shared.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_pair.h $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_ready_shared.so
libdevice_ready_shared.so: device_ready_shared.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_ready_shared.cu
.PHONY: all
