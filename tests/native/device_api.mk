# tests/native/device_api.mk -- TEST INFRASTRUCTURE: the device API test driver (device_api.cu), a user kernel built
# for sm_90a against the public header include/b200_device.cuh.
# make -C tests/native -f device_api.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_pair.h $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_api.so
libdevice_api.so: device_api.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_api.cu
.PHONY: all
