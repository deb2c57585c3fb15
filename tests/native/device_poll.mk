# tests/native/device_poll.mk -- TEST INFRASTRUCTURE: the device poll / status / Disconnect test driver
# (device_poll.cu), user kernels built for sm_90a against the public header include/b200_device.cuh.
# make -C tests/native -f device_poll.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_pair.h $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_poll.so
libdevice_poll.so: device_poll.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_poll.cu
.PHONY: all
