# tests/native/device_cluster.mk -- TEST INFRASTRUCTURE: the cluster-call test driver (device_cluster.cu), a user
# kernel built for sm_90a against the public header include/b200_device_block.cuh.
# make -C tests/native -f device_cluster.mk
NVCC ?= /usr/local/cuda/bin/nvcc
ROOT := ../..
HDRS := $(ROOT)/include/b200_device_block.cuh $(ROOT)/include/b200_device.cuh $(ROOT)/include/b200_pair.h \
        $(ROOT)/grpc-rdma_b200/csrc/b200_block.cuh $(ROOT)/grpc-rdma_b200/csrc/b200_warp.cuh \
        $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh
all: libdevice_cluster.so
libdevice_cluster.so: device_cluster.cu $(HDRS)
	$(NVCC) -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-Wall -Xptxas -v -shared -o $@ device_cluster.cu
.PHONY: all
