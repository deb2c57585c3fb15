# tests/native/stamp_arith.mk -- TEST INFRASTRUCTURE: the stamped-frame arithmetic of csrc/b200_dev.cuh and the
# b200_dev_pair layout, compiled for the host (stamp_arith.cc).
# make -C tests/native -f stamp_arith.mk
ROOT := ../..
all: libstamp_arith.so
libstamp_arith.so: stamp_arith.cc $(ROOT)/grpc-rdma_b200/csrc/b200_dev.cuh $(ROOT)/include/b200_pair.h
	g++ -O2 -std=c++17 -fPIC -shared -Wall -x c++ -o $@ stamp_arith.cc
.PHONY: all
