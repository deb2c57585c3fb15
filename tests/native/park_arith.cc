// park_arith.cc -- TEST INFRASTRUCTURE: the ready-set control words of grpc-rdma_b200/csrc/b200_dev.cuh with their
// parking fields, compiled for the host, for tests/test_device_ready_park_cpu.py.
#include <stddef.h>
#include <stdint.h>

#define __align__(n) __attribute__((aligned(n)))  // nvcc spelling, for the host compiler
#include "../../grpc-rdma_b200/csrc/b200_dev.cuh"

extern "C" {
uint64_t pa_sizeof_queue() { return sizeof(b200::ReadyQueue); }
uint64_t pa_offset_head() { return offsetof(b200::ReadyQueue, head); }
uint64_t pa_offset_tail() { return offsetof(b200::ReadyQueue, tail); }
uint64_t pa_offset_tail_hi() { return offsetof(b200::ReadyQueue, tail_hi); }
uint64_t pa_offset_rings() { return offsetof(b200::ReadyQueue, rings); }
uint64_t pa_offset_mask() { return offsetof(b200::ReadyQueue, mask); }
uint64_t pa_offset_bell() { return offsetof(b200::ReadyQueue, bell); }
uint64_t pa_entries_offset() { return (uint64_t)((const char*)b200::ready_entries(nullptr) - (const char*)nullptr); }
uint64_t pa_parked_bit() { return b200::kReadyParked; }
}
