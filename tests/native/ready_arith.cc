// ready_arith.cc -- TEST INFRASTRUCTURE: the ready-set queue arithmetic of grpc-rdma_b200/csrc/b200_dev.cuh (the
// B200_HD inlines the kernels and the host runtime share) compiled for the host, for tests/test_device_ready_cpu.py.
#include <stddef.h>
#include <stdint.h>

#define __align__(n) __attribute__((aligned(n)))  // nvcc spelling, for the host compiler
#include "../../grpc-rdma_b200/csrc/b200_dev.cuh"

extern "C" {
uint32_t ra_queue_size(uint32_t capacity) { return b200::ready_queue_size(capacity); }
int ra_add_check(uint32_t head, uint32_t tail, uint32_t members, uint32_t capacity, uint32_t size) {
  return b200::ready_add_check(head, tail, members, capacity, size);
}
uint64_t ra_entry(uint32_t key, uint32_t pos) { return b200::ready_entry(key, pos); }
int ra_entry_at(uint64_t e, uint32_t pos) { return b200::ready_entry_at(e, pos) ? 1 : 0; }
uint64_t ra_sizeof_queue() { return sizeof(b200::ReadyQueue); }
uint64_t ra_sizeof_note() { return sizeof(b200::ReadyNote); }
uint64_t ra_offset_tail() { return offsetof(b200::ReadyQueue, tail); }
uint64_t ra_offset_mask() { return offsetof(b200::ReadyQueue, mask); }
// byte offset of slot's note from the start of the connection table, and of the first entry from the queue's start
uint64_t ra_note_offset(int slot) {
  return (uint64_t)((const char*)b200::ready_note(nullptr, slot) - (const char*)nullptr);
}
uint64_t ra_entries_offset() { return (uint64_t)((const char*)b200::ready_entries(nullptr) - (const char*)nullptr); }
}
