// stamp_arith.cc -- TEST INFRASTRUCTURE: the stamped-frame arithmetic the kernels run (the B200_HD inlines of
// grpc-rdma_b200/csrc/b200_dev.cuh: stamp_of, frame_header / footer, frame_present / complete) compiled for the
// host, plus the layout of the frame counters (PairSeq) and of the b200_dev_pair handle through which the GPU tests
// seed them.  tests/test_stamp_limits_cpu.py compares all of it with a closed form.
#include <stddef.h>
#include <stdint.h>

#define __align__(n) __attribute__((aligned(n)))  // nvcc spelling, for the host compiler
#include "../../grpc-rdma_b200/csrc/b200_dev.cuh"
#include "../../include/b200_pair.h"

// a connection table of the real size (kMaxPairs rows, then the PairSeq side array), for pair_seq()'s addressing
static b200::PairDev g_table[b200::kMaxPairs + b200::kMaxPairs * sizeof(b200::PairSeq) / sizeof(b200::PairDev)];

extern "C" {
uint32_t sa_stamp_of(uint64_t s) { return b200::stamp_of(s); }
uint64_t sa_frame_header(uint64_t p, uint32_t st) { return b200::frame_header(p, st); }
uint64_t sa_frame_footer(uint64_t hdr, uint32_t st) { return b200::frame_footer(hdr, st); }
uint64_t sa_frame_present(uint64_t hdr, uint64_t cap, uint32_t st) { return b200::frame_present(hdr, cap, st); }
uint64_t sa_frame_complete(uint64_t hdr, uint64_t foot, uint64_t cap, uint32_t st) {
  return b200::frame_complete(hdr, foot, cap, st);
}
uint64_t sa_sizeof_pairdev() { return sizeof(b200::PairDev); }
uint64_t sa_sizeof_pairseq() { return sizeof(b200::PairSeq); }
uint64_t sa_offset_seq_tx() { return offsetof(b200::PairSeq, tx); }
uint64_t sa_offset_seq_rx() { return offsetof(b200::PairSeq, rx); }
// byte offset of slot's PairSeq from the side array (what b200_dev_pair::seq points at) and from the table
uint64_t sa_offset_pair_seq(int slot) {
  return (uint64_t)((const char*)b200::pair_seq(g_table, slot) - (const char*)b200::pair_seq(g_table, 0));
}
uint64_t sa_offset_pair_seq_table(int slot) {
  return (uint64_t)((const char*)b200::pair_seq(g_table, slot) - (const char*)g_table);
}
// the public handle b200_pair_device_claim fills (include/b200_pair.h)
uint64_t sa_sizeof_dev_pair() { return sizeof(b200_dev_pair); }
uint64_t sa_offset_dev_pair_seq() { return offsetof(b200_dev_pair, seq); }
uint64_t sa_offset_dev_pair_slot() { return offsetof(b200_dev_pair, slot); }
}
