/*
 * b200_device.cuh -- device-side Send / Recv on a pair, for user kernels (sm_90a).
 *
 * A kernel that already produces or consumes a connection's bytes on the GPU can drive the pair itself instead of
 * returning to the host for every call.  The host hands the pair over with b200_pair_device_claim (b200_pair.h),
 * which fills a b200_dev_pair; the kernel takes it by pointer.  Build with
 *     nvcc -gencode arch=compute_90a,code=sm_90a -I<repo>/include ...
 *
 * Every call is WARP-COLLECTIVE: all 32 lanes of one warp call it with the same arguments, every lane gets the
 * result.  The calls are those of the single-call C ABI, bit for bit (return value, partial_write, cursors,
 * credit, frames and ring image), in every framing mode the connection runs (per-slice, coalesced, stamped):
 *   b200_warp_send      one PairPollable::Send call: b200_pair_send from the same state
 *   b200_warp_recv      one PairPollable::Recv call: b200_pair_recv from the same state
 *   b200_warp_readable / b200_warp_has_message / b200_warp_has_pending_writes: the readiness queries
 * They never wait: Send returns 0 when there is no credit, Recv returns 0 when no complete frame is at the head.
 * The caller decides how to retry and bounds its own loop.
 *
 * Rules:
 *   - slices and dst are device memory or pinned, mapped host memory (the RDMA registered-memory rule);
 *   - at most one sender warp and one receiver warp per pair at a time (the ops-in-flight rule of b200_pair.h);
 *   - the handle is valid from b200_pair_device_claim until b200_pair_device_release, and the kernels that use it
 *     must have finished before the release.
 * At the end of each call the warp publishes the pair's host-visible mirror (and, on the loopback wire, the
 * peer's readiness and credit fields) under the per-pair mirror lock, so host readiness queries, the Poller and a
 * host-driven peer see the device-driven traffic.
 *
 * The code behind these calls (include'd below) is the one the library's service owner warps run.
 */
#ifndef B200_DEVICE_CUH
#define B200_DEVICE_CUH

#include "b200_pair.h"
// the implementation the library's own warps run, compiled into the caller's kernel (header-only by design)
#include "../grpc-rdma_b200/csrc/b200_warp.cuh"
#undef VL  // (the library's shorthand for a volatile access: not for user translation units)

static_assert(sizeof(b200_slice) == sizeof(b200::SliceDev), "b200_slice is the device slice layout");

__device__ __forceinline__ uint32_t b200_lane_id() { return threadIdx.x & 31; }

/* Payload bytes accepted; 0 = nothing (not connected, peer gone, no credit, n == 0). */
__device__ inline uint64_t b200_warp_send(const b200_dev_pair* h, const b200_slice* slices, uint32_t n,
                                          uint64_t byte_idx) {
  return b200::warp_send_call(reinterpret_cast<b200::PairDev*>(h->table), h->slot,
                              reinterpret_cast<const b200::SliceDev*>(slices), n, byte_idx, b200_lane_id());
}

/* Bytes delivered into dst (at most one frame, or the rest of a partially read one); 0 = nothing complete. */
__device__ inline uint64_t b200_warp_recv(const b200_dev_pair* h, void* dst, uint64_t cap) {
  return b200::warp_recv_call(reinterpret_cast<b200::PairDev*>(h->table), h->slot, static_cast<uint8_t*>(dst), cap,
                              b200_lane_id());
}

/* GetReadableSize / HasMessage / HasPendingWrites from the device truth (pair.cc:288-303). */
__device__ inline uint64_t b200_warp_readable(const b200_dev_pair* h) {
  return b200::warp_readable(reinterpret_cast<b200::PairDev*>(h->table), h->slot, nullptr);
}
__device__ inline int b200_warp_has_message(const b200_dev_pair* h) {
  uint32_t hm = 0;
  b200::warp_readable(reinterpret_cast<b200::PairDev*>(h->table), h->slot, &hm);
  return hm != 0;
}
__device__ inline int b200_warp_has_pending_writes(const b200_dev_pair* h) {
  return *(volatile const uint32_t*)&reinterpret_cast<b200::PairDev*>(h->table)[h->slot].partial_write != 0;
}

#endif /* B200_DEVICE_CUH */
