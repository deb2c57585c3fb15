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
 *   b200_warp_poll / b200_warp_status / b200_warp_writable / b200_warp_disconnect: the Poller's scan over many ends,
 *                       get_status, GetWritableSize and Disconnect (below)
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
 * host-driven peer see the device-driven traffic.  An end claimed with B200_CLAIM_UNMIRRORED (b200_pair_device_claim_ex)
 * has no mirror until its release: its calls skip its publication and its lock, and a peer's calls skip it too; the
 * peer's own mirror is published as above.  The results are the same, bit for bit.
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

/* ---- the poll loop of a BPEV server: poll, status, writable, Disconnect (DESIGN.md §13) ---------------------------
 *
 * b200_warp_poll: the readiness of n claimed ends, one lane per handle, 32 handles per round (any n, 0 included).
 * events[i] (may be NULL) gets the B200_EV_* bits b200_poller_scan gives the same pair from the same state: on a
 * CONNECTED end READABLE when the peer has left, otherwise READABLE on HasMessage (reference format: a header word
 * at the head counts, footer or not; stamped frames: a complete frame with the expected stamp) and WRITABLE on
 * HasPendingWrites; READABLE on an ERROR or HALF_CLOSED end; 0 otherwise.  ready (may be NULL) gets the indices i
 * with non-zero events in ascending order; the call returns how many there are.  It never waits, takes no lock and
 * writes no mirror: a device-owned end publishes its own mirror under the pair's lock in its Send / Recv calls, and a
 * lock-free scan that wrote mirrors could overwrite a newer view.  The rule is k_poll_scan's, in the same code.
 */
__device__ inline uint32_t b200_warp_poll(const b200_dev_pair* handles, uint32_t n, uint32_t* events,
                                          uint32_t* ready) {
  const uint32_t lane = b200_lane_id();
  uint32_t count = 0;
  for (uint32_t base = 0; base < n; base += 32) {
    const uint32_t i = base + lane;
    uint32_t ev = 0;
    if (i < n) {
      ev = b200::poll_events<false>(reinterpret_cast<b200::PairDev*>(handles[i].table), handles[i].slot);
      if (events) events[i] = ev;
    }
    const unsigned m = __ballot_sync(0xffffffffu, ev != 0);
    if (ready && ev) ready[count + __popc(m & ((1u << lane) - 1))] = i;
    count += __popc(m);
  }
  __syncwarp();
  return count;
}

/* get_status (pair.cc:349-375) from the device state: a b200_status, HALF_CLOSED on a CONNECTED end whose peer has
 * left.  b200_pair_status also probes, every 500 ms, whether the peer's process still exists (CUDA-IPC wire): a
 * kernel cannot ask that, so a peer process that died without Disconnect shows here only once the host has seen it. */
__device__ inline int b200_warp_status(const b200_dev_pair* h) {
  return (int)b200::pair_status(reinterpret_cast<b200::PairDev*>(h->table), h->slot);
}

/* GetWritableSize (pair.cc:294-301): b200_pair_writable's formula on the device's credit word and tail. */
__device__ inline uint64_t b200_warp_writable(const b200_dev_pair* h) {
  return b200::pair_writable(reinterpret_cast<b200::PairDev*>(h->table), h->slot);
}

/* PairPollable::Disconnect (pair.cc:325-347) from the device: 0 (nothing changed) unless the end is CONNECTED;
 * otherwise a fence (system scope on the nvlink wire) so that everything this end wrote is visible, the peer's
 * peer_exit = 1 with this end's moving head (as b200_pair_disconnect writes it; not when the peer has left already),
 * the end DISCONNECTED -- every later call on it returns 0 -- and 1.  The peer sees HALF_CLOSED at once; a
 * b200_pair_status of this end says DISCONNECTED.  b200_pair_device_release then finishes the Disconnect on the host
 * (the wire and the address go), with no second write to the peer.  Counts as both a Send and a Recv under the
 * ops-in-flight rule: no Send or Recv of this end may run beside it. */
__device__ inline int b200_warp_disconnect(const b200_dev_pair* h) {
  return b200::warp_disconnect(reinterpret_cast<b200::PairDev*>(h->table), h->slot, b200_lane_id());
}

/* ---- ready sets: the device's epoll (b200_pair.h, DESIGN.md §13 "Ready sets") -------------------------------------
 *
 * A server warp that holds many claimed ends takes the keys of the ends whose readiness changed instead of scanning
 * them all.  Any number of consumer warps may share one set (one CTA or many, one kernel or several); neither call
 * waits.
 *   b200_warp_ready_take(s, keys, max): pops up to max keys into keys[] (device or pinned memory) and returns how many;
 *     keys[] beyond that count are unspecified.  Each entry goes to exactly one warp: the warp claims the run it read
 *     with one atomicCAS on the queue's head and reads again when another warp took first.  An empty take does no
 *     atomic.  The keys are hints: the consumer drives those ends with the calls above (Recv until it returns 0,
 *     Send, Disconnect).  A taken key's frame, credit or close is visible to those calls.
 *   b200_warp_ready_rearm(s, h): the consumer has finished with member h for now.  It stores armed = 1, fences and
 *     probes.  When the end is READY (b200_warp_poll reports READABLE, or a write is pending and there is credit for
 *     one frame) and the call wins the end back from the producers, it returns the end's B200_EV_* bits: the consumer
 *     keeps the end and serves it again.  Otherwise 0: a producer has queued the key already, or nothing is pending
 *     and the next change will queue it.  Every change after a rearm is reported, by the rearm itself or by an entry
 *     (no lost wakeup), and a member never has two entries queued.
 * The first entry of a member is queued by b200_ready_set_add, with the member disarmed: take it, serve, rearm.  An
 * entry of a released member can still be taken once; its key then names an end that is no longer a member.
 * The holder rule, for consumers that share a set: a warp holds member m from the take that returned m's key, or from
 * its rearm of m that returned non-zero, until its rearm of m returns 0 or it disconnects m.  Only the holder drives m
 * (Recv, Send, Disconnect) and rearms it.  A member has at most one entry queued, and that entry is queued only after
 * the holder's rearm stored armed = 1, so no two warps hold a member at once and the ops-in-flight rule holds with no
 * lock in user code.  The new holder may take the entry while the old holder's rearm still probes; that probe only
 * reads.  A warp that shares its set runs __threadfence() before each rearm: the rearm's own fence follows its store
 * of armed = 1, and the next holder must see the cursors this warp's calls wrote and the warp's own per-member state.
 * (With one consumer warp per set the fence is not needed.)  A warp may take up to max keys, but the members it holds
 * are served by no other warp: take what the warp will serve soon.
 */
__device__ inline uint32_t b200_warp_ready_take(const b200_dev_ready_set* s, uint32_t* keys, uint32_t max) {
  return b200::ready_take(static_cast<b200::ReadyQueue*>(s->queue), keys, max, b200_lane_id());
}
__device__ inline uint32_t b200_warp_ready_rearm(const b200_dev_ready_set* s, const b200_dev_pair* h) {
  return b200::ready_rearm(static_cast<b200::ReadyQueue*>(s->queue), reinterpret_cast<b200::PairDev*>(h->table),
                           h->slot, b200_lane_id());
}

/* b200_warp_ready_park(s): park the set so that the server may exit, warp-collective (b200_pair.h and DESIGN.md §13
 * "Parking").  The next entry queued on a parked set rings its doorbell once, and the Poller kicks the set's eventfd.
 * The rule:
 *   - one warp calls it, once no other consumer warp of the set will take again;
 *   - that warp holds no member: each of its rearms returned 0, or it disconnected the member;
 *   - 0: the set is parked (or a ring is already on its way), and the kernel may exit;
 *   - non-zero: entries are queued and nothing rang; the warp must take and serve again (and park again later).  With
 *     many warps the last one to go idle may serve alone.
 * The multi-warp exit (tests/native/device_ready_park.cu): each warp counts empty takes, and after K in a row it adds
 * one to an idle counter in device memory and stops taking.  The warp whose atomicAdd returns warps - 1 is the last:
 * it parks; while the park returns non-zero it takes, serves and rearms alone, then parks again.  The kernel exits
 * when that park returns 0.
 *
 *   if (atomicAdd(&idle, 1) == warps - 1)           // lane 0, broadcast to the warp
 *     while (b200_warp_ready_park(s)) serve_until_empty(s);
 */
__device__ inline uint32_t b200_warp_ready_park(const b200_dev_ready_set* s) {
  return b200::ready_park(static_cast<b200::ReadyQueue*>(s->queue), b200_lane_id());
}

#endif /* B200_DEVICE_CUH */
