// b200_warp.cuh -- warp-level code shared by the library's kernels and by user kernels (include/b200_device.cuh).
//
// Everything here is run by ONE warp, all 32 lanes with the same arguments: no shared memory, no CTA barrier.
//   memory helpers   loads / stores with the scope a ring, a credit word or a host mirror needs
//   rx_probe, publish_mirror_*, mirror_lock   readiness of a pair and its host-visible mirror
//   warp movers      warp_copy_to_ring / warp_copy_from_ring / warp_zero_ring
//   send_plan, send_frames, warp_recv_frame   the per-slice Send planner, its frame mover and the Recv core: the
//                    service owner warps' small ops call them with their own limits
//   send_publish, credit_return   a Send's result and a Recv's credit, by one thread: shared by send_body /
//                    recv_body and the warp calls
//   warp_send_call / warp_recv_call   one PairPollable::Send / Recv call on a pair's line of the connection
//                    table, any size, every framing mode: the device API (DESIGN.md §13)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_dev.cuh"

namespace b200 {

// Resident kernels touch a pair's line from whichever SM serves the op, so nothing of it may come out of a
// stale L1 line: read through (volatile) every time.
#define VL(x) (*(volatile decltype(x)*)&(x))

__device__ __forceinline__ uint64_t ld_acquire_u64(const void* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_volatile_u64(const void* p) {
  uint64_t v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ uint32_t ld_acquire_u32(const void* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_v2u64(void* p, uint64_t a, uint64_t b) {
  // 16-byte status_report {remote_head, peer_exit}: fence + one vector store
  __threadfence_system();
  asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(p), "l"(a), "l"(b) : "memory");
}

__device__ __forceinline__ uint64_t ld_sys_u64(const void* p) {
  uint64_t v;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_sys_v4(const void* p) {
  uint4 r;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p)
               : "memory");
  return r;
}
__device__ __forceinline__ void st_sys_v4(void* p, uint4 v) {
  asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_sys_u64(void* p, uint64_t v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint8_t ld_volatile_u8(const void* p) { return *(const volatile uint8_t*)p; }

__device__ __forceinline__ uint8_t ld_sys_u8(const void* p) {
  uint16_t v;
  asm volatile("ld.relaxed.sys.global.u8 %0, [%1];" : "=h"(v) : "l"(p) : "memory");
  return (uint8_t)v;
}

// GetReadableSize / HasMessage of a pair whose cursor is (head, remain)
// (ring_buffer.cc:56-97).  A header larger than cap-24 is a torn read in the
// reference (it spins); here it reports "not readable yet".  `st` = the stamp expected at the head (0:
// reference format); a stamped ring has a message only when a complete frame with that stamp is there.
template <bool kSys = true>  // kSys: the ring may be written from outside this GPU (NIC, peer GPU)
__device__ __forceinline__ void rx_probe(const uint8_t* ring, uint64_t cap, uint64_t head, uint64_t remain,
                                         uint32_t st, uint32_t& has_msg, uint64_t& readable) {
  if (remain > 0) {
    has_msg = 1;
    readable = remain;
    return;
  }
  uint64_t hdr = kSys ? ld_acquire_u64(ring + head) : ld_volatile_u64(ring + head);
  has_msg = hdr != 0;
  readable = 0;
  const uint64_t p = frame_present(hdr, cap, st);
  if (p) {
    const uint8_t* fp = ring + ((head + 8 + round_up8(p)) & (cap - 1));
    uint64_t foot = kSys ? ld_acquire_u64(fp) : ld_volatile_u64(fp);
    if (foot == frame_footer(hdr, st)) readable = p;
  }
  if (st) has_msg = readable != 0;
}
// the stamp expected at the head of pair `slot`'s ring (0 when the pair runs the reference format)
__device__ __forceinline__ uint32_t rx_stamp(PairDev* pairs, int slot) {
  if (!(VL(pairs[slot].max_sge) & kSgeStamped)) return 0;
  return stamp_of(VL(pair_seq(pairs, slot)->rx));
}

// Host-visible mirror (pinned, mapped): posted writes only -- a kernel never reads host memory.
// The receive side and the send side of a pair may run concurrently (different streams), so each
// publishes only the fields it owns.
__device__ __forceinline__ void publish_mirror_rx(PairMirror* m, const PairDev* P, uint32_t has_msg,
                                                  uint64_t readable) {
  if (m == nullptr) return;
  volatile PairMirror* vm = m;
  vm->head = P->head;
  vm->moving_head = P->moving_head;
  vm->remain = P->remain;
  vm->acc = P->acc;
  vm->readable = readable;
  vm->has_message = has_msg;
}
__device__ __forceinline__ void publish_mirror_tx(PairMirror* m, const PairDev* P) {
  if (m == nullptr) return;
  volatile PairMirror* vm = m;
  vm->remote_tail = P->remote_tail;
  vm->credit_head = *(volatile const uint64_t*)&P->credit_head;
  vm->partial_write = P->partial_write;
  vm->peer_exit = *(volatile const uint32_t*)&P->credit_exit;
}

// A pair's readiness fields are written by its own Recv and by the peer's Send (which lands the
// bytes); its credit field by its own Send and by the peer's Recv (which returns the credit).  When
// the two ends' ops can run at the same time (the service kernel's workers, or batches on separate
// streams with B200_BATCH_CONCURRENT) each "read the device truth, write the mirror" runs under the
// pair's lock and is made visible system-wide before the lock is released, so the mirror always ends
// up with the newest view and the host never waits on a readiness that was overwritten by an older one.
__device__ __forceinline__ void mirror_lock(PairDev* P, bool on) {
  if (!on) return;
  while (atomicCAS(&P->mlock, 0u, 1u) != 0u) __nanosleep(64);
  __threadfence();
}
__device__ __forceinline__ void mirror_unlock(PairDev* P, bool on) {
  if (!on) return;
  __threadfence_system();
  atomicExch(&P->mlock, 0u);
}

// ---- warp-level byte movers of the small paths (no shared memory, no barrier) ----------------

// n bytes from `src` (any alignment; device or pinned host memory: system-coherent loads that bypass
// L1, the host reuses its buffers) into the ring at payload offset `off` (8-byte aligned; wraps at
// cap).  Whole 8-byte words are written, the tail padded with zeros (pad bytes are never delivered).
// With `eslot` the words also go to that host slot and their eager checksum contribution is returned.
constexpr int kCopyBatch = 8;  // 8-byte words per lane whose loads are in flight together (2 KiB per warp)

__device__ __forceinline__ uint64_t warp_copy_to_ring(uint8_t* ring, uint64_t mask, uint64_t off, const uint8_t* src,
                                                      uint32_t n, uint8_t* eslot, uint32_t lane) {
  const uintptr_t s = reinterpret_cast<uintptr_t>(src);
  const uint32_t sb = (uint32_t)(s & 7), sh = sb * 8;
  const uint64_t* s0 = reinterpret_cast<const uint64_t*>(s & ~(uintptr_t)7);
  const uint32_t words = (n + 7) >> 3;
  uint64_t cs = 0;
  for (uint32_t base = 0; base < words; base += 32 * kCopyBatch) {
    // all loads of the batch first (one trip over PCIe for host slices), then shifts and stores
    uint64_t lo[kCopyBatch], hi[kCopyBatch];
#pragma unroll
    for (int k = 0; k < kCopyBatch; k++) {
      const uint32_t j = base + 32 * k + lane;
      lo[k] = j < words ? ld_sys_u64(s0 + j) : 0;
    }
    if (sh) {
#pragma unroll
      for (int k = 0; k < kCopyBatch; k++) {
        const uint32_t j = base + 32 * k + lane;
        // the last payload byte of word j is byte min(8 j + 8, n) - 1; it lives in aligned word (sb + b) / 8
        const uint32_t lastb = (8 * j + 8 < n ? 8 * j + 8 : n) - 1;
        hi[k] = (j < words && (sb + lastb) / 8 > j) ? ld_sys_u64(s0 + j + 1) : 0;
      }
    }
#pragma unroll
    for (int k = 0; k < kCopyBatch; k++) {
      const uint32_t j = base + 32 * k + lane;
      if (j < words) {
        uint64_t w = sh ? (lo[k] >> sh) | (hi[k] << (64 - sh)) : lo[k];
        const uint32_t rem = n - 8 * j;
        if (rem < 8) w &= (1ull << (8 * rem)) - 1;
        *reinterpret_cast<uint64_t*>(ring + ((off + 8ull * j) & mask)) = w;
        if (eslot) {  // the same words to the receiver's host slot (eager push), folded into its checksum
          st_sys_u64(eslot + 8ull * j, w);
          cs ^= eager_word(w, j);
        }
      }
    }
  }
  return cs;
}

// n ring bytes starting at offset `off` (any alignment, wraps) to `dst` (any alignment; device or
// pinned host memory).
__device__ __forceinline__ void warp_copy_from_ring(uint8_t* dst, const uint8_t* ring, uint64_t mask, uint64_t off,
                                                    uint32_t n, uint32_t lane) {
  const uintptr_t d = reinterpret_cast<uintptr_t>(dst);
  uint32_t head = (uint32_t)((8 - (d & 7)) & 7);
  if (head > n) head = n;
  if (lane < head) dst[lane] = ld_volatile_u8(ring + ((off + lane) & mask));
  const uint32_t nwords = (n - head) >> 3;
  const uint64_t o = off + head;
  const uint32_t sh = (uint32_t)(o & 7) * 8;
  const uint64_t o0 = o & ~7ull;
  for (uint32_t base = 0; base < nwords; base += 32 * kCopyBatch) {
    uint64_t lo[kCopyBatch], hi[kCopyBatch];
#pragma unroll
    for (int k = 0; k < kCopyBatch; k++) {
      const uint32_t j = base + 32 * k + lane;
      lo[k] = j < nwords ? ld_volatile_u64(ring + ((o0 + 8ull * j) & mask)) : 0;
    }
    if (sh) {
#pragma unroll
      for (int k = 0; k < kCopyBatch; k++) {
        const uint32_t j = base + 32 * k + lane;
        hi[k] = j < nwords ? ld_volatile_u64(ring + ((o0 + 8ull * j + 8) & mask)) : 0;
      }
    }
#pragma unroll
    for (int k = 0; k < kCopyBatch; k++) {
      const uint32_t j = base + 32 * k + lane;
      if (j < nwords) *reinterpret_cast<uint64_t*>(dst + head + 8ull * j) = sh ? (lo[k] >> sh) | (hi[k] << (64 - sh)) : lo[k];
    }
  }
  const uint32_t tail = n - head - 8 * nwords;
  if (lane < tail) dst[head + 8 * nwords + lane] = ld_volatile_u8(ring + ((o + 8ull * nwords + lane) & mask));
}

// zero [zs, zs + zl) of the ring (any alignment, wraps)
__device__ __forceinline__ void warp_zero_ring(uint8_t* ring, uint64_t mask, uint64_t zs, uint64_t zl, uint32_t lane) {
  uint64_t head = (8 - (zs & 7)) & 7;
  if (head > zl) head = zl;
  if (lane < head) ring[(zs + lane) & mask] = 0;
  const uint64_t nwords = (zl - head) >> 3;
  const uint64_t o = zs + head;
  for (uint64_t k = lane; k < nwords; k += 32) *reinterpret_cast<uint64_t*>(ring + ((o + 8 * k) & mask)) = 0;
  const uint64_t tail = zl - head - 8 * nwords;
  if (lane < tail) ring[(o + 8 * nwords + lane) & mask] = 0;
}

// Both halves of pair `slot`'s mirror from the device truth, under the pair's lock (loopback wire).  Run by ONE
// lane: the service owner warps call it after an op on a connection whose other end a user kernel drives, so that
// a mirror field this warp wrote from values it loaded at the start of the op never outlives a newer one the kernel
// published meanwhile.
__device__ __forceinline__ void publish_mirror_locked(PairDev* table, int slot) {
  PairDev* X = table + slot;
  PairMirror* m = VL(X->mirror);
  if (m == nullptr) return;
  mirror_lock(X, true);
  const uint64_t head = VL(X->head), remain = VL(X->remain);
  uint32_t hm;
  uint64_t rd;
  rx_probe<false>(VL(X->ring), VL(X->cap), head, remain, rx_stamp(table, slot), hm, rd);
  volatile PairMirror* vm = m;
  vm->head = head;
  vm->moving_head = VL(X->moving_head);
  vm->remain = remain;
  vm->acc = VL(X->acc);
  vm->readable = rd;
  vm->has_message = hm;
  vm->remote_tail = VL(X->remote_tail);
  vm->credit_head = VL(X->credit_head);
  vm->partial_write = VL(X->partial_write);
  vm->peer_exit = VL(X->credit_exit);
  mirror_unlock(X, true);
}

// Ready sets (DESIGN.md §13 "Ready sets"), by ONE thread of a path that has just made a change of pair `peer_slot`'s
// readiness visible: a frame's footer in its ring, the credit in its credit block, or its peer_exit.  An end that
// belongs to no set costs the load of its note's set pointer.  A member: fence (the change before the exchange: with
// the consumer's store / fence / probe in b200_warp_ready_rearm, Dekker's pattern), then whoever takes `armed` from 1
// to 0 appends the key, so a member has at most one entry queued.  The entry is stored with release semantics after
// the change, and the consumer loads it with acquire semantics.
// Parking (DESIGN.md §13 "Parking"): the position is claimed by a 64-bit atomicAdd on the word whose low half is
// `tail`; when the value it returns has the parked bit, the producer clears the bit, and the one whose atomicAnd still
// saw it rings the doorbell after its entry is stored: one ring per park.
__device__ __forceinline__ void ready_ring(ReadyQueue* q) {
  if ((atomicAnd(ready_tail_word(q), ~kReadyParked) & kReadyParked) == 0) return;  // another producer rang
  const unsigned long long n = atomicAdd(reinterpret_cast<unsigned long long*>(&q->rings), 1ull) + 1ull;
  uint64_t* bell = VL(q->bell);
  __threadfence_system();  // the entry, and the change before it, reach the host's view before the count moves
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(bell), "l"(n) : "memory");
}
__device__ __forceinline__ void ready_push(ReadyQueue* q, uint32_t key) {
  const unsigned long long w = atomicAdd(ready_tail_word(q), 1ull);
  const uint32_t pos = (uint32_t)w;
  uint64_t* e = ready_entries(q) + (pos & VL(q->mask));
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(e), "l"(ready_entry(key, pos)) : "memory");
  if (w & kReadyParked) ready_ring(q);
}
// The member's half is inlined into user kernels and called out of line by the library's kernels (b200_kernels.cu
// defines B200_NOTIFY_OUT_OF_LINE).  Inlined with its ring path it made k_recv and k_svc_big spill; as a call it made
// the device-call test kernels spill.  Either way, no kernel changes its registers, stack or spills.
#ifdef B200_NOTIFY_OUT_OF_LINE
static __device__ __noinline__ void notify_member(ReadyNote* n, ReadyQueue* q) {
#else
__device__ __forceinline__ void notify_member(ReadyNote* n, ReadyQueue* q) {
#endif
  __threadfence();
  if (atomicExch(&n->armed, 0u) == 1u) ready_push(q, VL(n->key));
}
__device__ __forceinline__ void notify_peer(PairDev* table, int peer_slot) {
  if (peer_slot < 0) return;
  ReadyNote* n = ready_note(table, peer_slot);
  ReadyQueue* q = VL(n->set);
  if (q == nullptr) return;
  notify_member(n, q);
}

// ======================================================================= one call by one warp, any size

__device__ __forceinline__ uint64_t warp_sum(uint64_t v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// n bytes from `src` (any alignment) to ring offset `off` (any alignment, wraps): byte stores at the <8-byte
// edges, whole words in between.  A coalesced frame gathers slices at any frame offset; the words a slice
// shares with its neighbours are written byte by byte, so no two slices store to the same byte.
__device__ __forceinline__ void warp_put_bytes(uint8_t* ring, uint64_t mask, uint64_t off, const uint8_t* src,
                                               uint64_t n, uint32_t lane) {
  uint64_t head = (8 - (off & 7)) & 7;
  if (head > n) head = n;
  if (lane < head) ring[(off + lane) & mask] = ld_sys_u8(src + lane);
  const uint64_t body = (n - head) & ~7ull;
  if (body) warp_copy_to_ring(ring, mask, (off + head) & mask, src + head, (uint32_t)body, nullptr, lane);
  const uint64_t tail = n - head - body;
  if (lane < tail) ring[(off + head + body + lane) & mask] = ld_sys_u8(src + head + body + lane);
}

// Per-slice Send planning (pair.cc:667-700).  Lane i < look holds slice i (`valid`), `len` = its bytes from
// byte_idx on.  Frame i is slice i, cut to what is left of staging (C/2) and credit at the first slice that does not
// fit; a zero-length slice stops the call.  Returns this lane's frame payload (0: no frame; the frames are lanes
// 0 .. nframes-1), `a` = the ring bytes of the frames in front of it.  kLanes: the lanes that can hold a slice.
template <int kLanes>
__device__ __forceinline__ uint64_t send_plan(bool valid, uint64_t len, uint64_t cap, uint64_t rh, uint64_t rt,
                                              uint32_t lane, uint64_t& a, uint32_t& nframes, uint64_t& wsum,
                                              uint64_t& esum) {
  const uint64_t e = valid ? encoded_size(len) : 0;
  uint64_t incl = e;
  for (int o = 1; o < kLanes; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += t;
  }
  a = incl - e;
  const uint64_t fr = free_size(cap, rh, rt), staging = cap / 2;  // send_buf_size = recv_buf_size / 2, pair.cc:104
  const uint64_t lim = staging < fr ? staging : fr;
  const uint64_t room = calc_writable(lim > a ? lim - a : 0);
  const bool fits = valid && len != 0 && len <= room;
  const unsigned bad = __ballot_sync(0xffffffffu, !fits);
  const int nfull = (kLanes < 32 || bad) ? __ffs(bad) - 1 : 32;  // (kLanes < 32: the lanes >= kLanes are "bad")
  uint64_t p = 0;
  if ((int)lane < nfull) p = len;
  else if ((int)lane == nfull && valid && len != 0) p = room;  // cut: space ran out
  nframes = __popc(__ballot_sync(0xffffffffu, p != 0));
  wsum = p;
  esum = p ? encoded_size(p) : 0;
  for (int o = 16; o > 0; o >>= 1) {
    wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
    esum += __shfl_xor_sync(0xffffffffu, esum, o);
  }
  return p;
}

// The headers and payloads of a per-slice Send call's frames (lane f < nframes holds frame f's source, payload,
// ring offset and header); footers are the caller's, after its fence.  With `eslot` the first frame's payload words
// also go to that host slot and their eager checksum contribution is returned.
__device__ __forceinline__ uint64_t send_frames(uint8_t* ring, uint64_t mask, const uint8_t* ptr, uint64_t p,
                                                uint64_t foff, uint64_t hdr, uint32_t nframes, uint8_t* eslot,
                                                uint32_t lane) {
  uint64_t cs = 0;
  for (uint32_t f = 0; f < nframes; f++) {
    const uint8_t* fsrc = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<uint64_t>(ptr), f));
    const uint32_t fp = (uint32_t)__shfl_sync(0xffffffffu, p, f);
    const uint64_t fo = __shfl_sync(0xffffffffu, foff, f);
    const uint64_t fh = __shfl_sync(0xffffffffu, hdr, f);
    if (lane == 0) *reinterpret_cast<uint64_t*>(ring + fo) = fh;  // AppendHeader
    cs ^= warp_copy_to_ring(ring, mask, (fo + 8) & mask, fsrc, fp, f == 0 ? eslot : nullptr, lane);
  }
  return cs;
}

// The receive side of a pair as one Recv call changes it (PairDev cursor fields + PairSeq::rx)
struct RxCursor {
  uint64_t head, mh, remain, acc, rx;
};
constexpr uint64_t kRecvTooBig = ~0ull;

// The ring work of one PairPollable::Recv call (ring_buffer.cc:122-191 + the internal_read_size count of
// pair.cc:270-284): at most one frame, or the rest of a partially read one, min(readable, capacity) bytes to `dst`;
// the bytes read are cleared in the reference format (header on first touch, pad + footer once the frame is
// finished), nothing is stored in the stamped one.  Returns the bytes delivered (0: nothing complete at the head),
// or kRecvTooBig -- nothing touched -- when that would exceed `limit`.  `acquire`: the probe loads order the payload
// loads behind them (a writer outside this warp).  `discard`: the frame of `capacity` bytes at the head was already
// taken from its eager slot; it is retired without a look and without a copy.  `credit`: C/2 bytes have been retired
// since the last status_report, one is due now (with c.mh).
__device__ __forceinline__ uint64_t warp_recv_frame(uint8_t* ring, uint64_t cap, bool acquire, bool stamped,
                                                    RxCursor& c, uint8_t* dst, uint64_t capacity, bool discard,
                                                    uint64_t limit, bool& credit, uint32_t lane) {
  const uint64_t mask = cap - 1;
  uint64_t r, src;
  bool open;
  if (c.remain > 0) {
    r = c.remain;
    src = c.mh;
    open = false;
  } else if (discard) {
    r = capacity;
    src = (c.head + 8) & mask;
    open = true;
  } else {  // GetReadableSize, ring_buffer.cc:67-97
    const uint64_t hdr = acquire ? ld_acquire_u64(ring + c.head) : ld_volatile_u64(ring + c.head);
    const uint32_t st = stamped ? stamp_of(c.rx) : 0;
    const uint64_t len = frame_present(hdr, cap, st);
    if (len == 0) return 0;
    const uint8_t* fp = ring + ((c.head + 8 + round_up8(len)) & mask);
    const uint64_t foot = acquire ? ld_acquire_u64(fp) : ld_volatile_u64(fp);
    if (foot != frame_footer(hdr, st)) return 0;
    r = len;
    src = (c.head + 8) & mask;
    open = true;
  }
  const uint64_t n = r < capacity ? r : capacity;  // copy_size = min(readable, capacity)
  if (n == 0) return 0;
  if (n > limit) return kRecvTooBig;
  if (!discard) warp_copy_from_ring(dst, ring, mask, src, (uint32_t)n, lane);
  __syncwarp();
  const uint64_t end = (src + n) & mask;
  uint64_t ztail = 0, mh_after = end;
  if (n == r) {
    const uint64_t up = round_up8(end);
    ztail = (up - end) + 8;
    mh_after = ((up & mask) + 8) & mask;
  }
  const uint64_t zhead = open ? 8 : 0;
  if (!stamped) warp_zero_ring(ring, mask, (src + cap - zhead) & mask, zhead + n + ztail, lane);
  if (open) {
    c.head = (c.head + 16 + round_up8(r)) & mask;  // ring_buffer.cc:140-141
    c.rx++;
  }
  c.remain = r - n;
  c.mh = mh_after;
  c.acc += zhead + n + ztail;  // internal_bytes_read
  credit = false;
  if (c.acc >= cap / 2) {  // pair.cc:276-284
    credit = true;
    c.acc = 0;
  }
  return n;
}

// ======================================================================= a call's result, published by ONE thread
//
// Shared by the CTA pipeline (send_body / recv_body: k_send, k_recv, k_cluster_send, k_cluster_recv, k_svc_big, the
// block and cluster calls) and the warp calls.  `conc`: ops of the two ends may run at the same time (kFlagConcurrent;
// always for the warp calls), so a pair's mirror is written under that pair's lock.  A pair without a mirror (an end
// claimed with B200_CLAIM_UNMIRRORED) is not locked: there is nothing to publish.

// A Send's result: the cursors and the frame counter, this end's send-side mirror, and on the loopback wire the peer's
// readiness hint and ready set.  Every footer of the call is visible to this thread (the caller's barrier).
// `written`: the payload bytes the call accepted.
__device__ __forceinline__ void send_publish(PairDev* table, int slot, uint64_t rt, bool partial, bool stamped,
                                             uint64_t tx, uint64_t written, bool conc) {
  PairDev* P = table + slot;
  VL(P->remote_tail) = rt;
  VL(P->partial_write) = partial;  // pair.cc:712
  if (stamped) VL(pair_seq(table, slot)->tx) = tx;
  PairMirror* pm = VL(P->mirror);
  mirror_lock(P, conc && pm);
  publish_mirror_tx(pm, P);
  mirror_unlock(P, conc && pm);
  const int peer_slot = VL(P->peer_slot);
  if (peer_slot < 0 || written == 0) return;
  PairDev* Q = table + peer_slot;  // loopback wire: the peer lives in this table
  PairMirror* qm = VL(Q->mirror);
  if (qm) {
    uint32_t hm;
    uint64_t rd;
    mirror_lock(Q, conc);
    rx_probe<false>(VL(Q->ring), VL(Q->cap), VL(Q->head), VL(Q->remain), rx_stamp(table, peer_slot), hm, rd);
    volatile PairMirror* vm = qm;
    vm->has_message = hm;
    vm->readable = rd;
    mirror_unlock(Q, conc);
  }
  notify_peer(table, peer_slot);
}

// The credit a Recv returns (updateStatus, pair.cc:624-641): the 16-byte status_report {mh, peer_exit = 0} into the
// peer's credit block, on the loopback wire the peer mirror's credit_head, then the peer's ready set.  The caller has
// fenced what the credit frees (the clears; stamped: the reads) before it.
__device__ __forceinline__ void credit_return(PairDev* table, PairDev* P, uint64_t mh, bool conc) {
  const int peer_slot = VL(P->peer_slot);
  PairMirror* pm = VL(P->peer_mirror);  // (loopback wire; null when the peer end is claimed unmirrored)
  PairDev* Q = conc && peer_slot >= 0 && pm ? table + peer_slot : nullptr;
  if (Q) mirror_lock(Q, true);
  asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(VL(P->peer_credit)), "l"(mh), "l"(0ull) : "memory");
  if (pm) ((volatile PairMirror*)pm)->credit_head = mh;
  if (Q) mirror_unlock(Q, true);
  notify_peer(table, peer_slot);
}

// One PairPollable::Send call (pair.cc:645-734) by one warp on pair `slot` of `table`, from the pair's state in
// the table.  Per-slice framing: <= max_sge frames, one per slice, a slice is cut only where staging (C/2) or
// credit runs out, a zero-length slice stops the call.  kSgeCoalesce: ONE frame gathering the slices of the
// kCoalesceSlices window from byte_idx on.  Stamped frames when the connection negotiated them.  Slices: device
// or pinned host memory.  Returns the payload bytes accepted, after lane 0 has published the result with
// send_publish: cursors, frame counter, the pair's mirror, on the loopback wire the peer's readiness and ready set.
__device__ inline uint64_t warp_send_call(PairDev* table, int slot, const SliceDev* slices, uint64_t n,
                                          uint64_t byte_idx, uint32_t lane) {
  PairDev* P = table + slot;
  if (VL(P->status) != kStConnected || n == 0) return 0;  // pair.cc:657
  if (ld_acquire_u32(&P->credit_exit) == 1) return 0;     // the peer left: its ring may belong to somebody else
  const uint64_t cap = VL(P->cap), mask = cap - 1;
  uint8_t* ring = VL(P->peer_ring);
  const bool sys = VL(P->wire) != 0;
  const uint32_t sgew = VL(P->max_sge);
  const bool stamped = (sgew & kSgeStamped) != 0;
  const uint64_t rt = VL(P->remote_tail);
  const uint64_t rh = ld_acquire_u64(&P->credit_head);  // credit snapshot, once (pair.cc:650); the receiver's
                                                        // clears are ordered before our frames
  PairSeq* S = pair_seq(table, slot);
  const uint64_t tx = stamped ? VL(S->tx) : 0;
  uint64_t total = 0;  // total_slice_size, pair.cc:661-664
  for (uint64_t i = lane; i < n; i += 32) total += slices[i].len;
  total = warp_sum(total) - byte_idx;
  uint64_t written = 0, esum = 0;
  uint32_t nframes = 0;
  if (!(sgew & kSgeCoalesce)) {
    const uint32_t sge = sgew & ~kSgeModeBits;
    const uint32_t look = (uint32_t)(n < sge ? n : sge);  // <= kMaxSgeLimit: one lane per slice
    const bool valid = lane < look;
    const uint8_t* ptr = nullptr;
    uint64_t len = 0;
    if (valid) {
      const uint64_t skip = lane == 0 ? byte_idx : 0;
      ptr = slices[lane].ptr + skip;
      len = slices[lane].len - skip;
    }
    uint64_t a;
    const uint64_t p = send_plan<32>(valid, len, cap, rh, rt, lane, a, nframes, written, esum);
    const uint64_t foff = (rt + a) & mask;
    const uint32_t st = stamped ? stamp_of(tx + lane) : 0;
    const uint64_t hdr = frame_header(p, st);
    send_frames(ring, mask, ptr, p, foff, hdr, nframes, nullptr, lane);
    // footers last (ring_buffer.cc:75-96): the reader may be another warp, kernel or GPU
    if (sys) __threadfence_system();
    else __threadfence();
    __syncwarp();
    if (p != 0) *reinterpret_cast<uint64_t*>(ring + ((foff + 8 + round_up8(p)) & mask)) = frame_footer(hdr, st);
  } else {
    const uint64_t look = n < kCoalesceSlices ? n : kCoalesceSlices;
    uint64_t avail = 0;
    for (uint64_t i = lane; i < look; i += 32) avail += slices[i].len;
    avail = warp_sum(avail) - byte_idx;
    const uint64_t ws = calc_writable(cap / 2), wf = calc_writable(free_size(cap, rh, rt));
    uint64_t p = avail < ws ? avail : ws;
    if (p > wf) p = wf;
    if (p) {
      const uint32_t st = stamped ? stamp_of(tx) : 0;
      uint64_t off = 0;
      for (uint64_t i = 0; i < look && off < p; i++) {
        const uint64_t skip = i == 0 ? byte_idx : 0;
        uint64_t m = slices[i].len - skip;
        if (m > p - off) m = p - off;
        if (m) warp_put_bytes(ring, mask, (rt + 8 + off) & mask, slices[i].ptr + skip, m, lane);
        off += m;
      }
      if (lane < round_up8(p) - p) ring[(rt + 8 + p + lane) & mask] = 0;  // pad
      const uint64_t hdr = frame_header(p, st);
      if (lane == 0) *reinterpret_cast<uint64_t*>(ring + rt) = hdr;
      if (sys) __threadfence_system();
      else __threadfence();
      __syncwarp();
      if (lane == 0) *reinterpret_cast<uint64_t*>(ring + ((rt + 8 + round_up8(p)) & mask)) = frame_footer(hdr, st);
      nframes = 1;
      written = p;
      esum = encoded_size(p);
    }
  }
  __syncwarp();  // (every lane's footer before lane 0 publishes)
  if (lane == 0) send_publish(table, slot, (rt + esum) & mask, written < total, stamped, tx + nframes, written, true);
  __syncwarp();
  return written;
}

// One PairPollable::Recv call (ring_buffer.cc:122-191 + pair.cc:264-286) by one warp on pair `slot` of
// `table`: at most one frame, or the rest of a partially read one, into `dst` (device or pinned host memory,
// any alignment).  Clears what it read in the reference format, stores nothing into the ring in the stamped
// one.  Lane 0 returns credit with credit_return once C/2 bytes have been retired, then publishes the cursors, the
// frame counter and the pair's mirror.
__device__ inline uint64_t warp_recv_call(PairDev* table, int slot, uint8_t* dst, uint64_t capacity, uint32_t lane) {
  PairDev* Q = table + slot;
  if (VL(Q->status) != kStConnected || capacity == 0) return 0;  // pair.cc:266-268
  const uint64_t cap = VL(Q->cap);
  uint8_t* ring = VL(Q->ring);
  const bool sys = VL(Q->wire) != 0;
  const bool stamped = (VL(Q->max_sge) & kSgeStamped) != 0;
  PairSeq* S = pair_seq(table, slot);
  RxCursor c{VL(Q->head), VL(Q->moving_head), VL(Q->remain), VL(Q->acc), stamped ? VL(S->rx) : 0};
  bool credit;
  const uint64_t n = warp_recv_frame(ring, cap, true, stamped, c, dst, capacity, false, ~0ull, credit, lane);
  if (n == 0) return 0;
  // the sender may reuse the space only once it reads as zero (stamped: once it has been read)
  if (credit) {
    if (sys) __threadfence_system();
    else __threadfence();
  }
  __syncwarp();
  if (lane == 0) {
    if (credit) credit_return(table, Q, c.mh, true);
    VL(Q->head) = c.head;
    VL(Q->moving_head) = c.mh;
    VL(Q->remain) = c.remain;
    VL(Q->acc) = c.acc;
    if (stamped) VL(S->rx) = c.rx;
    PairMirror* m = VL(Q->mirror);  // null: claimed unmirrored, nothing to publish
    if (m) {
      uint32_t hm;
      uint64_t rd;
      mirror_lock(Q, true);
      if (sys) rx_probe<true>(ring, cap, c.head, c.remain, stamped ? stamp_of(c.rx) : 0, hm, rd);
      else rx_probe<false>(ring, cap, c.head, c.remain, stamped ? stamp_of(c.rx) : 0, hm, rd);
      publish_mirror_rx(m, Q, hm, rd);
      mirror_unlock(Q, true);
    }
  }
  __syncwarp();
  return n;
}

// GetReadableSize / HasMessage / HasPendingWrites of pair `slot` from the device truth (pair.cc:288-303)
__device__ inline uint64_t warp_readable(PairDev* table, int slot, uint32_t* has_msg) {
  PairDev* P = table + slot;
  uint32_t hm = 0;
  uint64_t rd = 0;
  if (VL(P->status) == kStConnected)
    rx_probe<true>(VL(P->ring), VL(P->cap), VL(P->head), VL(P->remain), rx_stamp(table, slot), hm, rd);
  if (has_msg) *has_msg = hm;
  return rd;
}

// ======================================================================= poll, status, writable, Disconnect

// The kEv* readiness of pair `slot`, by ONE lane: the per-pair body of Poller::begin_polling (poller.cc:66-101) and of
// the engine's busy-poll window (ev_epollex_rdma_bpev_linux.cc:1104-1145).  A CONNECTED pair whose peer has left is
// READABLE (the read that reports the close); otherwise READABLE on HasMessage, WRITABLE on HasPendingWrites.  An
// ERROR or HALF_CLOSED row is READABLE.  Acquire loads: the ring and the credit word may be written from outside this
// GPU.  k_poll_scan and b200_warp_poll both run this.  kPublish (k_poll_scan): also refresh the host mirror of a pair
// off the loopback wire, whose bytes and credit nothing on this GPU publishes; a lock-free scan beside the ops of the
// pair would overwrite a newer view with an older one, so the device API never publishes from here.
template <bool kPublish>
__device__ __forceinline__ uint32_t poll_events(PairDev* __restrict__ pairs, int slot) {
  PairDev* P = &pairs[slot];
  uint32_t ev = 0;
  const uint32_t st = *(volatile uint32_t*)&P->status;
  if (st == kStConnected) {
    const uint32_t exit_flag = ld_acquire_u32(&P->credit_exit);
    uint32_t hm;
    uint64_t rd;
    rx_probe(P->ring, P->cap, *(volatile uint64_t*)&P->head, *(volatile uint64_t*)&P->remain, rx_stamp(pairs, slot),
             hm, rd);
    const uint32_t pw = *(volatile uint32_t*)&P->partial_write;
    if (exit_flag == 1) {
      ev = kEvReadable;  // HalfClosed: force a read event (engine :1130-1137)
    } else {
      if (hm) ev |= kEvReadable;
      if (pw) ev |= kEvWritable;
    }
    // On the loopback wire the kernels that land bytes / return credit refresh the mirrors themselves, in
    // order with their own completion; a scan running beside them could only overwrite that with an older
    // view (and b200_pair_recv / send answer "nothing to do" from the mirror without launching anything).
    if (kPublish && P->peer_slot < 0) {
      publish_mirror_rx(P->mirror, P, hm, rd);
      publish_mirror_tx(P->mirror, P);
    }
  } else if (st == kStError || st == kStHalfClosed) {
    ev = kEvReadable;
  }
  return ev;
}

// get_status (pair.cc:349-375) as far as the device can tell: the row's status, HALF_CLOSED on a CONNECTED row whose
// peer has written peer_exit.  (Whether the peer's process still exists is a host question: b200_pair_status.)
__device__ __forceinline__ uint32_t pair_status(PairDev* table, int slot) {
  PairDev* P = table + slot;
  const uint32_t st = VL(P->status);
  return st == kStConnected && ld_acquire_u32(&P->credit_exit) == 1 ? kStHalfClosed : st;
}

// GetWritableSize (pair.cc:294-301) from the device state
__device__ __forceinline__ uint64_t pair_writable(PairDev* table, int slot) {
  PairDev* P = table + slot;
  return writable_size(VL(P->cap), ld_acquire_u64(&P->credit_head), VL(P->remote_tail));
}

// PairPollable::Disconnect (pair.cc:325-347) of a device-owned end, by one warp.  Returns 0 and changes nothing on a
// row that is not CONNECTED.  Otherwise: (1) a fence (system scope on the nvlink wire), so every frame and clear this
// end wrote is visible before the peer can see the close; (2) unless the peer has left already, the 16-byte
// status_report {moving_head, peer_exit = 1} into the peer's credit block -- on the loopback wire with the peer's
// mirror, under the peer's mirror lock; (3) the row's status = DISCONNECTED, so every later call on the end refuses;
// (4) the end's mirror flag that tells the host the rest of the Disconnect is due at the release (an end claimed
// unmirrored has no mirror: its release finds the DISCONNECTED row instead).  Returns 1.
__device__ inline int warp_disconnect(PairDev* table, int slot, uint32_t lane) {
  PairDev* P = table + slot;
  uint32_t st = 0;
  if (lane == 0) st = VL(P->status);
  st = __shfl_sync(0xffffffffu, st, 0);
  if (st != kStConnected) return 0;
  if (lane == 0) {
    if (VL(P->wire) != 0) __threadfence_system();
    else __threadfence();
    if (ld_acquire_u32(&P->credit_exit) != 1) {
      const uint64_t mh = VL(P->moving_head);
      const int peer_slot = VL(P->peer_slot);
      PairMirror* pm = VL(P->peer_mirror);
      PairDev* Q = peer_slot >= 0 && pm ? table + peer_slot : nullptr;
      if (Q) mirror_lock(Q, true);
      asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(VL(P->peer_credit)), "l"(mh), "l"(1ull) : "memory");
      if (pm) {
        volatile PairMirror* vm = pm;
        vm->credit_head = mh;
        vm->peer_exit = 1;
      }
      if (Q) mirror_unlock(Q, true);
      notify_peer(table, peer_slot);
    }
    VL(P->status) = kStDisconnected;
    PairMirror* m = VL(P->mirror);  // null (claimed unmirrored): the release reads the row's status instead
    if (m) {
      __threadfence_system();
      ((volatile PairMirror*)m)->dev_closed = 1;
    }
  }
  __syncwarp();
  return 1;
}

// ======================================================================= ready sets: the consumers (any number of warps)

// A member is ready when poll_events reports READABLE, or when it has a pending write and credit for at least one
// frame: the inverse of the host's "this Send cannot accept a byte" rule.  (The Poller's level-triggered WRITABLE on
// partial_write alone would hand a blocked sender back to an edge-triggered consumer at once, again and again.)
__device__ __forceinline__ uint32_t ready_events(PairDev* table, int slot) {
  const uint32_t ev = poll_events<false>(table, slot);
  uint32_t out = ev & kEvReadable;
  if (ev & kEvWritable) {  // (CONNECTED, the peer has not left, partial_write)
    PairDev* P = table + slot;
    const uint64_t cap = VL(P->cap);
    const uint64_t fr = free_size(cap, ld_acquire_u64(&P->credit_head), VL(P->remote_tail));
    if (calc_writable(fr < cap / 2 ? fr : cap / 2) != 0) out |= kEvWritable;
  }
  return out;
}

// Up to `max` keys from the head of the queue into keys[]; stops at the first position whose entry has not been
// stored yet.  Returns how many, every lane; keys[] beyond that count are unspecified.  Any number of consumer warps
// may take from one queue at once: the run [h, h + n) read from head h becomes this warp's by atomicCAS(head, h,
// h + n), and a lost CAS (another consumer took first) reads again from the new head.  An empty run costs no atomic.
// A won CAS returns the right keys: an entry is accepted only when its tag names its position, a slot is rewritten
// only for position p + size, and b200_ready_set_add keeps entries queued plus members below size, so while head ==
// h no producer holds a position at or beyond h + size; a CAS from h that wins saw head still at h.  (head is a
// 32-bit counter: an ABA needs 2^32 taken entries between one warp's load and its CAS.)  A ticket atomicAdd(head)
// would instead own positions whose producer may not have stored the entry yet, and the take would have to wait.
// `retries` (may be null): lane 0 adds the lost CASes.
__device__ inline uint32_t ready_take(ReadyQueue* q, uint32_t* keys, uint32_t max, uint32_t lane,
                                      uint32_t* retries = nullptr) {
  const uint32_t mask = VL(q->mask);
  for (;;) {
    uint32_t head = 0;
    if (lane == 0) head = VL(q->head);
    head = __shfl_sync(0xffffffffu, head, 0);
    uint32_t n = 0;
    while (n < max) {
      const uint32_t i = n + lane;
      bool ok = false;
      uint64_t e = 0;
      if (i < max) {
        const uint32_t pos = head + i;
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(e) : "l"(ready_entries(q) + (pos & mask)) : "memory");
        ok = ready_entry_at(e, pos);
      }
      const unsigned bad = __ballot_sync(0xffffffffu, !ok);
      const uint32_t run = bad ? __ffs(bad) - 1 : 32;
      if (lane < run) keys[i] = (uint32_t)e;
      n += run;
      if (run < 32) break;
    }
    if (n == 0) return 0;
    uint32_t won = 0;
    if (lane == 0) {
      won = atomicCAS(&q->head, head, head + n) == head;
      if (!won && retries) (*retries)++;
    }
    __syncwarp();
    if (__shfl_sync(0xffffffffu, won, 0)) return n;
  }
}

// The consumer is done with member `slot` of `q`: armed = 1, a fence, then the probe.  Ready and the exchange won:
// the member's events (the consumer keeps it, nothing is queued).  Otherwise 0: a producer that saw armed == 1 has
// queued the key, or nothing is pending and the next change will.  0 as well for an end that is not a member of `q`.
// Once armed = 1 is stored, another consumer warp may take the member's new entry while this probe still runs: the
// probe (poll_events, free_size) only reads, so the new holder's calls never run beside a write of this warp's.
__device__ inline uint32_t ready_rearm(ReadyQueue* q, PairDev* table, int slot, uint32_t lane) {
  uint32_t ev = 0;
  if (lane == 0) {
    ReadyNote* n = ready_note(table, slot);
    if (VL(n->set) == q) {
      VL(n->armed) = 1u;
      __threadfence();
      ev = ready_events(table, slot);
      if (ev && atomicExch(&n->armed, 0u) != 1u) ev = 0;
    }
  }
  return __shfl_sync(0xffffffffu, ev, 0);
}

// Park the set (DESIGN.md §13 "Parking"), by the one warp that still takes from it, holding no member: set the parked
// bit, and compare the tail it covered with head.  Equal: 0, the set is parked and the next push rings.  Not equal:
// entries are queued, so clear the bit again; if it was still set no producer rang, and the caller has work (1).  If a
// producer cleared it first, its ring is on its way and the set counts as parked (0).  Park and push are
// read-modify-writes of one word, so their order is that word's coherence order: no fence is needed.
// ready_park_one is the park by one thread (k_ready_park runs it for b200_ready_set_park).
__device__ inline uint32_t ready_park_one(ReadyQueue* q) {
  const unsigned long long w = atomicOr(ready_tail_word(q), kReadyParked);
  if ((uint32_t)w == VL(q->head)) return 0;
  return (atomicAnd(ready_tail_word(q), ~kReadyParked) & kReadyParked) ? 1u : 0u;
}
__device__ inline uint32_t ready_park(ReadyQueue* q, uint32_t lane) {
  const uint32_t busy = lane == 0 ? ready_park_one(q) : 0u;
  return __shfl_sync(0xffffffffu, busy, 0);
}

}  // namespace b200
