// b200_kernels.cu -- sm_90a (H100) kernels of the RDMA_BPEV endpoint hot path.
//
//   k_send       gather/encode: grpc_slice list -> [len][payload][pad][~0] frames
//                written straight at the remote tail of the peer's HBM ring
//                (replaces PairPollable::Send pair.cc:645-734 + AppendHeader/
//                Payload/Footer ring_buffer.h:84-99 + GetWriteRequests
//                ring_buffer.cc:261-330 + the NIC's RDMA write)
//   k_recv       deframe/scatter + clear-on-read + credit write-back (replaces
//                RingBufferPollable::Read ring_buffer.cc:122-191 and
//                PairPollable::Recv/updateStatus pair.cc:264-286,624-641)
//   k_poll_scan  readiness scan (replaces the per-pair body of
//                Poller::begin_polling poller.cc:66-101 and of the engine's
//                busy-poll window ev_epollex_rdma_bpev_linux.cc:1104-1145)
//
// Pure indexing / memcpy work: HBM-bound, no tensor cores.  One CTA serves one
// (pair, op): warp 0 runs the reference's integer logic with warp scans and
// publishes 4 KiB work items; the mover warps pull every item's source bytes
// into shared memory with the bulk-copy engine (cp.async.bulk + mbarrier
// complete_tx, several stages in flight per warp, so the HBM read latency is
// never held in registers) and write them out with bulk stores, re-aligning
// the stage in place through a funnel shift when source and destination
// differ mod 16 (gRPC slices sit at odd offsets, ring payloads at 8 mod 16).
// Byte granularity only at the <16-byte edges of a copy.
#include <cuda_runtime.h>
#include <stdint.h>

#include <mutex>

#include "b200_dev.cuh"
#include "b200_warp.cuh"  // memory helpers, readiness + mirrors, warp movers (shared with include/b200_device.cuh)

#ifndef B200_RECV_PROXY_FENCE
#define B200_RECV_PROXY_FENCE 1
#endif

namespace b200 {

// ------------------------------------------------------------ memory helpers

__device__ __forceinline__ uint4 ld_stream16(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
// ring reads must not use the non-coherent path: the ring is written by other
// kernels / the wire while we run
__device__ __forceinline__ uint4 ld_ring16(const void* p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

// ------------------------------------------------- bulk-copy engine (TMA) helpers

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// global -> shared, completion counted in bytes on `bar`.  dst, src 16-byte aligned, bytes % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* sdst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(sdst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// order this thread's earlier generic-proxy observations of global memory before its bulk copies
__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }
// shared -> global, byte-exact; completion is tracked in this thread's bulk groups.  gdst, ssrc 16-byte
// aligned, bytes % 16 == 0.
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* ssrc, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(ssrc)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }

// In place: vector i of the 16-byte aligned shared array sv becomes source bytes [16 i + m, 16 i + m + 16),
// m = 4 K + r/8 (a shift towards lower addresses).  Warp-cooperative, one 512-byte stripe at a time:
// every lane reads its two vectors before any lane of the stripe writes; the next stripe's reads start
// at the first vector this one did not write.
template <int K>
__device__ __forceinline__ void realign_vectors(uint4* sv, uint32_t nvec, uint32_t r, uint32_t lane) {
  for (uint32_t j = 0; j < nvec; j += 32) {
    const uint32_t i = j + lane;
    uint4 o = make_uint4(0, 0, 0, 0);
    if (i < nvec) {
      const uint4 A = sv[i], B = sv[i + 1];
      uint32_t x0, x1, x2, x3, x4;
      if (K == 0) { x0 = A.x; x1 = A.y; x2 = A.z; x3 = A.w; x4 = B.x; }
      else if (K == 1) { x0 = A.y; x1 = A.z; x2 = A.w; x3 = B.x; x4 = B.y; }
      else if (K == 2) { x0 = A.z; x1 = A.w; x2 = B.x; x3 = B.y; x4 = B.z; }
      else { x0 = A.w; x1 = B.x; x2 = B.y; x3 = B.z; x4 = B.w; }
      o.x = __funnelshift_r(x0, x1, r);
      o.y = __funnelshift_r(x1, x2, r);
      o.z = __funnelshift_r(x2, x3, r);
      o.w = __funnelshift_r(x3, x4, r);
    }
    __syncwarp();
    if (i < nvec) sv[i] = o;
  }
}

// Warp-cooperative copy of n bytes from shared memory (16-byte aligned base `sbase`, byte offset
// `soff`) to global memory at any alignment.  The <16-byte edges are stored byte by byte; the
// aligned interior is realigned in place to the destination's phase and lane 0 issues one bulk store
// for it (committed by the caller).  The stage holds at least one 16-byte block past the last source
// byte's block start, so vector i+1 is always readable.  Bytes of the stage below soff + n may be
// overwritten; the bytes from the block of soff + n on are left as they were.
__device__ __forceinline__ void smem_to_global(uint8_t* dst, uint8_t* sbase, uint32_t soff, uint32_t n,
                                               uint32_t lane) {
  if (n == 0) return;
  uint32_t head = (16 - (uint32_t)(reinterpret_cast<uintptr_t>(dst) & 15)) & 15;
  if (head > n) head = n;
  const uint32_t nvec = (n - head) >> 4;
  const uint32_t tail = n - head - (nvec << 4);
  if (lane < head) dst[lane] = sbase[soff + lane];
  if (lane < tail) dst[head + (nvec << 4) + lane] = sbase[soff + head + (nvec << 4) + lane];
  if (nvec == 0) return;
  const uint32_t vs = soff + head, m = vs & 15;
  uint4* sv = reinterpret_cast<uint4*>(sbase + (vs - m));
  if (m != 0) {
    __syncwarp();  // the edge bytes are read before the realignment overwrites them
    const uint32_t r = (m & 3) * 8;
    switch (m >> 2) {
      case 0: realign_vectors<0>(sv, nvec, r, lane); break;
      case 1: realign_vectors<1>(sv, nvec, r, lane); break;
      case 2: realign_vectors<2>(sv, nvec, r, lane); break;
      default: realign_vectors<3>(sv, nvec, r, lane); break;
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> the bulk store's reads
    __syncwarp();
  }
  if (lane == 0) bulk_s2g(dst + head, sv, nvec << 4);
}

// Warp-cooperative zero fill of n bytes at p (any alignment): byte stores at the <16-byte edges, bulk
// stores from the zero block `zero` (kZeroBytes of shared memory) for the aligned interior, issued by
// lane 0 (committed by the caller).
constexpr uint32_t kZeroBytes = 1024;
__device__ __forceinline__ void coop_zero(uint8_t* p, uint64_t n, const uint8_t* zero, uint32_t lane) {
  if (n == 0) return;
  uint64_t head = (16 - (reinterpret_cast<uintptr_t>(p) & 15)) & 15;
  if (head > n) head = n;
  if (lane < head) p[lane] = 0;
  p += head;
  n -= head;
  const uint64_t body = n & ~15ull;
  if (lane < n - body) p[body + lane] = 0;
  if (lane == 0)
    for (uint64_t o = 0; o < body; o += kZeroBytes)
      bulk_s2g(p + o, zero, body - o < kZeroBytes ? (uint32_t)(body - o) : kZeroBytes);
}

// =========================================================================
// Producer / mover skeleton shared by k_send and k_recv
// =========================================================================
//
// One CTA per (pair, op).  Warp 0 is the producer: it runs the reference's
// integer logic (Send planning / frame-list walking) ahead of the data and
// publishes 4 KiB work items into a ticket ring in shared memory.  The other
// warps are movers.  A mover owns kDepth private stages in shared memory: it
// takes a ticket, starts the bulk copy of that item's source bytes into a free
// stage (completion counted on the stage's mbarrier) and only then turns to its
// oldest landed stage and writes it out, so every mover keeps up to kDepth x
// 4 KiB of HBM reads in flight without holding them in registers.  There is no
// CTA barrier on the steady-state path; a "segment" ends only where the
// protocol needs everything before it to be finished: the footer flush of Send,
// the credit write of Recv, the end of the op.

#ifndef B200_MOVERS
#define B200_MOVERS 8
#endif
#ifndef B200_DEPTH
#define B200_DEPTH 3
#endif
#ifndef B200_CHUNK
#define B200_CHUNK 4096
#endif
constexpr int kMovers = B200_MOVERS;            // mover warps per CTA
constexpr int kThreads = 32 * (1 + kMovers);    // + the producer warp
constexpr int kDepth = B200_DEPTH;                     // stages (bulk copies in flight) per mover warp
constexpr uint32_t kChunk = B200_CHUNK;             // payload bytes per work item
constexpr uint32_t kStageBytes = kChunk + 32;   // + up to 15 bytes of alignment slack on either side
constexpr uint32_t kStageTotal = kMovers * kDepth * kStageBytes;  // dynamic shared memory per CTA
constexpr uint32_t kQI = 128;                   // ticket ring entries (descriptor look-ahead)

struct WorkItem {      // 32 bytes
  uint64_t a;          // send: source pointer          recv: ring offset of the payload bytes
  uint64_t b;          // send: ring offset (payload)   recv: offset in the destination
  uint64_t c;          // send: header value (chunk 0)  recv: zhead | ztail << 16
  uint32_t n;          // bytes
  uint32_t ready;      // ticket: item id + 1 when published, 0 when free
};

struct PipeCtl {
  uint32_t next;         // next item id to claim
  uint32_t total_items;  // valid once seg_done
  uint32_t seg_done;
  uint32_t op_done;
};

// Shared by every kernel of this file: the ticket ring, the stage barriers, the zero block the Recv movers
// clear from, and the stages (dynamic shared memory).
struct PipeSmem {
  WorkItem q[kQI];
  PipeCtl ctl;
  uint64_t bars[kMovers * kDepth];
  uint4 zero[kZeroBytes / 16];
};

__device__ __forceinline__ uint32_t ld_shared_volatile(const uint32_t* p) { return *(const volatile uint32_t*)p; }

// producer side: wait for the slot of item `id`, fill it, publish
__device__ __forceinline__ void publish_item(WorkItem* q, uint32_t id, uint64_t a, uint64_t b, uint64_t c,
                                             uint32_t n) {
  WorkItem* slot = &q[id % kQI];
  while (ld_shared_volatile(&slot->ready) != 0) __nanosleep(20);
  slot->a = a;
  slot->b = b;
  slot->c = c;
  slot->n = n;
  __threadfence_block();
  *(volatile uint32_t*)&slot->ready = id + 1;
}

// Callers pass a __syncthreads before the movers run.
__device__ __forceinline__ void movers_init(PipeSmem& pipe, uint32_t tid) {
  if (tid < kMovers * kDepth) mbar_init(&pipe.bars[tid], 1);
  for (uint32_t i = tid; i < kZeroBytes / 16; i += kThreads) pipe.zero[i] = make_uint4(0, 0, 0, 0);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// Mover warp, one segment.  Move::issue (lane 0) starts the bulk copy of an item into a stage;
// Move::process (whole warp) writes a landed stage out.  The item's descriptor stays in its
// ticket-ring slot until it has been written out; the next ticket is always claimed ahead of
// time so that a freed stage is refilled without waiting for the shared counter.  phase_bits
// carries the stages' mbarrier parities from segment to segment.
template <class Move>
__device__ __forceinline__ void mover_run(const Move& mv, WorkItem* q, PipeCtl* ctl, uint8_t* stages, uint64_t* bars,
                                          uint32_t& phase_bits, uint32_t lane) {
  static_assert(kQI <= 256 && kDepth <= 8, "slot_of packs one byte per stage");
  uint32_t head = 0, tail = 0, ticket = 0;
  uint64_t slot_of = 0;  // ticket-ring slot of the item in stage s, one byte per stage
  bool drained = false;
  if (lane == 0) ticket = atomicAdd(&ctl->next, 1u);
  while (true) {
    // ---- fill: start copies into free stages while published items are available
    while (!drained && tail - head < (uint32_t)kDepth) {
      uint32_t st = 0;  // 0 = ticket not published yet, 1 = copy started, 2 = segment drained
      if (lane == 0) {
        const uint32_t si = ticket % kQI;
        WorkItem* slot = &q[si];
        if (ld_shared_volatile(&slot->ready) == ticket + 1) {
          st = 1;
        } else if (ld_shared_volatile(&ctl->seg_done) && ticket >= ld_shared_volatile(&ctl->total_items)) {
          st = ld_shared_volatile(&slot->ready) == ticket + 1 ? 1 : 2;  // re-check: published in between?
        }
        if (st == 1) {
          __threadfence_block();
          const uint32_t s = tail % kDepth;
          // the stage is refilled only once the bulk stores of its previous item have read it
          asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
          mv.issue(slot->a, slot->n, stages + s * kStageBytes, &bars[s]);
          st |= si << 8;
          ticket = atomicAdd(&ctl->next, 1u);  // claim ahead
        }
      }
      st = __shfl_sync(0xffffffffu, st, 0);
      if ((st & 3) == 1) {
        const uint32_t sh = 8 * (tail % kDepth);
        slot_of = (slot_of & ~(0xffull << sh)) | ((uint64_t)(st >> 8) << sh);
        tail++;
      } else {
        drained = (st & 3) == 2;
        break;
      }
    }
    __syncwarp();
    if (head == tail) {
      if (drained) break;
      __nanosleep(32);
      continue;
    }
    // ---- write out the oldest stage
    const uint32_t s = head % kDepth;
    const uint32_t par = (phase_bits >> s) & 1u;
    while (!mbar_try_wait(&bars[s], par)) {
    }
    phase_bits ^= 1u << s;
    WorkItem* w = &q[(uint32_t)(slot_of >> (8 * s)) & 0xffu];
    const uint64_t ia = w->a, ib = w->b, ic = w->c;
    const uint32_t in = w->n;
    mv.process(ia, ib, ic, in, stages + s * kStageBytes, lane);
    __syncwarp();  // every lane is done with the stage and the descriptor before they are reused
    if (lane == 0) {
      bulk_commit();                            // the item's bulk stores: one group
      *(volatile uint32_t*)&w->ready = 0;  // the ticket-ring slot may be refilled
    }
    head++;
  }
  // The segment's bulk stores are complete and ordered before the generic-proxy fence and barrier that
  // end the segment (footers, credit, the op's answer), so nobody sees those before the bytes.
  if (lane == 0) {
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
    fence_proxy_async_global();
  }
  __syncwarp();
}

// =========================================================================
// k_send
// =========================================================================

constexpr uint32_t kTiny = 32;      // frames up to this size bypass the movers
constexpr uint32_t kFootCap = 1024;  // footers buffered per segment (ring offsets / 8)
// Stamped mode: the same buffer holds kFootCap / 2 entries of (ring offset / 8) | p << 32; frame i of the
// segment carries the stamp of frame PS.tx (at the segment's start) + i, so the footer ~header follows.
__device__ __forceinline__ void foot_put(uint32_t* foot8, bool stamped, uint32_t i, uint64_t off, uint64_t p) {
  if (stamped) reinterpret_cast<uint64_t*>(foot8)[i] = (off >> 3) | p << 32;
  else foot8[i] = (uint32_t)(off >> 3);
}

struct SendPlanState {  // producer-only
  uint64_t rt, cap, staging, total_left, written_total, ncalls, cur, bidx, last_rh;
  uint64_t tx;  // stamped mode: frames written so far (PairSeq::tx)
  uint32_t partial, max_sge, coalesce, stamped;
};

struct SendCallScratch {  // frames of the call being published
  const uint8_t* src[kMaxSgeLimit];
  uint64_t len[kMaxSgeLimit];
  uint64_t off[kMaxSgeLimit];
  uint32_t first_item[kMaxSgeLimit + 1];
};

// Producer: plan PairPollable::Send calls (pair.cc:645-734) one after another and publish
// their frames as work items until the op is finished or the footer buffer is full.  kStamped: stamped
// frames (a separate instantiation, so the reference-format planner is unchanged).
template <bool kStamped>
__device__ __noinline__ void send_produce_segment(const SendOpDev& op, const PairDev* P, uint8_t* ring,
                                                  SendPlanState& S, SendCallScratch& CS, WorkItem* q, PipeCtl* ctl,
                                                  uint32_t* foot8, uint32_t* nfoot_out, uint32_t lane) {
  const uint64_t cap = S.cap, mask = cap - 1;
  uint32_t base_item = 0, nfoot = 0;
  bool op_done = false;
  constexpr bool stamped = kStamped;
  const uint32_t fcap = stamped ? kFootCap / 2 : kFootCap;
  while (nfoot + kMaxSgeLimit <= fcap) {
    const uint64_t rt = S.rt, tx0 = S.tx;
    // credit snapshot, once per call (pair.cc:650).  The receiver publishes new credit with a
    // system-scope release after zeroing the space; the matching acquire is only needed when the
    // value moved, i.e. when this call may write into space that was just cleared.
    const uint64_t rh = ld_volatile_u64(&P->credit_head);
    if (rh != S.last_rh) {
      if (P->wire != 0) __threadfence_system();
      else __threadfence();  // loopback wire: the credit writer is a kernel on this GPU
      S.last_rh = rh;  // every lane writes the same value
    }
    const uint64_t cur = S.cur, bidx = S.bidx;
    const uint64_t idx = cur + lane;
    const bool valid = lane < S.max_sge && idx < op.nreal;  // never past the slices that may be dereferenced
    const uint8_t* ptr = nullptr;
    uint64_t len = 0;
    if (valid) {
      SliceDev sl = op.slices[idx];
      const uint64_t skip = lane == 0 ? bidx : 0;
      ptr = sl.ptr + skip;
      len = sl.len - skip;
    }
    const uint64_t e = valid ? encoded_size(len) : 0;
    uint64_t incl = e;
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= (uint32_t)o) incl += t;
    }
    const uint64_t a = incl - e;  // staging / ring bytes consumed before this slice
    // min(CWS(send_buf_free), CWS(recv_buf_free)) (pair.cc:676-681): both shrink by `a`
    const uint64_t fr = free_size(cap, rh, rt);
    const uint64_t lim = S.staging < fr ? S.staging : fr;
    const uint64_t room = calc_writable(lim > a ? lim - a : 0);
    const bool fits = valid && len != 0 && len <= room;
    const unsigned bad = __ballot_sync(0xffffffffu, !fits);
    const int first_bad = __ffs(bad) - 1;
    const int nfull = first_bad < 0 ? 32 : first_bad;
    uint64_t p = 0;
    if ((int)lane < nfull) p = len;
    else if ((int)lane == nfull && valid && len != 0) p = room;  // cut: space ran out
    const unsigned fmask = __ballot_sync(0xffffffffu, p != 0);
    const uint32_t nframes = __popc(fmask);  // frames are lanes 0..nframes-1
    uint64_t wsum = p, esum = p ? encoded_size(p) : 0;
    // Frames of <= kTiny bytes (chttp2's 9-byte DATA frame headers are every other slice) are
    // written by the planner lane itself: they would otherwise occupy a mover stage for a full
    // trip to memory each.
    const bool tiny = p != 0 && p <= kTiny;
    const uint32_t items = (p && !tiny) ? (uint32_t)((p + kChunk - 1) / kChunk) : 0;
    uint32_t items_incl = items;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, items_incl, o);
      if (lane >= (uint32_t)o) items_incl += t;
    }
    for (int o = 16; o > 0; o >>= 1) {
      wsum += __shfl_xor_sync(0xffffffffu, wsum, o);
      esum += __shfl_xor_sync(0xffffffffu, esum, o);
    }
    const uint32_t nitems = __shfl_sync(0xffffffffu, items_incl, 31);
    const uint64_t cut_p = __shfl_sync(0xffffffffu, p, nfull < 32 ? nfull : 0);
    const uint64_t foff = (rt + a) & mask;
    const uint64_t hdr = frame_header(p, stamped ? stamp_of(tx0 + lane) : 0);  // frames are lanes 0..nframes-1
    CS.first_item[lane] = items_incl - items;
    if (p) {
      CS.src[lane] = ptr;
      CS.len[lane] = p;
      CS.off[lane] = foff;
      foot_put(foot8, stamped, nfoot + lane, (foff + 8 + round_up8(p)) & mask, p);
    }
    if (tiny) {
      uint64_t w[kTiny / 8];
#pragma unroll
      for (int k = 0; k < (int)(kTiny / 8); k++) w[k] = 0;
#pragma unroll
      for (int i = 0; i < (int)kTiny; i++)
        if ((uint64_t)i < p) w[i >> 3] |= (uint64_t)__ldg(ptr + i) << (8 * (i & 7));
      *reinterpret_cast<uint64_t*>(ring + foff) = hdr;  // AppendHeader
      // payload words (8-byte aligned in the ring; pad bytes are never delivered)
#pragma unroll
      for (int k = 0; k < (int)(kTiny / 8); k++)
        if ((uint64_t)(8 * k) < p) *reinterpret_cast<uint64_t*>(ring + ((foff + 8 + 8 * k) & mask)) = w[k];
    }
    if (lane == 0) {
      CS.first_item[32] = nitems;
      S.rt = (rt + esum) & mask;
      S.tx = tx0 + nframes;
      S.partial = wsum < S.total_left;  // pair.cc:712
      S.total_left -= wsum;
      S.written_total += wsum;
      if (wsum) S.ncalls++;
      // cursor advance (rdma_flush, rdma_bp_posix.cc:480-493)
      uint64_t nb = 0;
      if (nfull < 32 && nframes > (uint32_t)nfull) nb = (nfull == 0 ? bidx : 0) + cut_p;  // cut slice stays current
      else if (nfull == 0) nb = bidx;                                                    // nothing consumed
      S.cur = cur + nfull;
      S.bidx = nb;
    }
    __syncwarp();
    nfoot += nframes;
    const unsigned big = __ballot_sync(0xffffffffu, items > 8);
    if (!big && nitems <= kQI) {
      // frame-parallel: lane f publishes the chunks of its own frame straight from registers.
      // (nitems <= kQI: no lane can wait for a ticket-ring slot that an item of this same call
      // still has to vacate.)
      const uint32_t first = items_incl - items;
      for (uint32_t t = 0; t < items; t++) {
        const uint64_t c0 = (uint64_t)t * kChunk;
        uint64_t n = p - c0;
        if (n > kChunk) n = kChunk;
        publish_item(q, base_item + first + t, reinterpret_cast<uint64_t>(ptr + c0), (foff + 8 + c0) & mask,
                     c0 == 0 ? hdr : 0, (uint32_t)n);
      }
    } else
    // publish this call's items in id order, 32 at a time
    for (uint32_t it = lane; it < nitems; it += 32) {
      uint32_t f = 0;
      while (f + 1 < nframes && CS.first_item[f + 1] <= it) f++;
      const uint64_t c0 = (uint64_t)(it - CS.first_item[f]) * kChunk;
      const uint64_t flen = CS.len[f];
      uint64_t n = flen - c0;
      if (n > kChunk) n = kChunk;
      publish_item(q, base_item + it, reinterpret_cast<uint64_t>(CS.src[f] + c0), (CS.off[f] + 8 + c0) & mask,
                   c0 == 0 ? frame_header(flen, stamped ? stamp_of(tx0 + f) : 0) : 0, (uint32_t)n);
    }
    __syncwarp();
    base_item += nitems;
    const bool last = (wsum == 0) || !(op.flags & kFlagUntilBlocked) || S.total_left == 0;
    if (last) {
      op_done = true;
      break;
    }
  }
  if (lane == 0) {
    *nfoot_out = nfoot;
    ctl->total_items = base_item;
    ctl->op_done = op_done ? 1u : 0u;
    __threadfence_block();
    *(volatile uint32_t*)&ctl->seg_done = 1;
  }
  __syncwarp();
}

// Producer, coalesced framing (B200_SEND_COALESCE, DESIGN.md §2): every Send call writes ONE frame that
// gathers the bytes of the slices [cur, cur + kCoalesceSlices) from byte `bidx` on, p = min(those bytes,
// CWS(staging), CWS(free)).  Two walks over the window, 32 slices at a time with a running prefix: the
// first finds p, the second publishes each slice's part of the frame at payload offset `prefix` and finds
// where the cursor stops.  Slices share 8-byte words of the frame, so nothing here writes whole words
// of payload: short parts are stored byte by byte by the planner lane, longer ones go to the movers,
// whose stores are byte-exact at the edges of an item.
template <bool kStamped>
__device__ __noinline__ void send_produce_coalesced(const SendOpDev& op, const PairDev* P, uint8_t* ring,
                                                    SendPlanState& S, SendCallScratch& CS, WorkItem* q, PipeCtl* ctl,
                                                    uint32_t* foot8, uint32_t* nfoot_out, uint32_t lane) {
  const uint64_t cap = S.cap, mask = cap - 1;
  uint32_t base_item = 0, nfoot = 0;
  bool op_done = false;
  constexpr bool stamped = kStamped;
  const uint32_t fcap = stamped ? kFootCap / 2 : kFootCap;
  while (nfoot < fcap) {
    const uint64_t rt = S.rt;
    const uint64_t rh = ld_volatile_u64(&P->credit_head);  // credit snapshot, once per call (see above)
    if (rh != S.last_rh) {
      if (P->wire != 0) __threadfence_system();
      else __threadfence();
      S.last_rh = rh;
    }
    const uint64_t cur = S.cur, bidx = S.bidx;
    const uint64_t wend = op.nreal < cur + kCoalesceSlices ? op.nreal : cur + kCoalesceSlices;
    const uint64_t ws = calc_writable(S.staging), wf = calc_writable(free_size(cap, rh, rt));
    const uint64_t pmax = ws < wf ? ws : wf;
    uint64_t p = 0;
    for (uint64_t g = cur; g < wend && p < pmax; g += 32) {
      const uint64_t idx = g + lane;
      uint64_t len = idx < wend ? op.slices[idx].len - (idx == cur ? bidx : 0) : 0;
      for (int o = 16; o > 0; o >>= 1) len += __shfl_xor_sync(0xffffffffu, len, o);
      p += len;
    }
    if (p > pmax) p = pmax;
    uint64_t pre = 0, passed = 0, nb = 0;
    bool cut = false;
    for (uint64_t g = cur; g < wend && pre < p; g += 32) {
      const uint64_t idx = g + lane;
      const bool valid = idx < wend;
      const uint8_t* ptr = nullptr;
      uint64_t len = 0, skip = 0;
      if (valid) {
        const SliceDev sl = op.slices[idx];
        skip = idx == cur ? bidx : 0;
        ptr = sl.ptr + skip;
        len = sl.len - skip;
      }
      uint64_t incl = len;
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= (uint32_t)o) incl += t;
      }
      const uint64_t a = pre + incl - len, e = pre + incl;  // this slice's bytes are frame payload [a, e)
      const uint64_t n = valid && a < p ? (e < p ? e : p) - a : 0;
      // cursor advance (rdma_flush, rdma_bp_posix.cc:480-493): a slice is passed when the bytes reach
      // past its end (zero-length slices too, unless the call ended right before them); the first slice
      // the bytes end inside stays current
      passed += __popc(__ballot_sync(0xffffffffu, valid && a < p && e <= p));
      const unsigned cm = __ballot_sync(0xffffffffu, valid && a < p && e > p);
      if (cm) {
        nb = __shfl_sync(0xffffffffu, skip + (p - a), __ffs(cm) - 1);
        cut = true;
      }
      const bool tiny = n != 0 && n <= kTiny;
      const uint32_t items = (n && !tiny) ? (uint32_t)((n + kChunk - 1) / kChunk) : 0;
      uint32_t items_incl = items;
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, items_incl, o);
        if (lane >= (uint32_t)o) items_incl += t;
      }
      const uint32_t nitems = __shfl_sync(0xffffffffu, items_incl, 31);
      const uint64_t foff = (rt + 8 + a) & mask;
      if (tiny) {
#pragma unroll 1
        for (uint32_t i = 0; i < (uint32_t)n; i++) ring[(foff + i) & mask] = __ldg(ptr + i);
      }
      CS.first_item[lane] = items_incl - items;
      CS.src[lane] = ptr;
      CS.len[lane] = n;
      CS.off[lane] = foff;
      __syncwarp();
      // items in id order, 32 at a time; item `it` belongs to the last slice whose first item is <= it
      for (uint32_t it = lane; it < nitems; it += 32) {
        uint32_t f = 0;
        while (f + 1 < 32 && CS.first_item[f + 1] <= it) f++;
        const uint64_t c0 = (uint64_t)(it - CS.first_item[f]) * kChunk;
        uint64_t m = CS.len[f] - c0;
        if (m > kChunk) m = kChunk;
        publish_item(q, base_item + it, reinterpret_cast<uint64_t>(CS.src[f] + c0), (CS.off[f] + c0) & mask, 0,
                     (uint32_t)m);
      }
      __syncwarp();
      base_item += nitems;
      pre = __shfl_sync(0xffffffffu, e, 31);
    }
    if (lane == 0) {
      if (p) {
        *reinterpret_cast<uint64_t*>(ring + rt) = frame_header(p, stamped ? stamp_of(S.tx) : 0);  // AppendHeader
        foot_put(foot8, stamped, nfoot, (rt + 8 + round_up8(p)) & mask, p);
        S.tx++;
        S.rt = (rt + encoded_size(p)) & mask;
        S.ncalls++;
        S.cur = cur + passed;
        S.bidx = cut ? nb : 0;
      }
      S.partial = p < S.total_left;  // pair.cc:712
      S.total_left -= p;
      S.written_total += p;
    }
    __syncwarp();
    if (p) nfoot++;
    if (p == 0 || !(op.flags & kFlagUntilBlocked) || S.total_left == 0) {
      op_done = true;
      break;
    }
  }
  if (lane == 0) {
    *nfoot_out = nfoot;
    ctl->total_items = base_item;
    ctl->op_done = op_done ? 1u : 0u;
    __threadfence_block();
    *(volatile uint32_t*)&ctl->seg_done = 1;
  }
  __syncwarp();
}

// Send mover: source = a slice at any alignment (linear), destination = the peer ring (may wrap).
struct SendMove {
  uint8_t* ring;
  uint64_t cap, mask;
  __device__ __forceinline__ void issue(uint64_t a, uint32_t n, uint8_t* stage, uint64_t* bar) const {
    const uint32_t pre = (uint32_t)(a & 15);
    const uint32_t len = (pre + n + 15u) & ~15u;  // the aligned 16-byte blocks that cover the chunk
    mbar_expect_tx(bar, len);
    bulk_g2s(stage, reinterpret_cast<const void*>(a - pre), len, bar);
  }
  __device__ __forceinline__ void process(uint64_t a, uint64_t b, uint64_t c, uint32_t n, uint8_t* stage,
                                          uint32_t lane) const {
    const uint32_t pre = (uint32_t)(a & 15);
    if (c != 0 && lane == 0) *reinterpret_cast<uint64_t*>(ring + ((b + cap - 8) & mask)) = c;  // AppendHeader
    uint64_t seg1 = cap - b;
    if (seg1 > n) seg1 = n;
    // the first part only rewrites stage bytes below its end, where the second part's source starts
    smem_to_global(ring + b, stage, pre, (uint32_t)seg1, lane);
    if (n > seg1) smem_to_global(ring, stage, pre + (uint32_t)seg1, n - (uint32_t)seg1, lane);  // wrap: WR1 at remote+0
  }
};

// One Send op (PairPollable::Send, or the rdma_flush loop around it) by the whole CTA.
// `phase_bits` carries the stage barriers' parities of this thread's warp from op to op.
__device__ __forceinline__ void send_body(PairDev* __restrict__ pairs, const SendOpDev& op, OpResult* result,
                                          PipeSmem& pipe, uint8_t* stage_mem, uint32_t& phase_bits) {
  WorkItem* q = pipe.q;
  PipeCtl& ctl = pipe.ctl;
  uint64_t* bars = pipe.bars;
  __shared__ SendPlanState PS;
  __shared__ SendCallScratch CS;
  __shared__ uint64_t foot_mem[kFootCap / 2];
  uint32_t* foot8 = reinterpret_cast<uint32_t*>(foot_mem);
  __shared__ uint32_t s_nfoot;
  __shared__ unsigned long long s_tx0;
  __shared__ unsigned long long s_total;
  __shared__ uint32_t s_status;
  PairDev* P = &pairs[op.slot];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid < kQI) q[tid].ready = 0;
  if (tid == 0) {
    s_total = 0;
    s_status = *(volatile uint32_t*)&P->status;
    PS.rt = *(volatile uint64_t*)&P->remote_tail;
    PS.cap = *(volatile uint64_t*)&P->cap;
    PS.staging = PS.cap / 2;  // send_buf_size = recv_buf_size / 2, pair.cc:104
    const uint32_t sge = *(volatile uint32_t*)&P->max_sge;
    PS.max_sge = sge & ~kSgeModeBits;
    PS.coalesce = (sge & kSgeCoalesce) != 0;
    PS.stamped = (sge & kSgeStamped) != 0;
    PS.tx = PS.stamped ? VL(pair_seq(pairs, op.slot)->tx) : 0;
    PS.cur = 0;
    PS.bidx = op.byte_idx;
    PS.written_total = 0;
    PS.ncalls = 0;
    PS.partial = *(volatile uint32_t*)&P->partial_write;
    PS.last_rh = ~0ull;  // not a ring offset: the first call always fences
  }
  __syncthreads();
  {  // total_slice_size, pair.cc:661-664
    unsigned long long part = 0;
    for (uint64_t i = tid; i < op.nslices; i += kThreads) part += op.slices[i].len;
    for (int o = 16; o > 0; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
    if (lane == 0 && part) atomicAdd(&s_total, part);
  }
  __syncthreads();
  if (s_status != kStConnected) {  // pair.cc:657
    if (tid == 0) {
      result->bytes = 0;
      result->calls = 0;
    }
    return;
  }
  if (tid == 0) PS.total_left = s_total - op.byte_idx;
  const uint64_t cap = VL(P->cap), mask = cap - 1;
  uint8_t* ring = VL(P->peer_ring);
  const bool sys_scope = VL(P->wire) != 0;

  while (true) {
    if (tid == 0) {
      ctl.next = 0;
      ctl.total_items = 0;
      ctl.seg_done = 0;
      ctl.op_done = 0;
      s_nfoot = 0;
      s_tx0 = PS.tx;
    }
    __syncthreads();
    if (warp == 0) {
      if (PS.stamped) {
        if (PS.coalesce) send_produce_coalesced<true>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
        else send_produce_segment<true>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
      } else {
        if (PS.coalesce) send_produce_coalesced<false>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
        else send_produce_segment<false>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
      }
    } else {  // ---------------------------------------------- move bytes
      const SendMove mv{ring, cap, mask};
      mover_run(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
    }
    // footers last: a frame is complete for the reader only when header != 0 and footer == ~0
    // (ring_buffer.cc:75-96; stamped: the expected stamp and footer == ~header), so everything else of the
    // segment is made visible first
    if (sys_scope) __threadfence_system();
    else __threadfence();
    __syncthreads();
    const uint32_t nfoot = s_nfoot;
    if (PS.stamped) {
      for (uint32_t i = tid; i < nfoot; i += kThreads) {
        const uint64_t v = foot_mem[i];
        const uint64_t hdr = frame_header(v >> 32, stamp_of(s_tx0 + i));
        *reinterpret_cast<uint64_t*>(ring + ((v & 0xffffffffu) << 3)) = ~hdr;
      }
    } else {
      for (uint32_t i = tid; i < nfoot; i += kThreads)
        *reinterpret_cast<uint64_t*>(ring + ((uint64_t)foot8[i] << 3)) = kFooter;
    }
    const bool done = ctl.op_done != 0;
    __syncthreads();
    if (done) break;
  }
  if (tid == 0) {
    P->remote_tail = PS.rt;
    P->partial_write = PS.partial;
    if (PS.stamped) pair_seq(pairs, op.slot)->tx = PS.tx;
    result->bytes = PS.written_total;
    result->calls = PS.ncalls;
    const bool conc = (op.flags & kFlagConcurrent) != 0;
    mirror_lock(P, conc);
    publish_mirror_tx(VL(P->mirror), P);
    mirror_unlock(P, conc);
    // loopback wire: the peer lives in this table, refresh its readiness hint
    const int peer_slot = VL(P->peer_slot);
    if (peer_slot >= 0 && PS.written_total) {
      PairDev* Q = &pairs[peer_slot];
      PairMirror* qm = VL(Q->mirror);
      if (qm) {
        uint32_t hm;
        uint64_t rd;
        mirror_lock(Q, conc);
        rx_probe<false>(VL(Q->ring), VL(Q->cap), *(volatile uint64_t*)&Q->head, *(volatile uint64_t*)&Q->remain,
                        rx_stamp(pairs, peer_slot), hm, rd);
        volatile PairMirror* vm = qm;
        vm->has_message = hm;
        vm->readable = rd;
        mirror_unlock(Q, conc);
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads, 2)
k_send(PairDev* __restrict__ pairs, const SendOpDev* __restrict__ ops, OpResult* __restrict__ results) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  movers_init(pipe, threadIdx.x);
  uint32_t phase_bits = 0;
  const SendOpDev op = ops[blockIdx.x];
  send_body(pairs, op, &results[blockIdx.x], pipe, stage_mem, phase_bits);
}

// =========================================================================
// k_recv
// =========================================================================
//
// The frames of a ring form a linked list (the next header sits right after the
// previous footer), so the producer is a scout: it walks the list through a
// 256-byte register window (one 8-byte word per lane: a 9-byte HTTP/2 header
// frame and the header of the payload frame behind it cost a single trip to
// memory), applies the Read/Recv integer logic and publishes 4 KiB items.
// Consumers: load, store to the destination slice, __syncwarp, then clear
// exactly the ring bytes just read (clear-on-read is part of the wire protocol,
// ring_buffer.cc:146,160,180).  A segment ends at a credit point or at the end.

struct ScoutState {  // producer-only, lives in shared memory between segments
  uint64_t head, mh, remain, acc, cap_left, delivered, ncalls;
  uint64_t credit_val;
  uint64_t rx;  // stamped mode: frames opened so far (PairSeq::rx)
  uint32_t credit_flag;
  uint32_t stamped;
};

// Producer: RingBufferPollable::Read (ring_buffer.cc:122-191) + PairPollable::Recv's credit
// rule (pair.cc:276-284) as integer logic over the frame list.  Two steps per batch of <= 32
// frames: (1) a minimal sequential walk of the list (header -> footer check -> next header)
// that leaves frame i in lane i; (2) everything else -- destination capacity, partial reads,
// pad/footer clearing, the credit threshold, work-item expansion -- lane-parallel with warp
// scans, exactly like the Send planner.  kStamped: stamped frames (separate instantiation).
template <bool kStamped>
__device__ __noinline__ void recv_produce_segment(const RecvOpDev& op, const uint8_t* ring, uint64_t cap,
                                                  ScoutState& SS, WorkItem* q, PipeCtl* ctl, uint32_t lane) {
  const uint64_t mask = cap - 1;
  uint64_t head = SS.head, mh = SS.mh, remain = SS.remain, acc = SS.acc, cap_left = SS.cap_left;
  uint64_t delivered = SS.delivered, ncalls = SS.ncalls, rx = SS.rx;
  constexpr bool stamped = kStamped;
  uint64_t win = 0, win_base = 0;
  bool win_valid = false;
  uint32_t base_item = 0, credit = 0, last = 0;
  uint64_t credit_val = 0;
  uint64_t last_reload = 0;
  bool have_last = false;
  auto peek = [&](uint64_t off) -> uint64_t {  // 8-byte ring word at `off` through the window
    uint64_t d = (off - win_base) & mask;
    if (!win_valid || d >= 256) {
      // Frame lists are usually periodic (chttp2: 9-byte header frame + 16 KiB payload frame), so
      // the distance between the last two window reloads predicts where the next ones will be:
      // pull those lines into L2 now, 16 hops ahead, so the list walk is not one DRAM trip per hop.
      if (have_last) {
        const uint64_t stride = (off - last_reload) & mask;
        if (stride >= 256) {
          const uint64_t pf = (off + (uint64_t)((lane & 15) + 1) * stride + (lane >> 4) * 128) & mask;
          asm volatile("prefetch.global.L2 [%0];" ::"l"(ring + pf));
        }
      }
      last_reload = off;
      have_last = true;
      win_base = off;
      win = ld_volatile_u64(ring + ((off + 8ull * lane) & mask));
      win_valid = true;
      d = 0;
    }
    return __shfl_sync(0xffffffffu, win, (int)(d >> 3));
  };
  const bool one_call = !(op.flags & kFlagUntilBlocked);
  // Frame streams are usually periodic with period two (chttp2: a 9-byte DATA header frame, then
  // its payload frame), so once two consecutive frame sizes are known the next 32 frames can be
  // checked speculatively: every lane loads the header at the position the pattern predicts, the
  // positions are exact up to (and including) the first lane whose size breaks the pattern, and
  // the footers of those lanes are loaded in a second parallel round -- two trips to memory per
  // batch instead of one or two per frame.  pstate: 0 = sizes unknown (walk two frames), 1 = predict,
  // 2 = the prediction just failed early (walk a full batch, predict again only if it shows period two).
  uint32_t pstate = 0;
  uint64_t pe1 = 0, pe2 = 0;  // encoded sizes of the last processed frame and of the one before
  while (true) {
    // ---- step 1: find up to 32 complete frames; lane i keeps frame i
    uint64_t my_r = 0, my_head = 0;
    bool my_open = false;
    uint32_t cnt = 0;
    bool stopped = false, predicted = false;
    uint64_t h = head;
    if (remain > 0) {  // rest of a partially consumed frame (its header is already cleared or consumed)
      if (lane == 0) my_r = remain;
      cnt = 1;
    }
    const uint32_t c0 = cnt;  // frames before lane c0 are not new: new frame j (lane c0 + j) is frame rx + j
    if (!one_call && pstate == 1) {
      predicted = true;
      const uint32_t j = lane - c0;  // frame index after the cursor (lanes >= c0)
      const uint64_t pred_e = (j & 1) ? pe1 : pe2;
      const uint64_t rel = (uint64_t)(j >> 1) * (pe1 + pe2) + ((j & 1) ? pe2 : 0);
      const bool mine = lane >= c0 && rel + pred_e <= cap;  // a genuine chain never laps the ring
      const uint64_t off = (h + rel) & mask;
      uint64_t hdr = 0;
      if (mine) hdr = ld_volatile_u64(ring + off);
      // stamped: a header that became visible late, or one left from the last lap, carries another stamp
      const uint32_t st = stamped ? stamp_of(rx + j) : 0;
      const uint64_t len = frame_present(hdr, cap, st);
      const uint64_t e = 16 + round_up8(len);
      const bool valid = mine && len != 0 && rel + e <= cap;
      const unsigned mism = __ballot_sync(0xffffffffu, lane >= c0 && !(valid && e == pred_e));
      const uint32_t k = mism ? (uint32_t)__ffs(mism) - 1 : 32u;  // first lane off the pattern: its position is still exact
      uint64_t foot = 0;
      if (valid && lane <= k) foot = ld_volatile_u64(ring + ((off + 8 + round_up8(len)) & mask));
      const bool complete = valid && lane <= k && foot == frame_footer(hdr, st);  // GetReadableSize, ring_buffer.cc:67-97
      const unsigned inc = __ballot_sync(0xffffffffu, lane >= c0 && !complete);
      const uint32_t stop_lane = inc ? (uint32_t)__ffs(inc) - 1 : 32u;
      if (lane >= c0 && lane < stop_lane) {
        my_r = len;
        my_head = off;
        my_open = true;
      }
      // the walk ends at a position known exactly whose frame is absent or incomplete: nothing more to read
      stopped = stop_lane < 32 && stop_lane <= k && ((__ballot_sync(0xffffffffu, mine) >> stop_lane) & 1u);
      cnt = stop_lane;
      if (cnt > c0) {
        const uint64_t off_l = __shfl_sync(0xffffffffu, off, cnt - 1);
        const uint64_t e_l = __shfl_sync(0xffffffffu, e, cnt - 1);
        h = (off_l + e_l) & mask;
      }
      if (!stopped && cnt - c0 < 4) pstate = 2;
    } else {
      const uint32_t want = one_call ? 1u : (pstate == 0 ? cnt + 2u : 32u);
      while (cnt < want) {  // GetReadableSize, ring_buffer.cc:67-97
        const uint64_t hdr = peek(h);
        const uint32_t st = stamped ? stamp_of(rx + (cnt - c0)) : 0;
        const uint64_t len = frame_present(hdr, cap, st);
        if (len == 0) { stopped = true; break; }
        const uint64_t foot = peek((h + 8 + round_up8(len)) & mask);
        if (foot != frame_footer(hdr, st)) { stopped = true; break; }
        if (lane == cnt) {
          my_r = len;
          my_head = h;
          my_open = true;
        }
        h = (h + 16 + round_up8(len)) & mask;
        cnt++;
      }
    }
    // ---- step 2: Read()/Recv() per frame, all lanes at once
    const bool valid = lane < cnt;
    uint64_t r_incl = valid ? my_r : 0;
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t t = __shfl_up_sync(0xffffffffu, r_incl, o);
      if (lane >= (uint32_t)o) r_incl += t;
    }
    const uint64_t r_excl = r_incl - (valid ? my_r : 0);
    const uint64_t room = cap_left > r_excl ? cap_left - r_excl : 0;  // destination space left for this frame
    const uint64_t n = valid ? (my_r < room ? my_r : room) : 0;     // copy_size = min(readable, capacity)
    const bool full = valid && n == my_r && n != 0;
    const unsigned notfull = __ballot_sync(0xffffffffu, !full);
    const int first_nf = __ffs(notfull) - 1;
    uint32_t nproc = first_nf < 0 ? 32u : (uint32_t)first_nf;
    {  // a partially delivered frame is still processed (and is then the last one)
      const uint64_t n_at = __shfl_sync(0xffffffffu, n, nproc < 32 ? nproc : 0);
      if (nproc < 32 && n_at != 0) nproc++;
    }
    const uint64_t src = my_open ? (my_head + 8) & mask : mh;  // first payload byte to deliver
    const uint64_t end = (src + n) & mask;
    uint32_t ztail = 0;
    uint64_t mh_after = end;
    if (n == my_r) {  // frame finished: pad + footer, ring_buffer.cc:170-183
      const uint64_t up = round_up8(end);
      ztail = (uint32_t)(up - end) + 8;
      mh_after = ((up & mask) + 8) & mask;
    }
    const uint32_t zhead = my_open ? 8u : 0u;
    const bool proc = lane < nproc;
    // credit threshold (pair.cc:276-284): the first frame whose retired bytes push the
    // accumulator to cap/2 closes the segment
    uint64_t a_incl = proc ? (uint64_t)zhead + n + ztail : 0;  // internal_bytes_read of this call
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t t = __shfl_up_sync(0xffffffffu, a_incl, o);
      if (lane >= (uint32_t)o) a_incl += t;
    }
    const unsigned cross = __ballot_sync(0xffffffffu, proc && acc + a_incl >= cap / 2);
    if (cross) {
      const uint32_t ci = (uint32_t)__ffs(cross) - 1;
      nproc = ci + 1;
      credit = 1;
      credit_val = __shfl_sync(0xffffffffu, mh_after, ci);
    }
    if (nproc == 0) {  // nothing deliverable: empty ring, incomplete frame, or no room in dst
      last = 1;
      break;
    }
    const bool proc2 = lane < nproc;
    // A whole frame of <= kTiny bytes is delivered and retired by its own lane (the words were
    // just read by the walk, so they come from L2): ring_buffer.cc:146-183 for one small frame.
    const bool tiny = proc2 && my_open && n == my_r && n <= kTiny;
    if (tiny) {
      uint64_t w[kTiny / 8];
#pragma unroll
      for (int k = 0; k < (int)(kTiny / 8); k++)
        w[k] = (uint64_t)(8 * k) < n ? ld_volatile_u64(ring + ((my_head + 8 + 8 * k) & mask)) : 0;
      uint8_t* d = op.dst + delivered + r_excl;
#pragma unroll
      for (int i = 0; i < (int)kTiny; i++)
        if ((uint64_t)i < n) d[i] = (uint8_t)(w[i >> 3] >> (8 * (i & 7)));
      if (!stamped) {  // stamped frames are not cleared
        uint8_t* wr = const_cast<uint8_t*>(ring);
        const uint32_t nw = (uint32_t)(round_up8(n) >> 3) + 2;  // header + payload words + footer
        for (uint32_t k = 0; k < nw; k++) *reinterpret_cast<uint64_t*>(wr + ((my_head + 8 * k) & mask)) = 0;
      }
    }
    const uint32_t items = (proc2 && !tiny) ? (uint32_t)((n + kChunk - 1) / kChunk) : 0;
    uint32_t items_incl = items;
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t t = __shfl_up_sync(0xffffffffu, items_incl, o);
      if (lane >= (uint32_t)o) items_incl += t;
    }
    const uint32_t nitems = __shfl_sync(0xffffffffu, items_incl, 31);
    const uint32_t my_first = items_incl - items;
    // publish in id order: item `it` belongs to the frame f with first[f] <= it < first[f+1]
    for (uint32_t it0 = 0; it0 < nitems; it0 += 32) {
      const uint32_t it = it0 + lane;
      // find the owning frame by asking every lane whether it starts at or before `it`
      uint32_t f = 0;
      for (uint32_t g = 0; g < nproc; g++) {
        const uint32_t fg = __shfl_sync(0xffffffffu, my_first, g);
        const uint32_t ig = __shfl_sync(0xffffffffu, items, g);
        if (ig && fg <= it) f = g;
      }
      const uint64_t f_src = __shfl_sync(0xffffffffu, src, f);
      const uint64_t f_n = __shfl_sync(0xffffffffu, n, f);
      const uint64_t f_dst = delivered + __shfl_sync(0xffffffffu, r_excl, f);
      const uint32_t f_first = __shfl_sync(0xffffffffu, my_first, f);
      const uint32_t f_zh = __shfl_sync(0xffffffffu, zhead, f);
      const uint32_t f_zt = __shfl_sync(0xffffffffu, ztail, f);
      if (it < nitems) {
        const uint64_t c0 = (uint64_t)(it - f_first) * kChunk;
        uint64_t m = f_n - c0;
        const bool tail_item = m <= kChunk;
        if (m > kChunk) m = kChunk;
        const uint64_t z = (c0 == 0 ? f_zh : 0u) | ((uint64_t)(tail_item ? f_zt : 0u) << 16);
        publish_item(q, base_item + it, (f_src + c0) & mask, f_dst + c0, z, (uint32_t)m);
      }
    }
    __syncwarp();
    base_item += nitems;
    // ---- new cursor = state after the last processed frame
    const uint32_t L = nproc - 1;
    const bool open_L = __shfl_sync(0xffffffffu, (int)my_open, L) != 0;
    const uint64_t head_L = __shfl_sync(0xffffffffu, my_head, L);
    const uint64_t r_L = __shfl_sync(0xffffffffu, my_r, L);
    const uint64_t n_L = __shfl_sync(0xffffffffu, n, L);
    const uint64_t moved = __shfl_sync(0xffffffffu, r_excl, L) + n_L;
    if (open_L) head = (head_L + 16 + round_up8(r_L)) & mask;  // ring_buffer.cc:140-141
    mh = __shfl_sync(0xffffffffu, mh_after, L);
    remain = r_L - n_L;
    acc = credit ? 0 : acc + __shfl_sync(0xffffffffu, a_incl, L);
    rx += __popc(__ballot_sync(0xffffffffu, lane < nproc && my_open));
    delivered += moved;
    cap_left -= moved;
    ncalls += nproc;
    if (one_call || cap_left == 0 || (stopped && nproc == cnt)) last = 1;
    if (last || credit) break;
    {  // pattern for the next batch: the encoded sizes of the last two frames processed
      const bool two = L >= 1 && __shfl_sync(0xffffffffu, (int)my_open, L - (L >= 1 ? 1 : 0)) != 0 && open_L && remain == 0;
      if (two) {
        const uint64_t ra = r_L, rb = __shfl_sync(0xffffffffu, my_r, L - 1);
        const uint64_t na = 16 + round_up8(ra), nb = 16 + round_up8(rb);
        bool ok = true;
        if (pstate == 2 && !predicted) {  // distrust: the window walk must itself show period two
          ok = false;
          if (L >= 3) {
            const uint64_t rc = __shfl_sync(0xffffffffu, my_r, L - 2), rd = __shfl_sync(0xffffffffu, my_r, L - 3);
            const bool oc = __shfl_sync(0xffffffffu, (int)my_open, L - 3) != 0;
            ok = oc && round_up8(rc) == round_up8(ra) && round_up8(rd) == round_up8(rb);
          }
        }
        pe1 = na;
        pe2 = nb;
        if (pstate == 0 || (pstate == 2 && !predicted && ok)) pstate = 1;
      } else if (pstate == 1) {
        pstate = 0;
      }
    }
  }
  if (lane == 0) {
    SS.head = head;
    SS.mh = mh;
    SS.remain = remain;
    SS.acc = acc;
    SS.cap_left = cap_left;
    SS.delivered = delivered;
    SS.ncalls = ncalls;
    SS.rx = rx;
    SS.credit_flag = credit;
    SS.credit_val = credit_val;
    ctl->total_items = base_item;
    ctl->op_done = last;
    __threadfence_block();
    *(volatile uint32_t*)&ctl->seg_done = 1;
  }
  __syncwarp();
}

// Recv mover: source = ring bytes (may wrap), destination = the caller's slice (linear);
// everything the item retires is zeroed once its bytes have landed in shared memory (reference format
// only: stamped frames are left where they are).
struct RecvMove {
  uint8_t* ring;
  uint8_t* dst;
  uint64_t cap, mask;
  const uint8_t* zero;  // kZeroBytes of zeros in shared memory
  bool clear;
  __device__ __forceinline__ void issue(uint64_t a, uint32_t n, uint8_t* stage, uint64_t* bar) const {
    const uint32_t pre = (uint32_t)(a & 15);
    const uint64_t start = a - pre;
#if B200_RECV_PROXY_FENCE
    fence_proxy_async_global();  // the frame was validated with generic loads; the copy reads through the async proxy
#endif
    if (a + n <= cap) {
      const uint32_t len = (pre + n + 15u) & ~15u;
      mbar_expect_tx(bar, len);
      bulk_g2s(stage, ring + start, len, bar);
    } else {  // the chunk crosses the ring end: two copies, contiguous in the stage
      const uint32_t len1 = (uint32_t)(cap - start);  // multiple of 16 (cap is a power of two >= 16)
      const uint32_t n2 = n - (uint32_t)(cap - a);
      const uint32_t len2 = (n2 + 15u) & ~15u;
      mbar_expect_tx(bar, len1 + len2);
      bulk_g2s(stage, ring + start, len1, bar);
      bulk_g2s(stage + len1, ring, len2, bar);
    }
  }
  __device__ __forceinline__ void process(uint64_t a, uint64_t b, uint64_t c, uint32_t n, uint8_t* stage,
                                          uint32_t lane) const {
    // ---- clear-on-read: exactly what the item retired (its bytes are already in shared memory)
    if (clear) {
      const uint32_t zhead = (uint32_t)(c & 0xffff), ztail = (uint32_t)(c >> 16);
      const uint64_t zs = (a + cap - zhead) & mask;
      const uint64_t zl = (uint64_t)zhead + n + ztail;
      uint64_t z1 = cap - zs;
      if (z1 > zl) z1 = zl;
      coop_zero(ring + zs, z1, zero, lane);
      if (zl > z1) coop_zero(ring, zl - z1, zero, lane);
    }
    // ---- scatter
    smem_to_global(dst + b, stage, (uint32_t)(a & 15), n, lane);
  }
};

// One Recv op (PairPollable::Recv, or rdma_do_read's loop around it) by the whole CTA.
__device__ __forceinline__ void recv_body(PairDev* __restrict__ pairs, const RecvOpDev& op, OpResult* result,
                                          PipeSmem& pipe, uint8_t* stage_mem, uint32_t& phase_bits) {
  WorkItem* q = pipe.q;
  PipeCtl& ctl = pipe.ctl;
  uint64_t* bars = pipe.bars;
  __shared__ ScoutState SS;
  __shared__ uint32_t s_status;
  PairDev* P = &pairs[op.slot];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  if (tid < kQI) q[tid].ready = 0;
  if (tid == 0) {
    s_status = *(volatile uint32_t*)&P->status;
    SS.head = *(volatile uint64_t*)&P->head;
    SS.mh = *(volatile uint64_t*)&P->moving_head;
    SS.remain = *(volatile uint64_t*)&P->remain;
    SS.acc = *(volatile uint64_t*)&P->acc;
    SS.cap_left = op.cap;
    SS.delivered = 0;
    SS.ncalls = 0;
    SS.credit_flag = 0;
    SS.stamped = (*(volatile uint32_t*)&P->max_sge & kSgeStamped) != 0;
    SS.rx = SS.stamped ? VL(pair_seq(pairs, op.slot)->rx) : 0;
  }
  __syncthreads();
  if (s_status != kStConnected) {  // pair.cc:266-268
    if (tid == 0) {
      result->bytes = 0;
      result->calls = 0;
    }
    return;
  }
  uint8_t* ring = VL(P->ring);
  const uint64_t cap = VL(P->cap), mask = cap - 1;

  while (true) {
    if (tid == 0) {
      ctl.next = 0;
      ctl.total_items = 0;
      ctl.seg_done = 0;
      ctl.op_done = 0;
    }
    __syncthreads();
    if (warp == 0) {
      if (SS.stamped) recv_produce_segment<true>(op, ring, cap, SS, q, &ctl, lane);
      else recv_produce_segment<false>(op, ring, cap, SS, q, &ctl, lane);
    } else {
      const RecvMove mv{ring, op.dst, cap, mask, reinterpret_cast<const uint8_t*>(pipe.zero), SS.stamped == 0};
      mover_run(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
    }
    const bool credit = ld_shared_volatile(&SS.credit_flag) != 0;  // stable: the producer finished this segment
    // the sender may reuse the space only once it reads as zero (stamped: once the movers have read it)
    if (credit) __threadfence_system();
    __syncthreads();
    const bool done = ctl.op_done != 0;
    if (tid == 0 && credit) {
      // updateStatus, pair.cc:624-641: 16-byte status_report to the peer
      const int peer_slot = VL(P->peer_slot);
      const bool conc = (op.flags & kFlagConcurrent) != 0 && peer_slot >= 0;
      PairDev* Q = conc ? &pairs[peer_slot] : nullptr;
      if (conc) mirror_lock(Q, true);
      st_release_v2u64(VL(P->peer_credit), SS.credit_val, 0);
      PairMirror* pm = VL(P->peer_mirror);
      if (pm) ((volatile PairMirror*)pm)->credit_head = SS.credit_val;
      if (conc) mirror_unlock(Q, true);
      SS.credit_flag = 0;
    }
    __syncthreads();
    if (done) break;
  }
  if (tid == 0) {
    P->head = SS.head;
    P->moving_head = SS.mh;
    P->remain = SS.remain;
    P->acc = SS.acc;
    if (SS.stamped) pair_seq(pairs, op.slot)->rx = SS.rx;
    result->bytes = SS.delivered;
    result->calls = SS.ncalls;
    uint32_t hm;
    uint64_t rd;
    const bool conc = (op.flags & kFlagConcurrent) != 0;
    mirror_lock(P, conc);
    rx_probe<false>(ring, cap, SS.head, SS.remain, SS.stamped ? stamp_of(SS.rx) : 0, hm, rd);
    publish_mirror_rx(VL(P->mirror), P, hm, rd);
    mirror_unlock(P, conc);
  }
}

__global__ void __launch_bounds__(kThreads, 2)
k_recv(PairDev* __restrict__ pairs, const RecvOpDev* __restrict__ ops, OpResult* __restrict__ results) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  movers_init(pipe, threadIdx.x);
  uint32_t phase_bits = 0;
  const RecvOpDev op = ops[blockIdx.x];
  recv_body(pairs, op, &results[blockIdx.x], pipe, stage_mem, phase_bits);
}

// =========================================================================
// k_poll_scan
// =========================================================================

__global__ void __launch_bounds__(128)
k_poll_scan(PairDev* __restrict__ pairs, const int32_t* __restrict__ slots, uint32_t* __restrict__ events,
            uint32_t* __restrict__ ready_count, int32_t* __restrict__ ready_slots, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t ev = 0;
  int32_t slot = -1;
  if (i < n) {
    slot = slots[i];
    PairDev* P = &pairs[slot];
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
      if (P->peer_slot < 0) {
        publish_mirror_rx(P->mirror, P, hm, rd);
        publish_mirror_tx(P->mirror, P);
      }
    } else if (st == kStError || st == kStHalfClosed) {
      ev = kEvReadable;
    }
    events[i] = ev;
  }
  // warp-aggregated append to the ready set
  const unsigned m = __ballot_sync(0xffffffffu, ev != 0);
  if (m) {
    uint32_t base = 0;
    if (lane == (uint32_t)(__ffs(m) - 1)) base = atomicAdd(ready_count, __popc(m));
    base = __shfl_sync(0xffffffffu, base, __ffs(m) - 1);
    if (ev) ready_slots[base + __popc(m & ((1u << lane) - 1))] = slot;
  }
}

// =========================================================================
// Persistent service: k_svc_owner (one warp per host command queue), k_svc_big (pool CTAs running
// send_body / recv_body on mailbox jobs), k_svc_poll (resident readiness scan).  See b200_dev.cuh.
// =========================================================================

#ifdef B200_SVC_TRACE
__device__ unsigned long long g_svc_trace[16];
__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define TRACE_MARK(i, t0) do { if (lane == 0) atomicAdd(&g_svc_trace[i], gtime() - (t0)); } while (0)
#else
#define TRACE_MARK(i, t0) do { } while (0)
#endif

// Per owner warp: a small cache of the connections it serves -- both pairs' lines and service state in
// shared memory.  Everything that changes a cached line is either this warp itself (small ops: it updates
// the cached copy and writes through), a pool job (the entry is dropped when the job is handed over) or
// the host (Init / Connect / Disconnect and kernels launched beside the service: the host bumps a generation
// that every command carries; a new generation drops the whole cache).  A hit costs no trip to memory at
// all; a miss reads both lines with one trip (16-byte system-coherent loads, lanes in parallel).  Pairs on
// the nvlink wire are never kept: their ring and credit word are written from another GPU.
constexpr int kConnCache = 8;
struct ConnEntry {
  PairDev line[2];   // [0] = the pair with the smaller slot ... no order implied: line[i] belongs to slot[i]
  PairSvc svc[2];
  PairSeq seq[2];    // stamped mode's frame counters
  int32_t slot[2];   // slot[1] = -1: no loopback peer
};
struct ConnView {    // what an op works on
  PairDev* P;        // the op's pair (cached copy)
  PairDev* Q;        // its loopback peer or nullptr
  PairSvc* SP;
  PairSvc* SQ;
  PairSeq* NP;       // the op's pair's frame counters (cached copy)
};

__device__ __forceinline__ ConnView conn_get(ConnEntry* cc, uint32_t& cc_next, const SvcParams& sp, int pslot,
                                             int peer_hint, uint32_t lane) {
  int hit = -1, side = 0;
  {
    bool mine = false;
    int myside = 0;
    if (lane < kConnCache) {
      if (cc[lane].slot[0] == pslot) mine = true, myside = 0;
      else if (cc[lane].slot[1] == pslot) mine = true, myside = 1;
    }
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (m) {
      hit = __ffs(m) - 1;
      side = __shfl_sync(0xffffffffu, myside, hit);
    }
  }
  if (hit < 0) {
    hit = (int)(cc_next % kConnCache);
    cc_next++;
    side = 0;
    ConnEntry& e = cc[hit];
    uint4 v = make_uint4(0, 0, 0, 0);
    if (lane < 8) v = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.pairs[pslot]) + lane);
    else if (lane < 16 && peer_hint >= 0) v = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.pairs[peer_hint]) + (lane - 8));
    else if (lane == 16) v = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.psvc[pslot]));
    else if (lane == 17 && peer_hint >= 0) v = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.psvc[peer_hint]));
    else if (lane == 18) v = ld_sys_v4(reinterpret_cast<const uint4*>(pair_seq(sp.pairs, pslot)));
    else if (lane == 19 && peer_hint >= 0) v = ld_sys_v4(reinterpret_cast<const uint4*>(pair_seq(sp.pairs, peer_hint)));
    if (lane < 8) reinterpret_cast<uint4*>(&e.line[0])[lane] = v;
    else if (lane < 16) reinterpret_cast<uint4*>(&e.line[1])[lane - 8] = v;
    else if (lane == 16) *reinterpret_cast<uint4*>(&e.svc[0]) = v;
    else if (lane == 17) *reinterpret_cast<uint4*>(&e.svc[1]) = v;
    else if (lane == 18) *reinterpret_cast<uint4*>(&e.seq[0]) = v;
    else if (lane == 19) *reinterpret_cast<uint4*>(&e.seq[1]) = v;
    __syncwarp();
    int peer = e.line[0].peer_slot;
    if (peer != peer_hint) {  // (stale hint from the host: read the right peer)
      if (lane < 8 && peer >= 0) reinterpret_cast<uint4*>(&e.line[1])[lane] = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.pairs[peer]) + lane);
      if (lane == 8 && peer >= 0) *reinterpret_cast<uint4*>(&e.svc[1]) = ld_sys_v4(reinterpret_cast<const uint4*>(&sp.psvc[peer]));
      if (lane == 9 && peer >= 0) *reinterpret_cast<uint4*>(&e.seq[1]) = ld_sys_v4(reinterpret_cast<const uint4*>(pair_seq(sp.pairs, peer)));
      __syncwarp();
    }
    if (lane == 0) {
      e.slot[0] = pslot;
      e.slot[1] = peer;
    }
    __syncwarp();
  }
  ConnEntry& e = cc[hit];
  ConnView v;
  v.P = &e.line[side];
  v.SP = &e.svc[side];
  v.NP = &e.seq[side];
  const bool has_q = e.slot[side ^ 1] >= 0 && e.slot[side ^ 1] == e.line[side].peer_slot;
  v.Q = has_q ? &e.line[side ^ 1] : nullptr;
  v.SQ = has_q ? &e.svc[side ^ 1] : nullptr;
  return v;
}

// forget the connection of `pslot` (a pool job or a remote GPU is about to change its lines)
__device__ __forceinline__ void conn_drop(ConnEntry* cc, int pslot, uint32_t lane) {
  if (lane < kConnCache && (cc[lane].slot[0] == pslot || cc[lane].slot[1] == pslot)) cc[lane].slot[0] = cc[lane].slot[1] = -1;
  __syncwarp();
}
__device__ __forceinline__ void conn_drop_all(ConnEntry* cc, uint32_t lane) {
  if (lane < kConnCache) cc[lane].slot[0] = cc[lane].slot[1] = -1;
  __syncwarp();
}

// the eager record of pair `qslot`: frame of `size` bytes at the head of its ring, pushed while its delivered
// count is `at`; `cs` = XOR of eager_word() over the payload words (reduced over the warp)
__device__ __forceinline__ void eager_publish(const SvcParams& sp, int qslot, PairSvc* SQ, uint64_t at, uint64_t size,
                                              uint64_t cs, uint32_t lane) {
  for (int o = 16; o > 0; o >>= 1) cs ^= __shfl_xor_sync(0xffffffffu, cs, o);
  cs ^= eager_mix(at * 31 + size);
  if (lane == 0) {
    EagerRec* r = &sp.erec[qslot];
    uint4 a, b;
    a.x = (uint32_t)at; a.y = (uint32_t)(at >> 32); a.z = (uint32_t)cs; a.w = (uint32_t)(cs >> 32);
    b.x = (uint32_t)size; b.y = kEagerMagic; b.z = 0; b.w = 0;
    st_sys_v4(r, a);
    st_sys_v4(reinterpret_cast<uint8_t*>(r) + 16, b);
    SQ->pushed_at = at;
    VL(sp.psvc[qslot].pushed_at) = at;
  }
}

// ---- readiness of pair Q (cursor values given) after its own Recv / Retire: mirror + eager push of the
// next frame.  Called by the owner warp only: everything that touches a connection's small ops is
// program-ordered in this warp.  The frame at the head, when complete and <= kEagerMax, is copied to Q's
// host slot first, then the mirror says "has message": a Recv that finds a valid record takes the bytes
// from the slot and owes a Retire instead of waiting for a trip to the GPU and back.
__device__ __forceinline__ void svc_rx_refresh(const SvcParams& sp, const PairDev& Q, int qslot, PairSvc* SQ,
                                               uint64_t head, uint64_t mh, uint64_t remain, uint64_t acc,
                                               bool known_empty, uint32_t st, uint32_t lane) {
  const uint64_t cap = Q.cap, mask = cap - 1;
  const uint8_t* ring = Q.ring;
  const uint64_t delivered = SQ->delivered, pushed_at = SQ->pushed_at;
  uint32_t hm = 0;
  uint64_t rd = 0;
  if (remain > 0) {
    hm = 1;
    rd = remain;
  } else if (!known_empty) {
    const uint64_t hdr = ld_volatile_u64(ring + head);
    const uint64_t len = frame_present(hdr, cap, st);
    hm = hdr != 0;
    if (len) {
      // the footer and (speculatively) the payload words in the same trip
      const bool small = len <= kEagerMax && sp.erec != nullptr && pushed_at != delivered;
      const uint32_t words = small ? (uint32_t)((len + 7) >> 3) : 0;
      uint64_t w[kEagerMax / 8 / 32];
#pragma unroll
      for (int k = 0; k < (int)(kEagerMax / 8 / 32); k++) {
        const uint32_t j = k * 32 + lane;
        w[k] = j < words ? ld_volatile_u64(ring + ((head + 8 + 8ull * j) & mask)) : 0;
      }
      const uint64_t foot = ld_volatile_u64(ring + ((head + 8 + round_up8(len)) & mask));
      if (foot == frame_footer(hdr, st)) {
        rd = len;
        if (small) {
          uint8_t* slot = sp.eslots + (size_t)qslot * kEagerMax;
          uint64_t cs = 0;
#pragma unroll
          for (int k = 0; k < (int)(kEagerMax / 8 / 32); k++) {
            const uint32_t j = k * 32 + lane;
            if (j < words) {
              uint64_t x = w[k];
              const uint32_t rem = (uint32_t)len - 8 * j;
              if (rem < 8) x &= (1ull << (8 * rem)) - 1;
              st_sys_u64(slot + 8ull * j, x);
              cs ^= eager_word(x, j);
            }
          }
          eager_publish(sp, qslot, SQ, delivered, len, cs, lane);
        }
      }
    }
    if (st) hm = rd != 0;  // stamped: a message is a complete frame with the expected stamp
  }
  __syncwarp();
  if (lane == 0 && Q.mirror) {
    volatile PairMirror* vm = Q.mirror;
    vm->head = head;
    vm->moving_head = mh;
    vm->remain = remain;
    vm->acc = acc;
    vm->readable = rd;
    vm->has_message = hm;
  }
}

// ---- one PairPollable::Send call by one warp (pair.cc:645-734): <= kSvcInline slices, <= kSmallMax bytes.
// Same planning arithmetic as send_produce_segment (credit snapshot once, prefix scan of encoded sizes,
// first slice that does not fit is cut to CWS(room), zero-length slice stops the call), then the warp
// moves the frames itself.  Memory trips: pair lines (one), payload (one, over PCIe for host slices),
// then only stores; when the first frame lands at the head of the peer's ring its payload goes to the
// peer's host slot straight from the words just loaded.
__device__ __forceinline__ void svc_send_small(const SvcParams& sp, const ConnView& cv, const SvcCmd& c, int pslot,
                                               OpResult& res, uint32_t lane) {
  res.bytes = 0;
  res.calls = 0;
  PairDev& P = *cv.P;
#ifdef B200_SVC_TRACE
  const unsigned long long ts0 = gtime();
#endif
  if (P.status != kStConnected) return;  // pair.cc:657
  const uint64_t cap = P.cap, mask = cap - 1;
  uint8_t* ring = P.peer_ring;
  const bool sys_scope = P.wire != 0;
  const uint64_t rt = P.remote_tail;
  const uint64_t rh = P.credit_head;  // credit snapshot, once (pair.cc:650)
  const int peer_slot = cv.Q ? P.peer_slot : -1;  // -1: no loopback peer
  if (sys_scope) __threadfence_system();  // remote receiver: its zeroes before its credit, our frames after it
  const uint32_t nsl = (uint32_t)c.n;
  const uint32_t sge = P.max_sge & ~kSgeModeBits;
  const bool stamped = (P.max_sge & kSgeStamped) != 0;
  const uint64_t tx = cv.NP->tx;
  const uint32_t look = (uint32_t)(c.nreal < sge ? c.nreal : sge);
  const uint8_t* ptr = nullptr;
  uint64_t len = 0, raw = 0;
  if (lane < nsl) {
    raw = c.inl[lane].len;
    if (lane < look) {
      const uint64_t skip = lane == 0 ? c.byte_idx : 0;
      ptr = c.inl[lane].ptr + skip;
      len = raw - skip;
    }
  }
  const bool valid = lane < look;
  uint64_t total = raw;  // total_slice_size, pair.cc:661-664
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  total -= c.byte_idx;
  uint64_t a, wsum, esum;
  uint32_t nframes;
  const uint64_t p = send_plan<8>(valid, len, cap, rh, rt, lane, a, nframes, wsum, esum);  // kSvcInline <= 8 lanes
  const uint64_t foff = (rt + a) & mask;
  const uint32_t st = stamped ? stamp_of(tx + lane) : 0;  // frames are lanes 0..nframes-1
  const uint64_t hdr = frame_header(p, st);
  // eager: the first frame lands exactly at the head of the peer's (empty) ring
  const uint64_t p0 = __shfl_sync(0xffffffffu, p, 0);
  const bool at_head = peer_slot >= 0 && nframes > 0 && cv.Q->remain == 0 && cv.Q->head == rt;
  const bool eager = at_head && p0 <= kEagerMax && sp.erec != nullptr && cv.SQ->pushed_at != cv.SQ->delivered;
  uint8_t* eslot = eager ? sp.eslots + (size_t)peer_slot * kEagerMax : nullptr;
  const uint64_t cs = send_frames(ring, mask, ptr, p, foff, hdr, nframes, eslot, lane);
  TRACE_MARK(5, ts0);  // after the pair lines: plan + payload loads + ring stores
  // footers last (ring_buffer.cc:75-96).  A remote reader (nvlink wire) must see everything else of the call
  // first: system fence.  On the loopback wire every reader of this ring is ordered behind this warp -- its own
  // later ops, or a pool / one-shot kernel that starts after a fenced hand-over -- and a fence here would
  // also wait for the posted PCIe stores of the previous answer: none.
  if (sys_scope) __threadfence_system();
  __syncwarp();
  if (p != 0) *reinterpret_cast<uint64_t*>(ring + ((foff + 8 + round_up8(p)) & mask)) = frame_footer(hdr, st);
  if (lane == 0) {
    PairDev* Pg = &sp.pairs[pslot];
    if (stamped) {
      cv.NP->tx = tx + nframes;
      VL(pair_seq(sp.pairs, pslot)->tx) = tx + nframes;
    }
    P.remote_tail = (rt + esum) & mask;
    P.partial_write = wsum < total;
    VL(Pg->remote_tail) = (rt + esum) & mask;
    VL(Pg->partial_write) = wsum < total;  // pair.cc:712
    if (P.mirror) {
      volatile PairMirror* vm = P.mirror;
      vm->remote_tail = (rt + esum) & mask;
      vm->partial_write = wsum < total;
      vm->credit_head = rh;
      vm->peer_exit = P.credit_exit;
    }
  }
  res.bytes = wsum;
  res.calls = wsum ? 1 : 0;
  if (at_head) {
    // the peer's readiness: it was empty, now the frame at its head is ours (complete: its footer is written)
    if (eager) eager_publish(sp, peer_slot, cv.SQ, cv.SQ->delivered, p0, cs, lane);
    if (lane == 0 && cv.Q->mirror) {
      volatile PairMirror* vm = cv.Q->mirror;
      vm->readable = p0;
      vm->has_message = 1;
    }
  }
  __syncwarp();
}

// ---- one coalesced Send call by one warp (B200_SEND_COALESCE, DESIGN.md §2): <= kSvcInline slices, <= kSmallMax
// bytes, ONE frame of p = min(bytes from byte_idx, CWS(staging), CWS(free)).  The slices sit at any offset of
// the frame, so every lane assembles whole payload words itself (word j = frame bytes [8 j, 8 j + 8), gathered
// from the one or more slices it covers) and no two lanes store to the same word.  The eager push to the peer's
// host slot works as for a per-slice first frame.
__device__ __forceinline__ void svc_send_small_coalesced(const SvcParams& sp, const ConnView& cv, const SvcCmd& c,
                                                         int pslot, OpResult& res, uint32_t lane) {
  res.bytes = 0;
  res.calls = 0;
  PairDev& P = *cv.P;
  if (P.status != kStConnected) return;  // pair.cc:657
  const uint64_t cap = P.cap, mask = cap - 1;
  uint8_t* ring = P.peer_ring;
  const bool sys_scope = P.wire != 0;
  const uint64_t rt = P.remote_tail;
  const uint64_t rh = P.credit_head;  // credit snapshot, once
  const int peer_slot = cv.Q ? P.peer_slot : -1;
  if (sys_scope) __threadfence_system();
  const uint32_t nsl = (uint32_t)c.n;
  const uint32_t look = c.nreal;  // <= kSvcInline here, so within the kCoalesceSlices window
  const bool stamped = (P.max_sge & kSgeStamped) != 0;
  const uint64_t tx = cv.NP->tx;
  const uint32_t st = stamped ? stamp_of(tx) : 0;
  uint64_t raw = 0, len = 0;
  const uint8_t* ptr = nullptr;
  if (lane < nsl) {
    raw = c.inl[lane].len;
    if (lane < look) {
      const uint64_t skip = lane == 0 ? c.byte_idx : 0;
      ptr = c.inl[lane].ptr + skip;
      len = raw - skip;
    }
  }
  uint64_t total = raw;  // total_slice_size
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
  total -= c.byte_idx;
  uint64_t incl = len;
  for (int o = 1; o < 8; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += t;
  }
  const uint64_t ws = calc_writable(cap / 2), wf = calc_writable(free_size(cap, rh, rt));
  const uint64_t pmax = ws < wf ? ws : wf;
  uint64_t p = __shfl_sync(0xffffffffu, incl, 7);
  if (p > pmax) p = pmax;
  const bool at_head = peer_slot >= 0 && p > 0 && cv.Q->remain == 0 && cv.Q->head == rt;
  const bool eager = at_head && p <= kEagerMax && sp.erec != nullptr && cv.SQ->pushed_at != cv.SQ->delivered;
  uint8_t* eslot = eager ? sp.eslots + (size_t)peer_slot * kEagerMax : nullptr;
  uint64_t cs = 0;
  const uint64_t a_mine = incl - len;  // frame payload offset of this lane's slice
  const uint32_t words = (uint32_t)((p + 7) >> 3);
  for (uint32_t base = 0; base < words; base += 32) {
    const uint32_t j = base + lane;
    const uint64_t b0 = 8ull * j, b1 = b0 + 8 < p ? b0 + 8 : p;
    uint64_t w = 0;
    for (int k = 0; k < (int)kSvcInline; k++) {  // the slices' (offset, length, source) from their lanes
      const uint64_t ak = __shfl_sync(0xffffffffu, a_mine, k), lk = __shfl_sync(0xffffffffu, len, k);
      const uint8_t* sk = reinterpret_cast<const uint8_t*>(__shfl_sync(0xffffffffu, reinterpret_cast<uint64_t>(ptr), k));
      const uint64_t s = ak > b0 ? ak : b0, e = ak + lk < b1 ? ak + lk : b1;
      if (j >= words || s >= e) continue;
      const uint8_t* src = sk + (s - ak);
      if (e - s == 8) {  // the whole word from one slice: two aligned loads at most
        const uintptr_t sa = reinterpret_cast<uintptr_t>(src);
        const uint32_t sh = (uint32_t)(sa & 7) * 8;
        const uint64_t* s0 = reinterpret_cast<const uint64_t*>(sa & ~(uintptr_t)7);
        w = sh ? (ld_sys_u64(s0) >> sh) | (ld_sys_u64(s0 + 1) << (64 - sh)) : ld_sys_u64(s0);
      } else {
#pragma unroll 1
        for (uint64_t i = s; i < e; i++) w |= (uint64_t)ld_sys_u8(src + (i - s)) << (8 * (i - b0));
      }
    }
    if (j < words) {
      *reinterpret_cast<uint64_t*>(ring + ((rt + 8 + b0) & mask)) = w;  // bytes past p are zero (pad)
      if (eslot) {
        st_sys_u64(eslot + b0, w);
        cs ^= eager_word(w, j);
      }
    }
  }
  const uint64_t hdr = frame_header(p, st);
  if (lane == 0 && p) *reinterpret_cast<uint64_t*>(ring + rt) = hdr;  // AppendHeader
  if (sys_scope) __threadfence_system();  // footer last (see svc_send_small)
  __syncwarp();
  const uint64_t esum = p ? encoded_size(p) : 0;
  if (lane == 0) {
    if (p) *reinterpret_cast<uint64_t*>(ring + ((rt + 8 + round_up8(p)) & mask)) = frame_footer(hdr, st);
    PairDev* Pg = &sp.pairs[pslot];
    if (stamped && p) {
      cv.NP->tx = tx + 1;
      VL(pair_seq(sp.pairs, pslot)->tx) = tx + 1;
    }
    P.remote_tail = (rt + esum) & mask;
    P.partial_write = p < total;
    VL(Pg->remote_tail) = (rt + esum) & mask;
    VL(Pg->partial_write) = p < total;  // pair.cc:712
    if (P.mirror) {
      volatile PairMirror* vm = P.mirror;
      vm->remote_tail = (rt + esum) & mask;
      vm->partial_write = p < total;
      vm->credit_head = rh;
      vm->peer_exit = P.credit_exit;
    }
  }
  res.bytes = p;
  res.calls = p ? 1 : 0;
  if (at_head) {
    if (eager) eager_publish(sp, peer_slot, cv.SQ, cv.SQ->delivered, p, cs, lane);
    if (lane == 0 && cv.Q->mirror) {
      volatile PairMirror* vm = cv.Q->mirror;
      vm->readable = p;
      vm->has_message = 1;
    }
  }
  __syncwarp();
}

// ---- one PairPollable::Recv call by one warp (ring_buffer.cc:122-191 + pair.cc:264-286).  Returns false
// when the call would move more than kSmallMax bytes (nothing touched: the pool takes it).  With `discard`
// the payload is not stored anywhere (Retire: the host already took it from the eager slot, the frame is the
// whole frame of `capacity` bytes at the head); every state transition is that of Recv(capacity).
__device__ __forceinline__ bool svc_recv_small(const SvcParams& sp, const ConnView& cv, int slot, uint8_t* dst,
                                               uint64_t capacity, bool discard, OpResult& res, uint32_t lane) {
  res.bytes = 0;
  res.calls = 0;
  PairDev& Q = *cv.P;
  if (Q.status != kStConnected) return true;  // pair.cc:266-268
  const uint64_t cap = Q.cap;
  const bool stamped = (Q.max_sge & kSgeStamped) != 0;
  RxCursor rc{Q.head, Q.moving_head, Q.remain, Q.acc, cv.NP->rx};
  bool credit;
  const uint64_t n = warp_recv_frame(Q.ring, cap, Q.wire != 0, stamped, rc, dst, capacity, discard, kSmallMax, credit,
                                     lane);
  if (n == 0) return true;
  if (n == kRecvTooBig) return false;
  const uint64_t head = rc.head, mh_after = rc.mh, remain = rc.remain, acc = rc.acc, rx = rc.rx;
  __syncwarp();
  if (credit) {  // updateStatus, pair.cc:624-641: the 16-byte status_report
    if (Q.wire != 0) {
      // a remote sender may reuse the space only once it reads as zero (stamped: once it has been read)
      __threadfence_system();
      __syncwarp();
      if (lane == 0) st_release_v2u64(Q.peer_credit, mh_after, 0);
    } else if (lane == 0) {  // loopback: the sender is ordered behind this warp (see svc_send_small)
      asm volatile("st.global.v2.u64 [%0], {%1,%2};" ::"l"(Q.peer_credit), "l"(mh_after), "l"(0ull) : "memory");
    }
    if (lane == 0 && Q.peer_mirror) ((volatile PairMirror*)Q.peer_mirror)->credit_head = mh_after;
    if (lane == 0 && cv.Q) cv.Q->credit_head = mh_after;  // the cached line of the sender
  }
  const uint64_t delivered = cv.SP->delivered + n;
  if (lane == 0) {
    PairDev* Qg = &sp.pairs[slot];
    Q.head = head;
    Q.moving_head = mh_after;
    Q.remain = remain;
    Q.acc = acc;
    cv.SP->delivered = delivered;
    if (stamped) {
      cv.NP->rx = rx;
      VL(pair_seq(sp.pairs, slot)->rx) = rx;
    }
    VL(Qg->head) = head;
    VL(Qg->moving_head) = mh_after;
    VL(Qg->remain) = remain;
    VL(Qg->acc) = acc;
    VL(sp.psvc[slot].delivered) = delivered;
  }
  __syncwarp();  // (the zeroes are ordered before anything this warp does next; see svc_send_small)
  res.bytes = n;
  res.calls = 1;
  // the ring is known to be empty when the new head has reached the loopback sender's tail: no probe needed
  const bool known_empty = remain == 0 && cv.Q != nullptr && cv.Q->remote_tail == head;
  svc_rx_refresh(sp, Q, slot, cv.SP, head, mh_after, remain, acc, known_empty, stamped ? stamp_of(rx) : 0, lane);
  return true;
}

struct OwnerShared {  // per owner warp
  ConnEntry cc[kConnCache];
  SvcCmd cmd[2];
  int32_t box_a[kOwnBoxes], box_b[kOwnBoxes];  // pair slot of a job in flight (-1: box free) and its loopback peer
  uint32_t box_kind[kOwnBoxes];
};

// reap finished pool jobs; when `slot_a`/`slot_b` >= 0 wait for every job that touches those pairs
__device__ __forceinline__ void owner_reap(const SvcParams& sp, BigBox* boxes, OwnerShared& os, int slot_a, int slot_b,
                                           uint32_t lane) {
  if (lane < kOwnBoxes && os.box_a[lane] >= 0) {
    const int a = os.box_a[lane], b = os.box_b[lane];
    const bool must = (slot_a >= 0 && (a == slot_a || b == slot_a)) || (slot_b >= 0 && (a == slot_b || b == slot_b));
    BigBox* bx = &boxes[lane];
    uint32_t st = *(volatile uint32_t*)&bx->state;
    while (must && st != 3) {
      __nanosleep(100);
      st = *(volatile uint32_t*)&bx->state;
    }
    if (st == 3) {
      __threadfence();
      if (os.box_kind[lane] == kSvcRecv) VL(sp.psvc[a].delivered) = VL(sp.psvc[a].delivered) + VL(bx->res.bytes);
      os.box_a[lane] = -1;
      *(volatile uint32_t*)&bx->state = 0;
    }
  }
  __syncwarp();
}

__global__ void __launch_bounds__(128) k_svc_owner(SvcParams sp) {
  __shared__ OwnerShared s_os[4];
  const uint32_t lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  const int q = blockIdx.x * 4 + wi;
  if (q >= sp.nowners) return;
  OwnerShared& os = s_os[wi];
  const SvcCmd* qcmds = sp.cmds + (size_t)q * kOwnQ;
  SvcDone* qdone = sp.done + (size_t)q * kOwnQ;
  BigBox* boxes = sp.boxes + (size_t)q * kOwnBoxes;
  if (lane < kOwnBoxes) os.box_a[lane] = os.box_b[lane] = -1;
  conn_drop_all(os.cc, lane);
  uint32_t expect = 1, avail = 0, cur = 0, idle = 0, cc_next = 0, gen = 0;
  while (true) {
    // ---- fetch: entries `expect` and `expect + 1` in one trip (16 lanes x 16 bytes); both halves of a
    // line carry the stamp because the two 64-byte halves may be read by separate PCIe reads
    if (avail == 0) {
      while (true) {
        if (idle > 256) {  // nothing for a while: one small read per poll, then look properly
          uint32_t st = 0;
          if (lane == 0) st = ld_acquire_u32(&qcmds[(expect - 1) % kOwnQ].stamp);
          st = __shfl_sync(0xffffffffu, st, 0);
          if (st != expect) {
            __nanosleep(400);
            continue;
          }
        }
        uint4 v = make_uint4(0, 0, 0, 0);
        const uint32_t e = lane >> 3, ch = lane & 7;
        if (lane < 16) v = ld_sys_v4(reinterpret_cast<const uint8_t*>(&qcmds[(expect - 1 + e) % kOwnQ]) + 16 * ch);
        const bool okh = lane < 16 && ((ch == 0 && v.x == expect + e) || (ch == 7 && v.w == expect + e));
        const unsigned okm = __ballot_sync(0xffffffffu, okh);
        const bool ok0 = (okm & 0x81u) == 0x81u, ok1 = (okm & 0x8100u) == 0x8100u;
        if (ok0) {
          if (lane < 8 || (ok1 && lane < 16)) reinterpret_cast<uint4*>(&os.cmd[e])[ch] = v;
          __syncwarp();
          avail = ok1 ? 2 : 1;
          cur = 0;
          idle = 0;
          break;
        }
        idle++;
      }
    }
    const SvcCmd& c = os.cmd[cur];
    const uint32_t opc = c.op & 0xffu;
    if (opc == kSvcStop) break;
    if ((c.op >> 8) != gen) {  // the host changed pair lines (or launched kernels beside us) since the last command
      gen = c.op >> 8;
      conn_drop_all(os.cc, lane);
    }
#ifdef B200_SVC_TRACE
    const unsigned long long tr0 = gtime();
#endif
    OpResult res;
    res.bytes = 0;
    res.calls = 0;
    bool answer = true;
    if (opc != kSvcNop) {
      // the host packs the loopback peer's slot next to the pair's own (saves a dependent load)
      const int pslot = c.slot & 0xffff, peer = (c.slot >> 16) - 1;
      bool small = false;
      if (opc == kSvcSend) {
        uint64_t bytes = 0;
        if (lane < c.nreal && lane < kSvcInline) bytes = c.inl[lane].len;
        for (int o = 4; o > 0; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
        bytes = __shfl_sync(0xffffffffu, bytes, 0);
        small = !(c.flags & kFlagUntilBlocked) && c.n <= kSvcInline && bytes <= kSmallMax;
      } else {
        small = !(c.flags & kFlagUntilBlocked);
      }
      bool done_small = false;
      // a Retire the host owes for this same pair rides on its next Send (flags >> 16 = frame size).  The two
      // commute (Retire touches the pair's receive side and the peer's credit, Send neither), so a small Send
      // goes first -- its bytes are what the peer is waiting for.
      const uint32_t owed = opc == kSvcSend ? c.flags >> 16 : 0;
      if (small || owed) owner_reap(sp, boxes, os, pslot, peer, lane);  // nothing of this connection may be in flight in the pool
      // the other end of the connection is driven by a user kernel: its lines are read fresh for this op only, and
      // both mirrors are published again under their locks once the op is done
      const bool conc = (c.flags & kFlagConcurrent) != 0;
      if (small || owed) {
        if (conc) conn_drop(os.cc, pslot, lane);
        const ConnView cv = conn_get(os.cc, cc_next, sp, pslot, peer, lane);
        if (owed && !small) {
          OpResult r2;
          svc_recv_small(sp, cv, pslot, nullptr, owed, true, r2, lane);
        }
        if (small) {
          if (opc == kSvcSend) {
            if (cv.P->max_sge & kSgeCoalesce) svc_send_small_coalesced(sp, cv, c, pslot, res, lane);
            else svc_send_small(sp, cv, c, pslot, res, lane);
            done_small = true;
            TRACE_MARK(0, tr0);  // small send: fetched -> frames landed, eager record + mirror stores issued
            if (owed) {
              OpResult r2;
              svc_recv_small(sp, cv, pslot, nullptr, owed, true, r2, lane);
              TRACE_MARK(1, tr0);  // ... -> piggybacked retire finished
            }
#ifdef B200_SVC_TRACE
            if (lane == 0) atomicAdd(&g_svc_trace[2], 1ull);
#endif
          } else {
            done_small = svc_recv_small(sp, cv, pslot, reinterpret_cast<uint8_t*>(c.ptr), c.n, opc == kSvcRetire, res, lane);
          }
        }
        if (conc) {
          __syncwarp();
          if (lane == 0) {
            publish_mirror_locked(sp.pairs, pslot);
            if (cv.Q) publish_mirror_locked(sp.pairs, cv.P->peer_slot);
          }
          __syncwarp();
        }
        if (cv.P->wire != 0 || conc) conn_drop(os.cc, pslot, lane);  // nvlink wire: ring and credit change from outside
      }
      if (!done_small) {
        // ---- hand the op to the pool; the CTA that runs it answers the host itself
        conn_drop(os.cc, pslot, lane);  // the job changes the connection's lines
        owner_reap(sp, boxes, os, -1, -1, lane);
        int bi = -1;
        while (true) {
          const unsigned freem = __ballot_sync(0xffffffffu, lane < kOwnBoxes && os.box_a[lane] < 0);
          if (freem) {
            bi = __ffs(freem) - 1;
            break;
          }
          __nanosleep(200);
          owner_reap(sp, boxes, os, -1, -1, lane);
        }
        BigBox* bx = &boxes[bi];
        if (lane == 0) {
          bx->kind = opc == kSvcSend ? kSvcSend : kSvcRecv;
          bx->slot = pslot;
          bx->flags = (c.flags & 0xffffu) | kFlagConcurrent;  // the two ends' jobs run side by side in the pool
          bx->ptr = c.ptr;
          bx->n = c.n;
          bx->byte_idx = c.byte_idx;
          bx->nreal = c.nreal;
          bx->done = &qdone[(expect - 1) % kOwnQ];
          bx->seq = expect;
          os.box_a[bi] = pslot;
          os.box_b[bi] = peer;
          os.box_kind[bi] = opc == kSvcSend ? kSvcSend : kSvcRecv;
        }
        if (lane < kSvcInline) bx->inl[lane] = c.inl[lane];
        __threadfence();
        __syncwarp();
        if (lane == 0) *(volatile uint32_t*)&bx->state = 1;
        answer = false;
      }
    }
    if (answer) {
      // a Recv may have scattered into host memory from every lane: all of it before the answer
      if (opc == kSvcRecv && res.bytes) __threadfence_system();
      __syncwarp();
      if (lane == 0) {
        uint4 d;
        d.x = (uint32_t)res.bytes;
        d.y = (uint32_t)(res.bytes >> 32);
        d.z = (uint32_t)res.calls;
        d.w = expect;
        st_sys_v4(&qdone[(expect - 1) % kOwnQ], d);
      }
      TRACE_MARK(3, tr0);  // every answered op: fetched -> answer store issued
#ifdef B200_SVC_TRACE
      if (lane == 0) atomicAdd(&g_svc_trace[4], 1ull);
#endif
    }
    expect++;
    cur++;
    avail--;
    __syncwarp();
  }
  // stop: wait for the pool jobs of this queue, then acknowledge
  for (int i = 0; i < (int)kOwnBoxes; i++) {
    if (lane == 0 && os.box_a[i] >= 0)
      while (*(volatile uint32_t*)&boxes[i].state != 3) __nanosleep(200);
  }
  __syncwarp();
  if (lane == 0) {
    __threadfence_system();
    uint4 d = make_uint4(0, 0, 0, expect);
    st_sys_v4(&qdone[(expect - 1) % kOwnQ], d);
  }
}

// pool: CTAs with the k_send / k_recv machinery; a CTA claims a posted mailbox, runs the op and answers.
__global__ void __launch_bounds__(kThreads, 2) k_svc_big(SvcParams sp) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  __shared__ OpResult s_res;
  __shared__ int s_pick;
  __shared__ uint32_t s_stop;
  __shared__ __align__(16) BigBox s_box;
  const uint32_t tid = threadIdx.x;
  movers_init(pipe, tid);
  uint32_t phase_bits = 0;
  const int nboxes = sp.nowners * (int)kOwnBoxes;
  uint32_t idle = 0;
  while (true) {
    if (tid == 0) {
      s_pick = 0x7fffffff;
      s_stop = *(volatile uint32_t*)&sp.ps->stop;
    }
    __syncthreads();
    if (s_stop) break;
    for (int i = tid; i < nboxes; i += kThreads) {
      const int b = (i + blockIdx.x * 37) % nboxes;  // CTAs start their scans at different boxes
      if (*(volatile uint32_t*)&sp.boxes[b].state == 1) atomicMin(&s_pick, i);
    }
    __syncthreads();
    int pick = s_pick;
    __syncthreads();
    if (pick != 0x7fffffff) {
      const int b = (pick + blockIdx.x * 37) % nboxes;
      if (tid == 0) s_pick = atomicCAS(&sp.boxes[b].state, 1u, 2u) == 1u ? b : -1;
      __syncthreads();
      pick = s_pick;
      __syncthreads();
    } else {
      pick = -1;
    }
    if (pick < 0) {
      if (++idle > 16) __nanosleep(idle > 4096 ? 2000 : 300);
      continue;
    }
    idle = 0;
    BigBox* bx = &sp.boxes[pick];
    __threadfence();
    // the mailbox was written from another SM: read it through to shared memory (never from a stale L1 line)
    if (tid < sizeof(BigBox) / 16) reinterpret_cast<uint4*>(&s_box)[tid] = ld_sys_v4(reinterpret_cast<const uint4*>(bx) + tid);
    if (tid == 0) {
      s_res.bytes = 0;
      s_res.calls = 0;
    }
    __syncthreads();
    const uint32_t kind = s_box.kind;
    if (kind == kSvcSend) {
      SendOpDev op;
      op.slot = s_box.slot;
      op.flags = s_box.flags;
      op.nslices = s_box.n;
      op.slices = op.nslices <= kSvcInline ? s_box.inl : reinterpret_cast<const SliceDev*>(s_box.ptr);
      op.byte_idx = s_box.byte_idx;
      op.nreal = s_box.nreal;
      send_body(sp.pairs, op, &s_res, pipe, stage_mem, phase_bits);
    } else {
      RecvOpDev op;
      op.slot = s_box.slot;
      op.flags = s_box.flags;
      op.dst = reinterpret_cast<uint8_t*>(s_box.ptr);
      op.cap = s_box.n;
      recv_body(sp.pairs, op, &s_res, pipe, stage_mem, phase_bits);
    }
    // every byte this op produced must be visible before the answer: a Recv may have scattered into host
    // memory from any mover; a Send only wrote host memory (the mirrors) under the mirror lock, whose release
    // already fenced system-wide
    if (kind == kSvcRecv) __threadfence_system();
    __syncthreads();
    if (tid == 0) {
      bx->res = s_res;
      uint4 d;
      d.x = (uint32_t)s_res.bytes;
      d.y = (uint32_t)(s_res.bytes >> 32);
      d.z = (uint32_t)s_res.calls;
      d.w = s_box.seq;
      st_sys_v4(s_box.done, d);
      __threadfence();
      *(volatile uint32_t*)&bx->state = 3;
    }
    __syncthreads();
  }
}

// resident poller of the BPEV design (Poller::begin_polling, poller.cc:52-106, and the engine's scan,
// ev_epollex_rdma_bpev_linux.cc:1104-1145)
__device__ __forceinline__ void service_poll_loop(PairDev* pairs, SvcPollState* ps, uint32_t* last_ev,
                                                  ReadyEntry* ready, uint32_t* host_scans) {
  const uint32_t tid = threadIdx.x, lane = tid & 31;
  __shared__ uint32_t s_hi, s_stop;
  while (true) {
    if (tid == 0) {
      s_hi = *(volatile uint32_t*)&ps->hi_slot;
      s_stop = *(volatile uint32_t*)&ps->stop;
    }
    __syncthreads();
    const uint32_t hi = s_hi;
    if (s_stop) break;
    for (uint32_t base = 0; base < hi; base += kThreads) {
      const uint32_t slot = base + tid;
      uint32_t ev = 0, changed = 0;
      if (slot < hi) {
        PairDev* P = &pairs[slot];
        const uint32_t st = *(volatile uint32_t*)&P->status;
        uint32_t hm = 0;
        uint64_t rd = 0;
        if (st == kStConnected) {
          const uint32_t exit_flag = ld_acquire_u32(&P->credit_exit);
          rx_probe(P->ring, P->cap, *(volatile uint64_t*)&P->head, *(volatile uint64_t*)&P->remain,
                   rx_stamp(pairs, (int)slot), hm, rd);
          const uint32_t pw = *(volatile uint32_t*)&P->partial_write;
          if (exit_flag == 1) {
            ev = kEvReadable;  // HalfClosed: force a read event (engine :1130-1137)
          } else {
            if (hm) ev |= kEvReadable;
            if (pw) ev |= kEvWritable;
          }
          ev |= (uint32_t)(rd != 0) << 8;  // a frame that became complete is a change too
        } else if (st == kStError || st == kStHalfClosed) {
          ev = kEvReadable;
        }
        changed = ev != last_ev[slot];
        if (changed) {
          last_ev[slot] = ev;
          // On the loopback wire the kernels that land bytes / return credit refresh the peer's
          // mirror themselves, in order with their own completion; a second writer here could
          // only overwrite that with an older view.  Any other wire has no such writer.
          if (st == kStConnected && P->peer_slot < 0) {
            publish_mirror_rx(P->mirror, P, hm, rd);
            publish_mirror_tx(P->mirror, P);
          }
        }
      }
      // warp-aggregated append of the changes to the ready ring (mapped host memory)
      const unsigned m = __ballot_sync(0xffffffffu, changed != 0);
      if (m) {
        const int leader = __ffs(m) - 1;
        uint32_t idx = 0;
        if ((int)lane == leader) idx = atomicAdd(&ps->ready_next, (uint32_t)__popc(m));
        idx = __shfl_sync(0xffffffffu, idx, leader) + __popc(m & ((1u << lane) - 1));
        if (changed) {
          __threadfence_system();  // the mirror fields first
          ReadyEntry e;
          e.stamp = idx + 1;
          e.slot = (uint16_t)slot;
          e.events = (uint16_t)(ev & 0xff);
          *reinterpret_cast<volatile uint64_t*>(&ready[idx % kReadyRing]) = *reinterpret_cast<uint64_t*>(&e);
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      const uint32_t n = ++ps->scans;
      if ((n & 1023u) == 0) *(volatile uint32_t*)host_scans = n;  // liveness beacon
    }
    __nanosleep(200);
  }
}

__global__ void __launch_bounds__(kThreads) k_svc_poll(SvcParams sp) {
  service_poll_loop(sp.pairs, sp.ps, sp.last_ev, sp.ready, sp.host_scans);
}

// =========================================================================
// k_probe_copy: calibration kernel.  Same decomposition as k_send / k_recv (one CTA per
// connection, a producer warp publishing 4 KiB items, the same movers and stages) but no
// framing logic: what this grid shape can reach on this GPU, for a source misaligned by `mis`.
// =========================================================================
__global__ void __launch_bounds__(kThreads, 2)
k_probe_copy(uint8_t* __restrict__ dst, uint8_t* __restrict__ src, uint64_t bytes_per_cta, uint64_t stride,
             uint32_t mis, uint32_t item_bytes, uint32_t mode) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  WorkItem* q = pipe.q;
  PipeCtl& ctl = pipe.ctl;
  uint64_t* bars = pipe.bars;
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  uint8_t* d = dst + (uint64_t)blockIdx.x * stride;
  uint8_t* sbase = src + (uint64_t)blockIdx.x * stride;  // 16-byte aligned like a ring
  uint8_t* sp = sbase + mis;
  if (item_bytes > kChunk) item_bytes = kChunk;
  const uint32_t nitems = (uint32_t)(bytes_per_cta / item_bytes);
  if (tid < kQI) q[tid].ready = 0;
  movers_init(pipe, tid);
  uint32_t phase_bits = 0;
  if (tid == 0) {
    ctl.next = 0;
    ctl.total_items = 0;
    ctl.seg_done = 0;
    ctl.op_done = 0;
  }
  __syncthreads();
  const bool zero_after = (mode & 2) != 0;  // recv-like traffic: read src, write dst, clear src
  constexpr uint64_t kBig = 1ull << 62;
  if (warp == 0) {
    for (uint32_t it = lane; it < nitems; it += 32) {
      const uint64_t off = (uint64_t)it * item_bytes;
      publish_item(q, it, zero_after ? off + mis : reinterpret_cast<uint64_t>(sp + off), off, 0, item_bytes);
    }
    __syncwarp();
    if (lane == 0) {
      ctl.total_items = nitems;
      __threadfence_block();
      *(volatile uint32_t*)&ctl.seg_done = 1;
    }
  } else if (zero_after) {
    const RecvMove mv{sbase, d, kBig, kBig - 1, reinterpret_cast<const uint8_t*>(pipe.zero)};
    mover_run(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
  } else {
    const SendMove mv{d, kBig, kBig - 1};
    mover_run(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
  }
}

static void ensure_kernel_attrs() {
  static std::once_flag once;
  std::call_once(once, [] {
  cudaFuncSetAttribute(k_send, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageTotal);
  cudaFuncSetAttribute(k_recv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageTotal);
  cudaFuncSetAttribute(k_probe_copy, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageTotal);
  cudaFuncSetAttribute(k_send, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  cudaFuncSetAttribute(k_recv, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  cudaFuncSetAttribute(k_probe_copy, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  cudaFuncSetAttribute(k_svc_big, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageTotal);
  cudaFuncSetAttribute(k_svc_big, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  // Load every kernel of the library now.  With lazy module loading the first launch of a kernel loads it,
  // and a load may wait for the device to go idle: beside a resident kernel that never happens.
  cudaFuncAttributes fa;
  cudaFuncGetAttributes(&fa, k_send);
  cudaFuncGetAttributes(&fa, k_recv);
  cudaFuncGetAttributes(&fa, k_poll_scan);
  cudaFuncGetAttributes(&fa, k_probe_copy);
  cudaFuncGetAttributes(&fa, k_svc_owner);
  cudaFuncGetAttributes(&fa, k_svc_big);
  cudaFuncGetAttributes(&fa, k_svc_poll);
  });
}

int svc_trace_read(unsigned long long* out16) {
#ifdef B200_SVC_TRACE
  return cudaMemcpyFromSymbol(out16, g_svc_trace, sizeof(unsigned long long) * 16) == cudaSuccess ? 0 : -1;
#else
  (void)out16;
  return -1;
#endif
}

bool launch_service(const SvcParams& sp, void* s_owner, void* s_big, void* s_poll) {
  ensure_kernel_attrs();
  // all three grids stay resident and wait for each other's work: they must fit on the device together
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_svc_big, kThreads, kStageTotal) != cudaSuccess ||
      sp.nbig + 2 > per_sm * sms)
    return false;
  const int octas = (sp.nowners + 3) / 4;
  k_svc_owner<<<octas, 128, 0, static_cast<cudaStream_t>(s_owner)>>>(sp);
  k_svc_big<<<sp.nbig, kThreads, kStageTotal, static_cast<cudaStream_t>(s_big)>>>(sp);
  k_svc_poll<<<1, kThreads, 0, static_cast<cudaStream_t>(s_poll)>>>(sp);
  return cudaGetLastError() == cudaSuccess;
}

void launch_probe_copy(uint8_t* dst, const uint8_t* src, uint64_t bytes_per_cta, uint64_t stride, int nctas,
                       int threads, uint32_t mis, uint32_t item_bytes, uint32_t dynamic, void* stream) {
  (void)threads;
  ensure_kernel_attrs();
  k_probe_copy<<<nctas, kThreads, kStageTotal, static_cast<cudaStream_t>(stream)>>>(
      dst, const_cast<uint8_t*>(src), bytes_per_cta, stride, mis, item_bytes, dynamic);
}

// ---------------------------------------------------------------- launchers

void launch_send(PairDev* pairs, const SendOpDev* ops, OpResult* results, int nops, void* stream) {
  if (nops <= 0) return;
  ensure_kernel_attrs();
  k_send<<<nops, kThreads, kStageTotal, static_cast<cudaStream_t>(stream)>>>(pairs, ops, results);
}
void launch_recv(PairDev* pairs, const RecvOpDev* ops, OpResult* results, int nops, void* stream) {
  if (nops <= 0) return;
  ensure_kernel_attrs();
  k_recv<<<nops, kThreads, kStageTotal, static_cast<cudaStream_t>(stream)>>>(pairs, ops, results);
}
void launch_poll_scan(PairDev* pairs, const int32_t* slots, uint32_t* events, uint32_t* ready_count,
                      int32_t* ready_slots, int n, void* stream) {
  if (n <= 0) return;
  ensure_kernel_attrs();
  k_poll_scan<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(pairs, slots, events, ready_count,
                                                                               ready_slots, n);
}

}  // namespace b200
