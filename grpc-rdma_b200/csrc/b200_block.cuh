// b200_block.cuh -- the CTA pipeline shared by the library's kernels and by user kernels
// (include/b200_device_block.cuh).
//
// Everything here is run by ONE CTA of kThreads threads: warp 0 plans, warps 1 .. kMovers move bytes through
// the bulk-copy engine (TMA) and shared memory.
//   pipeline layout   kMovers, kDepth, kChunk, the stages (dynamic shared memory) and PipeSmem
//   TMA helpers       bulk_g2s / bulk_s2g, mbarriers, realign_vectors, smem_to_global, coop_zero
//   skeleton          publish_item, movers_init, mover_run
//   send_body         one Send op (PairPollable::Send, or the rdma_flush loop around it): the planners
//                     send_produce_segment / send_produce_coalesced and the SendMove mover
//   recv_body         one Recv op (PairPollable::Recv, or rdma_do_read's loop): the scout
//                     recv_produce_segment and the RecvMove mover
// k_send, k_recv and the service pool k_svc_big (b200_kernels.cu) are thin wrappers around the two bodies.
// The skeleton, the producers and the bodies take kCl: false (the default) is the one-CTA pipeline the library's
// kernels and the block calls run; true runs one op on a thread-block cluster (the cluster calls).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200_dev.cuh"
#include "b200_warp.cuh"

#ifndef VL  // (a user translation unit has dropped the shorthand of b200_warp.cuh)
#define VL(x) (*(volatile decltype(x)*)&(x))
#endif

#ifndef B200_RECV_PROXY_FENCE
#define B200_RECV_PROXY_FENCE 1
#endif

namespace b200 {

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

// Shared by every kernel that runs the pipeline: the ticket ring, the stage barriers, the zero block the Recv movers
// clear from, and the stages (dynamic shared memory).
struct PipeSmem {
  WorkItem q[kQI];
  PipeCtl ctl;
  uint64_t bars[kMovers * kDepth];
  uint4 zero[kZeroBytes / 16];
};

__device__ __forceinline__ uint32_t ld_shared_volatile(const uint32_t* p) { return *(const volatile uint32_t*)p; }

// ------------------------------------------------- thread-block clusters (the cluster calls)
//
// kCl = true runs one op on a cluster of K CTAs (K = %cluster_nctarank): the producer warp of rank 0 publishes item i
// into the ticket ring of rank i mod K (as that CTA's item i / K), every CTA's movers claim from their own ring, and
// the segment ends are cluster barriers.  Addresses of the shared::cluster window are 32-bit (mapa).
__device__ __forceinline__ uint32_t cluster_nctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
// this CTA's shared variable p, in the shared memory of CTA `rank` of the cluster
__device__ __forceinline__ uint32_t cl_map(const void* p, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_u32(p)), "r"(rank));
  return r;
}
__device__ __forceinline__ uint32_t cl_ld_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t cl_ld_u64(uint32_t a) {
  uint64_t v;
  asm volatile("ld.shared::cluster.u64 %0, [%1];" : "=l"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void cl_st_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void cl_st_u64(uint32_t a, uint64_t v) {
  asm volatile("st.shared::cluster.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}
__device__ __forceinline__ uint32_t cl_ld_acquire_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.acquire.cluster.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void cl_st_release_u32(uint32_t a, uint32_t v) {
  asm volatile("st.release.cluster.shared::cluster.u32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
// every thread of every CTA of the cluster: release this thread's writes, acquire everybody's
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
}
// the barrier that separates the phases of an op: the CTA's, or the cluster's
template <bool kCl>
__device__ __forceinline__ void pipe_sync() {
  if constexpr (kCl) cluster_sync();
  else __syncthreads();
}

// producer side: wait for the slot of item `id`, fill it, publish
template <bool kCl = false>
__device__ __forceinline__ void publish_item(WorkItem* q, uint32_t id, uint64_t a, uint64_t b, uint64_t c,
                                             uint32_t n) {
  if constexpr (!kCl) {
    WorkItem* slot = &q[id % kQI];
    while (ld_shared_volatile(&slot->ready) != 0) __nanosleep(20);
    slot->a = a;
    slot->b = b;
    slot->c = c;
    slot->n = n;
    __threadfence_block();
    *(volatile uint32_t*)&slot->ready = id + 1;
  } else {
    // item id is item l = id / K of CTA id mod K; its movers free the slot with a release store
    const uint32_t K = cluster_nctarank(), l = id / K;
    const uint32_t s = cl_map(&q[l % kQI], id - l * K);
    while (cl_ld_acquire_u32(s + offsetof(WorkItem, ready)) != 0) __nanosleep(20);
    cl_st_u64(s + offsetof(WorkItem, a), a);
    cl_st_u64(s + offsetof(WorkItem, b), b);
    cl_st_u64(s + offsetof(WorkItem, c), c);
    cl_st_u32(s + offsetof(WorkItem, n), n);
    cl_st_release_u32(s + offsetof(WorkItem, ready), l + 1);
  }
}

// producer lane, cluster form of a segment's end: every CTA learns how many of the segment's `total` items are its
// own (ids r, r + K, ...) and whether the op ends here; seg_done is released last, after the producer's other writes
// (the planner state, the Recv credit flag) that the other CTAs read once they see it
__device__ __forceinline__ void cluster_seg_end(PipeCtl* ctl, uint32_t total, uint32_t op_done) {
  const uint32_t K = cluster_nctarank();
  for (uint32_t r = 0; r < K; r++) {
    const uint32_t c = cl_map(ctl, r);
    cl_st_u32(c + offsetof(PipeCtl, total_items), (total + K - 1 - r) / K);
    cl_st_u32(c + offsetof(PipeCtl, op_done), op_done);
    cl_st_release_u32(c + offsetof(PipeCtl, seg_done), 1);
  }
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
// carries the stages' mbarrier parities from segment to segment.  kCl: the producer is in another CTA of the
// cluster, so the tickets and the segment end are read with cluster-scope acquires and a slot is freed with a
// cluster-scope release.
template <bool kCl = false, class Move>
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
        if constexpr (kCl) {
          const uint32_t rs = smem_u32(&slot->ready);
          if (cl_ld_acquire_u32(rs) == ticket + 1) {
            st = 1;
          } else if (cl_ld_acquire_u32(smem_u32(&ctl->seg_done)) && ticket >= ld_shared_volatile(&ctl->total_items)) {
            st = cl_ld_acquire_u32(rs) == ticket + 1 ? 1 : 2;
          }
        } else {
          if (ld_shared_volatile(&slot->ready) == ticket + 1) {
            st = 1;
          } else if (ld_shared_volatile(&ctl->seg_done) && ticket >= ld_shared_volatile(&ctl->total_items)) {
            st = ld_shared_volatile(&slot->ready) == ticket + 1 ? 1 : 2;  // re-check: published in between?
          }
        }
        if (st == 1) {
          if constexpr (!kCl) __threadfence_block();
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
      if constexpr (kCl) cl_st_release_u32(smem_u32(&w->ready), 0);
      else *(volatile uint32_t*)&w->ready = 0;  // the ticket-ring slot may be refilled
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
template <bool kStamped, bool kCl = false>
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
        publish_item<kCl>(q, base_item + first + t, reinterpret_cast<uint64_t>(ptr + c0), (foff + 8 + c0) & mask,
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
      publish_item<kCl>(q, base_item + it, reinterpret_cast<uint64_t>(CS.src[f] + c0), (CS.off[f] + 8 + c0) & mask,
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
    if constexpr (kCl) {
      cluster_seg_end(ctl, base_item, op_done ? 1u : 0u);
    } else {
      ctl->total_items = base_item;
      ctl->op_done = op_done ? 1u : 0u;
      __threadfence_block();
      *(volatile uint32_t*)&ctl->seg_done = 1;
    }
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
template <bool kStamped, bool kCl = false>
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
        publish_item<kCl>(q, base_item + it, reinterpret_cast<uint64_t>(CS.src[f] + c0), (CS.off[f] + c0) & mask, 0,
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
    if constexpr (kCl) {
      cluster_seg_end(ctl, base_item, op_done ? 1u : 0u);
    } else {
      ctl->total_items = base_item;
      ctl->op_done = op_done ? 1u : 0u;
      __threadfence_block();
      *(volatile uint32_t*)&ctl->seg_done = 1;
    }
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
// kCl: by every CTA of a cluster.  Rank 0 holds the planner state and plans; every CTA's movers move its share of the
// items; the segment's barriers are cluster barriers, and rank 0 writes the footers, the cursors and the answer.
template <bool kCl = false>
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
  const uint32_t rank = kCl ? cluster_ctarank() : 0u;

  if (tid < kQI) q[tid].ready = 0;
  if (tid == 0 && rank == 0) {
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
  pipe_sync<kCl>();  // cluster: every CTA's ticket ring is free before rank 0 publishes into it
  if (rank == 0) {  // total_slice_size, pair.cc:661-664
    unsigned long long part = 0;
    for (uint64_t i = tid; i < op.nslices; i += kThreads) part += op.slices[i].len;
    for (int o = 16; o > 0; o >>= 1) part += __shfl_down_sync(0xffffffffu, part, o);
    if (lane == 0 && part) atomicAdd(&s_total, part);
  }
  __syncthreads();
  const uint32_t status = kCl ? cl_ld_u32(cl_map(&s_status, 0)) : s_status;  // cluster: rank 0's reading
  if (status != kStConnected) {  // pair.cc:657
    if (tid == 0 && rank == 0) {
      result->bytes = 0;
      result->calls = 0;
    }
    return;
  }
  if (tid == 0 && rank == 0) PS.total_left = s_total - op.byte_idx;
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
    pipe_sync<kCl>();
    if (warp == 0) {
      if (rank != 0) {
        // cluster: warp 0 of the other CTAs waits at the segment's barrier
      } else if (PS.stamped) {
        if (PS.coalesce) send_produce_coalesced<true, kCl>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
        else send_produce_segment<true, kCl>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
      } else {
        if (PS.coalesce) send_produce_coalesced<false, kCl>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
        else send_produce_segment<false, kCl>(op, P, ring, PS, CS, q, &ctl, foot8, &s_nfoot, lane);
      }
    } else {  // ---------------------------------------------- move bytes
      const SendMove mv{ring, cap, mask};
      mover_run<kCl>(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
    }
    // footers last: a frame is complete for the reader only when header != 0 and footer == ~0
    // (ring_buffer.cc:75-96; stamped: the expected stamp and footer == ~header), so everything else of the
    // segment is made visible first.  Cluster: every CTA fences before the cluster barrier, and only then does rank 0
    // write the footers (DESIGN.md §13, "Cluster calls").
    if (sys_scope) __threadfence_system();
    else __threadfence();
    pipe_sync<kCl>();
    const uint32_t nfoot = rank == 0 ? s_nfoot : 0u;
    if (rank != 0) {
      // cluster: the planner state and the footer buffer are rank 0's
    } else if (PS.stamped) {
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
    pipe_sync<kCl>();
    if (done) break;
  }
  if (tid == 0 && rank == 0) {
    result->bytes = PS.written_total;
    result->calls = PS.ncalls;
    // (the footers are behind the last segment's barrier)
    send_publish(pairs, op.slot, PS.rt, PS.partial != 0, PS.stamped != 0, PS.tx, PS.written_total,
                 (op.flags & kFlagConcurrent) != 0);
  }
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
template <bool kStamped, bool kCl = false>
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
        publish_item<kCl>(q, base_item + it, (f_src + c0) & mask, f_dst + c0, z, (uint32_t)m);
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
    if constexpr (kCl) {
      cluster_seg_end(ctl, base_item, last);
    } else {
      ctl->total_items = base_item;
      ctl->op_done = last;
      __threadfence_block();
      *(volatile uint32_t*)&ctl->seg_done = 1;
    }
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
// kCl: by every CTA of a cluster.  Rank 0 holds the scout state and scouts; every CTA's movers move its share of the
// items; the segment's barriers are cluster barriers, and rank 0 writes the credit, the cursors and the answer.
template <bool kCl = false>
__device__ __forceinline__ void recv_body(PairDev* __restrict__ pairs, const RecvOpDev& op, OpResult* result,
                                          PipeSmem& pipe, uint8_t* stage_mem, uint32_t& phase_bits) {
  WorkItem* q = pipe.q;
  PipeCtl& ctl = pipe.ctl;
  uint64_t* bars = pipe.bars;
  __shared__ ScoutState SS;
  __shared__ uint32_t s_status;
  PairDev* P = &pairs[op.slot];
  const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t rank = kCl ? cluster_ctarank() : 0u;

  if (tid < kQI) q[tid].ready = 0;
  if (tid == 0 && rank == 0) {
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
  pipe_sync<kCl>();  // cluster: every CTA's ticket ring is free before rank 0 publishes into it
  const uint32_t status = kCl ? cl_ld_u32(cl_map(&s_status, 0)) : s_status;  // cluster: rank 0's reading
  if (status != kStConnected) {  // pair.cc:266-268
    if (tid == 0 && rank == 0) {
      result->bytes = 0;
      result->calls = 0;
    }
    return;
  }
  uint8_t* ring = VL(P->ring);
  const uint64_t cap = VL(P->cap), mask = cap - 1;
  const uint32_t stamped = kCl ? cl_ld_u32(cl_map(&SS.stamped, 0)) : 0u;  // cluster: read once, rank 0's

  while (true) {
    if (tid == 0) {
      ctl.next = 0;
      ctl.total_items = 0;
      ctl.seg_done = 0;
      ctl.op_done = 0;
    }
    pipe_sync<kCl>();
    if (warp == 0) {
      if (rank != 0) {
        // cluster: warp 0 of the other CTAs waits at the segment's barrier
      } else if (SS.stamped) recv_produce_segment<true, kCl>(op, ring, cap, SS, q, &ctl, lane);
      else recv_produce_segment<false, kCl>(op, ring, cap, SS, q, &ctl, lane);
    } else {
      const RecvMove mv{ring, op.dst, cap, mask, reinterpret_cast<const uint8_t*>(pipe.zero),
                        (kCl ? stamped : SS.stamped) == 0};
      mover_run<kCl>(mv, q, &ctl, stage_mem + (warp - 1) * (kDepth * kStageBytes), &bars[(warp - 1) * kDepth], phase_bits, lane);
    }
    // stable: the producer finished this segment.  Cluster: a mover has acquired its CTA's seg_done, which rank 0's
    // producer released after writing the flag; warp 0 of the other CTAs wrote nothing and does not fence.
    bool credit;
    if constexpr (kCl) credit = (rank == 0 || warp != 0) && cl_ld_u32(cl_map(&SS.credit_flag, 0)) != 0;
    else credit = ld_shared_volatile(&SS.credit_flag) != 0;
    // the sender may reuse the space only once it reads as zero (stamped: once the movers have read it)
    if (credit) __threadfence_system();
    pipe_sync<kCl>();
    const bool done = ctl.op_done != 0;
    if (tid == 0 && rank == 0 && credit) {
      __threadfence_system();  // the thread that stores the status_report fences once more itself
      credit_return(pairs, P, SS.credit_val, (op.flags & kFlagConcurrent) != 0);
      SS.credit_flag = 0;
    }
    pipe_sync<kCl>();
    if (done) break;
  }
  if (tid == 0 && rank == 0) {
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

}  // namespace b200
