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
#define B200_NOTIFY_OUT_OF_LINE 1  // notify_member is a call here (b200_warp.cuh)
#include "b200_warp.cuh"  // memory helpers, readiness + mirrors, warp movers (shared with include/b200_device.cuh)
#include "b200_block.cuh"  // the CTA pipeline: send_body / recv_body (shared with include/b200_device_block.cuh)

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

// =========================================================================
// k_send
// =========================================================================

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
// k_cluster_send / k_cluster_recv: batches launched with B200_BATCH_CLUSTER(K), K >= 2
// =========================================================================
//
// One op per thread-block cluster of K CTAs (op = cluster index): every CTA runs the cluster form of the body on it,
// rank 0 plans and writes the answer, the movers of all K CTAs move its items (DESIGN.md §13).  The body's first
// cluster barrier comes before any access to another CTA's shared memory.  Each kernel ends on a cluster barrier on
// every path -- the body returns without one for a pair that is not connected -- so that no CTA leaves while another
// may still read its shared memory.

__global__ void __launch_bounds__(kThreads, 2)
k_cluster_send(PairDev* __restrict__ pairs, const SendOpDev* __restrict__ ops, OpResult* __restrict__ results) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  movers_init(pipe, threadIdx.x);
  uint32_t phase_bits = 0;
  const uint32_t o = blockIdx.x / cluster_nctarank();
  const SendOpDev op = ops[o];
  send_body<true>(pairs, op, &results[o], pipe, stage_mem, phase_bits);
  cluster_sync();
}

// The op and the table pointer are read from shared memory, as the cluster calls hold them in b200_block: with the
// op in registers, as k_recv takes it, this kernel spills 12 bytes.
struct RecvClArgs {
  RecvOpDev op;
  PairDev* table;
};

__global__ void __launch_bounds__(kThreads, 2)
k_cluster_recv(PairDev* __restrict__ pairs, const RecvOpDev* __restrict__ ops, OpResult* __restrict__ results) {
  extern __shared__ __align__(128) uint8_t stage_mem[];
  __shared__ PipeSmem pipe;
  __shared__ RecvClArgs args;
  movers_init(pipe, threadIdx.x);
  uint32_t phase_bits = 0;
  const uint32_t o = blockIdx.x / cluster_nctarank();
  if (threadIdx.x == 0) {
    args.op = ops[o];
    args.table = pairs;
  }
  __syncthreads();
  recv_body<true>(args.table, args.op, &results[o], pipe, stage_mem, phase_bits);
  cluster_sync();
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
    ev = poll_events<true>(pairs, slot);  // (b200_warp.cuh: the readiness rule b200_warp_poll shares)
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
  PairSeq* NQ;       // its loopback peer's, or nullptr
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
  v.NQ = has_q ? &e.seq[side ^ 1] : nullptr;
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

// ---- the start and the end of the owner's small Send, per-slice and coalesced alike

// The command's slices to lanes: lane i < look holds slice i from byte_idx on (`ptr`, `len`).  Returns
// total_slice_size (pair.cc:661-664) to every lane.
__device__ __forceinline__ uint64_t svc_send_slices(const SvcCmd& c, uint32_t look, const uint8_t*& ptr, uint64_t& len,
                                                    uint32_t lane) {
  ptr = nullptr;
  len = 0;
  uint64_t raw = 0;
  if (lane < (uint32_t)c.n) {
    raw = c.inl[lane].len;
    if (lane < look) {
      const uint64_t skip = lane == 0 ? c.byte_idx : 0;
      ptr = c.inl[lane].ptr + skip;
      len = raw - skip;
    }
  }
  for (int o = 16; o > 0; o >>= 1) raw += __shfl_xor_sync(0xffffffffu, raw, o);
  return raw - c.byte_idx;
}

// The call's result, once every lane has written its footers: the cached line, the table and PairSeq written through,
// the pair's mirror, the answer; when the first frame landed at the head of the peer's empty ring (`at_head`) the
// peer's readiness -- its eager record (`eager`: the frame's `p0` payload bytes went to its host slot, `cs` this
// lane's checksum part) and its mirror -- then the peer's ready set.  `tx`: the frame counter after the call.
__device__ __forceinline__ void svc_send_done(const SvcParams& sp, const ConnView& cv, int pslot, int peer_slot,
                                              uint64_t mask, uint64_t rt, uint64_t rh, uint64_t esum, uint64_t wsum,
                                              uint64_t total, bool stamped, uint64_t tx, bool at_head, bool eager,
                                              uint64_t p0, uint64_t cs, OpResult& res, uint32_t lane) {
  PairDev& P = *cv.P;
  if (lane == 0) {
    PairDev* Pg = &sp.pairs[pslot];
    if (stamped) {
      cv.NP->tx = tx;
      VL(pair_seq(sp.pairs, pslot)->tx) = tx;
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
  __syncwarp();  // (every lane's footer before lane 0's notify)
  if (lane == 0 && wsum) notify_peer(sp.pairs, P.peer_slot);
  __syncwarp();
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
  const uint32_t sge = P.max_sge & ~kSgeModeBits;
  const bool stamped = (P.max_sge & kSgeStamped) != 0;
  const uint64_t tx = cv.NP->tx;
  const uint32_t look = (uint32_t)(c.nreal < sge ? c.nreal : sge);
  const uint8_t* ptr;
  uint64_t len;
  const uint64_t total = svc_send_slices(c, look, ptr, len, lane);
  const bool valid = lane < look;
  uint64_t a, wsum, esum;
  uint32_t nframes;
  const uint64_t p = send_plan<8>(valid, len, cap, rh, rt, lane, a, nframes, wsum, esum);  // kSvcInline <= 8 lanes
  const uint64_t foff = (rt + a) & mask;
  const uint32_t st = stamped ? stamp_of(tx + lane) : 0;  // frames are lanes 0..nframes-1
  const uint64_t hdr = frame_header(p, st);
  // eager: the first frame lands exactly at the head of the peer's (empty) ring.  Stamped, it is the peer's next
  // message only if it carries the stamp the peer expects (its rx counter's), as every reader checks
  const uint64_t p0 = __shfl_sync(0xffffffffu, p, 0);
  const bool at_head = peer_slot >= 0 && nframes > 0 && cv.Q->remain == 0 && cv.Q->head == rt &&
                       (!stamped || stamp_of(cv.NQ->rx) == stamp_of(tx));
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
  svc_send_done(sp, cv, pslot, peer_slot, mask, rt, rh, esum, wsum, total, stamped, tx + nframes, at_head, eager, p0,
                cs, res, lane);
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
  const bool stamped = (P.max_sge & kSgeStamped) != 0;
  const uint64_t tx = cv.NP->tx;
  const uint32_t st = stamped ? stamp_of(tx) : 0;
  const uint8_t* ptr;
  uint64_t len;
  // every real slice (<= kSvcInline here, so within the kCoalesceSlices window)
  const uint64_t total = svc_send_slices(c, c.nreal, ptr, len, lane);
  uint64_t incl = len;
  for (int o = 1; o < 8; o <<= 1) {
    const uint64_t t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= (uint32_t)o) incl += t;
  }
  const uint64_t ws = calc_writable(cap / 2), wf = calc_writable(free_size(cap, rh, rt));
  const uint64_t pmax = ws < wf ? ws : wf;
  uint64_t p = __shfl_sync(0xffffffffu, incl, 7);
  if (p > pmax) p = pmax;
  const bool at_head = peer_slot >= 0 && p > 0 && cv.Q->remain == 0 && cv.Q->head == rt &&
                       (!stamped || stamp_of(cv.NQ->rx) == st);
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
  if (lane == 0 && p) *reinterpret_cast<uint64_t*>(ring + ((rt + 8 + round_up8(p)) & mask)) = frame_footer(hdr, st);
  svc_send_done(sp, cv, pslot, peer_slot, mask, rt, rh, esum, p, total, stamped, tx + (p != 0), at_head, eager, p, cs,
                res, lane);
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
    if (lane == 0) notify_peer(sp.pairs, Q.peer_slot);
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

// =========================================================================
// ready sets: one-thread library kernels (b200_ready_set_add, b200_pair_disconnect)
// =========================================================================
// k_ready_add: the note first, the set pointer last (a producer that finds the pointer finds the key), then one
// initial entry with armed = 0, so that a frame or a close that came before the add is not lost.
__global__ void k_ready_add(PairDev* pairs, int slot, ReadyQueue* q, uint32_t key) {
  ReadyNote* n = ready_note(pairs, slot);
  VL(n->key) = key;
  VL(n->armed) = 0u;
  __threadfence();
  VL(n->set) = q;
  __threadfence();
  ready_push(q, key);
}
__global__ void k_ready_notify(PairDev* pairs, int slot) { notify_peer(pairs, slot); }
// k_ready_park: b200_ready_set_park, the consumer's park run by one thread
__global__ void k_ready_park(ReadyQueue* q, volatile int* out) { *out = (int)ready_park_one(q); }

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
  for (const void* f : {(const void*)k_cluster_send, (const void*)k_cluster_recv}) {
    cudaFuncSetAttribute(f, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kStageTotal);
    cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
    cudaFuncSetAttribute(f, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);  // clusters of 9..16 CTAs
  }
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
  cudaFuncGetAttributes(&fa, k_cluster_send);
  cudaFuncGetAttributes(&fa, k_cluster_recv);
  cudaFuncGetAttributes(&fa, k_ready_add);
  cudaFuncGetAttributes(&fa, k_ready_notify);
  cudaFuncGetAttributes(&fa, k_ready_park);
  });
}

void load_kernels() { ensure_kernel_attrs(); }

void launch_ready_add(PairDev* pairs, int slot, ReadyQueue* q, uint32_t key, void* stream) {
  ensure_kernel_attrs();
  k_ready_add<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(pairs, slot, q, key);
}
void launch_ready_notify(PairDev* pairs, int slot, void* stream) {
  ensure_kernel_attrs();
  k_ready_notify<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(pairs, slot);
}
void launch_ready_park(ReadyQueue* q, int* out, void* stream) {
  ensure_kernel_attrs();
  k_ready_park<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(q, out);
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

// nops clusters of `cluster` CTAs
static cudaLaunchConfig_t cluster_config(int nops, int cluster, void* stream, cudaLaunchAttribute* attr) {
  cudaLaunchConfig_t c = {};
  c.gridDim = dim3((unsigned)nops * (unsigned)cluster);
  c.blockDim = dim3(kThreads);
  c.dynamicSmemBytes = kStageTotal;
  c.stream = static_cast<cudaStream_t>(stream);
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  c.attrs = attr;
  c.numAttrs = 1;
  return c;
}

void launch_send(PairDev* pairs, const SendOpDev* ops, OpResult* results, int nops, void* stream, int cluster) {
  if (nops <= 0) return;
  ensure_kernel_attrs();
  if (cluster <= 1) {
    k_send<<<nops, kThreads, kStageTotal, static_cast<cudaStream_t>(stream)>>>(pairs, ops, results);
    return;
  }
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t c = cluster_config(nops, cluster, stream, attr);
  cudaLaunchKernelEx(&c, k_cluster_send, pairs, ops, results);
}
void launch_recv(PairDev* pairs, const RecvOpDev* ops, OpResult* results, int nops, void* stream, int cluster) {
  if (nops <= 0) return;
  ensure_kernel_attrs();
  if (cluster <= 1) {
    k_recv<<<nops, kThreads, kStageTotal, static_cast<cudaStream_t>(stream)>>>(pairs, ops, results);
    return;
  }
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t c = cluster_config(nops, cluster, stream, attr);
  cudaLaunchKernelEx(&c, k_cluster_recv, pairs, ops, results);
}
int cluster_capacity(int kind, int cluster) {
  ensure_kernel_attrs();
  cudaLaunchAttribute attr[1];
  const cudaLaunchConfig_t c = cluster_config(1, cluster, nullptr, attr);
  int n = 0;
  const cudaError_t e = kind == 0 ? cudaOccupancyMaxActiveClusters(&n, k_cluster_send, &c)
                                  : cudaOccupancyMaxActiveClusters(&n, k_cluster_recv, &c);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  return n;
}
void launch_poll_scan(PairDev* pairs, const int32_t* slots, uint32_t* events, uint32_t* ready_count,
                      int32_t* ready_slots, int n, void* stream) {
  if (n <= 0) return;
  ensure_kernel_attrs();
  k_poll_scan<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(pairs, slots, events, ready_count,
                                                                               ready_slots, n);
}

}  // namespace b200
