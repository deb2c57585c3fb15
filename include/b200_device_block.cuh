/*
 * b200_device_block.cuh -- block-level device Send / Recv on a pair, for user kernels (sm_90a), and their cluster form
 * (b200_cluster_send / b200_cluster_recv, below).
 *
 * The warp calls of b200_device.cuh move a connection's bytes with one warp and plain loads and stores.  The calls
 * here put a whole CTA on the op and run the library's own k_send / k_recv pipeline on it: warp 0 plans the frames,
 * warps 1..8 move them through shared memory with the bulk-copy engine (TMA).  Build with
 *     nvcc -gencode arch=compute_90a,code=sm_90a -I<repo>/include ...
 *
 * Every call is BLOCK-COLLECTIVE: all B200_BLOCK_THREADS threads of the CTA call it with the same arguments and
 * every thread gets the same result.  The semantics are those of the C ABI, op for op:
 *   flags = B200_BATCH_ONE_CALL        one PairPollable::Send / Recv call: b200_pair_send / b200_pair_recv (and
 *                                      b200_warp_send / b200_warp_recv) from the same state, bit for bit
 *   flags = B200_BATCH_UNTIL_BLOCKED   the rdma_flush / rdma_do_read loop of a prepared batch op: the same bytes
 *                                      and the same number of calls that moved bytes (*calls)
 * in every framing mode the connection runs (per-slice with the max_sge cut, coalesced, stamped).
 *
 * Rules:
 *   - the calling block is exactly B200_BLOCK_THREADS x 1 x 1 threads and runs under
 *     __launch_bounds__(B200_BLOCK_THREADS, 2), which keeps two CTAs per SM;
 *   - the first B200_BLOCK_SMEM_BYTES of the kernel's dynamic shared memory are the movers' stages (the kernel may
 *     use what lies beyond them); its launcher passes at least that much and sets
 *     cudaFuncAttributeMaxDynamicSharedMemorySize accordingly, as the library does for k_send;
 *   - b200_block_init runs once per CTA before its first call;
 *   - slices and dst are device memory or pinned, mapped host memory (the RDMA registered-memory rule);
 *   - at most one sending CTA or warp and one receiving CTA or warp per pair at a time: the ops-in-flight rule of
 *     b200_pair.h, which also covers mixing these calls with the warp calls on one pair;
 *   - the handle is the one b200_pair_device_claim filled; the kernels that use it finish before the release.
 * The calls never wait: no credit, or no complete frame at the head, returns 0.  A kernel whose CTAs wait for each
 * other (a sender CTA and a receiver CTA of one connection) must make sure they are co-resident, and bounds its own
 * retry loops.  When b200_block_recv returns, the delivered bytes are visible to every thread of the calling CTA; a
 * consumer in another CTA or kernel needs the usual GPU-scope fence.  Every call publishes the pair's host-visible
 * mirror (and, on the loopback wire, the peer's readiness or credit) under the per-pair mirror lock.  A mirror that an
 * unmirrored claim (B200_CLAIM_UNMIRRORED) took away is skipped; with neither this end's nor its loopback peer's mirror
 * left, the call takes no lock at all.  The results are the same, bit for bit.
 *
 * Refusals return 0 (and *calls = 0) to every thread and change nothing: a block shape other than
 * B200_BLOCK_THREADS x 1 x 1, any flag bit other than B200_BATCH_UNTIL_BLOCKED, a pair that is not connected, a Send
 * to a peer that has gone, n == 0 or cap == 0.
 *
 * The code behind these calls (include'd below) is the one k_send, k_recv and the service pool run.
 */
#ifndef B200_DEVICE_BLOCK_CUH
#define B200_DEVICE_BLOCK_CUH

#include "b200_device.cuh"
// the library's CTA pipeline, compiled into the caller's kernel (header-only by design)
#include "../grpc-rdma_b200/csrc/b200_block.cuh"
#undef VL  // (the library's shorthand for a volatile access: not for user translation units)

#define B200_BLOCK_THREADS 288     /* 1 producer warp + 8 mover warps */
#define B200_BLOCK_SMEM_BYTES 99072 /* the movers' stages: dynamic shared memory the caller provides */

static_assert(B200_BLOCK_THREADS == b200::kThreads, "B200_BLOCK_THREADS is the pipeline's CTA size");
static_assert(B200_BLOCK_SMEM_BYTES == b200::kStageTotal, "B200_BLOCK_SMEM_BYTES is the pipeline's stage memory");

/* Per-CTA state of the calls: declare it __shared__ (one per CTA). */
typedef struct b200_block {
  b200::PipeSmem pipe;                  // ticket ring, stage barriers, the zero block
  b200::SendOpDev sop;                  // the op being run, as k_send / k_recv take it
  b200::RecvOpDev rop;
  b200::OpResult res;                   // the op's answer, broadcast to every thread
  uint32_t go;                          // the entry checks' answer
  uint32_t phase[1 + b200::kMovers];    // per warp: the parities of its stage barriers, carried from op to op
  b200::PairDev* table;                 // cluster calls: the connection table of the op (rank 0's handle)
} b200_block;

// The movers' stages: the first B200_BLOCK_SMEM_BYTES of the kernel's dynamic shared memory.  They are addressed from
// its start, as k_send does, so that their addresses are constants: a base kept in a register costs k_send's body six
// registers.
extern __shared__ __align__(128) uint8_t b200_block_stages[];

// The op's publication flag: kFlagConcurrent makes the bodies publish the mirrors under the per-pair locks.  When
// neither this end nor its loopback peer has a mirror -- both ends of a loopback connection claimed with
// B200_CLAIM_UNMIRRORED, or a CUDA-IPC end claimed so (such an end has no peer row here) -- the bodies have nothing to
// publish, and the flag, whose only effect is the locks, is left out.  Every mirrored end keeps it, on either wire.
__device__ __forceinline__ uint32_t b200_publish_flag(const b200::PairDev* P) {
  return *(volatile b200::PairMirror* const*)&P->mirror || *(volatile b200::PairMirror* const*)&P->peer_mirror
             ? b200::kFlagConcurrent
             : 0u;
}

__device__ __forceinline__ bool b200_block_shape_ok() {
  return blockDim.x == B200_BLOCK_THREADS && blockDim.y == 1 && blockDim.z == 1;
}

/* Block-collective, once per CTA before its first call. */
__device__ inline void b200_block_init(b200_block* st) {
  if (!b200_block_shape_ok()) return;
  b200::movers_init(st->pipe, threadIdx.x);
  if (threadIdx.x <= (uint32_t)b200::kMovers) st->phase[threadIdx.x] = 0;
  __syncthreads();
}

// Thread 0 has written the op and the entry checks' answer; the barrier shows them to every thread.  A refused op
// returns only after a second barrier, so that no thread can overwrite `go` with the next call's answer before every
// thread has read this one.  (The answer travels through shared memory rather than __syncthreads_or: an early return
// straight out of the barrier's value costs the Recv body spills.)
__device__ __forceinline__ bool b200_block_enter(b200_block* st) {
  __syncthreads();
  if (st->go) return true;
  __syncthreads();
  return false;
}

// The end of every op that ran: this warp's stage parities for the next op, then one barrier for the whole CTA (the
// bodies return early, skipping their last barrier, when the pair is not connected), then the answer to every thread.
__device__ __forceinline__ uint64_t b200_block_leave(b200_block* st, uint32_t phase, uint64_t* calls) {
  if ((threadIdx.x & 31) == 0) st->phase[threadIdx.x >> 5] = phase;
  __syncthreads();
  if (calls) *calls = st->res.calls;
  return st->res.bytes;
}

/* Payload bytes accepted; *calls (may be NULL) = Send calls that accepted bytes.  0: nothing (refused, not
 * connected, peer gone, no credit, n == 0). */
__device__ inline uint64_t b200_block_send(b200_block* st, const b200_dev_pair* h, const b200_slice* slices,
                                           uint64_t n, uint64_t byte_idx, int flags, uint64_t* calls) {
  if (calls) *calls = 0;
  if (!b200_block_shape_ok() || (flags & ~B200_BATCH_UNTIL_BLOCKED) != 0) return 0;
  b200::PairDev* table = reinterpret_cast<b200::PairDev*>(h->table);
  if (threadIdx.x == 0) {
    const b200::PairDev* P = table + h->slot;
    // pair.cc:657; and a peer that left: its ring may belong to somebody else
    st->go = *(volatile const uint32_t*)&P->status == b200::kStConnected && n != 0 &&
             b200::ld_acquire_u32(&P->credit_exit) != 1;
    b200::SendOpDev& op = st->sop;
    op.slot = h->slot;
    op.flags = (uint32_t)flags | b200_publish_flag(P);  // a device-owned end publishes under the per-pair lock
    op.slices = reinterpret_cast<const b200::SliceDev*>(slices);
    op.nslices = n;
    op.byte_idx = byte_idx;
    op.nreal = n;  // every slice is real memory: nothing is folded into a pseudo-slice
  }
  if (!b200_block_enter(st)) return 0;
  uint32_t phase = st->phase[threadIdx.x >> 5];
  b200::send_body(table, st->sop, &st->res, st->pipe, b200_block_stages, phase);
  return b200_block_leave(st, phase, calls);
}

/* Bytes delivered into dst; *calls (may be NULL) = Recv calls that delivered bytes.  0: nothing (refused, not
 * connected, cap == 0, no complete frame at the head). */
__device__ inline uint64_t b200_block_recv(b200_block* st, const b200_dev_pair* h, void* dst, uint64_t cap, int flags,
                                           uint64_t* calls) {
  if (calls) *calls = 0;
  if (!b200_block_shape_ok() || (flags & ~B200_BATCH_UNTIL_BLOCKED) != 0) return 0;
  b200::PairDev* table = reinterpret_cast<b200::PairDev*>(h->table);
  if (threadIdx.x == 0) {
    st->go = *(volatile const uint32_t*)&table[h->slot].status == b200::kStConnected && cap != 0;  // pair.cc:266-268
    b200::RecvOpDev& op = st->rop;
    op.slot = h->slot;
    op.flags = (uint32_t)flags | b200_publish_flag(table + h->slot);
    op.dst = static_cast<uint8_t*>(dst);
    op.cap = cap;
  }
  if (!b200_block_enter(st)) return 0;
  uint32_t phase = st->phase[threadIdx.x >> 5];
  b200::recv_body(table, st->rop, &st->res, st->pipe, b200_block_stages, phase);
  return b200_block_leave(st, phase, calls);
}

/* ---- cluster calls: a thread-block cluster of K CTAs drives one op ------------------------------------------------
 *
 * One CTA keeps at most 8 movers x 3 stages x 4 KiB of reads in flight, far below what HBM needs to run near its rate;
 * with few connections most of the GPU would sit idle.  b200_cluster_send / b200_cluster_recv run one op on a cluster:
 * the planner warp of CTA rank 0 plans it as the block calls do, and the mover warps of all K CTAs move its 4 KiB items,
 * item i in CTA i mod K, each CTA with its own stages and bulk-copy engine (DESIGN.md §13, "Cluster calls").
 *
 * Every call is CLUSTER-COLLECTIVE: every thread of every CTA of the cluster calls it.  The op is taken from the
 * arguments of CTA rank 0 (the other CTAs' arguments are ignored) and every thread gets the same result, with the
 * semantics of b200_block_send / b200_block_recv: return values, *calls, partial_write, cursors, credit, frames and
 * ring image bit for bit, in every framing mode.
 *
 * Rules, beyond those of the block calls (the CTA shape, __launch_bounds__(B200_BLOCK_THREADS, 2), the stages, one
 * b200_block per CTA with b200_block_init, the memory of slices and dst, the claim):
 *   - the cluster is K x 1 x 1 CTAs, 1 <= K <= 16 (K is read from %cluster_nctarank; K > 8 needs
 *     cudaFuncAttributeNonPortableClusterSizeAllowed on the kernel).  K = 1, a launch without clusters, runs the
 *     block calls' pipeline on the one CTA, with the same results;
 *   - at most one sending cluster, CTA or warp and one receiving cluster, CTA or warp per pair at a time;
 *   - the calls never wait; clusters that wait for each other must be co-resident (cudaOccupancyMaxActiveClusters);
 *   - when b200_cluster_recv returns, the delivered bytes are visible to every thread of the cluster.  Rank 0
 *     publishes the mirrors under the per-pair lock, once per op.
 * Refusals return 0 (and *calls = 0) to every thread and change nothing: those of the block calls, and a cluster that
 * is not K x 1 x 1 with K <= 16.
 */
__device__ __forceinline__ bool b200_cluster_shape_ok() {
  uint32_t y, z;
  asm volatile("mov.u32 %0, %%cluster_nctaid.y;" : "=r"(y));
  asm volatile("mov.u32 %0, %%cluster_nctaid.z;" : "=r"(z));
  return y == 1 && z == 1 && b200::cluster_nctarank() <= 16;
}

// Thread 0 of rank 0 has written the op, its table and the entry checks' answer into its b200_block; after the cluster
// barrier every other CTA copies them into its own.  A refused op returns only after a second cluster barrier, so that
// rank 0 cannot overwrite them with the next call's before every CTA has read them.
template <class Op>
__device__ __forceinline__ bool b200_cluster_enter(b200_block* st, Op* op) {
  static_assert(sizeof(Op) % 8 == 0, "the op is copied in 8-byte words");
  constexpr uint32_t kWords = sizeof(Op) / 8;
  b200::cluster_sync();
  if (b200::cluster_ctarank() != 0) {
    const uint32_t t = threadIdx.x;
    uint64_t* w = reinterpret_cast<uint64_t*>(op);
    if (t < kWords) w[t] = b200::cl_ld_u64(b200::cl_map(w + t, 0));
    else if (t == kWords) st->table = reinterpret_cast<b200::PairDev*>(b200::cl_ld_u64(b200::cl_map(&st->table, 0)));
    else if (t == kWords + 1) st->go = b200::cl_ld_u32(b200::cl_map(&st->go, 0));
  }
  __syncthreads();
  if (st->go) return true;
  b200::cluster_sync();
  return false;
}

// The end of every op that ran: this warp's stage parities, then rank 0's answer to every thread of the cluster.  The
// second barrier keeps every CTA in the call (and rank 0's shared memory alive) until every CTA has read the answer.
__device__ __forceinline__ uint64_t b200_cluster_leave(b200_block* st, uint32_t phase, uint64_t* calls) {
  if ((threadIdx.x & 31) == 0) st->phase[threadIdx.x >> 5] = phase;
  b200::cluster_sync();
  const uint32_t a = b200::cl_map(&st->res, 0);
  const uint64_t bytes = b200::cl_ld_u64(a + offsetof(b200::OpResult, bytes));
  const uint64_t c = b200::cl_ld_u64(a + offsetof(b200::OpResult, calls));
  b200::cluster_sync();
  if (calls) *calls = c;
  return bytes;
}

/* Cluster-collective b200_block_send: payload bytes accepted; *calls (may be NULL) = Send calls that accepted bytes. */
__device__ inline uint64_t b200_cluster_send(b200_block* st, const b200_dev_pair* h, const b200_slice* slices,
                                             uint64_t n, uint64_t byte_idx, int flags, uint64_t* calls) {
  if (calls) *calls = 0;
  if (!b200_block_shape_ok() || !b200_cluster_shape_ok()) return 0;
  if (threadIdx.x == 0 && b200::cluster_ctarank() == 0) {
    b200::PairDev* table = reinterpret_cast<b200::PairDev*>(h->table);
    const b200::PairDev* P = table + h->slot;
    st->go = (flags & ~B200_BATCH_UNTIL_BLOCKED) == 0 && *(volatile const uint32_t*)&P->status == b200::kStConnected &&
             n != 0 && b200::ld_acquire_u32(&P->credit_exit) != 1;
    st->table = table;
    b200::SendOpDev& op = st->sop;
    op.slot = h->slot;
    op.flags = (uint32_t)flags | b200_publish_flag(P);
    op.slices = reinterpret_cast<const b200::SliceDev*>(slices);
    op.nslices = n;
    op.byte_idx = byte_idx;
    op.nreal = n;
  }
  if (!b200_cluster_enter(st, &st->sop)) return 0;
  uint32_t phase = st->phase[threadIdx.x >> 5];
  b200::send_body<true>(st->table, st->sop, &st->res, st->pipe, b200_block_stages, phase);
  return b200_cluster_leave(st, phase, calls);
}

/* Cluster-collective b200_block_recv: bytes delivered into dst; *calls (may be NULL) = Recv calls that delivered
 * bytes. */
__device__ inline uint64_t b200_cluster_recv(b200_block* st, const b200_dev_pair* h, void* dst, uint64_t cap, int flags,
                                             uint64_t* calls) {
  if (calls) *calls = 0;
  if (!b200_block_shape_ok() || !b200_cluster_shape_ok()) return 0;
  if (threadIdx.x == 0 && b200::cluster_ctarank() == 0) {
    b200::PairDev* table = reinterpret_cast<b200::PairDev*>(h->table);
    st->go = (flags & ~B200_BATCH_UNTIL_BLOCKED) == 0 &&
             *(volatile const uint32_t*)&table[h->slot].status == b200::kStConnected && cap != 0;
    st->table = table;
    b200::RecvOpDev& op = st->rop;
    op.slot = h->slot;
    op.flags = (uint32_t)flags | b200_publish_flag(table + h->slot);
    op.dst = static_cast<uint8_t*>(dst);
    op.cap = cap;
  }
  if (!b200_cluster_enter(st, &st->rop)) return 0;
  uint32_t phase = st->phase[threadIdx.x >> 5];
  b200::recv_body<true>(st->table, st->rop, &st->res, st->pipe, b200_block_stages, phase);
  return b200_cluster_leave(st, phase, calls);
}

#endif /* B200_DEVICE_BLOCK_CUH */
