/*
 * b200_pair.h -- C ABI of the GPU-native (H100, sm_90a) RDMA_BPEV endpoint hot path.
 *
 * This is the drop-in boundary: plain pointers and sizes, no C++/torch types.
 * It replaces, for the reference (pwrliang/grpc-rdma, paths relative to its
 * root), exactly the surface that the endpoint (src/core/lib/iomgr/
 * rdma_bp_posix.cc), the BPEV event engine (src/core/lib/iomgr/
 * ev_epollex_rdma_bpev_linux.cc) and the background Poller (src/core/lib/
 * ibverbs/poller.cc) call on a connection:
 *
 *   grpc_core::ibverbs::PairPollable   src/core/lib/ibverbs/pair.h:82-271
 *   grpc_core::ibverbs::PairPool       src/core/lib/ibverbs/pair.h:273-333
 *   grpc_core::ibverbs::Poller         src/core/lib/ibverbs/poller.h:16-68
 *   grpc_core::ibverbs::Config         src/core/lib/ibverbs/config.h:15-55
 *
 * Implementation: libb200rdma.so (grpc-rdma_b200/csrc).  Ring buffers, credit
 * words and cursors live in HBM; gather/encode (Send), deframe/scatter/clear
 * (Recv), the credit write-back and the readiness scan are sm_90a kernels.
 * There is NO CPU fallback: every data-path entry point fails (returns 0 and
 * sets b200_last_error) if no CUDA device is usable.
 *
 * Conventions kept from the reference: byte counts are returned, never
 * negative; 0 means "nothing moved", the caller then looks at
 * b200_pair_status(); at most one send and one recv may be in flight per pair
 * (ContentAssertion, pair.h:64-81); the has_ and status queries are wait-free
 * and may be called from any thread.
 *
 * Memory rule (the RDMA "registered memory" rule, buffer.cc:9): the batch
 * entry points require slices/destinations that the GPU can address -- device
 * memory, or host memory from b200_mem_alloc_host / b200_mem_register_host.
 * The single-pair entry points accept ANY host pointer; unregistered memory is
 * bounced through a pinned staging buffer (the analogue of send_buffers_
 * [kDataBuffer], pair.cc:104,690).
 */
#ifndef B200_PAIR_H
#define B200_PAIR_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_pair b200_pair; /* opaque, pool-owned (PairPollable) */

/* Flattened grpc_slice: GRPC_SLICE_START_PTR / GRPC_SLICE_LENGTH
 * (include/grpc/impl/codegen/slice.h:96-101). */
typedef struct b200_slice {
  const void* ptr;
  uint64_t len;
} b200_slice;

/* PairStatus, pair.h:44-51 (same order, same values). */
enum b200_status {
  B200_UNINITIALIZED = 0,
  B200_INITIALIZED = 1,
  B200_CONNECTED = 2,
  B200_HALF_CLOSED = 3,
  B200_DISCONNECTED = 4,
  B200_ERROR = 5
};

/* Size of the bootstrap blob exchanged over the TCP fd
 * (Address::bytes(), address.h:24-31 / address.cc:19-23; exchange_data,
 * rdma_bp_posix.cc:640-692). */
#define B200_ADDRESS_BYTES 48
/* IBVERBS_PAIR_TAG_POLLABLE, pair.h:26 */
#define B200_PAIR_TAG_POLLABLE 0xa0u
/* GRPC_IBVERBS_POLLER_CAPACITY, poller.h:12 */
#define B200_POLLER_CAPACITY 4096

/* ------------------------------------------------------------------ runtime */

/* Bind the runtime to CUDA device `device` (-1: current device / env
 * B200_DEVICE).  Idempotent.  Returns 0 on success, -1 on failure (no CUDA
 * device, wrong architecture ...); there is no CPU fallback. */
int b200_init(int device);
void b200_shutdown(void);
int b200_device(void);
/* Thread-local description of the last failure ("" if none). */
const char* b200_last_error(void);

/* Config (config.cc:45-115): same keys as the reference's environment
 * variables -- GRPC_RDMA_RING_BUFFER_SIZE_KB (4096), GRPC_RDMA_POLLER_THREAD_NUM
 * (1), GRPC_RDMA_BUSY_POLLING_TIMEOUT_US (500), GRPC_RDMA_POLLER_SLEEP_TIMEOUT_MS
 * (1000), GRPC_RDMA_MAX_SGE (30: what ibv_query_device reported on the authors'
 * HCA, pair.cc:33-35) plus B200_RING_BUFFER_SIZE_BYTES for sub-KB test rings and
 * B200_SEND_COALESCE (0 / 1, default 0): 1 = coalesced send framing, every Send call
 * writes ONE frame gathering up to 1024 slices from byte_idx on, cut where staging or
 * credit runs out (max_sge does not apply; zero-length slices are skipped, not a stop).
 * The peer's receive side is unchanged and needs no negotiation (DESIGN.md §2).
 * Like GRPC_RDMA_MAX_SGE it is captured into the pair at b200_pair_init.
 * B200_RING_STAMPED (0 / 1, default 0): 1 = the pair offers stamped ring frames
 * (header = p | t << 40 with a per-frame stamp t, footer = ~header; the receiver
 * never clears what it retires).  Captured at b200_pair_init and offered in the
 * address blob when the ring is <= 256 MiB; a connection runs stamped frames only
 * when both ends offered them, otherwise the reference format (DESIGN.md §2).
 * Return values, cursors and the delivered stream are those of the reference.
 * The environment is read at b200_init; b200_config_set overrides afterwards
 * (affects pairs initialised later).  Returns 0 / -1 (unknown key, bad value). */
int b200_config_set(const char* key, const char* value);
int64_t b200_config_get(const char* key);

/* --------------------------------------------------------------- memory */
void* b200_mem_alloc_device(size_t bytes);
void b200_mem_free_device(void* p);
void* b200_mem_alloc_host(size_t bytes); /* pinned + GPU-addressable (UVA) */
void b200_mem_free_host(void* p);
int b200_mem_register_host(void* p, size_t bytes); /* ibv_reg_mr analogue */
int b200_mem_unregister_host(void* p);
/* Stream-ordered copies (dir: 0 = host->device, 1 = device->host, 2 = d->d). */
int b200_memcpy(void* dst, const void* src, size_t bytes, int dir, void* stream);
int b200_stream_sync(void* stream); /* NULL = the runtime's own stream */

/* ------------------------------------------------------------ pool / pair */

/* PairPool::Take / Putback, pair.h:288-310 */
b200_pair* b200_pool_take(const char* id);
void b200_pool_putback(b200_pair* p);
/* PairPool::Get(id), pair.h:312-320 */
b200_pair* b200_pool_get(const char* id);

/* PairPollable::Init, pair.cc:85-141: (re)allocate + zero the HBM ring and
 * cursors; status -> INITIALIZED. */
void b200_pair_init(b200_pair* p);
/* get_self_address().bytes(), pair.h:150 + address.cc:19: writes
 * B200_ADDRESS_BYTES, returns the size. */
size_t b200_pair_self_address(b200_pair* p, void* out48);
/* PairPollable::Connect, pair.cc:143-168.  1 = connected, 0 = failed (tag or
 * ring size mismatch, peer not reachable by an available wire). */
int b200_pair_connect(b200_pair* p, const void* peer48, size_t n);
/* PairPollable::Disconnect, pair.cc:325-347: tells the peer (peer_exit=1). */
void b200_pair_disconnect(b200_pair* p);

/* PairPollable::Send(grpc_slice*, count, byte_idx), pair.cc:645-734: one frame
 * per slice, <= max_sge frames, a slice is cut only when staging or remote
 * credit runs out (a pair initialised with B200_SEND_COALESCE=1: one frame per
 * call, see above).  Returns payload bytes accepted. */
uint64_t b200_pair_send(b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx);
/* PairPollable::Recv, pair.cc:264-286: at most one frame (or the rest of a
 * partially consumed one) into dst; returns bytes delivered. */
uint64_t b200_pair_recv(b200_pair* p, void* dst, uint64_t cap);

/* pair.cc:288-303 -- wait-free reads of the host-visible mirror that the
 * kernels keep current. */
int b200_pair_has_message(const b200_pair* p);
int b200_pair_has_pending_writes(const b200_pair* p);
uint64_t b200_pair_readable(const b200_pair* p);
uint64_t b200_pair_writable(const b200_pair* p);
/* get_status, pair.cc:349-375; get_error, pair.cc:643 */
enum b200_status b200_pair_status(b200_pair* p);
const char* b200_pair_error(const b200_pair* p);
/* 1 when the connected pair runs stamped ring frames (both ends offered
 * B200_RING_STAMPED), 0 otherwise. */
int b200_pair_stamped(const b200_pair* p);
/* get_wakeup_fd()->read_fd, pair.cc:377: an eventfd the engine registers in
 * epoll with tag ptr|2 (ev_epollex_rdma_bpev_linux.cc:725-741). */
int b200_pair_wakeup_read_fd(b200_pair* p);
/* grpc_wakeup_fd_consume_wakeup on that fd (engine :1018-1021). */
void b200_pair_consume_wakeup(b200_pair* p);

/* Debug / parity inspection (what tests compare with the oracle). */
typedef struct b200_pair_state {
  uint64_t head, moving_head, remain;        /* ring_buffer.h:203-208        */
  uint64_t remote_tail, internal_read_size;  /* pair.h:170-171               */
  uint64_t credit_remote_head;               /* status_report.remote_head    */
  uint32_t partial_write, peer_exit;
  uint64_t ring_capacity;
} b200_pair_state;
int b200_pair_get_state(b200_pair* p, b200_pair_state* out);
/* Copy the pair's HBM ring image to host memory (cap >= ring capacity). */
int b200_pair_copy_ring(b200_pair* p, void* host_dst, uint64_t cap);

/* ------------------------------------------------------------ device API */
/*
 * Hand one end of a connection to the caller's own kernels: they drive it with the warp-collective calls of
 * include/b200_device.cuh (b200_warp_send / b200_warp_recv / readiness) instead of b200_pair_send / recv.
 *
 * b200_pair_device_claim: the pair must be CONNECTED and have no host op in flight (a single call, a submit
 * pass, a posted op) -- otherwise -1 and b200_last_error.  It drains an eagerly received frame's owed Retire,
 * makes the service's owner warps drop their cached copy of the connection, marks the pair device-owned and
 * fills *out (0).  While the pair is device-owned, host operations on THIS end are refused: b200_pair_send /
 * recv return 0 (b200_pair_error says why), b200_pairs_send / recv / submit, b200_batch_prepare_* and
 * b200_pair_post_* with this pair fail.  The readiness queries, get_state and copy_ring keep working (from the
 * mirrors the device calls publish).  The PEER end is unaffected: it may stay host-driven, with or without the
 * service, or be claimed as well.
 * b200_pair_device_release: the caller guarantees that the kernels using the handle have finished.  The
 * mirrors are re-published from the device state and host calls resume (0; -1 if the pair is not claimed).
 * b200_pair_disconnect, b200_pair_init and b200_pool_putback on a claimed pair release the claim first.
 * An end the device closed with b200_warp_disconnect: b200_pair_status says DISCONNECTED from then on; the release
 * finishes the Disconnect on the host (the wire and the address go, nothing more is written to the peer), after which
 * b200_pair_init, Connect and b200_pool_putback work as after b200_pair_disconnect -- which, on such an end, is the
 * release and nothing else.
 */
typedef struct b200_dev_pair {
  void* table;     /* the connection table (PairDev rows, then the PairSeq side array) */
  void* seq;       /* the PairSeq side array (stamped frames' counters) */
  void* mirrors;   /* host-visible mirrors (pinned, mapped), indexed by slot */
  int32_t slot;    /* this pair's row */
  uint32_t wire;   /* 0 = loopback (same GPU), 1 = peer GPU over NVLink */
  uint64_t _reserved[4];
} b200_dev_pair;   /* POD, 64 bytes: pass it by pointer (device or pinned memory) or by value */
int b200_pair_device_claim(b200_pair* p, b200_dev_pair* out);
/*
 * b200_pair_device_claim_ex: b200_pair_device_claim with flags; b200_pair_device_claim(p, out) is
 * b200_pair_device_claim_ex(p, 0, out).  Unknown flag bits: -1 and b200_last_error.
 * B200_CLAIM_UNMIRRORED: while the end is claimed, nothing writes its host-visible mirror -- not the device calls of
 * either end, the service, the Poller nor the host calls of the peer.  For a connection whose bytes never leave the
 * GPU this takes the per-call publication (PCIe stores, system-scope fences, the per-pair mirror lock) off the device
 * calls.  Every data result is the mirrored claim's, bit for bit, in every framing mode.  The peer end keeps its own
 * mirror as before: a host-driven peer still sees its readiness after our Send and its credit after our Recv.
 *   - Frozen queries: b200_pair_status, b200_pair_has_message / has_pending_writes / readable / writable on this end
 *     answer from the mirror as the claim left it, until the release (a device Disconnect of the end included).
 *     get_state and copy_ring read the device and keep working; the kernel has the device queries of
 *     b200_device.cuh.
 *   - Refused (-1) besides the plain claim's refusals: while the loopback peer has a host op in flight.  A peer end
 *     that a kernel drives must not be inside a call at the claim.
 *   - On the CUDA-IPC wire with the service running, the claim waits for the device poller's scans in progress to
 *     pass, then rebuilds the frozen mirror from the device state.
 *   - b200_pair_device_release publishes again: the mirror is rebuilt from the device state, and a Disconnect the
 *     device made (b200_warp_disconnect) is finished as on a mirrored end.
 */
#define B200_CLAIM_UNMIRRORED 0x1
int b200_pair_device_claim_ex(b200_pair* p, int flags, b200_dev_pair* out);
int b200_pair_device_release(b200_pair* p);
/* 1 while the pair is device-owned */
int b200_pair_device_owned(const b200_pair* p);

/*
 * Ready sets: the device's epoll (DESIGN.md §13 "Ready sets").  A polling server kernel that holds many claimed ends
 * takes the ones whose readiness changed from a device queue, b200_warp_ready_take (b200_device.cuh), instead of
 * scanning them all with b200_warp_poll.  Edge-triggered and one-shot, like EPOLLONESHOT with re-arm:
 *   - members are claimed ends (either claim form) on the loopback wire, each with a 32-bit key the caller chooses; an
 *     end belongs to at most one set;
 *   - the peer's Send landing a frame, the peer's Recv returning credit and the peer's Disconnect (host or device)
 *     append the member's key when the member is armed, and disarm it: a member has at most one entry queued;
 *   - a member is READY when b200_warp_poll reports it READABLE, or when it has a pending write (partial_write) and
 *     credit for at least one frame.  The second rule is narrower than the Poller's WRITABLE (partial_write alone),
 *     which would hand a blocked sender back to an edge-triggered consumer again and again;
 *   - any number of consumer warps per set, in one CTA or in many, in one kernel or in several: each takes, drives
 *     the ends it took with the device calls, then b200_warp_ready_rearm each end it has finished with.  Each entry
 *     goes to exactly one warp, which holds the member until its rearm returns 0 (b200_device.cuh: the holder rule).
 * b200_ready_set_create: 1 <= capacity <= 8192 members; the queue and its control words live in device memory.  NULL
 * and b200_last_error on failure.
 * b200_ready_set_device fills the 64-byte handle the consumer kernel takes (0 / -1).
 * b200_ready_set_destroy: the caller guarantees that no kernel uses the set.  -1 while the set has members.
 * b200_ready_set_add: p must be device-owned, on the loopback wire and in no set.  A one-thread library kernel on the
 * runtime's stream writes the member's note and queues one initial entry with the member disarmed, so a frame or a
 * close that came before the add is not lost.  It may run while a consumer kernel takes from the set (a running
 * server gets a new connection).  -1 and b200_last_error: p not claimed, p on the CUDA-IPC wire (its peer's kernels
 * run in another process and cannot reach this queue), p already a member, the set full, or the queue could overflow
 * because of stale entries (entries queued plus members reach the queue's size, twice the capacity rounded up to a
 * power of two).
 * Membership ends with the claim: b200_pair_device_release (and with it b200_pair_disconnect, b200_pair_init and
 * b200_pool_putback) clears the member's note before it republishes.  The kernels that use the pair's handle must have
 * finished before the release, as always; ops of the peer must not run across it.  Once the release returns nothing
 * more is queued for the end, but an entry already queued can still be taken once, and counts against the queue's
 * size until then.
 *
 * Parking (DESIGN.md §13 "Parking"): a server kernel need not stay resident while its set is idle.  It parks the set
 * (b200_warp_ready_park) and exits; the next entry queued on a parked set -- a frame, credit or close of a member, or
 * b200_ready_set_add's initial entry -- rings the set's doorbell once: a 64-bit counter in pinned host memory.  The
 * Poller threads turn a doorbell that moved into a kick of the set's eventfd; the application polls that fd and
 * launches the server again.  A release of a member rings nothing.
 * b200_ready_set_park: the same park from the host, through a one-thread library kernel on the runtime's stream: 0 the
 * set is parked, 1 entries are queued (launch a server; the set is not parked), -1 and b200_last_error on failure.  No
 * consumer may take from the set while it runs.  A set starts unparked; parking it before any server runs launches
 * servers on demand, and parking it after the host stopped its server itself makes the next change ring.  The kernel is
 * loaded with the library's others, so a host park may run beside resident kernels.
 * b200_ready_set_wakeup_fd: the set's eventfd (-1 on failure).  The first call creates it, registers the set with the
 * Poller and starts the Poller's threads, as b200_poller_add does; a ring from before the call signals it as well.
 * b200_ready_set_consume_wakeup: reads the eventfd back to not-readable.
 * b200_ready_set_rings: the doorbell, the rings so far; a wait-free read of pinned memory, for a host that busy-polls
 * for a while before it waits on the fd.  b200_ready_set_destroy unregisters the set and closes its fd.
 */
typedef struct b200_ready_set b200_ready_set;
typedef struct b200_dev_ready_set {
  void* queue;        /* control words, then the entries (device memory) */
  uint32_t capacity;  /* members at most */
  uint32_t size;      /* entries of the queue */
  uint64_t _reserved[6];
} b200_dev_ready_set;  /* POD, 64 bytes: pass it by pointer (device or pinned memory) or by value */
b200_ready_set* b200_ready_set_create(uint32_t capacity);
int b200_ready_set_device(b200_ready_set* s, b200_dev_ready_set* out);
int b200_ready_set_destroy(b200_ready_set* s);
int b200_ready_set_add(b200_ready_set* s, b200_pair* p, uint32_t key);
int b200_ready_set_park(b200_ready_set* s);
int b200_ready_set_wakeup_fd(b200_ready_set* s);
void b200_ready_set_consume_wakeup(b200_ready_set* s);
uint64_t b200_ready_set_rings(const b200_ready_set* s);

#if defined(__cplusplus)
static_assert(sizeof(b200_dev_pair) == 64, "b200_dev_pair is 64 bytes");
static_assert(sizeof(b200_dev_ready_set) == 64, "b200_dev_ready_set is 64 bytes");
#endif

/* ------------------------------------------------------------------ poller */

/* Poller::AddPollable / RemovePollable / Shutdown, poller.cc:12-49, poller.h:37.
 * Background thread(s) launch the readiness-scan kernel over all registered
 * pairs and kick a pair's eventfd when it is readable, has a pending partial
 * write, or its peer went away (poller.cc:75-101). */
void b200_poller_add(b200_pair* p);
void b200_poller_remove(b200_pair* p);
void b200_poller_shutdown(void);

/* One synchronous readiness scan over `n` pairs (the body of the engine's
 * busy-poll window, ev_epollex_rdma_bpev_linux.cc:1104-1145): events[i] gets
 * B200_EV_* bits.  Returns the number of pairs with a non-zero event. */
#define B200_EV_READABLE 0x1u /* EPOLLIN: HasMessage, or HalfClosed / Error */
#define B200_EV_WRITABLE 0x4u /* EPOLLOUT: HasPendingWrites */
int b200_poller_scan(b200_pair* const* pairs, size_t n, uint32_t* events);

/* ----------------------------------------------------------------- service */
/*
 * The resident kernels of the unary path (the "persistent warp-per-connection kernel" and the busy-poll half of the
 * BPEV completion loop).  b200_service_start launches three of them and keeps them resident:
 *   owners  one WARP per host command queue.  b200_pair_send / recv post a 128-byte command into the queue of the
 *           pair's connection (both ends of a loopback connection share a queue) and spin on a 16-byte answer.  A
 *           small call (a unary message) is planned, moved, retired and published by that warp alone -- no launch,
 *           no stream synchronisation, no CTA barrier, no lock; a frame that lands at the head of the peer's ring
 *           is pushed to the peer's host slot at once, so the peer's Recv does not need a trip to the GPU.
 *   pool    `workers` CTAs with the k_send / k_recv machinery for everything larger (and for the rdma_flush /
 *           rdma_do_read loops of b200_pairs_submit), fed by the owners through mailboxes in device memory.
 *   poller  scans the connection table continuously, keeps the host-visible mirror of pairs on the nvlink wire
 *           current and appends readiness CHANGES to a ready ring in mapped host memory (one atomic per warp); the
 *           background Poller threads turn those into eventfd kicks instead of launching scans.
 * Returns 0 / -1.  While the service runs: no device-wide synchronisation (cudaDeviceSynchronize, cudaFree; the
 * library defers its own frees until b200_service_stop) and no FIRST launch of a kernel in the process (lazy module
 * loading waits for an idle device; the library loads all of its own kernels before it starts the service).
 */
/* `workers` = pool CTAs (B200_SERVICE_WORKERS, default 16); B200_SERVICE_OWNERS = owner warps = host command queues
 * (default 32).  Fails (-1) when the resident grids would not fit on the device together. */
int b200_service_start(int workers);
/* Call with no b200_pair_send / recv in flight (they would wait for a worker that has left). */
void b200_service_stop(void);
int b200_service_running(void); /* number of pool CTAs, 0 = not running */
/* out[0] commands executed, [1] ready-ring entries consumed, [2] ready-ring overruns,
 * [3] device poller scans (updated every 1024 scans) */
void b200_service_stats(uint64_t out[4]);
/* Recv calls answered from a pair's eagerly pushed host slot (no trip to the GPU and back). */
uint64_t b200_service_eager_hits(void);

/* ------------------------------------------------------------------- batch */
/*
 * GPU-native widening of Send/Recv: one kernel launch serves many pairs
 * (what the engine's event loop would otherwise do pair by pair).  Semantics
 * per op are those of the endpoint loops around the single calls:
 *   B200_BATCH_ONE_CALL      exactly one Send / one Recv per op
 *   B200_BATCH_UNTIL_BLOCKED rdma_flush re-entered while Send accepts bytes
 *                            (rdma_bp_posix.cc:470-557) / rdma_do_read's loop
 *                            until dst is full or no complete frame is left
 *                            (rdma_bp_posix.cc:180-286)
 * All pointers must be GPU-addressable (see the memory rule above).
 */
#define B200_BATCH_ONE_CALL 0x0
#define B200_BATCH_UNTIL_BLOCKED 0x1
#define B200_BATCH_ASYNC 0x2 /* do not synchronise; results valid after stream sync */
#define B200_BATCH_ZEROCOPY 0x4 /* pinned HOST buffers are dereferenced by the kernels over PCIe */
/* Sends and Recvs of the SAME connection may run at the same time (batches launched on separate
 * streams without an ordering between them): the kernels then update the host-visible mirrors under a
 * per-pair device lock so that an older readiness / credit view can never overwrite a newer one.
 * The service kernel always works this way; the library's own lanes order the two ends by events and
 * do not need it. */
#define B200_BATCH_CONCURRENT 0x8
/* Cluster width of a batch, 1 <= k <= 16, in bits 4..7 of the flags (they hold k - 1).  Field 0, the default and
 * B200_BATCH_CLUSTER(1), is one CTA per op.  k >= 2 runs each op on a thread-block cluster of k CTAs (kernels
 * k_cluster_send / k_cluster_recv, DESIGN.md §13): the planner of CTA rank 0 plans the op and the movers of all k
 * CTAs move its bytes, so one connection keeps up to k times as many reads in flight.  The results are those of the
 * same batch launched with field 0 from the same state, bit for bit -- per-op bytes and b200_batch_calls,
 * partial_write, cursors, credit, frames and ring images, the delivered bytes and (host-staged) the whole copied-back
 * window -- in every framing mode.  Accepted by b200_pairs_send / recv and b200_batch_prepare_send / recv on all three
 * memory paths (device, host-staged lanes, B200_BATCH_ZEROCOPY); bits above 7 are ignored.
 *   - The caller chooses k: whether clusters pay depends on the message size and on what else occupies the GPU.  With
 *     few connections and large messages they do; with 64 connections on an H100, clusters of 4 or more CTAs lose.
 *   - b200_batch_prepare_* and b200_pairs_send / recv fail (NULL / -1, b200_last_error) when
 *     cudaOccupancyMaxActiveClusters says the device cannot place one cluster of k CTAs of the kernel.  That query
 *     does not see resident kernels: beside the service or a user's device-API kernel, a cluster launch needs k free
 *     CTA slots within one GPC and waits for them, as a one-CTA launch waits for one free slot.
 *   - b200_pairs_submit and b200_pair_post_send / recv run on the service's owners and pool, not on these kernels:
 *     they refuse a nonzero field (-1; NULL with *again = 0) and say why in b200_last_error. */
#define B200_BATCH_CLUSTER(k) (((unsigned)(k) - 1u) << 4)
/*
 * Where the bytes live decides the path of a batch:
 *   device memory        kernels work in place (one launch per batch);
 *   pinned host memory   HOST-STAGED path (default): the batch owns a device staging arena and
 *                        runs as 8 independent lanes (internal streams), each H2D -> Send kernel
 *                        or Recv kernel -> D2H, so the copy engines and the SMs overlap; a
 *                        connection always maps to the same lane, which keeps its Send and Recv
 *                        ordered.  With a NULL stream the lanes run free (b200_lanes_join or
 *                        b200_batch_results to wait); with a stream the batch forks from / joins
 *                        back into it.  A Recv copies its WHOLE destination window back: bytes
 *                        past `delivered` are the batch's staging bytes there (zero, or what an
 *                        earlier launch of the same batch delivered).  B200_BATCH_ZEROCOPY
 *                        instead lets the kernels read and write the pinned buffers directly
 *                        (GPUDirect-style, no staging).
 */

/* Threading of this section: a prepared batch belongs to one thread at a time (launch / results / destroy are not
 * locked against each other); different batches may be driven from different threads, the host-staged lanes and the
 * runtime's default stream are shared, so concurrent launches interleave there in submission order.
 * b200_pairs_submit and the post / poll calls are thread-safe (per-queue posting sections, per-thread staging).
 *
 * A batch launched while the service runs (b200_service_start) may run beside single calls on the same connection,
 * within the rule above: one Send and one Recv of a pair at a time, e.g. a batch Send on one end and b200_pair_recv on
 * the other.  From the launch until b200_batch_results (or b200_batch_destroy), the service reads that connection's
 * state fresh for every call and publishes both ends' readiness under the per-pair locks, as the batch's kernels do
 * (B200_BATCH_CONCURRENT is implied); once the results are collected, no call works from a view taken before the
 * batch ran.  A single call that returns before the batch runs is ordered before it, one that starts after
 * b200_batch_results is ordered after it; in between, the per-op counts depend on timing and the byte stream does
 * not. */
typedef struct b200_send_op {
  b200_pair* pair;
  const b200_slice* slices; /* host array of n entries (copied at submit) */
  size_t nslices;
  size_t byte_idx;
} b200_send_op;

typedef struct b200_recv_op {
  b200_pair* pair;
  void* dst;
  uint64_t cap;
} b200_recv_op;

/* Returns 0 on success.  accepted/delivered: nops entries (may be NULL); with
 * B200_BATCH_ASYNC they must be pinned host memory (b200_mem_alloc_host). */
int b200_pairs_send(const b200_send_op* ops, size_t nops, int flags, uint64_t* accepted, void* stream);
int b200_pairs_recv(const b200_recv_op* ops, size_t nops, int flags, uint64_t* delivered, void* stream);

/* One event-loop pass: all ready Sends and Recvs posted together, waited for together (what
 * pollable_process_events does closure by closure, ev_epollex_rdma_bpev_linux.cc:977-1066).  With the service
 * running nothing is launched: every op is a command of its pair's owner queue, slices (any host memory;
 * unregistered slices are staged) and destinations (GPU-addressable) are used in place.  0 on success.
 * At most one Send op and one Recv op of a pair may be in flight at a time -- within one pass and across threads
 * (the ContentAssertion rule above): a pair's Send and Recv run side by side on the pool, but two Sends (or two
 * Recvs) of one pair would overlap too, because an owner hands a job to the pool after reaping only the jobs that
 * have already finished.  A pass that holds the Send of one direction of a connection and the Recv of the same
 * direction runs both concurrently: their per-op counts depend on timing, the delivered stream does not. */
int b200_pairs_submit(const b200_send_op* sops, size_t ns, uint64_t* accepted, const b200_recv_op* rops, size_t nr,
                      uint64_t* delivered, int flags);

/* Completion-queue form of the same (service running only): post now, poll later -- the event loop never waits
 * for the GPU, every connection advances at its own pace.  A posted op is an rdma_flush loop / rdma_do_read loop
 * (B200_BATCH_UNTIL_BLOCKED) or a single call.  Recv into pinned HOST memory is delivered into device staging and
 * taken down by the copy engine (one contiguous copy); the op completes when the bytes are in `dst`.
 * post: NULL + *again = 1 when the pair's command queue has no free entry right now (poll something, post later);
 *       NULL + *again = 0 on error.  poll: 1 = finished (bytes valid, handle released), 0 = still running, -1 = error. */
typedef struct b200_async b200_async;
b200_async* b200_pair_post_send(b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx, int flags, int* again);
b200_async* b200_pair_post_recv(b200_pair* p, void* dst, uint64_t cap, int flags, int* again);
int b200_async_poll(b200_async* op, uint64_t* bytes);

/* Prepared batches: descriptors uploaded to HBM once, launched many times
 * (streaming workloads that reuse their buffers; CUDA-graph friendly). */
typedef struct b200_batch b200_batch;
b200_batch* b200_batch_prepare_send(const b200_send_op* ops, size_t nops, int flags);
b200_batch* b200_batch_prepare_recv(const b200_recv_op* ops, size_t nops, int flags);
int b200_batch_launch(b200_batch* b, void* stream);       /* asynchronous */
/* Per-op byte counts of the most recent launch (synchronises the stream). */
int b200_batch_results(b200_batch* b, uint64_t* out, void* stream);
/* Lanes of the host-staged path: make them wait for `stream` / make `stream` (or, with NULL,
 * the calling thread) wait for them. */
int b200_lanes_fork(void* stream);
int b200_lanes_join(void* stream);
/* Per-op number of Send / Recv calls that moved bytes, as fetched by the last
 * b200_batch_results (parity with the endpoint loops' iteration counts). */
int b200_batch_calls(b200_batch* b, uint64_t* out);
void b200_batch_destroy(b200_batch* b);

/* Calibration: copy `bytes_per_cta` bytes per CTA (CTA i works at offset i*stride of src+mis
 * and dst) with the same one-CTA-per-connection decomposition and copy primitives as the Send
 * kernel but no framing.  Tells what that grid shape can reach on this GPU. */
int b200_probe_copy(void* dst, const void* src, uint64_t bytes_per_cta, uint64_t stride, int nctas, int threads,
                    uint32_t mis, uint32_t item_bytes, uint32_t dynamic, void* stream);

/* Number of kernels this library has launched so far (bench: gpu_launches). */
uint64_t b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_PAIR_H */
