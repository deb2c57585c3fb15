// b200_dev.cuh -- device-visible state of a connection and the integer helpers
// shared by the sm_90a kernels and the host runtime.
//
// Reference being replaced (paths relative to the reference root):
//   RingBufferPollable state      src/core/lib/ibverbs/ring_buffer.h:203-208
//   PairPollable cursors/credit   src/core/lib/ibverbs/pair.h:100-103,168-172
//   credit / framing arithmetic   src/core/lib/ibverbs/ring_buffer.h:180-189,
//                                 ring_buffer.cc:99-116
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif

namespace b200 {

constexpr uint64_t kAlign = 8;          // ring_buffer.h:49
constexpr uint64_t kReserved = 24;      // ring_buffer.h:52 (header, footer, one spare word)
constexpr uint64_t kFooter = ~0ull;     // ring_buffer.h:50
constexpr int kMaxSgeLimit = 32;        // planner handles one warp of slices per Send call
// Coalesced framing (B200_SEND_COALESCE=1): one frame per Send call gathering up to kCoalesceSlices
// slices.  The mode travels in the top bit of PairDev::max_sge (max_sge itself is <= kMaxSgeLimit).
constexpr uint32_t kCoalesceSlices = 1024;
constexpr uint32_t kSgeCoalesce = 0x80000000u;
// Stamped ring frames (B200_RING_STAMPED=1, negotiated at Connect, DESIGN.md §2): frame s of a direction
// carries t(s) = 1 + s mod (2^24 - 1) in the top 24 bits of its header, footer = ~header, and the receiver
// never clears what it retires.  The mode travels in bit 30 of PairDev::max_sge.
constexpr uint32_t kSgeStamped = 0x40000000u;
constexpr uint32_t kSgeModeBits = kSgeCoalesce | kSgeStamped;
constexpr uint64_t kStampMod = (1ull << 24) - 1;
constexpr uint64_t kLenMask = (1ull << 40) - 1;
// fewer than C/24 frames fit in one lap, so a leftover header of the last lap never carries the stamp
// expected at its position while C/24 < 2^24 - 1
constexpr uint64_t kStampedMaxCap = 256ull << 20;
constexpr int kMaxPairs = 8192;  // rows of the connection table

B200_HD uint64_t round_up8(uint64_t v) { return (v + 7) & ~7ull; }
B200_HD uint64_t round_down8(uint64_t v) { return v & ~7ull; }
// GetEncodedSize, ring_buffer.h:180-183
B200_HD uint64_t encoded_size(uint64_t payload) { return 16 + round_up8(payload); }
// CalculateWritableSize, ring_buffer.h:185-189
B200_HD uint64_t calc_writable(uint64_t space) { return space > kReserved ? round_down8(space - kReserved) : 0; }
// GetFreeSize, ring_buffer.cc:99-104
B200_HD uint64_t free_size(uint64_t cap, uint64_t head, uint64_t tail) {
  return cap - ((tail + cap - head) & (cap - 1));
}
// GetWritableSize(head, tail), ring_buffer.cc:106-116
B200_HD uint64_t writable_size(uint64_t cap, uint64_t head, uint64_t tail) {
  uint64_t f = free_size(cap, head, tail);
  return f > kReserved ? f - kReserved : 0;
}

// ---- stamped frames.  `st` is the stamp a frame must carry; st = 0 selects the reference format
// (header = p, footer = ~0), so one call site serves both modes.
B200_HD uint32_t stamp_of(uint64_t s) { return 1u + (uint32_t)(s % kStampMod); }
B200_HD uint64_t frame_header(uint64_t p, uint32_t st) { return p | (uint64_t)st << 40; }
B200_HD uint64_t frame_footer(uint64_t hdr, uint32_t st) { return st ? ~hdr : kFooter; }
// payload length of the frame whose header word is `hdr` when it is present at the head (a valid length, and
// in stamped mode the expected stamp), else 0
B200_HD uint64_t frame_present(uint64_t hdr, uint64_t cap, uint32_t st) {
  const uint64_t p = st ? hdr & kLenMask : hdr;
  if (st && (uint32_t)(hdr >> 40) != st) return 0;
  return p != 0 && p <= cap - kReserved ? p : 0;
}
// ... and complete: the footer word as well
B200_HD uint64_t frame_complete(uint64_t hdr, uint64_t foot, uint64_t cap, uint32_t st) {
  const uint64_t p = frame_present(hdr, cap, st);
  return p && foot == frame_footer(hdr, st) ? p : 0;
}

// Host-visible mirror of one pair (pinned, GPU-mapped).  Kernels refresh the
// fields they own at the end of every op that touches the pair (posted writes
// only) so that HasMessage / HasPendingWrites / get_status stay wait-free host
// reads (pair.cc:288-303).
struct PairMirror {
  uint64_t head, moving_head, remain, acc;
  uint64_t remote_tail, credit_head;
  uint64_t readable;       // GetReadableSize() as of the last refresh
  uint32_t partial_write;  // HasPendingWrites()
  uint32_t peer_exit;      // status_report.peer_exit seen by this pair
  uint32_t has_message;    // HasMessage()
  uint32_t dev_closed;     // 1 once b200_warp_disconnect closed this device-owned end (0 from Init on; the release
                           // finishes the Disconnect on the host)
};

// One connection endpoint in HBM.  Three blocks with distinct writers:
//   setup  : written by the host at Init/Connect/Disconnect only
//   cursor : owned by this pair's own send/recv kernels
//   credit : the 16-byte status_report the PEER writes (pair.h:100-103);
//            16-byte aligned so one v2.u64 store updates it atomically
struct __align__(128) PairDev {
  // ---- setup
  uint8_t* ring;         // this pair's receive ring (HBM), all-zero when empty
  uint64_t cap;          // power of two (ring_buffer.cc:22)
  uint8_t* peer_ring;    // where Send lands frames: the peer's ring (remote_addr)
  uint64_t* peer_credit; // address of the peer's credit block
  PairMirror* mirror;
  PairMirror* peer_mirror;  // loopback wire only, else nullptr
  uint32_t status;       // b200_status: set by the host at Init / Connect / Disconnect, and to DISCONNECTED by
                         // b200_warp_disconnect on a device-owned end
  uint32_t max_sge;      // frames per Send call (pair.cc:672); | kSgeCoalesce: one coalesced frame per call;
                         // | kSgeStamped: stamped frames both ways (set at Connect when both ends agree)
  int32_t peer_slot;     // loopback wire: index of the peer in this table, else -1
  uint32_t wire;         // 0 = same device, 1 = peer device over NVLink (system-scope fences)
  // ---- cursor
  uint64_t head;         // RingBufferPollable::head_
  uint64_t moving_head;  // moving_head_
  uint64_t remain;       // remain_
  uint64_t acc;          // PairPollable::internal_read_size_
  uint64_t remote_tail;  // PairPollable::remote_tail_
  uint32_t partial_write;
  uint32_t mlock;        // serialises "read the device truth, write the mirror" when ops of the two
                         // ends run concurrently (kFlagConcurrent)
  // ---- credit (offset 112, 16-byte aligned)
  uint64_t credit_head;  // status_report.remote_head
  uint32_t credit_exit;  // status_report.peer_exit
  uint32_t _pad1;        // covered by the peer's 16-byte status write: nothing of ours may live here
};
static_assert(sizeof(PairDev) == 128, "PairDev is one 128-byte line");

// Stamped mode's frame counters of a pair (reset at Init), in the side array that follows the kMaxPairs rows
// of the connection table in the same allocation.  Each is written only by the ops of its own direction.
struct __align__(16) PairSeq {
  uint64_t tx;  // frames this pair's Send calls have written into the peer's ring
  uint64_t rx;  // frames this pair's Recv calls have opened in its own ring
};
B200_HD PairSeq* pair_seq(PairDev* table, int slot) { return reinterpret_cast<PairSeq*>(table + kMaxPairs) + slot; }

// ---- device ready sets (b200_ready_set_*, DESIGN.md §13 "Ready sets").  A set is a queue of 32-bit member keys in
// device memory taken by any number of consumer warps; the paths that change a member's readiness append its key
// (notify_peer).  Control words: the consumers' head and the producers' tail on separate lines, then the entries.
// Parking (DESIGN.md §13 "Parking"): `tail` is the low half of the 64-bit word at offset 128, whose bit 63 is the
// parked bit; producers claim positions with a 64-bit atomicAdd on that word (carries out of the low half stop at bit
// 62), and the one that clears the bit rings the set's doorbell.
struct __align__(128) ReadyQueue {
  uint32_t head;  // next position a consumer takes (advanced by the consumers' atomicCAS in ready_take)
  uint32_t _h[31];
  uint32_t tail;     // next position a producer claims (low half of the 64-bit atomicAdd of ready_push)
  uint32_t tail_hi;  // carries of tail in bits 0..30, the parked bit in bit 31 (bit 63 of the word)
  uint64_t rings;    // doorbell rings so far (device count; each ring stores the new count into *bell)
  uint32_t _t[28];
  uint32_t mask;  // entries - 1, set at creation
  uint32_t _m0;
  uint64_t* bell;  // pinned, mapped host counter of the rings (b200_ready_set_rings), set at creation
  uint32_t _m[28];
};
static_assert(sizeof(ReadyQueue) == 384, "ReadyQueue: three 128-byte lines");
constexpr uint64_t kReadyParked = 1ull << 63;
B200_HD unsigned long long* ready_tail_word(ReadyQueue* q) { return reinterpret_cast<unsigned long long*>(&q->tail); }
// An entry is one 8-byte word: the key, and position + 1 in the top half (0: never written), so the consumer tells a
// written entry from a slot whose producer has claimed it but not yet stored into it.
B200_HD uint64_t* ready_entries(ReadyQueue* q) { return reinterpret_cast<uint64_t*>(q + 1); }
B200_HD uint64_t ready_entry(uint32_t key, uint32_t pos) { return (uint64_t)(pos + 1u) << 32 | key; }
B200_HD bool ready_entry_at(uint64_t e, uint32_t pos) { return (uint32_t)(e >> 32) == pos + 1u; }
// Entries of a set of `capacity` members: a power of two >= 2 * capacity.  Each member has at most one entry queued,
// and an entry of a released member stays until it is taken, so twice the members leaves room for that many stale
// entries before b200_ready_set_add has to refuse.
B200_HD uint32_t ready_queue_size(uint32_t capacity) {
  uint32_t s = 1;
  while (s < 2 * capacity) s <<= 1;
  return s;
}
constexpr int kReadyAddOk = 0, kReadyAddFull = 1, kReadyAddOverflow = 2;
// May one more member join a set whose queue holds positions [head, tail)?  Each present member can still append one
// entry and the new one appends its initial entry, so the entries in the queue plus the members must stay below its
// size.  (tail - head) counts stale entries of released members as well.
B200_HD int ready_add_check(uint32_t head, uint32_t tail, uint32_t members, uint32_t capacity, uint32_t size) {
  if (members >= capacity) return kReadyAddFull;
  return (uint64_t)(tail - head) + members < size ? kReadyAddOk : kReadyAddOverflow;
}
// The note of a ready-set member, in the side array that follows the PairSeq array of the connection table.  `set`
// is null for an end that belongs to no set: the one load every producer pays.
struct __align__(16) ReadyNote {
  ReadyQueue* set;
  uint32_t key;
  uint32_t armed;  // 1: the next readiness change appends the key; 0: an entry is queued or the consumer holds the end
};
B200_HD ReadyNote* ready_note(PairDev* table, int slot) {
  return reinterpret_cast<ReadyNote*>(pair_seq(table, kMaxPairs)) + slot;
}

struct SliceDev {  // same layout as b200_slice
  const uint8_t* ptr;
  uint64_t len;
};

struct SendOpDev {
  int32_t slot;
  uint32_t flags;  // B200_BATCH_*
  const SliceDev* slices;
  uint64_t nslices;
  uint64_t byte_idx;
  uint64_t nreal;  // slices [nreal, nslices) only count towards total_slice_size (pair.cc:661-664): the host folds
                   // what lies beyond max_sge (coalesced: kCoalesceSlices) into one trailing pseudo-slice that
                   // must never be dereferenced
};

struct RecvOpDev {
  int32_t slot;
  uint32_t flags;
  uint8_t* dst;
  uint64_t cap;
};

// per-op result: bytes moved and number of Send/Recv calls that moved > 0
struct OpResult {
  uint64_t bytes;
  uint64_t calls;
};

constexpr uint32_t kFlagUntilBlocked = 0x1;
constexpr uint32_t kFlagConcurrent = 0x8;  // B200_BATCH_CONCURRENT
constexpr uint32_t kEvReadable = 0x1;
constexpr uint32_t kEvWritable = 0x4;

constexpr uint32_t kStConnected = 2;
constexpr uint32_t kStHalfClosed = 3;
constexpr uint32_t kStDisconnected = 4;
constexpr uint32_t kStError = 5;

// ---- persistent service (b200_service_*): three resident kernels.
//   owners  (k_svc_owner): one WARP per command queue.  The host posts 128-byte commands into the
//           queue's ring in pinned mapped memory; the warp polls it (two entries per trip over PCIe),
//           executes small Send / Recv calls entirely by itself -- plan, copy, cursors, credit,
//           mirrors: no CTA barrier, no lock (both ends of a loopback connection map to the same
//           owner, so everything that touches a connection's small ops is program-ordered) -- and
//           hands anything larger to the pool through a mailbox in device memory.
//   pool    (k_svc_big): CTAs that run send_body / recv_body (the k_send / k_recv code) on mailbox
//           jobs and answer the host themselves.
//   poller  (k_svc_poll): the resident readiness scan of the BPEV design (ready ring).
constexpr uint32_t kSvcSend = 1, kSvcRecv = 2, kSvcStop = 3, kSvcRetire = 4, kSvcNop = 5;
constexpr uint32_t kSvcInline = 5;     // slices carried inside the command (a unary call has 2-4)
constexpr uint32_t kOwnQ = 16;         // command entries per owner queue
constexpr uint32_t kOwnBoxes = 8;      // pool jobs in flight per owner
constexpr uint32_t kSmallMax = 8192;   // bytes one warp moves by itself; larger ops go to the pool
constexpr uint32_t kEagerMax = 2048;   // frames up to this size are pushed to the receiver's host slot
constexpr uint32_t kSvcSliceArea = 1024;  // pinned slice descriptors per command entry (+1 for the pseudo-slice
                                          // behind a full coalesced look window)
struct __align__(128) SvcCmd {
  uint32_t stamp;    // ticket + 1, written last by the host (first 64-byte half of the line)
  uint32_t op;       // kSvc*
  int32_t slot;
  uint32_t flags;    // B200_BATCH_*
  uint64_t ptr;      // send: SliceDev* (GPU-addressable; unused when n <= kSvcInline)   recv: destination
  uint64_t n;        // send: nslices                        recv / retire: capacity
  uint64_t byte_idx;
  SliceDev inl[kSvcInline];  // send: the slice list itself when it is short -- no second trip over PCIe
  uint32_t nreal;    // send: slices [nreal, n) only count towards total_slice_size (never dereferenced)
  uint32_t stamp2;   // = stamp, in the second 64-byte half: the two halves may be read by separate PCIe reads
};
static_assert(sizeof(SvcCmd) == 128, "one command = one 128-byte line");
struct __align__(16) SvcDone {  // one 16-byte store: the fields become visible together
  uint64_t bytes;
  uint32_t calls;
  uint32_t seq;      // = SvcCmd.stamp once the op is finished and its bytes are visible
};
static_assert(sizeof(SvcDone) == 16, "one answer = one 16-byte store");
// service-only device state of a pair
struct PairSvc {
  uint64_t delivered;  // payload bytes this pair's Recv calls have returned since the service started
  uint64_t pushed_at;  // value of `delivered` for which the frame at the head was pushed to the host slot (~0: none)
};
// host-visible record of an eagerly pushed frame (pinned): the frame at the head of the ring, complete and
// <= kEagerMax bytes, copied to the pair's host slot so that Recv does not need a trip to the GPU.  No
// ordering between the payload stores and the record is assumed: `csum` covers payload, size and `at`.
struct __align__(32) EagerRec {
  uint64_t at;     // = PairSvc.delivered when the frame was pushed: valid only while the host's count agrees
  uint64_t csum;
  uint32_t size;
  uint32_t magic;
  uint64_t _pad;
};
constexpr uint32_t kEagerMagic = 0xEA6E7001u;
// mailbox owner -> pool (device memory)
struct __align__(128) BigBox {
  uint32_t state;    // 0 free, 1 posted, 2 running, 3 done (owner reaps)
  uint32_t kind;     // kSvcSend / kSvcRecv
  int32_t slot;
  uint32_t flags;
  uint64_t ptr, n, byte_idx, nreal;
  SliceDev inl[kSvcInline];
  SvcDone* done;     // host entry the pool answers into
  uint32_t seq;
  uint32_t _pad;
  OpResult res;
};
B200_HD uint64_t eager_mix(uint64_t x) {
  x ^= x >> 32;
  x *= 0xD6E8FEB86659FD93ull;
  x ^= x >> 32;
  return x;
}
// checksum contribution of payload word j (tail bytes beyond `size` zeroed); XOR of all + eager_mix(at * 31 + size)
B200_HD uint64_t eager_word(uint64_t w, uint32_t j) { return eager_mix(w + (uint64_t)(j + 1) * 0x9E3779B97F4A7C15ull); }

constexpr uint32_t kReadyRing = 4096;  // entries; entry i of the stream sits at i % kReadyRing
struct ReadyEntry {                    // one 8-byte store
  uint32_t stamp;                      // stream index + 1 (0 = never written)
  uint16_t slot;
  uint16_t events;                     // kEv* bits now set for the pair (0 = went idle)
};
struct SvcPollState {                  // device memory
  uint32_t hi_slot;                    // scan slots [0, hi_slot)
  uint32_t stop;
  uint32_t ready_next;                 // next stream index of the ready ring
  uint32_t scans;                      // completed scans (liveness)
};
struct SvcParams {
  PairDev* pairs;
  PairSvc* psvc;
  SvcCmd* cmds;        // [nowners][kOwnQ], pinned
  SvcDone* done;       // [nowners][kOwnQ], pinned
  BigBox* boxes;       // [nowners][kOwnBoxes], device
  EagerRec* erec;      // [kMaxPairs], pinned
  uint8_t* eslots;     // [kMaxPairs][kEagerMax], pinned
  SvcPollState* ps;
  uint32_t* last_ev;
  ReadyEntry* ready;
  uint32_t* host_scans;
  int nowners, nbig;
};

// launch wrappers (b200_kernels.cu)
// cluster >= 2 (B200_BATCH_CLUSTER): each op runs on a cluster of that many CTAs (k_cluster_send / k_cluster_recv)
void launch_send(PairDev* pairs, const SendOpDev* ops, OpResult* results, int nops, void* stream, int cluster = 1);
void launch_recv(PairDev* pairs, const RecvOpDev* ops, OpResult* results, int nops, void* stream, int cluster = 1);
// clusters of `cluster` CTAs of k_cluster_send (kind 0) / k_cluster_recv (kind 1) the device can hold at once, with
// nothing else resident (cudaOccupancyMaxActiveClusters); 0: it cannot place one
int cluster_capacity(int kind, int cluster);
void launch_poll_scan(PairDev* pairs, const int32_t* slots, uint32_t* events, uint32_t* ready_count,
                      int32_t* ready_slots, int n, void* stream);
// ready sets: load the library's kernels (before a user's consumer kernel may be resident); one-thread kernels that
// make pair `slot` a member of `q` with `key`, that run notify_peer for pair `slot` (b200_pair_disconnect), and that
// park `q` and write the park's result to *out (b200_ready_set_park)
void load_kernels();
void launch_ready_add(PairDev* pairs, int slot, ReadyQueue* q, uint32_t key, void* stream);
void launch_ready_notify(PairDev* pairs, int slot, void* stream);
void launch_ready_park(ReadyQueue* q, int* out, void* stream);

// owners / pool / poller on three streams; returns false when the resident grids cannot be co-resident
bool launch_service(const SvcParams& sp, void* s_owner, void* s_big, void* s_poll);
int svc_trace_read(unsigned long long* out16);  // -DB200_SVC_TRACE builds only (device-side phase timers)

void launch_probe_copy(uint8_t* dst, const uint8_t* src, uint64_t bytes_per_cta, uint64_t stride, int nctas,
                       int threads, uint32_t mis, uint32_t item_bytes, uint32_t dynamic, void* stream);

}  // namespace b200
