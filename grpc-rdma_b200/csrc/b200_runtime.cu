// b200_runtime.cu -- host runtime behind include/b200_pair.h.
//
// Owns the HBM-resident connection table (PairDev[]), the pinned host mirrors,
// the pair pool, the bootstrap blob / loopback wire registry, the single-call
// and batched submit paths and the background poller.  No data byte is touched
// by the CPU on the batch path; the single-pair calls bounce UNREGISTERED host
// memory through pinned staging exactly like the reference copies slices into
// its registered send buffer (pair.cc:690-694).
//
// Reference counterparts (relative to the reference root):
//   PairPollable lifecycle  src/core/lib/ibverbs/pair.cc:85-168,325-375
//   PairPool                src/core/lib/ibverbs/pair.h:273-333
//   Poller                  src/core/lib/ibverbs/poller.cc:12-106
//   Config                  src/core/lib/ibverbs/config.cc:45-115
//   Address blob            src/core/lib/ibverbs/address.h:24-31
#include <cuda_runtime.h>
#include <errno.h>
#include <poll.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <fcntl.h>
#include <signal.h>
#include <sys/eventfd.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <map>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/b200_pair.h"
#include "b200_dev.cuh"

using namespace b200;

// ----------------------------------------------------------------- errors

static thread_local std::string t_err;
static void set_err(const std::string& s) { t_err = s; }
#define CU_OK(call)                                                                      \
  ([&]() -> bool {                                                                       \
    cudaError_t e__ = (call);                                                            \
    if (e__ != cudaSuccess) {                                                            \
      set_err(std::string(#call) + ": " + cudaGetErrorString(e__));                      \
      return false;                                                                      \
    }                                                                                    \
    return true;                                                                         \
  }())

// ------------------------------------------------------------------ config

struct Config {
  uint64_t ring_bytes = 4096ull * 1024;  // GRPC_RDMA_RING_BUFFER_SIZE_KB, config.cc:90-96
  int poller_threads = 1;                // GRPC_RDMA_POLLER_THREAD_NUM, config.cc:66-73
  int busy_poll_us = 500;                // GRPC_RDMA_BUSY_POLLING_TIMEOUT_US, config.cc:75-81
  int poller_sleep_ms = 1000;            // GRPC_RDMA_POLLER_SLEEP_TIMEOUT_MS, config.cc:83-89
  int max_sge = 30;                      // ibv_device_attr.max_sge on the authors' HCA
  int send_coalesce = 0;                 // B200_SEND_COALESCE: one frame per Send call (DESIGN.md §2)
  int ring_stamped = 0;                  // B200_RING_STAMPED: offer stamped ring frames at Connect (DESIGN.md §2)
};

// Address blob: same 48-byte layout as grpc_core::ibverbs::Address::addr_
struct AddrBlob {
  uint32_t lid;
  uint32_t qpn;
  uint32_t psn;
  uint32_t _pad0;
  uint8_t gid[16];
  uint32_t tag;
  uint32_t _pad1;  // capability bits of this library (kBlob*); 0 in every blob written before they existed
  uint64_t ring_buffer_size;
};
static_assert(sizeof(AddrBlob) == B200_ADDRESS_BYTES, "address blob must stay 48 bytes");
constexpr uint32_t kBlobStamped = 0x1;  // this end offers stamped ring frames

struct b200_pair {
  int slot = -1;
  int status = B200_UNINITIALIZED;
  std::string id, error;
  uint8_t* ring = nullptr;
  uint64_t cap = 0;
  int wakeup_fd = -1;
  PairMirror* mirror = nullptr;
  AddrBlob self{};
  AddrBlob peer{};
  b200_pair* peer_local = nullptr;  // loopback wire
  // nvlink wire: the peer lives in another process (another GPU of the box); its ring and its
  // row of the connection table are mapped here through CUDA IPC
  bool remote = false;
  uint8_t* remote_ring = nullptr;
  uint64_t* remote_credit = nullptr;
  std::string wire_file;  // this pair's descriptor under /dev/shm (unlinked on Disconnect)
  bool in_poller = false;
  int peer_pid = 0;  // nvlink wire: the process that owns the peer; probed every 500 ms by get_status
  std::atomic<bool> peer_dead{false};  // ... and found gone (kept on the host: the mirror is re-published from the device)
  std::chrono::steady_clock::time_point last_probe{};
  int max_sge = 30;  // captured at Init (what the kernels use for this pair)
  bool coalesce = false;  // B200_SEND_COALESCE, captured at Init like max_sge
  bool stamp_offer = false;  // B200_RING_STAMPED at Init and a ring of <= kStampedMaxCap: the blob's kBlobStamped
  bool stamped = false;      // negotiated at Connect: both ends offered stamped frames
  // service: payload bytes Recv has returned since the service started (the device keeps the same count;
  // an eagerly pushed frame is valid only while both agree), and the asynchronous Retire of the last
  // eagerly received frame, if it has not been confirmed yet
  uint64_t svc_delivered = 0;
  std::atomic<bool> retire_pending{false};
  int retire_q = 0;
  uint64_t retire_ticket = 0;
  std::atomic<uint32_t> retire_owed{0};  // size of an eagerly received frame whose Retire has not been posted yet:
                                         // it rides on the pair's next Send, or is posted by whoever looks next
  // device API (b200_pair_device_claim): host ops on this end are refused while it is set.  A host op counts
  // itself in host_ops before it looks at device_owned, the claim sets device_owned before it looks at host_ops,
  // so one of the two always sees the other.
  std::atomic<bool> device_owned{false};
  std::atomic<int> host_ops{0};
  // claimed with B200_CLAIM_UNMIRRORED: the row's mirror (and, loopback wire, the peer row's peer_mirror) is null
  // until the release, so nothing writes this end's PairMirror
  std::atomic<bool> unmirrored{false};
  b200_ready_set* ready_set = nullptr;  // the set this claimed end is a member of (under the runtime lock)
};

struct b200_ready_set {
  ReadyQueue* q = nullptr;  // device memory: control lines, then `size` entries
  uint32_t capacity = 0, size = 0;
  uint32_t members = 0;  // under the runtime lock
  // parking (DESIGN.md §13 "Parking"): pinned, mapped; [0] the doorbell (the ring count the device stores), [1] the
  // result of a host park
  uint64_t* bell = nullptr;
  int wakeup_fd = -1;     // created by the first b200_ready_set_wakeup_fd, which registers the set with the Poller
  uint64_t bell_seen = 0; // the doorbell as the Poller last read it (under the Poller lock)
};

static const char* const kDeviceOwnedRefusal =
    "the pair is device-owned (b200_pair_device_claim): host operations are refused until the release";
// a host op on pair p for as long as it lives (refused: !ok, p->error says why)
struct HostOp {
  b200_pair* p;
  bool ok;
  explicit HostOp(b200_pair* pp) : p(pp) {
    p->host_ops.fetch_add(1);
    ok = !p->device_owned.load();
    if (!ok) p->error = kDeviceOwnedRefusal;
  }
  ~HostOp() { p->host_ops.fetch_sub(1); }
};
static bool any_device_owned(const b200_pair* const* pairs, size_t n, size_t stride_bytes, const char* who) {
  for (size_t i = 0; i < n; i++) {
    const b200_pair* p = *(const b200_pair* const*)((const char*)pairs + i * stride_bytes);
    if (p && p->device_owned.load()) {
      t_err = std::string(who) + ": a pair of the batch is device-owned (b200_pair_device_claim)";
      return true;
    }
  }
  return false;
}

constexpr int kLanes = 16;  // max internal lanes of the host-staged path (B200_LANES, default 8)

struct CopyRun {  // one cudaMemcpyAsync
  void* dst;
  const void* src;
  size_t bytes;
};

struct LanePlan {  // the ops of a lane are contiguous in d_ops
  int first_op = 0, nops = 0;
  std::vector<CopyRun> copies;
};

struct b200_batch {
  int kind = 0;  // 0 send, 1 recv
  int nops = 0;
  int flags = 0;
  void* d_ops = nullptr;       // SendOpDev[] / RecvOpDev[]
  SliceDev* d_slices = nullptr;
  OpResult* d_results = nullptr;
  OpResult* h_results = nullptr;  // pinned
  // host-staged path: slices / destinations are pinned HOST memory; the batch owns a device
  // staging arena and runs as kLanes independent H2D -> kernel (-> D2H) pipelines
  bool staged = false;
  int cluster = 1;  // CTAs per op (B200_BATCH_CLUSTER): >= 2 launches k_cluster_send / k_cluster_recv
  uint8_t* d_stage = nullptr;
  std::vector<int> perm;  // perm[k] = caller's index of device op k
  std::vector<b200_pair*> pairs;  // the pairs of a Recv batch (service: their eager records go stale at launch)
  std::vector<b200_pair*> op_pairs;  // the pair of every op: refused at launch when device-owned, and counted as
                                     // host ops of them from the launch until the results are collected
  bool counted = false;
  std::vector<SendOpDev> h_sops;  // host copies of the descriptors: B200_BATCH_CONCURRENT is added at launch when
  std::vector<RecvOpDev> h_rops;  // a peer has been claimed since the batch was prepared
  LanePlan lanes[kLanes];
};

static void drain_retire(b200_pair* p);

namespace {

struct Runtime {
  std::mutex mu;       // setup + single-call submit
  bool inited = false;
  int dev = -1;
  Config cfg;
  cudaStream_t stream = nullptr;       // single-call + setup stream
  cudaStream_t poll_stream = nullptr;  // readiness scans
  // host-staged lanes: an "up" stream (H2D + Send kernel) and a "down" stream (Recv kernel + D2H)
  // per lane, tied together by events only where the protocol has a real dependency
  cudaStream_t lane_up[kLanes] = {}, lane_down[kLanes] = {};
  cudaEvent_t send_done[kLanes] = {}, recv_done[kLanes] = {};
  cudaEvent_t join_up[kLanes] = {}, join_down[kLanes] = {};
  cudaEvent_t fork_event = nullptr;
  PairDev* d_pairs = nullptr;       // kMaxPairs rows, then the kMaxPairs PairSeq of pair_seq(), then the ReadyNotes
  PairMirror* h_mirrors = nullptr;  // pinned, mapped
  std::vector<b200_pair*> all_pairs;
  std::queue<b200_pair*> pool;
  std::vector<int> free_slots;
  std::unordered_map<std::string, b200_pair*> id_pair;
  std::map<uint32_t, b200_pair*> by_qpn;  // loopback wire registry
  uint32_t next_qpn = 0x200;
  uint32_t cookie = 0;
  bool ipc_wire = false;                 // publish CUDA IPC descriptors (B200_IPC_WIRE / WORLD_SIZE > 1)
  cudaIpcMemHandle_t pairs_handle{};     // d_pairs, exported once
  std::map<uint32_t, PairDev*> peer_tables;  // other processes' connection tables, by cookie
  // single-call staging (pinned, GPU-mapped)
  SendOpDev* h_sop = nullptr;
  RecvOpDev* h_rop = nullptr;
  SliceDev* h_slices = nullptr;  // kMaxSgeLimit + 1 entries
  OpResult* h_res = nullptr;
  std::atomic<uint64_t> launches{0};
  // poller
  std::mutex pmu;
  std::condition_variable pcv;
  std::vector<b200_pair*> pollables;
  std::vector<b200_ready_set*> bell_sets;  // ready sets with a wakeup fd: the Poller reads their doorbells
  std::vector<std::thread> poll_threads;
  std::atomic<bool> poll_running{false};
  // scan scratch (pinned)
  int32_t* h_scan_slots = nullptr;
  uint32_t* h_scan_events = nullptr;
  uint32_t* h_scan_count = nullptr;
  int32_t* h_scan_ready = nullptr;
  std::mutex scan_mu;
  // persistent service (b200_service_*): owner queues in pinned memory, pool mailboxes in HBM
  struct OwnerQ {
    std::mutex mu;          // posting only; nobody waits for an answer under it
    uint64_t next = 0;      // next ticket
  };
  std::atomic<bool> svc_running{false};
  int svc_workers = 0;      // pool CTAs
  int svc_nowners = 0;      // owner warps = command queues
  cudaStream_t svc_stream = nullptr, svc_stream_big = nullptr, svc_stream_poll = nullptr;
  OwnerQ* svc_q = nullptr;
  SvcCmd* svc_cmds = nullptr;          // pinned, mapped  [nowners][kOwnQ]
  SvcDone* svc_done = nullptr;         // pinned, mapped  [nowners][kOwnQ]
  std::atomic<uint32_t>* svc_consumed = nullptr;  // host only [nowners][kOwnQ]: stamp of the last answer its waiter has read
  SliceDev* svc_slices = nullptr;      // pinned, mapped  [nowners][kOwnQ][kSvcSliceArea + 1]
  EagerRec* svc_erec = nullptr;        // pinned, mapped  [kMaxPairs]
  uint8_t* svc_eslots = nullptr;       // pinned, mapped  [kMaxPairs][kEagerMax]
  BigBox* d_svc_boxes = nullptr;
  PairSvc* d_svc_psvc = nullptr;
  ReadyEntry* svc_ready = nullptr;     // pinned, mapped
  uint32_t* svc_host_scans = nullptr;  // pinned, mapped
  SvcPollState* d_svc_ps = nullptr;
  uint32_t* d_svc_last_ev = nullptr;
  uint32_t svc_hi_slot = 0;
  std::atomic<uint64_t> svc_ops{0}, svc_ready_seen{0}, svc_ready_overflows{0}, svc_eager_hits{0};
  // bumped whenever the host changes pair lines on the device or launches kernels beside the service; every
  // command carries it (SvcCmd.op >> 8) and an owner warp that sees a new value drops its cached lines
  std::atomic<uint32_t> svc_gen{1};
  // slots claimed by b200_pair_device_claim: a command for a connection with a claimed end carries
  // B200_BATCH_CONCURRENT, so the owner warp reads that connection's lines fresh and publishes its mirrors under the
  // per-pair locks (a user kernel changes them meanwhile)
  std::atomic<uint8_t> dev_slot[kMaxPairs] = {};
  // ops of launched prepared batches whose results have not been collected, per slot: a command for a connection
  // with such an op carries B200_BATCH_CONCURRENT as well (the batch's kernels change its lines meanwhile)
  std::atomic<uint16_t> batch_slot[kMaxPairs] = {};
  uint32_t svc_ready_head = 0;      // next stream index the host expects (under scan_mu)
  std::vector<uint16_t> svc_level;  // events pending per slot, as last reported by the device poller
  std::mutex grave_mu;
  std::vector<std::pair<void*, int>> graveyard;  // frees deferred while the persistent kernel runs
  // registry of memory this library handed out (skips cudaPointerGetAttributes on the unary path)
  std::mutex reg_mu;
  std::map<uintptr_t, std::pair<size_t, int>> reg_ranges;  // base -> (bytes, 1 = pinned host / 2 = device)
};

Runtime& R() {
  static Runtime r;
  return r;
}

bool ensure_init() {
  if (R().inited) return true;
  return b200_init(-1) == 0;
}

long env_long(const char* k, long dflt) {
  const char* v = getenv(k);
  return v ? atol(v) : dflt;
}

bool is_pow2(uint64_t v) { return v && (v & (v - 1)) == 0; }

bool write_setup(Runtime& r, b200_pair* p, const PairDev& hd) {
  // setup block = first 64 bytes of PairDev
  return CU_OK(cudaMemcpyAsync(&r.d_pairs[p->slot], &hd, 64, cudaMemcpyHostToDevice, r.stream)) &&
         CU_OK(cudaStreamSynchronize(r.stream));
}

// what kind of memory is this? 0 = unregistered host, 1 = pinned / registered host, 2 = device or managed
int reg_kind(const void* p);
int mem_kind3(const void* p) {
  const int k = reg_kind(p);
  if (k) return k;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return 0;
  }
  if (a.type == cudaMemoryTypeUnregistered) return 0;
  return a.type == cudaMemoryTypeHost ? 1 : 2;
}
int mem_kind(const void* p) { return mem_kind3(p) != 0; }  // 0 = unregistered host, 1 = GPU-addressable

void kick(b200_pair* p) {
  if (p->wakeup_fd >= 0) (void)eventfd_write(p->wakeup_fd, 1);
}

// cudaFree / cudaFreeHost synchronise the whole device, which never completes while the
// persistent service kernel is resident: such frees wait in a graveyard until it stops.
void rt_free(void* p, int host) {
  if (!p) return;
  Runtime& r = R();
  if (r.svc_running.load()) {
    std::lock_guard<std::mutex> lk(r.grave_mu);
    r.graveyard.push_back({p, host});
    return;
  }
  if (host) cudaFreeHost(p);
  else cudaFree(p);
}

std::atomic<uint64_t> g_reg_epoch{1};
void reg_add(const void* p, size_t n, int kind) {
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.reg_mu);
  r.reg_ranges[(uintptr_t)p] = {n, kind};
  g_reg_epoch++;
}
void reg_del(const void* p) {
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.reg_mu);
  r.reg_ranges.erase((uintptr_t)p);
  g_reg_epoch++;
}
// nvlink wire bootstrap.  The 48-byte address blob has no room for CUDA IPC handles, so -- like the
// reference's memory-region exchange after the QP is up (pair.cc:472-486,513-526) -- the handles
// travel out of band: every pair publishes a descriptor under /dev/shm keyed by (process cookie,
// qpn), both of which are in the blob.
struct WireDesc {
  uint32_t magic, psn;
  int32_t dev, slot;
  uint64_t cap;
  cudaIpcMemHandle_t ring, pairs;
  int32_t pid, _pad;  // owner process: the survivor's liveness probe (get_status, pair.cc:358-372)
};
constexpr uint32_t kWireMagic = 0xB2001BC0u;
std::string wire_path(uint32_t cookie, uint32_t qpn) {
  char b[96];
  snprintf(b, sizeof b, "/dev/shm/b200wire-%08x-%08x", cookie, qpn);
  return b;
}

// 0 = not in the registry, 1 = pinned host, 2 = device.  The slices of a message usually come from one
// allocation: the last range a thread hit answers without the lock (reg_epoch: any change drops it).
int reg_kind(const void* p) {
  static thread_local uintptr_t c_base = 0, c_end = 0;
  static thread_local int c_kind = 0;
  static thread_local uint64_t c_epoch = 0;
  const uint64_t ep = g_reg_epoch.load(std::memory_order_acquire);
  if (c_epoch == ep && (uintptr_t)p >= c_base && (uintptr_t)p < c_end) return c_kind;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.reg_mu);
  auto it = r.reg_ranges.upper_bound((uintptr_t)p);
  if (it == r.reg_ranges.begin()) return 0;
  --it;
  if ((uintptr_t)p >= it->first + it->second.first) return 0;
  c_base = it->first;
  c_end = it->first + it->second.first;
  c_kind = it->second.second;
  c_epoch = ep;
  return c_kind;
}

}  // namespace

// The calling thread's pinned bounce buffers for unregistered memory of single calls and submit passes (several
// threads post to one queue at the same time, so the staging cannot belong to the queue; a call has finished with
// them when it returns).  Released at b200_shutdown.
struct TlsBounce {
  uint8_t* tx = nullptr;
  uint8_t* rx = nullptr;
  uint64_t tx_cap = 0, rx_cap = 0;
};
static std::mutex g_tls_mu;
static std::vector<TlsBounce*> g_tls_all;
static TlsBounce& tls_bounce() {
  static thread_local TlsBounce* t = nullptr;
  if (!t) {
    t = new TlsBounce();
    std::lock_guard<std::mutex> lk(g_tls_mu);
    g_tls_all.push_back(t);
  }
  return *t;
}

// =================================================================== runtime

static int init_locked(int device);
extern "C" int b200_init(int device) {
  const bool was = R().inited;
  const int rc = init_locked(device);
  // B200_SERVICE_AUTOSTART=<pool CTAs>: bring the resident service kernels up with the runtime, for programs that
  // reach this library through the reference-side shim and never call b200_service_start themselves
  if (rc == 0 && !was) {
    const long n = env_long("B200_SERVICE_AUTOSTART", 0);
    if (n > 0 && b200_service_start((int)n) != 0) return -1;
  }
  return rc;
}
static int init_locked(int device) {
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (r.inited) return 0;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    set_err("b200_init: no CUDA device (this library has no CPU fallback)");
    return -1;
  }
  if (device < 0) {
    const char* e = getenv("B200_DEVICE");
    if (e) device = atoi(e);
    else if (cudaGetDevice(&device) != cudaSuccess) device = 0;
  }
  if (!CU_OK(cudaSetDevice(device))) return -1;
  cudaDeviceProp prop;
  if (!CU_OK(cudaGetDeviceProperties(&prop, device))) return -1;
  if (prop.major != 9 || prop.minor != 0) {  // sm_90a code loads on compute capability 9.0 only
    set_err("b200_init: device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
            ", this library is built for sm_90a only");
    return -1;
  }
  r.dev = device;
  // environment, same keys as the reference (config.cc:45-115)
  r.cfg.ring_bytes = (uint64_t)env_long("GRPC_RDMA_RING_BUFFER_SIZE_KB", 4096) * 1024;
  if (getenv("B200_RING_BUFFER_SIZE_BYTES")) r.cfg.ring_bytes = (uint64_t)env_long("B200_RING_BUFFER_SIZE_BYTES", 0);
  r.cfg.poller_threads = (int)env_long("GRPC_RDMA_POLLER_THREAD_NUM", 1);
  r.cfg.busy_poll_us = (int)env_long("GRPC_RDMA_BUSY_POLLING_TIMEOUT_US", 500);
  r.cfg.poller_sleep_ms = (int)env_long("GRPC_RDMA_POLLER_SLEEP_TIMEOUT_MS", 1000);
  r.cfg.max_sge = (int)env_long("GRPC_RDMA_MAX_SGE", 30);
  if (r.cfg.max_sge < 1 || r.cfg.max_sge > kMaxSgeLimit) r.cfg.max_sge = 30;
  r.cfg.send_coalesce = env_long("B200_SEND_COALESCE", 0) == 1 ? 1 : 0;
  r.cfg.ring_stamped = env_long("B200_RING_STAMPED", 0) == 1 ? 1 : 0;

  if (!CU_OK(cudaStreamCreateWithFlags(&r.stream, cudaStreamNonBlocking))) return -1;
  if (!CU_OK(cudaStreamCreateWithFlags(&r.poll_stream, cudaStreamNonBlocking))) return -1;
  for (int i = 0; i < kLanes; i++) {
    if (!CU_OK(cudaStreamCreateWithFlags(&r.lane_up[i], cudaStreamNonBlocking))) return -1;
    if (!CU_OK(cudaStreamCreateWithFlags(&r.lane_down[i], cudaStreamNonBlocking))) return -1;
    for (cudaEvent_t* e : {&r.send_done[i], &r.recv_done[i], &r.join_up[i], &r.join_down[i]})
      if (!CU_OK(cudaEventCreateWithFlags(e, cudaEventDisableTiming))) return -1;
  }
  if (!CU_OK(cudaEventCreateWithFlags(&r.fork_event, cudaEventDisableTiming))) return -1;
  const size_t table_bytes = (sizeof(PairDev) + sizeof(PairSeq) + sizeof(ReadyNote)) * kMaxPairs;
  if (!CU_OK(cudaMalloc(&r.d_pairs, table_bytes))) return -1;
  if (!CU_OK(cudaMemset(r.d_pairs, 0, table_bytes))) return -1;
  if (!CU_OK(cudaHostAlloc(&r.h_mirrors, sizeof(PairMirror) * kMaxPairs, cudaHostAllocMapped | cudaHostAllocPortable)))
    return -1;
  memset(r.h_mirrors, 0, sizeof(PairMirror) * kMaxPairs);
  auto halloc = [&](void** p, size_t n) {
    return CU_OK(cudaHostAlloc(p, n, cudaHostAllocMapped | cudaHostAllocPortable));
  };
  if (!halloc((void**)&r.h_sop, sizeof(SendOpDev)) || !halloc((void**)&r.h_rop, sizeof(RecvOpDev)) ||
      !halloc((void**)&r.h_slices, sizeof(SliceDev) * (kCoalesceSlices + 1)) ||
      !halloc((void**)&r.h_res, sizeof(OpResult)) ||
      !halloc((void**)&r.h_scan_slots, sizeof(int32_t) * kMaxPairs) ||
      !halloc((void**)&r.h_scan_events, sizeof(uint32_t) * kMaxPairs) ||
      !halloc((void**)&r.h_scan_count, sizeof(uint32_t) * 4) ||
      !halloc((void**)&r.h_scan_ready, sizeof(int32_t) * kMaxPairs))
    return -1;
  r.ipc_wire = getenv("B200_IPC_WIRE") ? env_long("B200_IPC_WIRE", 0) != 0 : env_long("WORLD_SIZE", 1) > 1;
  if (r.ipc_wire && !CU_OK(cudaIpcGetMemHandle(&r.pairs_handle, r.d_pairs))) return -1;
  r.free_slots.clear();
  for (int i = kMaxPairs - 1; i >= 0; i--) r.free_slots.push_back(i);
  r.cookie = (uint32_t)getpid() * 2654435761u ^ (uint32_t)(uintptr_t)&r;
  static bool at_exit_registered = false;
  if (!at_exit_registered) {
    at_exit_registered = true;
    atexit([] {  // poller threads joined and the persistent kernel gone before static destruction
      b200_poller_shutdown();
      b200_service_stop();
      for (b200_pair* p : R().all_pairs)  // wire descriptors of pairs nobody disconnected
        if (!p->wire_file.empty()) unlink(p->wire_file.c_str());
    });
  }
  r.inited = true;
  return 0;
}

extern "C" void b200_shutdown(void) {
  b200_poller_shutdown();
  b200_service_stop();
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (!r.inited) return;
  cudaSetDevice(r.dev);
  cudaDeviceSynchronize();
  for (b200_pair* p : r.all_pairs) {
    if (p->ring) cudaFree(p->ring);
    if (p->wakeup_fd >= 0) close(p->wakeup_fd);
    delete p;
  }
  r.all_pairs.clear();
  while (!r.pool.empty()) r.pool.pop();
  r.id_pair.clear();
  r.by_qpn.clear();
  cudaFree(r.d_pairs);
  cudaFreeHost(r.h_mirrors);
  cudaFreeHost(r.h_sop);
  cudaFreeHost(r.h_rop);
  cudaFreeHost(r.h_slices);
  cudaFreeHost(r.h_res);
  cudaFreeHost(r.h_scan_slots);
  cudaFreeHost(r.h_scan_events);
  cudaFreeHost(r.h_scan_count);
  cudaFreeHost(r.h_scan_ready);
  {
    std::lock_guard<std::mutex> tl(g_tls_mu);
    for (TlsBounce* t : g_tls_all) {
      if (t->tx) cudaFreeHost(t->tx);
      if (t->rx) cudaFreeHost(t->rx);
      t->tx = t->rx = nullptr;
      t->tx_cap = t->rx_cap = 0;
    }
  }
  cudaStreamDestroy(r.stream);
  cudaStreamDestroy(r.poll_stream);
  for (int i = 0; i < kLanes; i++) {
    cudaStreamDestroy(r.lane_up[i]);
    cudaStreamDestroy(r.lane_down[i]);
    for (cudaEvent_t e : {r.send_done[i], r.recv_done[i], r.join_up[i], r.join_down[i]}) cudaEventDestroy(e);
  }
  cudaEventDestroy(r.fork_event);
  r.inited = false;
}

extern "C" int b200_device(void) { return R().dev; }
extern "C" const char* b200_last_error(void) { return t_err.c_str(); }
extern "C" uint64_t b200_launch_count(void) { return R().launches.load(); }

extern "C" int b200_config_set(const char* key, const char* value) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  std::string k(key);
  long v = atol(value);
  if (k == "GRPC_RDMA_RING_BUFFER_SIZE_KB") {
    if (v <= 0) return -1;
    r.cfg.ring_bytes = (uint64_t)v * 1024;
  } else if (k == "B200_RING_BUFFER_SIZE_BYTES") {
    if (v <= (long)kReserved) return -1;
    r.cfg.ring_bytes = (uint64_t)v;
  } else if (k == "GRPC_RDMA_POLLER_THREAD_NUM") {
    if (v <= 0) return -1;
    r.cfg.poller_threads = (int)v;
  } else if (k == "GRPC_RDMA_BUSY_POLLING_TIMEOUT_US") {
    if (v < 0) return -1;
    r.cfg.busy_poll_us = (int)v;
  } else if (k == "GRPC_RDMA_POLLER_SLEEP_TIMEOUT_MS") {
    if (v < 0) return -1;
    r.cfg.poller_sleep_ms = (int)v;
  } else if (k == "GRPC_RDMA_MAX_SGE") {
    if (v < 1 || v > kMaxSgeLimit) return -1;
    r.cfg.max_sge = (int)v;
  } else if (k == "B200_SEND_COALESCE") {
    if (v != 0 && v != 1) return -1;
    r.cfg.send_coalesce = (int)v;
  } else if (k == "B200_RING_STAMPED") {
    if (v != 0 && v != 1) return -1;
    r.cfg.ring_stamped = (int)v;
  } else {
    set_err("b200_config_set: unknown key " + k);
    return -1;
  }
  return 0;
}

extern "C" int64_t b200_config_get(const char* key) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  std::string k(key);
  if (k == "GRPC_RDMA_RING_BUFFER_SIZE_KB") return (int64_t)(r.cfg.ring_bytes / 1024);
  if (k == "B200_RING_BUFFER_SIZE_BYTES") return (int64_t)r.cfg.ring_bytes;
  if (k == "GRPC_RDMA_POLLER_THREAD_NUM") return r.cfg.poller_threads;
  if (k == "GRPC_RDMA_BUSY_POLLING_TIMEOUT_US") return r.cfg.busy_poll_us;
  if (k == "GRPC_RDMA_POLLER_SLEEP_TIMEOUT_MS") return r.cfg.poller_sleep_ms;
  if (k == "GRPC_RDMA_MAX_SGE") return r.cfg.max_sge;
  if (k == "B200_SEND_COALESCE") return r.cfg.send_coalesce;
  if (k == "B200_RING_STAMPED") return r.cfg.ring_stamped;
  return -1;
}

// ==================================================================== memory

extern "C" void* b200_mem_alloc_device(size_t bytes) {
  if (!ensure_init()) return nullptr;
  void* p = nullptr;
  cudaSetDevice(R().dev);
  if (!CU_OK(cudaMalloc(&p, bytes ? bytes : 1))) return nullptr;
  reg_add(p, bytes ? bytes : 1, 2);
  return p;
}
extern "C" void b200_mem_free_device(void* p) {
  if (!p) return;
  reg_del(p);
  rt_free(p, 0);
}
extern "C" void* b200_mem_alloc_host(size_t bytes) {
  if (!ensure_init()) return nullptr;
  void* p = nullptr;
  cudaSetDevice(R().dev);
  if (!CU_OK(cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocMapped | cudaHostAllocPortable))) return nullptr;
  reg_add(p, bytes ? bytes : 1, 1);
  return p;
}
extern "C" void b200_mem_free_host(void* p) {
  if (!p) return;
  reg_del(p);
  rt_free(p, 1);
}
extern "C" int b200_mem_register_host(void* p, size_t bytes) {
  if (!ensure_init()) return -1;
  if (!CU_OK(cudaHostRegister(p, bytes, cudaHostRegisterMapped | cudaHostRegisterPortable))) return -1;
  reg_add(p, bytes, 1);
  return 0;
}
extern "C" int b200_mem_unregister_host(void* p) {
  reg_del(p);
  return CU_OK(cudaHostUnregister(p)) ? 0 : -1;
}
extern "C" int b200_memcpy(void* dst, const void* src, size_t bytes, int dir, void* stream) {
  if (!ensure_init()) return -1;
  cudaMemcpyKind k = dir == 0 ? cudaMemcpyHostToDevice : dir == 1 ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
  cudaStream_t s = stream ? (cudaStream_t)stream : R().stream;
  return CU_OK(cudaMemcpyAsync(dst, src, bytes, k, s)) ? 0 : -1;
}
extern "C" int b200_stream_sync(void* stream) {
  if (!ensure_init()) return -1;
  cudaStream_t s = stream ? (cudaStream_t)stream : R().stream;
  return CU_OK(cudaStreamSynchronize(s)) ? 0 : -1;
}

// ================================================================ pool / pair

static void device_release_locked(Runtime& r, b200_pair* p);
static void close_host_side(Runtime& r, b200_pair* p);

extern "C" b200_pair* b200_pool_take(const char* id) {
  if (!ensure_init()) return nullptr;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  b200_pair* p = nullptr;
  if (!r.pool.empty()) {
    p = r.pool.front();
    r.pool.pop();
  } else {
    if (r.free_slots.empty()) {
      set_err("b200_pool_take: connection table full");
      return nullptr;
    }
    p = new b200_pair();
    p->slot = r.free_slots.back();
    r.free_slots.pop_back();
    p->mirror = &r.h_mirrors[p->slot];
    p->wakeup_fd = eventfd(0, EFD_NONBLOCK | EFD_CLOEXEC);  // grpc_wakeup_fd_init, pair.cc:74
    r.all_pairs.push_back(p);
  }
  p->id = id ? id : "";
  if (!p->id.empty()) r.id_pair[p->id] = p;
  return p;
}

extern "C" void b200_pool_putback(b200_pair* p) {
  if (!p) return;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  device_release_locked(r, p);
  auto it = r.id_pair.find(p->id);
  if (it != r.id_pair.end() && it->second == p) r.id_pair.erase(it);
  r.pool.push(p);
}

extern "C" b200_pair* b200_pool_get(const char* id) {
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  auto it = r.id_pair.find(id ? id : "");
  return it == r.id_pair.end() ? nullptr : it->second;
}

// the pair's max_sge word of PairDev: the modes ride in its top bits so the line stays 128 bytes
static uint32_t sge_word(const b200_pair* p) {
  return (uint32_t)p->max_sge | (p->coalesce ? kSgeCoalesce : 0u) | (p->stamped ? kSgeStamped : 0u);
}

extern "C" void b200_pair_init(b200_pair* p) {
  if (!p || !ensure_init()) return;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  device_release_locked(r, p);
  // pair.cc:88-89: only from Uninitialized / Error / Disconnected
  if (!(p->status == B200_UNINITIALIZED || p->status == B200_ERROR || p->status == B200_DISCONNECTED)) return;
  cudaSetDevice(r.dev);
  const uint64_t cap = r.cfg.ring_bytes;
  if (!is_pow2(cap) || cap <= kReserved) {  // ring_buffer.cc:22-23
    p->error = "ring buffer size must be a power of two > 24";
    set_err(p->error);
    p->status = B200_ERROR;
    return;
  }
  if (p->ring && p->cap != cap) {
    rt_free(p->ring, 0);
    p->ring = nullptr;
  }
  if (!p->ring) {
    if (!CU_OK(cudaMalloc(&p->ring, cap))) {
      p->error = t_err;
      p->status = B200_ERROR;
      return;
    }
  }
  p->cap = cap;
  PairDev hd;
  memset(&hd, 0, sizeof(hd));
  hd.ring = p->ring;
  hd.cap = cap;
  hd.mirror = p->mirror;
  hd.status = B200_INITIALIZED;
  p->max_sge = r.cfg.max_sge;
  p->coalesce = r.cfg.send_coalesce != 0;
  p->stamp_offer = r.cfg.ring_stamped != 0 && cap <= kStampedMaxCap;
  p->stamped = false;
  hd.max_sge = sge_word(p);
  hd.peer_slot = -1;
  p->svc_delivered = 0;
  p->retire_pending = false;
  p->peer_dead = false;
  p->peer_pid = 0;
  memset(p->mirror, 0, sizeof(PairMirror));
  bool ok = CU_OK(cudaMemsetAsync(p->ring, 0, cap, r.stream)) &&  // RingBufferPollable::Init
            CU_OK(cudaMemcpyAsync(&r.d_pairs[p->slot], &hd, sizeof(hd), cudaMemcpyHostToDevice, r.stream)) &&
            CU_OK(cudaMemsetAsync(pair_seq(r.d_pairs, p->slot), 0, sizeof(PairSeq), r.stream)) &&
            CU_OK(cudaStreamSynchronize(r.stream));
  if (!ok) {
    p->error = t_err;
    p->status = B200_ERROR;
    return;
  }
  if (r.svc_running.load()) {
    const PairSvc fresh{0, ~0ull};
    memset((void*)&r.svc_erec[p->slot], 0, sizeof(EagerRec));
    cudaMemcpyAsync(&r.d_svc_psvc[p->slot], &fresh, sizeof(fresh), cudaMemcpyHostToDevice, r.stream);
    if ((uint32_t)p->slot + 1 > r.svc_hi_slot) {
      r.svc_hi_slot = (uint32_t)p->slot + 1;
      cudaMemcpyAsync(&r.d_svc_ps->hi_slot, &r.svc_hi_slot, 4, cudaMemcpyHostToDevice, r.stream);
    }
    cudaStreamSynchronize(r.stream);
    r.svc_gen++;
  }
  // drop a stale registration, then publish the new address
  if (p->self.qpn) r.by_qpn.erase(p->self.qpn);
  memset(&p->self, 0, sizeof(p->self));
  p->self.lid = 0xB200;
  p->self.qpn = r.next_qpn++;
  p->self.psn = (uint32_t)rand() & 0xffffff;
  memcpy(p->self.gid, &r.cookie, 4);           // which process
  memcpy(p->self.gid + 4, &r.dev, 4);          // which GPU
  memcpy(p->self.gid + 8, &p->slot, 4);        // which row of the connection table
  p->self.tag = B200_PAIR_TAG_POLLABLE;
  p->self._pad1 = p->stamp_offer ? kBlobStamped : 0u;
  p->self.ring_buffer_size = cap;  // "used to check peer has the same size", pair.cc:107
  r.by_qpn[p->self.qpn] = p;
  p->peer_local = nullptr;
  p->remote = false;
  if (r.ipc_wire) {
    WireDesc d{};
    d.magic = kWireMagic;
    d.psn = p->self.psn;
    d.dev = r.dev;
    d.slot = p->slot;
    d.cap = cap;
    d.pid = (int32_t)getpid();
    d.pairs = r.pairs_handle;
    if (CU_OK(cudaIpcGetMemHandle(&d.ring, p->ring))) {
      p->wire_file = wire_path(r.cookie, p->self.qpn);
      const std::string tmp = p->wire_file + ".tmp";
      int fd = open(tmp.c_str(), O_CREAT | O_TRUNC | O_WRONLY, 0600);
      if (fd >= 0) {
        const bool okw = write(fd, &d, sizeof d) == (ssize_t)sizeof d;
        close(fd);
        if (okw) rename(tmp.c_str(), p->wire_file.c_str());
      }
    }
  }
  p->error.clear();
  eventfd_t junk;
  (void)eventfd_read(p->wakeup_fd, &junk);
  p->status = B200_INITIALIZED;
}

extern "C" size_t b200_pair_self_address(b200_pair* p, void* out48) {
  if (!p || !out48) return 0;
  memcpy(out48, &p->self, sizeof(AddrBlob));
  return sizeof(AddrBlob);
}

extern "C" int b200_pair_connect(b200_pair* p, const void* peer48, size_t n) {
  if (!p || !ensure_init()) return 0;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (p->status != B200_INITIALIZED) return 0;  // pair.cc:144
  if (n != sizeof(AddrBlob)) {                  // address.cc:13 asserts
    p->error = "peer address blob has the wrong size";
    set_err(p->error);
    return 0;
  }
  memcpy(&p->peer, peer48, sizeof(AddrBlob));
  if (p->peer.tag != p->self.tag) {  // pair.cc:148 (GPR_ASSERT there)
    p->error = "peer pair tag mismatch";
    set_err(p->error);
    return 0;
  }
  if (p->peer.ring_buffer_size != p->self.ring_buffer_size) {  // pair.cc:149
    p->error = "peer ring buffer size mismatch";
    set_err(p->error);
    return 0;
  }
  // stamped frames when both ends offer them: both compute the same AND, and a peer without the bit (any
  // blob written before the bit existed) gets the reference format.  Set right before the setup line is written.
  const bool stamped = p->stamp_offer && (p->peer._pad1 & kBlobStamped) != 0;
  uint32_t cookie;
  memcpy(&cookie, p->peer.gid, 4);
  if (cookie != r.cookie) {
    // ---- nvlink wire: the peer is another process on this box (one process per GPU)
    WireDesc d{};
    const std::string path = wire_path(cookie, p->peer.qpn);
    int fd = open(path.c_str(), O_RDONLY);
    const bool got = fd >= 0 && read(fd, &d, sizeof d) == (ssize_t)sizeof d;
    if (fd >= 0) close(fd);
    if (!got || d.magic != kWireMagic || d.psn != p->peer.psn || d.cap != p->cap) {
      p->error = "peer is not reachable: no wire descriptor " + path +
                 " (wires built: in-process loopback, CUDA-IPC/NVLink within one box; no NIC wire)";
      set_err(p->error);
      return 0;
    }
    cudaSetDevice(r.dev);
    void* rring = nullptr;
    if (!CU_OK(cudaIpcOpenMemHandle(&rring, d.ring, cudaIpcMemLazyEnablePeerAccess))) {
      p->error = t_err;
      return 0;
    }
    PairDev* table = nullptr;
    auto pt = r.peer_tables.find(cookie);
    if (pt != r.peer_tables.end()) {
      table = pt->second;
    } else {
      void* tp = nullptr;
      if (!CU_OK(cudaIpcOpenMemHandle(&tp, d.pairs, cudaIpcMemLazyEnablePeerAccess))) {
        p->error = t_err;
        cudaIpcCloseMemHandle(rring);
        return 0;
      }
      table = (PairDev*)tp;
      r.peer_tables[cookie] = table;
    }
    PairDev hd;
    memset(&hd, 0, sizeof(hd));
    hd.ring = p->ring;
    hd.cap = p->cap;
    hd.peer_ring = (uint8_t*)rring;
    hd.peer_credit = &table[d.slot].credit_head;
    hd.mirror = p->mirror;
    hd.peer_mirror = nullptr;
    hd.status = B200_CONNECTED;
    p->stamped = stamped;
    hd.max_sge = sge_word(p);
    hd.peer_slot = -1;
    hd.wire = 1;  // system-scope fences: the ring is in another GPU's HBM, reached over NVLink
    if (!write_setup(r, p, hd)) {
      p->error = t_err;
      p->status = B200_ERROR;
      return 0;
    }
    p->remote = true;
    p->peer_pid = d.pid;
    p->remote_ring = (uint8_t*)rring;
    p->remote_credit = hd.peer_credit;
    p->peer_local = nullptr;
    p->status = B200_CONNECTED;
    r.svc_gen++;
    return 1;
  }
  auto it = r.by_qpn.find(p->peer.qpn);
  if (it == r.by_qpn.end() || it->second->self.psn != p->peer.psn) {
    p->error = "peer is not reachable: unknown qpn on the in-process loopback wire";
    set_err(p->error);
    return 0;
  }
  b200_pair* q = it->second;
  if (!q->ring) {
    p->error = "peer ring not allocated";
    set_err(p->error);
    return 0;
  }
  cudaSetDevice(r.dev);
  PairDev hd;
  memset(&hd, 0, sizeof(hd));
  hd.ring = p->ring;
  hd.cap = p->cap;
  hd.peer_ring = q->ring;
  hd.peer_credit = &r.d_pairs[q->slot].credit_head;
  hd.mirror = p->mirror;
  hd.peer_mirror = q->mirror;
  hd.status = B200_CONNECTED;
  p->stamped = stamped;
  hd.max_sge = sge_word(p);
  hd.peer_slot = q->slot;
  hd.wire = 0;
  if (!write_setup(r, p, hd)) {
    p->error = t_err;
    p->status = B200_ERROR;
    return 0;
  }
  p->peer_local = q;
  p->status = B200_CONNECTED;
  r.svc_gen++;
  return 1;
}

extern "C" void b200_pair_disconnect(b200_pair* p) {
  if (!p || !R().inited) return;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  device_release_locked(r, p);
  if (p->status == B200_UNINITIALIZED || p->status == B200_DISCONNECTED) return;  // pair.cc:326-327
  drain_retire(p);
  cudaSetDevice(r.dev);
  const bool was_connected = p->status == B200_CONNECTED && p->mirror->peer_exit == 0;
  if (was_connected && p->peer_local) {
    // peer_exit = 1 + current head, one 16-byte status write (pair.cc:330-337)
    cudaStreamSynchronize(r.stream);
    struct {
      uint64_t remote_head;
      uint32_t peer_exit, pad;
    } st = {p->mirror->moving_head, 1, 0};
    b200_pair* q = p->peer_local;
    cudaMemcpyAsync(&r.d_pairs[q->slot].credit_head, &st, 16, cudaMemcpyHostToDevice, r.stream);
    cudaStreamSynchronize(r.stream);
    if (!q->unmirrored.load()) {  // (an unmirrored end's release publishes it from the credit block)
      q->mirror->credit_head = st.remote_head;
      q->mirror->peer_exit = 1;
    }
    if (q->ready_set) {  // the peer's readiness changed: its ready set hears of it
      launch_ready_notify(r.d_pairs, q->slot, r.stream);
      r.launches++;
      cudaStreamSynchronize(r.stream);
    }
  }
  if (p->remote && was_connected) {  // the same 16-byte status write, over NVLink into the peer's table
    cudaStreamSynchronize(r.stream);
    struct {
      uint64_t remote_head;
      uint32_t peer_exit, pad;
    } st = {p->mirror->moving_head, 1, 0};
    cudaMemcpyAsync(p->remote_credit, &st, 16, cudaMemcpyDefault, r.stream);
    cudaStreamSynchronize(r.stream);
  }
  uint32_t st = B200_DISCONNECTED;
  cudaMemcpyAsync(&r.d_pairs[p->slot].status, &st, 4, cudaMemcpyHostToDevice, r.stream);
  cudaStreamSynchronize(r.stream);
  close_host_side(r, p);
}

// The host half of Disconnect, once the peer has been told and the row says DISCONNECTED (b200_pair_disconnect, or
// b200_warp_disconnect on a device-owned end, whose release calls this): the wire mapping, the wire descriptor and
// the address go.  Caller holds r.mu.
static void close_host_side(Runtime& r, b200_pair* p) {
  if (p->remote) {
    if (!r.svc_running.load()) cudaIpcCloseMemHandle(p->remote_ring);  // (device-wide sync: skipped beside the service)
    p->remote = false;
    p->remote_ring = nullptr;
    p->remote_credit = nullptr;
  }
  if (!p->wire_file.empty()) {
    unlink(p->wire_file.c_str());
    p->wire_file.clear();
  }
  if (p->self.qpn) r.by_qpn.erase(p->self.qpn);
  p->self.qpn = 0;
  p->peer_local = nullptr;
  p->status = B200_DISCONNECTED;
  r.svc_gen++;
}

// On the nvlink wire the bytes, the credit and the peer_exit flag are written by another GPU, so
// nothing on this side knows when the mirror went stale: the wait-free answer comes from the
// service kernel's poller when it runs, from a one-pair scan otherwise.
static void refresh_remote(const b200_pair* cp) {
  b200_pair* p = const_cast<b200_pair*>(cp);
  if (!p->remote || p->status != B200_CONNECTED || R().svc_running.load()) return;
  b200_pair* one[1] = {p};
  b200_poller_scan(one, 1, nullptr);
}

extern "C" enum b200_status b200_pair_status(b200_pair* p) {
  if (!p) return B200_UNINITIALIZED;
  // a device-owned end that b200_warp_disconnect closed (the release finishes the Disconnect on the host)
  if (p->device_owned.load() && ((volatile PairMirror*)p->mirror)->dev_closed) return B200_DISCONNECTED;
  if (p->remote && p->status == B200_CONNECTED && p->peer_pid > 0) {
    // the liveness leg of get_status (pair.cc:358-372: ibv_query_qp every 500 ms, anything but RTS -> HalfClosed).
    // On the CUDA-IPC wire there is no QP to ask: the owner process of the peer pair is probed instead -- a peer
    // that died without Disconnect (no peer_exit write) leaves nobody to answer, and the survivor must not stay
    // Connected forever.
    const auto now = std::chrono::steady_clock::now();
    if (now - p->last_probe > std::chrono::milliseconds(500)) {
      p->last_probe = now;
      if (kill((pid_t)p->peer_pid, 0) != 0 && errno == ESRCH) p->peer_dead = true;
    }
  }
  if (p->peer_dead.load() && p->status == B200_CONNECTED) return B200_HALF_CLOSED;
  refresh_remote(p);
  if (p->status == B200_CONNECTED && ((volatile PairMirror*)p->mirror)->peer_exit == 1)
    return B200_HALF_CLOSED;  // pair.cc:354-356
  return (enum b200_status)p->status;
}
extern "C" const char* b200_pair_error(const b200_pair* p) { return p ? p->error.c_str() : ""; }
extern "C" int b200_pair_stamped(const b200_pair* p) {
  return p && p->stamped && (p->status == B200_CONNECTED || p->status == B200_HALF_CLOSED) ? 1 : 0;
}
extern "C" int b200_pair_wakeup_read_fd(b200_pair* p) { return p ? p->wakeup_fd : -1; }
extern "C" void b200_pair_consume_wakeup(b200_pair* p) {
  if (!p) return;
  eventfd_t v;
  (void)eventfd_read(p->wakeup_fd, &v);
}
extern "C" int b200_pair_has_message(const b200_pair* p) {
  if (!p) return 0;
  drain_retire(const_cast<b200_pair*>(p));
  refresh_remote(p);
  return ((volatile PairMirror*)p->mirror)->has_message != 0;
}
extern "C" int b200_pair_has_pending_writes(const b200_pair* p) {
  return p && ((volatile PairMirror*)p->mirror)->partial_write != 0;
}
extern "C" uint64_t b200_pair_readable(const b200_pair* p) {
  if (!p || p->status != B200_CONNECTED) return 0;  // pair.cc:290-292
  drain_retire(const_cast<b200_pair*>(p));
  refresh_remote(p);
  return ((volatile PairMirror*)p->mirror)->readable;
}
extern "C" uint64_t b200_pair_writable(const b200_pair* p) {
  if (!p || !p->cap) return 0;
  if (p->peer_local) drain_retire(p->peer_local);  // a Retire of the peer may return credit
  refresh_remote(p);
  volatile PairMirror* m = p->mirror;
  return writable_size(p->cap, m->credit_head, m->remote_tail);  // pair.cc:294-301
}

extern "C" int b200_pair_get_state(b200_pair* p, b200_pair_state* out) {
  if (!p || !out || !ensure_init()) return -1;
  Runtime& r = R();
  drain_retire(p);
  if (p->peer_local) drain_retire(p->peer_local);
  std::lock_guard<std::mutex> lk(r.mu);
  cudaSetDevice(r.dev);
  PairDev hd;
  if (!CU_OK(cudaMemcpy(&hd, &r.d_pairs[p->slot], sizeof(hd), cudaMemcpyDeviceToHost))) return -1;
  out->head = hd.head;
  out->moving_head = hd.moving_head;
  out->remain = hd.remain;
  out->remote_tail = hd.remote_tail;
  out->internal_read_size = hd.acc;
  out->credit_remote_head = hd.credit_head;
  out->partial_write = hd.partial_write;
  out->peer_exit = hd.credit_exit;
  out->ring_capacity = hd.cap;
  return 0;
}

extern "C" int b200_pair_copy_ring(b200_pair* p, void* host_dst, uint64_t cap) {
  if (!p || !p->ring || cap < p->cap) return -1;
  drain_retire(p);
  cudaSetDevice(R().dev);
  return CU_OK(cudaMemcpy(host_dst, p->ring, p->cap, cudaMemcpyDeviceToHost)) ? 0 : -1;
}

static void refresh_remote(const b200_pair* cp);

// ================================================================== service
//
// The persistent kernel of the unary path: worker CTAs take Send / Recv commands from pinned
// mapped memory (no launch, no stream synchronisation per call) and a poller CTA keeps the
// mirrors and the ready ring current (no scan launches).  While it runs, b200_pair_send / recv
// are routed through it; the batch entry points keep launching their own kernels beside it.

static bool ensure_bounce(uint8_t** buf, uint64_t* cap, uint64_t need);

static int owner_of(const Runtime& r, const b200_pair* p) {
  uint32_t key = (uint32_t)p->slot;
  if (p->peer_local && (uint32_t)p->peer_local->slot < key) key = (uint32_t)p->peer_local->slot;  // both ends: one owner
  return (int)(((key * 2654435761u) >> 12) % (uint32_t)r.svc_nowners);
}

extern "C" int b200_service_start(int workers) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (r.svc_running.load()) return 0;
  if (workers <= 0) workers = (int)env_long("B200_SERVICE_WORKERS", 16);
  if (workers > 256) workers = 256;
  int owners = (int)env_long("B200_SERVICE_OWNERS", 32);
  if (owners < 1) owners = 1;
  if (owners > 256) owners = 256;
  cudaSetDevice(r.dev);
  auto halloc = [&](void** p, size_t n) {
    if (!CU_OK(cudaHostAlloc(p, n, cudaHostAllocMapped | cudaHostAllocPortable))) return false;
    memset(*p, 0, n);
    return true;
  };
  for (cudaStream_t* st : {&r.svc_stream, &r.svc_stream_big, &r.svc_stream_poll})
    if (!*st && !CU_OK(cudaStreamCreateWithFlags(st, cudaStreamNonBlocking))) return -1;
  const size_t nent = (size_t)owners * kOwnQ;
  if (!halloc((void**)&r.svc_cmds, sizeof(SvcCmd) * nent) || !halloc((void**)&r.svc_done, sizeof(SvcDone) * nent) ||
      !halloc((void**)&r.svc_slices, sizeof(SliceDev) * nent * (kSvcSliceArea + 1)) ||
      !halloc((void**)&r.svc_erec, sizeof(EagerRec) * kMaxPairs) ||
      !halloc((void**)&r.svc_eslots, (size_t)kEagerMax * kMaxPairs) ||
      !halloc((void**)&r.svc_ready, sizeof(ReadyEntry) * kReadyRing) || !halloc((void**)&r.svc_host_scans, 64))
    return -1;
  if (!CU_OK(cudaMalloc(&r.d_svc_ps, sizeof(SvcPollState))) || !CU_OK(cudaMalloc(&r.d_svc_last_ev, 4 * kMaxPairs)) ||
      !CU_OK(cudaMalloc(&r.d_svc_boxes, sizeof(BigBox) * owners * kOwnBoxes)) ||
      !CU_OK(cudaMalloc(&r.d_svc_psvc, sizeof(PairSvc) * kMaxPairs)))
    return -1;
  r.svc_hi_slot = 0;
  for (b200_pair* p : r.all_pairs) {
    if ((uint32_t)p->slot + 1 > r.svc_hi_slot) r.svc_hi_slot = (uint32_t)p->slot + 1;
    p->svc_delivered = 0;
    p->retire_pending = false;
  }
  SvcPollState ps{};
  ps.hi_slot = r.svc_hi_slot;
  std::vector<PairSvc> psvc(kMaxPairs, PairSvc{0, ~0ull});
  if (!CU_OK(cudaMemcpyAsync(r.d_svc_ps, &ps, sizeof(ps), cudaMemcpyHostToDevice, r.stream)) ||
      !CU_OK(cudaMemsetAsync(r.d_svc_last_ev, 0, 4 * kMaxPairs, r.stream)) ||
      !CU_OK(cudaMemsetAsync(r.d_svc_boxes, 0, sizeof(BigBox) * owners * kOwnBoxes, r.stream)) ||
      !CU_OK(cudaMemcpyAsync(r.d_svc_psvc, psvc.data(), sizeof(PairSvc) * kMaxPairs, cudaMemcpyHostToDevice, r.stream)) ||
      !CU_OK(cudaStreamSynchronize(r.stream)))
    return -1;
  r.svc_q = new Runtime::OwnerQ[owners];
  r.svc_consumed = new std::atomic<uint32_t>[nent];
  for (size_t i = 0; i < nent; i++) r.svc_consumed[i].store(0);
  r.svc_workers = workers;
  r.svc_nowners = owners;
  r.svc_ready_head = 0;
  r.svc_level.assign(kMaxPairs, 0);
  SvcParams sp{};
  sp.pairs = r.d_pairs;
  sp.psvc = r.d_svc_psvc;
  sp.cmds = r.svc_cmds;
  sp.done = r.svc_done;
  sp.boxes = r.d_svc_boxes;
  sp.erec = env_long("B200_SERVICE_EAGER", 1) ? r.svc_erec : nullptr;
  sp.eslots = r.svc_eslots;
  sp.ps = r.d_svc_ps;
  sp.last_ev = r.d_svc_last_ev;
  sp.ready = r.svc_ready;
  sp.host_scans = r.svc_host_scans;
  sp.nowners = owners;
  sp.nbig = workers;
  if (!launch_service(sp, r.svc_stream, r.svc_stream_big, r.svc_stream_poll)) {
    set_err("b200_service_start: the resident kernels (" + std::to_string(workers) +
            " pool CTAs + owners + poller) do not fit on the device together");
    cudaGetLastError();
    return -1;
  }
  r.launches += 3;
  r.svc_running = true;
  return 0;
}

extern "C" int b200_service_running(void) { return R().svc_running.load() ? R().svc_workers : 0; }

// ---- owner queues: post = claim the next ticket of the queue and fill its entry; the answer lands in the
// entry's SvcDone.  An entry is reused every kOwnQ tickets, once the answer of its previous ticket was seen.
// An entry is reused every kOwnQ tickets -- once the answer of its previous ticket has been CONSUMED by the
// thread that waits for it (svc_consumed), not merely written by the GPU: a thread that posts many commands
// before it waits (b200_pairs_submit) would otherwise have its early answers overwritten by its later ones.
template <class Fill>
static bool svc_try_post(Runtime& r, int q, Fill fill, uint64_t* ticket) {
  Runtime::OwnerQ& Q = r.svc_q[q];
  std::lock_guard<std::mutex> lk(Q.mu);
  const uint64_t t = Q.next;
  const size_t e = (size_t)q * kOwnQ + t % kOwnQ;
  if (t >= kOwnQ && r.svc_consumed[e].load(std::memory_order_acquire) != (uint32_t)(t - kOwnQ + 1)) return false;
  Q.next = t + 1;
  SvcCmd* c = &r.svc_cmds[e];
  c->nreal = 0;
  fill(c, r.svc_slices + e * (kSvcSliceArea + 1));
  const int s0 = c->slot & 0xffff, s1 = (c->slot >> 16) - 1;
  if ((s0 < kMaxPairs && (r.dev_slot[s0].load() || r.batch_slot[s0].load())) ||
      (s1 >= 0 && s1 < kMaxPairs && (r.dev_slot[s1].load() || r.batch_slot[s1].load())))
    c->flags |= B200_BATCH_CONCURRENT;
  c->op = (c->op & 0xffu) | ((r.svc_gen.load(std::memory_order_acquire) & 0xffffffu) << 8);
  std::atomic_thread_fence(std::memory_order_release);
  *(volatile uint32_t*)&c->stamp2 = (uint32_t)(t + 1);
  *(volatile uint32_t*)&c->stamp = (uint32_t)(t + 1);
  *ticket = t;
  return true;
}
// blocking form: only for callers that hold no unconsumed answers themselves (they wait right after posting)
template <class Fill>
static uint64_t svc_post(Runtime& r, int q, Fill fill) {
  uint64_t t = 0;
  while (!svc_try_post(r, q, fill, &t)) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
  return t;
}

static bool svc_wait(Runtime& r, int q, uint64_t t, uint64_t* bytes, uint64_t* calls) {
  const size_t e = (size_t)q * kOwnQ + t % kOwnQ;
  volatile SvcDone* d = &r.svc_done[e];
  const uint32_t want = (uint32_t)(t + 1);
  uint32_t spins = 0;
  std::chrono::steady_clock::time_point t0;
  while (d->seq != want) {
    // already reused: somebody else waited for this ticket too and consumed it (a Retire: no result to read)
    if ((int32_t)(d->seq - want) > 0) return true;
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
    if ((++spins & 0xfffff) == 0) {
      if (spins == 0x100000) t0 = std::chrono::steady_clock::now();
      else if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(30)) {
        set_err("b200 service: command timed out");
        return false;
      }
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  if (bytes) *bytes = d->bytes;
  if (calls) *calls = d->calls;
  r.svc_consumed[e].store(want, std::memory_order_release);  // the entry may be reused now
  r.svc_ops++;
  return true;
}

// the asynchronous Retire of the last eagerly received frame must have run before anything looks at the
// pair's receive side again (mirror, state, ring image) -- it is a couple of microseconds behind at most
static int owner_of(const Runtime& r, const b200_pair* p);
static int32_t slot_word(const b200_pair* p) {  // SvcCmd.slot: the pair's slot, the loopback peer's slot + 1 above it
  return (int32_t)((uint32_t)p->slot | (p->peer_local ? ((uint32_t)p->peer_local->slot + 1) << 16 : 0));
}
// a command for p: a Recv's destination and capacity, a Send's slice list and its length, or (ptr unused) the size
// of the frame a Retire retires
static void fill_cmd(SvcCmd* c, const b200_pair* p, uint32_t op, uint32_t flags, const void* ptr, uint64_t n) {
  c->op = op;
  c->slot = slot_word(p);
  c->flags = flags;
  c->ptr = (uint64_t)(uintptr_t)ptr;
  c->n = n;
  c->byte_idx = 0;
}
static void fill_retire(SvcCmd* c, const b200_pair* p, uint32_t owed) {  // nothing owed: a no-op
  fill_cmd(c, p, owed ? kSvcRetire : kSvcNop, B200_BATCH_ONE_CALL, nullptr, owed);
}
static void drain_retire(b200_pair* p) {
  Runtime& r = R();
  if (p->retire_owed.load(std::memory_order_acquire) && r.svc_running.load()) {
    // The owed Retire is claimed INSIDE the queue's posting section: whoever claims it has its Retire in
    // the queue before anybody else can post another command for this connection (a Recv posted by the
    // pair's own thread while another thread -- the peer's sender looking for credit -- sat between "claimed"
    // and "posted" would deliver the frame a second time).
    const int q = owner_of(r, p);
    const uint64_t t = svc_post(r, q, [&](SvcCmd* c, SliceDev*) {
      fill_retire(c, p, p->retire_owed.exchange(0, std::memory_order_acq_rel));
    });
    // wait for what was posted (the Retire, or the no-op behind somebody else's Retire: the queue is in order,
    // so either way the pair's Retire has run when this returns)
    svc_wait(r, q, t, nullptr, nullptr);
  }
}

extern "C" void b200_service_stop(void) {
  Runtime& r = R();
  if (!r.inited || !r.svc_running.load()) return;
  cudaSetDevice(r.dev);
  for (b200_pair* p : r.all_pairs) drain_retire(p);
  for (int q = 0; q < r.svc_nowners; q++) {
    const uint64_t t = svc_post(r, q, [&](SvcCmd* c, SliceDev*) { c->op = kSvcStop; });
    svc_wait(r, q, t, nullptr, nullptr);  // the owner has left (its pool jobs are finished)
  }
  uint32_t one = 1;
  cudaMemcpyAsync(&r.d_svc_ps->stop, &one, 4, cudaMemcpyHostToDevice, r.stream);
  cudaStreamSynchronize(r.stream);
  cudaStreamSynchronize(r.svc_stream);  // the kernels exit
  cudaStreamSynchronize(r.svc_stream_big);
  cudaStreamSynchronize(r.svc_stream_poll);
  r.svc_running = false;
  delete[] r.svc_q;
  r.svc_q = nullptr;
  delete[] r.svc_consumed;
  r.svc_consumed = nullptr;
  {
    // the host poller thread reads the ready ring under scan_mu: hand it a null pointer before the free
    std::lock_guard<std::mutex> lk(r.scan_mu);
    ReadyEntry* ring = r.svc_ready;
    r.svc_ready = nullptr;
    cudaFreeHost(ring);
  }
  cudaFreeHost(r.svc_cmds);
  cudaFreeHost(r.svc_done);
  cudaFreeHost(r.svc_slices);
  cudaFreeHost(r.svc_erec);
  cudaFreeHost(r.svc_eslots);
  cudaFreeHost(r.svc_host_scans);
  cudaFree(r.d_svc_ps);
  cudaFree(r.d_svc_last_ev);
  cudaFree(r.d_svc_boxes);
  cudaFree(r.d_svc_psvc);
  r.svc_cmds = nullptr;
  r.svc_done = nullptr;
  r.svc_slices = nullptr;
  r.svc_erec = nullptr;
  r.svc_eslots = nullptr;
  r.svc_host_scans = nullptr;
  r.d_svc_ps = nullptr;
  r.d_svc_last_ev = nullptr;
  r.d_svc_boxes = nullptr;
  r.d_svc_psvc = nullptr;
  r.svc_workers = 0;
  r.svc_nowners = 0;
  std::vector<std::pair<void*, int>> dead;
  {
    std::lock_guard<std::mutex> lk(r.grave_mu);
    dead.swap(r.graveyard);
  }
  for (auto& d : dead) {
    if (d.second) cudaFreeHost(d.first);
    else cudaFree(d.first);
  }
}

// [0] ops executed, [1] ready-ring entries consumed by the host poller, [2] ready-ring overruns,
// [3] poller scans reported by the device (updated every 1024 scans)
extern "C" void b200_service_stats(uint64_t out[4]) {
  Runtime& r = R();
  out[0] = r.svc_ops.load();
  out[1] = r.svc_ready_seen.load();
  out[2] = r.svc_ready_overflows.load();
  out[3] = r.svc_host_scans ? *(volatile uint32_t*)r.svc_host_scans : 0;
}
extern "C" uint64_t b200_service_eager_hits(void) { return R().svc_eager_hits.load(); }
// experiment builds (-DB200_SVC_TRACE): accumulated device-side phase timers of the owner warps, see b200_kernels.cu
extern "C" int b200_debug_service_trace(unsigned long long* out16) { return svc_trace_read(out16); }

// Where a Send stages its unregistered slices: [base, base + cap), filled from off.  grow: the calling thread's tx
// buffer, grown at the first unregistered slice to the ring plus a 16-byte step per slice of the larger window
// (kCoalesceSlices >= kMaxSgeLimit), more than a one-call op stages.
struct SendStage {
  uint8_t* base;
  uint64_t cap, off;
  bool grow;
};
constexpr uint64_t kSendSlack = 16ull * (kCoalesceSlices + 4);

// The slice list of one Send op in out[]: <= max_sge slices (coalesced: kCoalesceSlices; until-blocked:
// kSvcSliceArea - 1) are looked at (*nreal), the rest only counts towards total_slice_size (pair.cc:661-664) and is
// folded into one trailing pseudo-slice that is never dereferenced.  Unregistered host memory is copied to st like the
// reference copies slices into its registered send buffer (pair.cc:690-694), in 16-byte steps, with (ptr + skip)
// pointing at the staged bytes.
//   One call: the kernel never accepts more than C/2 bytes (one frame of at most CWS(C/2), or frames that share a
//   C/2 staging size) and reads them from the front of the slices, so only the first C/2 bytes from byte_idx on are
//   staged: at most C/2 plus a 16-byte step per looked-at slice.  st must hold all of it (-1 otherwise).
//   Until blocked: the looked-at slices are staged whole while they fit.  The slice that does not fit is staged as far
//   as st reaches and its entry shortened; the rest of it is folded into the pseudo-slice with what follows, so
//   total_slice_size is unchanged and the op stops at the end of the staged prefix as if the ring had filled there.
//   A slice that finds st full ends the prefix before it.
// out == nullptr measures: nothing is copied or written, st.off ends at the bytes the op stages (stage_need).
// Returns the number of entries, -1 when the staging cannot be allocated or does not hold a one-call op.
static long stage_send(const b200_pair* p, SliceDev* out, const b200_slice* slices, size_t n, size_t byte_idx,
                       bool one_call, SendStage& st, size_t* nreal) {
  size_t look = one_call ? (p->coalesce ? kCoalesceSlices : (size_t)p->max_sge) : kSvcSliceArea - 1;
  if (look > n) look = n;
  uint64_t budget = p->cap / 2;  // one call: bytes the kernel may still read, in slice order
  uint64_t cut = 0;              // until blocked: bytes of the last looked-at slice beyond the staged prefix
  for (size_t i = 0; i < look; i++) {
    const uint8_t* ptr = (const uint8_t*)slices[i].ptr;
    const uint64_t len = slices[i].len;
    const uint64_t skip = i == 0 ? byte_idx : 0;
    uint64_t take = len > skip ? len - skip : 0;
    if (one_call) {
      if (take > budget) take = budget;
      budget -= take;
    }
    if (out) out[i] = SliceDev{ptr, len};
    if (!len || mem_kind(ptr) != 0) continue;
    if (st.grow) {
      TlsBounce& tb = tls_bounce();
      if (!ensure_bounce(&tb.tx, &tb.tx_cap, p->cap + kSendSlack)) return -1;
      st = SendStage{tb.tx, tb.tx_cap, 0, false};
    }
    const uint64_t room = st.cap > st.off ? st.cap - st.off : 0;
    bool last = false;
    if (take > room) {
      if (one_call) {
        set_err("stage_send: the staging buffer does not hold what one call reads");
        return -1;
      }
      if (!room) {
        look = i;
        break;
      }
      cut = take - room;
      take = room;
      last = true;
    }
    if (out) {
      memcpy(st.base + st.off, ptr + skip, take);
      out[i].ptr = st.base + st.off - skip;
      if (last) out[i].len = skip + take;
    }
    st.off += (take + 15) & ~15ull;
    if (last) {
      look = i + 1;
      break;
    }
  }
  *nreal = look;
  uint64_t rest = cut;
  for (size_t i = look; i < n; i++) rest += slices[i].len;
  if (!rest || !out) return (long)look;
  out[look].ptr = nullptr;
  out[look].len = rest;
  return (long)look + 1;
}

// The bytes stage_send stages for this op: what its SendStage must hold to stage it whole
static uint64_t stage_need(const b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx, bool one_call) {
  SendStage st{nullptr, ~0ull, 0, false};
  size_t nreal = 0;
  stage_send(p, nullptr, slices, n, byte_idx, one_call, st, &nreal);
  return st.off;
}

// A Send command that carries the pair's owed Retire (the owner warp runs it right after the Send), claimed inside
// the queue's posting section, see drain_retire.  When the slices cannot be staged the command is the Retire alone
// and the answer is false.
static bool fill_send_cmd(b200_pair* p, SvcCmd* c, SliceDev* area, const b200_slice* slices, size_t n, size_t byte_idx,
                          uint32_t flags, SendStage& st) {
  const uint32_t owed = p->retire_owed.exchange(0, std::memory_order_acq_rel);
  size_t nreal = 0;
  const long nsl = stage_send(p, area, slices, n, byte_idx, !(flags & B200_BATCH_UNTIL_BLOCKED), st, &nreal);
  if (nsl < 0) {
    fill_retire(c, p, owed);
    return false;
  }
  if (nsl <= (long)kSvcInline) memcpy(c->inl, area, nsl * sizeof(SliceDev));
  fill_cmd(c, p, kSvcSend, flags | (owed << 16), area, nsl);
  c->nreal = (uint32_t)nreal;
  c->byte_idx = byte_idx;
  return true;
}

static uint64_t svc_send(Runtime& r, b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx) {
  const int q = owner_of(r, p);
  bool ok = true;
  SendStage st{nullptr, 0, 0, true};
  const uint64_t t = svc_post(r, q, [&](SvcCmd* c, SliceDev* area) {
    ok = fill_send_cmd(p, c, area, slices, n, byte_idx, B200_BATCH_ONE_CALL, st);
  });
  uint64_t bytes = 0;
  if (!svc_wait(r, q, t, &bytes, nullptr) || !ok) {
    p->error = t_err;
    p->status = B200_ERROR;
    return 0;
  }
  return bytes;
}

// Recv into unregistered host memory goes through the calling thread's pinned rx buffer (one frame never exceeds
// the ring, so the capacity is clipped to it); recv_bounce_out copies what was delivered to dst
static uint8_t* recv_bounce_in(const b200_pair* p, void* dst, int kind, uint64_t* cap) {
  if (kind != 0) return (uint8_t*)dst;
  if (*cap > p->cap) *cap = p->cap;
  TlsBounce& tb = tls_bounce();
  return ensure_bounce(&tb.rx, &tb.rx_cap, p->cap) ? tb.rx : nullptr;
}
static uint64_t recv_bounce_out(void* dst, const uint8_t* kdst, uint64_t got) {
  if (kdst != dst && got) memcpy(dst, kdst, got);
  return got;
}

static uint64_t eager_checksum(const uint8_t* slot, uint32_t size, uint64_t at) {
  uint64_t cs = eager_mix(at * 31 + size);
  const uint32_t words = (size + 7) >> 3;
  for (uint32_t j = 0; j < words; j++) {
    uint64_t w = *(const volatile uint64_t*)(slot + 8ull * j);
    const uint32_t rem = size - 8 * j;
    if (rem < 8) w &= (1ull << (8 * rem)) - 1;
    cs ^= eager_word(w, j);
  }
  return cs;
}

static uint64_t svc_recv(Runtime& r, b200_pair* p, void* dst, uint64_t cap) {
  const int q = owner_of(r, p);
  const int kind = mem_kind3(dst);
  // ---- eager: the frame at the head of the ring was already pushed to this pair's host slot by the kernel
  // that landed it (or that retired its predecessor): take it from there, retire it asynchronously
  if (r.svc_erec && kind != 2 && !p->remote) {
    volatile EagerRec* rec = &r.svc_erec[p->slot];
    const uint8_t* slot = r.svc_eslots + (size_t)p->slot * kEagerMax;
    for (int attempt = 0; attempt < 4; attempt++) {
      const uint64_t at = rec->at;
      const uint32_t size = rec->size;
      if (rec->magic != kEagerMagic || at != p->svc_delivered || size == 0 || size > kEagerMax || size > cap) break;
      const uint64_t cs = rec->csum;
      memcpy(dst, slot, size);
      if (eager_checksum((const uint8_t*)dst, size, at) != cs) continue;  // payload stores still in flight: look again
      p->svc_delivered += size;
      p->retire_owed.store(size, std::memory_order_release);  // rides on the next Send, or drain_retire posts it
      r.svc_eager_hits++;
      return size;
    }
  }
  uint64_t kcap = cap;
  uint8_t* kdst = recv_bounce_in(p, dst, kind, &kcap);
  if (!kdst) return 0;
  const uint64_t t = svc_post(r, q, [&](SvcCmd* c, SliceDev*) { fill_cmd(c, p, kSvcRecv, B200_BATCH_ONE_CALL, kdst, kcap); });
  uint64_t bytes = 0;
  if (!svc_wait(r, q, t, &bytes, nullptr)) {
    p->error = t_err;
    p->status = B200_ERROR;
    return 0;
  }
  p->svc_delivered += bytes;
  return recv_bounce_out(dst, kdst, bytes);
}

// ================================================================ device API

// The host-visible mirror of p from the device state (readiness as rx_probe computes it).  dev_closed is left as it
// is: b200_warp_disconnect sets it (the release of an unmirrored end does, from the row), Init clears it with the
// rest of the mirror.  Returns the row's status (-1 when the device could not be read).
static int republish_mirror(Runtime& r, b200_pair* p) {
  PairDev hd;
  PairSeq sq;
  if (!CU_OK(cudaMemcpy(&hd, &r.d_pairs[p->slot], sizeof(hd), cudaMemcpyDeviceToHost)) ||
      !CU_OK(cudaMemcpy(&sq, pair_seq(r.d_pairs, p->slot), sizeof(sq), cudaMemcpyDeviceToHost)))
    return -1;
  uint32_t hm = 0;
  uint64_t rd = 0;
  if (hd.remain > 0) {
    hm = 1;
    rd = hd.remain;
  } else if (hd.ring) {
    const uint32_t st = (hd.max_sge & kSgeStamped) ? stamp_of(sq.rx) : 0;
    uint64_t hdr = 0, foot = 0;
    if (!CU_OK(cudaMemcpy(&hdr, hd.ring + hd.head, 8, cudaMemcpyDeviceToHost))) return -1;
    hm = hdr != 0;
    const uint64_t len = frame_present(hdr, hd.cap, st);
    if (len && CU_OK(cudaMemcpy(&foot, hd.ring + ((hd.head + 8 + round_up8(len)) & (hd.cap - 1)), 8,
                                cudaMemcpyDeviceToHost)) && foot == frame_footer(hdr, st))
      rd = len;
    if (st) hm = rd != 0;
  }
  volatile PairMirror* m = p->mirror;
  m->head = hd.head;
  m->moving_head = hd.moving_head;
  m->remain = hd.remain;
  m->acc = hd.acc;
  m->readable = rd;
  m->has_message = hm;
  m->remote_tail = hd.remote_tail;
  m->credit_head = hd.credit_head;
  m->partial_write = hd.partial_write;
  m->peer_exit = hd.credit_exit;
  return (int)hd.status;
}

// The mirror pointers of p's row and, on the loopback wire, of its peer's row (peer_mirror): null for an unmirrored
// claim, p->mirror again at its release.  The peer's row is left alone once the peer has left the connection.
// Caller holds r.mu.
static bool set_mirror_pointers(Runtime& r, b200_pair* p, bool on) {
  PairMirror* const m = on ? p->mirror : nullptr;
  bool ok = CU_OK(cudaMemcpyAsync(&r.d_pairs[p->slot].mirror, &m, sizeof(m), cudaMemcpyHostToDevice, r.stream));
  b200_pair* q = p->peer_local;
  if (q && q->peer_local == p)
    ok = ok && CU_OK(cudaMemcpyAsync(&r.d_pairs[q->slot].peer_mirror, &m, sizeof(m), cudaMemcpyHostToDevice, r.stream));
  return CU_OK(cudaStreamSynchronize(r.stream)) && ok;
}

extern "C" int b200_pair_device_claim(b200_pair* p, b200_dev_pair* out) { return b200_pair_device_claim_ex(p, 0, out); }

extern "C" int b200_pair_device_claim_ex(b200_pair* p, int flags, b200_dev_pair* out) {
  if (flags & ~B200_CLAIM_UNMIRRORED) {
    set_err("b200_pair_device_claim_ex: unknown flag bits");
    return -1;
  }
  const bool unmirrored = (flags & B200_CLAIM_UNMIRRORED) != 0;
  if (!p || !out || !ensure_init()) {
    set_err("b200_pair_device_claim: no pair / no output / no CUDA device");
    return -1;
  }
  Runtime& r = R();
  if (p->status != B200_CONNECTED) {
    set_err("b200_pair_device_claim: the pair is not connected");
    return -1;
  }
  drain_retire(p);
  bool was = false;
  if (!p->device_owned.compare_exchange_strong(was, true)) {
    set_err("b200_pair_device_claim: the pair is already device-owned");
    return -1;
  }
  if (p->host_ops.load() != 0) {
    p->device_owned = false;
    set_err("b200_pair_device_claim: host operations on the pair are in flight");
    return -1;
  }
  drain_retire(p);  // (an eager Recv that finished between the first drain and the claim)
  {
    std::lock_guard<std::mutex> lk(r.mu);
    if (unmirrored) {
      // A host op of the loopback peer may have loaded this end's mirror pointer before it goes null and publish
      // through it afterwards: refused while one is in flight.  An op counted after this check starts after the
      // pointers are null (single calls wait for r.mu, held here).  On the CUDA-IPC wire the host scans publish an
      // end's mirror: none runs while scan_mu is held.
      b200_pair* q = p->peer_local;
      if (q && q->host_ops.load() != 0) {
        p->device_owned = false;
        set_err("b200_pair_device_claim_ex: host operations on the peer end are in flight");
        return -1;
      }
      std::unique_lock<std::mutex> sl(r.scan_mu, std::defer_lock);
      if (p->remote) sl.lock();
      cudaSetDevice(r.dev);
      if (!set_mirror_pointers(r, p, false)) {
        set_mirror_pointers(r, p, true);
        p->device_owned = false;
        set_err("b200_pair_device_claim_ex: " + std::string(t_err));
        return -1;
      }
      p->unmirrored = true;
    }
    r.dev_slot[p->slot] = 1;
    if (r.svc_running.load()) memset((void*)&r.svc_erec[p->slot], 0, sizeof(EagerRec));  // no eager Recv any more
    ((volatile PairMirror*)p->mirror)->dev_closed = 0;  // (a CONNECTED end: clear since Init; set only by the device)
    r.svc_gen++;
    memset(out, 0, sizeof(*out));
    out->table = r.d_pairs;
    out->seq = pair_seq(r.d_pairs, 0);
    out->mirrors = r.h_mirrors;
    out->slot = p->slot;
    out->wire = p->remote ? 1 : 0;
  }
  if (r.svc_running.load()) {
    // the connection's queue is in order: once this no-op is answered, every command of the peer posted before the
    // claim has run, and the owner has seen the new generation (its cached lines of the connection are gone)
    const int q = owner_of(r, p);
    const uint64_t t = svc_post(r, q, [&](SvcCmd* c, SliceDev*) {
      c->op = kSvcNop;
      c->slot = slot_word(p);
      c->flags = B200_BATCH_ONE_CALL;
    });
    svc_wait(r, q, t, nullptr, nullptr);
    if (unmirrored && p->remote) {
      // the device poller publishes the mirrors of CUDA-IPC ends: a scan that loaded the pointer before it went null
      // may publish once more.  Two completed scans later none can; the mirror is then rebuilt from the device.  The
      // wait does not hold r.mu: the other pairs' host calls go on meanwhile.
      uint32_t s0 = 0, s = 0;
      cudaMemcpyAsync(&s0, &r.d_svc_ps->scans, 4, cudaMemcpyDeviceToHost, r.stream);
      cudaStreamSynchronize(r.stream);
      const auto until = std::chrono::steady_clock::now() + std::chrono::seconds(5);
      do {
        std::this_thread::sleep_for(std::chrono::microseconds(20));
        cudaMemcpyAsync(&s, &r.d_svc_ps->scans, 4, cudaMemcpyDeviceToHost, r.stream);
        cudaStreamSynchronize(r.stream);
      } while (s - s0 < 2 && std::chrono::steady_clock::now() < until);
      std::lock_guard<std::mutex> lk(r.mu);
      if (s - s0 < 2) {
        device_release_locked(r, p);
        set_err("b200_pair_device_claim_ex: the device poller did not complete a scan");
        return -1;
      }
      republish_mirror(r, p);
    }
  }
  return 0;
}

// caller holds r.mu.  The device Recv calls do not count in the service's delivered counts (host and device
// agree on them still); the eager record may have been pushed from a stale view: it is dropped.
static void device_release_locked(Runtime& r, b200_pair* p) {
  if (!p->device_owned.load()) return;
  cudaSetDevice(r.dev);
  if (p->ready_set) {  // membership ends with the claim: no producer finds the note from here on
    cudaMemsetAsync(ready_note(r.d_pairs, p->slot), 0, sizeof(ReadyNote), r.stream);
    cudaStreamSynchronize(r.stream);
    p->ready_set->members--;
    p->ready_set = nullptr;
  }
  const bool unmirrored = p->unmirrored.load();
  if (unmirrored) {
    // publication resumes before the mirror is rebuilt from the device, so no update falls between the two
    set_mirror_pointers(r, p, true);
    p->unmirrored = false;
  }
  if (r.svc_running.load()) {
    const PairSvc fresh{p->svc_delivered, ~0ull};
    memset((void*)&r.svc_erec[p->slot], 0, sizeof(EagerRec));
    cudaMemcpyAsync(&r.d_svc_psvc[p->slot], &fresh, sizeof(fresh), cudaMemcpyHostToDevice, r.stream);
    cudaStreamSynchronize(r.stream);
  }
  const int row_status = republish_mirror(r, p);
  // an unmirrored end's b200_warp_disconnect could not set the mirror's flag: the row's status tells
  if (unmirrored && p->status == B200_CONNECTED && row_status == B200_DISCONNECTED)
    ((volatile PairMirror*)p->mirror)->dev_closed = 1;
  r.svc_gen++;
  r.dev_slot[p->slot] = 0;
  p->device_owned = false;
  if (p->error == kDeviceOwnedRefusal) p->error.clear();
  // b200_warp_disconnect told the peer and marked the row: the rest of the Disconnect, with no second peer_exit write
  if (p->status == B200_CONNECTED && ((volatile PairMirror*)p->mirror)->dev_closed) close_host_side(r, p);
}

extern "C" int b200_pair_device_release(b200_pair* p) {
  if (!p || !p->device_owned.load()) {
    set_err("b200_pair_device_release: the pair is not device-owned");
    return -1;
  }
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  device_release_locked(r, p);
  return 0;
}

extern "C" int b200_pair_device_owned(const b200_pair* p) { return p && p->device_owned.load() ? 1 : 0; }

// ================================================================ ready sets

extern "C" b200_ready_set* b200_ready_set_create(uint32_t capacity) {
  if (capacity < 1 || capacity > (uint32_t)kMaxPairs) {
    set_err("b200_ready_set_create: capacity must be 1.." + std::to_string(kMaxPairs));
    return nullptr;
  }
  if (!ensure_init()) return nullptr;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  cudaSetDevice(r.dev);
  load_kernels();  // (a consumer kernel may be resident by the time of the first add)
  b200_ready_set* s = new b200_ready_set();
  s->capacity = capacity;
  s->size = ready_queue_size(capacity);
  const size_t bytes = sizeof(ReadyQueue) + sizeof(uint64_t) * s->size;
  const uint32_t mask = s->size - 1;
  if (!CU_OK(cudaHostAlloc((void**)&s->bell, 2 * sizeof(uint64_t), cudaHostAllocMapped | cudaHostAllocPortable)) ||
      !CU_OK(cudaMalloc(&s->q, bytes)) || !CU_OK(cudaMemsetAsync(s->q, 0, bytes, r.stream)) ||
      !CU_OK(cudaMemcpyAsync(&s->q->mask, &mask, 4, cudaMemcpyHostToDevice, r.stream)) ||
      !CU_OK(cudaMemcpyAsync(&s->q->bell, &s->bell, sizeof(s->bell), cudaMemcpyHostToDevice, r.stream)) ||
      !CU_OK(cudaStreamSynchronize(r.stream))) {
    if (s->q) rt_free(s->q, 0);
    if (s->bell) rt_free(s->bell, 1);
    delete s;
    return nullptr;
  }
  s->bell[0] = s->bell[1] = 0;
  return s;
}

extern "C" int b200_ready_set_device(b200_ready_set* s, b200_dev_ready_set* out) {
  if (!s || !out) {
    set_err("b200_ready_set_device: no set / no output");
    return -1;
  }
  memset(out, 0, sizeof(*out));
  out->queue = s->q;
  out->capacity = s->capacity;
  out->size = s->size;
  return 0;
}

extern "C" int b200_ready_set_destroy(b200_ready_set* s) {
  if (!s) return -1;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (s->members) {
    set_err("b200_ready_set_destroy: the set has " + std::to_string(s->members) + " members");
    return -1;
  }
  {  // the Poller reads the doorbell under its lock: after this block it never looks at the set again
    std::lock_guard<std::mutex> plk(r.pmu);
    auto& v = r.bell_sets;
    v.erase(std::remove(v.begin(), v.end(), s), v.end());
  }
  if (s->wakeup_fd >= 0) close(s->wakeup_fd);
  rt_free(s->q, 0);
  rt_free(s->bell, 1);
  delete s;
  return 0;
}

extern "C" int b200_ready_set_park(b200_ready_set* s) {
  if (!s) {
    set_err("b200_ready_set_park: no set");
    return -1;
  }
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  cudaSetDevice(r.dev);
  volatile int* res = reinterpret_cast<volatile int*>(&s->bell[1]);
  *res = -1;
  launch_ready_park(s->q, (int*)res, r.stream);
  r.launches++;
  if (!CU_OK(cudaGetLastError()) || !CU_OK(cudaStreamSynchronize(r.stream))) return -1;
  return *res;
}

static void poller_start_locked(Runtime& r);

extern "C" int b200_ready_set_wakeup_fd(b200_ready_set* s) {
  if (!s) return -1;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.pmu);
  if (s->wakeup_fd < 0) {
    s->wakeup_fd = eventfd(0, EFD_NONBLOCK | EFD_CLOEXEC);
    if (s->wakeup_fd < 0) {
      set_err("b200_ready_set_wakeup_fd: eventfd failed");
      return -1;
    }
    s->bell_seen = 0;  // (a ring before this call signals the new fd on the Poller's first pass)
    r.bell_sets.push_back(s);
    poller_start_locked(r);
    r.pcv.notify_all();
  }
  return s->wakeup_fd;
}

extern "C" void b200_ready_set_consume_wakeup(b200_ready_set* s) {
  if (!s || s->wakeup_fd < 0) return;
  eventfd_t v;
  (void)eventfd_read(s->wakeup_fd, &v);
}

extern "C" uint64_t b200_ready_set_rings(const b200_ready_set* s) {
  return s ? *(const volatile uint64_t*)&s->bell[0] : 0;
}

extern "C" int b200_ready_set_add(b200_ready_set* s, b200_pair* p, uint32_t key) {
  if (!s || !p) {
    set_err("b200_ready_set_add: no set / no pair");
    return -1;
  }
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.mu);
  if (!p->device_owned.load()) {
    set_err("b200_ready_set_add: the pair is not device-owned (b200_pair_device_claim)");
    return -1;
  }
  if (p->remote || !p->peer_local) {
    set_err("b200_ready_set_add: the pair is not on the loopback wire (its peer's kernels cannot reach the set)");
    return -1;
  }
  if (p->ready_set) {
    set_err("b200_ready_set_add: the pair is already a member of a ready set");
    return -1;
  }
  cudaSetDevice(r.dev);
  uint32_t head = 0, tail = 0;
  if (!CU_OK(cudaMemcpyAsync(&head, &s->q->head, 4, cudaMemcpyDeviceToHost, r.stream)) ||
      !CU_OK(cudaMemcpyAsync(&tail, &s->q->tail, 4, cudaMemcpyDeviceToHost, r.stream)) ||
      !CU_OK(cudaStreamSynchronize(r.stream)))
    return -1;
  const int chk = ready_add_check(head, tail, s->members, s->capacity, s->size);
  if (chk == kReadyAddFull) {
    set_err("b200_ready_set_add: the set is full (" + std::to_string(s->capacity) + " members)");
    return -1;
  }
  if (chk == kReadyAddOverflow) {
    set_err("b200_ready_set_add: the queue could overflow: " + std::to_string(tail - head) +
            " entries queued (stale entries of released members included) and " + std::to_string(s->members) +
            " members against " + std::to_string(s->size) + " entries; take from the set first");
    return -1;
  }
  launch_ready_add(r.d_pairs, p->slot, s->q, key, r.stream);
  r.launches++;
  if (!CU_OK(cudaGetLastError()) || !CU_OK(cudaStreamSynchronize(r.stream))) return -1;
  s->members++;
  p->ready_set = s;
  return 0;
}

// ================================================================ single call

static bool ensure_bounce(uint8_t** buf, uint64_t* cap, uint64_t need) {
  if (*cap >= need) return true;
  if (*buf) rt_free(*buf, 1);
  *buf = nullptr;
  *cap = 0;
  if (!CU_OK(cudaHostAlloc((void**)buf, need, cudaHostAllocMapped | cudaHostAllocPortable))) return false;
  *cap = need;
  return true;
}

// The endpoint re-enters Send from the poll loop for as long as a write is pending, whether or not
// the peer has returned credit (poller.cc:83, rdma_bp_posix.cc:527-557).  On the CPU that is a cheap
// call; here it would be a launch per spin.  When the host-visible mirror already shows that the
// call cannot accept a byte (no credit for even one frame and the partial-write flag already set),
// the answer and the resulting state are exactly those of the kernel, so no kernel runs.
// The mirror short-cuts below are not taken when a user kernel drives the other end (b200_pair_device_claim): its
// warps and ours publish the mirror concurrently, so the answer comes from the device state instead.
static bool peer_device_owned(const b200_pair* p) { return p->peer_local && p->peer_local->device_owned.load(); }
static bool send_is_a_no_op(const b200_pair* p) {
  if (peer_device_owned(p)) return false;
  volatile PairMirror* m = p->mirror;
  if (!m->partial_write) return false;
  const uint64_t fr = free_size(p->cap, m->credit_head, m->remote_tail);
  const uint64_t lim = p->cap / 2 < fr ? p->cap / 2 : fr;
  return calc_writable(lim) == 0;
}

extern "C" uint64_t b200_pair_send(b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx) {
  if (!p || !ensure_init()) return 0;
  Runtime& r = R();
  const HostOp op(p);
  if (!op.ok) return 0;
  if (p->peer_dead.load()) return 0;  // nobody owns the remote ring any more: get_status reports HalfClosed
  if (p->status == B200_CONNECTED && n) {
    if (p->peer_local) drain_retire(p->peer_local);  // its Retire may be about to return credit
    refresh_remote(p);
    if (send_is_a_no_op(p)) return 0;
  }
  if (r.svc_running.load()) {
    if (p->status != B200_CONNECTED || n == 0) return 0;
    if (((volatile PairMirror*)p->mirror)->peer_exit == 1) return 0;
    return svc_send(r, p, slices, n, byte_idx);
  }
  std::lock_guard<std::mutex> lk(r.mu);
  if (p->status != B200_CONNECTED || n == 0) return 0;
  // The peer told us it left (peer_exit): its ring may already belong to a new
  // connection, so nothing is written; rdma_flush then reports "Peer has been
  // exited" from get_status() exactly as with the reference (rdma_bp_posix.cc:507-511).
  if (((volatile PairMirror*)p->mirror)->peer_exit == 1) return 0;
  cudaSetDevice(r.dev);
  SendStage st{nullptr, 0, 0, true};
  size_t nreal = 0;
  const long nsl = stage_send(p, r.h_slices, slices, n, byte_idx, true, st, &nreal);
  if (nsl < 0) return 0;
  r.h_sop->slot = p->slot;
  // a device-owned peer publishes its mirror fields under the per-pair lock: so must we
  const bool conc = p->peer_local && p->peer_local->device_owned.load();
  r.h_sop->flags = B200_BATCH_ONE_CALL | (conc ? B200_BATCH_CONCURRENT : 0);
  r.h_sop->slices = r.h_slices;
  r.h_sop->nslices = nsl;
  r.h_sop->nreal = nreal;
  r.h_sop->byte_idx = byte_idx;
  r.h_res->bytes = 0;
  r.h_res->calls = 0;
  launch_send(r.d_pairs, r.h_sop, r.h_res, 1, r.stream);
  r.launches++;
  if (!CU_OK(cudaGetLastError()) || !CU_OK(cudaStreamSynchronize(r.stream))) {
    p->error = t_err;
    p->status = B200_ERROR;
    return 0;
  }
  return r.h_res->bytes;
}

extern "C" uint64_t b200_pair_recv(b200_pair* p, void* dst, uint64_t cap) {
  if (!p || !ensure_init()) return 0;
  Runtime& r = R();
  const HostOp op(p);
  if (!op.ok) return 0;
  drain_retire(p);
  // same reasoning for a Recv on a ring the mirror shows empty: it delivers nothing, changes nothing
  if (p->status == B200_CONNECTED && !p->remote && !peer_device_owned(p) &&
      ((volatile PairMirror*)p->mirror)->has_message == 0)
    return 0;
  if (r.svc_running.load()) {
    if (p->status != B200_CONNECTED || cap == 0) return 0;
    return svc_recv(r, p, dst, cap);
  }
  std::lock_guard<std::mutex> lk(r.mu);
  if (p->status != B200_CONNECTED || cap == 0) return 0;
  cudaSetDevice(r.dev);
  uint64_t kcap = cap;
  uint8_t* kdst = recv_bounce_in(p, dst, mem_kind(dst), &kcap);
  if (!kdst) return 0;
  r.h_rop->slot = p->slot;
  const bool conc = p->peer_local && p->peer_local->device_owned.load();
  r.h_rop->flags = B200_BATCH_ONE_CALL | (conc ? B200_BATCH_CONCURRENT : 0);
  r.h_rop->dst = kdst;
  r.h_rop->cap = kcap;
  r.h_res->bytes = 0;
  r.h_res->calls = 0;
  launch_recv(r.d_pairs, r.h_rop, r.h_res, 1, r.stream);
  r.launches++;
  if (!CU_OK(cudaGetLastError()) || !CU_OK(cudaStreamSynchronize(r.stream))) {
    p->error = t_err;
    p->status = B200_ERROR;
    return 0;
  }
  return recv_bounce_out(dst, kdst, r.h_res->bytes);
}

// ===================================================================== batch

static int lane_of(const b200_pair* p) {
  static const int nl = [] { long v = env_long("B200_LANES", 8); return (int)(v < 1 ? 1 : v > kLanes ? kLanes : v); }();
  static const int shift = (int)env_long("B200_LANE_SHIFT", 1);
  int key = p->slot;
  if (p->peer_local && p->peer_local->slot < key) key = p->peer_local->slot;
  return (key >> shift) % nl;  // both ends of a loopback connection share a lane: per-connection order
}

constexpr size_t kDmaAlign = 4096;

static size_t stage_place(size_t& cursor, const void* host_ptr, size_t bytes) {
  // keep the host buffer's alignment modulo 4 KiB: the kernels see the same (mis)alignment and
  // the DMA engine sees page-aligned transfers on both sides
  size_t off = ((cursor + kDmaAlign - 1) & ~(kDmaAlign - 1)) + ((uintptr_t)host_ptr & (kDmaAlign - 1));
  cursor = off + bytes;
  return off;
}

// A DMA copy whose HOST address is not 256-byte aligned runs well below the PCIe rate when both
// directions are busy (the device address and the size do not matter; splitting off small edge copies
// costs more than it saves -- tools/pcie_probe*.py calibrate this).
//   H2D: the transfer is widened to the enclosing 256-byte blocks of the host buffer (a few extra bytes
//        of the same pinned page land in the staging arena next to the slice and are never read);
//   D2H: must be exact, so destinations should be 256-byte aligned -- the endpoint allocates its read
//        slices itself (rdma_bp_posix.cc:308-317), from b200_mem_alloc_host they are.
constexpr size_t kHostDmaAlign = 256;
static void push_h2d(std::vector<CopyRun>& out, uint8_t* stage, const uint8_t* src, size_t bytes) {
  if (!bytes) return;
  // only the START needs the alignment (the size does not matter), and only inside the registered
  // range the bytes belong to: the driver rejects a copy that leaves it
  size_t lead = (uintptr_t)src & (kHostDmaAlign - 1);
  if (lead) {
    Runtime& r = R();
    std::lock_guard<std::mutex> lk(r.reg_mu);
    auto it = r.reg_ranges.upper_bound((uintptr_t)src);
    if (it == r.reg_ranges.begin()) {
      lead = 0;  // memory registered by someone else: its base is unknown
    } else {
      --it;
      if ((uintptr_t)src >= it->first + it->second.first || (uintptr_t)src - lead < it->first) lead = 0;
    }
  }
  out.push_back({stage - lead, src - lead, lead + bytes});
}

// the cluster width of a batch's flags (B200_BATCH_CLUSTER; field 0 = 1)
static int cluster_of(int flags) { return (int)(((unsigned)flags >> 4) & 15u) + 1; }
constexpr int kClusterField = 0xf0;

// Can this device place one cluster of `k` CTAs of the batch kernel at all?  Asked once per kind and k.
static bool cluster_placeable(int kind, int k) {
  static std::atomic<int> known[2][17];  // 0 = not asked yet, 1 = no, 2 = yes
  std::atomic<int>& a = known[kind][k];
  if (a.load() == 0) a.store(cluster_capacity(kind, k) > 0 ? 2 : 1);
  return a.load() == 2;
}

static b200_batch* prepare_common(int kind, const void* ops_v, size_t nops, int flags) {
  if (!ensure_init()) return nullptr;
  const int cluster = cluster_of(flags);
  if (cluster > 1 && !cluster_placeable(kind, cluster)) {
    set_err("b200_batch_prepare: this device cannot place a cluster of " + std::to_string(cluster) + " CTAs of the " +
            (kind == 0 ? "Send" : "Recv") + " kernel (B200_BATCH_CLUSTER)");
    return nullptr;
  }
  if (any_device_owned((const b200_pair* const*)ops_v, nops, kind == 0 ? sizeof(b200_send_op) : sizeof(b200_recv_op),
                       "b200_batch_prepare"))
    return nullptr;
  Runtime& r = R();
  cudaSetDevice(r.dev);
  b200_batch* b = new b200_batch();
  b->kind = kind;
  b->nops = (int)nops;
  b->flags = flags;
  b->cluster = cluster;
  const b200_send_op* sops = (const b200_send_op*)ops_v;
  const b200_recv_op* rops = (const b200_recv_op*)ops_v;
  bool ok = true;
  // ---- where do the payload bytes live?
  int cls = -1;
  for (size_t i = 0; ok && i < nops; i++) {
    const b200_pair* pr = kind == 0 ? sops[i].pair : rops[i].pair;
    if (!pr) {
      set_err("batch: null pair");
      ok = false;
      break;
    }
    const void* probe = nullptr;
    if (kind == 0) {
      for (size_t j = 0; j < sops[i].nslices && !probe; j++)
        if (sops[i].slices[j].len) probe = sops[i].slices[j].ptr;
    } else if (rops[i].cap) {
      probe = rops[i].dst;
    }
    if (!probe) continue;
    const int c = mem_kind3(probe);
    if (c == 0) {
      set_err("batch: slices / destinations must be GPU-addressable (device memory, b200_mem_alloc_host or "
              "b200_mem_register_host); unregistered host memory is only accepted by b200_pair_send/recv");
      ok = false;
    } else if (cls >= 0 && c != cls) {
      set_err("batch: host and device buffers cannot be mixed in one batch");
      ok = false;
    }
    cls = c;
  }
  b->staged = ok && cls == 1 && !(flags & B200_BATCH_ZEROCOPY);
  // ---- device order of the ops: lane-sorted for the staged path, caller's order otherwise
  b->perm.resize(nops);
  if (ok && b->staged) {
    int k = 0;
    for (int L = 0; L < kLanes; L++) {
      b->lanes[L].first_op = k;
      for (size_t i = 0; i < nops; i++)
        if (lane_of(kind == 0 ? sops[i].pair : rops[i].pair) == L) b->perm[k++] = (int)i;
      b->lanes[L].nops = k - b->lanes[L].first_op;
    }
  } else {
    for (size_t i = 0; i < nops; i++) b->perm[i] = (int)i;
  }
  const uint32_t kflags = (uint32_t)(flags & (B200_BATCH_UNTIL_BLOCKED | B200_BATCH_CONCURRENT));
  for (size_t k = 0; ok && k < nops; k++) b->op_pairs.push_back(kind == 0 ? sops[b->perm[k]].pair : rops[b->perm[k]].pair);
  if (ok && kind == 0) {
    size_t total_slices = 0;
    for (size_t i = 0; i < nops; i++) total_slices += sops[i].nslices;
    std::vector<SendOpDev> h(nops ? nops : 1);
    std::vector<SliceDev> hs(total_slices ? total_slices : 1);
    std::vector<size_t> stage_off(total_slices ? total_slices : 1, 0);
    ok = CU_OK(cudaMalloc(&b->d_slices, sizeof(SliceDev) * hs.size())) &&
         CU_OK(cudaMalloc(&b->d_ops, sizeof(SendOpDev) * (nops ? nops : 1)));
    size_t off = 0, cursor = 0;
    struct Run { int lane; const uint8_t* src; size_t bytes, stage; };
    std::vector<Run> runs;
    for (size_t k = 0; ok && k < nops; k++) {
      const b200_send_op& o = sops[b->perm[k]];
      h[k].slot = o.pair->slot;
      h[k].flags = kflags;
      h[k].slices = b->d_slices + off;
      h[k].nslices = o.nslices;
      h[k].nreal = o.nslices;
      h[k].byte_idx = o.byte_idx;
      const int L = b->staged ? lane_of(o.pair) : 0;
      const uint8_t* run_end = nullptr;
      for (size_t j = 0; j < o.nslices; j++) {
        const uint8_t* ptr = (const uint8_t*)o.slices[j].ptr;
        const uint64_t len = o.slices[j].len;
        hs[off + j].ptr = ptr;
        hs[off + j].len = len;
        if (b->staged && len) {
          // adjacent slices (a message cut into DATA frames) are staged by one copy
          if (runs.empty() || runs.back().lane != L || ptr != run_end) {
            Run nr = {L, ptr, 0, 0};
            nr.stage = stage_place(cursor, ptr, 0);
            runs.push_back(nr);
          }
          stage_off[off + j] = runs.back().stage + runs.back().bytes;
          runs.back().bytes += len;
          cursor = runs.back().stage + runs.back().bytes;
          run_end = ptr + len;
        }
      }
      off += o.nslices;
    }
    if (ok && b->staged) {
      ok = CU_OK(cudaMalloc(&b->d_stage, cursor + kDmaAlign));
      for (size_t q = 0; ok && q < total_slices; q++)
        if (hs[q].len) hs[q].ptr = b->d_stage + stage_off[q];
      for (const Run& rn : runs) push_h2d(b->lanes[rn.lane].copies, b->d_stage + rn.stage, rn.src, rn.bytes);
    }
    ok = ok && CU_OK(cudaMemcpy(b->d_slices, hs.data(), sizeof(SliceDev) * hs.size(), cudaMemcpyHostToDevice)) &&
         CU_OK(cudaMemcpy(b->d_ops, h.data(), sizeof(SendOpDev) * (nops ? nops : 1), cudaMemcpyHostToDevice));
    b->h_sops.swap(h);
  } else if (ok) {
    std::vector<RecvOpDev> h(nops ? nops : 1);
    ok = CU_OK(cudaMalloc(&b->d_ops, sizeof(RecvOpDev) * (nops ? nops : 1)));
    size_t cursor = 0;
    std::vector<size_t> place(nops ? nops : 1, 0);
    for (size_t k = 0; k < nops; k++) {
      const b200_recv_op& o = rops[b->perm[k]];
      h[k].slot = o.pair->slot;
      h[k].flags = kflags;
      h[k].dst = (uint8_t*)o.dst;
      h[k].cap = o.cap;
      b->pairs.push_back(o.pair);
      if (b->staged && o.cap) place[k] = stage_place(cursor, o.dst, o.cap);
    }
    if (ok && b->staged) {
      // zeroed once: the whole destination window is copied back, whatever was delivered into it
      ok = CU_OK(cudaMalloc(&b->d_stage, cursor + kDmaAlign)) && CU_OK(cudaMemset(b->d_stage, 0, cursor + kDmaAlign));
      for (size_t k = 0; ok && k < nops; k++) {
        const b200_recv_op& o = rops[b->perm[k]];
        if (!o.cap) continue;
        h[k].dst = b->d_stage + place[k];
        // the whole destination window comes back: callers size it to what they expect, like
        // the endpoint's max(256, GetReadableSize()) slice (rdma_bp_posix.cc:308-317)
        b->lanes[lane_of(o.pair)].copies.push_back({o.dst, b->d_stage + place[k], (size_t)o.cap});
      }
    }
    ok = ok && CU_OK(cudaMemcpy(b->d_ops, h.data(), sizeof(RecvOpDev) * (nops ? nops : 1), cudaMemcpyHostToDevice));
    b->h_rops.swap(h);
  }
  ok = ok && CU_OK(cudaMalloc(&b->d_results, sizeof(OpResult) * (nops ? nops : 1))) &&
       CU_OK(cudaHostAlloc(&b->h_results, sizeof(OpResult) * (nops ? nops : 1), cudaHostAllocPortable));
  if (!ok) {
    b200_batch_destroy(b);
    return nullptr;
  }
  return b;
}

extern "C" b200_batch* b200_batch_prepare_send(const b200_send_op* ops, size_t nops, int flags) {
  return prepare_common(0, ops, nops, flags);
}
extern "C" b200_batch* b200_batch_prepare_recv(const b200_recv_op* ops, size_t nops, int flags) {
  return prepare_common(1, ops, nops, flags);
}

extern "C" int b200_lanes_fork(void* stream) {
  if (!ensure_init() || !stream) return -1;
  Runtime& r = R();
  if (!CU_OK(cudaEventRecord(r.fork_event, (cudaStream_t)stream))) return -1;
  for (int L = 0; L < kLanes; L++)
    if (!CU_OK(cudaStreamWaitEvent(r.lane_up[L], r.fork_event, 0)) ||
        !CU_OK(cudaStreamWaitEvent(r.lane_down[L], r.fork_event, 0)))
      return -1;
  return 0;
}

extern "C" int b200_lanes_join(void* stream) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  for (int L = 0; L < kLanes; L++) {
    if (stream) {
      if (!CU_OK(cudaEventRecord(r.join_up[L], r.lane_up[L])) ||
          !CU_OK(cudaEventRecord(r.join_down[L], r.lane_down[L])) ||
          !CU_OK(cudaStreamWaitEvent((cudaStream_t)stream, r.join_up[L], 0)) ||
          !CU_OK(cudaStreamWaitEvent((cudaStream_t)stream, r.join_down[L], 0)))
        return -1;
    } else if (!CU_OK(cudaStreamSynchronize(r.lane_up[L])) || !CU_OK(cudaStreamSynchronize(r.lane_down[L]))) {
      return -1;
    }
  }
  return 0;
}

// a device-owned peer, and the service's owner warps, publish mirror fields under the per-pair locks: so must the
// batch's kernels
static bool batch_make_concurrent(b200_batch* b) {
  bool need = R().svc_running.load();
  for (const b200_pair* p : b->op_pairs) need = need || (p->peer_local && p->peer_local->device_owned.load());
  if (!need || (b->flags & B200_BATCH_CONCURRENT)) return true;
  b->flags |= B200_BATCH_CONCURRENT;
  if (b->kind == 0) {
    for (SendOpDev& o : b->h_sops) o.flags |= kFlagConcurrent;
    return CU_OK(cudaMemcpy(b->d_ops, b->h_sops.data(), sizeof(SendOpDev) * b->h_sops.size(), cudaMemcpyHostToDevice));
  }
  for (RecvOpDev& o : b->h_rops) o.flags |= kFlagConcurrent;
  return CU_OK(cudaMemcpy(b->d_ops, b->h_rops.data(), sizeof(RecvOpDev) * b->h_rops.size(), cudaMemcpyHostToDevice));
}
static void batch_uncount(b200_batch* b) {
  if (!b->counted) return;
  Runtime& r = R();
  // the kernels have changed the pairs' lines behind the owners' caches: a new generation first, so that a command
  // that no longer sees the batch's ops in batch_slot carries it
  if (r.svc_running.load()) r.svc_gen++;
  for (b200_pair* p : b->op_pairs) {
    r.batch_slot[p->slot].fetch_sub(1);
    p->host_ops.fetch_sub(1);
  }
  b->counted = false;
}

extern "C" int b200_batch_launch(b200_batch* b, void* stream) {
  if (!b) return -1;
  Runtime& r = R();
  if (b->nops == 0) return 0;
  // from here until its results are collected the batch is a host op of each of its pairs (counted first, then the
  // ownership looked at: see HostOp)
  if (!b->counted) {
    for (b200_pair* p : b->op_pairs) {
      p->host_ops.fetch_add(1);
      r.batch_slot[p->slot].fetch_add(1);
    }
    b->counted = true;
  }
  if (any_device_owned((const b200_pair* const*)b->op_pairs.data(), b->op_pairs.size(), sizeof(b200_pair*),
                       "b200_batch_launch")) {
    batch_uncount(b);
    return -1;
  }
  if (!batch_make_concurrent(b)) return -1;
  if (r.svc_running.load()) r.svc_gen++;  // kernels beside the service change pair lines behind the owners' caches
  if (b->kind == 1 && r.svc_running.load()) {
    // frames are about to be consumed behind the service's back: whatever it pushed eagerly for these pairs
    // is stale from now on, and stays so (host and device counts no longer agree -> Recv takes the normal path)
    for (b200_pair* p : b->pairs) {
      drain_retire(p);
      ((volatile EagerRec*)&r.svc_erec[p->slot])->magic = 0;
      p->svc_delivered += 1ull << 40;
    }
  }
  if (!b->staged) {
    cudaStream_t s = stream ? (cudaStream_t)stream : r.stream;
    if (b->kind == 0) launch_send(r.d_pairs, (const SendOpDev*)b->d_ops, b->d_results, b->nops, s, b->cluster);
    else launch_recv(r.d_pairs, (const RecvOpDev*)b->d_ops, b->d_results, b->nops, s, b->cluster);
    r.launches++;
    return CU_OK(cudaGetLastError()) ? 0 : -1;
  }
  // Host-staged: per lane, Send = H2D of the slices then the kernel on the "up" stream, Recv =
  // the kernel then D2H of the destinations on the "down" stream.  A connection always maps to
  // the same lane.  Dependencies are the protocol's own: Recv after the Send kernels that wrote
  // the ring, Send kernel (not its H2D) after the Recv kernels that returned credit -- so the
  // two copy engines and the SMs run concurrently across lanes and across consecutive batches.
  if (stream && b200_lanes_fork(stream) != 0) return -1;
  for (int L = 0; L < kLanes; L++) {
    LanePlan& lp = b->lanes[L];
    if (lp.nops == 0) continue;
    if (b->kind == 0) {
      cudaStream_t s = r.lane_up[L];
      for (const CopyRun& c : lp.copies)
        if (!CU_OK(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyHostToDevice, s))) return -1;
      if (!CU_OK(cudaStreamWaitEvent(s, r.recv_done[L], 0))) return -1;
      launch_send(r.d_pairs, (const SendOpDev*)b->d_ops + lp.first_op, b->d_results + lp.first_op, lp.nops, s,
                  b->cluster);
      if (!CU_OK(cudaEventRecord(r.send_done[L], s))) return -1;
    } else {
      cudaStream_t s = r.lane_down[L];
      if (!CU_OK(cudaStreamWaitEvent(s, r.send_done[L], 0))) return -1;
      launch_recv(r.d_pairs, (const RecvOpDev*)b->d_ops + lp.first_op, b->d_results + lp.first_op, lp.nops, s,
                  b->cluster);
      if (!CU_OK(cudaEventRecord(r.recv_done[L], s))) return -1;
      for (const CopyRun& c : lp.copies)
        if (!CU_OK(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToHost, s))) return -1;
    }
    r.launches++;
    if (!CU_OK(cudaGetLastError())) return -1;
  }
  if (stream && b200_lanes_join(stream) != 0) return -1;
  return 0;
}

extern "C" int b200_batch_results(b200_batch* b, uint64_t* out, void* stream) {
  if (!b) return -1;
  Runtime& r = R();
  if (b->nops == 0) return 0;
  cudaStream_t s = stream ? (cudaStream_t)stream : r.stream;
  if (b->staged) {
    for (int L = 0; L < kLanes; L++)
      if (b->lanes[L].nops &&
          (!CU_OK(cudaStreamSynchronize(r.lane_up[L])) || !CU_OK(cudaStreamSynchronize(r.lane_down[L]))))
        return -1;
  }
  if (!CU_OK(cudaMemcpyAsync(b->h_results, b->d_results, sizeof(OpResult) * b->nops, cudaMemcpyDeviceToHost, s)) ||
      !CU_OK(cudaStreamSynchronize(s)))
    return -1;
  if (out)
    for (int k = 0; k < b->nops; k++) out[b->perm[k]] = b->h_results[k].bytes;
  batch_uncount(b);
  return 0;
}

extern "C" int b200_batch_calls(b200_batch* b, uint64_t* out) {
  if (!b || !out) return -1;
  for (int k = 0; k < b->nops; k++) out[b->perm[k]] = b->h_results[k].calls;
  return 0;
}

extern "C" void b200_batch_destroy(b200_batch* b) {
  if (!b) return;
  batch_uncount(b);
  rt_free(b->d_ops, 0);
  rt_free(b->d_slices, 0);
  rt_free(b->d_results, 0);
  rt_free(b->d_stage, 0);
  rt_free(b->h_results, 1);
  delete b;
}

static int run_unprepared(int kind, const void* ops, size_t nops, int flags, uint64_t* out, void* stream) {
  b200_batch* b = prepare_common(kind, ops, nops, flags);
  if (!b) return -1;
  int rc = b200_batch_launch(b, stream);
  // descriptors live in HBM owned by the batch object, so even the ASYNC form
  // has to wait before they are released
  if (rc == 0) rc = b200_batch_results(b, out, stream);
  b200_batch_destroy(b);
  return rc;
}

extern "C" int b200_pairs_send(const b200_send_op* ops, size_t nops, int flags, uint64_t* accepted, void* stream) {
  return run_unprepared(0, ops, nops, flags, accepted, stream);
}
extern "C" int b200_pairs_recv(const b200_recv_op* ops, size_t nops, int flags, uint64_t* delivered, void* stream) {
  return run_unprepared(1, ops, nops, flags, delivered, stream);
}

// ------------------------------------------------------------------ device staging of service Recvs

namespace {
// device staging blocks of the service's Recvs and pinned staging blocks of posted Sends (power-of-two classes: 2^31
// bytes at most for a Recv, any size a one-call Send stages) and finished posted-op handles, recycled
struct AsyncPool {
  std::mutex mu;
  std::vector<uint8_t*> free_stage[32], free_hstage[64];
  std::vector<b200_async*> free_ops;
  cudaStream_t copy[4] = {nullptr, nullptr, nullptr, nullptr};
  std::atomic<uint32_t> rr{0};
};
AsyncPool& AP() {
  static AsyncPool a;
  return a;
}
uint8_t* stage_get(uint64_t bytes, int* cls) {
  int c = 16;  // 64 KiB
  while ((1ull << c) < bytes) c++;
  *cls = c;
  AsyncPool& a = AP();
  {
    std::lock_guard<std::mutex> lk(a.mu);
    if (!a.free_stage[c].empty()) {
      uint8_t* p = a.free_stage[c].back();
      a.free_stage[c].pop_back();
      return p;
    }
  }
  uint8_t* p = nullptr;
  if (cudaMalloc(&p, 1ull << c) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void stage_put(uint8_t* p, int cls) {
  AsyncPool& a = AP();
  std::lock_guard<std::mutex> lk(a.mu);
  a.free_stage[cls].push_back(p);
}
// the D2H copies out of the staging blocks take the copy streams in turn
cudaStream_t copy_stream() {
  AsyncPool& a = AP();
  const uint32_t k = a.rr++ & 3;
  std::lock_guard<std::mutex> lk(a.mu);
  if (!a.copy[k]) cudaStreamCreateWithFlags(&a.copy[k], cudaStreamNonBlocking);
  return a.copy[k];
}
// Optional (B200_SUBMIT_STAGE_MIN=<bytes>, off by default): a Recv of the service (a b200_pairs_submit op or a posted
// Recv) into pinned HOST memory (kind 1) of at least that size goes through a device staging block and ONE contiguous
// D2H copy by the copy engine instead of SM stores over PCIe.  (SM-issued PCIe reads and writes share one ceiling,
// tools/zc_overlap.py; on the endpoint streaming workload the staged form measured the same as the in-place form.)
// nullptr: the Recv writes in place, as does one whose cap is larger than the largest block class (2^31 bytes).  The
// block goes back with stage_put once its copy has finished.
uint8_t* recv_stage(int kind, uint64_t cap, int* cls) {
  static const uint64_t kStageMin = (uint64_t)env_long("B200_SUBMIT_STAGE_MIN", 1l << 40);
  if (kind != 1 || cap < kStageMin || cap > (1ull << 31)) return nullptr;
  cudaSetDevice(R().dev);
  return stage_get(cap, cls);
}
}  // namespace

// One engine pass worth of work: every Send and every Recv the event loop has ready, posted together and
// waited for together.  With the service running nothing is launched: each op becomes a command of the pair's
// owner queue (large ones run on the pool CTAs, all of them side by side), slices and destinations are read
// and written in place over PCIe.  Without it the two batch launches are used.
extern "C" int b200_pairs_submit(const b200_send_op* sops, size_t ns, uint64_t* accepted, const b200_recv_op* rops,
                                 size_t nr, uint64_t* delivered, int flags) {
  if (!ensure_init()) return -1;
  if (flags & kClusterField) {
    set_err("b200_pairs_submit: B200_BATCH_CLUSTER applies to batch launches only; the service's owners and pool run "
            "one CTA per op");
    return -1;
  }
  Runtime& r = R();
  // the pass counts as a host op of each of its pairs until it returns
  static thread_local std::vector<b200_pair*> held;
  held.clear();
  for (size_t i = 0; i < ns; i++)
    if (sops[i].pair) held.push_back(sops[i].pair);
  for (size_t i = 0; i < nr; i++)
    if (rops[i].pair) held.push_back(rops[i].pair);
  for (b200_pair* p : held) p->host_ops.fetch_add(1);
  struct Release {
    ~Release() {
      for (b200_pair* p : held) p->host_ops.fetch_sub(1);
    }
  } release;
  if (any_device_owned((const b200_pair* const*)sops, ns, sizeof(b200_send_op), "b200_pairs_submit") ||
      any_device_owned((const b200_pair* const*)rops, nr, sizeof(b200_recv_op), "b200_pairs_submit"))
    return -1;
  if (!r.svc_running.load()) {
    int rc = 0;
    if (ns) rc = b200_pairs_send(sops, ns, flags, accepted, nullptr);
    if (rc == 0 && nr) rc = b200_pairs_recv(rops, nr, flags, delivered, nullptr);
    return rc;
  }
  struct Ticket {
    int q;
    uint64_t t;
    bool posted;
  };
  static thread_local std::vector<Ticket> st, rt;
  st.assign(ns, Ticket{0, 0, false});
  rt.assign(nr, Ticket{0, 0, false});
  // staging for unregistered slices: one pinned buffer for the whole pass, sized for what its Sends stage
  // (stage_need), at most kMaxBounce unless one one-call op stages more (it is staged whole or not at all).  A Send
  // that does not fit in what is left waits for the pass's posted ops -- the only readers of the buffer -- and
  // starts it again from the front; an until-blocked op larger than the buffer stages a prefix.
  const uint32_t fl = (uint32_t)(flags & (B200_BATCH_UNTIL_BLOCKED));
  static thread_local std::vector<uint64_t> sneed;
  sneed.assign(ns, 0);
  uint64_t need = 0, most = 0;
  for (size_t i = 0; i < ns; i++) {
    if (!sops[i].pair || !sops[i].nslices) continue;
    sneed[i] = stage_need(sops[i].pair, sops[i].slices, sops[i].nslices, sops[i].byte_idx, !fl);
    need += sneed[i];
    if (sneed[i] > most) most = sneed[i];
  }
  const uint64_t kMaxBounce = 1ull << 30;
  uint64_t size = need < kMaxBounce ? need : kMaxBounce;
  if (!fl && size < most) size = most;
  TlsBounce& tb = tls_bounce();
  if (size && !ensure_bounce(&tb.tx, &tb.tx_cap, size)) return -1;
  SendStage stage{tb.tx, tb.tx_cap, 0, false};
  int rc = 0;
  static thread_local std::vector<uint8_t*> rstage;  // device staging of a Recv (recv_stage), by op
  static thread_local std::vector<int> rcls;
  rstage.assign(nr, nullptr);
  rcls.assign(nr, -1);
  cudaStream_t copies = nullptr;  // the stream of the pass's D2H copies out of rstage
  // answers are collected at the end -- or earlier, when a queue has no free entry: a thread never blocks on
  // a queue while it sits on answers of its own that somebody else's post may be waiting for
  auto harvest = [&]() {
    for (size_t i = 0; i < ns; i++) {
      if (!st[i].posted) continue;
      st[i].posted = false;
      uint64_t bytes = 0;
      if (!svc_wait(r, st[i].q, st[i].t, &bytes, nullptr)) rc = -1;
      if (accepted) accepted[i] = bytes;
    }
    for (size_t i = 0; i < nr; i++) {
      if (!rt[i].posted) continue;
      rt[i].posted = false;
      uint64_t bytes = 0;
      if (!svc_wait(r, rt[i].q, rt[i].t, &bytes, nullptr)) rc = -1;
      rops[i].pair->svc_delivered += bytes;
      if (delivered) delivered[i] = bytes;
      if (rstage[i] && bytes) {
        if (!copies) copies = copy_stream();
        if (!CU_OK(cudaMemcpyAsync(rops[i].dst, rstage[i], bytes, cudaMemcpyDeviceToHost, copies))) rc = -1;
      }
    }
  };
  for (size_t i = 0; i < ns; i++) {
    b200_pair* p = sops[i].pair;
    if (accepted) accepted[i] = 0;
    if (!p || p->status != B200_CONNECTED || sops[i].nslices == 0) continue;
    if (((volatile PairMirror*)p->mirror)->peer_exit == 1) continue;
    if (p->peer_local && p->peer_local->retire_owed.load(std::memory_order_acquire)) {
      harvest();
      drain_retire(p->peer_local);
    }
    if (send_is_a_no_op(p)) continue;
    if (stage.off && sneed[i] > stage.cap - stage.off) {
      harvest();
      stage.off = 0;
    }
    const int q = owner_of(r, p);
    auto fill = [&](SvcCmd* c, SliceDev* area) {
      fill_send_cmd(p, c, area, sops[i].slices, sops[i].nslices, sops[i].byte_idx, fl, stage);
    };
    while (!svc_try_post(r, q, fill, &st[i].t)) harvest();
    st[i].q = q;
    st[i].posted = true;
  }
  for (size_t i = 0; i < nr; i++) {
    b200_pair* p = rops[i].pair;
    if (delivered) delivered[i] = 0;
    if (!p || p->status != B200_CONNECTED || rops[i].cap == 0) continue;
    if (p->retire_owed.load(std::memory_order_acquire)) {
      harvest();
      drain_retire(p);
    }
    if (!p->remote && ((volatile PairMirror*)p->mirror)->has_message == 0) continue;
    const int kind = mem_kind3(rops[i].dst);
    if (kind == 0) {
      set_err("b200_pairs_submit: destinations must be GPU-addressable (b200_mem_alloc_host / register_host / device)");
      rc = -1;
      continue;
    }
    rstage[i] = recv_stage(kind, rops[i].cap, &rcls[i]);
    const int q = owner_of(r, p);
    auto fill = [&](SvcCmd* c, SliceDev*) {
      fill_cmd(c, p, kSvcRecv, fl, rstage[i] ? rstage[i] : rops[i].dst, rops[i].cap);
    };
    while (!svc_try_post(r, q, fill, &rt[i].t)) harvest();
    rt[i].q = q;
    rt[i].posted = true;
  }
  harvest();
  if (copies && !CU_OK(cudaStreamSynchronize(copies))) rc = -1;
  for (size_t i = 0; i < nr; i++)
    if (rstage[i]) stage_put(rstage[i], rcls[i]);
  return rc;
}

// ------------------------------------------------------------------ post / poll (completion-queue form)

struct b200_async {
  int kind = 0;          // 0 send, 1 recv
  b200_pair* p = nullptr;
  int q = 0;
  uint64_t t = 0;
  int state = 0;         // 0 posted, 1 copying down, 2 done
  uint64_t bytes = 0;
  uint8_t* stage = nullptr;
  int stage_cls = -1;
  uint8_t* hstage = nullptr;  // send: pinned staging of unregistered slices, owned until the op has finished
  int hstage_cls = -1;
  void* dst = nullptr;
  cudaEvent_t ev = nullptr;
  bool counted = false;  // posted: counts in p->host_ops until it is finished
};

namespace {
b200_async* async_get() {
  AsyncPool& a = AP();
  {
    std::lock_guard<std::mutex> lk(a.mu);
    if (!a.free_ops.empty()) {
      b200_async* o = a.free_ops.back();
      a.free_ops.pop_back();
      return o;
    }
  }
  b200_async* o = new b200_async();
  cudaEventCreateWithFlags(&o->ev, cudaEventDisableTiming);
  return o;
}
void async_put(b200_async* o) {
  if (o->counted) o->p->host_ops.fetch_sub(1);
  o->counted = false;
  AsyncPool& a = AP();
  std::lock_guard<std::mutex> lk(a.mu);
  if (o->stage) a.free_stage[o->stage_cls].push_back(o->stage);
  if (o->hstage) a.free_hstage[o->hstage_cls].push_back(o->hstage);
  o->stage = o->hstage = nullptr;
  o->stage_cls = o->hstage_cls = -1;
  o->state = 0;
  a.free_ops.push_back(o);
}
}  // namespace

extern "C" b200_async* b200_pair_post_send(b200_pair* p, const b200_slice* slices, size_t n, size_t byte_idx, int flags,
                                           int* again) {
  if (again) *again = 0;
  Runtime& r = R();
  if (!p || !r.svc_running.load()) {
    set_err("b200_pair_post_send: the service is not running");
    return nullptr;
  }
  if (flags & kClusterField) {
    set_err("b200_pair_post_send: B200_BATCH_CLUSTER applies to batch launches only; the service's owners and pool run "
            "one CTA per op");
    return nullptr;
  }
  b200_async* o = async_get();
  o->p = p;
  o->counted = true;  // a host op of p until it is polled to the end
  p->host_ops.fetch_add(1);
  if (p->device_owned.load()) {
    set_err("b200_pair_post_send: the pair is device-owned (b200_pair_device_claim)");
    async_put(o);
    return nullptr;
  }
  o->kind = 0;
  o->p = p;
  o->bytes = 0;
  o->state = 2;  // finished with 0 bytes unless something is posted
  if (p->status != B200_CONNECTED || n == 0 || ((volatile PairMirror*)p->mirror)->peer_exit == 1) return o;
  if (p->peer_local) drain_retire(p->peer_local);
  if (send_is_a_no_op(p)) return o;
  const int q = owner_of(r, p);
  uint64_t t = 0;
  const uint32_t fl = (uint32_t)(flags & B200_BATCH_UNTIL_BLOCKED);
  {  // unregistered slices are staged in pinned memory that belongs to the op: a block of the power-of-two class of
     // what it stages (stage_need).  A one-call op's block holds all of it; an until-blocked op's is at most 2^28
     // bytes, and when it needs more it stages a prefix.
    const uint64_t need = stage_need(p, slices, n, byte_idx, !fl);
    if (need) {
      int c = 12;
      while ((1ull << c) < need && (c < 28 || !fl)) c++;
      AsyncPool& a = AP();
      {
        std::lock_guard<std::mutex> lk(a.mu);
        if (!a.free_hstage[c].empty()) {
          o->hstage = a.free_hstage[c].back();
          a.free_hstage[c].pop_back();
        }
      }
      if (!o->hstage && cudaHostAlloc((void**)&o->hstage, 1ull << c, cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        o->hstage = nullptr;
      }
      o->hstage_cls = c;
      if (!o->hstage) {
        set_err("b200_pair_post_send: pinned staging allocation failed");
        async_put(o);
        return nullptr;
      }
    }
  }
  SendStage st{o->hstage, o->hstage ? 1ull << o->hstage_cls : 0, 0, false};
  auto fill = [&](SvcCmd* c, SliceDev* area) {
    fill_send_cmd(p, c, area, slices, n, byte_idx, fl, st);
  };
  if (!svc_try_post(r, q, fill, &t)) {
    async_put(o);
    if (again) *again = 1;
    return nullptr;
  }
  o->q = q;
  o->t = t;
  o->state = 0;
  return o;
}

extern "C" b200_async* b200_pair_post_recv(b200_pair* p, void* dst, uint64_t cap, int flags, int* again) {
  if (again) *again = 0;
  Runtime& r = R();
  if (!p || !r.svc_running.load()) {
    set_err("b200_pair_post_recv: the service is not running");
    return nullptr;
  }
  if (flags & kClusterField) {
    set_err("b200_pair_post_recv: B200_BATCH_CLUSTER applies to batch launches only; the service's owners and pool run "
            "one CTA per op");
    return nullptr;
  }
  b200_async* o = async_get();
  o->p = p;
  o->counted = true;  // a host op of p until it is polled to the end
  p->host_ops.fetch_add(1);
  if (p->device_owned.load()) {
    set_err("b200_pair_post_recv: the pair is device-owned (b200_pair_device_claim)");
    async_put(o);
    return nullptr;
  }
  o->kind = 1;
  o->p = p;
  o->bytes = 0;
  o->dst = dst;
  o->state = 2;
  if (p->status != B200_CONNECTED || cap == 0) return o;
  drain_retire(p);
  if (!p->remote && !peer_device_owned(p) && ((volatile PairMirror*)p->mirror)->has_message == 0) return o;
  const int kind = mem_kind3(dst);
  if (kind == 0) {
    set_err("b200_pair_post_recv: the destination must be GPU-addressable (b200_mem_alloc_host / register_host / device)");
    async_put(o);
    return nullptr;
  }
  o->stage = recv_stage(kind, cap, &o->stage_cls);
  const int q = owner_of(r, p);
  uint64_t t = 0;
  auto fill = [&](SvcCmd* c, SliceDev*) {
    fill_cmd(c, p, kSvcRecv, (uint32_t)(flags & B200_BATCH_UNTIL_BLOCKED), o->stage ? o->stage : dst, cap);
  };
  if (!svc_try_post(r, q, fill, &t)) {
    async_put(o);
    if (again) *again = 1;
    return nullptr;
  }
  o->q = q;
  o->t = t;
  o->state = 0;
  return o;
}

extern "C" int b200_async_poll(b200_async* o, uint64_t* bytes) {
  if (!o) return -1;
  Runtime& r = R();
  if (o->state == 0) {
    const size_t e = (size_t)o->q * kOwnQ + o->t % kOwnQ;
    volatile SvcDone* d = &r.svc_done[e];
    if (d->seq != (uint32_t)(o->t + 1)) return 0;
    std::atomic_thread_fence(std::memory_order_acquire);
    o->bytes = d->bytes;
    r.svc_consumed[e].store((uint32_t)(o->t + 1), std::memory_order_release);
    r.svc_ops++;
    if (o->kind == 1) {
      o->p->svc_delivered += o->bytes;
      if (o->stage && o->bytes) {  // the copy engine takes the delivered bytes down
        cudaStream_t cs = copy_stream();
        if (cudaMemcpyAsync(o->dst, o->stage, o->bytes, cudaMemcpyDeviceToHost, cs) != cudaSuccess ||
            cudaEventRecord(o->ev, cs) != cudaSuccess) {
          cudaGetLastError();
          async_put(o);
          return -1;
        }
        o->state = 1;
        return 0;
      }
    }
    o->state = 2;
  }
  if (o->state == 1) {
    const cudaError_t e = cudaEventQuery(o->ev);
    if (e == cudaErrorNotReady) return 0;
    if (e != cudaSuccess) {
      cudaGetLastError();
      async_put(o);
      return -1;
    }
    o->state = 2;
  }
  if (bytes) *bytes = o->bytes;
  async_put(o);
  return 1;
}

// ================================================================ calibration

extern "C" int b200_probe_copy(void* dst, const void* src, uint64_t bytes_per_cta, uint64_t stride, int nctas,
                               int threads, uint32_t mis, uint32_t item_bytes, uint32_t dynamic, void* stream) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  cudaStream_t s = stream ? (cudaStream_t)stream : r.stream;
  launch_probe_copy((uint8_t*)dst, (const uint8_t*)src, bytes_per_cta, stride, nctas, threads, mis, item_bytes,
                    dynamic, s);
  r.launches++;
  return CU_OK(cudaGetLastError()) ? 0 : -1;
}

// ==================================================================== poller

extern "C" int b200_poller_scan(b200_pair* const* pairs, size_t n, uint32_t* events) {
  if (!ensure_init()) return -1;
  Runtime& r = R();
  if (n > (size_t)kMaxPairs) return -1;
  std::lock_guard<std::mutex> lk(r.scan_mu);
  cudaSetDevice(r.dev);
  for (size_t i = 0; i < n; i++) r.h_scan_slots[i] = pairs[i]->slot;
  r.h_scan_count[0] = 0;
  launch_poll_scan(r.d_pairs, r.h_scan_slots, r.h_scan_events, r.h_scan_count, r.h_scan_ready, (int)n,
                   r.poll_stream);
  r.launches++;
  if (!CU_OK(cudaGetLastError()) || !CU_OK(cudaStreamSynchronize(r.poll_stream))) return -1;
  if (events)
    for (size_t i = 0; i < n; i++) events[i] = r.h_scan_events[i];
  return (int)r.h_scan_count[0];
}

// Service mode: the device poller reports readiness CHANGES through the ready ring; the host keeps
// the level per pair and kicks the eventfd of every registered pair that has events pending and
// whose eventfd is not signalled already (poller.cc:73-101) -- no kernel launch on this path.
static void poller_service_pass(Runtime& r, const std::vector<b200_pair*>& snap) {
  std::unique_lock<std::mutex> lk(r.scan_mu, std::try_to_lock);
  if (!lk.owns_lock()) return;
  if (r.svc_level.size() != (size_t)kMaxPairs) r.svc_level.assign(kMaxPairs, 0);
  uint64_t n = 0;
  while (r.svc_ready) {
    const uint64_t raw = *reinterpret_cast<volatile uint64_t*>(&r.svc_ready[r.svc_ready_head % kReadyRing]);
    ReadyEntry e;
    memcpy(&e, &raw, 8);
    if (e.stamp == r.svc_ready_head + 1) {
      r.svc_level[e.slot] = e.events;
      r.svc_ready_head++;
      n++;
    } else if ((int32_t)(e.stamp - (r.svc_ready_head + 1)) > 0) {
      // the device lapped the ring: rebuild the levels from the mirrors and resume at this entry
      r.svc_ready_overflows++;
      for (b200_pair* p : snap) {
        volatile PairMirror* m = p->mirror;
        r.svc_level[p->slot] = (uint16_t)((m->has_message || m->peer_exit ? kEvReadable : 0) |
                                           (m->partial_write ? kEvWritable : 0));
      }
      r.svc_ready_head = e.stamp - 1;
    } else {
      break;
    }
  }
  if (n) r.svc_ready_seen += n;
  for (b200_pair* p : snap) {
    if (!r.svc_level[p->slot]) continue;
    if (p->retire_owed.load(std::memory_order_acquire)) {
      // the frame the device still reports was already taken from the eager slot: post its Retire now
      // (nobody sent on the pair since) instead of waking the engine for it
      drain_retire(p);
      continue;
    }
    struct pollfd pfd = {p->wakeup_fd, POLLIN, 0};
    if (poll(&pfd, 1, 0) <= 0) kick(p);
  }
}

// Ready sets with a wakeup fd (DESIGN.md §13 "Parking"): a doorbell that moved since the last pass kicks the set's
// eventfd unless it is signalled already.  Caller holds r.pmu, under which b200_ready_set_destroy unregisters a set.
static void poller_bell_pass_locked(Runtime& r) {
  for (b200_ready_set* s : r.bell_sets) {
    const uint64_t v = *(volatile uint64_t*)&s->bell[0];
    if (v == s->bell_seen) continue;
    s->bell_seen = v;
    struct pollfd pfd = {s->wakeup_fd, POLLIN, 0};
    if (poll(&pfd, 1, 0) <= 0) (void)eventfd_write(s->wakeup_fd, 1);
  }
}

static void poller_main(int /*id*/) {
  Runtime& r = R();
  std::vector<b200_pair*> snap;
  std::vector<uint32_t> ev;
  uint32_t idle = 0;
  while (r.poll_running.load()) {
    {
      std::unique_lock<std::mutex> lk(r.pmu);
      if (r.pollables.empty() && r.bell_sets.empty()) {  // poller.cc:58-63: sleep while there is nothing to poll
        r.pcv.wait_for(lk, std::chrono::milliseconds(r.cfg.poller_sleep_ms), [&] {
          return !r.pollables.empty() || !r.bell_sets.empty() || !r.poll_running.load();
        });
        continue;
      }
      poller_bell_pass_locked(r);
      snap = r.pollables;
    }
    if (snap.empty()) {  // only ready sets to watch: no scan to launch
      if ((++idle & 63) == 0) std::this_thread::yield();
      continue;
    }
    if (r.svc_running.load()) {
      poller_service_pass(r, snap);
      if ((++idle & 63) == 0) std::this_thread::yield();
      continue;
    }
    ev.assign(snap.size(), 0);
    int nready = b200_poller_scan(snap.data(), snap.size(), ev.data());
    if (nready <= 0) continue;
    for (size_t i = 0; i < snap.size(); i++) {
      if (!ev[i]) continue;
      struct pollfd pfd = {snap[i]->wakeup_fd, POLLIN, 0};
      if (poll(&pfd, 1, 0) <= 0) kick(snap[i]);  // skip a pair whose eventfd is already signalled (poller.cc:73-75)
    }
  }
}

extern "C" void b200_poller_add(b200_pair* p) {
  if (!p || !ensure_init()) return;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.pmu);
  if ((int)r.pollables.size() >= B200_POLLER_CAPACITY) return;  // poller.cc:13 asserts
  if (p->in_poller) return;  // (O(1): 4096 connections register one after the other)
  r.pollables.push_back(p);
  p->in_poller = true;
  poller_start_locked(r);
  r.pcv.notify_all();
}

// caller holds r.pmu
static void poller_start_locked(Runtime& r) {
  if (r.poll_running.load()) return;
  r.poll_running = true;
  for (int i = 0; i < r.cfg.poller_threads; i++) r.poll_threads.emplace_back(poller_main, i);
}

extern "C" void b200_poller_remove(b200_pair* p) {
  if (!p) return;
  Runtime& r = R();
  std::lock_guard<std::mutex> lk(r.pmu);
  for (size_t i = 0; i < r.pollables.size(); i++) {
    if (r.pollables[i] == p) {
      r.pollables.erase(r.pollables.begin() + i);
      break;
    }
  }
  p->in_poller = false;
}

extern "C" void b200_poller_shutdown(void) {
  Runtime& r = R();
  if (!r.poll_running.exchange(false)) return;
  {
    std::lock_guard<std::mutex> lk(r.pmu);
    r.pcv.notify_all();
  }
  for (auto& t : r.poll_threads) t.join();
  r.poll_threads.clear();
}
